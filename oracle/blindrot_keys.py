"""CPU restatement of blindrot.GenEvaluationKeyNew (core/rgsw/blindrot/keys.go:52-108), with the samples as arguments: RGSW(X^{s_i}) per
LWE-key coefficient (rgsw.Encryptor.Encrypt of the NTT-domain monomial NewMonomialXi(s_i)) and the Galois keys of GaloisElement(1..window)
and NthRoot - GaloisGen (KeyGenerator.GenGaloisKeysNew).

TEST INFRASTRUCTURE ONLY. tests/test_oracle_blindrot_keys.py pins it by decryption through oracle/blindrot_evaluate.py."""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence

import numpy as np

from . import rgsw_keygen as E
from . import oracle as O

U64 = np.uint64


def monomial(ringQ: O.Ring, k: int) -> np.ndarray:
    """ring.NewMonomialXi (ring/ring.go:374-396) over every limb of ringQ."""
    N = ringQ.N()
    p = ringQ.NewPoly()
    k &= 2 * N - 1
    if k >= N:
        k -= 2 * N
    for r, q in enumerate(ringQ.ModuliChain()[: ringQ.Level() + 1]):
        if k < 0:
            p[r, N + k] = q - 1
        else:
            p[r, k] = 1
    return p


def galois_elements(params: O.Parameters, window: int) -> List[int]:
    return [params.GaloisElement(k) for k in range(1, window + 1)] + [params.ringQ.NthRoot() - 5]


def GenEvaluationKeyNew(params: O.Parameters, sk, s_lwe: Sequence[int], levelQ: int, levelP: int, pw2: int, window: int,
                        samples: Callable[[int], tuple]):
    """sk: (nQ + nP, N) blind-rotation secret key, NTT + Montgomery; s_lwe: the centred LWE-key coefficients (keys.go:57-65 computes
    them). samples(m) -> (a, e) of the m-th gadget ciphertext, a[i][j] (levelQ+1 + levelP+1, N) uniform rows and e[i][j] signed, where
    m = 2 i + v is Value[v] of RGSW i and m = 2 len(s_lwe) + t the t-th Galois key. Returns (brk, {galEl: GadgetCiphertext}), brk[i] =
    [Value0, Value1]."""
    pts: Dict[int, np.ndarray] = {}
    brk = []
    for i, si in enumerate(s_lwe):
        si = int(si)
        if si not in pts:
            pt = monomial(params.ringQ, si)
            params.ringQ.NTT(pt, pt)          # IsNTT = true, IsMontgomery = false: Encrypt takes it to Montgomery form
            pts[si] = pt
        a0, e0 = samples(2 * i)
        a1, e1 = samples(2 * i + 1)
        brk.append(E.rgsw_encrypt(params, sk, pts[si], [a0, a1], [e0, e1], levelQ, levelP, pw2, is_ntt=True, is_montgomery=False))
    gks = {}
    for t, g in enumerate(galois_elements(params, window)):
        a, e = samples(2 * len(s_lwe) + t)
        gks[g] = E.gen_galois_key(params, g, sk, a, e, pw2, levelQ, levelP)
    return brk, gks

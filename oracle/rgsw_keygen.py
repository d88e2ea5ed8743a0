"""CPU restatement of the gadget encryptions behind RGSW encryption and key generation at any levels, with the samplers' outputs as
explicit arguments (as in oracle/encryptor.py, whose encryptZeroSkFromC1QP it builds on):

    AddPolyTimesGadgetVectorToGadgetCiphertext   core/rlwe/gadgetciphertext.go:171-241   (one or two ciphertexts, any levelP)
    KeyGenerator.genEvaluationKey                core/rlwe/keygenerator.go:287-330       (at any levels)
    KeyGenerator.GenGaloisKey                    :139-177
    rgsw.Encryptor.Encrypt / EncryptZero         core/rgsw/encryptor.go:25-121

TEST INFRASTRUCTURE ONLY. tests/test_rgsw_keygen_cpu.py pins it by decryption, as core/rgsw/rgsw_test.go pins the reference."""
from __future__ import annotations

import numpy as np

from . import encryptor as E
from . import oracle as O

U64 = np.uint64


def add_poly_times_gadget_vector(params: O.Parameters, pt, cts):
    """AddPolyTimesGadgetVectorToGadgetCiphertext (core/rlwe/gadgetciphertext.go:171-241): adds pt * P_levelP * w^j to component u of
    cts[u] on the limbs of digit i (P_levelP = 1 when levelP = -1). cts: one GadgetCiphertext or a list of at most two. pt:
    (>= levelQ+1, N) NTT + Montgomery rows."""
    cts = cts if isinstance(cts, (list, tuple)) else [cts]
    assert len(cts) <= 2
    levelQ, levelP = cts[0].LevelQ(), cts[0].LevelP()
    ringQ = params.ringQ.AtLevel(levelQ)
    buff = np.empty((levelQ + 1, params.N()), dtype=U64)
    if levelP != -1:
        ringQ.MulScalarBigint(pt[: levelQ + 1], params.ringP.AtLevel(levelP).ModulusAtLevel[levelP], buff)
    else:
        levelP = 0
        buff[...] = pt[: levelQ + 1]
    sizes = cts[0].BaseTwoDecompositionVectorSize()
    for j in range(max(sizes)):
        for i in range(cts[0].data.shape[0]):
            if j < sizes[i]:
                for k in range(levelP + 1):
                    index = i * (levelP + 1) + k
                    if index >= levelQ + 1:
                        break
                    for u, ct in enumerate(cts):
                        ringQ.SubRings[index].vecop("Add", ct.data[i, j, u, index], buff[index], ct.data[i, j, u, index])
        ringQ.MulScalar(buff, 1 << cts[0].BaseTwoDecomposition, buff)


def gadget_layout(params: O.Parameters, levelQ, levelP, pw2):
    n = params.BaseRNSDecompositionVectorSize(levelQ, levelP)
    return n, params.BaseTwoDecompositionVectorSize(levelQ, levelP, pw2)[:n]


def encrypt_zero_gadget(params: O.Parameters, sk, a, e, levelQ, levelP, pw2):
    """A gadget encryption of zero under sk at the given levels: entry (i, j) = (e_ij - a_ij sk, a_ij), NTT + Montgomery (the loop of
    genEvaluationKey, keygenerator.go:313-322, and of rgsw.Encryptor.EncryptZero, encryptor.go:88-118). a[i][j]: (levelQ+1 + levelP+1, N)."""
    n, sizes = gadget_layout(params, levelQ, levelP, pw2)
    rows = levelQ + 1 + levelP + 1
    data = np.zeros((n, max(sizes), 2, rows, params.N()), dtype=U64)
    enc = E.Encryptor(params)
    for i in range(n):
        for j in range(sizes[i]):
            c1 = np.array(a[i][j], dtype=U64, copy=True)
            data[i, j, 0] = enc.encryptZeroSkFromC1QP(levelQ, levelP, sk, c1, e[i][j], True, True)
            data[i, j, 1] = c1
    return O.GadgetCiphertext(data, levelQ + 1, levelP + 1, pw2, sizes)


def gen_evaluation_key(params: O.Parameters, skIn, skOut, a, e, pw2=0, levelQ=None, levelP=None):
    """KeyGenerator.genEvaluationKey (core/rlwe/keygenerator.go:287-330) with the samples given: a[i][j]: (levelQ+1 + levelP+1, N)
    uniform rows (the key's component 1), e[i][j]: signed small polynomial. skIn: (>= levelQ+1, N) rows, skOut: (nQ + nP, N) rows at
    the maximum levels, both NTT + Montgomery. Levels default to the maximum."""
    levelQ = params.MaxLevelQ() if levelQ is None else levelQ
    levelP = params.MaxLevelP() if levelP is None else levelP
    evk = encrypt_zero_gadget(params, skOut, a, e, levelQ, levelP, pw2)
    add_poly_times_gadget_vector(params, skIn, evk)
    return evk


def gen_galois_key(params: O.Parameters, galEl, sk, a, e, pw2=0, levelQ=None, levelP=None):
    """KeyGenerator.GenGaloisKey (keygenerator.go:139-177): sk under AutomorphismNTT(sk, galEl^-1 mod 2N) on Q and P. sk: (nQ + nP, N)."""
    nQ = len(params.qi)
    inv = pow(int(galEl), -1, params.ringQ.NthRoot())
    skOut = np.empty_like(sk)
    params.ringQ.AutomorphismNTT(sk[:nQ], inv, skOut[:nQ])
    if params.ringP is not None:
        params.ringP.AutomorphismNTT(sk[nQ:], inv, skOut[nQ:])
    return gen_evaluation_key(params, sk[:nQ], skOut, a, e, pw2, levelQ, levelP)


def rgsw_encrypt(params: O.Parameters, sk, pt, a, e, levelQ, levelP, pw2=0, is_ntt=True, is_montgomery=False):
    """rgsw.Encryptor.Encrypt (core/rgsw/encryptor.go:25-70), or EncryptZero (:74-121) when pt is None, with the samples given: a[v][i][j]
    and e[v][i][j] for Value[v]. pt: (>= levelQ+1, N) rows, in the NTT domain / Montgomery form as flagged. Returns [Value0, Value1]."""
    ct = [encrypt_zero_gadget(params, sk, a[v], e[v], levelQ, levelP, pw2) for v in range(2)]
    if pt is not None:
        ringQ = params.ringQ.AtLevel(levelQ)
        buf = np.array(pt[: levelQ + 1], dtype=U64, copy=True)
        if not is_ntt:
            ringQ.NTT(buf, buf)
            if not is_montgomery:
                ringQ.MForm(buf, buf)
        elif not is_montgomery:
            ringQ.MForm(buf, buf)
        add_poly_times_gadget_vector(params, buf, ct)
    return ct

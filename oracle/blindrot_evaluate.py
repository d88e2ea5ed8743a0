"""CPU restatement of blindrot.Evaluator.Evaluate and InitTestPolynomial -- `core/rgsw/blindrot/`:

    Evaluator.Evaluate              evaluator.go:49-132   (on top of oracle/blindrot.py's BlindRotateCore)
    modSwitchRLWETo2NLvl            evaluator.go:254-283  (level 0: the coefficient itself is PolyToBigint's value)
    mulBySmallMonomialMod2N         utils.go:11-21
    InitTestPolynomial              blindrot.go:12-44     (scaleUp, normalizeInv: utils.go:23-57)

TEST INFRASTRUCTURE ONLY. tests/test_oracle_blindrot_evaluate.py pins it by decryption, as blindrot_test.go does."""
from __future__ import annotations

from typing import Callable, Dict, List

import numpy as np

from . import blindrot as BR
from . import oracle as O

U64 = np.uint64


def div_round(a: int, b: int) -> int:
    """bignum.DivRound (utils/bignum/int.go:52-64): Quo, then away from zero when 2|Rem| >= |b|."""
    q = abs(a) // abs(b) * (1 if (a >= 0) == (b > 0) else -1)
    r = a - q * b
    if 2 * abs(r) >= abs(b):
        q += 1 if (a >= 0) == (b > 0) else -1
    return q


def mod_switch_to_2n(coeffs, q_lwe: int, twoN: int, make_odd: bool) -> List[int]:
    """modSwitchRLWETo2NLvl at level 0: round(x * 2N / q) & (2N - 1), made odd by ^1 when even and non-zero."""
    out = []
    for x in coeffs:
        r = div_round((int(x) % q_lwe) * twoN, q_lwe) & (twoN - 1)
        if make_odd and r & 1 == 0 and r != 0:
            r ^= 1
        out.append(r)
    return out


def mul_by_small_monomial_mod2n(mask: int, pol: List[int], n: int) -> List[int]:
    if n != 0:
        N = len(pol)
        pol = pol[N - n:] + pol[: N - n]
        for j in range(n):
            pol[j] = -pol[j] & mask
    return pol


def scale_up(value: float, scale: float, Q: int) -> int:
    """utils.go:27-57: big.NewFloat keeps 53 bits, so the + 0.5 rounds like a float64 addition; Int() truncates toward zero."""
    neg = value < 0
    x = (-scale * value) if neg else (scale * value)
    x = int(x + 0.5)
    res = x % Q
    return Q - res if neg else res


def InitTestPolynomial(g: Callable[[float], float], scale: float, ringQ: O.Ring, a: float, b: float):
    N = ringQ.N()
    F = ringQ.NewPoly()
    interval = 2.0 / float(N)
    norm_inv = lambda x: (x * (b - a) + b + a) / 2.0
    for j, qi in enumerate(ringQ.ModuliChain()[: ringQ.Level() + 1]):
        for i in range((N >> 1) + 1):
            F[j, i] = scale_up(g(norm_inv(-interval * float(i))), scale, qi)
        for i in range((N >> 1) + 1, N):
            F[j, i] = scale_up(-g(norm_inv(interval * float(N - i))), scale, qi)
    ringQ.NTT(F, F)
    return F


class Evaluator:
    def __init__(self, paramsBR: O.Parameters, paramsLWE: O.Parameters, window_size: int = BR.WINDOW_SIZE):
        self.paramsBR, self.paramsLWE = paramsBR, paramsLWE
        self.core = BR.Evaluator(paramsBR, window_size)

    def Evaluate(self, ct, testPolyWithSlotIndex: Dict[int, np.ndarray], brk: List[list], galois_keys, is_ntt=True, ntt_flag=True):
        """ct: [c0, c1] level-0 rows of the LWE ring; brk[j] = [Value0, Value1] of RGSW(X^{s_j}); returns {slot: [c0, c1]}."""
        level = brk[0][0].LevelQ()
        ringQBR = self.paramsBR.ringQ.AtLevel(level)
        ringQLWE = self.paramsLWE.ringQ.AtLevel(0)
        NBR, NLWE = ringQBR.N(), ringQLWE.N()
        qLWE = self.paramsLWE.qi[0]
        c = [np.array(ct[0][:1], dtype=U64), np.array(ct[1][:1], dtype=U64)]
        if is_ntt:
            ringQLWE.INTT(c[0], c[0]); ringQLWE.INTT(c[1], c[1])
        twoN = NBR << 1
        mask = twoN - 1
        tmp1 = mod_switch_to_2n(c[1][0], qLWE, twoN, True)
        aRLWEMod2N = [tmp1[0]] + [-tmp1[NLWE - j] & mask for j in range(1, NLWE)]
        bRLWEMod2N = mod_switch_to_2n(c[0][0], qLWE, twoN, False)
        res = {}
        prev = 0
        for index in range(NLWE):
            if index not in testPolyWithSlotIndex:
                continue
            aRLWEMod2N = mul_by_small_monomial_mod2n(mask, aRLWEMod2N, index - prev)
            prev = index
            b = bRLWEMod2N[index]
            xb = ringQBR.NewPoly()                      # NewMonomialXi(b), ring/ring.go:374-396
            i = b & (twoN - 1)
            i = i - twoN if i >= NBR else i
            for k, q in enumerate(ringQBR.ModuliChain()[: level + 1]):
                if i < 0:
                    xb[k, NBR + i] = q - 1
                else:
                    xb[k, i] = 1
            ringQBR.NTT(xb, xb)
            ringQBR.MForm(xb, xb)
            acc1 = ringQBR.NewPoly()
            ringQBR.MulCoeffsMontgomery(np.asarray(testPolyWithSlotIndex[index], dtype=U64)[: level + 1], xb, acc1)
            acc0 = ringQBR.NewPoly()
            ringQBR.AutomorphismNTT(acc1, ringQBR.NthRoot() - 5, acc0)
            acc = [acc0, np.zeros_like(acc0)]
            self.core.BlindRotateCore(np.array(aRLWEMod2N, dtype=U64), acc, brk, galois_keys, level)
            if not ntt_flag:
                ringQBR.INTT(acc[0], acc[0]); ringQBR.INTT(acc[1], acc[1])
            res[index] = acc
        return res

"""CPU restatement of schemes/bgv's ciphertext x ciphertext multiplication (TEST INFRASTRUCTURE ONLY), composed from the
oracle's ring / BasisExtender / rlwe.Evaluator pieces (oracle/oracle.py) the way schemes/bgv/evaluator.go composes the Go ones:
QMul generation and levelQMul (params.go:98-109, evaluator.go:38-70), tensorStandard (:592-667), tensorScaleInvariant with
modUpAndNTT / tensorLowDeg / quantize (:898-1070) and Rescale (:1363-1393). Ciphertexts are lists [c0, c1] of (limbs, N) uint64
arrays in the NTT domain; passing the same list twice is the squaring case (op0.El() == op1.El())."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np

from oracle import oracle as O

U64 = np.uint64


def qmul_moduli(logN: int, Q: Sequence[int]) -> List[int]:
    """ringQMul's moduli: NextDownstreamPrimes(61, NthRoot) x ceil((BitLen(Q) + logN) / 61) (params.go:98-109)."""
    prod = 1
    for q in Q:
        prod *= int(q)
    n = int(math.ceil(float(prod.bit_length() + logN) / 61.0))
    g = O.NTTFriendlyPrimesGenerator(61, 2 << logN)
    return [g.NextDownstreamPrime() for _ in range(n)]


def level_qmul(logN: int, Q: Sequence[int]) -> List[int]:
    """levelQMul[i] = ceil((BitLen(Q_i) + logN) / 61) - 1 (evaluator.go:43-48)."""
    out, prod = [], 1
    for q in Q:
        prod *= int(q)
        out.append(int(math.ceil(float(prod.bit_length() + logN) / 61.0)) - 1)
    return out


class BGVEvaluator(O.Evaluator):
    """bgv.Evaluator (evaluator.go:18-29) restricted to MulRelin[ScaleInvariant] of degree-1 ciphertexts and Rescale."""

    def __init__(self, params: O.Parameters, t: int, qmul: Sequence[int], rlk: Optional[O.GadgetCiphertext] = None,
                 scale_invariant: bool = False):
        super().__init__(params)
        self.t = int(t)
        self.rlk = rlk
        self.ScaleInvariant = scale_invariant
        self.ringQMul = O.Ring(params.N(), [int(x) for x in qmul])
        self.levelQMul = level_qmul(params.logN, params.qi)
        self.basisExtenderQ1toQ2 = O.BasisExtender(params.ringQ, self.ringQMul)
        # tMontgomery = MForm(t * 2^64 mod q_i) (evaluator.go:60-62)
        self.tMontgomery = [O.mform((self.t << 64) % q, q) for q in params.qi]

    def _new(self, ring, level):
        return np.zeros((level + 1, ring.N()), dtype=U64)

    def MulRelinNew(self, op0, op1):
        """MulRelinNew (:576-590) -> MulRelin (:529-556) / MulRelinScaleInvariant (:806-864)."""
        level = min(op0[0].shape[0], op1[0].shape[0]) - 1
        if self.ScaleInvariant:
            return self.tensorScaleInvariant(level, op0, op1)
        return self.tensorStandard(level, op0, op1)

    def _relinearize(self, level, c0, c1, c2):
        ringQ = self.params.ringQ.AtLevel(level)
        tmp = [self._new(ringQ, level), self._new(ringQ, level)]
        self.GadgetProduct(level, c2, self.rlk, tmp)
        ringQ.Add(c0, tmp[0], c0)
        ringQ.Add(c1, tmp[1], c1)
        return [c0, c1]

    def tensorStandard(self, level, op0, op1):
        """:592-667 (degree 1 x degree 1, relin = true)."""
        ringQ = self.params.ringQ.AtLevel(level)
        c00, c01 = self._new(ringQ, level), self._new(ringQ, level)
        c0, c1, c2 = self._new(ringQ, level), self._new(ringQ, level), self._new(ringQ, level)
        ringQ.MulRNSScalarMontgomery(op0[0], self.tMontgomery, c00)
        ringQ.MulRNSScalarMontgomery(op0[1], self.tMontgomery, c01)
        if op0 is op1:
            ringQ.MulCoeffsMontgomery(c00, op1[0], c0)
            ringQ.MulCoeffsMontgomery(c01, op1[1], c2)
            ringQ.MulCoeffsMontgomery(c00, op1[1], c1)
            ringQ.Add(c1, c1, c1)
        else:
            ringQ.MulCoeffsMontgomery(c00, op1[0], c0)
            ringQ.MulCoeffsMontgomery(c01, op1[1], c2)
            ringQ.MulCoeffsMontgomery(c00, op1[1], c1)
            ringQ.MulCoeffsMontgomeryThenAdd(c01, op1[0], c1)
        return self._relinearize(level, c0, c1, c2)

    def modUpAndNTT(self, level, levelQMul, ctQ0):
        """:991-1001"""
        ringQ, ringQMul = self.params.ringQ.AtLevel(level), self.ringQMul.AtLevel(levelQMul)
        buffQ = self._new(ringQ, level)
        out = []
        for v in ctQ0:
            p = self._new(ringQMul, levelQMul)
            ringQ.INTT(v, buffQ)
            self.basisExtenderQ1toQ2.ModUpQtoP(level, levelQMul, buffQ, p)
            ringQMul.NTTLazy(p, p)
            out.append(p)
        return out

    def tensorLowDeg(self, level, levelQMul, ct0Q0, ct1Q0, ct0Q1, ct1Q1, square):
        """:1003-1048"""
        ringQ, ringQMul = self.params.ringQ.AtLevel(level), self.ringQMul.AtLevel(levelQMul)
        c00, c01 = self._new(ringQ, level), self._new(ringQ, level)
        ringQ.MForm(ct0Q0[0], c00)
        ringQ.MForm(ct0Q0[1], c01)
        c00M, c01M = self._new(ringQMul, levelQMul), self._new(ringQMul, levelQMul)
        ringQMul.MForm(ct0Q1[0], c00M)
        ringQMul.MForm(ct0Q1[1], c01M)
        ct2Q0 = [self._new(ringQ, level) for _ in range(3)]
        ct2Q1 = [self._new(ringQMul, levelQMul) for _ in range(3)]
        for ring, a, b, m0, m1, d in ((ringQ, ct0Q0, ct1Q0, c00, c01, ct2Q0), (ringQMul, ct0Q1, ct1Q1, c00M, c01M, ct2Q1)):
            if square:
                ring.MulCoeffsMontgomery(m0, a[0], d[0])
                ring.MulCoeffsMontgomery(m1, a[1], d[2])
                ring.MulCoeffsMontgomery(m0, a[1], d[1])
                ring.AddLazy(d[1], d[1], d[1])
            else:
                ring.MulCoeffsMontgomery(m0, b[0], d[0])
                ring.MulCoeffsMontgomery(m1, b[1], d[2])
                ring.MulCoeffsMontgomery(m0, b[1], d[1])
                ring.MulCoeffsMontgomeryThenAddLazy(m1, b[0], d[1])
        return ct2Q0, ct2Q1

    def quantize(self, level, levelQMul, c2Q1, c2Q2):
        """:1050-1070"""
        ringQ, ringQMul = self.params.ringQ.AtLevel(level), self.ringQMul.AtLevel(levelQMul)
        ringQ.INTTLazy(c2Q1, c2Q1)
        ringQMul.INTTLazy(c2Q2, c2Q2)
        self.basisExtenderQ1toQ2.ModDownQPtoP(level, levelQMul, c2Q1, c2Q2, c2Q2)
        self.basisExtenderQ1toQ2.ModUpPtoQ(levelQMul, level, c2Q2, c2Q1)
        ringQ.MulScalar(c2Q1, self.t, c2Q1)
        ringQ.NTT(c2Q1, c2Q1)

    def tensorScaleInvariant(self, level, ct0, ct1):
        """:898-978 (relin = true)."""
        levelQMul = self.levelQMul[level]
        square = ct0 is ct1
        tmp0Q1 = self.modUpAndNTT(level, levelQMul, ct0)
        tmp1Q1 = tmp0Q1 if square else self.modUpAndNTT(level, levelQMul, ct1)
        ct2Q0, ct2Q1 = self.tensorLowDeg(level, levelQMul, ct0, ct1, tmp0Q1, tmp1Q1, square)
        for k in range(3):
            self.quantize(level, levelQMul, ct2Q0[k], ct2Q1[k])
        return self._relinearize(level, ct2Q0[0], ct2Q0[1], ct2Q0[2])

    def Rescale(self, op0):
        """:1363-1393: DivRoundByLastModulusNTT of both polynomials; a copy for the scale-invariant evaluator."""
        if self.ScaleInvariant:
            return [v.copy() for v in op0]
        level = op0[0].shape[0] - 1
        assert level > 0, "cannot rescale: op0 already at level 0"
        ringQ = self.params.ringQ.AtLevel(level)
        out = [np.zeros((level, ringQ.N()), dtype=U64) for _ in op0]
        for i in range(len(op0)):
            ringQ.DivRoundByLastModulusNTT(op0[i], out[i])
        return out

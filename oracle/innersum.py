"""CPU restatement of the slot-aggregation family, `core/rlwe/inner_sum.go` (reference, pure Go):

    Trace                        :36-116    (X -> sum of the automorphisms of the subgroup, pre-multiplied by gap^-1)
    GaloisElementsForTrace       :120-141
    PartialTracesSum             :147-292   (double hoisting: log2(n) + HW(n) - 1 key switches)
    GaloisElementsForInnerSum    :442-466
    Replicate                    :475-477
    GaloisElementsForReplicate   :481-483

and the scheme wrappers that reach PartialTracesSum: ckks.Evaluator.InnerSum / RotateAndAdd (schemes/ckks/evaluator.go:1285-1317),
ckks.Evaluator.Average (schemes/ckks/linear_transformation.go:27-52), bgv.Evaluator.InnerSum / RotateAndAdd
(schemes/bgv/evaluator.go:1475-1535, with its RotateRows branch for n * batchSize == slots).

TEST INFRASTRUCTURE ONLY, like the rest of oracle/: built from oracle/oracle.py's Evaluator methods (DecomposeNTT,
AutomorphismHoisted[Lazy], Automorphism, BasisExtender.ModDownQPtoQNTT) and ring ops, as oracle/lintrans.py is. Parity status: the
reference holds no bit-level vectors for these methods; tests/test_oracle_innersum.py pins the restatement by decryption with real
Galois keys.

Conventions: ciphertexts are pairs [c0, c1] of (level+1, N) uint64 arrays, `is_ntt` tells their domain (the reference's
MetaData.IsNTT); Galois keys are {galEl: oracle.GadgetCiphertext}. Standard ring only."""
from __future__ import annotations

from typing import Dict, List

import numpy as np

from . import oracle as O

U64 = np.uint64


def GaloisElementsForTrace(params: O.Parameters, logN: int) -> List[int]:
    """:120-141 (Standard ring)."""
    gal = [params.GaloisElement(1 << i) for i in range(logN, params.logN - 1)]
    if logN == 0:
        gal.append(params.GaloisElementOrderTwoOrthogonalSubgroup())
    return gal


def GaloisElementsForInnerSum(params: O.Parameters, batch: int, n: int) -> List[int]:
    """:442-466; the reference returns the elements in map order, here they are sorted."""
    rot = set()
    i = 1
    while i < n:
        rot.add(i * batch)
        rot.add((n - (n & ((i << 1) - 1))) * batch)
        i <<= 1
    return sorted({params.GaloisElement(k) for k in rot})


def GaloisElementsForReplicate(params: O.Parameters, batch: int, n: int) -> List[int]:
    """:481-483."""
    return GaloisElementsForInnerSum(params, -batch, n)


class Evaluator:
    """rlwe.Evaluator's inner_sum.go methods over oracle.Evaluator. `asked` records every Galois element looked up."""

    def __init__(self, params: O.Parameters, galois_keys: Dict[int, O.GadgetCiphertext]):
        self.params = params
        self.ev = O.Evaluator(params)
        self.keys = galois_keys
        self.asked: List[int] = []

    def _key(self, galEl: int) -> O.GadgetCiphertext:
        self.asked.append(galEl)
        if galEl not in self.keys:
            raise KeyError("GaloisKey[%d] is missing" % galEl)      # CheckAndGetGaloisKey
        return self.keys[galEl]

    # --- :36-116 ---------------------------------------------------------------------------------------------
    def Trace(self, ctIn, logN: int, opOut, is_ntt: bool = True):
        """opOut: pair of arrays with at least min(levels) + 1 rows; rows 0..level are written. Returns the level."""
        params = self.params
        level = min(ctIn[0].shape[0], opOut[0].shape[0]) - 1
        N = params.N()
        gap = 1 << (params.logN - logN - 1)
        if logN == 0:
            gap <<= 1
        if gap > 1:
            ringQ = params.ringQ.AtLevel(level)
            NInv = pow(gap, -1, ringQ.ModulusAtLevel[level])
            cur = [np.empty((level + 1, N), dtype=U64) for _ in range(2)]
            ringQ.MulScalarBigint(ctIn[0][: level + 1], NInv, cur[0])
            ringQ.MulScalarBigint(ctIn[1][: level + 1], NInv, cur[1])
            if not is_ntt:
                ringQ.NTT(cur[0], cur[0]); ringQ.NTT(cur[1], cur[1])
            buff = [np.empty((level + 1, N), dtype=U64) for _ in range(2)]
            gals = [params.GaloisElement(1 << i) for i in range(logN, params.logN - 1)]
            if logN == 0:
                gals.append(ringQ.NthRoot() - 1)
            for g in gals:
                self.ev.Automorphism(cur, g, self._key(g), buff, level=level)
                ringQ.Add(cur[0], buff[0], cur[0]); ringQ.Add(cur[1], buff[1], cur[1])
            if not is_ntt:
                ringQ.INTT(cur[0], cur[0]); ringQ.INTT(cur[1], cur[1])
            for k in range(2):
                opOut[k][: level + 1] = cur[k]
        else:
            for k in range(2):
                opOut[k][: level + 1] = ctIn[k][: level + 1]
        return level

    # --- :147-292 --------------------------------------------------------------------------------------------
    def PartialTracesSum(self, ctIn, offset: int, n: int, opOut, is_ntt: bool = True):
        if n == 0 or offset == 0:
            raise ValueError("partialtrace: invalid parameter (n = 0 or batchSize = 0)")
        params = self.params
        levelQ = ctIn[0].shape[0] - 1
        levelP = params.MaxLevelP()
        N = params.N()
        ringQ = params.ringQ.AtLevel(levelQ)
        nq = levelQ + 1
        ctInNTT = [np.empty((nq, N), dtype=U64) for _ in range(2)]
        if not is_ntt:
            ringQ.NTT(ctIn[0], ctInNTT[0]); ringQ.NTT(ctIn[1], ctInNTT[1])
        else:
            ctInNTT[0][...] = ctIn[0]; ctInNTT[1][...] = ctIn[1]
        out = [np.empty((nq, N), dtype=U64) for _ in range(2)]
        if n == 1:
            out[0][...] = ctIn[0]; out[1][...] = ctIn[1]
        else:
            ringP = params.ringP.AtLevel(levelP)
            accQ = [np.zeros((nq, N), dtype=U64) for _ in range(2)]; accP = [np.zeros((levelP + 1, N), dtype=U64) for _ in range(2)]
            cQ = [np.zeros((nq, N), dtype=U64) for _ in range(2)]; cP = [np.zeros((levelP + 1, N), dtype=U64) for _ in range(2)]
            nd = params.BaseRNSDecompositionVectorSize(levelQ, levelP)
            decompQ = [np.zeros((nq, N), dtype=U64) for _ in range(nd)]
            decompP = [np.zeros((levelP + 1, N), dtype=U64) for _ in range(nd)]
            state, copy = False, True
            i, j = 0, n
            while j > 0:
                self.ev.DecomposeNTT(levelQ, levelP, levelP + 1, ctInNTT[1].copy(), True, decompQ, decompP)
                if j & 1 == 1:
                    k = (n - (n & ((2 << i) - 1))) * offset
                    if k != 0:
                        rot = params.GaloisElement(k)
                        if copy:
                            self.ev.AutomorphismHoistedLazy(levelQ, ctInNTT, decompQ, decompP, rot, self._key(rot), accQ, accP)
                            copy = False
                        else:
                            self.ev.AutomorphismHoistedLazy(levelQ, ctInNTT, decompQ, decompP, rot, self._key(rot), cQ, cP)
                            for c in range(2):
                                ringQ.Add(accQ[c], cQ[c], accQ[c]); ringP.Add(accP[c], cP[c], accP[c])
                    else:
                        state = True
                        if n & (n - 1) != 0:
                            be = self.ev.BasisExtender
                            be.ModDownQPtoQNTT(levelQ, levelP, accQ[0], accP[0], out[0])
                            be.ModDownQPtoQNTT(levelQ, levelP, accQ[1], accP[1], out[1])
                            ringQ.Add(out[0], ctInNTT[0], out[0]); ringQ.Add(out[1], ctInNTT[1], out[1])
                        else:
                            out[0][...] = ctInNTT[0]; out[1][...] = ctInNTT[1]
                if not state:
                    rot = params.GaloisElement((1 << i) * offset)
                    buf = [np.empty((nq, N), dtype=U64) for _ in range(2)]
                    self.ev.AutomorphismHoisted(levelQ, ctInNTT, decompQ, decompP, rot, self._key(rot), buf)
                    ringQ.Add(ctInNTT[0], buf[0], ctInNTT[0]); ringQ.Add(ctInNTT[1], buf[1], ctInNTT[1])
                i, j = i + 1, j >> 1
        if not is_ntt:
            ringQ.INTT(out[0], out[0]); ringQ.INTT(out[1], out[1])
        opOut[0][:nq] = out[0]; opOut[1][:nq] = out[1]

    def Replicate(self, ctIn, batchSize: int, n: int, opOut, is_ntt: bool = True):
        self.PartialTracesSum(ctIn, -batchSize, n, opOut, is_ntt)

    # --- scheme wrappers -------------------------------------------------------------------------------------
    def InnerSum(self, ctIn, batchSize: int, n: int, opOut, slots: int, bgv: bool = False, is_ntt: bool = True):
        """ckks.Evaluator.InnerSum (bgv = False) or bgv.Evaluator.InnerSum (bgv = True); slots = ctIn.Slots()."""
        check_inner_sum(batchSize, n, slots)
        if bgv and n * batchSize == slots:
            if n == 1:
                opOut[0][: ctIn[0].shape[0]] = ctIn[0]; opOut[1][: ctIn[1].shape[0]] = ctIn[1]
                return
            self.PartialTracesSum(ctIn, batchSize, n // 2, opOut, is_ntt)
            level = ctIn[0].shape[0] - 1
            ringQ = self.params.ringQ.AtLevel(level)
            cur = [opOut[0][: level + 1].copy(), opOut[1][: level + 1].copy()]
            tmp = [np.empty_like(cur[0]), np.empty_like(cur[1])]
            g = self.params.GaloisElementOrderTwoOrthogonalSubgroup()       # bgv.Evaluator.RotateRows
            self.ev.Automorphism(cur, g, self._key(g), tmp, level=level)
            ringQ.Add(cur[0], tmp[0], opOut[0][: level + 1]); ringQ.Add(cur[1], tmp[1], opOut[1][: level + 1])
            return
        self.PartialTracesSum(ctIn, batchSize, n, opOut, is_ntt)

    def Average(self, ctIn, logBatchSize: int, opOut, log_slots: int, is_ntt: bool = True):
        """ckks.Evaluator.Average: opOut = InnerSum(n^-1 * ctIn, 2^logBatchSize, n), n = 2^(log_slots - logBatchSize)."""
        if logBatchSize > log_slots:
            raise ValueError("cannot Average: batchSize must be smaller or equal to the number of slots")
        level = min(ctIn[0].shape[0], opOut[0].shape[0]) - 1
        n = 1 << (log_slots - logBatchSize)
        ringQ = self.params.ringQ.AtLevel(level)
        scaled = [np.empty((level + 1, self.params.N()), dtype=U64) for _ in range(2)]
        inv = [O.mform(pow(n, s.Modulus - 2, s.Modulus), s.Modulus) for s in ringQ.SubRings[: level + 1]]
        ringQ.MulRNSScalarMontgomery(ctIn[0][: level + 1], inv, scaled[0])
        ringQ.MulRNSScalarMontgomery(ctIn[1][: level + 1], inv, scaled[1])
        self.InnerSum(scaled, 1 << logBatchSize, n, opOut, 1 << log_slots, False, is_ntt)


def check_inner_sum(batchSize: int, n: int, slots: int):
    """The scheme-level checks of ckks / bgv InnerSum."""
    l = n * batchSize
    if n <= 0 or batchSize <= 0:
        raise ValueError("innersum: invalid parameter (n <= 0 or batchSize <= 0)")
    if l > slots:
        raise ValueError("innersum: invalid parameters (n*batchSize=%d > #slots=%d)" % (l, slots))
    if l & (l - 1) != 0:
        raise ValueError("innersum: invalid parameters (n*batchSize=%d does not divide #slots=%d)" % (l, slots))

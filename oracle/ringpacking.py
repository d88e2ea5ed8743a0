"""CPU restatement of the ring-packing family, `core/rlwe/ring_packing.go` and `ring_packing_keys.go` (reference, pure Go), on a
single ring degree (RingPackingEvaluator with MinLogN == MaxLogN):

    Extract                      :56-171    (logNFactor = 0: Expand + selection)
    Repack                       :252-374   (logNFactor = 0: Pack(cts, LogN, true))
    Expand                       :457-571
    Pack                         :600-770
    GenXPow2NTT                  :773-810
    getMinimumGap                :812-845
    GaloisElementsForExpand      ring_packing_keys.go:143-153
    GaloisElementsForPack        ring_packing_keys.go:156-180

TEST INFRASTRUCTURE ONLY, like the rest of oracle/: built from oracle/oracle.py's Evaluator.Automorphism and ring ops, as
oracle/innersum.py is. Parity status: the reference holds no bit-level vectors for these methods; tests/test_oracle_ringpacking.py
pins the restatement by decryption with real Galois keys.

Conventions: ciphertexts are pairs [c0, c1] of (level+1, N) uint64 arrays, `is_ntt` tells their domain (the reference's
MetaData.IsNTT); Galois keys are {galEl: oracle.GadgetCiphertext}. Standard ring only. Unlike the reference, Pack works on copies:
the caller's arrays are left as they were."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import oracle as O

U64 = np.uint64


def GaloisElementsForExpand(params: O.Parameters, logN: int) -> List[int]:
    NthRoot = params.ringQ.NthRoot()
    return [NthRoot // (2 << i) + 1 for i in range(logN)]


def GaloisElementsForPack(params: O.Parameters, logGap: int) -> List[int]:
    if logGap > params.logN or logGap < 0:
        raise ValueError("cannot GaloisElementsForPack: logGap > logN || logGap < 0")
    galEls = [params.GaloisElement(1 << i) for i in range(logGap)]
    if params.ringQ.Type != "Standard":
        raise ValueError("cannot GaloisElementsForPack: invalid ring type")
    if logGap == params.logN:
        galEls.append(params.GaloisElementOrderTwoOrthogonalSubgroup())
    return galEls


def GenXPow2NTT(r: O.Ring, logN: int, div: bool) -> List[np.ndarray]:
    """X^(+-2^i) for 0 <= i < logN, NTT domain, Montgomery form."""
    xPow = []
    N = r.N()
    for i in range(logN):
        idx = 1 << i
        if div:
            idx = N - idx
        p = r.NewPoly()
        if i == 0:
            for j, s in enumerate(r.SubRings[: r.Level() + 1]):
                p[j][idx] = O.mform(1, s.Modulus)
            r.NTT(p, p)
        else:
            r.MulCoeffsMontgomery(xPow[i - 1], xPow[i - 1], p)
        xPow.append(p)
    if div:
        r.Neg(xPow[0], xPow[0])
    return xPow


def getMinimumGap(lst: List[int]):
    gap, logGap = 0x7FFFFFFFFFFFFFFF, 0
    for i in range(1, len(lst)):
        a, b = lst[i - 1], lst[i]
        if a > b:
            raise ValueError("invalid index list: element must be sorted from smallest to largest")
        elif a == b:
            raise ValueError("invalid index list: contains duplicated elements")
        if b - a < gap:
            gap = b - a
        if gap == 1:
            break
    while gap & 1 == 0:
        logGap += 1
        gap >>= 1
    return gap, logGap


class RingPackingEvaluator:
    """rlwe.RingPackingEvaluator at one ring degree over oracle.Evaluator. `asked` records every Galois element looked up."""

    def __init__(self, params: O.Parameters, extract_keys: Dict[int, O.GadgetCiphertext], repack_keys: Dict[int, O.GadgetCiphertext]):
        self.params = params
        self.ev = O.Evaluator(params)
        self.extract_keys, self.repack_keys = extract_keys, repack_keys
        ringQ = params.ringQ.AtLevel(params.MaxLevelQ())
        self.XPow2NTT = GenXPow2NTT(ringQ, params.logN, False)
        self.XInvPow2NTT = GenXPow2NTT(ringQ, params.logN, True)
        self.asked: List[int] = []

    def _key(self, keys, galEl: int) -> O.GadgetCiphertext:
        self.asked.append(galEl)
        if galEl not in keys:
            raise KeyError("GaloisKey[%d] is missing" % galEl)
        return keys[galEl]

    def _automorphism(self, keys, ctIn, galEl, opOut, level):
        self.ev.Automorphism(ctIn, galEl, self._key(keys, galEl), opOut, level=level)

    # --- :457-571 --------------------------------------------------------------------------------------------
    def Expand(self, ct, logGap: int, is_ntt: bool = True) -> Dict[int, list]:
        params = self.params
        logN = params.logN
        xPow2 = self.XInvPow2NTT
        level = ct[0].shape[0] - 1
        ringQ = params.ringQ.AtLevel(level)
        cts = {0: [ct[0].copy(), ct[1].copy()]}
        if not is_ntt:
            ringQ.NTT(cts[0][0], cts[0][0]); ringQ.NTT(cts[0][1], cts[0][1])
        NInv = pow(1 << logN, -1, ringQ.ModulusAtLevel[level])
        ringQ.MulScalarBigint(cts[0][0], NInv, cts[0][0]); ringQ.MulScalarBigint(cts[0][1], NInv, cts[0][1])
        gap = 1 << logGap
        tmp = [np.empty_like(cts[0][0]) for _ in range(2)]
        for i in range(logN):
            n = 1 << i
            galEl = ringQ.N() // n + 1
            for j in range(0, n, gap):
                c0 = cts[j]
                self._automorphism(self.extract_keys, c0, galEl, tmp, level)
                if j + n // gap > 0:
                    c1 = [c0[0].copy(), c0[1].copy()]
                    ringQ.Add(c0[0], tmp[0], c0[0]); ringQ.Add(c0[1], tmp[1], c0[1])
                    ringQ.Sub(c1[0], tmp[0], c1[0]); ringQ.Sub(c1[1], tmp[1], c1[1])
                    ringQ.MulCoeffsMontgomery(c1[0], xPow2[i][: level + 1], c1[0])
                    ringQ.MulCoeffsMontgomery(c1[1], xPow2[i][: level + 1], c1[1])
                    cts[j + n] = c1
                else:
                    ringQ.Add(c0[0], tmp[0], c0[0]); ringQ.Add(c0[1], tmp[1], c0[1])
        # cts[0] was marked IsNTT = true above, so the reference's trailing INTT loop (:563-569) never fires
        return cts

    # --- :600-770 --------------------------------------------------------------------------------------------
    def Pack(self, cts_in: Dict[int, list], inputLogGap: int, zeroGarbageSlots: bool, is_ntt: bool = True) -> Optional[list]:
        if len(cts_in) == 0:
            raise ValueError("len(cts) = 0")
        params = self.params
        cts = {k: [v[0].copy(), v[1].copy()] for k, v in cts_in.items()}
        keys = sorted(cts)
        logN = params.logN
        xPow2 = self.XPow2NTT
        level = cts[keys[0]][0].shape[0] - 1
        if len(keys) > 1:
            try:
                gap, logGap = getMinimumGap(keys)
            except ValueError as e:
                raise ValueError("getMinimumGap: %s" % e) from None
        else:
            gap, logGap = params.N(), logN
        ringQ = params.ringQ.AtLevel(level)
        logStart, logEnd = logN - inputLogGap, logN
        if not zeroGarbageSlots:
            if gap > 0:
                logEnd -= logGap
        if logStart >= logEnd:
            raise ValueError("gaps between ciphertexts is smaller than inputLogGap > N")
        NInv = pow(1 << (logEnd - logStart), -1, ringQ.ModulusAtLevel[level])
        for key in keys:
            ct = cts[key]
            if not is_ntt:
                ringQ.NTT(ct[0], ct[0]); ringQ.NTT(ct[1], ct[1])
            ringQ.MulScalarBigint(ct[0], NInv, ct[0]); ringQ.MulScalarBigint(ct[1], NInv, ct[1])
        N = params.N()
        tmpa = [np.zeros((level + 1, N), dtype=U64) for _ in range(2)]
        for i in range(logStart, logEnd):
            t = 1 << (logN - 1 - i)
            for jx in range(t):
                jy = jx + t
                a, b = cts.get(jx), cts.get(jy)
                if b is not None:
                    x = xPow2[len(xPow2) - i - 1][: level + 1]
                    ringQ.MulCoeffsMontgomery(b[0], x, b[0]); ringQ.MulCoeffsMontgomery(b[1], x, b[1])
                    if a is not None:
                        ringQ.Sub(a[0], b[0], tmpa[0]); ringQ.Sub(a[1], b[1], tmpa[1])
                        ringQ.Add(a[0], b[0], a[0]); ringQ.Add(a[1], b[1], a[1])
                    else:
                        cts[jx] = cts[jy]
                    cts[jy] = None
                if a is not None or b is not None:
                    galEl = ringQ.NthRoot() - 1 if i == 0 else params.GaloisElement(1 << (i - 1))
                    if a is not None:
                        self._automorphism(self.repack_keys, tmpa if b is not None else a, galEl, tmpa, level)
                        ringQ.Add(a[0], tmpa[0], a[0]); ringQ.Add(a[1], tmpa[1], a[1])
                    else:
                        self._automorphism(self.repack_keys, b, galEl, tmpa, level)
                        ringQ.Sub(b[0], tmpa[0], b[0]); ringQ.Sub(b[1], tmpa[1], b[1])
        return cts.get(0)

    # --- :56-171 and :252-374 with MinLogN == MaxLogN ---------------------------------------------------------
    def Extract(self, ct, idx, is_ntt: bool = True) -> Dict[int, list]:
        keys = sorted(idx)
        try:
            _, logGap = getMinimumGap(keys)
        except ValueError as e:
            raise ValueError("getMinimumGap: %s" % e) from None
        ciphertexts = self.Expand(ct, logGap, is_ntt)
        cts = {}
        for j in keys:
            if j in ciphertexts:
                cts[j] = ciphertexts[j]
            else:
                raise ValueError("invalid ciphertexts map: index i+j*(NFactor*gap)=%d is nil" % (j * (1 << logGap)))
        return cts

    def Repack(self, cts: Dict[int, list], is_ntt: bool = True) -> Optional[list]:
        return self.Pack(cts, self.params.logN, True, is_ntt)

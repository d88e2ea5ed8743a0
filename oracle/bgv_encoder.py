"""oracle/bgv_encoder.py -- TEST INFRASTRUCTURE ONLY: a literal CPU restatement of bgv.Encoder (schemes/bgv/encoder.go, all of it) and of
the plaintext ring of bgv.NewParameters (schemes/bgv/params.go:76-135), on oracle.oracle's Ring (the coefficient-wise ops and transforms
of lattigo_oracle.c), its mod_up_exact, and Python integers for the big-integer branch of RingQ2T.

Values are Python / numpy integers; `signed` selects the reference's []int64 path, otherwise []uint64 (taken mod 2^64). One difference
from the reference is kept on purpose, as in the device encoder: plaintext rings of fewer than 16 slots are not built."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

from oracle import oracle as O

U64 = np.uint64
M64 = (1 << 64) - 1


def plaintext_order(t: int) -> int:
    """The largest cyclotomic order enabled by t (params.go:119-123)."""
    order = 1 << t.bit_length()
    while order != 0 and t & (order - 1) != 1:
        order >>= 1
    return order


def permute_matrix(logN: int) -> list:
    """permuteMatrix (encoder.go:110-133)."""
    N, pow_, mask = 1 << logN, 1, (2 << logN) - 1
    perm = [0] * N
    half = N >> 1
    for i in range(half):
        pos = O.bit_reverse64(pow_ >> 1, logN)
        perm[i] = pos
        perm[half + i] = N - pos - 1
        pow_ = pow_ * 5 & mask
    return perm


def bred_add(a: int, q: int) -> int:
    """ring.BRedAdd: exact a mod q for a < 2^64."""
    return a % q


def signed_word(c: int, T: int) -> int:
    """encoder.go:183-185 / :247-250: sign = uint64(c) >> 63; abs = BRedAdd(uint64(c * (1 - 2 sign))); sign * (T - abs) | (1 - sign) * abs
    (the word T itself when abs = 0)."""
    c = int(c)
    sign = (c & M64) >> 63
    mag = (c * (1 - 2 * sign)) & M64                               # int64 multiplication wraps: INT64_MIN stays 2^63
    ab = bred_add(mag, T)
    return (T - ab) if sign else ab


class BGVEncoder:
    """bgv.Encoder over ringQ (and ringP for Embed into a ringqp.Poly) with plaintext modulus t."""

    def __init__(self, ringQ: O.Ring, t: int, ringP: Optional[O.Ring] = None):
        t = int(t)
        Q = ringQ.ModuliChain()
        assert t >= 2 and t not in Q and t < Q[0]
        order = plaintext_order(t)
        assert order >= 16
        self.n = min(ringQ.N(), order >> 1)
        assert self.n >= 16, "plaintext rings of fewer than 16 slots are not built"
        self.ringQ, self.ringP, self.t = ringQ, ringP, t
        self.ringT = O.Ring(self.n, [t])
        self.indexMatrix = permute_matrix(self.n.bit_length() - 1)
        # NewEncoder (encoder.go:52-83)
        self.paramsQP = [None] + [O.ModUpConstants(Q[: i + 1], [t]) for i in range(1, len(Q))]
        self.qHalf = [None] + [ringQ.ModulusAtLevel[i] >> 1 for i in range(1, len(Q))]
        self.tInvModQ = [pow(t, -1, ringQ.ModulusAtLevel[i]) for i in range(len(Q))]

    def MaxSlots(self):
        return self.n

    # ---- encoding ----------------------------------------------------------------------------------------------
    def EncodeRingT(self, values: Sequence[int], signed: bool, scale: int):
        """encoder.go:213-270."""
        T, n = self.t, self.n
        assert len(values) <= n
        pt = np.zeros((1, n), dtype=U64)
        for i, c in enumerate(values):
            pt[0, self.indexMatrix[i]] = signed_word(c, T) if signed else int(c) & M64
        if not signed:
            self.ringT.Reduce(pt, pt)
        for i in range(len(values), n):
            pt[0, self.indexMatrix[i]] = 0
        self.ringT.INTT(pt, pt)
        self.ringT.MulScalar(pt, int(scale) & M64, pt)
        return pt

    def RingT2Q(self, level: int, scaleUp: bool, pT, ring: O.Ring):
        """encoder.go:378-407 onto the rows of `ring` at `level` (the reference passes RingQ for P rows too; only Embed writes P rows)."""
        N, n = ring.N(), pT.shape[1]
        gap = N // n
        pQ = np.zeros((level + 1, N), dtype=U64)
        for i in range(level + 1):
            pQ[i, ::gap] = pT[0]
        if scaleUp:
            self.ringQ.AtLevel(level).MulScalarBigint(pQ, self.tInvModQ[level], pQ)
        return pQ

    def EmbedScale(self, values, signed: bool, scaleUp: bool, scale: int, ntt: bool, mont: bool, level_q: int, level_p: int = -1):
        """encoder.go:276-333: the Q rows and, with level_p >= 0, the P rows of a ringqp.Poly (None otherwise)."""
        pT = self.EncodeRingT(values, signed, scale)
        rq = self.ringQ.AtLevel(level_q)
        pq = self.RingT2Q(level_q, scaleUp, pT, rq)
        if ntt:
            rq.NTT(pq, pq)
        if mont:
            rq.MForm(pq, pq)
        pp = None
        if level_p >= 0:
            assert not scaleUp, "RingT2Q would scale the P rows with the Q moduli (encoder.go:404-406)"
            rp = self.ringP.AtLevel(level_p)
            pp = self.RingT2Q(level_p, False, pT, rp)
            if ntt:
                rp.NTT(pp, pp)
            if mont:
                rp.MForm(pp, pp)
        return pq, pp

    def Embed(self, values, signed, scale, ntt, mont, level_q, level_p=-1):
        return self.EmbedScale(values, signed, False, scale, ntt, mont, level_q, level_p)

    def Encode(self, values, signed: bool, scale: int, ntt: bool, mont: bool, level: int, batched: bool = True):
        """encoder.go:140-199."""
        if batched:
            return self.EmbedScale(values, signed, True, scale, ntt, mont, level)[0]
        T, N = self.t, self.ringQ.N()
        assert len(values) <= N
        buff = np.zeros((1, N), dtype=U64)
        for i, c in enumerate(values):
            buff[0, i] = signed_word(c, T) if signed else int(c) & M64
        self.ringT.SubRings[0].vecop("MulScalarMontgomery", buff[0], None, buff[0], O.mform(int(scale) % T, T))   # ringT.MulScalar over N words
        pq = self.RingT2Q(level, True, buff, self.ringQ.AtLevel(level))
        if ntt:
            self.ringQ.AtLevel(level).NTT(pq, pq)
        return pq

    # ---- decoding ----------------------------------------------------------------------------------------------
    def RingQ2T(self, level: int, pQ, nT: int):
        """RingQ2T(level, scaleDown = true, pQ, pT) (encoder.go:412-467) with pT of nT coefficients (RingT's n, or N for coefficients)."""
        ringQ = self.ringQ.AtLevel(level)
        T = self.t
        N = pQ.shape[1]
        poly = np.empty((level + 1, N), dtype=U64)
        ringQ.MulScalar(pQ[: level + 1], T, poly)
        gap = N // nT
        pT = np.zeros((1, nT), dtype=U64)
        subT = self.ringT.SubRings[0]                                  # its ops take their length from the buffer
        q0 = ringQ.SubRings[0].Modulus
        if level > 0:
            if gap == 1:
                buffQ = np.empty_like(poly)
                ringQ.AddScalarBigint(poly, self.qHalf[level], buffQ)
                O.mod_up_exact(buffQ, pT, ringQ, self.ringT, self.paramsQP[level])
                subT.vecop("SubScalar", pT[0], None, pT[0], self.qHalf[level] % T)
            else:
                big = _poly_to_bigint_centered(ringQ, poly, gap)
                pT[0] = np.array([c % T for c in big], dtype=U64)          # SetCoefficientsBigint: big.Int.Mod is Euclidean
        else:
            buf = poly[0, ::gap].copy()
            ringQ.SubRings[0].vecop("AddScalar", buf, None, buf, q0 >> 1)
            subT.vecop("Reduce", buf, None, pT[0])
            subT.vecop("SubScalar", pT[0], None, pT[0], bred_add(q0 >> 1, T))
        return pT

    def DecodeRingT(self, pT, scale: int, signed: bool):
        """encoder.go:340-375: all MaxSlots values."""
        T = self.t
        buf = pT.copy()
        self.ringT.MulScalar(buf, pow(int(scale) % T, T - 2, T), buf)
        self.ringT.NTT(buf, buf)
        vals = [int(buf[0, self.indexMatrix[i]]) for i in range(self.n)]
        if signed:
            vals = [v - T if v >= T >> 1 else v for v in vals]
        return vals

    def Decode(self, pt, level: int, scale: int, ntt: bool, batched: bool = True, signed: bool = False, values: Optional[list] = None):
        """encoder.go:471-521. Coefficient mode returns N values; signed, only the first RingT().N() are written into `values` (N words,
        zeros by default) and the rest stay as they were."""
        N = self.ringQ.N()
        pq = np.array(pt[: level + 1], dtype=U64)
        if ntt:
            self.ringQ.AtLevel(level).INTT(pq, pq)
        nT = self.n if batched else N
        pT = self.RingQ2T(level, pq, nT)
        if batched:
            return self.DecodeRingT(pT, scale, signed)
        T = self.t
        self.ringT.SubRings[0].vecop("MulScalarMontgomery", pT[0], None, pT[0], O.mform(pow(int(scale) % T, T - 2, T), T))
        out = list(values) if values is not None else [0] * N
        if not signed:
            return [int(x) for x in pT[0]]
        for i in range(self.n):
            v = int(pT[0, i])
            out[i] = v - T if v >= T >> 1 else v
        return out


def _poly_to_bigint_centered(ringQ: O.Ring, p, gap: int) -> list:
    """ring.Ring.PolyToBigintCentered (ring/ring.go:469-508): X = CRT mod Q of coefficients j * gap, X - Q when X >= floor(Q / 2)."""
    level = ringQ.Level()
    Q = ringQ.ModulusAtLevel[level]
    crt = []
    for s in ringQ.SubRings[: level + 1]:
        Qi = Q // s.Modulus
        crt.append(Qi * (pow(Qi, -1, s.Modulus) % s.Modulus))
    half = Q >> 1
    out = []
    for j in range(0, ringQ.N(), gap):
        x = sum(int(p[k, j]) * crt[k] for k in range(level + 1)) % Q
        out.append(x - Q if x >= half else x)
    return out

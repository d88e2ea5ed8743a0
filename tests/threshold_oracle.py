"""CPU restatement of the t-out-of-N threshold scheme of multiparty/threshold.go that csrc/multiparty.cu and lattigo_b200.multiparty
serve, with Python integers for every scalar:

    Thresholdizer.GenShamirSecretShare   threshold.go:102-104 -> ringqp.Ring.EvalPolyScalar (ring/ringqp/operations.go:92-102,
                                         ring/operations.go:269-275): MulScalar = MRed(x, MForm(pt)), MForm in its Barrett form on the
                                         unreduced point (ring/modular_reduction.go:11-35), then Add = CRed on the wrapping 64-bit sum
    NewCombiner / GenAdditiveShare       threshold.go:117-179: MForm(1), SubRNSScalar, Inverse = ModexpMontgomery(x, q - 2)
                                         (ring/utils.go:58-69), MulRNSScalar = MRedLazy (ring/scalar.go:63-67), and the final
                                         MulRNSScalarMontgomery = MRed per word

eval_poly_scalar_word is the per-word statement; eval_poly_scalar applies the same steps to whole rows through the oracle's vector ops
(MulScalarMontgomery = MRed, Add = CRed of the wrapping sum), and the CPU tests hold the two equal.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np

from oracle import oracle as O

U64 = np.uint64
MASK = (1 << 64) - 1


def mform(a: int, q: int) -> int:
    """ring.MForm: -(a bhi + mulhi(a, blo)) q mod 2^64, then one conditional subtraction."""
    bhi, blo = O.gen_bred_constant(q)
    mhi = (a * blo) >> 64
    r = (-(a * bhi + mhi) * q) & MASK
    return r - q if r >= q else r


def mred_lazy(x: int, y: int, q: int) -> int:
    """ring.MRedLazy: hi(x y) - hi(lo(lo(x y) qinv) q) + q mod 2^64."""
    qinv = O.gen_mred_constant(q)
    p = x * y
    h = (((p & MASK) * qinv & MASK) * q) >> 64
    return ((p >> 64) - h + q) & MASK


def mred(x: int, y: int, q: int) -> int:
    r = mred_lazy(x, y, q)
    return r - q if r >= q else r


def cred(a: int, q: int) -> int:
    return a - q if a >= q else a


def modexp_montgomery(x: int, e: int, q: int) -> int:
    result = mform(1, q)
    while e > 0:
        if e & 1:
            result = mred(result, x, q)
        x = mred(x, x, q)
        e >>= 1
    return result


def eval_poly_scalar_word(coeffs, pt: int, q: int) -> int:
    """One word of EvalPolyScalar: coeffs[i] is the word of coefficient i (any 64-bit value)."""
    m = mform(pt, q)
    acc = int(coeffs[-1])
    for i in range(len(coeffs) - 1, 0, -1):
        acc = cred((mred(acc, m, q) + int(coeffs[i - 1])) & MASK, q)
    return acc


def eval_poly_scalar(poly, pt: int, moduli, N: int):
    """poly: (t, rows, N) uint64 words; moduli: one per row. Returns the (rows, N) share."""
    out = np.array(poly[-1], dtype=U64, copy=True)
    for r, q in enumerate(moduli):
        s = O.get_subring(N, int(q))
        m = mform(pt, int(q))
        for i in range(poly.shape[0] - 1, 0, -1):
            s.vecop("MulScalarMontgomery", out[r], None, out[r], m)
            s.vecop("Add", out[r], np.ascontiguousarray(poly[i - 1, r]), out[r])
    return out


def shamir_shares(poly, points, moduli, N: int):
    return np.stack([eval_poly_scalar(poly, int(x), moduli, N) for x in points])


def aggregate(shares, moduli):
    """agg = shares[0]; agg = Add(agg, s) for the rest."""
    agg = np.array(shares[0], dtype=U64, copy=True)
    for s in shares[1:]:
        for r, q in enumerate(moduli):
            with np.errstate(over="ignore"):
                t = agg[r] + s[r]
            agg[r] = np.where(t >= U64(q), t - U64(q), t)
    return agg


class Combiner:
    def __init__(self, moduli, own: int, others, threshold: int):
        self.moduli = [int(q) for q in moduli]
        self.threshold = threshold
        self.one = [mform(1, q) for q in self.moduli]
        self.lagrangeCoeffs = {}
        for spk in others:
            if spk != own:
                self.lagrangeCoeffs[spk] = self.lagrange_coeff(own, spk)

    def lagrange_coeff(self, this: int, that: int):
        out = []
        for q in self.moduli:
            a, b = that % q, this % q
            d = a + q - b if b > a else a - b
            out.append(mred_lazy(modexp_montgomery(d, q - 2, q), a, q))
        return out

    def prod(self, actives, own: int):
        assert len(actives) >= self.threshold
        prod = list(self.one)
        for active in actives[: self.threshold]:
            if active != own:
                prod = [mred_lazy(x, y, q) for x, y, q in zip(prod, self.lagrangeCoeffs[active], self.moduli)]
        return prod

    def gen_additive_share(self, actives, own: int, share, N: int):
        prod = self.prod(actives, own)
        out = np.empty_like(share)
        for r, q in enumerate(self.moduli):
            O.get_subring(N, q).vecop("MulScalarMontgomery", np.ascontiguousarray(share[r]), None, out[r], prod[r])
        return out

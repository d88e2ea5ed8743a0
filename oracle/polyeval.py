"""Literal restatement of ckks polynomial.Evaluator.Evaluate (circuits/ckks/polynomial/polynomial_evaluator.go:42-57) for one
bignum.Polynomial (Lazy = false), op by op, on the oracle's CKKS evaluator:
  circuits/common/polynomial/polynomial_evaluator.go:29-359   Evaluate, EvaluatePatersonStockmeyerPolynomialVector, EvaluateBabyStep,
                                                              EvaluateGiantStep, EvaluateMonomial, EvaluatePolynomialVectorFromPowerBasis
  circuits/common/polynomial/power_basis.go:32-182            SplitDegree, GenPower, genPower
  circuits/common/polynomial/polynomial.go:37-153             Factorize, PatersonStockmeyerPolynomial, recursePS
  circuits/ckks/polynomial/polynomial_evaluator_sim.go        simEvaluator
  utils/bignum/polynomial.go:14-23, :257-314                  OptimalSplit, Polynomial.Factorize
  schemes/ckks/evaluator.go                                   Add / Sub (evaluateInPlace, scalar), Mul (tensor / scalar), MulThenAdd, Rescale
  schemes/ckks/scaling.go:10-43                               bigComplexToRNSScalar
Every ciphertext object carries its own level and scale, as the reference's do. big.Float values are (Fraction, precision) pairs rounded
to nearest-even at every operation, as math/big does; rlwe.Scale is a big.Float at ScalePrecision = 128 bits.
TEST INFRASTRUCTURE ONLY: lattigo_b200/polyeval.py is the product's planner and does not import this module."""
from __future__ import annotations

from fractions import Fraction
from typing import Dict, List, Optional

import numpy as np

from oracle import oracle as O

U64 = np.uint64
SCALE_PREC = 128
MONOMIAL, CHEBYSHEV = 0, 1


# ---------------------------------------------------------------------------------------------------------------- math/big
def rnd(x: Fraction, prec: int) -> Fraction:
    """x rounded to `prec` significant bits, ties to even (big.Float's default ToNearestEven)."""
    x = Fraction(x)
    if x == 0:
        return x
    s = -1 if x < 0 else 1
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()       # 2^e <= a < 2^(e+2)
    if Fraction(2) ** e > a:
        e -= 1
    sh = prec - 1 - e                                                 # a * 2^sh in [2^(prec-1), 2^prec)
    v = a * (Fraction(2) ** sh)
    n, r = divmod(v.numerator, v.denominator)
    if 2 * r > v.denominator or (2 * r == v.denominator and n & 1):
        n += 1
    return s * Fraction(n) / (Fraction(2) ** sh)


def trunc(x: Fraction) -> int:
    """big.Float.Int: truncation toward zero."""
    return int(x)


class BF:
    """big.Float with its precision."""
    __slots__ = ("v", "prec")

    def __init__(self, v, prec):
        self.v, self.prec = Fraction(v), prec


def scale_mul(a: Fraction, b: Fraction) -> Fraction: return rnd(a * b, SCALE_PREC)      # rlwe.Scale.Mul
def scale_div(a: Fraction, b: Fraction) -> Fraction: return rnd(a / b, SCALE_PREC)      # rlwe.Scale.Div
def new_scale(x) -> Fraction: return rnd(Fraction(x), SCALE_PREC)                         # rlwe.NewScale


def in_delta(a: Fraction, b: Fraction, log2delta: int) -> bool:
    """rlwe.Scale.InDelta: -log2(|a - b| / max(a, b)) >= log2delta."""
    d = abs(a - b)
    return d == 0 or d * (Fraction(2) ** log2delta) <= max(a, b)


def to_complex(c, prec):
    """bignum.ToComplex(c, prec) for a (BF, BF) coefficient or an int."""
    if isinstance(c, int):
        return (BF(rnd(c, prec), prec), BF(0, prec))
    return (BF(rnd(c[0].v, prec), prec), BF(rnd(c[1].v, prec), prec))


def is_int(c) -> bool:
    return c[0].v.denominator == 1 and c[1].v.denominator == 1


def big_complex_to_rns_scalar(mods, scale: Fraction, cmplx):
    """schemes/ckks/scaling.go:10-43. scale is a 128-bit rlwe.Scale value."""
    out = []
    for part in cmplx:
        p = max(part.prec, SCALE_PREC)
        r = rnd(part.v * scale, p)
        if part.v > 0:
            r = rnd(r + Fraction(1, 2), p)
        elif part.v < 0:
            r = rnd(r - Fraction(1, 2), p)
        v = trunc(r)
        out.append([v % q for q in mods])
    return out[0], out[1]


# ---------------------------------------------------------------------------------------------------------------- polynomials
class Poly:
    """polynomial.Polynomial around a bignum.Polynomial: Coeffs (list of (BF, BF) or None), Basis, IsOdd, IsEven, MaxDeg, Lead, Level, Scale."""

    def __init__(self, coeffs, basis, is_odd=True, is_even=True):
        self.Coeffs, self.Basis, self.IsOdd, self.IsEven = coeffs, basis, is_odd, is_even
        self.MaxDeg, self.Lead, self.Level, self.Scale = len(coeffs) - 1, True, 0, Fraction(0)

    def Degree(self): return len(self.Coeffs) - 1

    def Depth(self):                                   # bignum.Polynomial.Depth: ceil(log2(degree))
        return (self.Degree() - 1).bit_length()


def new_polynomial(basis, coeffs, is_odd=True, is_even=True) -> Poly:
    """bignum.NewPolynomial with []float64 / []complex128 coefficients: 53-bit big.Floats."""
    cs = []
    for c in coeffs:
        c = complex(c)
        cs.append((BF(Fraction(c.real), 53), BF(Fraction(c.imag), 53)))
    return Poly(cs, basis, is_odd, is_even)


def _clone(c): return (BF(c[0].v, c[0].prec), BF(c[1].v, c[1].prec))


def optimal_split(logDegree: int) -> int:         # utils/bignum/polynomial.go:14-23
    logSplit = logDegree >> 1
    a = (1 << logSplit) + (1 << (logDegree - logSplit)) + logDegree - logSplit - 3
    b = (1 << (logSplit + 1)) + (1 << (logDegree - logSplit - 1)) + logDegree - logSplit - 4
    if a > b:
        logSplit += 1
    return logSplit


def split_degree(n: int):                          # power_basis.go:34-52
    if n <= 0:
        raise ValueError("invalid n: n=%d should be greater than zero" % n)
    if n & (n - 1) == 0:
        return n // 2, n // 2
    k = (n - 1).bit_length() - 1
    return (1 << k) - 1, n + 1 - (1 << k)


def bignum_factorize(p: Poly, n: int):             # utils/bignum/polynomial.go:257-314
    if n < p.Degree() >> 1:
        raise ValueError("cannot Factorize: n < p.Degree()/2")
    pr = [(_clone(p.Coeffs[i]) if p.Coeffs[i] is not None else None) for i in range(n)]
    pq = [None] * (p.Degree() - n + 1)
    if p.Coeffs[n] is not None:
        pq[0] = _clone(p.Coeffs[n])
    odd, even = p.IsOdd, p.IsEven
    keep = lambda i: (not (even or odd)) or (i & 1 == 0 and even) or (i & 1 == 1 and odd)
    if p.Basis == MONOMIAL:
        for i in range(n + 1, p.Degree() + 1):
            if p.Coeffs[i] is not None and keep(i):
                pq[i - n] = _clone(p.Coeffs[i])
    else:
        j = 1
        for i in range(n + 1, p.Degree() + 1):
            if p.Coeffs[i] is not None and keep(i):
                c = _clone(p.Coeffs[i])
                pq[i - n] = tuple(BF(rnd(x.v + x.v, x.prec), x.prec) for x in c)                 # Add(x, x)
                if pr[n - j] is not None:
                    pr[n - j] = tuple(BF(rnd(z.v - y.v, z.prec), z.prec) for z, y in zip(pr[n - j], p.Coeffs[i]))   # Sub
                else:
                    pr[n - j] = tuple(BF(-x.v, x.prec) for x in _clone(p.Coeffs[i]))
            j += 1
    q_, r_ = Poly(pq, p.Basis, p.IsOdd, p.IsEven), Poly(pr, p.Basis, p.IsOdd, p.IsEven)
    return q_, r_


def factorize(p: Poly, n: int):                    # common/polynomial/polynomial.go:37-58
    pq, pr = bignum_factorize(p, n)
    pq.MaxDeg = p.MaxDeg
    pr.MaxDeg = n - 1 if p.MaxDeg == p.Degree() else p.MaxDeg - (p.Degree() - n + 1)
    pq.Lead = bool(p.Lead)
    pr.Lead = False
    return pq, pr


class SimOp:
    def __init__(self, level, scale): self.Level, self.Scale = level, scale


class SimEval:                                     # circuits/ckks/polynomial/polynomial_evaluator_sim.go
    def __init__(self, Q, lpr): self.Q, self.lpr = Q, lpr

    def PolynomialDepth(self, degree):
        if degree <= 0:
            raise ValueError("invalid degree")
        return self.lpr * (degree.bit_length() - 1)

    def Rescale(self, op):
        for _ in range(self.lpr):
            op.Scale = scale_div(op.Scale, new_scale(self.Q[op.Level])); op.Level -= 1

    def MulNew(self, a, b): return SimOp(min(a.Level, b.Level), scale_mul(a.Scale, b.Scale))

    def UpdateLevelAndScaleBabyStep(self, lead, tLevelOld, tScaleOld):
        s = tScaleOld
        if lead:
            for i in range(self.lpr):
                s = scale_mul(s, new_scale(self.Q[tLevelOld - i]))
        return tLevelOld, s

    def UpdateLevelAndScaleGiantStep(self, lead, tLevelOld, tScaleOld, xPowScale):
        if lead:
            qi = self.Q[tLevelOld]
            for i in range(1, self.lpr):
                qi *= self.Q[tLevelOld - i]
        else:
            qi = self.Q[tLevelOld + self.lpr]
            for i in range(1, self.lpr):
                qi *= self.Q[tLevelOld + self.lpr - i]
        return tLevelOld + self.lpr, scale_div(scale_mul(tScaleOld, new_scale(qi)), xPowScale)


def sim_gen_power(pb, n, ev):                      # polynomial_evaluator_sim.go SimPowerBasis.GenPower
    if n < 2:
        return
    a, b = split_degree(n)
    sim_gen_power(pb, a, ev); sim_gen_power(pb, b, ev)
    pb[n] = ev.MulNew(pb[a], pb[b]); ev.Rescale(pb[n])


def recurse_ps(logSplit, targetLevel, p: Poly, pb, outputScale, ev: SimEval):     # polynomial.go:109-153
    if p.Degree() < (1 << logSplit):
        if p.Lead and logSplit > 1 and p.MaxDeg > (1 << p.MaxDeg.bit_length()) - (1 << (logSplit - 1)):
            return recurse_ps(optimal_split(p.Degree().bit_length()), targetLevel, p, pb, outputScale, ev)
        p.Level, p.Scale = ev.UpdateLevelAndScaleBabyStep(p.Lead, targetLevel, outputScale)
        return [p], SimOp(p.Level, p.Scale)
    nextPower = 1 << logSplit
    while nextPower < (p.Degree() >> 1) + 1:
        nextPower <<= 1
    XPow = pb[nextPower]
    coeffsq, coeffsr = factorize(p, nextPower)
    tLevelNew, tScaleNew = ev.UpdateLevelAndScaleGiantStep(p.Lead, targetLevel, outputScale, XPow.Scale)
    bsgsQ, res = recurse_ps(logSplit, tLevelNew, coeffsq, pb, tScaleNew, ev)
    ev.Rescale(res)
    res = ev.MulNew(res, XPow)
    bsgsR, tmp = recurse_ps(logSplit, targetLevel, coeffsr, pb, res.Scale, ev)
    if not in_delta(tmp.Scale, res.Scale, SCALE_PREC - 12):
        raise ValueError("recursePS: res.Scale != tmp.Scale")
    return bsgsQ + bsgsR, res


def paterson_stockmeyer(p: Poly, Q, lpr, inputLevel, inputScale, outputScale):   # polynomial.go:74-106
    logDegree = p.Degree().bit_length()
    logSplit = optimal_split(logDegree)
    ev = SimEval(Q, lpr)
    pb = {1: SimOp(inputLevel, inputScale)}
    sim_gen_power(pb, 1 << logDegree, ev)
    for i in range((1 << logSplit) - 1, 2, -1):
        sim_gen_power(pb, i, ev)
    ps, _ = recurse_ps(logSplit, inputLevel - ev.PolynomialDepth(p.Degree()), p, pb, outputScale, ev)
    return ps


# ---------------------------------------------------------------------------------------------------------------- ciphertexts
class Ct:
    """rlwe.Ciphertext: Value (degree+1 polynomials of level+1 rows, NTT domain), Scale."""

    def __init__(self, value, scale):
        self.Value, self.Scale = [np.array(v, dtype=U64) for v in value], Fraction(scale)

    def Level(self): return self.Value[0].shape[0] - 1
    def Degree(self): return len(self.Value) - 1


class PolyEvaluator:
    """polynomial.Evaluator[*bignum.Complex] over the oracle CKKS evaluator. encoding_precision = Parameters.EncodingPrecision()
    = max(53, log2(DefaultScale))."""

    def __init__(self, params: O.Parameters, rlk: O.GadgetCiphertext, levels_per_rescale=1, encoding_precision=53):
        self.params, self.rlk, self.lpr, self.prec = params, rlk, levels_per_rescale, encoding_precision
        self.ev = O.CKKSEvaluator(params, rlk, levels_per_rescale)
        self.Q = list(params.qi)

    def _ring(self, level): return self.params.ringQ.AtLevel(level)

    def _roots1(self, level): return [int(s.RootsForward[1]) for s in self.params.ringQ.SubRings[: level + 1]]

    # ---- schemes/ckks/evaluator.go -------------------------------------------------------------------------------
    def _with_scalar(self, level, p0, re, im, p1, op):            # evaluateWithScalar :410-424
        mods = self.Q[: level + 1]
        r1 = self._roots1(level)
        s0, s1 = [], []
        for i, q in enumerate(mods):
            m = O.mform(1, q)
            imag = im[i] * r1[i] * pow(m, -1, q) % q                 # MRed(imag, RootsForward[1])
            s0.append((re[i] + imag) % q); s1.append((re[i] + q - imag) % q)
        ring = self._ring(level)
        for a, b in zip(p0, p1):
            getattr(ring, op)(a, s0, s1, b)

    def mul_scalar(self, op0: Ct, c, opOut_rows=None) -> Ct:        # Mul, scalar case :629-666
        level = op0.Level() if opOut_rows is None else min(op0.Level(), opOut_rows)
        cmplx = to_complex(c, self.prec)
        if is_int(cmplx):
            scale = new_scale(1)
        else:
            scale = new_scale(self.Q[level])
            for i in range(1, self.lpr):
                scale = scale_mul(scale, new_scale(self.Q[level - i]))
        re, im = big_complex_to_rns_scalar(self.Q[: level + 1], scale, cmplx)
        out = [np.empty((level + 1, self.params.N()), dtype=U64) for _ in op0.Value]
        self._with_scalar(level, [v[: level + 1] for v in op0.Value], re, im, out, "MulDoubleRNSScalar")
        return Ct(out, scale_mul(op0.Scale, scale))

    def add_const(self, op0: Ct, c, sub=False) -> Ct:              # Add / Sub with a scalar :67-86, :158-177
        level = op0.Level()
        re, im = big_complex_to_rns_scalar(self.Q[: level + 1], op0.Scale, to_complex(c, self.prec))
        out = [v.copy() for v in op0.Value]
        self._with_scalar(level, op0.Value[:1], re, im, out[:1], "SubDoubleRNSScalar" if sub else "AddDoubleRNSScalar")
        return Ct(out, op0.Scale)

    def add_ct(self, c0: Ct, c1: Ct, sub=False) -> Ct:              # Add / Sub (ct, ct) with opOut == c0 (evaluateInPlace :221-408)
        level = min(c0.Level(), c1.Level())
        ring = self._ring(level)
        cmp = (c0.Scale > c1.Scale) - (c0.Scale < c1.Scale)
        tmp0, tmp1 = Ct([v[: level + 1] for v in c0.Value], c0.Scale), Ct([v[: level + 1] for v in c1.Value], c1.Scale)
        out_scale = c0.Scale
        if cmp == 1:
            ratio = trunc(scale_div(c0.Scale, c1.Scale))
            if ratio > 0:
                tmp1 = self.mul_scalar(tmp1, ratio)
        elif cmp == -1:
            ratio = trunc(scale_div(c1.Scale, c0.Scale))
            if ratio > 0:
                tmp0 = self.mul_scalar(tmp0, ratio)
                out_scale = c1.Scale
        maxd, mind = max(c0.Degree(), c1.Degree()), min(c0.Degree(), c1.Degree())
        out = [np.empty((level + 1, self.params.N()), dtype=U64) for _ in range(maxd + 1)]
        for i in range(mind + 1):
            (ring.Sub if sub else ring.Add)(tmp0.Value[i], tmp1.Value[i], out[i])
        for i in range(mind + 1, maxd + 1):
            if c0.Degree() > c1.Degree():
                out[i][:] = tmp0.Value[i]
            else:
                out[i][:] = tmp1.Value[i]
                if sub:
                    ring.Neg(out[i], out[i])
        return Ct(out, max(out_scale, c1.Scale))

    def mul_relin(self, a: Ct, b: Ct) -> Ct:                         # MulRelinNew :719-872
        v = self.ev.MulRelinNew(a.Value, b.Value)
        return Ct(v, scale_mul(a.Scale, b.Scale))

    def mul_tensor(self, op0: Ct, op1: Ct) -> Ct:                    # Mul (ct x ct, relin = false): mulRelin :764-839
        level = min(op0.Level(), op1.Level())
        ring = self._ring(level)
        N = self.params.N()
        mk = lambda: np.empty((level + 1, N), dtype=U64)
        c00, c01, c0, c1, c2 = mk(), mk(), mk(), mk(), mk()
        ring.MForm(op0.Value[0], c00); ring.MForm(op0.Value[1], c01)
        ring.MulCoeffsMontgomery(c00, op1.Value[0], c0)
        ring.MulCoeffsMontgomery(c01, op1.Value[1], c2)
        ring.MulCoeffsMontgomery(c00, op1.Value[1], c1)
        ring.MulCoeffsMontgomeryThenAdd(c01, op1.Value[0], c1)
        return Ct([c0, c1, c2], scale_mul(op0.Scale, op1.Scale))

    def relinearize(self, ct: Ct) -> Ct:                             # rlwe.Evaluator.Relinearize
        out = [np.empty_like(ct.Value[0]) for _ in range(2)]
        self.ev.Relinearize(ct.Value, self.rlk, out)
        return Ct(out, ct.Scale)

    def rescale(self, ct: Ct) -> Ct:                                 # Rescale :477-515
        if ct.Level() <= self.lpr - 1:
            raise ValueError("cannot Rescale: input Ciphertext level is too low")
        s = ct.Scale
        for i in range(self.lpr):
            s = scale_div(s, new_scale(self.Q[ct.Level() - i]))
        return Ct(self.ev.Rescale(ct.Value), s)

    def mul_then_add(self, op0: Ct, c, opOut: Ct) -> Ct:             # MulThenAdd, scalar case :928-975
        level = min(op0.Level(), opOut.Level())
        cmplx = to_complex(c, self.prec)
        cmp = (op0.Scale > opOut.Scale) - (op0.Scale < opOut.Scale)
        if cmp == 0:
            if is_int(cmplx):
                scaleRLWE = new_scale(1)
            else:
                scaleRLWE = new_scale(self.Q[level])
                for i in range(1, self.lpr):
                    scaleRLWE = scale_mul(scaleRLWE, new_scale(self.Q[level - i]))
                opOut = self.mul_scalar(opOut, trunc(scaleRLWE))
                opOut.Scale = scale_mul(opOut.Scale, scaleRLWE)
        elif cmp == -1:
            scaleRLWE = scale_div(opOut.Scale, op0.Scale)
        else:
            raise ValueError("cannot MulThenAdd: op0.Scale > opOut.Scale is not supported")
        re, im = big_complex_to_rns_scalar(self.Q[: level + 1], scaleRLWE, cmplx)
        out = [v.copy() for v in opOut.Value]
        self._with_scalar(level, [v[: level + 1] for v in op0.Value], re, im, [v[: level + 1] for v in out], "MulDoubleRNSScalarThenAdd")
        return Ct(out, opOut.Scale)

    # ---- power_basis.go ------------------------------------------------------------------------------------------
    def gen_power(self, pb: Dict[int, Ct], basis, n):
        if n not in pb:
            if self._gen_power(pb, basis, n):
                pb[n] = self.rescale(pb[n])

    def _gen_power(self, pb, basis, n) -> bool:
        if n in pb:
            return False
        a, b = split_degree(n)
        rA = self._gen_power(pb, basis, a)
        rB = self._gen_power(pb, basis, b)
        if rA:
            pb[a] = self.rescale(pb[a])
        if rB:
            pb[b] = self.rescale(pb[b])
        pb[n] = self.mul_relin(pb[a], pb[b])
        if basis == CHEBYSHEV:
            c = abs(a - b)
            pb[n] = self.add_ct(pb[n], pb[n])
            if c == 0:
                pb[n] = self.add_const(pb[n], -1)
            else:
                self.gen_power(pb, basis, c)
                pb[n] = self.add_ct(pb[n], pb[c], sub=True)
        return True

    # ---- polynomial_evaluator.go ---------------------------------------------------------------------------------
    def baby_step(self, pol: Poly, pb, targetLevel, targetScale) -> Ct:     # EvaluatePolynomialVectorFromPowerBasis :254-359
        even, odd = pol.IsEven, pol.IsOdd
        minDeg = len(pol.Coeffs) - 1
        if even and not odd:
            minDeg -= 1
        maxCtDeg = 0
        for i in range(pol.Degree(), 0, -1):
            if i in pb:
                maxCtDeg = max(maxCtDeg, pb[i].Degree())
        N = self.params.N()
        if minDeg == 0:
            res = Ct([np.zeros((targetLevel + 1, N), dtype=U64) for _ in range(2)], targetScale)
            if even:
                res = self.add_const(res, self._coeff(pol, 0))
            return res
        res = Ct([np.zeros((targetLevel + 1, N), dtype=U64) for _ in range(maxCtDeg + 1)], targetScale)
        if even:
            res = self.add_const(res, self._coeff(pol, 0))
        for key in range(pol.Degree(), 0, -1):
            if (not (even or odd)) or (key & 1 == 0 and even) or (key & 1 == 1 and odd):
                res = self.mul_then_add(pb[key], self._coeff(pol, key), res)
        return res

    @staticmethod
    def _coeff(pol, k):
        c = pol.Coeffs[k]
        if c is None:
            raise ValueError("nil coefficient %d (the reference dereferences it)" % k)
        return c

    def evaluate_monomial(self, a: Ct, b: Ct, xpow: Ct) -> Ct:      # :226-251
        if b.Degree() == 2:
            b = self.relinearize(b)
        b = self.rescale(b)
        b = self.mul_tensor(b, xpow)
        if not in_delta(a.Scale, b.Scale, SCALE_PREC - 12):
            raise ValueError("evalMonomial: scale discrepency")
        return self.add_ct(b, a)

    def Evaluate(self, ct: Ct, p: Poly, targetScale) -> Ct:
        targetScale = Fraction(targetScale)
        if p.Degree() < 1:
            raise ValueError("the polynomial must have degree >= 1")
        pb = {1: Ct([v.copy() for v in ct.Value], ct.Scale)}
        if pb[1].Level() < self.lpr * p.Depth():
            raise ValueError("%d levels < %d log(d) -> cannot evaluate poly" % (pb[1].Level(), self.lpr * p.Depth()))
        logDegree = p.Degree().bit_length()
        logSplit = optimal_split(logDegree)
        odd, even = p.IsOdd, p.IsEven
        self.gen_power(pb, p.Basis, 1 << (logDegree - 1))
        for i in range((1 << logSplit) - 1, 2, -1):
            if (not (even or odd)) or (i & 1 == 0 and even) or (i & 1 == 1 and odd):
                self.gen_power(pb, p.Basis, i)
        ps = paterson_stockmeyer(p, self.Q, self.lpr, pb[1].Level(), pb[1].Scale, targetScale)
        # EvaluatePatersonStockmeyerPolynomialVector :101-161
        split = len(ps)
        babySteps: List[Optional[list]] = [None] * split
        for i in range(split):
            bs = ps[i]
            babySteps[split - i - 1] = [bs.Degree(), self.baby_step(bs, pb, bs.Level, bs.Scale)]
        while len(babySteps) != 1:
            giant = [0] * len(babySteps)
            i = 0
            while i < len(babySteps):
                if i == len(babySteps) - 1:
                    giant[i] = 2
                elif babySteps[i][0] == babySteps[i + 1][0]:
                    giant[i] = 1
                    i += 1
                i += 1
            i = 0
            while i < len(babySteps):                                      # EvaluateGiantStep :193-223
                if giant[i] == 2:
                    babySteps[i][0] = babySteps[i - 1][0]
                elif giant[i] == 1:
                    ev_, od_ = babySteps[i], babySteps[i + 1]
                    deg = 1 << ev_[0].bit_length()
                    od_[1] = self.evaluate_monomial(ev_[1], od_[1], pb[deg])
                    od_[0] = 2 * deg - 1
                    babySteps[i] = None
                    i += 1
                i += 1
            babySteps = [b for b in babySteps if b is not None]
        res = babySteps[0][1]
        if res.Degree() == 2:
            res = self.relinearize(res)
        return self.rescale(res)

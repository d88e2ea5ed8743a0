"""Literal restatement of bgv polynomial.Evaluator.Evaluate (circuits/bgv/polynomial/polynomial_evaluator.go:38-51) op by op, on the
BGV / BFV evaluator of tests/bgv_oracle.py (TEST INFRASTRUCTURE ONLY; lattigo_b200/bgv_polyeval.py is the product's planner and does
not import this module). The scheme-independent control flow (power basis, Paterson-Stockmeyer, baby and giant steps) is
oracle/polyeval.py's PolyEvaluator; this subclass replaces its scheme operations with schemes/bgv/evaluator.go's:
  Add / Sub (ct, ct) with evaluateInPlace or matchScaleThenEvaluateInPlace + matchScalesBinary   :122-244, :1569-1615
  Add (ct, uint64): c scale mod T, centred, times tInvModQ[level], AddScalarBigint                 :142-172
  MulThenAdd (ct, uint64) with the op0.Scale / opOut.Scale ratio                                  :1088-1141
  Mul / MulRelinNew dispatching on ScaleInvariant (tensorStandard / tensorScaleInvariant)          :391-396, :529-532, :592-667, :898-989
  Rescale (DivRoundByLastModulusNTT; nothing for the scale-invariant evaluator)                    :1363-1393
and the simEvaluator with circuits/bgv/polynomial/polynomial_evaluator_sim.go's. Scales are rlwe.Scale with Mod = T: Python ints,
Mul and Div mod T (core/rlwe/scale.go:77-119), Cmp on the values."""
from __future__ import annotations

from math import gcd
from typing import List, Optional

import numpy as np

from oracle import oracle as O
from oracle import polyeval as P
from tests import bgv_oracle as B

U64 = np.uint64
MONOMIAL, CHEBYSHEV = P.MONOMIAL, P.CHEBYSHEV


def scale_mul(a: int, b: int, t: int) -> int:
    return int(a) * int(b) % t


def scale_div(a: int, b: int, t: int) -> int:
    try:
        inv = pow(int(b), -1, t)
    except ValueError:                 # big.Int.ModInverse leaves the receiver (b) unchanged
        inv = int(b)
    return int(a) * inv % t


def modulus_at_level(Q, level):
    out = 1
    for q in Q[: level + 1]:
        out *= int(q)
    return out


def mul_scale_invariant(Q, t, a, b, level):      # evaluator.go:983-989
    c = scale_mul(a, b, t)
    return scale_div(c, t - modulus_at_level(Q, level) % t, t)


def match_scales_binary(scale0: int, scale1: int, t: int):      # evaluator.go:1569-1615
    tHalf = t >> 1
    center = lambda x: t - x if x >= tHalf else x
    if gcd(scale0, t) != 1:
        raise ValueError("cannot matchScalesBinary: invalid ciphertext scale: gcd(scale, t) != 1")
    a, b = t, 0
    A, Bv = pow(scale0, t - 2, t) * scale1 % t, 1
    r0, r1 = A, Bv
    e = center(A) + 1
    while A != 0:
        q = a // A
        a, A = A, a % A
        b, Bv = Bv, (t + b - Bv * q % t) % t
        if A != 0 and gcd(A, t) == 1:
            tmp = center(A) + center(Bv)
            if tmp < e:
                e = tmp
                r0, r1 = A, Bv
    return r0, r1, e


def new_polynomial(coeffs, is_odd=True, is_even=True, basis=MONOMIAL) -> P.Poly:
    """bignum.NewPolynomial(basis, []uint64, nil): exact big.Floats (SetUint64)."""
    return P.Poly([(P.BF(int(c), 64), P.BF(0, 64)) for c in coeffs], basis, is_odd, is_even)


class SimEval:                                    # circuits/bgv/polynomial/polynomial_evaluator_sim.go
    def __init__(self, Q, t, invariant):
        self.Q, self.t, self.inv = [int(q) for q in Q], t, invariant

    def PolynomialDepth(self, degree):
        if self.inv:
            return 0
        if degree <= 0:
            raise ValueError("invalid degree")
        return degree.bit_length() - 1

    def Rescale(self, op):
        if not self.inv:
            op.Scale = scale_div(op.Scale, self.Q[op.Level], self.t)
            op.Level -= 1

    def MulNew(self, a, b):
        lv = min(a.Level, b.Level)
        s = mul_scale_invariant(self.Q, self.t, a.Scale, b.Scale, lv) if self.inv else scale_mul(a.Scale, b.Scale, self.t)
        return P.SimOp(lv, s)

    def UpdateLevelAndScaleBabyStep(self, lead, tLevelOld, tScaleOld):
        if not self.inv and lead:
            return tLevelOld, scale_mul(tScaleOld, self.Q[tLevelOld], self.t)
        return tLevelOld, tScaleOld

    def UpdateLevelAndScaleGiantStep(self, lead, tLevelOld, tScaleOld, xPowScale):
        s = scale_div(tScaleOld, xPowScale, self.t)
        if not self.inv:
            s = scale_mul(s, self.Q[tLevelOld] if lead else self.Q[tLevelOld + 1], self.t)
            return tLevelOld + 1, s
        return tLevelOld, scale_mul(s, self.t - modulus_at_level(self.Q, tLevelOld) % self.t, self.t)


class Evaluator(B.BGVEvaluator):
    """bgv.Evaluator with Mul (no relinearization) for both tensorings."""

    def MulNew(self, op0, op1):
        level = min(op0[0].shape[0], op1[0].shape[0]) - 1
        if self.ScaleInvariant:
            lm = self.levelQMul[level]
            square = op0 is op1
            t0 = self.modUpAndNTT(level, lm, op0)
            t1 = t0 if square else self.modUpAndNTT(level, lm, op1)
            cQ, cM = self.tensorLowDeg(level, lm, op0, op1, t0, t1, square)
            for k in range(3):
                self.quantize(level, lm, cQ[k], cM[k])
            return cQ
        ring = self.params.ringQ.AtLevel(level)
        c00, c01 = self._new(ring, level), self._new(ring, level)
        c = [self._new(ring, level) for _ in range(3)]
        ring.MulRNSScalarMontgomery(op0[0], self.tMontgomery, c00)
        ring.MulRNSScalarMontgomery(op0[1], self.tMontgomery, c01)
        ring.MulCoeffsMontgomery(c00, op1[0], c[0])
        ring.MulCoeffsMontgomery(c01, op1[1], c[2])
        ring.MulCoeffsMontgomery(c00, op1[1], c[1])
        ring.MulCoeffsMontgomeryThenAdd(c01, op1[0], c[1])
        return c


class PolyEvaluator(P.PolyEvaluator):
    """polynomial.Evaluator[uint64] over bgv.Evaluator; invariant = InvariantTensoring = the evaluator's ScaleInvariant."""

    def __init__(self, params: O.Parameters, rlk: O.GadgetCiphertext, t: int, qmul, invariant: bool):
        self.params, self.rlk, self.lpr, self.prec = params, rlk, 1, 64
        self.t, self.inv = int(t), bool(invariant)
        self.ev = Evaluator(params, t, qmul, rlk, invariant)
        self.Q = [int(q) for q in params.qi]
        self.counts = {"matchScalesBinary": 0}

    def _ct(self, value, scale): return P.Ct(value, int(scale))

    # ---- schemes/bgv/evaluator.go -------------------------------------------------------------------------------
    def add_const(self, op0: P.Ct, c, sub=False) -> P.Ct:          # Add (ct, uint64) :142-172
        if sub:
            raise NotImplementedError("Sub with a scalar is not on the monomial path")
        level = op0.Level()
        v = int(c[0].v) * int(op0.Scale) % self.t
        if v > self.t >> 1:
            v -= self.t
        v *= pow(self.t, -1, modulus_at_level(self.Q, level))
        out = [x.copy() for x in op0.Value]
        self._ring(level).AddScalarBigint(op0.Value[0], v, out[0])
        return self._ct(out, op0.Scale)

    def add_ct(self, c0: P.Ct, c1: P.Ct, sub=False) -> P.Ct:        # Add / Sub (ct, ct) with opOut == c0 :122-244
        level = min(c0.Level(), c1.Level())
        ring = self._ring(level)
        N = self.params.N()
        deg = max(c0.Degree(), c1.Degree())
        out = [np.zeros((level + 1, N), dtype=U64) for _ in range(deg + 1)]
        if int(c0.Scale) == int(c1.Scale):                           # evaluateInPlace
            small, large = (c0, c1) if c0.Degree() <= c1.Degree() else (c1, c0)
            for i in range(small.Degree() + 1):
                (ring.Sub if sub else ring.Add)(c0.Value[i], c1.Value[i], out[i])
            for i in range(small.Degree() + 1, deg + 1):
                out[i][:] = large.Value[i][: level + 1]
            return self._ct(out, max(int(c0.Scale), int(c1.Scale)))
        self.counts["matchScalesBinary"] += 1                        # matchScaleThenEvaluateInPlace
        r0, r1, _ = match_scales_binary(int(c0.Scale), int(c1.Scale), self.t)
        for i in range(c0.Degree() + 1):
            ring.MulScalar(c0.Value[i], r0, out[i])
        for i in range(c1.Degree() + 1):
            (ring.MulScalarThenSub if sub else ring.MulScalarThenAdd)(c1.Value[i], r1, out[i])
        return self._ct(out, scale_mul(c0.Scale, r0, self.t))

    def mul_relin(self, a: P.Ct, b: P.Ct) -> P.Ct:                   # MulRelinNew
        level = min(a.Level(), b.Level())
        v = self.ev.MulRelinNew(a.Value, a.Value if a is b else b.Value)
        return self._ct(v, self._mul_scale(a.Scale, b.Scale, level))

    def mul_tensor(self, op0: P.Ct, op1: P.Ct) -> P.Ct:              # Mul (ct x ct, relin = false)
        level = min(op0.Level(), op1.Level())
        if op0.Degree() == 0:
            if self.inv:                                              # tensorScaleInvariant reads ct0.Value[1]
                raise IndexError("index out of range [1] with length 1")
            # tensorStandard's plaintext branch (:668-681): opOut keeps op0's degree 0 and reads op1.Value[0] only
            ring = self._ring(level)
            c00, out = np.empty((level + 1, self.params.N()), dtype=U64), np.empty((level + 1, self.params.N()), dtype=U64)
            ring.MulRNSScalarMontgomery(op1.Value[0], self.ev.tMontgomery, c00)
            ring.MulCoeffsMontgomery(op0.Value[0], c00, out)
            return self._ct([out], self._mul_scale(op0.Scale, op1.Scale, level))
        return self._ct(self.ev.MulNew(op0.Value, op1.Value), self._mul_scale(op0.Scale, op1.Scale, level))

    def _mul_scale(self, a, b, level):
        return mul_scale_invariant(self.Q, self.t, a, b, level) if self.inv else scale_mul(a, b, self.t)

    def rescale(self, ct: P.Ct) -> P.Ct:                             # Rescale :1363-1393
        if self.inv:
            return self._ct([v.copy() for v in ct.Value], ct.Scale)
        if ct.Level() == 0:
            raise ValueError("cannot rescale: op0 already at level 0")
        return self._ct(self.ev.Rescale(ct.Value), scale_div(ct.Scale, self.Q[ct.Level()], self.t))

    def mul_then_add(self, op0: P.Ct, c, opOut: P.Ct) -> P.Ct:       # MulThenAdd (ct, uint64) :1088-1141
        level = min(op0.Level(), opOut.Level())
        v = int(c[0].v)
        if int(op0.Scale) != int(opOut.Scale):
            v *= pow(int(op0.Scale), self.t - 2, self.t) * int(opOut.Scale) % self.t
        v %= self.t
        if v > self.t >> 1:
            v -= self.t
        out = [x.copy() for x in opOut.Value]
        ring = self._ring(level)
        for i in range(op0.Degree() + 1):
            ring.MulScalarBigintThenAdd(op0.Value[i], v, out[i])
        return self._ct(out, opOut.Scale)

    # ---- circuits/common/polynomial/polynomial_evaluator.go:29-161 with the BGV simEvaluator ---------------------
    def Evaluate(self, ct: P.Ct, p: P.Poly, targetScale) -> P.Ct:
        if p.Basis != MONOMIAL:
            raise ValueError("the Chebyshev basis is not supported for BGV polynomial evaluation (uint64 coefficients)")
        targetScale = int(targetScale)
        if p.Degree() < 1:
            raise ValueError("the polynomial must have degree >= 1")
        pb = {1: self._ct([v.copy() for v in ct.Value], ct.Scale)}
        if pb[1].Level() < p.Depth():
            raise ValueError("%d levels < %d log(d) -> cannot evaluate poly" % (pb[1].Level(), p.Depth()))
        logDegree = p.Degree().bit_length()
        logSplit = P.optimal_split(logDegree)
        odd, even = p.IsOdd, p.IsEven
        self.gen_power(pb, p.Basis, 1 << (logDegree - 1))
        for i in range((1 << logSplit) - 1, 2, -1):
            if (not (even or odd)) or (i & 1 == 0 and even) or (i & 1 == 1 and odd):
                self.gen_power(pb, p.Basis, i)
        # PatersonStockmeyerPolynomial (polynomial.go:74-106)
        sim = SimEval(self.Q, self.t, self.inv)
        spb = {1: P.SimOp(pb[1].Level(), int(pb[1].Scale))}
        P.sim_gen_power(spb, 1 << logDegree, sim)
        for i in range((1 << logSplit) - 1, 2, -1):
            P.sim_gen_power(spb, i, sim)
        ps, _ = P.recurse_ps(logSplit, pb[1].Level() - sim.PolynomialDepth(p.Degree()), p, spb, targetScale, sim)
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
            while i < len(babySteps):
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

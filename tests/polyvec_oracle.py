"""Literal restatement of polynomial.Evaluator.Evaluate on a PolynomialVector with a Mapping, op by op, for CKKS (on oracle/polyeval.py's
PolyEvaluator) and BGV / BFV (on tests/bgv_polyeval_oracle.py's). TEST INFRASTRUCTURE ONLY: lattigo_b200/polyeval.py and bgv_polyeval.py
are the product's planners and do not import this module.
  circuits/common/polynomial/polynomial_evaluator.go:29-91    Evaluate: power basis from Value[0] with the odd / even flags OR-ed
  circuits/common/polynomial/polynomial.go:165-260            NewPolynomialVector, IsOdd / IsEven (AND-ed), PatersonStockmeyerPolynomial
  circuits/common/polynomial/polynomial_evaluator.go:254-320  EvaluatePolynomialVectorFromPowerBasis with a mapping
  circuits/{ckks,bgv}/polynomial/polynomial_evaluator.go      GetVectorCoefficient (nil / 0 in unmapped slots)
  schemes/ckks/evaluator.go:88-109, :977-1025, :1081-1170     Add(ct, vector), MulThenAdd(ct, vector, ct), mulRelinThenAdd (degree 0)
  schemes/bgv/evaluator.go:180-205, :1148-1180, :1230-1350    the same for BGV, with matchScalesBinary
Slot vectors are encoded with the oracle encoders (oracle/encoder.py embed_double at scale.Float64(), oracle/bgv_encoder.py Encode)."""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from oracle import bgv_encoder as OE
from oracle import encoder as E
from oracle import polyeval as P
from tests import bgv_polyeval_oracle as BP

U64 = np.uint64


def new_polynomial_vector(polys: List[P.Poly], mapping):
    """NewPolynomialVector (polynomial.go:165-195)."""
    maxDeg = max(p.Degree() for p in polys)
    basis = polys[-1].Basis
    for p in polys:
        if basis != p.Basis:
            raise ValueError("polynomial basis must be the same for all polynomials in a polynomial vector")
        if maxDeg != p.Degree():
            raise ValueError("polynomial degree must all be the same")
    return polys, mapping


class _VectorEvaluate:
    """The scheme-independent Evaluate of a PolynomialVector with a Mapping; the scheme supplies _ps, max_slots, vector_coefficient,
    add_vector and mul_then_add_vector."""

    def EvaluateVector(self, ct: P.Ct, polys: List[P.Poly], mapping, targetScale):
        p = polys[0]
        if p.Degree() < 1:
            raise ValueError("the polynomial must have degree >= 1")
        pb = {1: self._ct([v.copy() for v in ct.Value], ct.Scale)}
        if pb[1].Level() < self.lpr * p.Depth():
            raise ValueError("%d levels < %d log(d) -> cannot evaluate poly" % (pb[1].Level(), self.lpr * p.Depth()))
        logDegree = p.Degree().bit_length()
        logSplit = P.optimal_split(logDegree)
        odd = any(q.IsOdd for q in polys)
        even = any(q.IsEven for q in polys)
        self.gen_power(pb, p.Basis, 1 << (logDegree - 1))
        for i in range((1 << logSplit) - 1, 2, -1):
            if (not (even or odd)) or (i & 1 == 0 and even) or (i & 1 == 1 and odd):
                self.gen_power(pb, p.Basis, i)
        pss = [self._ps(q, pb[1].Level(), pb[1].Scale, targetScale) for q in polys]
        split = len(pss[0])
        babySteps: List[Optional[list]] = [None] * split
        for i in range(split):                                           # EvaluateBabyStep: the transposed vector, Value[0]'s level / scale
            bs = pss[0][i]
            babySteps[split - i - 1] = [bs.Degree(), self.baby_step_vector([s[i] for s in pss], mapping, pb, bs.Level, bs.Scale)]
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

    def baby_step_vector(self, pols, mapping, pb, targetLevel, targetScale):     # polynomial_evaluator.go:254-320, mapping != nil
        even, odd = all(q.IsEven for q in pols), all(q.IsOdd for q in pols)
        minDeg = len(pols[0].Coeffs) - 1
        if even and not odd:
            minDeg -= 1
        maxCtDeg = 0
        for i in range(pols[0].Degree(), 0, -1):
            if i in pb:
                maxCtDeg = max(maxCtDeg, pb[i].Degree())
        N = self.params.N()
        deg = 1 if minDeg == 0 else maxCtDeg
        res = self._ct([np.zeros((targetLevel + 1, N), dtype=U64) for _ in range(deg + 1)], targetScale)
        if even:
            res = self.add_vector(res, self.vector_coefficient(pols, mapping, 0))
        if minDeg == 0:
            return res
        for key in range(pols[0].Degree(), 0, -1):
            if (not (even or odd)) or (key & 1 == 0 and even) or (key & 1 == 1 and odd):
                res = self.mul_then_add_vector(pb[key], self.vector_coefficient(pols, mapping, key), res)
        return res


class CKKSPolyVectorEvaluator(_VectorEvaluate, P.PolyEvaluator):
    def _ct(self, value, scale): return P.Ct(value, scale)

    def _ps(self, q, level, scale, target):
        return P.paterson_stockmeyer(q, self.Q, self.lpr, level, scale, target)

    def max_slots(self): return self.params.N() // 2

    def vector_coefficient(self, pols, mapping, k):
        values = [None] * self.max_slots()
        for i, p in enumerate(pols):
            for j in mapping.get(i, ()):
                values[j] = p.Coeffs[k]
        return [0j if c is None else complex(float(c[0].v), float(c[1].v)) for c in values]     # Embed: Complex128(), nil -> 0

    def encode(self, values, level, scale):
        """Encoder.Encode at pt.Scale (prec <= 53: Scale.Float64()), NTT, not Montgomery."""
        logN = self.params.N().bit_length() - 1
        pt, _ = E.embed_double(self.params.ringQ, None, values, logN - 1, float(scale), True, False, level)
        return pt

    def add_vector(self, op0: P.Ct, values) -> P.Ct:                 # Add(op0, vector, op0)
        level = op0.Level()
        pt = self.encode(values, level, op0.Scale)
        out = [v.copy() for v in op0.Value]
        self._ring(level).Add(op0.Value[0], pt, out[0])               # evaluateInPlace: equal scales, degree 0 + degree d
        return P.Ct(out, op0.Scale)

    def mul_then_add_vector(self, op0: P.Ct, values, opOut: P.Ct) -> P.Ct:
        level = min(op0.Level(), opOut.Level())
        cmp = (op0.Scale > opOut.Scale) - (op0.Scale < opOut.Scale)
        if cmp == 0:
            scaleRLWE = P.new_scale(self.Q[level])
            for i in range(1, self.lpr):
                scaleRLWE = P.scale_mul(scaleRLWE, P.new_scale(self.Q[level - i]))
            opOut = self.mul_scalar(opOut, P.trunc(scaleRLWE))
            opOut.Scale = P.scale_mul(opOut.Scale, scaleRLWE)
        elif cmp == -1:
            scaleRLWE = P.scale_div(opOut.Scale, op0.Scale)
        else:
            raise ValueError("cannot MulThenAdd: op0.Scale > opOut.Scale is not supported")
        pt = self.encode(values, level, scaleRLWE)
        # MulThenAdd(op0, pt, opOut): InitOutputBinaryOp and Resize to min(op0, pt, opOut) levels, then mulRelinThenAdd
        opOut = P.Ct([v[: level + 1] for v in opOut.Value], opOut.Scale)
        resScale = P.scale_mul(op0.Scale, scaleRLWE)
        if opOut.Scale < resScale:
            ratio = P.scale_div(resScale, opOut.Scale)
            if float(ratio) >= 2.0:
                opOut = self.mul_scalar(opOut, (P.BF(ratio, P.SCALE_PREC), P.BF(0, P.SCALE_PREC)))
                opOut.Scale = resScale
        ring = self._ring(level)
        c00 = np.empty_like(pt)
        ring.MForm(pt, c00)
        out = [v.copy() for v in opOut.Value]
        for i in range(op0.Degree() + 1):
            ring.MulCoeffsMontgomeryThenAdd(op0.Value[i][: level + 1], c00, out[i])
        return P.Ct(out, opOut.Scale)


class BGVPolyVectorEvaluator(_VectorEvaluate, BP.PolyEvaluator):
    def __init__(self, params, rlk, t, qmul, invariant):
        super().__init__(params, rlk, t, qmul, invariant)
        self.enc = OE.BGVEncoder(params.ringQ, self.t)
        self.counts["vector_matchScalesBinary"] = 0

    def _ps(self, q, level, scale, target):
        logDegree = q.Degree().bit_length()
        logSplit = P.optimal_split(logDegree)
        sim = BP.SimEval(self.Q, self.t, self.inv)
        spb = {1: P.SimOp(level, int(scale))}
        P.sim_gen_power(spb, 1 << logDegree, sim)
        for i in range((1 << logSplit) - 1, 2, -1):
            P.sim_gen_power(spb, i, sim)
        ps, _ = P.recurse_ps(logSplit, level - sim.PolynomialDepth(q.Degree()), q, spb, int(target), sim)
        return ps

    def vector_coefficient(self, pols, mapping, k):
        values = [0] * self.enc.MaxSlots()
        for i, p in enumerate(pols):
            for j in mapping.get(i, ()):
                if p.Coeffs[k] is None:
                    raise ValueError("nil coefficient %d (the reference dereferences it)" % k)
                values[j] = int(p.Coeffs[k][0].v)                       # Coeffs[k].Uint64()
        return values

    def add_vector(self, op0: P.Ct, values) -> P.Ct:                 # Add(op0, []uint64, op0): pt at op0's scale
        level = op0.Level()
        pt = np.array(self.enc.Encode(values, False, int(op0.Scale), True, False, level), dtype=U64)
        out = [v.copy() for v in op0.Value]
        self._ring(level).Add(op0.Value[0], pt, out[0])
        return self._ct(out, op0.Scale)

    def mul_then_add_vector(self, op0: P.Ct, values, opOut: P.Ct) -> P.Ct:
        level = min(op0.Level(), opOut.Level())
        if int(op0.Scale) != int(opOut.Scale):
            pt_scale = pow(int(op0.Scale), self.t - 2, self.t) * int(opOut.Scale) % self.t
        else:
            pt_scale = 1
        pt = np.array(self.enc.Encode(values, False, pt_scale, True, False, level), dtype=U64)
        opOut = self._ct([v[: level + 1] for v in opOut.Value], opOut.Scale)      # InitOutputBinaryOp + Resize
        ring = self._ring(level)
        c00 = np.empty_like(pt)
        ring.MulRNSScalarMontgomery(pt, self.ev.tMontgomery, c00)
        out = [v.copy() for v in opOut.Value]
        scale = int(opOut.Scale)
        r0 = 1
        target = int(op0.Scale) * pt_scale % self.t
        if target != scale:
            self.counts["vector_matchScalesBinary"] += 1
            r0, r1, _ = BP.match_scales_binary(target, scale, self.t)
            for v in out:
                ring.MulScalar(v, r1, v)
            scale = scale * r1 % self.t
        if r0 != 1:
            ring.MulScalar(c00, r0, c00)
        for i in range(op0.Degree() + 1):
            ring.MulCoeffsMontgomeryThenAdd(op0.Value[i][: level + 1], c00, out[i])
        return self._ct(out, scale)

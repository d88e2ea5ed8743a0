"""bgv polynomial.Evaluator.Evaluate (circuits/bgv/polynomial/polynomial_evaluator.go:38-51) on the device: one bignum.Polynomial in the
monomial basis with uint64 coefficients (Lead = true, Lazy = false), a batch of degree-1 NTT-domain ciphertexts sharing one level and
scale, for the BGV evaluator (InvariantTensoring = false) or the BFV one (InvariantTensoring = true, the evaluator's ScaleInvariant).

The scheme-independent planning (power basis, SplitDegree, OptimalSplit, Factorize, the Paterson-Stockmeyer recursion, the giant-step
loop, the program format) is lattigo_b200/polyeval.py's; this module adds the BGV parts:
  - the BGV simEvaluator (polynomial_evaluator_sim.go): PolynomialDepth, Rescale, MulNew and the baby / giant step updates in both
    tensoring modes, including -Q_level mod t for BFV;
  - rlwe.Scale with Mod = t (core/rlwe/scale.go:77-119): Mul and Div are exact mod t, Cmp compares the values; here Python ints;
  - the schemes/bgv rules folded into the LINCOMB weights: Add(res, c0) as c0 scale mod t, centred, times tInvModQ[level]
    (evaluator.go:142-172), and MulThenAdd(X^k, c, res) with the op0.Scale / opOut.Scale ratio mod t, centred (:1088-1141);
  - Mul / MulRelin dispatching on ScaleInvariant (:391-396, :529-532, MulScaleInvariant :983-989) and Rescale, a no-op for BFV
    (:1363-1393).
EvaluateMonomial checks a.Scale.InDelta(b.Scale, ScalePrecision - 12) before its Add. Scales mod t are integers below 2^64, so that
check passes only when they are equal, and the Add never reaches matchScalesBinary: every TENSOR has r_b = r_a = 1."""
from __future__ import annotations

import ctypes
from math import gcd
from typing import Sequence

import numpy as np

from . import _lib
from .polyeval import (CHEBYSHEV, MONOMIAL, MULRELIN, RESCALE, TENSOR, Polynomial, PolynomialVector, PreparedVector, Program, _check_vector,
                       _Evaluator, _Lin, _Planner, _Poly, _pt_block, _Sim, _Sym, _VLin)
from .ring import _stream

U64_MAX = (1 << 64) - 1


class ScaleModT:
    """rlwe.Scale with Mod = t on integer values (core/rlwe/scale.go:77-119)."""

    def __init__(self, t: int):
        self.t = t

    def mul(self, a: int, b: int) -> int:
        return a * b % self.t

    def div(self, a: int, b: int) -> int:
        try:
            inv = pow(b, -1, self.t)
        except ValueError:                       # big.Int.ModInverse leaves its receiver unchanged when there is no inverse
            inv = b
        return a * inv % self.t


def q_mod_t_neg(Q: Sequence[int], level: int, t: int) -> int:
    """T - (ModulusAtLevel[level] mod T), the factor of MulScaleInvariant and of the BFV giant step."""
    prod = 1
    for q in Q[: level + 1]:
        prod *= q
    return t - prod % t


def centred(c: int, t: int) -> int:
    """c mod T (Euclidean), minus T above T/2 (the scalar cases of Add / Mul / MulThenAdd)."""
    c %= t
    return c - t if c > t >> 1 else c


def match_scales_binary(scale0: int, scale1: int, t: int):
    """Evaluator.matchScalesBinary (schemes/bgv/evaluator.go:1569-1615): (r0, r1) with scale0 r0 = scale1 r1 mod t and small centred
    r0 + r1."""
    tHalf = t >> 1
    center = lambda x: t - x if x >= tHalf else x
    if gcd(scale0, t) != 1:
        raise ValueError("cannot matchScalesBinary: invalid ciphertext scale: gcd(scale, t) != 1")
    a, b = t, 0
    A, B = pow(scale0, t - 2, t) * scale1 % t, 1
    r0, r1 = A, B
    e = center(A) + 1
    while A != 0:
        q = a // A
        a, A = A, a % A
        b, B = B, (t + b - B * q % t) % t
        if A != 0 and gcd(A, t) == 1:
            tmp = center(A) + center(B)
            if tmp < e:
                e = tmp
                r0, r1 = A, B
    return r0, r1


class _BGVSim(_Sim):                              # circuits/bgv/polynomial/polynomial_evaluator_sim.go
    def __init__(self, Q, t, si):
        super().__init__(Q, 1)
        self.t, self.si, self.S = t, si, ScaleModT(t)

    def depth(self, degree):
        if self.si:
            return 0
        if degree <= 0:
            raise ValueError("invalid degree: degree=%d should be greater than zero" % degree)
        return degree.bit_length() - 1

    def rescale(self, lv, s):
        if self.si:
            return lv, s
        return lv - 1, self.S.div(s, self.Q[lv])

    def mul(self, a, b):
        lv = min(a[0], b[0])
        s = self.S.mul(a[1], b[1])
        return lv, self.S.div(s, q_mod_t_neg(self.Q, lv, self.t)) if self.si else s

    def same_scale(self, a, b):                  # InDelta(.., 116) on integers below 2^64 is equality
        return a == b

    def baby(self, lead, lv, s):
        if not self.si and lead:
            s = self.S.mul(s, self.Q[lv])
        return lv, s

    def giant(self, lead, lv, s, xs):
        s = self.S.div(s, xs)
        if self.si:
            return lv, self.S.mul(s, q_mod_t_neg(self.Q, lv, self.t))
        return lv + 1, self.S.mul(s, self.Q[lv] if lead else self.Q[lv + 1])


class _BGVPlanner(_Planner):
    def __init__(self, Q, t, si, max_slots=0):
        super().__init__(Q, 1, 64, None, max_slots)
        self.t, self.si = t, si
        self.sim = _BGVSim(self.Q, t, si)

    def _sim(self):
        return self.sim

    # ---- rounding ops --------------------------------------------------------------------------------------------
    def rescale(self, x: _Sym) -> _Sym:          # Rescale (:1363-1393): DivRoundByLastModulusNTT, or nothing for BFV
        if self.si:
            return x
        if x.level == 0:
            raise ValueError("cannot rescale: op0 already at level 0")
        y = _Sym(self._slot(), x.level - 1, self.sim.S.div(x.scale, self.Q[x.level]), x.deg)
        self.prog.ops.append(dict(kind=RESCALE, dst=y.slot, src0=x.slot, level=y.level))
        return y

    def mul_relin(self, a: _Sym, b: _Sym) -> _Sym:
        lv, s = self.sim.mul((a.level, a.scale), (b.level, b.scale))
        y = _Sym(self._slot(), lv, s, 1)
        self.prog.ops.append(dict(kind=MULRELIN, dst=y.slot, src0=a.slot, src1=b.slot, level=lv))
        return y

    @staticmethod
    def _degree0_check(even, odd, degree):
        if even and not odd and degree == 0:
            # NewCiphertext(params, 0, level): Mul(b, X^k) then takes the plaintext branch of tensorStandard, which reads X^k's first
            # component only (BGV), and tensorScaleInvariant indexes a second component that is not there (BFV)
            raise ValueError("an even-only polynomial whose giant-step quotient is a constant gives a degree-0 baby step, which the "
                             "reference's Mul does not multiply as a ciphertext; not supported")

    def baby_step(self, pol, pb, level, scale) -> _Lin:
        self._degree0_check(pol.IsEven, pol.IsOdd, pol.Degree())
        return super().baby_step(pol, pb, level, scale)

    def vec_baby_step(self, pols, pb, level, scale, mapping) -> _VLin:
        self._degree0_check(all(p.IsEven for p in pols), all(p.IsOdd for p in pols), pols[0].Degree())
        return super().vec_baby_step(pols, pb, level, scale, mapping)

    # ---- schemes/bgv vector ops: Add(res, []uint64) and MulThenAdd(X^k, []uint64, res) -------------------------------------
    def vector_coefficient(self, pols, mapping, k):       # CoefficientGetter.GetVectorCoefficient: Coeffs[k].Uint64()
        out = []
        for p in pols:
            if p.Coeffs[k] is None:
                raise ValueError("nil coefficient %d" % k)
            out.append(int(p.Coeffs[k]))
        return out

    def vec_mul_then_add(self, x: _Sym, values, f: _VLin):     # :1148-1180, then mulRelinThenAdd's plaintext branch :1310-1345
        if x.level < f.level:
            raise ValueError("baby step above the level of its power X^k is not supported (MulThenAdd would lower res to X^k's level)")
        t = self.t
        pt_scale = 1 if x.scale == f.scale else pow(x.scale, t - 2, t) * f.scale % t
        r0 = 1
        if x.scale * pt_scale % t != f.scale:       # the scale of op0 (x) pt against opOut's: equal by construction of pt_scale
            r0, r1 = match_scales_binary(x.scale * pt_scale % t, f.scale, t)
            f.scale_by([r1 % q for q in f.Q])
            f.scale = f.scale * r1 % t
        f.w[x.slot] = (self._pt(values, f.level, pt_scale), [t * r0 % q for q in f.Q])      # MRed(pt, tMontgomery), then r0
        f.seq.append(("pt", x.slot))

    def monomial(self, a: _Sym, b: _Sym, x: _Sym) -> _Sym:      # EvaluateMonomial: Mul(b, X^k) + Add(.., a) as one TENSOR
        if b.deg == 2:
            b = self.relin(b)
        b = self.rescale(b)
        lv, bs = self.sim.mul((b.level, b.scale), (x.level, x.scale))
        if not self.sim.same_scale(a.scale, bs):
            raise ValueError("evalMonomial: scale discrepency: (rescale(b) * X^{n}).Scale = %d != a.Scale = %d" % (bs, a.scale))
        lv = min(lv, a.level)
        y = _Sym(self._slot(), lv, bs, 2)
        self.prog.ops.append(dict(kind=TENSOR, dst=y.slot, src0=b.slot, src1=x.slot, addend=a.slot, level=lv, weights=[1] * (2 * (lv + 1))))
        return y

    # ---- schemes/bgv linear ops, folded ----------------------------------------------------------------------
    def add_const(self, f: _Lin, c: int):        # Add(ct, uint64): AddScalarBigint of c scale T^-1 on component 0
        Ql = 1
        for q in self.Q[: f.level + 1]:
            Ql *= q
        v = centred(c * f.scale, self.t) * pow(self.t, -1, Ql)
        for i, q in enumerate(self.Q[: f.level + 1]):
            f.const[i] = [(f.const[i][h] + v) % q for h in range(2)]

    def mul_then_add(self, x: _Sym, c: int, f: _Lin):         # MulThenAdd(X^k, uint64, res): MulScalarBigintThenAdd
        if x.scale != f.scale:
            ratio = pow(x.scale, self.t - 2, self.t) * f.scale % self.t
            c = c * ratio
        v = centred(c, self.t)
        cur = f.w.get(x.slot) or [[0, 0] for _ in range(f.level + 1)]
        # rows above X^k's level are not written (the ring runs at min(op0.Level(), opOut.Level()))
        f.w[x.slot] = [[(cur[i][h] + (v if i <= x.level else 0)) % q for h in range(2)] for i, q in enumerate(self.Q[: f.level + 1])]


def plan(Q: Sequence[int], t: int, level: int, scale: int, coeffs: Sequence[int], target_scale: int, scale_invariant: bool = False,
         odd: bool = True, even: bool = True, basis: int = MONOMIAL) -> Program:
    """The device program of Evaluate(ct, bignum.NewPolynomial(Monomial, coeffs, nil) with IsOdd = odd, IsEven = even, targetScale) for a
    ciphertext at `level` with rlwe.Scale `scale` (Mod = t); scale_invariant is the evaluator's ScaleInvariant (InvariantTensoring)."""
    return plan_vector(Q, t, level, scale, PolynomialVector([Polynomial(coeffs, basis, odd, even)], None), target_scale, scale_invariant)


def plan_vector(Q: Sequence[int], t: int, level: int, scale: int, pv: PolynomialVector, target_scale: int, scale_invariant: bool = False,
                max_slots: int = 0) -> Program:
    """The device program of Evaluate(ct, pv, targetScale) for a PolynomialVector of monomial-basis uint64 polynomials: with a Mapping,
    every baby step in one PTLINCOMB plus program.plaintexts (slot vectors Encode'd at (level, scale), scale mod t); without one, the
    scalar program of Value[0]. max_slots: MaxSlots of the parameters (the length of the slot vectors), needed with a Mapping."""
    p0 = pv.Value[0]
    if p0.basis == CHEBYSHEV:
        raise ValueError("the Chebyshev basis is not supported for BGV polynomial evaluation (uint64 coefficients); use the monomial basis")
    if p0.basis != MONOMIAL:
        raise ValueError("basis must be MONOMIAL")
    polys = []
    for q in pv.Value:
        coeffs = [int(c) for c in q.coeffs]
        if any(c < 0 or c > U64_MAX for c in coeffs):
            raise ValueError("coefficients must be uint64")
        polys.append(_Poly(coeffs, MONOMIAL, q.odd, q.even))
    t = int(t)
    for name, s in (("scale", scale), ("target_scale", target_scale)):
        if not 1 <= int(s) < t:
            raise ValueError("%s must be an integer in [1, t)" % name)
    if polys[0].Degree() > 255:
        raise ValueError("degree %d > 255 is not supported" % polys[0].Degree())
    if pv.Mapping is not None:
        if max_slots < 1:
            raise ValueError("max_slots must be the parameters' MaxSlots (>= 1), got %d" % max_slots)
        _check_vector(pv, max_slots, max_slots)
    return _BGVPlanner(Q, t, bool(scale_invariant), max_slots).evaluate(level, int(scale), polys[0], int(target_scale), polys[1:], pv.Mapping)


class BGVPolynomialEvaluator(_Evaluator):
    """polynomial.Evaluator (circuits/bgv/polynomial) over a BGVEvaluator: InvariantTensoring = bgv_evaluator.ScaleInvariant."""

    def __init__(self, bgv_evaluator):
        self.ev = bgv_evaluator
        self.ctx = bgv_evaluator.ctx
        self.InvariantTensoring = bgv_evaluator.ScaleInvariant
        self.lpr = 1                              # Rescale drops one modulus

    def plan(self, level, scale, coeffs, target_scale, odd=True, even=True, basis=MONOMIAL) -> Program:
        return self.plan_vector(level, scale, PolynomialVector([Polynomial(coeffs, basis, odd, even)], None), target_scale)

    def Evaluate(self, ct, scale, coeffs, target_scale, odd=True, even=True, basis=MONOMIAL):
        """ct: (batch, 2, level+1, N) or (2, level+1, N) int64 CUDA tensor, NTT domain. Returns (ct_out, level, scale)."""
        return self.EvaluateVector(ct, scale, PolynomialVector([Polynomial(coeffs, basis, odd, even)], None), target_scale, None)

    # ---- PolynomialVector (Evaluate with a Mapping) ----------------------------------------------------------------------
    def plan_vector(self, level, scale, pv: PolynomialVector, target_scale) -> Program:
        from .bgv_encoder import plaintext_slots
        return plan_vector(self.ctx.Q, self.ev.t, level, scale, pv, target_scale, self.InvariantTensoring, plaintext_slots(self.ctx.N, self.ev.t))

    def encode_plaintexts(self, prog: Program, encoder):
        """The program's slot vectors, Encode'd with lgpu_bgv_encode (EncodeRingT at the plaintext's scale, RingT2Q with t^-1, NTT): one
        batched call per distinct (level, scale). encoder: a BGVEncoder of the same context and t."""
        import torch
        from .bgv_encoder import ENC_NTT, ENC_SCALE_UP, _vp
        if encoder.t != self.ev.t:
            raise ValueError("the encoder's plaintext modulus differs from the evaluator's")

        def encode_group(values, level, scale, out_ptr, stride):
            v = torch.from_numpy(np.ascontiguousarray(values.view(np.int64))).to("cuda:%d" % self.ctx.device)
            _lib.check(_lib.lib().lgpu_bgv_encode(encoder.h, _vp(v), values.shape[1], ENC_SCALE_UP | ENC_NTT, int(scale), level,
                                                  ctypes.c_void_p(out_ptr), -1, None, values.shape[0], values.shape[1], stride, 0, _stream()))
        return _pt_block(self.ctx, prog, encode_group, np.uint64)

    def PrepareVector(self, level, scale, pv: PolynomialVector, target_scale, encoder) -> PreparedVector:
        """Plans Evaluate(ct, pv, target_scale) for ciphertexts at (level, scale) and encodes its slot vectors on the device."""
        return self._prepare(self.plan_vector(level, scale, pv, target_scale), pv, encoder)

    def EvaluateVector(self, ct, scale, pv: PolynomialVector, target_scale, encoder):
        """Evaluate(ct, PolynomialVector, targetScale) = PrepareVector + RunVector. Returns (ct_out, level, scale)."""
        return self._evaluate(ct, self.PrepareVector(ct.shape[-2] - 1, scale, pv, target_scale, encoder))

    def _call(self, level, ct, batch, prog, pts, out):
        rlk = self.ev.rlk.ref() if self.ev.rlk is not None else None
        si = 1 if self.InvariantTensoring else 0
        if pts is None:
            return _lib.lib().lgpu_bgv_polynomial_evaluate(self.ev.h, level, ct, batch, prog, rlk, si, out, _stream())
        return _lib.lib().lgpu_bgv_polynomial_vector_evaluate(self.ev.h, level, ct, batch, prog, pts, rlk, si, out, _stream())

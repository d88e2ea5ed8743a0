"""ckks polynomial.Evaluator.Evaluate (circuits/ckks/polynomial/polynomial_evaluator.go:42-57) on the device: one bignum.Polynomial
(monomial or Chebyshev basis, Lazy = false), a batch of degree-1 NTT-domain ciphertexts sharing one level and scale.

The host plans, the device runs. plan() restates the reference's control flow and scale bookkeeping
(common/polynomial/polynomial_evaluator.go:29-359, power_basis.go:32-182, polynomial.go:37-153, the CKKS simEvaluator, and the
schemes/ckks Add / Sub / Mul / MulThenAdd scale rules) and emits a program with one op per rounding boundary:
  MULRELIN a, b -> n     MulRelinNew (tensor, GadgetProduct of c2, ModDown, Add)
  TENSOR   b, x [, a]    Mul(b, x) without relinearization, then Add(.., a) with its scale ratio: t = r_b (b (x) x) + r_a a
  RELIN    t             Relinearize
  RESCALE  x             Rescale (DivRoundByLastModulusManyNTT, LevelsConsumedPerRescaling primes)
  LINCOMB                out_i = sum_k W[i,k] X_k (+ w_i0 on component 0), per limb and NTT half
Everything the reference does between two rounding ops (x2, - r T_c, Add(-1), Add(const), the MulThenAdd constants and the
scaleRLWE pre-multiplication, the Add ratios) is linear over the residues with canonical outputs, so it folds into LINCOMB / TENSOR
weights: all baby steps of a call become ONE LINCOMB that reads each power once (DESIGN 3.4).

Scales are rlwe.Scale big.Floats at 128 bits, restated as exact rationals rounded to nearest-even at every operation; coefficient
arithmetic (Factorize) runs at the coefficients' own precision (53 bits: bignum.NewPolynomial from float64 / complex128)."""
from __future__ import annotations

import ctypes
from fractions import Fraction

import numpy as np
from typing import Dict, List, Optional, Sequence

from . import _lib
from .ring import Context, _dptr, _stream

SCALE_PREC = 128
MONOMIAL, CHEBYSHEV = 0, 1
MULRELIN, TENSOR, RELIN, RESCALE, LINCOMB, PTLINCOMB = 0, 1, 2, 3, 4, 5
MAX_TERMS = 16            # LGPU_POLY_MAX_TERMS: powers X^1 .. X^15 for degree <= 255 (OptimalSplit(8) = 4)
MAX_OUTPUTS = 64          # LGPU_POLY_MAX_OUTPUTS


# ---------------------------------------------------------------------------------------------------------------- math/big
def rnd(x, prec: int) -> Fraction:
    """x rounded to `prec` significant bits, ties to even (big.Float's default rounding mode)."""
    x = Fraction(x)
    if x == 0:
        return x
    s = -1 if x < 0 else 1
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    sh = prec - 1 - e
    v = a * (Fraction(2) ** sh)
    n, r = divmod(v.numerator, v.denominator)
    if 2 * r > v.denominator or (2 * r == v.denominator and n & 1):
        n += 1
    return s * Fraction(n) / (Fraction(2) ** sh)


def _smul(a, b): return rnd(a * b, SCALE_PREC)
def _sdiv(a, b): return rnd(Fraction(a) / b, SCALE_PREC)
def _snew(x): return rnd(Fraction(x), SCALE_PREC)


def _in_delta(a, b, log2delta):
    d = abs(a - b)
    return d == 0 or d * (Fraction(2) ** log2delta) <= max(a, b)


class _C:
    """bignum.Complex: real and imaginary big.Floats as (value, precision)."""
    __slots__ = ("re", "im", "prec")

    def __init__(self, re, im, prec):
        self.re, self.im, self.prec = Fraction(re), Fraction(im), prec


def _to_complex(c, prec) -> _C:                  # bignum.ToComplex
    if isinstance(c, int):
        return _C(rnd(c, prec), 0, prec)
    return _C(rnd(c.re, prec), rnd(c.im, prec), prec)


def _rns_scalar(mods, scale, c: _C):             # schemes/ckks/scaling.go:10-43 (rounding half away from zero)
    out = []
    for part in (c.re, c.im):
        p = max(c.prec, SCALE_PREC)
        r = rnd(part * scale, p)
        if part > 0:
            r = rnd(r + Fraction(1, 2), p)
        elif part < 0:
            r = rnd(r - Fraction(1, 2), p)
        v = int(r)
        out.append([v % q for q in mods])
    return out


# ---------------------------------------------------------------------------------------------------------------- polynomials
class _Poly:
    def __init__(self, coeffs, basis, is_odd, is_even):
        self.Coeffs, self.Basis, self.IsOdd, self.IsEven = coeffs, basis, is_odd, is_even
        self.MaxDeg, self.Lead, self.Level, self.Scale = len(coeffs) - 1, True, 0, Fraction(0)

    def Degree(self): return len(self.Coeffs) - 1


def optimal_split(logDegree: int) -> int:       # utils/bignum/polynomial.go:14-23
    logSplit = logDegree >> 1
    a = (1 << logSplit) + (1 << (logDegree - logSplit)) + logDegree - logSplit - 3
    b = (1 << (logSplit + 1)) + (1 << (logDegree - logSplit - 1)) + logDegree - logSplit - 4
    return logSplit + 1 if a > b else logSplit


def split_degree(n: int):                        # power_basis.go:34-52
    if n <= 0:
        raise ValueError("invalid n: n=%d should be greater than zero" % n)
    if n & (n - 1) == 0:
        return n // 2, n // 2
    k = (n - 1).bit_length() - 1
    return (1 << k) - 1, n + 1 - (1 << k)


def _factorize(p: _Poly, n: int):                # bignum.Polynomial.Factorize + polynomial.Polynomial.Factorize
    if n < p.Degree() >> 1:
        raise ValueError("cannot Factorize: n < p.Degree()/2")
    pr = list(p.Coeffs[:n])
    pq = [None] * (p.Degree() - n + 1)
    pq[0] = p.Coeffs[n]
    odd, even = p.IsOdd, p.IsEven
    keep = lambda i: (not (even or odd)) or (i & 1 == 0 and even) or (i & 1 == 1 and odd)
    for j, i in enumerate(range(n + 1, p.Degree() + 1), 1):
        c = p.Coeffs[i]
        if c is None or not keep(i):
            continue
        if p.Basis == MONOMIAL:
            pq[i - n] = c
        else:
            pq[i - n] = _C(rnd(2 * c.re, c.prec), rnd(2 * c.im, c.prec), c.prec)
            z = pr[n - j]
            pr[n - j] = _C(rnd(z.re - c.re, z.prec), rnd(z.im - c.im, z.prec), z.prec) if z is not None else _C(-c.re, -c.im, c.prec)
    q_, r_ = _Poly(pq, p.Basis, p.IsOdd, p.IsEven), _Poly(pr, p.Basis, p.IsOdd, p.IsEven)
    q_.MaxDeg = p.MaxDeg
    r_.MaxDeg = n - 1 if p.MaxDeg == p.Degree() else p.MaxDeg - (p.Degree() - n + 1)
    q_.Lead, r_.Lead = bool(p.Lead), False
    return q_, r_


class _Sim:                                      # circuits/ckks/polynomial/polynomial_evaluator_sim.go
    """The CKKS simEvaluator over (level, scale) pairs. gen_power and recurse are the scheme-independent SimPowerBasis.GenPower and
    recursePS; a scheme's simEvaluator overrides depth, rescale, mul, baby, giant and same_scale."""

    def __init__(self, Q, lpr): self.Q, self.lpr = Q, lpr

    def depth(self, degree):                     # PolynomialDepth
        return self.lpr * (degree.bit_length() - 1)

    def rescale(self, lv, s):
        for _ in range(self.lpr):
            s = _sdiv(s, _snew(self.Q[lv])); lv -= 1
        return lv, s

    def mul(self, a, b):                         # MulNew
        return min(a[0], b[0]), _smul(a[1], b[1])

    def same_scale(self, a, b):                  # Scale.InDelta(.., ScalePrecision - 12)
        return _in_delta(a, b, SCALE_PREC - 12)

    def gen_power(self, pb, n):
        if n < 2:
            return
        a, b = split_degree(n)
        self.gen_power(pb, a); self.gen_power(pb, b)
        pb[n] = self.rescale(*self.mul(pb[a], pb[b]))

    def baby(self, lead, lv, s):
        if lead:
            for i in range(self.lpr):
                s = _smul(s, _snew(self.Q[lv - i]))
        return lv, s

    def giant(self, lead, lv, s, xs):
        qi = 1
        for i in range(self.lpr):
            qi *= self.Q[lv - i] if lead else self.Q[lv + self.lpr - i]
        return lv + self.lpr, _sdiv(_smul(s, _snew(qi)), xs)

    def recurse(self, logSplit, tl, p: _Poly, pb, os_):      # polynomial.go:109-153
        if p.Degree() < (1 << logSplit):
            if p.Lead and logSplit > 1 and p.MaxDeg > (1 << p.MaxDeg.bit_length()) - (1 << (logSplit - 1)):
                return self.recurse(optimal_split(p.Degree().bit_length()), tl, p, pb, os_)
            p.Level, p.Scale = self.baby(p.Lead, tl, os_)
            return [p], (p.Level, p.Scale)
        nextPower = 1 << logSplit
        while nextPower < (p.Degree() >> 1) + 1:
            nextPower <<= 1
        xs = pb[nextPower][1]
        cq, cr = _factorize(p, nextPower)
        tln, tsn = self.giant(p.Lead, tl, os_, xs)
        bq, res = self.recurse(logSplit, tln, cq, pb, tsn)
        res = self.mul(self.rescale(*res), pb[nextPower])
        br, tmp = self.recurse(logSplit, tl, cr, pb, res[1])
        if not self.same_scale(tmp[1], res[1]):
            raise ValueError("recursePS: res.Scale != tmp.Scale")
        return bq + br, res


# ---------------------------------------------------------------------------------------------------------------- the planner
class _Sym:
    """A planned ciphertext: its slot, level, scale (rlwe.Scale value) and degree."""
    __slots__ = ("slot", "level", "scale", "deg")

    def __init__(self, slot, level, scale, deg):
        self.slot, self.level, self.scale, self.deg = slot, level, scale, deg


class _Lin:
    """A pending linear form sum_k w_k X_k + const (const on component 0): w and const are [limb][half] residues."""

    def __init__(self, level, scale, Q):
        self.level, self.scale, self.Q = level, scale, Q[: level + 1]
        self.w: Dict[int, list] = {}
        self.const = [[0, 0] for _ in self.Q]

    def scale_by(self, m):
        for key in self.w:
            self.w[key] = [[x * m[i] % q for x in row] for i, (row, q) in enumerate(zip(self.w[key], self.Q))]
        self.const = [[x * m[i] % q for x in row] for i, (row, q) in enumerate(zip(self.const, self.Q))]


class _VLin:
    """A pending plaintext-weighted form (a baby step with a Mapping): w[slot] = (plaintext, s) for the terms and const = (plaintext, s)
    for component 0, s the per-limb scalar that multiplies the plaintext. seq: the reference's order of the steps the form folds,
    ("pt", slot or None for the constant) for an added plaintext product and ("mul", m) for a per-limb multiplication of res."""

    def __init__(self, level, scale, Q):
        self.level, self.scale, self.Q = level, scale, Q[: level + 1]
        self.w: Dict[int, tuple] = {}
        self.const = None
        self.seq: List[tuple] = []

    def scale_by(self, m):
        self.seq.append(("mul", [int(x) % q for x, q in zip(m, self.Q)]))
        mul = lambda s: [x * m[i] % q for i, (x, q) in enumerate(zip(s, self.Q))]
        self.w = {k: (pt, mul(s)) for k, (pt, s) in self.w.items()}
        if self.const is not None:
            self.const = (self.const[0], mul(self.const[1]))


class Program:
    """A planned evaluation: ops (dicts), the slot count, the output slot / level / scale. A vector program also lists the slot vectors
    its PTLINCOMB op multiplies: plaintexts[j] = dict(coeffs, level, scale), coeffs[i] the value of the slots of polynomial i, and
    slot_map[j] the polynomial of slot j (-1: unmapped, 0); values(j) is the vector to encode."""

    def __init__(self):
        self.ops: List[dict] = []
        self.n_slots = 1
        self.out_slot = self.out_level = -1
        self.out_scale = Fraction(0)
        self.plaintexts: List[dict] = []
        self.slot_map = None

    def values(self, j: int, dtype=np.complex128):
        """The slot vector of plaintext j (MaxSlots entries)."""
        table = np.array(list(self.plaintexts[j]["coeffs"]) + [0], dtype=dtype)
        return table[self.slot_map]

    def kinds(self) -> List[int]:
        return [o["kind"] for o in self.ops]

    def to_c(self, levels_per_rescale: int):
        """The lgpu_poly_program struct (and the arrays it points to, kept alive on the returned object)."""
        keep = []
        ops = (PolyOpStruct * max(1, len(self.ops)))()
        for i, o in enumerate(self.ops):
            s = ops[i]
            s.kind, s.dst, s.src0, s.src1, s.addend, s.level = o["kind"], o.get("dst", -1), o.get("src0", -1), o.get("src1", -1), o.get("addend", -1), o["level"]
            if o["kind"] in (LINCOMB, PTLINCOMB):
                outs = (ctypes.c_int * len(o["outs"]))(*o["outs"])
                lv = (ctypes.c_int * len(o["outs"]))(*o["out_levels"])
                terms = (ctypes.c_int * max(1, len(o["terms"])))(*o["terms"])
                keep += [outs, lv, terms]
                s.n_out, s.n_terms = len(o["outs"]), len(o["terms"])
                s.outs, s.out_levels, s.terms = outs, lv, terms
                if o["kind"] == LINCOMB:
                    w = (ctypes.c_uint64 * len(o["weights"]))(*o["weights"])
                    keep.append(w)
                    s.weights = ctypes.cast(w, ctypes.POINTER(ctypes.c_uint64))
            elif o["kind"] == TENSOR:
                w = (ctypes.c_uint64 * len(o["weights"]))(*o["weights"])
                keep.append(w)
                s.weights = ctypes.cast(w, ctypes.POINTER(ctypes.c_uint64))
        prog = PolyProgramStruct(self.n_slots, len(self.ops), ops, self.out_slot, levels_per_rescale)
        prog._keep = (ops, keep)
        return prog


    def pt_weights_to_c(self, pt_ptr: int, pt_stride: int, pt_levels: Sequence[int]):
        """The lgpu_poly_pt_weights struct of the program's PTLINCOMB op for plaintexts at device address pt_ptr, pt_stride words apart."""
        o = [o for o in self.ops if o["kind"] == PTLINCOMB][0]
        lv = (ctypes.c_int * len(pt_levels))(*pt_levels)
        idx = (ctypes.c_int * len(o["index"]))(*o["index"])
        sc = (ctypes.c_uint64 * len(o["scalars"]))(*o["scalars"])
        st = PolyPtWeightsStruct(ctypes.c_void_p(pt_ptr), pt_stride, len(pt_levels), lv, idx, ctypes.cast(sc, ctypes.POINTER(ctypes.c_uint64)))
        st._keep = (lv, idx, sc)
        return st


class PolyPtWeightsStruct(ctypes.Structure):
    """lgpu_poly_pt_weights (include/lattigo_b200.h)."""
    _fields_ = [("pt", ctypes.c_void_p), ("pt_stride", ctypes.c_size_t), ("n_pt", ctypes.c_int), ("pt_levels", ctypes.POINTER(ctypes.c_int)),
                ("index", ctypes.POINTER(ctypes.c_int)), ("scalars", ctypes.POINTER(ctypes.c_uint64))]


class PolyOpStruct(ctypes.Structure):
    """lgpu_poly_op (include/lattigo_b200.h)."""
    _fields_ = [("kind", ctypes.c_int), ("dst", ctypes.c_int), ("src0", ctypes.c_int), ("src1", ctypes.c_int), ("addend", ctypes.c_int),
                ("level", ctypes.c_int), ("n_out", ctypes.c_int), ("n_terms", ctypes.c_int), ("outs", ctypes.POINTER(ctypes.c_int)),
                ("out_levels", ctypes.POINTER(ctypes.c_int)), ("terms", ctypes.POINTER(ctypes.c_int)), ("weights", ctypes.POINTER(ctypes.c_uint64))]


class PolyProgramStruct(ctypes.Structure):
    """lgpu_poly_program (include/lattigo_b200.h)."""
    _fields_ = [("n_slots", ctypes.c_int), ("n_ops", ctypes.c_int), ("ops", ctypes.POINTER(PolyOpStruct)), ("out_slot", ctypes.c_int),
                ("levels_per_rescale", ctypes.c_int)]


class _Planner:
    def __init__(self, Q, lpr, prec, roots1, max_slots=0):
        self.Q, self.lpr, self.prec, self.roots1 = [int(q) for q in Q], lpr, prec, roots1
        self.max_slots = max_slots
        self.prog = Program()

    def _slot(self):
        s = self.prog.n_slots
        self.prog.n_slots += 1
        return s

    def _halves(self, level, re, im):
        """evaluateWithScalar (schemes/ckks/evaluator.go:410-424): the scalars of the lower and upper NTT halves."""
        out = []
        for i, q in enumerate(self.Q[: level + 1]):
            if im[i]:
                if self.roots1 is None:
                    raise ValueError("complex coefficients need the ring's RootsForward[1]")
                x = im[i] * int(self.roots1[i]) * pow(1 << 64, -1, q) % q       # MRed(imag, RootsForward[1])
            else:
                x = 0
            out.append([(re[i] + x) % q, (re[i] + q - x) % q])
        return out

    def _int_mul_weight(self, level, v: int):
        """Mul(ct, *big.Int v): the RNS scalar (v rounded to EncodingPrecision bits, scale 1) per limb."""
        c = _to_complex(v, self.prec)
        re, _ = _rns_scalar(self.Q[: level + 1], Fraction(1), c)
        return re

    # ---- rounding ops --------------------------------------------------------------------------------------------
    def rescale(self, x: _Sym) -> _Sym:
        if x.level <= self.lpr - 1:
            raise ValueError("cannot Rescale: input Ciphertext level is too low")
        s = x.scale
        for i in range(self.lpr):
            s = _sdiv(s, _snew(self.Q[x.level - i]))
        y = _Sym(self._slot(), x.level - self.lpr, s, x.deg)
        self.prog.ops.append(dict(kind=RESCALE, dst=y.slot, src0=x.slot, level=y.level))
        return y

    def mul_relin(self, a: _Sym, b: _Sym) -> _Sym:
        y = _Sym(self._slot(), min(a.level, b.level), _smul(a.scale, b.scale), 1)
        self.prog.ops.append(dict(kind=MULRELIN, dst=y.slot, src0=a.slot, src1=b.slot, level=y.level))
        return y

    def relin(self, x: _Sym) -> _Sym:
        y = _Sym(self._slot(), x.level, x.scale, 1)
        self.prog.ops.append(dict(kind=RELIN, dst=y.slot, src0=x.slot, level=y.level))
        return y

    def _ratio(self, big, small):
        return int(_sdiv(big, small))                      # ratioFlo.Int(nil): truncation

    def lincomb(self, forms: List[_Lin], outs: List[_Sym]):
        terms = sorted({k for f in forms for k in f.w})
        if len(terms) > MAX_TERMS or len(forms) > MAX_OUTPUTS:
            raise ValueError("polynomial too large for one LINCOMB (%d terms, %d outputs)" % (len(terms), len(forms)))
        L = max(f.level for f in forms)
        w = []
        for f in forms:
            for k in terms + [None]:
                rows = f.const if k is None else f.w.get(k)
                for r in range(L + 1):
                    w += rows[r] if rows is not None and r <= f.level else [0, 0]
        self.prog.ops.append(dict(kind=LINCOMB, level=L, outs=[o.slot for o in outs], out_levels=[f.level for f in forms], terms=terms, weights=w))

    # ---- schemes/ckks linear ops, folded ----------------------------------------------------------------------
    def add_const(self, f: _Lin, c):                        # Add(ct, scalar): AddDoubleRNSScalar on component 0
        re, im = _rns_scalar(self.Q[: f.level + 1], f.scale, _to_complex(c, self.prec))
        for i, (h0, h1) in enumerate(self._halves(f.level, re, im)):
            q = self.Q[i]
            f.const[i] = [(f.const[i][0] + h0) % q, (f.const[i][1] + h1) % q]

    def mul_then_add(self, x: _Sym, c, f: _Lin):           # MulThenAdd(x, scalar, res): schemes/ckks/evaluator.go:928-975
        if x.level < f.level:
            raise ValueError("baby step above the level of its power X^k is not supported")
        level = f.level
        cm = _to_complex(c, self.prec)
        if x.scale == f.scale:
            if cm.re.denominator == 1 and cm.im.denominator == 1:
                sr = _snew(1)
            else:
                sr = _snew(self.Q[level])
                for i in range(1, self.lpr):
                    sr = _smul(sr, _snew(self.Q[level - i]))
                m = self._int_mul_weight(level, int(sr))
                f.scale_by(m)
                f.scale = _smul(f.scale, sr)
        elif x.scale < f.scale:
            sr = _sdiv(f.scale, x.scale)
        else:
            raise ValueError("cannot MulThenAdd: op0.Scale > opOut.Scale is not supported")
        re, im = _rns_scalar(self.Q[: level + 1], sr, cm)
        h = self._halves(level, re, im)
        cur = f.w.get(x.slot) or [[0, 0] for _ in range(level + 1)]
        f.w[x.slot] = [[(cur[i][0] + h[i][0]) % q, (cur[i][1] + h[i][1]) % q] for i, q in enumerate(self.Q[: level + 1])]

    # ---- power_basis.go -------------------------------------------------------------------------------------------
    def gen_power(self, pb, basis, n):
        if n not in pb and self._gen_power(pb, basis, n):
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
        M = self.mul_relin(pb[a], pb[b])
        if basis != CHEBYSHEV:
            pb[n] = M
            return True
        # C[n] = 2 C[a] C[b] - C[c]: Add(n, n, n) keeps the scale; Sub multiplies the smaller-scale operand by the truncated ratio
        c = abs(a - b)
        out = _Lin(M.level, M.scale, self.Q)
        two = [[2, 2] for _ in range(M.level + 1)]
        out.w[M.slot] = two
        if c == 0:
            self.add_const(out, -1)
        else:
            self.gen_power(pb, basis, c)
            C = pb[c]
            lv = min(M.level, C.level)
            if lv != M.level:
                raise ValueError("power basis: T_%d below the level of its product" % c)
            if M.scale > C.scale:
                r = self._int_mul_weight(lv, self._ratio(M.scale, C.scale))
                out.w[C.slot] = [[(-r[i]) % q] * 2 for i, q in enumerate(self.Q[: lv + 1])]
            elif M.scale < C.scale:
                r = self._int_mul_weight(lv, self._ratio(C.scale, M.scale))
                out.w[M.slot] = [[2 * r[i] % q] * 2 for i, q in enumerate(self.Q[: lv + 1])]
                out.w[C.slot] = [[q - 1] * 2 for q in self.Q[: lv + 1]]
                out.scale = C.scale
            else:
                out.w[C.slot] = [[q - 1] * 2 for q in self.Q[: lv + 1]]
        y = _Sym(self._slot(), out.level, out.scale, 1)
        self.lincomb([out], [y])
        pb[n] = y
        return True

    # ---- polynomial_evaluator.go -------------------------------------------------------------------------------------
    def baby_step(self, pol: _Poly, pb, level, scale) -> _Lin:     # EvaluatePolynomialVectorFromPowerBasis :254-359
        even, odd = pol.IsEven, pol.IsOdd
        minDeg = len(pol.Coeffs) - 1 - (1 if even and not odd else 0)
        f = _Lin(level, scale, self.Q)
        if even:
            self.add_const(f, self._coeff(pol, 0))
        if minDeg == 0:
            return f
        for key in range(pol.Degree(), 0, -1):
            if (not (even or odd)) or (key & 1 == 0 and even) or (key & 1 == 1 and odd):
                self.mul_then_add(pb[key], self._coeff(pol, key), f)
        return f

    @staticmethod
    def _coeff(pol, k):
        if pol.Coeffs[k] is None:
            raise ValueError("nil coefficient %d" % k)
        return pol.Coeffs[k]

    def monomial(self, a: _Sym, b: _Sym, x: _Sym) -> _Sym:      # EvaluateMonomial :226-251, Mul + Add fused into one TENSOR op
        if b.deg == 2:
            b = self.relin(b)
        b = self.rescale(b)
        lv = min(b.level, x.level)
        bs = _smul(b.scale, x.scale)
        if not _in_delta(a.scale, bs, SCALE_PREC - 12):
            raise ValueError("evalMonomial: scale discrepency")
        lv = min(lv, a.level)
        one = [1] * (lv + 1)
        rb, ra, scale = one, one, bs
        if bs > a.scale:
            ra = self._int_mul_weight(lv, self._ratio(bs, a.scale))
        elif bs < a.scale:
            rb = self._int_mul_weight(lv, self._ratio(a.scale, bs))
            scale = a.scale
        y = _Sym(self._slot(), lv, scale, 2)
        self.prog.ops.append(dict(kind=TENSOR, dst=y.slot, src0=b.slot, src1=x.slot, addend=a.slot, level=lv, weights=list(rb) + list(ra)))
        return y

    # ---- the baby step of a PolynomialVector with a Mapping (polynomial_evaluator.go:281-320) ------------------------------
    def _pt(self, values, level, scale) -> int:
        """A slot vector to encode at (level, scale); returns its plaintext index."""
        self.prog.plaintexts.append(dict(coeffs=values, level=level, scale=scale))
        return len(self.prog.plaintexts) - 1

    def set_mapping(self, n_polys, mapping):
        """slot_map: which polynomial's coefficient each of the MaxSlots slots takes (GetVectorCoefficient writes the polynomials in
        order, so a later polynomial wins a slot mapped twice); -1 for an unmapped slot."""
        sm = np.full(self.max_slots, n_polys, dtype=np.int64)
        for i in range(n_polys):
            for j in mapping.get(i, ()):
                sm[j] = i
        sm[sm == n_polys] = -1
        self.prog.slot_map = sm

    def vector_coefficient(self, pols, mapping, k):       # CoefficientGetter.GetVectorCoefficient: nil (CKKS) slots encode as 0
        return [0j if p.Coeffs[k] is None else complex(float(p.Coeffs[k].re), float(p.Coeffs[k].im)) for p in pols]   # Complex128()

    def vec_add(self, f: _VLin, values):                 # Add(res, vector): encoded at res.Scale, added to component 0
        f.const = (self._pt(values, f.level, f.scale), [1] * (f.level + 1))
        f.seq.append(("pt", None))

    def _mul_big_float(self, level, v: Fraction):
        """Mul(ct, *big.Float v) (schemes/ckks/evaluator.go:629-666): the per-limb scalar and the scale it multiplies by."""
        cm = _to_complex(_C(v, 0, SCALE_PREC), self.prec)
        if cm.re.denominator == 1:
            sc = _snew(1)
        else:
            sc = _snew(self.Q[level])
            for i in range(1, self.lpr):
                sc = _smul(sc, _snew(self.Q[level - i]))
        re, _ = _rns_scalar(self.Q[: level + 1], sc, cm)
        return re, sc

    def vec_mul_then_add(self, x: _Sym, values, f: _VLin):     # MulThenAdd(X^k, vector, res): schemes/ckks/evaluator.go:977-1025
        if x.level < f.level:
            raise ValueError("baby step above the level of its power X^k is not supported")
        level = f.level
        if x.scale == f.scale:
            sr = _snew(self.Q[level])
            for i in range(1, self.lpr):
                sr = _smul(sr, _snew(self.Q[level - i]))
            f.scale_by(self._int_mul_weight(level, int(sr)))
            f.scale = _smul(f.scale, sr)
        elif x.scale < f.scale:
            sr = _sdiv(f.scale, x.scale)
        else:
            raise ValueError("cannot MulThenAdd: op0.Scale > opOut.Scale is not supported")
        # mulRelinThenAdd (:1081-1170), degree-0 branch: Mul(opOut, ratio) when the ratio to op0.Scale * pt.Scale is >= 2
        res_scale = _smul(x.scale, sr)
        if f.scale < res_scale:
            ratio = _sdiv(res_scale, f.scale)
            if float(ratio) >= 2.0:
                m, _ = self._mul_big_float(level, ratio)
                f.scale_by(m)
                f.scale = res_scale
        f.w[x.slot] = (self._pt(values, level, sr), [1] * (level + 1))
        f.seq.append(("pt", x.slot))

    def vec_baby_step(self, pols, pb, level, scale, mapping) -> _VLin:
        even, odd = all(p.IsEven for p in pols), all(p.IsOdd for p in pols)      # PolynomialVector.IsEven / IsOdd
        p0 = pols[0]
        minDeg = len(p0.Coeffs) - 1 - (1 if even and not odd else 0)
        f = _VLin(level, scale, self.Q)
        if even:
            self.vec_add(f, self.vector_coefficient(pols, mapping, 0))
        if minDeg == 0:
            return f
        for key in range(p0.Degree(), 0, -1):
            if (not (even or odd)) or (key & 1 == 0 and even) or (key & 1 == 1 and odd):
                self.vec_mul_then_add(pb[key], self.vector_coefficient(pols, mapping, key), f)
        return f

    def ptlincomb(self, forms: List[_VLin], outs: List[_Sym]):
        terms = sorted({k for f in forms for k in f.w})
        if len(terms) > MAX_TERMS or len(forms) > MAX_OUTPUTS:
            raise ValueError("polynomial too large for one PTLINCOMB (%d terms, %d outputs)" % (len(terms), len(forms)))
        L = max(f.level for f in forms)
        index, scalars = [], []
        for f in forms:
            for k in terms + [None]:
                e = f.const if k is None else f.w.get(k)
                index.append(-1 if e is None else e[0])
                for r in range(L + 1):
                    scalars.append(e[1][r] if e is not None and r <= f.level else 0)
        # sequence[i]: output i's steps in the reference's order, ("pt", term position, n_terms for the constant) or ("mul", m per
        # limb); the device runs the folded form, tools that replay the reference's op sequence read this
        seq = [[("pt", len(terms) if k is None else terms.index(k)) if kind == "pt" else ("mul", k) for kind, k in f.seq] for f in forms]
        self.prog.ops.append(dict(kind=PTLINCOMB, level=L, outs=[o.slot for o in outs], out_levels=[f.level for f in forms], terms=terms,
                                  index=index, scalars=scalars, sequence=seq))

    def _sim(self) -> _Sim:
        return _Sim(self.Q, self.lpr)

    def evaluate(self, level, scale, p: _Poly, target_scale, others=(), mapping=None) -> Program:
        """The scheme-independent part of Evaluate (common/polynomial/polynomial_evaluator.go:29-161): level check, power basis,
        Paterson-Stockmeyer split on the scheme's simEvaluator, every baby step in one LINCOMB (one PTLINCOMB with a Mapping), the
        giant steps, the final Relinearize / Rescale. Scale values are the scheme's (Fractions for CKKS, ints mod t for BGV).
        others: the PolynomialVector's polynomials after p = Value[0]; the power basis takes their odd / even flags OR-ed, the baby
        steps AND-ed, and each is split on its own."""
        if p.Degree() < 1:
            raise ValueError("the polynomial must have degree >= 1")
        pols = [p] + list(others)
        pb: Dict[int, _Sym] = {1: _Sym(0, level, scale, 1)}
        depth = (p.Degree() - 1).bit_length()
        if level < self.lpr * depth:
            raise ValueError("%d levels < %d log(d) -> cannot evaluate poly" % (level, self.lpr * depth))
        logDegree = p.Degree().bit_length()
        logSplit = optimal_split(logDegree)
        odd, even = any(q.IsOdd for q in pols), any(q.IsEven for q in pols)
        self.gen_power(pb, p.Basis, 1 << (logDegree - 1))
        for i in range((1 << logSplit) - 1, 2, -1):
            if (not (even or odd)) or (i & 1 == 0 and even) or (i & 1 == 1 and odd):
                self.gen_power(pb, p.Basis, i)
        # PatersonStockmeyerPolynomial with the simulated power basis (polynomial.go:74-106)
        sim = self._sim()
        spb = {1: (level, scale)}
        sim.gen_power(spb, 1 << logDegree)
        for i in range((1 << logSplit) - 1, 2, -1):
            sim.gen_power(spb, i)
        pss = [sim.recurse(logSplit, level - sim.depth(p.Degree()), q, spb, target_scale)[0] for q in pols]
        ps = pss[0]
        if mapping is not None:                                    # every baby step in one PTLINCOMB
            self.set_mapping(len(pols), mapping)
            forms = [self.vec_baby_step([s[i] for s in pss], pb, bs.Level, bs.Scale, mapping) for i, bs in enumerate(ps)]
            outs = [_Sym(self._slot(), f.level, f.scale, 1) for f in forms]
            self.ptlincomb(forms, outs)
        else:                                                      # every baby step in one LINCOMB
            for i, bs in enumerate(ps):                            # GetSingleCoefficient of Value[0] under the vector's AND-ed flags
                bs.IsEven, bs.IsOdd = all(s[i].IsEven for s in pss), all(s[i].IsOdd for s in pss)
            forms = [self.baby_step(bs, pb, bs.Level, bs.Scale) for bs in ps]
            outs = [_Sym(self._slot(), f.level, f.scale, 1) for f in forms]
            self.lincomb(forms, outs)
        split = len(ps)
        babySteps = [None] * split
        for i in range(split):
            babySteps[split - i - 1] = [ps[i].Degree(), outs[i]]
        while len(babySteps) != 1:                                 # EvaluatePatersonStockmeyerPolynomialVector :117-148
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
                    e, o = babySteps[i], babySteps[i + 1]
                    deg = 1 << e[0].bit_length()
                    o[1] = self.monomial(e[1], o[1], pb[deg])
                    o[0] = 2 * deg - 1
                    babySteps[i] = None
                    i += 1
                i += 1
            babySteps = [b for b in babySteps if b is not None]
        res = babySteps[0][1]
        if res.deg == 2:
            res = self.relin(res)
        res = self.rescale(res)
        self.prog.out_slot, self.prog.out_level, self.prog.out_scale = res.slot, res.level, res.scale
        return self.prog


def _coeffs(coeffs) -> List[_C]:
    """bignum.NewPolynomial from []float64 / []complex128: 53-bit big.Floats."""
    out = []
    for c in coeffs:
        c = complex(c)
        out.append(_C(Fraction(c.real), Fraction(c.imag), 53))
    return out


def plan(Q: Sequence[int], level: int, scale, coeffs, basis: int, target_scale, levels_per_rescale: int = 1, encoding_precision: int = 53,
         odd: bool = True, even: bool = True, roots1: Optional[Sequence[int]] = None) -> Program:
    """The device program of Evaluate(ct, bignum.NewPolynomial(basis, coeffs, .) with IsOdd = odd, IsEven = even, targetScale) for
    a ciphertext at `level` and `scale`. roots1[i]: RootsForward[1] of Q limb i (needed for non-real coefficients only)."""
    return plan_vector(Q, level, scale, PolynomialVector([Polynomial(coeffs, basis, odd, even)], None), target_scale, levels_per_rescale,
                       encoding_precision, roots1=roots1)


class Polynomial:
    """bignum.NewPolynomial(basis, coeffs, nil) with its IsOdd / IsEven flags (polynomial.NewPolynomial)."""

    def __init__(self, coeffs, basis: int = MONOMIAL, odd: bool = True, even: bool = True):
        self.coeffs, self.basis, self.odd, self.even = list(coeffs), basis, odd, even

    def Degree(self):
        return len(self.coeffs) - 1


class PolynomialVector:
    """polynomial.PolynomialVector: Value (the polynomials) and Mapping {i: slots that take polynomial i} or None."""

    def __init__(self, value: Sequence[Polynomial], mapping: Optional[Dict[int, Sequence[int]]]):
        self.Value, self.Mapping = list(value), mapping


def NewPolynomialVector(polys: Sequence[Polynomial], mapping) -> PolynomialVector:
    """polynomial.NewPolynomialVector (circuits/common/polynomial/polynomial.go:165-195), with the reference's errors."""
    if not polys:
        raise ValueError("a polynomial vector needs at least one polynomial")
    maxDeg = max(p.Degree() for p in polys)
    basis = polys[-1].basis
    for p in polys:
        if basis != p.basis:
            raise ValueError("polynomial basis must be the same for all polynomials in a polynomial vector")
        if maxDeg != p.Degree():
            raise ValueError("polynomial degree must all be the same")
    return PolynomialVector(polys, None if mapping is None else {int(k): [int(j) for j in v] for k, v in mapping.items()})


def _check_vector(pv: PolynomialVector, max_slots: int, slots: int):
    if pv.Mapping is None:
        return
    for i, js in pv.Mapping.items():
        for j in js:
            if i < len(pv.Value) and not 0 <= j < max_slots:
                raise ValueError("mapping slot %d of polynomial %d out of range [0, %d)" % (j, i, max_slots))
    if slots < max_slots:                         # the slot vectors have MaxSlots entries: Embed refuses them on fewer slots
        raise ValueError("cannot Embed: ensure that #values (%d) <= slots (%d) <= maxCols (%d)" % (max_slots, slots, max_slots))


def plan_vector(Q: Sequence[int], level: int, scale, pv: PolynomialVector, target_scale, levels_per_rescale: int = 1,
                encoding_precision: int = 53, log_n: int = 0, log_slots: Optional[int] = None, roots1: Optional[Sequence[int]] = None) -> Program:
    """The device program of Evaluate(ct, pv, targetScale) for a PolynomialVector. With a Mapping: every baby step in one PTLINCOMB and
    program.plaintexts, the slot vectors to encode (values, level, scale). Without one: the scalar program of Value[0] (the reference's
    scalar path), with the vector's odd / even flags. log_n: LogN of the ring (MaxSlots = 2^(LogN - 1)), needed unless pv is one polynomial
    without a Mapping; log_slots: the ciphertext's LogSlots. roots1[i]: RootsForward[1] of Q limb i (needed for non-real coefficients
    without a Mapping only)."""
    p0 = pv.Value[0]
    if p0.basis not in (MONOMIAL, CHEBYSHEV):
        raise ValueError("basis must be MONOMIAL or CHEBYSHEV")
    if levels_per_rescale < 1:
        raise ValueError("levels_per_rescale must be >= 1")
    polys = [_Poly(_coeffs(q.coeffs), q.basis, q.odd, q.even) for q in pv.Value]
    if polys[0].Degree() > 255:
        raise ValueError("degree %d > 255 is not supported" % polys[0].Degree())
    max_slots = 0
    if pv.Mapping is not None or len(pv.Value) > 1:
        if log_n < 1:
            raise ValueError("log_n must be the ring's LogN (>= 1), got %d" % log_n)
        max_slots = 1 << (log_n - 1)
    if pv.Mapping is not None:
        if encoding_precision > 53:
            raise ValueError("the polynomial-vector path encodes its slot vectors with the float64 encoder (EncodingPrecision <= 53); "
                             "EncodingPrecision %d is not supported" % encoding_precision)
        _check_vector(pv, max_slots, 1 << (log_n - 1 if log_slots is None else log_slots))
    elif roots1 is None and any(complex(c).imag != 0 for c in p0.coeffs):
        raise ValueError("complex coefficients need the ring's RootsForward[1]")
    return _Planner(Q, levels_per_rescale, encoding_precision, roots1, max_slots).evaluate(level, Fraction(scale), polys[0], Fraction(target_scale),
                                                                                          polys[1:], pv.Mapping)


class PreparedVector:
    """A vector program with its slot vectors encoded on the device: reusable for any batch of ciphertexts at the level and scale it was
    planned for. pt: (n_pt, rows, N) int64 plaintext block, plaintext j's rows 0..pt_levels[j] written."""

    def __init__(self, prog: Program, pt, pt_levels):
        self.prog, self.pt, self.pt_levels = prog, pt, pt_levels
        self.out_level, self.out_scale = prog.out_level, prog.out_scale

    def structs(self, lpr: int):
        cp = self.prog.to_c(lpr)
        if self.pt is None:
            return cp, None
        return cp, self.prog.pt_weights_to_c(self.pt.data_ptr(), self.pt.shape[1] * self.pt.shape[2], self.pt_levels)


def _pt_block(ctx: Context, prog: Program, encode_group, dtype):
    """Allocates the plaintext block and encodes prog.plaintexts into it with one encode_group(values, level, scale, out_ptr, stride)
    call per distinct (level, scale); returns (block, pt_levels) with the op's indices renumbered to the block's order."""
    import torch
    if not prog.plaintexts:
        return None, []
    groups: Dict[tuple, List[int]] = {}
    for j, p in enumerate(prog.plaintexts):
        groups.setdefault((p["level"], p["scale"]), []).append(j)
    order = [j for g in groups.values() for j in g]
    vals = [prog.values(j, dtype) for j in range(len(prog.plaintexts))]
    new = {j: n for n, j in enumerate(order)}
    rows = max(p["level"] for p in prog.plaintexts) + 1
    N = ctx.N
    block = torch.zeros((len(order), rows, N), dtype=torch.int64, device="cuda:%d" % ctx.device)
    stride = rows * N
    first = 0
    for (lv, sc), js in groups.items():
        encode_group(np.stack([vals[j] for j in js]), lv, sc, block.data_ptr() + 8 * first * stride, stride)
        first += len(js)
    o = [o for o in prog.ops if o["kind"] == PTLINCOMB][0]
    o["index"] = [new[j] if j >= 0 else -1 for j in o["index"]]
    prog.plaintexts = [prog.plaintexts[j] for j in order]
    return block, [prog.plaintexts[n]["level"] for n in range(len(order))]


class _Evaluator:
    """What the CKKS and BGV polynomial evaluators share. A scheme supplies plan_vector, encode_plaintexts (its encode_group) and
    _call(level, ct, batch, prog, pts, out): its scalar entry point when pts is None, its vector entry point otherwise."""

    def _prepare(self, prog: Program, pv: PolynomialVector, *encoder) -> PreparedVector:
        """PrepareVector of a planned program: with a Mapping, its slot vectors encoded by encode_plaintexts(prog, *encoder)."""
        pt, lv = self.encode_plaintexts(prog, *encoder) if pv.Mapping is not None else (None, [])
        return PreparedVector(prog, pt, lv)

    def _evaluate(self, ct, prep: PreparedVector):
        return self.RunVector(prep, ct), prep.out_level, prep.out_scale

    def RunVector(self, prep: PreparedVector, ct):
        """Runs a prepared plan on ct (batch, 2, level+1, N) or (2, level+1, N). Returns the output ciphertexts."""
        import torch
        b = ct.shape[0] if ct.dim() == 4 else 1
        shape = (b, 2, prep.out_level + 1, self.ctx.N) if ct.dim() == 4 else (2, prep.out_level + 1, self.ctx.N)
        out = torch.empty(shape, dtype=torch.int64, device=ct.device)
        self._launch(*prep.structs(self.lpr), ct, out, b)
        return out

    def run(self, prog: Program, ct, out, batch: int):
        self._launch(prog.to_c(self.lpr), None, ct, out, batch)

    def _launch(self, cp, vw, ct, out, batch: int):
        _lib.check(self._call(ct.shape[-2] - 1, _dptr(ct), batch, ctypes.byref(cp), None if vw is None else ctypes.byref(vw), _dptr(out)))


class PolynomialEvaluator(_Evaluator):
    """polynomial.Evaluator (circuits/ckks/polynomial) for one polynomial. encoding_precision = ckks.Parameters.EncodingPrecision()
    = max(53, log2(DefaultScale))."""

    def __init__(self, ctx: Context, rlk, levels_per_rescale: int = 1, encoding_precision: int = 53):
        self.ctx, self.rlk, self.lpr, self.prec = ctx, rlk, levels_per_rescale, encoding_precision
        self._roots1 = None

    def roots1(self):
        if self._roots1 is None:
            self._roots1 = [int(self.ctx.table(0, i, 1)[1]) for i in range(len(self.ctx.Q))]
        return self._roots1

    def plan(self, level, scale, coeffs, basis, target_scale, odd=True, even=True) -> Program:
        return self.plan_vector(level, scale, PolynomialVector([Polynomial(coeffs, basis, odd, even)], None), target_scale)

    def Evaluate(self, ct, scale, coeffs, basis, target_scale, odd=True, even=True):
        """ct: (batch, 2, level+1, N) or (2, level+1, N) int64 CUDA tensor, NTT domain. Returns (ct_out, level, scale)."""
        return self.EvaluateVector(ct, scale, PolynomialVector([Polynomial(coeffs, basis, odd, even)], None), target_scale)

    # ---- PolynomialVector (Evaluate with a Mapping) ----------------------------------------------------------------------
    def plan_vector(self, level, scale, pv: PolynomialVector, target_scale, log_slots=None) -> Program:
        cplx = pv.Mapping is None and any(complex(c).imag != 0 for c in pv.Value[0].coeffs)
        return plan_vector(self.ctx.Q, level, scale, pv, target_scale, self.lpr, self.prec, self.ctx.logN, log_slots,
                           self.roots1() if cplx else None)

    def encode_plaintexts(self, prog: Program):
        """The program's slot vectors, encoded with lgpu_ckks_encode (NTT, Embed at the plaintext's scale as float64, no host FFT): one
        batched call per distinct (level, scale)."""
        import torch
        from .encoder import Encoder, ENC_NTT, _vp
        if getattr(self, "_enc", None) is None:
            self._enc = Encoder(self.ctx)
        enc = self._enc
        n = self.ctx.N // 2

        def encode_group(values, level, scale, out_ptr, stride):
            v = torch.from_numpy(values).to("cuda:%d" % self.ctx.device)
            _lib.check(_lib.lib().lgpu_ckks_encode(self.ctx.h, _vp(v), n, self.ctx.logN - 1, float(scale), ENC_NTT, _vp(enc.rot_group),
                                                   _vp(enc.roots), level, ctypes.c_void_p(out_ptr), -1, None, len(values), n, stride, 0,
                                                   _stream()))
        return _pt_block(self.ctx, prog, encode_group, np.complex128)

    def PrepareVector(self, level, scale, pv: PolynomialVector, target_scale, log_slots=None) -> PreparedVector:
        """Plans Evaluate(ct, pv, target_scale) for ciphertexts at (level, scale) and encodes its slot vectors on the device."""
        return self._prepare(self.plan_vector(level, scale, pv, target_scale, log_slots), pv)

    def EvaluateVector(self, ct, scale, pv: PolynomialVector, target_scale, log_slots=None):
        """Evaluate(ct, PolynomialVector, targetScale) = PrepareVector + RunVector. Returns (ct_out, level, scale)."""
        return self._evaluate(ct, self.PrepareVector(ct.shape[-2] - 1, scale, pv, target_scale, log_slots))

    def _call(self, level, ct, batch, prog, pts, out):
        rlk = self.rlk.ref() if self.rlk is not None else None
        if pts is None:
            return _lib.lib().lgpu_ckks_polynomial_evaluate(self.ctx.h, level, ct, batch, prog, rlk, out, _stream())
        return _lib.lib().lgpu_ckks_polynomial_vector_evaluate(self.ctx.h, level, ct, batch, prog, pts, rlk, out, _stream())

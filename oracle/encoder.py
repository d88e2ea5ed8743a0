"""Restatement of the CKKS encoder on the prec <= 53 path (schemes/ckks/encoder.go, schemes/ckks/utils.go, core/rlwe/utils.go:187-244,
ring/ring.go:433-462, schemes/ckks/scaling.go:46-52). TEST INFRASTRUCTURE ONLY.

Python floats are IEEE doubles evaluated without fusion, like Go on amd64, so every float expression below is the reference's. The scalar
functions are literal; `fixed_point_rows` is the same branch structure vectorised with numpy for the large rings, and the CPU tests pin
it to the scalar form on every branch. Transforms come from oracle/specialfft.py (the FFT) and oracle/oracle.py (the C restatement of
the ring NTT)."""
from __future__ import annotations

import math

import numpy as np

from . import oracle as O
from . import specialfft as SF

U64 = np.uint64
MASK64 = (1 << 64) - 1
M32 = np.uint64(0xFFFFFFFF)
TWO64 = 1.8446744073709552e+19


# ---- tables (schemes/ckks/encoder.go:83-112, utils.go:53-77) ---------------------------------------------------------------
def rot_group(m: int):
    """Encoder.rotGroup: 5^i mod m, i < m/4."""
    return SF.rot_group(m)


def get_roots_complex128(m: int):
    """GetRootsComplex128(NthRoot) with its symmetries (utils.go:53-77)."""
    roots = [0j] * (m + 1)
    quarm = m >> 2
    angle = 2 * 3.141592653589793 / float(m)
    for i in range(quarm):
        roots[i] = complex(math.cos(angle * float(i)), 0)
    for i in range(quarm):
        roots[quarm - i] += complex(0, roots[i].real)
    for i in range(1, quarm + 1):
        roots[i + 1 * quarm] = complex(-roots[quarm - i].real, roots[quarm - i].imag)
        roots[i + 2 * quarm] = -roots[i]
        roots[i + 3 * quarm] = complex(roots[quarm - i].real, -roots[quarm - i].imag)
    roots[m] = roots[0]
    return roots


# ---- scalar modular primitives (ring/modular_reduction.go) ------------------------------------------------------------------
def BRedAdd(a: int, q: int, brc) -> int:
    mhi = (a * brc[0]) >> 64
    r = (a - mhi * q) & MASK64
    return r - q if r >= q else r


def MForm(a: int, q: int, brc) -> int:
    mhi = (a * brc[1]) >> 64
    r = (-(a * brc[0] + mhi) * q) & MASK64
    return r - q if r >= q else r


# ---- numpy uint64 forms of the same --------------------------------------------------------------------------------------
def _mulhi(a, b: int):
    a = np.asarray(a, dtype=U64)
    b0, b1 = U64(b & 0xFFFFFFFF), U64(b >> 32)
    a0, a1 = a & M32, a >> U64(32)
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> U64(32)) + (p01 & M32) + (p10 & M32)
    return p11 + (p01 >> U64(32)) + (p10 >> U64(32)) + (mid >> U64(32))


def bred_add_vec(a, q: int, brc):
    with np.errstate(over="ignore"):
        r = np.asarray(a, dtype=U64) - _mulhi(a, brc[0]) * U64(q)
    return np.where(r >= U64(q), r - U64(q), r)


def mform_vec(a, q: int, brc):
    a = np.asarray(a, dtype=U64)
    with np.errstate(over="ignore"):
        r = (U64(0) - (a * U64(brc[0]) + _mulhi(a, brc[1]))) * U64(q)
    return np.where(r >= U64(q), r - U64(q), r)


# ---- quantisation (schemes/ckks/utils.go:130-234) ------------------------------------------------------------------------
def SingleFloat64ToFixedPointCRT(r: "O.Ring", i: int, value: float, scale: float, coeffs):
    if value == 0:
        for j in range(len(coeffs)):
            coeffs[j][i] = 0
        return
    isNegative = False
    if value < 0:
        isNegative = True
        scale *= -1
    value *= scale
    moduli = r.ModuliChain()[: r.Level() + 1]
    if value >= 1.8446744073709552e+19:
        # big.NewFloat(value).Add(0.5) at 53 bits: value is an integer with ulp >= 2^12, so the sum rounds back to value; Int() is
        # exact. For +Inf, Float.Int returns nil and leaves xInt at 0.
        xInt = 0 if math.isinf(value) else int(value)
        for j, qj in enumerate(moduli):
            tmp = xInt % qj
            coeffs[j][i] = qj - tmp if isNegative else tmp
    else:
        brc = [s.BRedConstant for s in r.SubRings]
        c = int(value + 0.5)
        if isNegative:
            for j, qi in enumerate(moduli):
                coeffs[j][i] = qi - BRedAdd(c, qi, brc[j]) if c > qi else qi - c
        else:
            for j, qi in enumerate(moduli):
                coeffs[j][i] = BRedAdd(c, qi, brc[j]) if c > 0x1fffffffffffffff else c


def fixed_point_rows(r: "O.Ring", values, scale: float):
    """SingleFloat64ToFixedPointCRT of every value (numpy float64 vector) -> (level+1, len) uint64 words, vectorised."""
    v = np.asarray(values, dtype=np.float64)
    moduli = r.ModuliChain()[: r.Level() + 1]
    out = np.zeros((len(moduli), v.size), dtype=U64)
    zero = v == 0
    neg = v < 0
    x = v * np.where(neg, -scale, scale)
    big = ~zero & (x >= TWO64)
    small = ~zero & ~big
    c = np.zeros(v.size, dtype=U64)
    c[small] = (x[small] + 0.5).astype(U64)
    for j, qj in enumerate(moduli):
        brc = r.SubRings[j].BRedConstant
        red = bred_add_vec(c, qj, brc)
        qv = U64(qj)
        with np.errstate(over="ignore"):
            w_neg = np.where(c > qv, qv - red, qv - c)
        w_pos = np.where(c > U64(0x1fffffffffffffff), red, c)
        row = np.where(neg, w_neg, w_pos)
        for i in np.nonzero(big)[0]:
            tmp = 0 if math.isinf(x[i]) else int(x[i]) % qj
            row[i] = qj - tmp if neg[i] else tmp
        row[zero] = 0
        out[j] = row
    return out


def Complex128ToFixedPointCRT(r: "O.Ring", values, scale: float, coeffs):
    """Standard ring: real parts at 0..slots-1, imaginary parts at slots..2 slots-1, zeros after."""
    v = np.asarray(values, dtype=np.complex128)
    slots = v.size
    coeffs[:, :] = 0
    coeffs[:, :slots] = fixed_point_rows(r, v.real, scale)
    coeffs[:, slots:2 * slots] = fixed_point_rows(r, v.imag, scale)


def Float64ToFixedPointCRT(r: "O.Ring", values, scale: float, coeffs):
    v = np.asarray(values, dtype=np.float64)
    coeffs[:, :] = 0
    coeffs[:, :v.size] = fixed_point_rows(r, v, scale)


# ---- NTTSparseAndMontgomery (core/rlwe/utils.go:187-244) ----------------------------------------------------------------
def _ntt_n(s: "O.SubRing", a, n: int):
    """NTTStandard(coeffs[:n], coeffs[:n], n, ..., s.RootsForward): the n-point transform with the N-point table."""
    a = np.ascontiguousarray(a, dtype=U64)
    out = np.empty_like(a)
    O.lib().lo_ntt(O._ptr(a), O._ptr(out), n, s.Modulus, s.MRedConstant, O._ptr(s.brc), O._ptr(s.RootsForward))
    return out


def sparse_spread_literal(coeffs, n: int, gap: int):
    """The coefficient-domain branch (utils.go:234-241) exactly as written: the inner loop's j shadows the outer one. Raises IndexError
    where Go panics."""
    N = len(coeffs)
    for j in range(n - 1, -1, -1):
        coeffs[j * gap] = coeffs[j]
        for jj in range(1, gap):
            k = jj * gap - jj
            if k >= N:
                raise IndexError("index out of range [%d] with length %d" % (k, N))
            coeffs[k] = 0


def NTTSparseAndMontgomery(r: "O.Ring", log_slots: int, is_ntt: bool, is_montgomery: bool, pol):
    N = r.N()
    if 1 << log_slots == r.NthRoot() >> 2:
        if is_ntt:
            r.NTT(pol, pol)
        if is_montgomery:
            for i, s in enumerate(r.SubRings[: r.Level() + 1]):
                pol[i] = mform_vec(pol[i], s.Modulus, s.BRedConstant)
        return
    n = 2 << log_slots
    gap = N // n
    for i, s in enumerate(r.SubRings[: r.Level() + 1]):
        coeffs = pol[i]
        if is_montgomery:
            coeffs[:n] = mform_vec(coeffs[:n], s.Modulus, s.BRedConstant)
        if is_ntt:
            coeffs[:n] = _ntt_n(s, coeffs[:n], n)
            coeffs[:] = np.repeat(coeffs[:n].copy(), gap)
        else:
            sparse_spread_literal(coeffs, n, gap)


# ---- Embed / Encode (schemes/ckks/encoder.go:156-337) --------------------------------------------------------------------
def embed_double(ringQ: "O.Ring", ringP, values, log_slots: int, scale: float, is_ntt: bool, is_montgomery: bool, level_q: int,
                 level_p: int = -1, rt=None):
    """Encoder.embedDouble on a ring.Poly (level_p < 0) or a ringqp.Poly; returns the Q rows and the P rows (or None)."""
    N = ringQ.N()
    m = 2 * N
    slots = 1 << log_slots
    v = [complex(z) for z in np.asarray(values, dtype=np.complex128).reshape(-1)]
    assert len(v) <= slots
    buff = v + [0j] * (slots - len(v))
    SF.special_ifft(buff, slots, m, rot_group(m), rt if rt is not None else get_roots_complex128(m))
    outs = []
    for ring, level in ((ringQ, level_q), (ringP, level_p)):
        if level < 0:
            outs.append(None)
            continue
        r = ring.AtLevel(level)
        pol = np.zeros((level + 1, N), dtype=U64)
        Complex128ToFixedPointCRT(r, buff, scale, pol)
        NTTSparseAndMontgomery(r, log_slots, is_ntt, is_montgomery, pol)
        outs.append(pol)
    return outs[0], outs[1]


def encode_coeffs(ringQ: "O.Ring", values, level: int, scale: float, is_ntt: bool):
    """Encoder.Encode with IsBatched = false on []float64 (encoder.go:163-185)."""
    r = ringQ.AtLevel(level)
    pol = np.zeros((level + 1, ringQ.N()), dtype=U64)
    Float64ToFixedPointCRT(r, values, scale, pol)
    if is_ntt:
        r.NTT(pol, pol)
    return pol


# ---- decoding (encoder.go:497-762, 823-1160; ring/ring.go:433-462; scaling.go:46-52) ---------------------------------------
def PolyToBigint(r: "O.Ring", p, gap: int):
    Q = r.ModulusAtLevel[r.Level()]
    crt = []
    for s in r.SubRings[: r.Level() + 1]:
        Qi = Q // s.Modulus
        crt.append(Qi * (pow(Qi, -1, s.Modulus) % s.Modulus))
    N = r.N()
    out = np.zeros(len(range(0, N, gap)), dtype=object)
    for k in range(r.Level() + 1):
        out = out + p[k][::gap].astype(object) * crt[k]
    return [int(x) % Q for x in out]


def to_float64(x: int) -> float:
    """big.Float.SetInt(x).Float64(): round half to even, +-Inf when the rounded value exceeds the largest double."""
    try:
        return float(x)
    except OverflowError:
        return math.inf if x > 0 else -math.inf


def scaleDown(coeff: int, n: float) -> float:
    x = to_float64(coeff)
    x /= n
    return x


def _centre(c: int, Q: int) -> int:
    c %= Q
    return c - Q if c >= Q >> 1 else c


def complex128div(n: complex, m: complex) -> complex:
    """Go's runtime complex division (runtime/complex.go), for the finite, non-zero real divisors used here."""
    a, b, c, d = n.real, n.imag, m.real, m.imag
    assert abs(c) >= abs(d) and math.isfinite(c) and c != 0
    ratio = d / c
    denom = c + ratio * d
    e = (a + b * ratio) / denom
    f = (b - a * ratio) / denom
    assert not (math.isnan(e) and math.isnan(f))
    return complex(e, f)


def polyToComplexNoCRT(coeffs, log_slots: int, scale: float, N: int, Q: int):
    slots = 1 << log_slots
    maxCols = N >> 1
    gap = maxCols // slots
    values = [0j] * slots
    for i in range(slots):
        c = int(coeffs[i * gap])
        values[i] = complex(-float((Q - c) & MASK64), 0) if c >= Q >> 1 else complex(float(c), 0)
    for i in range(slots):
        c = int(coeffs[maxCols + i * gap])
        y = complex(0, -float((Q - c) & MASK64)) if c >= Q >> 1 else complex(0, float(c))
        values[i] = complex(values[i].real + y.real, values[i].imag + y.imag)
    return [complex128div(v, complex(scale, 0)) for v in values]


def polyToComplexCRT(r: "O.Ring", p, log_slots: int, scale: float):
    maxCols = r.NthRoot() >> 2
    slots = 1 << log_slots
    gap = maxCols // slots
    big = PolyToBigint(r, p, gap)
    Q = r.ModulusAtLevel[r.Level()]
    values = [complex(scaleDown(_centre(big[i], Q), scale), 0) for i in range(slots)]
    for i in range(slots):
        y = complex(0, scaleDown(_centre(big[slots + i], Q), scale))
        values[i] = complex(values[i].real + y.real, values[i].imag + y.imag)
    return values


def polyToFloatNoCRT(coeffs, scale: float, Q: int):
    return [-float((Q - int(c)) & MASK64) / scale if int(c) >= Q >> 1 else float(int(c)) / scale for c in coeffs]


def polyToFloatCRT(r: "O.Ring", p, scale: float):
    Q = r.ModulusAtLevel[r.Level()]
    return [scaleDown(_centre(x, Q), scale) for x in PolyToBigint(r, p, 1)]


def go_round(x: float) -> float:
    """math.Round: half away from zero, sign of zero kept, NaN / Inf unchanged."""
    if math.isnan(x) or math.isinf(x):
        return x
    t = float(math.trunc(x))
    if abs(x - t) >= 0.5:
        t += math.copysign(1.0, x)
    return math.copysign(t, x)


def decode_public(ringQ: "O.Ring", pt, level: int, log_slots: int, scale: float, is_ntt: bool, logprec: float = 0, is_batched: bool = True,
                  rt=None):
    """Encoder.decodePublic into []complex128 (batched) or []float64 (IsBatched = false, N values)."""
    r = ringQ.AtLevel(level)
    buff = np.array(pt[: level + 1], dtype=U64)
    if is_ntt:
        r.INTT(buff, buff)
    N = ringQ.N()
    Q0 = ringQ.SubRings[0].Modulus
    if not is_batched:
        return polyToFloatNoCRT(buff[0], scale, Q0) if level == 0 else polyToFloatCRT(r, buff, scale)
    slots = 1 << log_slots
    vals = polyToComplexNoCRT(buff[0], log_slots, scale, N, Q0) if level == 0 else polyToComplexCRT(r, buff, log_slots, scale)
    m = 2 * N
    SF.special_fft(vals, slots, m, rot_group(m), rt if rt is not None else get_roots_complex128(m))
    if logprec != 0:
        s = math.pow(2.0, logprec)
        vals = [complex(go_round(v.real * s) / s, go_round(v.imag * s) / s) for v in vals]
    return vals

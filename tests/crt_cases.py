"""Chains and edge sets for the multiword CRT decoders (csrc/crt.cuh under dec_crt_kernel<W> and bgv_dec_crt_kernel<W>), shared by
tests/test_crt_model_cpu.py (a restatement of the device arithmetic, no GPU) and tests/test_gpu_crt_decode.py (the kernels).

The register width W (16, 32 or 64 words) follows from the SUMMED bit lengths of q_0..q_level (crt_words), not from bits(Q_level). The
chains put those sums exactly on the word boundaries, with primes just below 2^b so that bits(Q_level) is the full 64 W and the top word
of Q is set. All values are Python ints; the exact reference is plain integer arithmetic."""
from __future__ import annotations

import functools
import math

import numpy as np

from oracle import oracle as O

LOGN = 10
N = 1 << LOGN
MAX_WORDS = 64


def primes_below(bits, m, count, above=False):
    """`count` distinct primes = 1 mod m with `bits` bits: the largest ones below 2^bits, or the smallest above 2^(bits-1)."""
    out = []
    x = ((1 << (bits - 1)) // m + 1) * m + 1 if above else ((1 << bits) - 1) // m * m + 1
    while len(out) < count:
        if O.is_prime(x):
            out.append(x)
        x += m if above else -m
    assert all(p.bit_length() == bits for p in out)
    return out


def build_chain(spec, m=2 * N, above=False):
    """Moduli for a list of bit lengths, each taken from its own descending stream of primes, so repeated lengths stay distinct."""
    pools = {b: iter(primes_below(b, m, spec.count(b), above)) for b in set(spec)}
    return [next(pools[b]) for b in spec]


def crt_words(q, level):
    """crt_words (crt.cuh): ceil(sum of bit lengths of q_0..q_level / 64)."""
    return (sum(x.bit_length() for x in q[: level + 1]) + 63) // 64


def crt_width(words):
    """crt_width (crt.cuh): the register width the decoders launch, or None past kMaxCrtWords (refused before any launch)."""
    if words > MAX_WORDS:
        return None
    return 16 if words <= 16 else 32 if words <= 32 else 64


def modulus(q, level):
    Q = 1
    for x in q[: level + 1]:
        Q *= x
    return Q


# Chain A (61-bit rows on the integer pipe): the bit-length prefix sums reach 1024 at level 16, 2048 at level 33 and 4096 at level 67;
# the prime after each of those opens one more word (17, 33 and 65 words).
SPEC_A = [61] * 16 + [48] + [61] * 16 + [48] + [61] * 32 + [48] * 2 + [61]
# level -> (words, W); W None = refused
BOUNDARY_A = {16: (16, 16), 17: (17, 32), 33: (32, 32), 34: (33, 64), 67: (64, 64), 68: (65, None)}
FULL_A = (16, 33, 67)                      # levels where bits(Q_level) = 64 W exactly
# Chain B: 45-bit rows (FP64-pipe transforms at N = 2^10) inside the W = 32 and W = 64 prefixes.
SPEC_B = [61] * 12 + [45] * 8 + [61] * 16
BOUNDARY_B = {19: (18, 32), 35: (33, 64)}
# Chain R: 61-bit primes just ABOVE 2^60. 68 of them sum to 4148 bits (65 words, refused) while Q itself has only 4081 bits.
SPEC_R = [61] * 68
REFUSE_R = 67


@functools.lru_cache(None)
def t60():
    """A 60-bit plaintext modulus = 1 mod 1024 but not mod 2048: ring T has 512 slots, so N = 2^10 decodes at gap 2, and t > 2^59
    makes the Horner step's MForm and BRedAdd work on full-width residues."""
    x = ((1 << 60) - 1) // 2048 * 2048 + 1025
    while not O.is_prime(x):
        x -= 2048
    return x


@functools.lru_cache(None)
def chain_a():
    return build_chain(SPEC_A)


@functools.lru_cache(None)
def chain_b():
    return build_chain(SPEC_B)


@functools.lru_cache(None)
def chain_r():
    return build_chain(SPEC_R, above=True)


# ---- the device arithmetic, restated (crt.cuh crt_exact_load<W>) ----------------------------------------------------------

class Crt:
    """CRT constants of one level, as build_crt lays them out (q, (Q/q_k)^-1 mod q_k, 1 / q_k as a double, Q/q_k, Q, Q >> 1)."""

    def __init__(self, q, level, W=None):
        self.q = list(q[: level + 1])
        self.L = level + 1
        self.Q = modulus(q, level)
        self.Qh = self.Q >> 1
        self.words = crt_words(q, level)
        self.W = W or crt_width(self.words)
        self.qhat = [self.Q // x for x in self.q]
        self.inv = [pow(h % x, -1, x) for h, x in zip(self.qhat, self.q)]
        self.rq = [1.0 / float(x) for x in self.q]            # Python floats are IEEE doubles, round to nearest


def quotient(C: Crt, v):
    """f = sum_k v_k * (1 / q_k) in limb order, each product and sum rounded to nearest (__dmul_rn / __dadd_rn), and t = (u64) f."""
    f = 0.0
    for vk, r in zip(v, C.rq):
        f = f + float(vk) * r                                   # float(int) rounds to nearest even, like the (double) cast of a u64
    return int(f)


def crt_exact(C: Crt, X):
    """crt_exact_load<W> for the rows X mod q_k. Returns (acc, info): acc the W + 1 words as one int (must equal X), info the branches."""
    v = [(X % x) * i % x for x, i in zip(C.q, C.inv)]
    S = sum(vk * h for vk, h in zip(v, C.qhat))
    t = quotient(C, v)
    mod = 1 << (64 * (C.W + 1))
    acc = (S - t * C.Q) % mod                                   # two's complement over W + 1 words
    top = acc >> (64 * C.W)
    info = {"S_carry": S >> (64 * C.W) != 0}
    if top >> 63:                                               # t overestimated: + Q
        info["t"] = "over"
        acc = (acc + C.Q) % mod
    else:
        info["accW"] = top != 0
        low = acc & ((1 << (64 * C.W)) - 1)
        info["ge_Q"] = low >= C.Q
        if top != 0 or low >= C.Q:                              # acc[W] != 0 || mw_ge(acc, Q)
            info["t"] = "under"
            acc = (acc - C.Q) % mod
        else:
            info["t"] = "exact"
    return acc, info


def f_error_bound(C: Crt):
    """An upper bound on |f - S/Q|: per term, the rounding of (double)v, of 1/q, of the product and of the running sum."""
    u = 2.0 ** -53
    bound, s = 0.0, 0.0
    for _ in range(C.L):
        s += 1.0
        bound += 4 * u + u * s                                  # v/q < 1: three relative roundings of a term below 1, one of a sum <= s
    return bound


def words_to_double(m, W):
    """words_to_double<W> (encoder.cu) of the magnitude m < 2^(64 W). Returns (double, info)."""
    info = {}
    if m == 0:
        return 0.0, {"path": "zero"}
    bl = m.bit_length()
    if bl <= 64:
        return float(m), {"path": "u64"}
    s = bl - 64
    ws, bs = s >> 6, s & 63
    words = [(m >> (64 * w)) & ((1 << 64) - 1) for w in range(W)]
    win, sticky_low, sticky_ws = 0, 0, 0
    for w in range(W):
        if w < ws:
            sticky_low |= words[w]
        elif w == ws:
            win = (words[w] >> bs) if bs else words[w]
            sticky_ws = ((words[w] << (64 - bs)) & ((1 << 64) - 1)) if bs else 0
        elif w == ws + 1 and bs:
            win |= (words[w] << (64 - bs)) & ((1 << 64) - 1)
    mant = win >> 11
    rnd = (win >> 10) & 1
    st_win = (win & 0x3FF) != 0 or sticky_ws != 0
    st = st_win or sticky_low != 0
    info = {"path": "window", "ws": ws, "bs0": bs == 0, "rnd": bool(rnd)}
    if rnd and not st:
        info["round"] = "tie_up" if mant & 1 else "tie_down"
    elif rnd and not st_win and sticky_low:
        info["round"] = "sticky_low_up"                          # a tie broken only by a word below the window
    elif rnd:
        info["round"] = "up"
    else:
        info["round"] = "down"
    if rnd and (st or (mant & 1)):
        mant += 1
    info["carry"] = mant >> 53 != 0
    e = s + 11
    if e >= 972:
        info["inf"] = "big"
        return float("inf"), info
    if e == 971 and mant >> 53:
        info["inf"] = "tie"
        return float("inf"), info
    return math.ldexp(float(mant), e), info


def ckks_value(C: Crt, X, scale):
    """dec_crt_kernel<W>: crt_exact, centre at Q >> 1 (mw_ge against Qh), round to double, negate, divide by the scale."""
    acc, info = crt_exact(C, X)
    ge = acc >= C.Qh
    info["ge"] = ge
    mag = C.Q - acc if ge else acc
    x, winfo = words_to_double(mag, C.W)
    info.update({"w_" + k: val for k, val in winfo.items()})
    if ge:
        x = -x
    return x / scale, acc, info


def bgv_value(C: Crt, X, t):
    """bgv_dec_crt_kernel<W> before its final MulScalar(scale^-1): Horner r <- MForm(r) + BRedAdd(w) mod t over the words from the top,
    then - Q mod t when acc >= Q >> 1. Returns (r, acc, ge)."""
    acc, info = crt_exact(C, X)
    ge = acc >= C.Qh
    r = 0
    for w in range(C.W - 1, -1, -1):
        word = (acc >> (64 * w)) & ((1 << 64) - 1)
        a = (r << 64) % t                                       # mform: canonical r 2^64 mod t
        b = word % t                                            # bred_add
        r = a + b
        assert r < 2 * t < 1 << 64
        r = r - t if r >= t else r                              # cred
    if ge:
        r = r + t - C.Q % t
        r = r - t if r >= t else r
    return r, acc, ge


# ---- exact references ---------------------------------------------------------------------------------------------------

def to_float64(x: int) -> float:
    """big.Float.SetInt(x).Float64(): round half to even, +-Inf once the rounded value passes the largest double."""
    try:
        return float(x)
    except OverflowError:
        return float("inf") if x > 0 else float("-inf")


def centred(X, Q):
    return X - Q if X >= Q >> 1 else X


# ---- edge sets ----------------------------------------------------------------------------------------------------------

def near_integer(C: Crt, limit=1 << 12):
    """X whose S/Q lies within 2^-40 of an integer (X or Q - X small), chosen so that the double quotient estimate is exact,
    one too small (the >= Q subtraction) and one too large (the + Q on the negative branch): two of each kind where found."""
    found = {"exact": [], "under": [], "over": []}
    for j in range(3, limit):
        for X in (j, C.Q - j):
            kind = crt_exact(C, X)[1]["t"]
            if len(found[kind]) < 2:
                found[kind].append(X)
        if all(len(v) == 2 for v in found.values()):
            break
    return found["exact"] + found["under"] + found["over"]


def tie(mant54_odd, e):
    """M 2^e with M an odd 54-bit integer: exactly halfway between two doubles."""
    return mant54_odd << e


def magnitudes(rng):
    """CKKS magnitudes at the edges of words_to_double. The tie below rounds down (even mantissa), the next up (odd mantissa)."""
    even_tie = (1 << 53) | (0x5A5A5A5A5A5A4 << 1) | 1              # 54 bits, mantissa (M >> 1) even, round bit set
    odd_tie = even_tie + 2                                          # mantissa odd
    out = []
    for b in (53, 54, 64, 65, 127, 128, 129):                      # top bit b - 1 set, random below
        out.append((1 << (b - 1)) | int.from_bytes(rng.bytes(17), "little") & ((1 << (b - 1)) - 1))
    for e in (0, 11, 20, 90, 150, 400):                              # window inside word 0, straddling words, high
        out += [tie(even_tie, e), tie(odd_tie, e)]
    for e in (150, 300):                                            # a tie whose only sticky bit lives in word 0, below the window
        out.append(tie(even_tie, e) + 1)
    for bl in (128, 192, 640):                                      # window = one whole word (bs = 0): ties and a sticky below
        e = bl - 54
        out += [tie(even_tie, e), tie(odd_tie, e), tie(even_tie, e) + 1, tie(even_tie, e) + (1 << (e - 1))]
    for e in (11, 74, 300):                                         # 53 ones, round bit set: the mantissa carries to 2^53
        out.append(((1 << 54) - 1) << e)
    out += [((1 << 53) - 1) << 971,                                 # largest finite double
            (1 << 1024) - (1 << 970) - 1,                           # just below the tie: rounds to the largest finite
            (1 << 1024) - (1 << 970),                               # the tie: rounds to 2^1024 = +Inf
            1 << 1024,
            (1 << 4000) - 1, 1 << 4000, (1 << 4000) + (1 << 3946), (1 << 4000) + 12345]
    return out


def edge_values(C: Crt, rng):
    """The CRT values X in [0, Q) the kernels must rebuild: trivial values, the centring boundary, near-integer quotients, all-ones
    words, then the CKKS magnitudes as m and Q - m where m < Q / 2."""
    Q, Qh = C.Q, C.Qh
    xs = [0, 1, 2, Q - 1, Q - 2, Qh - 1, Qh, Qh + 1]
    xs += near_integer(C)
    for k in (1, 2, C.W // 2, C.W - 1):                             # the low k words all ones, and Q minus that
        ones = (1 << (64 * k)) - 1
        if ones < Q:
            xs += [ones, Q - ones]
    alt = sum(((1 << 64) - 1) << (128 * i) for i in range(C.W // 2)) % Q
    xs += [alt, Q - 1 - alt]
    for m in magnitudes(rng):
        if m < Q - Qh:                                              # -m centres back to -m: Q - m >= Qh
            xs += [m, Q - m] if m < Qh else [Q - m]
    return [x % Q for x in xs]


def fill_uniform(xs, count, Q, rng):
    """xs followed by uniform values of [0, Q) up to `count`."""
    assert len(xs) <= count, (len(xs), count)
    out = list(xs)
    nbytes = (Q.bit_length() + 71) // 8
    while len(out) < count:
        out.append(int.from_bytes(rng.bytes(nbytes), "little") % Q)
    return out


def rows_of(xs, q, level, mul=1):
    """(level + 1, len(xs)) uint64 rows: (X mul) mod q_k."""
    if mul != 1:
        Q = modulus(q, level)
        xs = [x * mul % Q for x in xs]
    return np.array([[x % qk for x in xs] for qk in q[: level + 1]], dtype=np.uint64)

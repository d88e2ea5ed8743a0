"""CPU restatement of the device samplers' random streams (csrc/encrypt.cu, counter layout in include/lattigo_b200.h): Philox4x32-10
and, for every sampler, exactly what its kernel writes for a given (seed, stream_id, moduli / limbs, batch, N, parameters).
Vectorised numpy; words are held in uint64 arrays with values below 2^32.

The Gaussian is the exception: the kernel's log / sqrt / cospi are not correctly rounded, so this module gives the exact inputs
of every attempt (u1, u2, sign) and a float64 evaluation that flags the coefficients whose outcome a few ulps could change.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np

U64 = np.uint64
M32 = U64(0xFFFFFFFF)
KIND_UNIFORM, KIND_TERNARY_P, KIND_TERNARY_H, KIND_GAUSSIAN = 0, 1, 2, 3
KIND_SHIFT = 30          # the kind sits in bits 30..31 of the polynomial word
MAX_ROWS = 128           # kMaxRows (csrc/engine.h): the uniform's polynomial index is batch * MAX_ROWS + limb
TWO_M53 = 1.0 / 9007199254740992.0


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11). ctr: four broadcastable integer arrays (or ints), key: two. Returns four uint64
    arrays of 32-bit words."""
    x, y, z, w = (np.asarray(c, dtype=U64) & M32 for c in ctr)
    k0, k1 = (np.asarray(k, dtype=U64) & M32 for k in key)
    x, y, z, w = np.broadcast_arrays(x, y, z, w)
    for _ in range(10):
        p0 = U64(0xD2511F53) * x                 # < 2^64: exact
        p1 = U64(0xCD9E8D57) * z
        x, y, z, w = (p1 >> U64(32)) ^ y ^ k0, p1 & M32, (p0 >> U64(32)) ^ w ^ k1, p0 & M32
        k0 = (k0 + U64(0x9E3779B9)) & M32
        k1 = (k1 + U64(0xBB67AE85)) & M32
    return x, y, z, w


def make_key(seed: int, stream_id: int):
    """(k0, k1, counter word 2) of a (seed, stream_id) pair: make_key in csrc/encrypt.cu."""
    seed &= (1 << 64) - 1
    stream_id &= (1 << 64) - 1
    k1 = ((seed >> 32) ^ ((stream_id >> 32) * 0x85EBCA6B)) & 0xFFFFFFFF
    return seed & 0xFFFFFFFF, k1, stream_id & 0xFFFFFFFF


def counter(kind: int, seed: int, stream_id: int, poly, coeff, attempt):
    """The full Philox input (c0, c1, c2, c3, k0, k1) of one draw. For ternary {H} `coeff` is the attempt and `attempt` is 0,
    as in the kernel."""
    k0, k1, s = make_key(seed, stream_id)
    poly = np.asarray(poly, dtype=U64) | U64(kind << KIND_SHIFT)
    return (np.asarray(coeff, dtype=U64), poly, U64(s), np.asarray(attempt, dtype=U64), U64(k0), U64(k1))


def draw(kind: int, seed: int, stream_id: int, poly, coeff, attempt):
    c = counter(kind, seed, stream_id, poly, coeff, attempt)
    return philox4x32_10(c[:4], c[4:])


def _word53(hi, lo):
    return (hi << U64(21)) | (lo >> U64(11))


def uniform(seed: int, stream_id: int, moduli, limbs, batch: int, N: int) -> np.ndarray:
    """lgpu_sample_uniform: (batch, rows, N) with row r uniform in [0, moduli[r]); limbs[r] is the row's global limb index (P limbs
    are nQ + j). Per attempt, the masked words (x:y) then (z:w); the first below q is taken."""
    out = np.zeros((batch, len(moduli), N), dtype=U64)
    for r, (q, limb) in enumerate(zip(moduli, limbs)):
        q = int(q)
        mask = U64((1 << (q - 1).bit_length()) - 1)
        qq = U64(q)
        b, i = np.meshgrid(np.arange(batch, dtype=U64), np.arange(N, dtype=U64), indexing="ij")
        b, i = b.ravel(), i.ravel()
        poly = b * U64(MAX_ROWS) + U64(limb)
        val = np.zeros(batch * N, dtype=U64)
        pending = np.arange(batch * N)
        a = 0
        while pending.size:
            x, y, z, w = draw(KIND_UNIFORM, seed, stream_id, poly[pending], i[pending], a)
            v1 = ((x << U64(32)) | y) & mask
            v2 = ((z << U64(32)) | w) & mask
            ok1, ok2 = v1 < qq, v2 < qq
            val[pending] = np.where(ok1, v1, v2)
            pending = pending[~(ok1 | ok2)]
            a += 1
        out[:, r] = val.reshape(batch, N)
    return out


def ternary_p(seed: int, stream_id: int, batch: int, N: int, p: float) -> np.ndarray:
    """lgpu_sample_ternary with hamming_weight = 0: (batch, N) int64; non-zero when u = 53 bits / 2^53 < p, sign from bit 0 of z."""
    b = np.arange(batch, dtype=U64)[:, None]
    i = np.arange(N, dtype=U64)[None, :]
    x, y, z, _ = draw(KIND_TERNARY_P, seed, stream_id, b, i, 0)
    u = _word53(x, y).astype(np.float64) * TWO_M53
    return np.where(u < p, np.where(z & U64(1), 1, -1), 0).astype(np.int64)


def ternary_p_nonzero_probability(p: float) -> float:
    """P(coefficient != 0) of ternary_p: ceil(p 2^53) / 2^53."""
    return float(np.ceil(p * 9007199254740992.0)) * TWO_M53


def ternary_h(seed: int, stream_id: int, batch: int, N: int, h: int) -> np.ndarray:
    """lgpu_sample_ternary with hamming_weight = h > 0 (clamped to N): (batch, N) int64. Attempt a gives the candidates
    (x & (N-1), sign y & 1) then (z & (N-1), sign w & 1); the non-zero coefficients are the first h distinct positions of the
    interleaved sequence x0, z0, x1, z1, ..."""
    h = min(h, N)
    out = np.zeros((batch, N), dtype=np.int64)
    # expected candidates for h distinct positions: N (H_N - H_{N-h}); draw a margin above it and extend if short
    need = N * float(np.sum(1.0 / np.arange(N - h + 1, N + 1))) if h else 0.0
    attempts = int(need * 0.6) + 64
    for b in range(batch):
        while True:
            x, y, z, w = draw(KIND_TERNARY_H, seed, stream_id, b, np.arange(attempts, dtype=U64), 0)
            pos = np.stack([x, z], axis=1).ravel() & U64(N - 1)
            neg = (np.stack([y, w], axis=1).ravel() & U64(1)) == 0
            _, first = np.unique(pos, return_index=True)
            if len(first) >= h:
                break
            attempts *= 2
        order = np.sort(first)[:h]
        out[b, pos[order].astype(np.int64)] = np.where(neg[order], -1, 1)
    return out


def gaussian_draws(seed: int, stream_id: int, b, i, a):
    """(u1, u2, negative) of attempt a of coefficient i of polynomial b: u1 in (0, 1] and u2 in [0, 1) are exact float64
    (53-bit words), negative is bit 0 of w (not part of u2)."""
    x, y, z, w = draw(KIND_GAUSSIAN, seed, stream_id, b, i, a)
    u1 = (_word53(x, y).astype(np.float64) + 1.0) * TWO_M53
    u2 = _word53(z, w).astype(np.float64) * TWO_M53
    return u1, u2, (w & U64(1)) == 1


def abs_cospi2(u2):
    """|cos(2 pi u2)| within a few ulps, also near its zeros: 2 u2 is reduced exactly to t in [-1/4, 1/4] around a multiple of 1/2."""
    r = 2.0 * u2
    n = np.rint(2.0 * r)
    t = r - 0.5 * n                                  # exact
    return np.where(n % 2 == 0, np.cos(np.pi * t), np.abs(np.sin(np.pi * t)))


def gaussian_m(u1, u2, sigma: float):
    """m = sqrt(-2 ln u1) |cos 2 pi u2| sigma in float64, within a few ulps of the exact value."""
    return np.sqrt(-2.0 * np.log(u1)) * abs_cospi2(u2) * sigma


def gaussian_float64(seed: int, stream_id: int, batch: int, N: int, sigma: float, bound: float, margin: float = 2.0 ** -40):
    """lgpu_sample_gaussian evaluated in float64: the first attempt with m <= bound gives sign * floor(m + 1/2). Returns
    (values (batch, N) int64, decisive m, decisive attempt, near): near marks the coefficients where some attempt up to the
    decisive one has m within `margin` (relative) of the bound, or the decisive m is within `margin` of a half-integer -- the
    only ones where the device's last-ulp differences can change the value."""
    n = batch * N
    val = np.zeros(n, dtype=np.int64)
    m_dec = np.zeros(n)
    att = np.zeros(n, dtype=np.int64)
    near = np.zeros(n, dtype=bool)
    b_all = np.repeat(np.arange(batch, dtype=U64), N)
    i_all = np.tile(np.arange(N, dtype=U64), batch)
    pending = np.arange(n)
    a0, k = 0, 1
    while pending.size:
        a = np.arange(a0, a0 + k, dtype=U64)[None, :]
        u1, u2, neg = gaussian_draws(seed, stream_id, b_all[pending][:, None], i_all[pending][:, None], a)
        m = gaussian_m(u1, u2, sigma)
        acc = m <= bound
        hit = acc.any(axis=1)
        j = np.argmax(acc, axis=1)                        # first accepted attempt in this window
        last = np.where(hit, j, k - 1)
        upto = np.arange(k)[None, :] <= last[:, None]
        near[pending] |= (upto & (np.abs(m - bound) <= margin * bound)).any(axis=1)
        rows = np.arange(len(pending))
        md = m[rows, j]
        v = np.floor(md + 0.5).astype(np.int64)
        v = np.where(neg[rows, j], -v, v)
        done = pending[hit]
        val[done] = v[hit]
        m_dec[done] = md[hit]
        att[done] = a0 + j[hit]
        near[done] |= np.abs(md[hit] - (np.floor(md[hit]) + 0.5)) <= margin * np.maximum(md[hit], 0.5)
        pending = pending[~hit]
        a0 += k
        k = min(2 * k, 4096)
    return val.reshape(batch, N), m_dec.reshape(batch, N), att.reshape(batch, N), near.reshape(batch, N)


# ---- the exact laws the samplers draw from (goodness-of-fit references) ----------------------------------------------------
def uniform_bin_probabilities(q: int, nbins: int) -> np.ndarray:
    """P(floor(v nbins / q) = k) for v uniform in [0, q): bin k holds v in [ceil(k q / nbins), ceil((k+1) q / nbins))."""
    edges = [-(-k * q // nbins) for k in range(nbins + 1)]
    return np.array([(edges[k + 1] - edges[k]) / q for k in range(nbins)])


def uniform_residue_probabilities(q: int, m: int) -> np.ndarray:
    """P(v mod m = r) for v uniform in [0, q)."""
    return np.array([(q - r + m - 1) // m / q for r in range(m)])


def gaussian_law(sigma: float, bound: float, edges) -> np.ndarray:
    """Probabilities of the truncated discrete Gaussian over signed bins. edges: increasing integers 0 = e_0 < 1 = e_1 < ... with
    e_n above every |v|; bin j of |v| is [e_j, e_{j+1}), i.e. m in [e_j - 1/2, e_{j+1} - 1/2) cut to [0, bound]. Returned in the
    order (-bin n-1, ..., -bin 1, bin 0 = {0}, +bin 1, ..., +bin n-1): 0 has P(m < 1/2), every other bin half its mass per sign."""
    from scipy.special import ndtr
    e = np.asarray(edges, dtype=np.float64)
    lo = np.clip(e[:-1] - 0.5, 0.0, bound)
    hi = np.clip(e[1:] - 0.5, 0.0, bound)
    mass = ndtr(-lo / sigma) - ndtr(-hi / sigma)           # P(lo <= |Z| sigma < hi) / 2
    mass[-1] = ndtr(-lo[-1] / sigma) - ndtr(-bound / sigma)
    total = 0.5 - ndtr(-bound / sigma)
    half = mass[1:] / (2.0 * total)
    return np.concatenate([half[::-1], [mass[0] / total], half])


def gaussian_bin_index(v, edges) -> np.ndarray:
    """The gaussian_law bin of every value v."""
    n = len(edges) - 1
    j = np.searchsorted(np.asarray(edges), np.abs(v), side="right") - 1
    return np.where(v < 0, n - 1 - j, n - 1 + j)

// crt.cuh -- exact CRT reconstruction of one coefficient mod Q_level in W 64-bit register words (W = 16, 32 or 64), shared by the CKKS
// decoder (encoder.cu: rounded to double) and the BGV decoder (bgv_encoder.cu: reduced mod t). Device side: the CrtTab view of the per-call
// constant blob, mw_ge and crt_exact; host side: the blob (build_crt) and the word-count helpers.
#pragma once
#include <algorithm>
#include <cstring>
#include <vector>
#include "engine.h"
#include "modarith.cuh"

namespace lgpu {

constexpr int kMaxCrtWords = 64;     // the bit lengths of q_0..q_level sum to at most 4096 (crt_words)

// Per-call constants of the CRT reconstruction at `level` (host-built): for k <= level, q_k, BRed hi / lo, (Q/q_k)^-1 mod q_k and 1/q_k;
// then Q/q_k as W words each, Q and floor(Q / 2) as W words.
struct CrtTab {
    const u64* q;        // [L]
    const u64* bhi;      // [L]
    const u64* blo;      // [L]
    const u64* inv;      // [L]
    const double* rq;    // [L] 1 / q_k (quotient estimate)
    const u64* qhat;     // [L][W]
    const u64* Q;        // [W]
    const u64* Qh;       // [W]
    int L;
};

// a >= b over the low W words, branch-free from the least significant word up (the most significant difference decides)
template <int W>
__device__ __forceinline__ bool mw_ge(const u64 (&a)[W + 1], const u64* __restrict__ b) {
    bool ge = true;
#pragma unroll
    for (int w = 0; w < W; w++) {
        const u64 bw = b[w];
        ge = a[w] > bw ? true : (a[w] < bw ? false : ge);
    }
    return ge;
}

// exact X = CRT(rows 0..L-1) mod Q: S = sum_k [x_k (Q/q_k)^-1]_{q_k} (Q/q_k) < L Q, t = floor(S / Q) = floor(sum_k [.]_{q_k} / q_k) estimated
// in double (error below 2^-37, so within one of t), S - t Q corrected by at most one +-Q. Result canonical in [0, Q).
// `load(k)` gives the word of row k (any 64-bit value: it is reduced here).
template <int W, class Load>
__device__ __forceinline__ void crt_exact_load(Load load, const CrtTab& T, u64 (&acc)[W + 1]) {
#pragma unroll
    for (int w = 0; w <= W; w++) acc[w] = 0;
    double f = 0.0;
    for (int k = 0; k < T.L; k++) {
        const u64 qk = T.q[k];
        const u64 v = bred(bred_add(load(k), qk, T.bhi[k]), T.inv[k], qk, T.bhi[k], T.blo[k]);
        f = __dadd_rn(f, __dmul_rn((double)v, T.rq[k]));
        const u64* h = T.qhat + (size_t)k * W;
        u64 carry = 0;
#pragma unroll
        for (int w = 0; w < W; w++) {
            u64 hi, lo;
            mul128(v, h[w], hi, lo);
            lo += carry; hi += lo < carry;
            acc[w] += lo; hi += acc[w] < lo;
            carry = hi;
        }
        acc[W] += carry;
    }
    u64 t = (u64)f;                                         // f >= 0: truncation = floor
    // acc -= t Q (two's complement over W + 1 words)
    u64 borrow = 0, carry = 0;
#pragma unroll
    for (int w = 0; w < W; w++) {
        u64 hi, lo;
        mul128(t, T.Q[w], hi, lo);
        lo += carry; hi += lo < carry; carry = hi;
        const u64 a = acc[w];
        const u64 d = a - lo - borrow;
        borrow = (a < lo) || (a - lo < borrow);
        acc[w] = d;
    }
    acc[W] = acc[W] - carry - borrow;
    if ((long long)acc[W] < 0) {                            // t overestimated: add Q back
        u64 c = 0;
#pragma unroll
        for (int w = 0; w < W; w++) {
            const u64 s = acc[w] + T.Q[w];
            const u64 c1 = s < acc[w];
            acc[w] = s + c;
            c = c1 | (acc[w] < s);
        }
        acc[W] += c;
    } else {
        if (acc[W] != 0 || mw_ge<W>(acc, T.Q)) {         // acc >= Q
            u64 br = 0;
#pragma unroll
            for (int w = 0; w < W; w++) {
                const u64 a = acc[w], bq = T.Q[w];
                acc[w] = a - bq - br;
                br = (a < bq) || (a - bq < br);
            }
            acc[W] -= br;
        }
    }
}

template <int W>
__device__ __forceinline__ void crt_exact(const u64* __restrict__ x, size_t row_stride, const CrtTab& T, u64 (&acc)[W + 1]) {
    crt_exact_load<W>([&](int k) { return x[(size_t)k * row_stride]; }, T, acc);
}

// ---- host side -------------------------------------------------------------------------------------------------------

// little-endian multiword helpers
inline void mw_mul_small(std::vector<u64>& a, u64 m) {
    unsigned __int128 c = 0;
    for (auto& w : a) { c += (unsigned __int128)w * m; w = (u64)c; c >>= 64; }
    if (c) a.push_back((u64)c);
}
inline std::vector<u64> mw_div_small(const std::vector<u64>& a, u64 d) {
    std::vector<u64> q(a.size());
    unsigned __int128 r = 0;
    for (size_t i = a.size(); i-- > 0;) { r = (r << 64) | a[i]; q[i] = (u64)(r / d); r %= d; }
    return q;
}

inline int crt_words(const Ctx& c, int level) {
    int bits = 0;
    for (int k = 0; k <= level; k++) bits += 64 - __builtin_clzll(c.Q[k]);
    return (bits + 63) / 64;
}
inline int crt_width(int words) { return words <= 16 ? 16 : words <= 32 ? 32 : 64; }

// blob layout: q | bhi | blo | inv | rq (doubles) | qhat [L][W] | Q [W] | Qh [W]
inline std::vector<u64> build_crt(const Ctx& c, int level, int W) {
    const int L = level + 1;
    std::vector<u64> Q{1};
    for (int k = 0; k < L; k++) mw_mul_small(Q, c.Q[k]);
    Q.resize(W, 0);
    std::vector<u64> blob((size_t)5 * L + (size_t)L * W + 2 * (size_t)W, 0);
    for (int k = 0; k < L; k++) {
        const u64 qk = c.Q[k];
        u64 hm = 1;                                               // (Q/q_k) mod q_k
        for (int j = 0; j < L; j++)
            if (j != k) hm = h_mulmod(hm, c.Q[j] % qk, qk);
        blob[k] = qk;
        blob[L + k] = c.sub[k].bred_hi;
        blob[2 * L + k] = c.sub[k].bred_lo;
        blob[3 * L + k] = h_invmod(hm, qk);
        const double rq = 1.0 / (double)qk;
        memcpy(&blob[4 * L + k], &rq, 8);
        const std::vector<u64> qh = mw_div_small(Q, qk);
        std::copy(qh.begin(), qh.begin() + W, blob.begin() + 5 * L + (size_t)k * W);
    }
    std::copy(Q.begin(), Q.end(), blob.begin() + 5 * L + (size_t)L * W);
    for (int w = 0; w < W; w++)                                   // Q >> 1
        blob[5 * L + (size_t)L * W + W + w] = (Q[w] >> 1) | (w + 1 < W ? Q[w + 1] << 63 : 0);
    return blob;
}

}  // namespace lgpu

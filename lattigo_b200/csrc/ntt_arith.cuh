// ntt_arith.cuh -- butterfly arithmetic shared by the transform kernels (ntt.cu, ntt_fp64.cu) and the fused
// key-switch kernels (keyswitch_fused.cu): the integer-pipe Shoup path and the FP64-pipe path.
#pragma once
#include "modarith.cuh"

namespace lgpu {

// ---- FAST path primitives ---------------------------------------------------------------------------
// x*w mod q in [0, 2q) for any x < 2^64, given wp = floor(w * 2^64 / q)
__device__ __forceinline__ u64 shoup_mul(u64 x, ulonglong2 w, u64 q) { return x * w.x - __umul64hi(x, w.y) * q; }

// CT butterfly: X = U + V*w, Y = U - V*w + 2q (lazy). nq = -q mod 2^64. The sum U + V*w - hi*q is accumulated in
// the multiplier's addend so that no separate 64-bit additions are issued for X.
__device__ __forceinline__ void fast_fwd_bfly(u64& X, u64& Y, ulonglong2 w, u64 nq, u64 twoq, u64 kq, bool corr) {
    u64 U = X;
    if (corr) U = (U >= kq) ? U - kq : U;
    const u64 V = Y;
    const u64 hi = __umul64hi(V, w.y);
    const u32 v0 = (u32)V, v1 = (u32)(V >> 32), w0 = (u32)w.x, w1 = (u32)(w.x >> 32);
    const u32 h0 = (u32)hi, h1 = (u32)(hi >> 32), n0 = (u32)nq, n1 = (u32)(nq >> 32);
    u64 acc = U + (u64)v0 * w0;
    acc += (u64)h0 * n0;
    const u32 t = v0 * w1 + v1 * w0 + h0 * n1 + h1 * n0;
    acc += (u64)t << 32;
    X = acc;
    Y = (U << 1) + twoq - acc;
}
// GS butterfly: X = U + V (optionally corrected to [0, 2q)), Y = (U - V + addq) * w in [0, 2q)
__device__ __forceinline__ void fast_inv_bfly(u64& X, u64& Y, ulonglong2 w, u64 q, u64 addq, bool corr) {
    const u64 U = X, V = Y;
    u64 s = U + V;
    if (corr) { const u64 twoq = q << 1; s = (s >= twoq) ? s - twoq : s; }
    X = s;
    Y = shoup_mul(U - V + addq, w, q);
}


// ---- FP64-pipe primitives (primes below 2^46, see ntt_fp64.cu) ----------------------------------------
#define FP_MAGIC 6755399441055744.0   /* 1.5 * 2^52 */
#define FP_TWO52 4503599627370496.0   /* 2^52 */

__device__ __forceinline__ double u2d(u64 x) { return __longlong_as_double((long long)(x | 0x4330000000000000ull)) - FP_TWO52; }
// The magic-number conversion is exact only below 2^52. The reference's NTTStandard / INTTStandard accept any uint64 that
// does not wrap its lazy arithmetic (lazily accumulated sums, AddLazy / MulCoeffsLazy outputs; ring/ntt.go:174-206 end in
// a full reduction), so user-supplied words are Barrett-reduced first when a high bit is set (rare, warp-divergent only
// when it happens).
__device__ __forceinline__ double u2d_any(u64 x, u64 q, u64 bred_hi) {
    if (x >> 52) x = bred_add(x, q, bred_hi);
    return u2d(x);
}
// integer-valued 0 <= d < 2^52
__device__ __forceinline__ u64 d2u(double d) { return (u64)__double_as_longlong(d + FP_TWO52) & 0x000FFFFFFFFFFFFFull; }

__device__ __forceinline__ double fp_mulmod(double v, double w, double q, double qinv) {
    const double h = __dmul_rn(v, w);
    const double l = __fma_rn(v, w, -h);
    const double t = __dadd_rn(__fma_rn(h, qinv, FP_MAGIC), -FP_MAGIC);
    const double r = __fma_rn(-t, q, h);
    return __dadd_rn(r, l);
}
// x mod q into (-0.66q, 0.66q)
__device__ __forceinline__ double fp_reduce(double x, double q, double qinv) {
    const double t = __dadd_rn(__fma_rn(x, qinv, FP_MAGIC), -FP_MAGIC);
    return __fma_rn(-t, q, x);
}
__device__ __forceinline__ u64 fp_canon(double x, double q, double qinv) {
    double r = fp_reduce(x, q, qinv);
    r = r < 0.0 ? r + q : r;
    return d2u(r);
}
__device__ __forceinline__ void fp_fwd_bfly(double& X, double& Y, double w, double q, double qinv) {
    const double v = fp_mulmod(Y, w, q, qinv);
    const double u = X;
    X = __dadd_rn(u, v);
    Y = __dadd_rn(u, -v);
}
__device__ __forceinline__ void fp_inv_bfly(double& X, double& Y, double w, double q, double qinv) {
    const double u = X, v = Y;
    X = __dadd_rn(u, v);
    Y = fp_mulmod(__dadd_rn(u, -v), w, q, qinv);
}

__device__ __forceinline__ int fpad(int i) { return i + (i >> 4); }



// ---- reference (Montgomery) butterflies and the chunk-round machinery ------------------------------------
// reference schedule for the forward U >= 4q correction, ring/ntt.go:275-310 (never on stage 0),
// :318 (bits.Len64(m) odd <=> stage index even), :500-518 (always on the last stage).
__device__ __forceinline__ bool fwd_reduce_flag(int s, int logN) { return (s == logN - 1) || (s > 0 && (s & 1) == 0); }

__device__ __forceinline__ void fwd_bfly(u64& X, u64& Y, u64 psi, u64 q, u64 qinv, bool reduce) {
    u64 U = X;
    u64 fourq = q << 2;
    if (reduce) U = (U >= fourq) ? U - fourq : U;
    u64 V = mred_lazy(Y, psi, q, qinv);
    X = U + V;
    Y = U + (q << 1) - V;
}
// invbutterfly, ring/ntt.go:164-171
__device__ __forceinline__ void inv_bfly(u64& X, u64& Y, u64 psi, u64 q, u64 qinv) {
    u64 U = X, V = Y;
    u64 twoq = q << 1;
    u64 s = U + V;
    X = (s >= twoq) ? s - twoq : s;
    Y = mred_lazy(U + (q << 2) - V, psi, q, qinv);
}

__host__ __device__ constexpr int round_bits(int cl, int i) {
    // radix schedule (bits per register round) for a chunk of 2^cl elements
    return cl == 12 ? 4
         : cl == 11 ? (i < 2 ? 4 : 3)
         : cl == 10 ? (i < 1 ? 4 : 3)
         : cl == 9  ? 3
         : cl == 8  ? (i < 2 ? 4 : 0)
         : cl == 7  ? (i == 0 ? 4 : (i == 1 ? 3 : 0))
         : cl == 6  ? (i < 2 ? 3 : 0)
         : cl == 5  ? (i == 0 ? 3 : (i == 1 ? 2 : 0))
         :            (i == 0 ? 4 : 0);
}
__host__ __device__ constexpr int num_rounds(int cl) { return cl >= 9 ? 3 : (cl >= 5 ? 2 : 1); }

__device__ __forceinline__ int pad_idx(int i) { return i + (i >> 4); }

// One register round of the forward transform on chunk-local stages [A, A+RB).
template <int CL, int A, int RB, bool FROM_GLOBAL, int FAST>
__device__ __forceinline__ void fwd_round(u64* sm, const u64* gsrc, const LimbConst& L,
                                          int s1, int logN, int chunk, int tid) {
    const u64 q = L.q, qinv = L.qinv;
    const u64* roots = L.roots_fwd;
    const ulonglong2* twp = L.tw_fwd;
    const u64 nq = 0ull - q, twoq = q << 1;
    constexpr int G = 16 >> RB;          // groups per thread
    constexpr int RR = 1 << RB;          // elements per group
    constexpr int LOB = CL - A - RB;     // bits of `lo`
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int g = tid * G + gi;
        const int hi = g >> LOB, lo = g & ((1 << LOB) - 1);
        const int base = (hi << (CL - A)) + lo;
        u64 x[RR];
#pragma unroll
        for (int k = 0; k < RR; k++) {
            const int idx = base + (k << LOB);
            x[k] = FROM_GLOBAL ? __ldcg(gsrc + idx) : sm[pad_idx(idx)];
        }
#pragma unroll
        for (int u = 0; u < RB; u++) {
            const int half = 1 << (RB - 1 - u);
            const int s = s1 + A + u;
            const int twbase = (1 << s) + (chunk << (A + u)) + (hi << u);
            if constexpr (FAST) {
                const bool corr = (FAST == 1) && ((L.fwd_mask >> s) & 1u);
#pragma unroll
                for (int k = 0; k < RR; k++) {
                    if (k & half) continue;
                    const ulonglong2 w = __ldg(twp + twbase + (k >> (RB - u)));
                    fast_fwd_bfly(x[k], x[k + half], w, nq, twoq, L.kq, corr);
                }
            } else {
                const bool red = fwd_reduce_flag(s, logN);
#pragma unroll
                for (int k = 0; k < RR; k++) {
                    if (k & half) continue;
                    u64 tw = __ldg(roots + twbase + (k >> (RB - u)));
                    fwd_bfly(x[k], x[k + half], tw, q, qinv, red);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < RR; k++) sm[pad_idx(base + (k << LOB))] = x[k];
    }
}


// ---- FP64 chunk rounds ---------------------------------------------------------------------------------
__host__ __device__ constexpr int fp_round_bits(int cl, int i) {
    return cl == 12 ? 4 : cl == 11 ? (i < 2 ? 4 : 3) : cl == 10 ? (i < 1 ? 4 : 3) : 0;
}

template <int CL, int A, int RB, int SRC /*0 smem, 1 global u64, 2 global raw double*/>
__device__ __forceinline__ void fp_fwd_round(double* sm, const u64* gsrc, const LimbConst& L, int s1, int chunk, int tid) {
    constexpr int G = 16 >> RB, RR = 1 << RB, LOB = CL - A - RB;
    const double q = L.fq, qinv = L.fqinv;
    const double* tw = L.ftw_fwd;
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int g = tid * G + gi;
        const int hi = g >> LOB, lo = g & ((1 << LOB) - 1);
        const int base = (hi << (CL - A)) + lo;
        double x[RR];
#pragma unroll
        for (int k = 0; k < RR; k++) {
            const int idx = base + (k << LOB);
            if (SRC == 1) x[k] = u2d(__ldcg(gsrc + idx));
            else if (SRC == 2) x[k] = __longlong_as_double((long long)__ldcg(gsrc + idx));
            else x[k] = sm[fpad(idx)];
        }
#pragma unroll
        for (int u = 0; u < RB; u++) {
            const int half = 1 << (RB - 1 - u);
            const int s = s1 + A + u;
            const int twbase = (1 << s) + (chunk << (A + u)) + (hi << u);
#pragma unroll
            for (int k = 0; k < RR; k++) {
                if (k & half) continue;
                fp_fwd_bfly(x[k], x[k + half], __ldg(tw + twbase + (k >> (RB - u))), q, qinv);
            }
        }
#pragma unroll
        for (int k = 0; k < RR; k++) sm[fpad(base + (k << LOB))] = x[k];
    }
}

// Twiddles of one forward round for this thread: G groups x (2^RB - 1) values, loaded BEFORE the barrier that
// precedes the round so that their L2 latency overlaps the barrier wait instead of following it.
template <int CL, int A, int RB>
__device__ __forceinline__ void fp_load_tw(double (&t)[15], const double* tw, int s1, int chunk, int tid) {
    constexpr int G = 16 >> RB, RR = 1 << RB, LOB = CL - A - RB;
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int hi = (tid * G + gi) >> LOB;
#pragma unroll
        for (int u = 0; u < RB; u++) {
            const int twbase = (1 << (s1 + A + u)) + (chunk << (A + u)) + (hi << u);
#pragma unroll
            for (int m = 0; m < (1 << u); m++) t[gi * (RR - 1) + (1 << u) - 1 + m] = __ldg(tw + twbase + m);
        }
    }
}
template <int CL, int A, int RB>
__device__ __forceinline__ void fp_fwd_round_tw(double* sm, const double (&t)[15], double q, double qinv, int tid) {
    constexpr int G = 16 >> RB, RR = 1 << RB, LOB = CL - A - RB;
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int g = tid * G + gi;
        const int hi = g >> LOB, lo = g & ((1 << LOB) - 1);
        const int base = (hi << (CL - A)) + lo;
        double x[RR];
#pragma unroll
        for (int k = 0; k < RR; k++) x[k] = sm[fpad(base + (k << LOB))];
#pragma unroll
        for (int u = 0; u < RB; u++) {
            const int half = 1 << (RB - 1 - u);
#pragma unroll
            for (int k = 0; k < RR; k++) {
                if (k & half) continue;
                fp_fwd_bfly(x[k], x[k + half], t[gi * (RR - 1) + (1 << u) - 1 + (k >> (RB - u))], q, qinv);
            }
        }
#pragma unroll
        for (int k = 0; k < RR; k++) sm[fpad(base + (k << LOB))] = x[k];
    }
}

// Last forward round (A + RB == CL): every group is 2^RB CONSECUTIVE coefficients, so the canonical results go straight
// from registers to global memory as 128-bit stores (no store / barrier / reload of the tile for a coalesced copy-out).
template <int CL, int A, int RB>
__device__ __forceinline__ void fp_fwd_round_tw_out(const double* sm, const double (&t)[15], double q, double qinv, int tid, u64* gdst) {
    static_assert(A + RB == CL && RB >= 1, "last round only");
    constexpr int G = 16 >> RB, RR = 1 << RB;
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int base = (tid * G + gi) << RB;
        double x[RR];
#pragma unroll
        for (int k = 0; k < RR; k++) x[k] = sm[fpad(base + k)];
#pragma unroll
        for (int u = 0; u < RB; u++) {
            const int half = 1 << (RB - 1 - u);
#pragma unroll
            for (int k = 0; k < RR; k++) {
                if (k & half) continue;
                fp_fwd_bfly(x[k], x[k + half], t[gi * (RR - 1) + (1 << u) - 1 + (k >> (RB - u))], q, qinv);
            }
        }
#pragma unroll
        for (int k = 0; k < RR; k += 2)
            *reinterpret_cast<ulonglong2*>(gdst + base + k) = make_ulonglong2(fp_canon(x[k], q, qinv), fp_canon(x[k + 1], q, qinv));
    }
}


// ---- moved here so that the persistent transform kernels (ntt_persist.cu) share them ---------------------------------
// One register round of the inverse transform (GS) on chunk-local stages [A, A+RB), processed deepest first.
template <int CL, int A, int RB, bool TO_GLOBAL, bool SCALE, int FAST>
__device__ __forceinline__ void inv_round(u64* sm, u64* gdst, const LimbConst& L,
                                          int s1, int chunk, int tid) {
    static_assert(FAST != 0, "the inverse transform has fast kernels only");
    const u64 q = L.q;
    const ulonglong2* twp = L.tw_bwd;
    const bool lazy = L.inv_lazy != 0;
    constexpr int G = 16 >> RB;
    constexpr int RR = 1 << RB;
    constexpr int LOB = CL - A - RB;
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int g = tid * G + gi;
        const int hi = g >> LOB, lo = g & ((1 << LOB) - 1);
        const int base = (hi << (CL - A)) + lo;
        u64 x[RR];
#pragma unroll
        for (int k = 0; k < RR; k++) x[k] = sm[pad_idx(base + (k << LOB))];
#pragma unroll
        for (int u = RB - 1; u >= 0; u--) {
            const int half = 1 << (RB - 1 - u);
            const int s = s1 + A + u;
            const int twbase = (1 << s) + (chunk << (A + u)) + (hi << u);
            // `done` inverse stages precede this one; lazy inputs are < 2^(done+1) q
            const int done = (CL - 1) - (A + u);
            if (SCALE && A + u == 0) {
                // very last stage of a single-pass transform: fold N^-1, canonical outputs
                const u64 addq = lazy ? (q << (done + 1)) : (q << 1);
#pragma unroll
                for (int k = 0; k < RR; k++) {
                    if (k & half) continue;
                    const u64 U = x[k], V = x[k + half];
                    const u64 a = shoup_mul(U + V, L.ninv_s, q);
                    const u64 c = shoup_mul(U - V + addq, L.last_inv_s, q);
                    x[k] = a >= q ? a - q : a;
                    x[k + half] = c >= q ? c - q : c;
                }
            } else {
                const u64 addq = lazy ? (q << (done + 1)) : (q << 1);
#pragma unroll
                for (int k = 0; k < RR; k++) {
                    if (k & half) continue;
                    const ulonglong2 w = __ldg(twp + twbase + (k >> (RB - u)));
                    fast_inv_bfly(x[k], x[k + half], w, q, addq, !lazy);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < RR; k++) {
            const int idx = base + (k << LOB);
            if (TO_GLOBAL) gdst[idx] = x[k];
            else sm[pad_idx(idx)] = x[k];
        }
    }
}


// inverse round over chunk-local stages [A, A+RB), deepest first; inputs |x| < 0.66q; DST: 0 smem (renormalised),
// 1 global raw doubles (renormalised), 2 global canonical u64 with N^-1 folded into the last stage (single pass)
template <int CL, int A, int RB, int DST>
__device__ __forceinline__ void fp_inv_round(double* sm, u64* gdst, const LimbConst& L, int s1, int chunk, int tid) {
    constexpr int G = 16 >> RB, RR = 1 << RB, LOB = CL - A - RB;
    const double q = L.fq, qinv = L.fqinv;
    const double* tw = L.ftw_bwd;
#pragma unroll
    for (int gi = 0; gi < G; gi++) {
        const int g = tid * G + gi;
        const int hi = g >> LOB, lo = g & ((1 << LOB) - 1);
        const int base = (hi << (CL - A)) + lo;
        double x[RR];
#pragma unroll
        for (int k = 0; k < RR; k++) x[k] = sm[fpad(base + (k << LOB))];
#pragma unroll
        for (int u = RB - 1; u >= 0; u--) {
            const int half = 1 << (RB - 1 - u);
            const int s = s1 + A + u;
            const int twbase = (1 << s) + (chunk << (A + u)) + (hi << u);
            if (DST == 2 && A + u == 0) {
#pragma unroll
                for (int k = 0; k < RR; k++) {
                    if (k & half) continue;
                    const double a = x[k], c = x[k + half];
                    x[k] = fp_mulmod(__dadd_rn(a, c), L.fninv, q, qinv);
                    x[k + half] = fp_mulmod(__dadd_rn(a, -c), L.flast_inv, q, qinv);
                }
            } else {
#pragma unroll
                for (int k = 0; k < RR; k++) {
                    if (k & half) continue;
                    fp_inv_bfly(x[k], x[k + half], __ldg(tw + twbase + (k >> (RB - u))), q, qinv);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < RR; k++) {
            const int idx = base + (k << LOB);
            if (DST == 2) gdst[idx] = d2u(x[k] < 0.0 ? x[k] + q : x[k]);
            else {
                const double r = fp_reduce(x[k], q, qinv);     // sums grew up to 2^RB * 0.66q: renormalise once per round
                if (DST == 1) gdst[idx] = (u64)__double_as_longlong(r);
                else sm[fpad(idx)] = r;
            }
        }
    }
}


// 512-thread x 8-element FP64 rounds (four radix-8 rounds per 4096-element chunk)
// The 1 + 2 + 4 twiddles of a radix-8 round are three CONTIGUOUS runs of the table (8, 16 and 32 bytes, aligned to their size: the table is
// allocated 256-byte aligned and every run starts at a multiple of its length), so they are fetched as one 64-bit and three 128-bit loads
// (128 bits is the widest global access on sm_90). In the last round (A = 9, one group per thread) the seven scalar loads touch
// 2 + 8 + 32 = 42 L1 wavefronts per warp (stride-2 / stride-4 8-byte accesses use a quarter of every sector they pull); the vector loads
// touch 2 + 4 + 2 x 8.
#ifndef LGPU_TW_VEC
#define LGPU_TW_VEC 1
#endif
__device__ __forceinline__ void ldg_f64x4(const double* p, double& a, double& b, double& c, double& d) {
    const double2 lo = __ldg(reinterpret_cast<const double2*>(p)), hi = __ldg(reinterpret_cast<const double2*>(p + 2));
    a = lo.x; b = lo.y; c = hi.x; d = hi.y;
}
// VOL: the loads are `asm volatile`, i.e. issued where they are written. Inside the digit loop of the key-switch MAC kernel the twiddles are
// loop-invariant; left to the compiler they are hoisted out of the loop, do not fit in the 64-register budget and come back as local-memory
// reloads (2 L1 wavefronts per 8-byte LDL against 1 for a CTA-uniform LDG) -- on exactly the unit that bounds that kernel.
template <int A, bool VOL = false>
__device__ __forceinline__ void fp8_load_tw(double (&t)[7], const double* tw, int s1, int chunk, int tid) {
    constexpr int LOB = 9 - A;
    const int hi = tid >> LOB;
#if LGPU_TW_VEC
    const double* p0 = tw + (1 << (s1 + A)) + (chunk << A) + hi;
    const double* p1 = tw + (1 << (s1 + A + 1)) + (chunk << (A + 1)) + (hi << 1);
    const double* p2 = tw + (1 << (s1 + A + 2)) + (chunk << (A + 2)) + (hi << 2);
    if (VOL) {
        asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(t[0]) : "l"(p0));
        asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(t[1]), "=d"(t[2]) : "l"(p1));
        asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(t[3]), "=d"(t[4]) : "l"(p2));
        asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(t[5]), "=d"(t[6]) : "l"(p2 + 2));
    } else {
        t[0] = __ldg(p0);
        const double2 v = __ldg(reinterpret_cast<const double2*>(p1));
        t[1] = v.x; t[2] = v.y;
        ldg_f64x4(p2, t[3], t[4], t[5], t[6]);
    }
#else
#pragma unroll
    for (int u = 0; u < 3; u++) {
        const int twbase = (1 << (s1 + A + u)) + (chunk << (A + u)) + (hi << u);
#pragma unroll
        for (int m = 0; m < (1 << u); m++) t[(1 << u) - 1 + m] = __ldg(tw + twbase + m);
    }
#endif
}
template <int A>
__device__ __forceinline__ void fp8_round(double* sm, const double (&t)[7], double q, double qinv, int tid) {
    constexpr int LOB = 9 - A;
    const int hi = tid >> LOB, lo = tid & ((1 << LOB) - 1);
    const int base = (hi << (12 - A)) + lo;
    double x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = sm[fpad(base + (k << LOB))];
#pragma unroll
    for (int u = 0; u < 3; u++) {
        const int half = 4 >> u;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (k & half) continue;
            fp_fwd_bfly(x[k], x[k + half], t[(1 << u) - 1 + (k >> (3 - u))], q, qinv);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; k++) sm[fpad(base + (k << LOB))] = x[k];
}


__device__ __forceinline__ u64 fp_biased_u64(double x, double off52) {
    return (u64)__double_as_longlong(__dadd_rn(x, off52)) & 0x000FFFFFFFFFFFFFull;
}


__device__ __forceinline__ int swz(int i) { return i ^ (((i >> 4) & 3) << 1) ^ (((i >> 6) & 1) * 9); }

// swz is GF(2)-linear, so swz(base + (k << s)) = swz(base) ^ swz(k << s) whenever base has no bits where k << s has:
// the k-dependent part is a compile-time constant and each round needs at most 8 address registers per thread
// (computed once, used for the loads and the stores) instead of a shift / xor / select chain per access.
__host__ __device__ constexpr int swzc(int i) { return i ^ (((i >> 4) & 3) << 1) ^ (((i >> 6) & 1) * 9); }

__device__ __forceinline__ void fp8_bflys(double (&x)[8], const double (&t)[7], double q, double qinv) {
#pragma unroll
    for (int u = 0; u < 3; u++) {
        const int half = 4 >> u;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (k & half) continue;
            fp_fwd_bfly(x[k], x[k + half], t[(1 << u) - 1 + (k >> (3 - u))], q, qinv);
        }
    }
}


// The four radix-8 rounds of a 4096-element chunk on a swizzled tile (512 threads x 8 elements). Round 1 is done by the
// caller from registers; its results are stored with fp8s_store_r1 and followed by a CTA barrier. Round 2 works inside
// 512-element groups (one pair of warps: fp8s_pair_sync), rounds 3 and 4 inside one warp's 256 elements (__syncwarp).
__device__ __forceinline__ void fp8s_store_r1(double* fsm, const double (&x)[8], int tid) {
    double* a = fsm + swz(tid);                            // swz(tid + 512 k) = swz(tid) + 512 k
#pragma unroll
    for (int k = 0; k < 8; k++) a[512 * k] = x[k];
}
__device__ __forceinline__ void fp8s_round2(double* fsm, const double (&tt)[7], double q, double qinv, int tid) {
    // base = hi * 512 + lo, elements base + 64 k; swzc(64 k) = 64 k ^ ((k & 1) * 9)
    const int tb = swz(((tid >> 6) << 9) + (tid & 63));
    double* a0 = fsm + tb;
    double* a1 = fsm + (tb ^ 9);
    double x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = ((k & 1) ? a1 : a0)[64 * k];
    fp8_bflys(x, tt, q, qinv);
#pragma unroll
    for (int k = 0; k < 8; k++) ((k & 1) ? a1 : a0)[64 * k] = x[k];
}
__device__ __forceinline__ void fp8s_pair_sync(int tid) {
    asm volatile("bar.sync %0, 64;" ::"r"(1 + (tid >> 6)) : "memory");          // the two warps of one 512-element group
}
__device__ __forceinline__ void fp8s_round3(double* fsm, const double (&tt)[7], double q, double qinv, int tid) {
    // base = hi * 64 + lo, elements base + 8 k; swzc(8 k) = 8 k ^ ((k >> 1) << 1)
    const int tb = swz(((tid >> 3) << 6) + (tid & 7));
    double* a[8];
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = fsm + ((tb ^ ((k & 1) << 3) ^ ((k >> 1) << 1)) + ((k >> 1) << 4));
    double x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = *a[k];
    fp8_bflys(x, tt, q, qinv);
#pragma unroll
    for (int k = 0; k < 8; k++) *a[k] = x[k];
}
// round 4 operands: elements 8 tid + k live at swz(8 tid) ^ k
__device__ __forceinline__ void fp8s_load_r4(const double* fsm, double (&x)[8], int tid) {
    const int tb = swz(tid << 3);
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = fsm[tb ^ k];
}


// ---- the same four radix-8 rounds for the integer (Shoup) butterflies: 512 threads x 8 elements on the XOR-swizzled u64 tile. Twiddle pairs are
// read where they are used (16 bytes each, L1-resident; rounds 1-2 are warp-uniform) instead of being held in 28 registers. `mask` is the
// prime's lazy-correction schedule (LimbConst.fwd_mask: 0 below 2^57, every other stage for 60-bit primes, every stage for 61-bit ones).
// CORR = false compiles the correction out (launches whose primes all have an empty schedule: q0 and the 55-bit special primes of the CKKS sets).
template <int A, bool CORR = true>
__device__ __forceinline__ void int8_bflys(u64 (&x)[8], const ulonglong2* tw, int s1, int chunk, int hi, u64 nq, u64 twoq, u64 kq, unsigned mask) {
#pragma unroll
    for (int u = 0; u < 3; u++) {
        const int half = 4 >> u;
        const int twbase = (1 << (s1 + A + u)) + (chunk << (A + u)) + (hi << u);
        const bool corr = CORR && ((mask >> (s1 + A + u)) & 1u);
#pragma unroll
        for (int k = 0; k < 8; k++) {
            if (k & half) continue;
            fast_fwd_bfly(x[k], x[k + half], __ldg(tw + twbase + (k >> (3 - u))), nq, twoq, kq, corr);
        }
    }
}
__device__ __forceinline__ void i8s_store_r1(u64* sm, const u64 (&x)[8], int tid) {
    u64* a = sm + swz(tid);
#pragma unroll
    for (int k = 0; k < 8; k++) a[512 * k] = x[k];
}
template <bool CORR = true>
__device__ __forceinline__ void i8s_round2(u64* sm, const ulonglong2* tw, int s1, int chunk, int tid, u64 nq, u64 twoq, u64 kq, unsigned mask) {
    const int tb = swz(((tid >> 6) << 9) + (tid & 63));
    u64* a0 = sm + tb;
    u64* a1 = sm + (tb ^ 9);
    u64 x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = ((k & 1) ? a1 : a0)[64 * k];
    int8_bflys<3, CORR>(x, tw, s1, chunk, tid >> 6, nq, twoq, kq, mask);
#pragma unroll
    for (int k = 0; k < 8; k++) ((k & 1) ? a1 : a0)[64 * k] = x[k];
}
template <bool CORR = true>
__device__ __forceinline__ void i8s_round3(u64* sm, const ulonglong2* tw, int s1, int chunk, int tid, u64 nq, u64 twoq, u64 kq, unsigned mask) {
    const int tb = swz(((tid >> 3) << 6) + (tid & 7));
    u64* a[8];
#pragma unroll
    for (int k = 0; k < 8; k++) a[k] = sm + ((tb ^ ((k & 1) << 3) ^ ((k >> 1) << 1)) + ((k >> 1) << 4));
    u64 x[8];
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = *a[k];
    int8_bflys<6, CORR>(x, tw, s1, chunk, tid >> 3, nq, twoq, kq, mask);
#pragma unroll
    for (int k = 0; k < 8; k++) *a[k] = x[k];
}
__device__ __forceinline__ void i8s_load_r4(const u64* sm, u64 (&x)[8], int tid) {
    const int tb = swz(tid << 3);
#pragma unroll
    for (int k = 0; k < 8; k++) x[k] = sm[tb ^ k];
}

}  // namespace lgpu

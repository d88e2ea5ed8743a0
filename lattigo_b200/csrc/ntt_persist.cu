// ntt_persist.cu -- single-launch, single-HBM-pass negacyclic transforms for 2^13 <= N <= 2^16.
//
// The two-pass transforms of ntt.cu / ntt_fp64.cu (strided pass over the whole launch, then chunk pass over the whole
// launch) move every coefficient through HBM twice: the intermediate of a launch (rows x batch x N x 8 B, 184 MB for
// 44 limbs x 8 polynomials) is long gone from the 50 MB L2 when the second kernel reads it. Here ONE persistent kernel
// (one CTA slot per SM x occupancy) executes both passes of every limb-transform as TILES drawn from a global ticket
// counter, in an order that keeps producer and consumer tiles a bounded distance apart:
//
//     step s :  [ pass-1 tiles of limb-transform s ]  [ pass-2 tiles of limb-transform s - D ]
//
// A pass-2 tile waits (acquire-load on a per-limb-transform counter) until the pass-1 tiles of ITS limb-transform have
// published their stores (barrier, then thread 0: fence + atomic add -- the cooperative-groups grid-sync pattern at the
// granularity of one polynomial row). Tickets are handed out in order and a pass-1 tile never waits, so every tile a
// waiter depends on is already running: no deadlock, whatever the grid size. The intermediate lives in the output buffer
// and is consumed ~D x 0.5 MB later, i.e. from L2: D is 2.5 x the resident CTAs / tiles per limb-transform, 10-14 MB of
// intermediate in flight at N = 2^16 on 132 SMs, well inside the 50 MB L2. HBM sees each coefficient once in and once out: 16 B per coefficient,
// the algorithmic minimum (SURVEY 8(d) C2).
//
// Arithmetic: the same butterflies as the two-pass kernels (FP64-pipe path for primes with LimbConst.fp_ok, Shoup
// integer path otherwise); only canonical values leave, so outputs equal ring.NTT / ring.INTT bit for bit
// (ring/ntt.go:127-152,174-206). The exact-lazy variant (NTTLazy) stays on the two-pass reference-arithmetic kernels.
//
// Forward FP64 pass-1 can run on the INTEGER pipes instead (PH1INT): the strided stages are 25 % of the butterflies at
// N = 2^16; with them on IMAD/ALU and the chunk stages on the FP64 pipe, CTAs of the two kinds share an SM and the two
// pipes overlap by construction (off by default, LGPU_NTT_PH1INT=1; A/B with tools/bench_ntt.py).
#include <cstdlib>
#include "../../include/lattigo_b200.h"
#include "engine.h"
#include "modarith.cuh"
#include "ntt_arith.cuh"

namespace lgpu {

struct PersistParams {
    const LimbConst* limbs;
    RowMap rm;
    const u64* in;
    u64* out;
    size_t in_rs, in_bs, out_rs, out_bs;
    int logN, batch, nLT;   // nLT = rows x batch limb-transforms, lt = row_index * batch + b
    int n1, n2;             // tiles per limb-transform in pass 1 / pass 2
    int D;                  // distance (in limb-transforms) between the pass-1 and the pass-2 tiles of one step
    int total;              // tickets = (nLT + D) * (n1 + n2)
    unsigned* ctr;          // [0]: ticket dispenser; [1 + lt]: finished pass-1 tiles of lt
    // optional fused epilogue (forward transforms): out = MulCoeffsMontgomery(NTT(in), mul) -- ring/ntt.go:127-131 followed by
    // ring/operations.go:88-92 in one pass (SURVEY 8(d) C2(ii): 3 rows of traffic instead of 5); the product runs on the integer
    // pipes, which the FP64-pipe transform leaves idle
    const u64* mul; size_t mul_rs, mul_bs;
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

struct TileRef {
    const u64* in;
    u64* out;
    const u64* mul;
    int limb;
};
__device__ __forceinline__ TileRef tile_ref(const PersistParams& p, int lt) {
    const int r = lt / p.batch, b = lt - r * p.batch;
    const int row = p.rm.drow[r];
    TileRef t;
    t.in = p.in + (size_t)b * p.in_bs + (size_t)row * p.in_rs;
    t.out = p.out + (size_t)b * p.out_bs + (size_t)row * p.out_rs;
    t.mul = p.mul ? p.mul + (size_t)b * p.mul_bs + (size_t)row * p.mul_rs : nullptr;
    t.limb = p.rm.limb[r];
    return t;
}

// ---------------------------------------------------------------------------------------------------------------------
// forward, FP64-pipe primes: 512 threads. pass 1 = strided stages [0, RL) on 512 columns x 2^RL rows (registers only);
// pass 2 = the 12 chunk stages as four radix-8 rounds (fp8_*), canonical output copied out through the tile.
// ---------------------------------------------------------------------------------------------------------------------
template <int RL, int PH1INT>
struct FpFwdOps {
    static constexpr int T = 512, MINB = 2;
    static constexpr bool kInverse = false;
    static constexpr size_t kSmem = (size_t)(4096 + 256 + 8) * sizeof(u64);
    static constexpr int kN1 = 4096 / T;                 // 8 column tiles
    static constexpr int kN2 = 1 << RL;                  // chunks

    static __device__ __forceinline__ void pass1(const PersistParams& p, int lt, int j, u64*) {
        constexpr int R = 1 << RL, stride = 4096;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        const int l = j * T + threadIdx.x;
        const u64 qi = L.q, bhi = L.bred_hi;
        if constexpr (PH1INT == 0) {
            const double q = L.fq, qinv = L.fqinv;
            const double* tw = L.ftw_fwd;
            double x[R];
#pragma unroll
            for (int k = 0; k < R; k++) x[k] = u2d_any(t.in[(size_t)k * stride + l], qi, bhi);
#pragma unroll
            for (int u = 0; u < RL; u++) {
                const int half = 1 << (RL - 1 - u);
#pragma unroll
                for (int k = 0; k < R; k++) {
                    if (k & half) continue;
                    fp_fwd_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), q, qinv);
                }
            }
#pragma unroll
            for (int k = 0; k < R; k++) t.out[(size_t)k * stride + l] = (u64)__double_as_longlong(x[k]);   // raw signed lazy doubles
        } else {
            // integer pipes: Shoup butterflies without corrections (q < 2^46: RL stages add < 2 RL q to a value < 2q),
            // intermediate = lazy u64 below 2^52, converted exactly by pass 2
            const ulonglong2* tw = L.tw_fwd;
            const u64 nq = 0ull - qi, twoq = qi << 1;
            u64 x[R];
#pragma unroll
            for (int k = 0; k < R; k++) {
                u64 v = t.in[(size_t)k * stride + l];
                if (v >= twoq) v = bred_add(v, qi, bhi);
                x[k] = v;
            }
#pragma unroll
            for (int u = 0; u < RL; u++) {
                const int half = 1 << (RL - 1 - u);
#pragma unroll
                for (int k = 0; k < R; k++) {
                    if (k & half) continue;
                    fast_fwd_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), nq, twoq, 0, false);
                }
            }
#pragma unroll
            for (int k = 0; k < R; k++) t.out[(size_t)k * stride + l] = x[k];
        }
    }

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int chunk, u64* smem) {
        constexpr int s1 = RL;
        const int tid = threadIdx.x;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        double* fsm = reinterpret_cast<double*>(smem);
        const double fq = L.fq, fqinv = L.fqinv;
        const double* tw = L.ftw_fwd;
        u64* io = t.out + ((size_t)chunk << 12);
        {
            double x[8];
#pragma unroll
            for (int k = 0; k < 8; k++) {
                const u64 raw = __ldcg(io + k * T + tid);
                x[k] = PH1INT ? u2d(raw) : __longlong_as_double((long long)raw);
            }
#pragma unroll
            for (int u = 0; u < 3; u++) {
                const int half = 4 >> u;
                const int twbase = (1 << (s1 + u)) + (chunk << u);
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    if (k & half) continue;
                    fp_fwd_bfly(x[k], x[k + half], __ldg(tw + twbase + (k >> (3 - u))), fq, fqinv);
                }
            }
#pragma unroll
            for (int k = 0; k < 8; k++) fsm[fpad(k * T + tid)] = x[k];
        }
        double tt[7];
        fp8_load_tw<3>(tt, tw, s1, chunk, tid);
        __syncthreads();
        fp8_round<3>(fsm, tt, fq, fqinv, tid);
        fp8_load_tw<6>(tt, tw, s1, chunk, tid);
        __syncthreads();
        fp8_round<6>(fsm, tt, fq, fqinv, tid);
        fp8_load_tw<9>(tt, tw, s1, chunk, tid);
        __syncthreads();
        {   // last round: 8 consecutive coefficients per thread, read and written back by the same thread
            const int base = tid << 3;
            double x[8];
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = fsm[fpad(base + k)];
#pragma unroll
            for (int u = 0; u < 3; u++) {
                const int half = 4 >> u;
#pragma unroll
                for (int k = 0; k < 8; k++) {
                    if (k & half) continue;
                    fp_fwd_bfly(x[k], x[k + half], tt[(1 << u) - 1 + (k >> (3 - u))], fq, fqinv);
                }
            }
            // canonicalisation on the INTEGER pipes (one biased conversion + one Barrett step) instead of 5 FP64 operations
            const double off52 = __dmul_rn((double)(10 + p.logN), fq) + 4503599627370496.0;
            const u64 q = L.q, bhi = L.bred_hi;
#pragma unroll
            for (int k = 0; k < 8; k++) smem[fpad(base + k)] = bred_add(fp_biased_u64(x[k], off52), q, bhi);
        }
        __syncthreads();
        if (t.mul) {
            const u64* mu = t.mul + ((size_t)chunk << 12);
            const u64 q = L.q, qinv = L.qinv;
#pragma unroll
            for (int k = 0; k < 8; k++) io[k * T + tid] = mred(smem[fpad(k * T + tid)], mu[k * T + tid], q, qinv);
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) io[k * T + tid] = smem[fpad(k * T + tid)];
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// forward FP64, second generation of pass 2 (the first stalled on CTA-wide barriers and its padded
// shared-memory tile had 2-way bank conflicts in the stride-8 round):
//   * the 4096-word tile is XOR-swizzled instead of padded: slot = i[3:0] ^ {i6, i5, i4, i6}; every access pattern of
//     the four radix-8 rounds (stride 512 / 64 / 8 / 1 across a half-warp) and the coalesced copy-out are conflict-free;
//   * only the exchange after round 1 is CTA-wide. Round 2 -> 3 exchanges data inside one 512-element group = one pair
//     of warps (named barrier, 64 threads), round 3 -> 4 and the copy-out inside one warp's 256 consecutive elements
//     (__syncwarp): warps drift apart and the FP64 phases of some overlap the exchange phases of others.
// ---------------------------------------------------------------------------------------------------------------------
template <int RL>
struct FpFwdOps2 : FpFwdOps<RL, 0> {
    static constexpr int T = 512;
    static constexpr size_t kSmem = (size_t)4096 * sizeof(u64);

    // pass 1 with the >= 2^52 guard as ONE warp-uniform branch: the per-element form is if-converted by the compiler into
    // ~12 predicated-off instructions per coefficient that still take issue slots (ncu: IMAD 36 per coefficient)
    static __device__ __forceinline__ void pass1(const PersistParams& p, int lt, int j, u64*) {
        constexpr int R = 1 << RL, stride = 4096;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        const int l = j * T + threadIdx.x;
        const double q = L.fq, qinv = L.fqinv;
        const double* tw = L.ftw_fwd;
        u64 raw[R];
#pragma unroll
        for (int k = 0; k < R; k++) raw[k] = t.in[(size_t)k * stride + l];
        unsigned hi = 0;
#pragma unroll
        for (int k = 0; k < R; k++) hi |= (unsigned)(raw[k] >> 32);
        if (__any_sync(0xffffffffu, (hi >> 20) != 0)) {
            const u64 qi = L.q, bhi = L.bred_hi;
#pragma unroll
            for (int k = 0; k < R; k++) if (raw[k] >> 52) raw[k] = bred_add(raw[k], qi, bhi);
        }
        double x[R];
#pragma unroll
        for (int k = 0; k < R; k++) x[k] = u2d(raw[k]);
#pragma unroll
        for (int u = 0; u < RL; u++) {
            const int half = 1 << (RL - 1 - u);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                fp_fwd_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), q, qinv);   // the same for every column
            }
        }
#pragma unroll
        for (int k = 0; k < R; k++) t.out[(size_t)k * stride + l] = (u64)__double_as_longlong(x[k]);
    }

    // round 1 (stages 0..2 of the chunk): element k of this thread = k * 512 + tid. SRC 0: straight from L2 (ld.global.cg);
    // SRC 1: from the tile itself, where a bulk-async copy (TMA) landed the chunk linearly -- the swizzled store goes to
    // words of the same 16-word group, i.e. words read by lanes of the same half-warp, hence the __syncwarp.
    template <int SRC>
    static __device__ __forceinline__ void round1(const LimbConst& L, const u64* io, u64* smem, int chunk, int tid) {
        constexpr int s1 = RL;
        double* fsm = reinterpret_cast<double*>(smem);
        const double fq = L.fq, fqinv = L.fqinv;
        const double* tw = L.ftw_fwd;
        double tt[7];
        fp8_load_tw<0>(tt, tw, s1, chunk, tid);           // CTA-uniform: hi = 0
        double x[8];
        if (SRC == 0) {
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = __longlong_as_double((long long)__ldcg(io + k * T + tid));
        } else {
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = fsm[k * T + tid];
            __syncwarp();
        }
        fp8_bflys(x, tt, fq, fqinv);
        double* a = fsm + swz(tid);                        // swz(tid + 512 k) = swz(tid) + 512 k
#pragma unroll
        for (int k = 0; k < 8; k++) a[512 * k] = x[k];
    }

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int chunk, u64* smem) {
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        u64* io = t.out + ((size_t)chunk << 12);
        round1<0>(L, io, smem, chunk, threadIdx.x);
        __syncthreads();
        tail(p, L, io, smem, chunk, threadIdx.x, t.mul);
    }

    // rounds 2..4 and the copy-out; the caller has issued the CTA barrier that follows round 1
    static __device__ __forceinline__ void tail(const PersistParams& p, const LimbConst& L, u64* io, u64* smem, int chunk, int tid,
                                                const u64* mul = nullptr) {
        constexpr int s1 = RL;
        double* fsm = reinterpret_cast<double*>(smem);
        const double fq = L.fq, fqinv = L.fqinv;
        const double* tw = L.ftw_fwd;
        double tt[7];
        fp8_load_tw<3>(tt, tw, s1, chunk, tid);
        fp8s_round2(fsm, tt, fq, fqinv, tid);              // stages 3..5
        fp8_load_tw<6>(tt, tw, s1, chunk, tid);
        fp8s_pair_sync(tid);
        fp8s_round3(fsm, tt, fq, fqinv, tid);              // stages 6..8
        fp8_load_tw<9>(tt, tw, s1, chunk, tid);
        __syncwarp();
        {   // round 4 (stages 9..11): elements 8 tid + k -> swz(8 tid) ^ k; canonical residues go back to the same words
            const int tb = swz(tid << 3);
            double* a[8];
#pragma unroll
            for (int k = 0; k < 8; k++) a[k] = fsm + (tb ^ k);
            double x[8];
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = *a[k];
            fp8_bflys(x, tt, fq, fqinv);
#ifdef NTT_CANON_INT
            // A/B (tools/build_variant.sh canon_int ntt_persist.cu -DNTT_CANON_INT): canonicalise on the integer pipes (one biased conversion + one
            // Barrett step) instead of 5 FP64 operations per coefficient
            const double off52 = __dmul_rn((double)(10 + p.logN), fq) + 4503599627370496.0;
            const u64 qi = L.q, bhi = L.bred_hi;
#pragma unroll
            for (int k = 0; k < 8; k++) *reinterpret_cast<u64*>(a[k]) = bred_add(fp_biased_u64(x[k], off52), qi, bhi);
#else
#pragma unroll
            for (int k = 0; k < 8; k++) *reinterpret_cast<u64*>(a[k]) = fp_canon(x[k], fq, fqinv);
#endif
        }
        __syncwarp();
        {   // this warp's 256 consecutive coefficients, 256 B per store instruction; swzc(32 m) = 32 m ^ ((m & 1) << 2) ^ (((m >> 1) & 1) * 9)
            const int w0 = (tid >> 5) << 8, lane = tid & 31;
            const int tb = swz(w0 + lane);
            u64* g = io + w0 + lane;
            if (mul) {
                const u64* mu = mul + ((size_t)chunk << 12) + w0 + lane;
                const u64 q = L.q, qinv = L.qinv;
                u64 o[8];
#pragma unroll
                for (int m = 0; m < 8; m++) o[m] = __ldg(mu + 32 * m);
#pragma unroll
                for (int m = 0; m < 8; m++) g[32 * m] = mred(smem[(tb ^ ((m & 1) << 2) ^ (((m >> 1) & 1) * 9)) + 32 * m], o[m], q, qinv);
            } else {
#pragma unroll
                for (int m = 0; m < 8; m++) g[32 * m] = smem[(tb ^ ((m & 1) << 2) ^ (((m >> 1) & 1) * 9)) + 32 * m];
            }
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// forward FP64, register copy-out (LGPU_NTT_PERSIST_V=5, A/B): after round 4 every thread holds 8 CONSECUTIVE canonical coefficients, so they go
// straight to global memory as four 128-bit stores (64 contiguous bytes per thread, as in the key-switch MAC kernel) instead of being written
// back to the tile, exchanged inside the warp and copied out 8 bytes at a time: 8 STS + 8 LDS + a warp barrier + 4 STG less per thread and tile.
// Needs 16-byte aligned output rows (the dispatcher checks and falls back to FpFwdOps2).
// ---------------------------------------------------------------------------------------------------------------------
template <int RL>
struct FpFwdOps3 : FpFwdOps2<RL> {
    static constexpr int T = 512;
    static constexpr size_t kSmem = (size_t)4096 * sizeof(u64);

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int chunk, u64* smem) {
        constexpr int s1 = RL;
        const int tid = threadIdx.x;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        u64* io = t.out + ((size_t)chunk << 12);
        FpFwdOps2<RL>::template round1<0>(L, io, smem, chunk, tid);
        __syncthreads();
        double* fsm = reinterpret_cast<double*>(smem);
        const double fq = L.fq, fqinv = L.fqinv;
        const double* tw = L.ftw_fwd;
        double tt[7];
        fp8_load_tw<3>(tt, tw, s1, chunk, tid);
        fp8s_round2(fsm, tt, fq, fqinv, tid);              // stages 3..5
        fp8_load_tw<6>(tt, tw, s1, chunk, tid);
        fp8s_pair_sync(tid);
        fp8s_round3(fsm, tt, fq, fqinv, tid);              // stages 6..8
        fp8_load_tw<9>(tt, tw, s1, chunk, tid);
        __syncwarp();
        double x[8];
        fp8s_load_r4(fsm, x, tid);
        fp8_bflys(x, tt, fq, fqinv);                       // stages 9..11
        u64* g = io + 8 * tid;
        if (t.mul) {
            const u64* mu = t.mul + ((size_t)chunk << 12) + 8 * tid;
            const u64 q = L.q, qinv = L.qinv;
#pragma unroll
            for (int k = 0; k < 8; k += 2) {
                const ulonglong2 m = __ldg(reinterpret_cast<const ulonglong2*>(mu + k));
                *reinterpret_cast<ulonglong2*>(g + k) = make_ulonglong2(mred(fp_canon(x[k], fq, fqinv), m.x, q, qinv), mred(fp_canon(x[k + 1], fq, fqinv), m.y, q, qinv));
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; k += 2)
                *reinterpret_cast<ulonglong2*>(g + k) = make_ulonglong2(fp_canon(x[k], fq, fqinv), fp_canon(x[k + 1], fq, fqinv));
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// inverse, FP64-pipe primes: 256 threads x 16 elements (fp_inv_round). pass 1 = chunk stages (deepest first), raw
// renormalised doubles out; pass 2 = strided stages with N^-1 folded into the last one, canonical output.
// ---------------------------------------------------------------------------------------------------------------------
template <int RL>
struct FpInvOps {
    static constexpr int T = 256, MINB = 2;
    static constexpr bool kInverse = true;
    static constexpr size_t kSmem = (size_t)(4096 + 256 + 1) * sizeof(double);
    static constexpr int kN1 = 1 << RL;                  // chunks
    static constexpr int kN2 = 4096 / T;                 // 16 column tiles

    static __device__ __forceinline__ void pass1(const PersistParams& p, int lt, int chunk, u64* smem) {
        constexpr int CL = 12;
        const int tid = threadIdx.x;
        const TileRef t = tile_ref(p, lt);
        const LimbConst L = p.limbs[t.limb];
        double* fsm = reinterpret_cast<double*>(smem);
        const u64* src = t.in + ((size_t)chunk << CL);
        u64* dst = t.out + ((size_t)chunk << CL);
        const double q = L.fq, qinv = L.fqinv;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int idx = k * T + tid;
            fsm[fpad(idx)] = fp_reduce(u2d_any(src[idx], L.q, L.bred_hi), q, qinv);
        }
        __syncthreads();
        fp_inv_round<CL, 8, 4, 0>(fsm, nullptr, L, RL, chunk, tid);
        __syncthreads();
        fp_inv_round<CL, 4, 4, 0>(fsm, nullptr, L, RL, chunk, tid);
        __syncthreads();
        fp_inv_round<CL, 0, 4, 1>(fsm, dst, L, RL, chunk, tid);
    }

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int j, u64*) {
        constexpr int R = 1 << RL, stride = 4096;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        const int l = j * T + threadIdx.x;
        const double q = L.fq, qinv = L.fqinv;
        const double* tw = L.ftw_bwd;
        double x[R];
#pragma unroll
        for (int k = 0; k < R; k++) x[k] = __longlong_as_double((long long)__ldcg(t.out + (size_t)k * stride + l));
#pragma unroll
        for (int u = RL - 1; u >= 1; u--) {
            const int half = 1 << (RL - 1 - u);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                fp_inv_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), q, qinv);
            }
        }
        constexpr int half = 1 << (RL - 1);
        const double fninv = L.fninv, flast = L.flast_inv;
#pragma unroll
        for (int k = 0; k < half; k++) {
            const double u = x[k], v = x[k + half];
            const double a = fp_mulmod(__dadd_rn(u, v), fninv, q, qinv);
            const double c = fp_mulmod(__dadd_rn(u, -v), flast, q, qinv);
            t.out[(size_t)k * stride + l] = d2u(a < 0.0 ? a + q : a);
            t.out[(size_t)(k + half) * stride + l] = d2u(c < 0.0 ? c + q : c);
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// integer (Shoup) primes, 256 threads x 16 elements, FAST = 1 (per-prime correction schedule) or 2 (no corrections)
// ---------------------------------------------------------------------------------------------------------------------
template <int RL, int FAST>
struct IntFwdOps {
    static constexpr int T = 256, MINB = 2;
    static constexpr bool kInverse = false;
    static constexpr size_t kSmem = (size_t)(4096 + 256 + 1) * sizeof(u64);
    static constexpr int kN1 = 4096 / T;
    static constexpr int kN2 = 1 << RL;

    static __device__ __forceinline__ void pass1(const PersistParams& p, int lt, int j, u64*) {
        constexpr int R = 1 << RL, stride = 4096;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        const int l = j * T + threadIdx.x;
        const u64 q = L.q;
        const ulonglong2* tw = L.tw_fwd;
        const u64 nq = 0ull - q, twoq = q << 1, kq = L.kq;
        const unsigned mask = L.fwd_mask;
        u64 x[R];
#pragma unroll
        for (int k = 0; k < R; k++) x[k] = t.in[(size_t)k * stride + l];
#pragma unroll
        for (int u = 0; u < RL; u++) {
            const int half = 1 << (RL - 1 - u);
            const bool corr = (FAST == 1) && ((mask >> u) & 1u);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                fast_fwd_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), nq, twoq, kq, corr);
            }
        }
#pragma unroll
        for (int k = 0; k < R; k++) t.out[(size_t)k * stride + l] = x[k];
    }

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int chunk, u64* sm) {
        constexpr int CL = 12;
        const int tid = threadIdx.x;
        const TileRef t = tile_ref(p, lt);
        const LimbConst L = p.limbs[t.limb];
        u64* io = t.out + ((size_t)chunk << CL);
        fwd_round<CL, 0, 4, true, FAST>(sm, io, L, RL, p.logN, chunk, tid);     // global reads are ld.global.cg
        __syncthreads();
        fwd_round<CL, 4, 4, false, FAST>(sm, nullptr, L, RL, p.logN, chunk, tid);
        __syncthreads();
        fwd_round<CL, 8, 4, false, FAST>(sm, nullptr, L, RL, p.logN, chunk, tid);
        __syncthreads();
        const u64 q = L.q, bhi = L.bred_hi;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int idx = k * T + tid;
            const u64 v = bred_add(sm[pad_idx(idx)], q, bhi);                     // reducevec, ring/ntt.go:176
            io[idx] = t.mul ? mred(v, t.mul[((size_t)chunk << CL) + idx], q, L.qinv) : v;
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// forward, integer primes, second generation: the tile code of FpFwdOps2 with Shoup butterflies (512 threads x 8 elements, swizzled tile,
// one CTA barrier, pair / warp exchanges, coalesced copy-out of canonical residues). The 256 x 16 IntFwdOps ran 16 warps per SM at 128
// registers; this one runs 32 at 64. The per-prime correction schedule is evaluated at run time (all-zero below 2^57).
// ---------------------------------------------------------------------------------------------------------------------
template <int RL, bool CORR>
struct IntFwdOps2 {
    static constexpr int T = 512, MINB = 2;
    static constexpr bool kInverse = false;
    static constexpr size_t kSmem = (size_t)4096 * sizeof(u64);
    static constexpr int kN1 = 4096 / T;
    static constexpr int kN2 = 1 << RL;

    static __device__ __forceinline__ void pass1(const PersistParams& p, int lt, int j, u64*) {
        constexpr int R = 1 << RL, stride = 4096;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        const int l = j * T + threadIdx.x;
        const u64 q = L.q;
        const ulonglong2* tw = L.tw_fwd;
        const u64 nq = 0ull - q, twoq = q << 1, kq = L.kq;
        const unsigned mask = L.fwd_mask;
        u64 x[R];
#pragma unroll
        for (int k = 0; k < R; k++) x[k] = t.in[(size_t)k * stride + l];
#pragma unroll
        for (int u = 0; u < RL; u++) {
            const int half = 1 << (RL - 1 - u);
            const bool corr = CORR && ((mask >> u) & 1u);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                fast_fwd_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), nq, twoq, kq, corr);
            }
        }
#pragma unroll
        for (int k = 0; k < R; k++) t.out[(size_t)k * stride + l] = x[k];
    }

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int chunk, u64* sm) {
        constexpr int s1 = RL;
        const int tid = threadIdx.x;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        u64* io = t.out + ((size_t)chunk << 12);
        const u64 q = L.q, nq = 0ull - q, twoq = q << 1, kq = L.kq, bhi = L.bred_hi;
        const unsigned mask = L.fwd_mask;
        const ulonglong2* tw = L.tw_fwd;
        {
            u64 x[8];
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = __ldcg(io + k * T + tid);
            int8_bflys<0, CORR>(x, tw, s1, chunk, 0, nq, twoq, kq, mask);
            i8s_store_r1(sm, x, tid);
        }
        __syncthreads();
        i8s_round2<CORR>(sm, tw, s1, chunk, tid, nq, twoq, kq, mask);
        fp8s_pair_sync(tid);
        i8s_round3<CORR>(sm, tw, s1, chunk, tid, nq, twoq, kq, mask);
        __syncwarp();
        {
            const int tb = swz(tid << 3);
            u64 x[8];
#pragma unroll
            for (int k = 0; k < 8; k++) x[k] = sm[tb ^ k];
            int8_bflys<9, CORR>(x, tw, s1, chunk, tid, nq, twoq, kq, mask);
#pragma unroll
            for (int k = 0; k < 8; k++) sm[tb ^ k] = bred_add(x[k], q, bhi);            // reducevec, ring/ntt.go:176
        }
        __syncwarp();
        {
            const int w0 = (tid >> 5) << 8, lane = tid & 31;
            const int tb = swz(w0 + lane);
            u64* g = io + w0 + lane;
            if (t.mul) {
                const u64* mu = t.mul + ((size_t)chunk << 12) + w0 + lane;
                const u64 qinv = L.qinv;
#pragma unroll
                for (int m = 0; m < 8; m++) g[32 * m] = mred(sm[(tb ^ ((m & 1) << 2) ^ (((m >> 1) & 1) * 9)) + 32 * m], __ldg(mu + 32 * m), q, qinv);
            } else {
#pragma unroll
                for (int m = 0; m < 8; m++) g[32 * m] = sm[(tb ^ ((m & 1) << 2) ^ (((m >> 1) & 1) * 9)) + 32 * m];
            }
        }
    }
};

template <int RL, int FAST>
struct IntInvOps {
    static constexpr int T = 256, MINB = 2;
    static constexpr bool kInverse = true;
    static constexpr size_t kSmem = (size_t)(4096 + 256 + 1) * sizeof(u64);
    static constexpr int kN1 = 1 << RL;
    static constexpr int kN2 = 4096 / T;

    static __device__ __forceinline__ void pass1(const PersistParams& p, int lt, int chunk, u64* sm) {
        constexpr int CL = 12;
        const int tid = threadIdx.x;
        const TileRef t = tile_ref(p, lt);
        const LimbConst L = p.limbs[t.limb];
        const u64* src = t.in + ((size_t)chunk << CL);
        u64* dst = t.out + ((size_t)chunk << CL);
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const int idx = k * T + tid;
            sm[pad_idx(idx)] = src[idx];
        }
        __syncthreads();
        inv_round<CL, 8, 4, false, false, FAST>(sm, nullptr, L, RL, chunk, tid);
        __syncthreads();
        inv_round<CL, 4, 4, false, false, FAST>(sm, nullptr, L, RL, chunk, tid);
        __syncthreads();
        inv_round<CL, 0, 4, true, false, FAST>(sm, dst, L, RL, chunk, tid);
    }

    static __device__ __forceinline__ void pass2(const PersistParams& p, int lt, int j, u64*) {
        constexpr int R = 1 << RL, stride = 4096;
        const TileRef t = tile_ref(p, lt);
        const LimbConst& L = p.limbs[t.limb];
        const int l = j * T + threadIdx.x;
        const u64 q = L.q;
        const ulonglong2* tw = L.tw_bwd;
        const bool lazy = (FAST == 2) || (FAST == 1 && L.inv_lazy != 0);
        constexpr int cl = 12;
        u64 x[R];
#pragma unroll
        for (int k = 0; k < R; k++) x[k] = __ldcg(t.out + (size_t)k * stride + l);
#pragma unroll
        for (int u = RL - 1; u >= 1; u--) {
            const int half = 1 << (RL - 1 - u);
            const u64 addq = lazy ? (q << (cl + (RL - 1 - u) + 1)) : (q << 1);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                fast_inv_bfly(x[k], x[k + half], __ldg(tw + (1 << u) + (k >> (RL - u))), q, addq, !lazy);
            }
        }
        constexpr int half = 1 << (RL - 1);
        const u64 addq = lazy ? (q << p.logN) : (q << 1);
        const ulonglong2 ninv_s = L.ninv_s, last_s = L.last_inv_s;
#pragma unroll
        for (int k = 0; k < half; k++) {
            const u64 U = x[k], V = x[k + half];
            const u64 a = shoup_mul(U + V, ninv_s, q);
            const u64 c = shoup_mul(U - V + addq, last_s, q);
            t.out[(size_t)k * stride + l] = a >= q ? a - q : a;
            t.out[(size_t)(k + half) * stride + l] = c >= q ? c - q : c;
        }
    }
};

// ---------------------------------------------------------------------------------------------------------------------
// the persistent tile loop
// ---------------------------------------------------------------------------------------------------------------------
template <class Ops>
__global__ void __launch_bounds__(Ops::T, Ops::MINB) ntt_persist_kernel(PersistParams p) {
    extern __shared__ u64 psm[];
    __shared__ int s_ticket;
    const int per = p.n1 + p.n2;
    for (;;) {
        if (threadIdx.x == 0) s_ticket = (int)atomicAdd(p.ctr, 1u);
        __syncthreads();
        const int t = s_ticket;
        if (t >= p.total) break;
        const int s = t / per, j = t - s * per;
        if (j < p.n1) {
            if (s < p.nLT) {
                Ops::pass1(p, s, j, psm);
                __syncthreads();                       // every thread's stores precede thread 0's fence
                if (threadIdx.x == 0) {
                    __threadfence();
                    atomicAdd(p.ctr + 1 + s, 1u);
                }
            }
        } else {
            const int lt = s - p.D;
            if (lt >= 0) {
                if (threadIdx.x == 0) {
                    const unsigned* c = p.ctr + 1 + lt;
                    while (ld_acquire_u32(c) < (unsigned)p.n1) __nanosleep(64);
                }
                __syncthreads();
                Ops::pass2(p, lt, j - p.n1, psm);
            }
        }
        __syncthreads();                               // s_ticket and the tile are free again
    }
}

// Second-generation tile loop: the next ticket is drawn (and, for a pass-2 tile, its dependency checked) by thread 0
// WHILE the current tile runs, and handed over through the end-of-tile barrier -- the first generation serialised an L2
// atomic round trip, a barrier, an acquire poll and another barrier in front of every tile (ncu: the three hottest
// stall sites of the kernel).
template <class Ops>
__global__ void __launch_bounds__(Ops::T, Ops::MINB) ntt_persist2_kernel(PersistParams p) {
    extern __shared__ u64 psm[];
    __shared__ int s_next[2], s_ready[2];
    const int per = p.n1 + p.n2;
    const int tid = threadIdx.x;
    if (tid == 0) { s_next[0] = (int)atomicAdd(p.ctr, 1u); s_ready[0] = 0; }
    __syncthreads();
    int par = 0;
    for (;;) {
        const int t = s_next[par];
        const int ready = s_ready[par];
        if (t >= p.total) break;
        unsigned nxt = 0;
        if (tid == 0) nxt = atomicAdd(p.ctr, 1u);          // consumed at the end of the tile: the L2 round trip is hidden
        const int s = t / per, j = t - s * per;
        int lt1 = -1;
        if (j < p.n1) {
            if (s < p.nLT) { Ops::pass1(p, s, j, psm); lt1 = s; }
        } else {
            const int lt = s - p.D;
            if (lt >= 0) {
                if (!ready) {
                    const unsigned* c = p.ctr + 1 + lt;
                    while (ld_acquire_u32(c) < (unsigned)p.n1) __nanosleep(64);
                }
                Ops::pass2(p, lt, j - p.n1, psm);
            }
        }
        if (tid == 0) {
            int rdy = 0;
            const int tn = (int)nxt;
            if (tn < p.total) {
                const int sn = tn / per, jn = tn - sn * per;
                const int ltn = sn - p.D;
                if (jn >= p.n1 && ltn >= 0) rdy = ld_acquire_u32(p.ctr + 1 + ltn) >= (unsigned)p.n1;
            }
            s_next[par ^ 1] = tn;
            s_ready[par ^ 1] = rdy;
        }
        __syncthreads();            // tile buffer free, next ticket visible, this tile's global stores ordered before thread 0
        if (lt1 >= 0 && tid == 0) {
            __threadfence();
            atomicAdd(p.ctr + 1 + lt1, 1u);
        }
        par ^= 1;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Third-generation loop, forward FP64 only: the chunk of the NEXT pass-2 tile is brought from L2 into the other half of a
// double-buffered tile by ONE bulk-async copy (cp.async.bulk = TMA, 32 KB, completion on an mbarrier) issued by thread 0
// as soon as the next ticket is known and its pass-1 tiles are published -- the L2 round trip that opened every pass-2
// tile (8 dependent-free LDG per thread, then nothing to do until they return) disappears behind the current tile.
// Round 1 then reads the landed chunk from shared memory. Needs 16-byte aligned rows (p.tma), else round 1 loads directly.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait_parity(unsigned bar, unsigned parity) {
    unsigned done;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    } while (!done);
}

template <int RL>
__global__ void __launch_bounds__(512, 2) ntt_persist_tma_kernel(PersistParams p, int tma_ok) {
    using Ops = FpFwdOps2<RL>;
    constexpr int T = 512;
    extern __shared__ __align__(1024) u64 psm[];          // two 4096-word tiles
    __shared__ __align__(8) u64 s_mbar[2];
    __shared__ int s_next[2], s_land[2];
    const int per = p.n1 + p.n2;
    const int tid = threadIdx.x;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_mbar[0])) : "memory");
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&s_mbar[1])) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        s_next[0] = (int)atomicAdd(p.ctr, 1u);
        s_land[0] = 0;
    }
    __syncthreads();
    unsigned phase[2] = {0u, 0u};
    int par = 0;
    for (;;) {
        const int t = s_next[par];
        const int landed = s_land[par];
        if (t >= p.total) break;
        unsigned nxt = 0;
        if (tid == 0) nxt = atomicAdd(p.ctr, 1u);
        const int s = t / per, j = t - s * per;
        u64* buf = psm + par * 4096;
        // thread 0: publish the next ticket; if it is a pass-2 tile whose pass-1 tiles are done, start its bulk copy now
        auto publish = [&]() {
            const int tn = (int)nxt;
            int land = 0;
            if (tn < p.total && tma_ok) {
                const int sn = tn / per, jn = tn - sn * per;
                const int ltn = sn - p.D;
                if (jn >= p.n1 && ltn >= 0 && ld_acquire_u32(p.ctr + 1 + ltn) >= (unsigned)p.n1) {
                    const TileRef tr = tile_ref(p, ltn);
                    const u64* src = tr.out + ((size_t)(jn - p.n1) << 12);
                    const unsigned dst = smem_u32(psm + (par ^ 1) * 4096), bar = smem_u32(&s_mbar[par ^ 1]);
                    asm volatile("fence.proxy.async;" ::: "memory");      // generic-proxy stores of the producers -> async-proxy read
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(32768u) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(dst), "l"(src), "r"(32768u), "r"(bar) : "memory");
                    land = 1;
                }
            }
            s_next[par ^ 1] = tn;
            s_land[par ^ 1] = land;
        };
        int lt1 = -1;
        bool done_publish = false;
        if (j < p.n1) {
            if (s < p.nLT) { Ops::pass1(p, s, j, buf); lt1 = s; }
        } else {
            const int lt = s - p.D;
            if (lt >= 0) {
                const int chunk = j - p.n1;
                const TileRef tr = tile_ref(p, lt);
                const LimbConst& L = p.limbs[tr.limb];
                u64* io = tr.out + ((size_t)chunk << 12);
                if (landed) {
                    mbar_wait_parity(smem_u32(&s_mbar[par]), phase[par]);
                    phase[par] ^= 1u;
                    Ops::template round1<1>(L, io, buf, chunk, tid);
                } else {
                    const unsigned* c = p.ctr + 1 + lt;
                    while (ld_acquire_u32(c) < (unsigned)p.n1) __nanosleep(64);
                    Ops::template round1<0>(L, io, buf, chunk, tid);
                }
                if (tid == 0) publish();
                done_publish = true;
                __syncthreads();
                Ops::tail(p, L, io, buf, chunk, tid, tr.mul);
            }
        }
        if (!done_publish && tid == 0) publish();
        __syncthreads();
        if (lt1 >= 0 && tid == 0) {
            __threadfence();
            atomicAdd(p.ctr + 1 + lt1, 1u);
        }
        par ^= 1;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Fourth-generation loop (LGPU_NTT_PERSIST_V=6, A/B), forward FP64 with the register copy-out: STATIC tile schedule (tile t belongs to CTA t mod grid;
// every CTA of the persistent grid is resident and walks its tiles in increasing order, and a pass-2 tile only ever waits for tiles with smaller
// numbers, so the smallest unfinished tile is never blocked) and a DOUBLE-BUFFERED tile: no ticket atomics, no ticket hand-over, and the only CTA
// barrier left is the one after round 1 of a pass-2 tile (it also separates the two uses of a buffer, since every warp passes it between them).
// Pass-1 tiles (registers only) publish per warp: __syncwarp, then lane 0 fences and bumps the limb-transform's counter (target n1 x warps).
// ---------------------------------------------------------------------------------------------------------------------
template <class Ops>
__global__ void __launch_bounds__(Ops::T, Ops::MINB) ntt_persist3_kernel(PersistParams p) {
    extern __shared__ u64 psm[];
    const int per = p.n1 + p.n2;
    const unsigned need = (unsigned)p.n1 * (Ops::T / 32);
    int par = 0;
    for (int t = blockIdx.x; t < p.total; t += gridDim.x) {
        const int s = t / per, j = t - s * per;
        if (j < p.n1) {
            if (s < p.nLT) {
                Ops::pass1(p, s, j, psm);
                __syncwarp();
                if ((threadIdx.x & 31) == 0) { __threadfence(); atomicAdd(p.ctr + 1 + s, 1u); }
            }
        } else {
            const int lt = s - p.D;
            if (lt >= 0) {
                if ((threadIdx.x & 31) == 0) {
                    const unsigned* c = p.ctr + 1 + lt;
                    while (ld_acquire_u32(c) < need) __nanosleep(64);
                }
                __syncwarp();
                Ops::pass2(p, lt, j - p.n1, psm + (par << 12));
                par ^= 1;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static int env_int(const char* name, int dflt) {
    const char* e = getenv(name);
    return e ? atoi(e) : dflt;
}

// The development switches of the persistent kernels, read once per process.
//   v: 1 = first generation (padded tile, CTA barriers, serial ticket), 2 = first-generation tile code under the claim-ahead loop,
//      3 (default) = swizzled tile + pair/warp syncs + claim-ahead loop, 4 = 3 + TMA bulk prefetch of the next chunk (no faster than
//      3 on the H100: 0.73 vs 0.71 us per limb-transform, profiles/h100_ntt_ab.json), 5 = 3 with the register copy-out (FpFwdOps3),
//      6 = 5 under the static-schedule / double-buffered loop
//   iv: integer forward tile code, 3 (default) = 512 x 8 swizzled (IntFwdOps2), 2 = 256 x 16 padded (IntFwdOps)
//   ph1int: FpFwdOps with an integer first pass
//   d: the distance D, > 0 overrides the default
struct PersistSwitches {
    int v, iv, ph1int, d;
};
static const PersistSwitches& switches() {
    static const PersistSwitches s = {env_int("LGPU_NTT_PERSIST_V", 3), env_int("LGPU_NTT_PERSIST_IV", 3), env_int("LGPU_NTT_PH1INT", 0),
                                      env_int("LGPU_NTT_PERSIST_D", 0)};
    return s;
}

struct Occupancy {
    int blocks;        // resident CTAs per SM, at least 1
    cudaError_t err;
};
template <class K>
static Occupancy occupancy(K kern, int threads, size_t smem) {
    Occupancy o = {0, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)};
    if (o.err == cudaSuccess) o.err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o.blocks, kern, threads, smem);
    if (o.blocks < 1) o.blocks = 1;
    return o;
}

// One launch of the persistent loop KERN running the tile code Ops, p filled but for the tiles, the distance and the counters. The
// grid is every resident CTA (SMs x occupancy; the static schedule relies on never having more), clamped to the number of tiles.
template <class Ops, auto KERN, class... Extra>
static int persist_launch(const char* name, size_t smem, const Ctx* c, PersistParams p, cudaStream_t st, Extra... extra) {
    static const Occupancy occ = occupancy(KERN, Ops::T, smem);
    if (occ.err != cudaSuccess) { set_error(std::string(name) + ": " + cudaGetErrorString(occ.err)); return -1; }
    p.n1 = Ops::kN1; p.n2 = Ops::kN2;
    const int per = p.n1 + p.n2;
    const long tiles = (long)p.nLT * per;
    int grid = c->sms * occ.blocks;
    if ((long)grid > tiles) grid = (int)tiles;
    // distance: the pass-1 tiles of a step must have left the machine when its pass-2 tiles are drawn, i.e. D steps should
    // hold ~2.5x the resident CTAs
    int D = switches().d > 0 ? switches().d : (int)((5L * grid / 2 + per - 1) / per);
    if (D < 1) D = 1;
    p.D = D;
    p.total = (p.nLT + D) * per;
    const size_t bytes = (size_t)(1 + p.nLT) * sizeof(unsigned);
    LGPU_CUDA_OK(cudaMallocAsync((void**)&p.ctr, bytes, st));
    LGPU_CUDA_OK(cudaMemsetAsync(p.ctr, 0, bytes, st));
    KERN<<<grid, Ops::T, smem, st>>>(p, extra...);
    cudaError_t e = cudaGetLastError();
    cudaFreeAsync(p.ctr, st);
    if (e != cudaSuccess) { set_error(std::string(name) + ": " + cudaGetErrorString(e)); return -1; }
    return 0;
}

// the first-generation loop (v = 1) or the claim-ahead loop (v >= 2)
template <class Ops>
static int ticket_loop(const Ctx* c, const PersistParams& p, cudaStream_t st, bool claim_ahead) {
    if (claim_ahead) return persist_launch<Ops, ntt_persist2_kernel<Ops>>("ntt_persist2_kernel", Ops::kSmem, c, p, st);
    return persist_launch<Ops, ntt_persist_kernel<Ops>>("ntt_persist_kernel", Ops::kSmem, c, p, st);
}

// vec: the output (and the multiplicand, if any) takes 128-bit accesses
template <int RL>
static int persist_dispatch(const Ctx* c, const PersistParams& p, bool inverse, int kind, bool vec, bool vec_out, cudaStream_t st) {
    const PersistSwitches& sw = switches();
    if (kind == 0) {
        if (inverse) return ticket_loop<FpInvOps<RL>>(c, p, st, sw.v >= 2);
        if (sw.ph1int) return ticket_loop<FpFwdOps<RL, 1>>(c, p, st, false);
        if (sw.v == 4)
            return persist_launch<FpFwdOps2<RL>, ntt_persist_tma_kernel<RL>>("ntt_persist_tma_kernel", 2 * 4096 * sizeof(u64), c, p, st,
                                                                            vec_out ? 1 : 0);
        if (sw.v == 6 && vec)
            return persist_launch<FpFwdOps3<RL>, ntt_persist3_kernel<FpFwdOps3<RL>>>("ntt_persist3_kernel", 2 * FpFwdOps3<RL>::kSmem, c, p, st);
        if (sw.v == 5 && vec) return ticket_loop<FpFwdOps3<RL>>(c, p, st, true);
        if (sw.v >= 3) return ticket_loop<FpFwdOps2<RL>>(c, p, st, true);
        return ticket_loop<FpFwdOps<RL, 0>>(c, p, st, sw.v == 2);
    }
    if (!inverse && sw.iv >= 3)
        return kind == 1 ? ticket_loop<IntFwdOps2<RL, true>>(c, p, st, true) : ticket_loop<IntFwdOps2<RL, false>>(c, p, st, true);
    if (kind == 1) return inverse ? ticket_loop<IntInvOps<RL, 1>>(c, p, st, sw.v >= 2) : ticket_loop<IntFwdOps<RL, 1>>(c, p, st, sw.v >= 2);
    return inverse ? ticket_loop<IntInvOps<RL, 2>>(c, p, st, sw.v >= 2) : ticket_loop<IntFwdOps<RL, 2>>(c, p, st, sw.v >= 2);
}

bool ntt_persist_supported(const Ctx* c) {
    return c->ring_type == 0 && c->logN >= 13 && c->logN <= 16;
}

// kind: 0 = FP64-pipe rows (all rows fp_ok), 1 / 2 = integer rows with / without lazy corrections
int launch_ntt_persist(const Ctx* c, const RowMap& rm, bool inverse, int kind, CSpan in, Span out, int batch, cudaStream_t st, CSpan mul) {
    if (mul.p && inverse) { set_error("the fused multiply epilogue exists for forward transforms only"); return -1; }
    PersistParams p;
    p.limbs = c->d_limbs; p.rm = rm; p.in = in.p; p.out = out.p;
    p.in_rs = in.row_stride; p.in_bs = in.batch_stride; p.out_rs = out.row_stride; p.out_bs = out.batch_stride;
    p.logN = c->logN; p.batch = batch; p.nLT = rm.nrows * batch;
    p.mul = mul.p; p.mul_rs = mul.row_stride; p.mul_bs = mul.batch_stride;
    const bool vec_out = aligned16(out.p) && even_words(out.row_stride, out.batch_stride);
    const bool vec = vec_out && (!mul.p || (aligned16(mul.p) && even_words(mul.row_stride, mul.batch_stride)));
    switch (c->logN - 12) {
        case 1: return persist_dispatch<1>(c, p, inverse, kind, vec, vec_out, st);
        case 2: return persist_dispatch<2>(c, p, inverse, kind, vec, vec_out, st);
        case 3: return persist_dispatch<3>(c, p, inverse, kind, vec, vec_out, st);
        case 4: return persist_dispatch<4>(c, p, inverse, kind, vec, vec_out, st);
    }
    set_error("persistent transform: unsupported ring degree");
    return -1;
}

}  // namespace lgpu

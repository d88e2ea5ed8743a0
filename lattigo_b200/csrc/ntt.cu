// ntt.cu -- forward / inverse negacyclic NTT over (limb, coeff) row-major uint64 polynomials.
//
// Replaces ring.Ring.NTT / NTTLazy / INTT / INTTLazy and the per-row SubRing forms
// (reference: ring/ntt.go:127-152,174-206, hot loops nttUnrolled16Lazy :258-552 and
// inttLazyUnrolled16 :608-714).
//
// Decomposition (N = 2^logN, one launch covers rows x batch):
//   forward : [strided pass: first s1 = max(0, logN-12) stages, radix-2^s1 in registers, no smem]
//             -> [chunk pass: remaining c = logN - s1 <= 12 stages on contiguous 2^c-element chunks,
//                 radix-16 register rounds exchanged through padded shared memory]
//   inverse : chunk pass (stages in reverse order, Gentleman-Sande) -> strided pass (+ N^-1 scaling).
// Every element crosses HBM twice per transform when logN > 12 (the intermediate stays L2-resident only while
// the launch's working set fits in the 50 MB L2), once when logN <= 12.
//
// Arithmetic, two variants selected at compile time (template parameter FAST):
//   FAST = false : forward only: the reference's lazy Montgomery butterflies (ring/ntt.go:155-171) with the reference's own
//                  4q-correction schedule, so NTT_EXACT_LAZY reproduces NTTLazy's representative in [0, 6q)
//                  bit for bit (used only when a caller asks for the Lazy API).
//   FAST = true  : free-form path for canonical outputs (NTT / INTT / INTTLazy for N >= 16): Shoup products with
//                  precomputed quotients {w, floor(w 2^64 / q)} -- 6 IMAD.WIDE + 4 IMAD per modular product instead
//                  of ~17 IMAD-class instructions for MRedLazy -- Harvey-style lazy ranges whose correction schedule
//                  is computed per prime (none at all for primes below 2^58), the forward output canonicalised by one
//                  Barrett pass in the store epilogue, the inverse's N^-1 folded into its last stage. The canonical
//                  residue is unique, so the result is bit-identical to the reference's NTTStandard / INTTStandard.
#include <cstdlib>
#include "../../include/lattigo_b200.h"
#include "engine.h"
#include "modarith.cuh"
#include "ntt_arith.cuh"

namespace lgpu {

struct NttParams {
    const LimbConst* limbs;
    RowMap rm;
    const u64* in;
    u64* out;
    size_t in_rs, in_bs, out_rs, out_bs;
    int logN;
    int mode;     // NttMode
    int ci;       // conjugate-invariant ring (stage numbering differs) -- not handled by these kernels
};

// ---------------------------------------------------------------------------------------------------
// strided pass: global stages [0, RL). Thread l handles elements {k * (N >> RL) + l}.
// ---------------------------------------------------------------------------------------------------
template <int RL, bool INVERSE, int FAST>
__global__ void __launch_bounds__(256) ntt_strided_kernel(NttParams p) {
    static_assert(!INVERSE || FAST != 0, "the inverse transform has fast kernels only");
    constexpr int R = 1 << RL;
    const int b = blockIdx.z;
    const LimbConst L = p.limbs[p.rm.limb[blockIdx.y]];
    const int row = p.rm.drow[blockIdx.y];
    const int N = 1 << p.logN;
    const int stride = N >> RL;
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= stride) return;
    const u64* in = p.in + (size_t)b * p.in_bs + (size_t)row * p.in_rs;
    u64* out = p.out + (size_t)b * p.out_bs + (size_t)row * p.out_rs;
    const u64 q = L.q, qinv = L.qinv;
    u64 x[R];
#pragma unroll
    for (int k = 0; k < R; k++) x[k] = in[(size_t)k * stride + l];
    if constexpr (!INVERSE && !FAST) {
        const u64* roots = L.roots_fwd;
#pragma unroll
        for (int u = 0; u < RL; u++) {
            const int half = 1 << (RL - 1 - u);
            const bool red = fwd_reduce_flag(u, p.logN);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                u64 tw = __ldg(roots + (1 << u) + (k >> (RL - u)));
                fwd_bfly(x[k], x[k + half], tw, q, qinv, red);
            }
        }
    } else if constexpr (!INVERSE && FAST) {
        const ulonglong2* tw = L.tw_fwd;
        const u64 nq = 0ull - q, twoq = q << 1;
#pragma unroll
        for (int u = 0; u < RL; u++) {
            const int half = 1 << (RL - 1 - u);
            const bool corr = (FAST == 1) && ((L.fwd_mask >> u) & 1u);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                const ulonglong2 w = __ldg(tw + (1 << u) + (k >> (RL - u)));
                fast_fwd_bfly(x[k], x[k + half], w, nq, twoq, L.kq, corr);
            }
        }
    } else {
        const ulonglong2* tw = L.tw_bwd;
        const bool lazy = (FAST == 2) || (FAST == 1 && L.inv_lazy != 0);
        const int cl = p.logN - RL;   // stages already done by the chunk pass
#pragma unroll
        for (int u = RL - 1; u >= 1; u--) {
            const int half = 1 << (RL - 1 - u);
            // stage index counted from the first inverse stage: cl + (RL-1-u); inputs are < 2^(idx+1) q when lazy
            const u64 addq = lazy ? (q << (cl + (RL - 1 - u) + 1)) : (q << 1);
#pragma unroll
            for (int k = 0; k < R; k++) {
                if (k & half) continue;
                const ulonglong2 w = __ldg(tw + (1 << u) + (k >> (RL - u)));
                fast_inv_bfly(x[k], x[k + half], w, q, addq, !lazy);
            }
        }
        {   // last stage (u = 0) with N^-1 folded in: X = (U + V) * N^-1, Y = (U - V) * (w * N^-1); canonical outputs
            constexpr int half = 1 << (RL - 1);
            const u64 addq = lazy ? (q << p.logN) : (q << 1);
#pragma unroll
            for (int k = 0; k < half; k++) {
                const u64 U = x[k], V = x[k + half];
                const u64 a = shoup_mul(U + V, L.ninv_s, q);
                const u64 c = shoup_mul(U - V + addq, L.last_inv_s, q);
                x[k] = a >= q ? a - q : a;
                x[k + half] = c >= q ? c - q : c;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < R; k++) out[(size_t)k * stride + l] = x[k];
}

// ---------------------------------------------------------------------------------------------------
// chunk pass: global stages [s1, logN) on a contiguous chunk of C = 2^CL elements held in shared memory.
// ---------------------------------------------------------------------------------------------------
template <int CL, int FAST, int MINB = 1>
__global__ void __launch_bounds__((1 << CL) >= 16 ? ((1 << CL) / 16) : 1, MINB)
ntt_chunk_fwd_kernel(NttParams p) {
    constexpr int C = 1 << CL;
    constexpr int T = C / 16;
    constexpr int R0 = round_bits(CL, 0), R1 = round_bits(CL, 1), R2 = round_bits(CL, 2);
    extern __shared__ u64 sm[];
    const int b = blockIdx.z, chunk = blockIdx.x, tid = threadIdx.x;
    const LimbConst L = p.limbs[p.rm.limb[blockIdx.y]];
    const int row = p.rm.drow[blockIdx.y];
    const int s1 = p.logN - CL;
    // for logN > 12 the strided pass already moved the data to `out`
    const u64* src = (s1 > 0 ? (const u64*)p.out + (size_t)b * p.out_bs + (size_t)row * p.out_rs
                             : p.in + (size_t)b * p.in_bs + (size_t)row * p.in_rs) + ((size_t)chunk << CL);
    u64* dst = p.out + (size_t)b * p.out_bs + (size_t)row * p.out_rs + ((size_t)chunk << CL);
    const u64 q = L.q;
    if constexpr (FAST != 0 && CL == 12) {
        // the last round reads 15 twiddle pairs per thread (61 KB per CTA): pull their lines into L1 now, while
        // the first two rounds run, so the round does not start on an L2 round trip
        const ulonglong2* tw = L.tw_fwd;
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int s = s1 + 8 + u;
            const ulonglong2* a = tw + (1 << s) + (chunk << (8 + u)) + (tid << u);
            asm volatile("prefetch.global.L1 [%0];" ::"l"(a));
        }
    }
    fwd_round<CL, 0, R0, true, FAST>(sm, src, L, s1, p.logN, chunk, tid);
    __syncthreads();
    if constexpr (R1 > 0) {
        fwd_round<CL, R0, R1, false, FAST>(sm, nullptr, L, s1, p.logN, chunk, tid);
        __syncthreads();
    }
    if constexpr (R2 > 0) {
        fwd_round<CL, R0 + R1, R2, false, FAST>(sm, nullptr, L, s1, p.logN, chunk, tid);
        __syncthreads();
    }
    const bool canon = (FAST != 0) || (p.mode == NTT_CANONICAL);
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const int idx = k * T + tid;
        u64 v = sm[pad_idx(idx)];
        if (canon) v = bred_add(v, q, L.bred_hi);   // reducevec, ring/ntt.go:176
        dst[idx] = v;
    }
}

template <int CL, int FAST>
__global__ void __launch_bounds__((1 << CL) >= 16 ? ((1 << CL) / 16) : 1)
ntt_chunk_inv_kernel(NttParams p) {
    static_assert(FAST != 0, "the inverse transform has fast kernels only");
    constexpr int C = 1 << CL;
    constexpr int T = C / 16;
    constexpr int NR = num_rounds(CL);
    constexpr int R0 = round_bits(CL, 0), R1 = round_bits(CL, 1), R2 = round_bits(CL, 2);
    extern __shared__ u64 sm[];
    const int b = blockIdx.z, chunk = blockIdx.x, tid = threadIdx.x;
    const LimbConst L = p.limbs[p.rm.limb[blockIdx.y]];
    const int row = p.rm.drow[blockIdx.y];
    const int s1 = p.logN - CL;
    const u64* src = p.in + (size_t)b * p.in_bs + (size_t)row * p.in_rs + ((size_t)chunk << CL);
    u64* dst = p.out + (size_t)b * p.out_bs + (size_t)row * p.out_rs + ((size_t)chunk << CL);
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const int idx = k * T + tid;
        sm[pad_idx(idx)] = src[idx];
    }
    __syncthreads();
    // deepest round first
    if constexpr (NR == 3) {
        inv_round<CL, R0 + R1, R2, false, false, FAST>(sm, nullptr, L, s1, chunk, tid);
        __syncthreads();
    }
    if constexpr (NR >= 2) {
        inv_round<CL, R0, R1, false, false, FAST>(sm, nullptr, L, s1, chunk, tid);
        __syncthreads();
    }
    if (s1 == 0) inv_round<CL, 0, R0, true, true, FAST>(sm, dst, L, s1, chunk, tid);
    else         inv_round<CL, 0, R0, true, false, FAST>(sm, dst, L, s1, chunk, tid);
}

// ---------------------------------------------------------------------------------------------------
// host launchers
// ---------------------------------------------------------------------------------------------------
template <bool INV, int FAST, int CL>
static void launch_chunk(const NttParams& p, dim3 grid, cudaStream_t st) {
    constexpr int C = 1 << CL;
    constexpr int T = C >= 16 ? C / 16 : 1;
    const size_t smem = (size_t)(C + (C >> 4) + 1) * sizeof(u64);
    if constexpr (INV) {
        ntt_chunk_inv_kernel<CL, FAST><<<grid, T, smem, st>>>(p);
    } else if constexpr (FAST == 2 && CL == 12) {
        static const int minb = [] { const char* e = getenv("LGPU_NTT_MINB"); return e ? atoi(e) : 2; }();
        if (minb == 3) ntt_chunk_fwd_kernel<CL, 2, 3><<<grid, T, smem, st>>>(p);
        else if (minb == 4) ntt_chunk_fwd_kernel<CL, 2, 4><<<grid, T, smem, st>>>(p);
        else ntt_chunk_fwd_kernel<CL, 2, 2><<<grid, T, smem, st>>>(p);
    } else {
        ntt_chunk_fwd_kernel<CL, FAST><<<grid, T, smem, st>>>(p);
    }
}

template <bool INV, int FAST>
static int launch_chunk_dyn(int cl, const NttParams& p, dim3 grid, cudaStream_t st) {
    switch (cl) {
        case 4: launch_chunk<INV, FAST, 4>(p, grid, st); break;
        case 5: launch_chunk<INV, FAST, 5>(p, grid, st); break;
        case 6: launch_chunk<INV, FAST, 6>(p, grid, st); break;
        case 7: launch_chunk<INV, FAST, 7>(p, grid, st); break;
        case 8: launch_chunk<INV, FAST, 8>(p, grid, st); break;
        case 9: launch_chunk<INV, FAST, 9>(p, grid, st); break;
        case 10: launch_chunk<INV, FAST, 10>(p, grid, st); break;
        case 11: launch_chunk<INV, FAST, 11>(p, grid, st); break;
        case 12: launch_chunk<INV, FAST, 12>(p, grid, st); break;
        default: set_error("unsupported chunk size"); return -1;
    }
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

template <bool INV, int FAST>
static int launch_strided(int rl, const NttParams& p, int rows, int batch, cudaStream_t st) {
    const int N = 1 << p.logN;
    const int threads_total = N >> rl;
    const int bs = threads_total < 256 ? threads_total : 256;
    dim3 grid((threads_total + bs - 1) / bs, rows, batch);
    switch (rl) {
        case 1: ntt_strided_kernel<1, INV, FAST><<<grid, bs, 0, st>>>(p); break;
        case 2: ntt_strided_kernel<2, INV, FAST><<<grid, bs, 0, st>>>(p); break;
        case 3: ntt_strided_kernel<3, INV, FAST><<<grid, bs, 0, st>>>(p); break;
        case 4: ntt_strided_kernel<4, INV, FAST><<<grid, bs, 0, st>>>(p); break;
        case 5: ntt_strided_kernel<5, INV, FAST><<<grid, bs, 0, st>>>(p); break;
        default: set_error("unsupported strided radix"); return -1;
    }
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// the two-pass integer transform: forward strided pass then chunk pass, inverse chunk pass then strided pass (in place on `out`)
template <bool INV, int FAST>
static int launch_int_two_pass(const Ctx* c, const RowMap& rm, int mode, CSpan in, Span out, int batch, cudaStream_t st) {
    NttParams p;
    p.limbs = c->d_limbs; p.rm = rm; p.in = in.p; p.out = out.p;
    p.in_rs = in.row_stride; p.in_bs = in.batch_stride; p.out_rs = out.row_stride; p.out_bs = out.batch_stride;
    p.logN = c->logN; p.mode = mode; p.ci = 0;
    const int cl = c->logN > 12 ? 12 : c->logN;
    const int s1 = c->logN - cl;
    const dim3 grid(1u << s1, rm.nrows, batch);
    if constexpr (INV) {
        if (launch_chunk_dyn<true, FAST>(cl, p, grid, st)) return -1;
        if (s1 == 0) return 0;
        p.in = out.p; p.in_rs = out.row_stride; p.in_bs = out.batch_stride;
        return launch_strided<true, FAST>(s1, p, rm.nrows, batch, st);
    } else {
        if (s1 > 0 && launch_strided<false, FAST>(s1, p, rm.nrows, batch, st)) return -1;
        return launch_chunk_dyn<false, FAST>(cl, p, grid, st);
    }
}

// fast: 2 = every limb of the launch needs no lazy correction at all (forward: fwd_mask == 0; inverse: inv_lazy), so the
// correction code is compiled out; 1 = per-limb schedules evaluated at run time; 0 = the reference's Montgomery arithmetic
// (forward NTT_EXACT_LAZY only: INTTLazy == INTT for N >= 16, ring/ntt.go:197-206, so both inverse modes are canonical).
static int fast_variant(const Ctx* c, const RowMap& rm, bool inverse) {
    for (int r = 0; r < rm.nrows; r++) {
        const LimbConst& L = c->h_limbs[rm.limb[r]];
        if (inverse ? (L.inv_lazy == 0) : (L.fwd_mask != 0)) return 1;
    }
    return 2;
}

static int launch_int_two_pass(const Ctx* c, const RowMap& rm, bool inverse, int fast, int mode, CSpan in, Span out, int batch,
                               cudaStream_t st) {
    if (inverse) return fast == 2 ? launch_int_two_pass<true, 2>(c, rm, mode, in, out, batch, st)
                                  : launch_int_two_pass<true, 1>(c, rm, mode, in, out, batch, st);
    return fast == 2 ? launch_int_two_pass<false, 2>(c, rm, mode, in, out, batch, st)
         : fast == 1 ? launch_int_two_pass<false, 1>(c, rm, mode, in, out, batch, st)
                     : launch_int_two_pass<false, 0>(c, rm, mode, in, out, batch, st);
}

// LGPU_NTT_PERSIST: 0 = never, 1 = every canonical transform the persistent kernels serve, unset = launches of at least 64
// limb-transforms. H100 (700 W), N = 2^16 x 44 limbs x 16 polynomials, us per limb-transform persistent vs two-pass
// (profiles/h100_ntt_ab.json): forward 0.71 vs 1.14 (45-bit chain) and 1.05 vs 1.27 (61-bit primes), inverse 0.76 vs 0.99 and
// 1.17 vs 1.24. But the tile queue pays a fill / drain of ~D limb-transforms: one 44-limb polynomial (44 limb-transforms), forward
// 1.57 vs 1.87 us per limb-transform on the 45-bit chain but 1.78 vs 1.76 on 61-bit primes, inverse 1.71 vs 1.66 and 1.86 vs
// 1.78, so launches below 64 limb-transforms keep the two-pass kernels.
static bool persistent(const Ctx* c, int limb_transforms) {
    static const int forced = [] { const char* e = getenv("LGPU_NTT_PERSIST"); return e ? atoi(e) : -1; }();
    return forced != 0 && ntt_persist_supported(c) && (forced == 1 || limb_transforms >= 64);
}

// one row class of a transform: the FP64-pipe rows (fp64) or the integer rows (their fast_variant), persistent or two-pass;
// mul: the product fused into a persistent forward FP64 launch
static int launch_rows(const Ctx* c, const RowMap& rm, bool inverse, bool fp64, int fast, bool persist, int mode, CSpan in, Span out,
                       int batch, CSpan mul, cudaStream_t st) {
    ProfScope ps(inverse ? LGPU_KCLASS_NTT_INV : LGPU_KCLASS_NTT_FWD, st, (mul.p ? 24.0 : 16.0) * c->N * rm.nrows * batch,
                 persist ? 1 : (c->logN > 12 ? 2 : 1));
    if (persist) return launch_ntt_persist(c, rm, inverse, fp64 ? 0 : fast, in, out, batch, st, mul);
    if (fp64) return launch_ntt_fp64(c, rm, inverse, in, out, batch, st);
    return launch_int_two_pass(c, rm, inverse, fast, mode, in, out, batch, st);
}

// out = out * mul (MulCoeffsMontgomery) on the rows of rm; nothing when there is no multiplicand
static int mul_coeffs(const Ctx* c, const RowMap& rm, CSpan mul, Span out, int batch, cudaStream_t st) {
    if (!mul.p || rm.nrows == 0) return 0;
    return launch_vecop(c, rm, LGPU_OP_MULCOEFFSMONTGOMERY, CSpan{out.p, out.row_stride, out.batch_stride}, mul, out, batch, nullptr, nullptr, 0, 0,
                        c->N, st);
}

static int check_common(const Ctx* c, const RowMap& rm, int batch) {
    if (c->logN < 4 || c->logN > 17) { set_error("NTT requires 16 <= N <= 2^17"); return -1; }
    if (rm.nrows <= 0 || rm.nrows > kMaxRows || batch <= 0 || batch > 65535) { set_error("bad rows/batch"); return -1; }
    return 0;
}

// Every transform's kernels, chosen per row class; mul.p: Ring.NTT followed by Ring.MulCoeffsMontgomery(., mul, out).
//   inverse (both modes): each class goes persistent on its own size;
//   forward, NTT_EXACT_LAZY: the integer Montgomery kernels (FAST = 0) on every row, never persistent;
//   forward, canonical: the FP64 rows go persistent on the size of the whole launch, the integer rows on their own size. The
//     two-pass FP64 forward chunk pass stores 128 bits at a time (the persistent kernels use 64-bit accesses only), so without the
//     persistent kernels an output that is not 16-byte aligned with even strides sends every row to the integer kernels.
//   The product (SURVEY 8(d) C2(ii): 3 rows of traffic instead of the 5 of the two-call sequence) is fused into a persistent FP64
//     launch; the integer rows are bound by the integer pipes, which the product would share, so they and every row of a launch
//     that is not persistent take the coefficient-wise kernel after their transform.
static int transform(const Ctx* c, const RowMap& rm, bool inverse, int mode, CSpan in, Span out, int batch, CSpan mul, cudaStream_t st) {
    if (check_common(c, rm, batch)) return -1;
    if (c->ring_type != 0) {
        if (launch_ntt_ci(c, rm, inverse, in, out, batch, mode == NTT_EXACT_LAZY, st)) return -1;
        return mul_coeffs(c, rm, mul, out, batch, st);
    }
    RowMap fp, rest;
    split_fp64_rows(c, rm, fp, rest);
    if (inverse) {
        if (fp.nrows && launch_rows(c, fp, true, true, 0, persistent(c, fp.nrows * batch), mode, in, out, batch, {}, st)) return -1;
        if (rest.nrows == 0) return 0;
        return launch_rows(c, rest, true, false, fast_variant(c, rest, true), persistent(c, rest.nrows * batch), mode, in, out, batch, {}, st);
    }
    if (mode == NTT_EXACT_LAZY) return launch_rows(c, rm, false, false, 0, false, mode, in, out, batch, {}, st);
    const bool whole = persistent(c, rm.nrows * batch);
    if (!whole && !(aligned16(out.p) && even_words(out.row_stride, out.batch_stride))) { fp.nrows = 0; rest = rm; }
    if (fp.nrows && launch_rows(c, fp, false, true, 0, whole, mode, in, out, batch, whole ? mul : CSpan{}, st)) return -1;
    if (rest.nrows &&
        launch_rows(c, rest, false, false, fast_variant(c, rest, false), persistent(c, rest.nrows * batch), mode, in, out, batch, {}, st))
        return -1;
    return mul_coeffs(c, whole ? rest : rm, mul, out, batch, st);
}

int launch_ntt(const Ctx* c, const RowMap& rm, CSpan in, Span out, int batch, int mode, cudaStream_t st) {
    return transform(c, rm, false, mode, in, out, batch, {}, st);
}

int launch_intt(const Ctx* c, const RowMap& rm, CSpan in, Span out, int batch, int mode, cudaStream_t st) {
    return transform(c, rm, true, mode, in, out, batch, {}, st);
}

int launch_ntt_mul_montgomery(const Ctx* c, const RowMap& rm, CSpan in, CSpan other, Span out, int batch, cudaStream_t st) {
    if (check_common(c, rm, batch)) return -1;
    if (!other.p) { set_error("null operand"); return -1; }
    if (other.p == out.p) { set_error("NTT+MulCoeffsMontgomery: the multiplicand cannot be the output"); return -1; }
    return transform(c, rm, false, NTT_CANONICAL, in, out, batch, other, st);
}

}  // namespace lgpu

// bgv_encoder.cu -- bgv.Encoder (schemes/bgv/encoder.go), batched on the device, ring.Standard only. BFV uses the same encoder.
//   NewEncoder / permuteMatrix                encoder.go:49-133, params.go:76-135   lgpu_bgv_encoder_create (host, once)
//   Encode / Embed (IsBatched)                encoder.go:201-333                    EncodeRingT, RingT2Q(scaleUp), NTT, MForm
//   Encode (!IsBatched)                       encoder.go:148-199                    MulScalar(scale), RingT2Q(true), NTT
//   Decode                                    encoder.go:471-521                    INTT, RingQ2T(scaleDown), DecodeRingT
// Everything is integer arithmetic: the outputs are the reference's words bit for bit (tests/test_gpu_bgv_encoder.py, tolerance 0).
//
// Ring T is a context of its own (degree n = min(N, order / 2) over {t}), so its INTT / NTT are the engine's launchers. Kernels:
//   bgv_enc_load_kernel     values -> the n-word ring-T scratch at perm[i], unmapped slots zero (BRedAdd / the signed rule)
//   bgv_enc_lift_kernel     one thread per (coefficient, batch entry), every Q and P row: MulScalar(scale) mod t, the spread to j * gap,
//                           MulScalarMontgomery(MForm(t^-1 mod q_i)) with SCALE_UP, MForm with IsMontgomery; the NTT launchers follow
//   bgv_dec_level0_kernel   RingQ2T at level 0 (gap 1 and gap > 1)
//   bgv_dec_modup_kernel    RingQ2T at level > 0, gap = 1: MulScalar(t), AddScalar(floor(Q/2)), ModUpExact to {t}, SubScalar, in one
//                           pass over the l + 1 rows
//   bgv_dec_crt_kernel<W>   RingQ2T at level > 0, gap > 1: PolyToBigintCentered + SetCoefficientsBigint through crt.cuh, exact mod t
//   bgv_dec_store_kernel    the ring-T words at perm[i] (or in order in coefficient mode), centred with SIGNED
// Every RingQ2T kernel folds in DecodeRingT's MulScalar(scale^-1 mod t).
#include <algorithm>
#include <vector>
#include "capi_common.h"
#include "composite.h"
#include "bgv_encoder.h"
#include "crt.cuh"
#include "modarith.cuh"

namespace lgpu {

constexpr int kBgvThreads = 256;

struct TMod {                 // ring T's modulus and its reduction constants
    u64 t, qinv, bhi, blo;
};

// int64 word -> ring T (EncodeRingT / Encode, encoder.go:179-186, :243-251): abs = BRedAdd(|c|) (|INT64_MIN| = 2^63 through the
// wrapping negation), T - abs for c < 0. The reference keeps the word T when abs = 0; T and 0 are the same residue and every consumer
// here (the ring-T INTT, MRed) is a function of the residue, so the canonical 0 is stored instead.
__device__ __forceinline__ u64 signed_to_t(u64 c, const TMod& T) {
    const bool neg = (long long)c < 0;
    const u64 abs = bred_add(neg ? 0ull - c : c, T.t, T.bhi);
    return neg ? (abs ? T.t - abs : 0) : abs;
}

// grid (ceil(n / 256), batch): slot i -> coefficient perm[i] of the ring-T polynomial, 0 for i >= n_values
__global__ void __launch_bounds__(kBgvThreads) bgv_enc_load_kernel(const u64* __restrict__ vals, size_t vs, int n_values, int sgn, int n,
                                                                   const unsigned* __restrict__ perm, TMod T, u64* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t b = blockIdx.y;
    u64 w = 0;
    if (i < n_values) {
        const u64 c = vals[b * vs + i];
        w = sgn ? signed_to_t(c, T) : bred_add(c, T.t, T.bhi);       // ringT.Reduce
    }
    out[b * n + perm[i]] = w;
}

// grid (ceil(N / 256), batch). Batched: coefficient col = j * gap takes word j of the ring-T INTT output (RingT2Q's spread), 0 elsewhere.
// Coefficient mode: word col of the values (raw uint64, or the signed rule), 0 past n_values, at gap 1. Then MulScalar(scale) mod t
// (MRed by MForm(scale mod t): any 64-bit word in, canonical out) and per row: MRed by MForm(t^-1 mod q_i) with tinv (RingT2Q's
// MulScalarBigint); otherwise BRedAdd mod q_i when a transform or MForm follows (the reference's NTT and MForm of a word below 2^61 are
// those of its residue, DESIGN.md §3.4), or the literal word; MForm when mont (before the transform: both are linear, the output canonical).
// RAW (RingT2Q of a ring-T polynomial as it is, the multiparty masks): the ring-T word is lifted as the integer it is, without MulScalar,
// so a word in [t, 2^64) keeps the reference's lift.
template <bool RAW = false>
__global__ void __launch_bounds__(kBgvThreads) bgv_enc_lift_kernel(const u64* __restrict__ src, size_t src_bs, int coeffs, int sgn, int n_values,
                                                                   int log_gap, TMod T, u64 smont, const u64* __restrict__ tinv, int canon,
                                                                   int mont, const LimbConst* __restrict__ limbs, int nrows_q, int limb_p0,
                                                                   int nrows_p, u64* __restrict__ out_q, size_t sq, u64* __restrict__ out_p,
                                                                   size_t sp, int N) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= N) return;
    const size_t b = blockIdx.y;
    u64 w = 0;
    if (coeffs) {
        if (col < n_values) {
            const u64 c = src[b * src_bs + col];
            w = mred(sgn ? signed_to_t(c, T) : c, smont, T.t, T.qinv);
        }
    } else if ((col & ((1 << log_gap) - 1)) == 0) {
        w = src[b * src_bs + (col >> log_gap)];
        if (!RAW) w = mred(w, smont, T.t, T.qinv);
    }
    for (int r = 0; r < nrows_q + nrows_p; r++) {
        const bool isq = r < nrows_q;
        const LimbConst& L = limbs[isq ? r : limb_p0 + r - nrows_q];
        u64 x = w;
        if (tinv) x = mred(w, tinv[r], L.q, L.qinv);                   // SCALE_UP: Q rows only
        else if (canon) x = bred_add(w, L.q, L.bred_hi);
        if (mont) x = mform(x, L.q, L.bred_hi, L.bred_lo);
        if (isq) out_q[b * sq + (size_t)r * N + col] = x;
        else out_p[b * sp + (size_t)(r - nrows_q) * N + col] = x;
    }
}

// RingQ2T(level 0, scaleDown) (encoder.go:449-466) of coefficient j << log_gap: MulScalar(t) mod q0, AddScalar(q0 >> 1) (CRed), Reduce mod t,
// SubScalar(BRedAdd(q0 >> 1)) (CRed), then DecodeRingT's MulScalar(scale^-1)
__global__ void __launch_bounds__(kBgvThreads) bgv_dec_level0_kernel(const u64* __restrict__ src, size_t src_bs, int count, int log_gap,
                                                                     LimbConst L0, u64 tmul0, TMod T, u64 half_t, u64 sinv,
                                                                     u64* __restrict__ out, size_t out_bs) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const size_t b = blockIdx.y;
    u64 x = mred(src[b * src_bs + ((size_t)j << log_gap)], tmul0, L0.q, L0.qinv);
    x = cred(x + (L0.q >> 1), L0.q);
    x = bred_add(x, T.t, T.bhi);
    x = cred(x + T.t - half_t, T.t);
    out[b * out_bs + j] = mred(x, sinv, T.t, T.qinv);
}

// ModUpConstants(Q[:l+1], {t}) of one level as device pointers (gen_modup's layout)
struct ModUpT {
    const u64* cinv;     // [L] MForm((Q/q_k)^-1 mod q_k)
    const u64* cmod;     // [L] MForm((Q/q_k) mod t)
    const u64* vt;       // [L + 1] v (t - Q mod t) mod t
    const u64* half_s;   // [L] floor(Q/2) mod q_k
    u64 half_t;          // floor(Q/2) mod t
    int L;
};

// RingQ2T(level > 0, gap = 1, scaleDown) (encoder.go:429-432): per row MulScalar(t), AddScalarBigint(floor(Q/2)), then ModUpExact to {t}
// (ring/basis_extension.go:282-308): y_k = MRed(x_k, cinv_k), v = uint64(sum_k float64(y_k) / float64(q_k)) in limb order with IEEE
// division and no FMA, result = sum_k y_k (Q/q_k) + v (t - Q mod t) mod t. The reference's word is that value plus a multiple of t (its
// lazy multSum); SubScalarBigint's CRed keeps it congruent and the MulScalar(scale^-1) that follows reduces it, so the residue suffices.
// RAW (RingQ2T alone, for the multiparty protocols): the reference's own word instead of the residue -- multSum's 128-bit sum of
// y_k MForm((Q/q_k) mod t), MRedLazy'd, plus v (t - Q mod t) mod t, then SubScalarBigint's CRed: a word in [0, 3t), no MulScalar.
template <bool RAW = false>
__global__ void __launch_bounds__(kBgvThreads) bgv_dec_modup_kernel(const u64* __restrict__ src, size_t src_bs, int N, const LimbConst* __restrict__ limbs,
                                                                    const u64* __restrict__ tmul, ModUpT M, TMod T, u64 sinv,
                                                                    u64* __restrict__ out, size_t out_bs) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= N) return;
    const size_t b = blockIdx.y;
    const u64* x = src + b * src_bs + j;
    double vf = 0.0;
    u64 s = 0, hi = 0, lo = 0;
    for (int k = 0; k < M.L; k++) {
        const u64 q = limbs[k].q, qinv = limbs[k].qinv;
        u64 a = mred(x[(size_t)k * N], tmul[k], q, qinv);
        a = cred(a + M.half_s[k], q);
        const u64 y = mred(a, M.cinv[k], q, qinv);
        vf = __dadd_rn(vf, __ddiv_rn(__ull2double_rn(y), __ull2double_rn(q)));
        if (RAW) {
            u64 ph, pl;
            mul128(y, M.cmod[k], ph, pl);
            lo += pl;
            hi += ph + (lo < pl);
        } else {
            s = cred(s + mred(y, M.cmod[k], T.t, T.qinv), T.t);
        }
    }
    const u64 v = __double2ull_rz(vf);
    if (RAW) {
        out[b * out_bs + j] = cred(mred128_lazy(hi, lo, T.t, T.qinv) + M.vt[v] + T.t - M.half_t, T.t);
        return;
    }
    s = cred(s + M.vt[v], T.t);
    s = cred(s + T.t - M.half_t, T.t);
    out[b * out_bs + j] = mred(s, sinv, T.t, T.qinv);
}

// RingQ2T(level > 0, gap > 1, scaleDown) (encoder.go:433-439): PolyToBigintCentered(MulScalar(t) of the rows, gap) (ring/ring.go:469-508:
// X = CRT mod Q, X - Q when X >= floor(Q/2)), then SetCoefficientsBigint into ring T (Euclidean mod t). X mod t by Horner over the W words
// (r <- r 2^64 + w mod t); the centred value's residue is X mod t - Q mod t.
template <int W>
__global__ void __launch_bounds__(kBgvThreads) bgv_dec_crt_kernel(const u64* __restrict__ src, size_t src_bs, int N, int count, int log_gap,
                                                                  CrtTab C, const LimbConst* __restrict__ limbs, const u64* __restrict__ tmul,
                                                                  u64 qmod_t, TMod T, u64 sinv, u64* __restrict__ out, size_t out_bs) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const size_t b = blockIdx.y;
    const u64* x = src + b * src_bs + ((size_t)j << log_gap);
    u64 acc[W + 1];
    crt_exact_load<W>([&](int k) { return mred(x[(size_t)k * N], tmul[k], limbs[k].q, limbs[k].qinv); }, C, acc);
    const bool ge = mw_ge<W>(acc, C.Qh);
    u64 r = 0;
#pragma unroll
    for (int w = W - 1; w >= 0; w--) r = cred(mform(r, T.t, T.bhi, T.blo) + bred_add(acc[w], T.t, T.bhi), T.t);
    if (ge) r = cred(r + T.t - qmod_t, T.t);
    out[b * out_bs + j] = mred(r, sinv, T.t, T.qinv);
}

// DecodeRingT's gather (encoder.go:356-379) or the coefficient-mode copy (:497-518): out[i] = word perm[i] (i when perm is null), and with
// sgn the int64 rule v >= t >> 1 -> v - t
__global__ void __launch_bounds__(kBgvThreads) bgv_dec_store_kernel(const u64* __restrict__ tb, size_t tb_bs, const unsigned* __restrict__ perm,
                                                                    int count, int sgn, u64 t, u64* __restrict__ out, size_t out_bs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const size_t b = blockIdx.y;
    u64 v = tb[b * tb_bs + (perm ? perm[i] : (unsigned)i)];
    if (sgn && v >= (t >> 1)) v -= t;
    out[b * out_bs + i] = v;
}

// permuteMatrix(logN) (encoder.go:110-133)
static std::vector<unsigned> permute_matrix(int logn) {
    const u64 n = 1ull << logn, mask = 2 * n - 1;
    std::vector<unsigned> perm(n);
    u64 pow = 1;
    for (u64 i = 0, j = n >> 1; i < (n >> 1); i++, j++) {
        u64 pos = 0, x = pow >> 1;                                   // BitReverse64(pow >> 1, logN)
        for (int k = 0; k < logn; k++) pos |= ((x >> k) & 1) << (logn - 1 - k);
        perm[i] = (unsigned)pos;
        perm[j] = (unsigned)(n - pos - 1);
        pow = (pow * 5) & mask;                                      // GaloisGen
    }
    return perm;
}

}  // namespace lgpu

using namespace lgpu;

struct lgpu_bgv_encoder {
    lgpu_ctx* ctx = nullptr;
    Ctx T;                                 // ring T: degree n over {t}
    u64 t = 0;
    int n = 0, log_gap = 0;
    TMod tm{};
    std::vector<unsigned> perm;
    // blob: tmul[nQ] = MForm(t mod q_i) | tinv[nQ] = MForm(t^-1 mod q_i) | GenModUpConstants(Q[:l+1], {t}) for l = 1 .. nQ - 1
    std::vector<u64> blob;
    std::vector<ModUpSet> muc;            // [level], level 0 unused
    unsigned* d_perm = nullptr;
    u64* d_blob = nullptr;
};

extern "C" void lgpu_bgv_encoder_destroy(lgpu_bgv_encoder* e) {
    if (!e) return;
    if (e->T.device >= 0) {
        cudaSetDevice(e->T.device);
        cudaFree(e->d_perm);
        cudaFree(e->d_blob);
    }
    destroy_context(&e->T);
    delete e;
}

extern "C" int lgpu_bgv_encoder_create(lgpu_ctx* ctx, uint64_t t, lgpu_bgv_encoder** out) {
    REQUIRE(ctx && out, "null argument");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "BGV encoding is only supported on the Standard ring (the ConjugateInvariant ring is not)");
    REQUIRE(t >= 2, "invalid parameters: plaintext modulus t must be >= 2");
    REQUIRE(t < c.Q[0], "invalid parameters: t must be smaller than Q[0]");
    for (int i = 0; i < c.nQ; i++) REQUIRE(c.Q[i] != t, "insecure parameters: t|Q");
    // the largest cyclotomic order enabled by t (params.go:119-123): the largest power of two `order` with t = 1 mod order
    const int bl = 64 - __builtin_clzll(t);
    u64 order = bl >= 64 ? 0 : 1ull << bl;
    while (order != 0 && (t & (order - 1)) != 1) order >>= 1;
    REQUIRE(order >= 16, "provided plaintext modulus t has cyclotomic order < 16 (ring degree of minimum 8 is required by the backend)");
    const u64 n = std::min<u64>((u64)c.N, order >> 1);
    REQUIRE(n >= 16, "plaintext ring T of fewer than 16 slots (t = 1 mod 16 but not mod 32) is not supported: the engine's transforms "
                     "start at 16 points");
    int logn = 0;
    while ((1ull << logn) < n) logn++;
    lgpu_bgv_encoder* e = new lgpu_bgv_encoder;
    e->ctx = ctx;
    e->t = t;
    const u64 tw = t;
    if (build_context(&e->T, c.device, logn, 0, &tw, 1, nullptr, 0, false)) {
        const std::string why = last_error();
        lgpu_bgv_encoder_destroy(e);
        set_error("provided plaintext modulus t is invalid: " + why);
        return -1;
    }
    e->n = (int)n;
    while ((e->n << e->log_gap) < c.N) e->log_gap++;
    const HostSubRing& s = e->T.sub[0];
    e->tm = TMod{t, s.qinv, s.bred_hi, s.bred_lo};
    e->perm = permute_matrix(logn);
    std::vector<u64>& b = e->blob;
    for (int i = 0; i < c.nQ; i++) b.push_back(h_mform(t % c.Q[i], c.Q[i]));
    for (int i = 0; i < c.nQ; i++) b.push_back(h_mform(h_invmod(t % c.Q[i], c.Q[i]), c.Q[i]));
    e->muc.resize(c.nQ);
    for (int l = 1; l < c.nQ; l++) e->muc[l] = gen_modup(b, c.Q.data(), l + 1, &tw, 1);
    if (c.device >= 0) {
        if (cudaMalloc(&e->d_perm, n * sizeof(unsigned)) != cudaSuccess || cudaMalloc(&e->d_blob, b.size() * sizeof(u64)) != cudaSuccess ||
            cudaMemcpy(e->d_perm, e->perm.data(), n * sizeof(unsigned), cudaMemcpyHostToDevice) != cudaSuccess ||
            cudaMemcpy(e->d_blob, b.data(), b.size() * sizeof(u64), cudaMemcpyHostToDevice) != cudaSuccess) {
            lgpu_bgv_encoder_destroy(e);
            set_error("BGV encoder: device allocation failed");
            return -1;
        }
    }
    *out = e;
    return 0;
}

static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }

extern "C" int lgpu_bgv_encode(lgpu_bgv_encoder* enc, const uint64_t* values, int n_values, int flags, uint64_t scale, int level_q, uint64_t* out_q,
                               int level_p, uint64_t* out_p, int batch, size_t values_stride, size_t out_q_stride, size_t out_p_stride,
                               void* stream) {
    REQUIRE(enc, "null encoder");
    lgpu_ctx* ctx = enc->ctx;
    const Ctx& c = ctx->c;
    REQUIRE((flags & ~(LGPU_ENC_NTT | LGPU_ENC_MONTGOMERY | LGPU_ENC_COEFFS | LGPU_ENC_SIGNED | LGPU_ENC_SCALE_UP)) == 0, "unknown encoder flags");
    const bool coeffs = flags & LGPU_ENC_COEFFS, ntt = flags & LGPU_ENC_NTT, sgn = flags & LGPU_ENC_SIGNED, up = flags & LGPU_ENC_SCALE_UP;
    const bool mont = !coeffs && (flags & LGPU_ENC_MONTGOMERY);
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(level_q >= 0 && level_q < c.nQ, "level_q out of range");
    REQUIRE(level_p >= -1 && level_p < c.nP, c.nP ? "level_p out of range" : "level_p out of range: the context has no P moduli");
    const int N = c.N, n = enc->n;
    if (coeffs) {
        REQUIRE(up, "coefficient encoding (IsBatched = false) exists only as Encode: LGPU_ENC_SCALE_UP is required");
        REQUIRE(n_values >= 0 && n_values <= N, "cannot Encode (TimeDomain): len(values) > N");
        REQUIRE(level_p == -1, "coefficient encoding (IsBatched = false) writes a ring.Poly: level_p must be -1");
    } else {
        REQUIRE(n_values >= 0 && n_values <= n, "cannot EncodeRingT (FrequencyDomain): len(values) > slots");
    }
    REQUIRE(!(up && level_p >= 0), "Encode (LGPU_ENC_SCALE_UP) writes a ring.Poly: P rows are only written by Embed (the reference's RingT2Q "
                                   "would scale them with the Q moduli)");
    REQUIRE(n_values == 0 || values, "null values");
    REQUIRE(aligned8(values), "values must be 8-byte aligned");
    REQUIRE(out_q && aligned8(out_q), "null or misaligned out_q");
    REQUIRE(level_p < 0 || (out_p && aligned8(out_p)), "null or misaligned out_p");
    REQUIRE(batch == 1 || (values_stride >= (size_t)n_values && out_q_stride >= (size_t)(level_q + 1) * N &&
                           (level_p < 0 || out_p_stride >= (size_t)(level_p + 1) * N)), "batch strides smaller than one entry");
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    const TMod& T = enc->tm;
    const u64 smont = h_mform(scale % T.t, T.t);
    const u64* src = (const u64*)values;
    size_t src_bs = values_stride;
    Scratch buf;
    if (!coeffs) {
        if (buf.alloc((size_t)n * batch, st)) return -1;
        count_launch(1);
        bgv_enc_load_kernel<<<dim3((n + kBgvThreads - 1) / kBgvThreads, batch), kBgvThreads, 0, st>>>(src, values_stride, n_values, sgn, n,
                                                                                                    enc->d_perm, T, buf.p);
        LGPU_CUDA_OK(cudaGetLastError());
        RowMap rt;
        if (make_rowmap(enc->T, LGPU_RING_Q, 0, rt)) return -1;
        if (launch_intt(&enc->T, rt, CSpan{buf.p, (size_t)n, (size_t)n}, Span{buf.p, (size_t)n, (size_t)n}, batch, NTT_CANONICAL, st)) return -1;
        src = buf.p;
        src_bs = n;
    }
    count_launch(1);
    bgv_enc_lift_kernel<<<dim3((N + kBgvThreads - 1) / kBgvThreads, batch), kBgvThreads, 0, st>>>(
        src, src_bs, coeffs, sgn, n_values, coeffs ? 0 : enc->log_gap, T, smont, up ? enc->d_blob + c.nQ : nullptr, ntt || mont, mont,
        c.d_limbs, level_q + 1, c.nQ, level_p + 1, (u64*)out_q, out_q_stride, (u64*)out_p, out_p_stride, N);
    LGPU_CUDA_OK(cudaGetLastError());
    if (ntt) {
        RowMap rm;
        if (make_rowmap(c, LGPU_RING_Q, level_q, rm)) return -1;
        if (launch_ntt(&c, rm, CSpan{(const u64*)out_q, (size_t)N, out_q_stride}, Span{(u64*)out_q, (size_t)N, out_q_stride}, batch, NTT_CANONICAL, st))
            return -1;
        if (level_p >= 0) {
            if (make_rowmap(c, LGPU_RING_P, level_p, rm)) return -1;
            if (launch_ntt(&c, rm, CSpan{(const u64*)out_p, (size_t)N, out_p_stride}, Span{(u64*)out_p, (size_t)N, out_p_stride}, batch,
                           NTT_CANONICAL, st))
                return -1;
        }
    }
    return 0;
}

template <int W>
static void launch_bgv_crt(dim3 grid, cudaStream_t st, const u64* src, size_t src_bs, int N, int count, int log_gap, const CrtTab& C,
                           const LimbConst* limbs, const u64* tmul, u64 qmod_t, const TMod& T, u64 sinv, u64* out, size_t out_bs) {
    bgv_dec_crt_kernel<W><<<grid, kBgvThreads, 0, st>>>(src, src_bs, N, count, log_gap, C, limbs, tmul, qmod_t, T, sinv, out, out_bs);
}

namespace lgpu {

int bgv_q2t_check(const lgpu_bgv_encoder* enc, int level, int log_gap) {
    if (level > 0 && log_gap > 0 && crt_words(enc->ctx->c, level) > kMaxCrtWords) {
        set_error("the bit lengths of q_0..q_level sum past 4096: the CRT accumulator exceeds 4096 bits");
        return -1;
    }
    return 0;
}

// RingQ2T(level, scaleDown = true) of coefficient-domain rows into tn-word ring-T entries (coefficients j << log_gap), followed by
// MulScalar(sinv): the branch choice of encoder.go:429-466 over the three kernels above. setup() stages the CRT table of the big-integer
// branch once; launch() runs one sub-batch. raw keeps the ModUpExact branch's own word (bgv_dec_modup_kernel<true>, sinv = MForm(1)).
struct Q2T {
    const lgpu_bgv_encoder* enc;
    int level, log_gap, tn, W = 0;
    bool big;
    Scratch tab;
    CrtTab C{};
    ModUpT M{};
    u64 qmod_t = 0;
    Q2T(const lgpu_bgv_encoder* e, int l, int lg, int n) : enc(e), level(l), log_gap(lg), tn(n), big(l > 0 && lg > 0) {}
    int setup(cudaStream_t st) {
        const Ctx& c = enc->ctx->c;
        const TMod& T = enc->tm;
        if (big) {
            W = crt_width(crt_words(c, level));
            std::vector<u64> blob = build_crt(c, level, W);
            if (tab.alloc(blob.size(), st)) return -1;
            // pageable source: the call returns once `blob` is staged, so it may die with this function
            LGPU_CUDA_OK(cudaMemcpyAsync(tab.p, blob.data(), blob.size() * 8, cudaMemcpyHostToDevice, st));
            const int L = level + 1;
            C.q = tab.p; C.bhi = tab.p + L; C.blo = tab.p + 2 * L; C.inv = tab.p + 3 * L; C.rq = reinterpret_cast<const double*>(tab.p + 4 * L);
            C.qhat = tab.p + 5 * L; C.Q = C.qhat + (size_t)L * W; C.Qh = C.Q + W; C.L = L;
        }
        qmod_t = 1 % T.t;
        for (int k = 0; k <= level; k++) qmod_t = h_mulmod(qmod_t, c.Q[k] % T.t, T.t);
        if (level > 0) {
            const ModUpSet& s = enc->muc[level];
            M.cinv = enc->d_blob + s.off_qoverqiinvqi; M.cmod = enc->d_blob + s.off_qoverqimodp; M.vt = enc->d_blob + s.off_vtimesqmodp;
            M.half_s = enc->d_blob + s.off_half_s; M.half_t = enc->blob[s.off_half_t]; M.L = level + 1;
        }
        return 0;
    }
    int launch(const u64* src, size_t sstride, u64 sinv, bool raw, u64* out, size_t out_bs, int nb, cudaStream_t st) const {
        const Ctx& c = enc->ctx->c;
        const TMod& T = enc->tm;
        const u64* tmul = enc->d_blob;
        const int N = c.N;
        count_launch(1);
        if (level == 0) {
            bgv_dec_level0_kernel<<<dim3((tn + kBgvThreads - 1) / kBgvThreads, nb), kBgvThreads, 0, st>>>(
                src, sstride, tn, log_gap, c.h_limbs[0], enc->blob[0], T, (c.Q[0] >> 1) % T.t, sinv, out, out_bs);
        } else if (!big) {
            const dim3 grid((N + kBgvThreads - 1) / kBgvThreads, nb);
            if (raw) bgv_dec_modup_kernel<true><<<grid, kBgvThreads, 0, st>>>(src, sstride, N, c.d_limbs, tmul, M, T, sinv, out, out_bs);
            else bgv_dec_modup_kernel<false><<<grid, kBgvThreads, 0, st>>>(src, sstride, N, c.d_limbs, tmul, M, T, sinv, out, out_bs);
        } else {
            const dim3 grid((tn + kBgvThreads - 1) / kBgvThreads, nb);
            switch (W) {
                case 16: launch_bgv_crt<16>(grid, st, src, sstride, N, tn, log_gap, C, c.d_limbs, tmul, qmod_t, T, sinv, out, out_bs); break;
                case 32: launch_bgv_crt<32>(grid, st, src, sstride, N, tn, log_gap, C, c.d_limbs, tmul, qmod_t, T, sinv, out, out_bs); break;
                default: launch_bgv_crt<64>(grid, st, src, sstride, N, tn, log_gap, C, c.d_limbs, tmul, qmod_t, T, sinv, out, out_bs); break;
            }
        }
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }
};

}  // namespace lgpu

extern "C" int lgpu_bgv_decode(lgpu_bgv_encoder* enc, const uint64_t* pt, int level, int flags, uint64_t scale, uint64_t* values, int batch,
                               size_t pt_stride, size_t values_stride, void* stream) {
    REQUIRE(enc, "null encoder");
    lgpu_ctx* ctx = enc->ctx;
    const Ctx& c = ctx->c;
    REQUIRE((flags & ~(LGPU_ENC_NTT | LGPU_ENC_MONTGOMERY | LGPU_ENC_COEFFS | LGPU_ENC_SIGNED)) == 0, "unknown decoder flags");
    const bool coeffs = flags & LGPU_ENC_COEFFS, ntt = flags & LGPU_ENC_NTT, sgn = flags & LGPU_ENC_SIGNED;
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    const int N = c.N, n = enc->n;
    const int tn = coeffs ? N : n;                                   // words of the ring-T buffer per entry
    const int log_gap = coeffs ? 0 : enc->log_gap;
    REQUIRE(pt && aligned8(pt), "null or misaligned plaintext");
    REQUIRE(values && aligned8(values), "null or misaligned values");
    REQUIRE(batch == 1 || (pt_stride >= (size_t)(level + 1) * N && values_stride >= (size_t)tn), "batch strides smaller than one entry");
    if (bgv_q2t_check(enc, level, log_gap)) return -1;
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    const TMod& T = enc->tm;
    const u64 sinv = h_mform(h_powmod(scale % T.t, T.t - 2, T.t), T.t);     // MForm(ModExp(scale, t - 2, t))
    Q2T q2t(enc, level, log_gap, tn);
    if (q2t.setup(st)) return -1;
    const size_t poly = (size_t)(level + 1) * N;
    Scratch tbuf;
    if (tbuf.alloc((size_t)tn * batch, st)) return -1;
    // INTT into scratch in sub-batches of at most ~256 MB (the plaintext is never written)
    const int ch = ntt ? (int)std::max<size_t>(1, std::min<size_t>(batch, ((size_t)256 << 20) / (poly * 8))) : batch;
    Scratch buf;
    if (ntt && buf.alloc(poly * ch, st)) return -1;
    RowMap rm;
    if (make_rowmap(c, LGPU_RING_Q, level, rm)) return -1;
    for (int k = 0; k < batch; k += ch) {
        const int nb = std::min(ch, batch - k);
        const u64* src = (const u64*)pt + (size_t)k * pt_stride;
        size_t sstride = pt_stride;
        if (ntt) {
            if (launch_intt(&c, rm, CSpan{src, (size_t)N, pt_stride}, Span{buf.p, (size_t)N, poly}, nb, NTT_CANONICAL, st)) return -1;
            src = buf.p; sstride = poly;
        }
        if (q2t.launch(src, sstride, sinv, false, tbuf.p + (size_t)k * tn, tn, nb, st)) return -1;
    }
    if (!coeffs) {
        RowMap rt;
        if (make_rowmap(enc->T, LGPU_RING_Q, 0, rt)) return -1;
        if (launch_ntt(&enc->T, rt, CSpan{tbuf.p, (size_t)n, (size_t)n}, Span{tbuf.p, (size_t)n, (size_t)n}, batch, NTT_CANONICAL, st)) return -1;
    }
    // coefficient mode: uint64 returns all N words; int64 centres only the first RingT().N() and leaves the rest (encoder.go:505-518)
    const int count = coeffs && !sgn ? N : n;
    count_launch(1);
    bgv_dec_store_kernel<<<dim3((count + kBgvThreads - 1) / kBgvThreads, batch), kBgvThreads, 0, st>>>(
        tbuf.p, tn, coeffs ? nullptr : enc->d_perm, count, sgn, T.t, (u64*)values, values_stride);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

namespace lgpu {

BgvEncInfo bgv_encoder_info(const lgpu_bgv_encoder* e) { return BgvEncInfo{e->ctx, &e->T, e->t, e->n}; }

int bgv_ring_q2t(const lgpu_bgv_encoder* e, int level, const u64* src, size_t src_bs, u64* out, size_t out_bs, int batch, cudaStream_t st) {
    Q2T q2t(e, level, e->log_gap, e->n);
    if (q2t.setup(st)) return -1;
    return q2t.launch(src, src_bs, h_mform(1, e->t), true, out, out_bs, batch, st);
}

int bgv_ring_t2q(const lgpu_bgv_encoder* e, int level, const u64* pT, size_t pT_bs, u64* out, size_t out_bs, int batch, cudaStream_t st) {
    const Ctx& c = e->ctx->c;
    count_launch(1);
    bgv_enc_lift_kernel<true><<<dim3((c.N + kBgvThreads - 1) / kBgvThreads, batch), kBgvThreads, 0, st>>>(
        pT, pT_bs, 0, 0, 0, e->log_gap, e->tm, 0, e->d_blob + c.nQ, 0, 0, c.d_limbs, level + 1, c.nQ, 0, out, out_bs, nullptr, 0, c.N);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int bgv_encode_ring_t(const lgpu_bgv_encoder* e, const u64* values, size_t vs, u64 scale, u64* pT, int batch, cudaStream_t st) {
    const int n = e->n;
    count_launch(1);
    bgv_enc_load_kernel<<<dim3((n + kBgvThreads - 1) / kBgvThreads, batch), kBgvThreads, 0, st>>>(values, vs, n, 0, n, e->d_perm, e->tm, pT);
    LGPU_CUDA_OK(cudaGetLastError());
    RowMap rt;
    if (make_rowmap(e->T, LGPU_RING_Q, 0, rt)) return -1;
    const Span P{pT, (size_t)n, (size_t)n};
    if (launch_intt(&e->T, rt, CSpan{pT, (size_t)n, (size_t)n}, P, batch, NTT_CANONICAL, st)) return -1;
    return launch_vecop(&e->T, rt, LGPU_OP_MULSCALARMONTGOMERY, CSpan{pT, (size_t)n, (size_t)n}, CSpan{nullptr, 0, 0}, P, batch, nullptr, nullptr,
                        h_mform(scale % e->t, e->t), 0, n, st);
}

int bgv_decode_ring_t(const lgpu_bgv_encoder* e, const u64* pT, size_t pT_bs, u64 scale, u64* values, size_t vs, int batch, cudaStream_t st) {
    const int n = e->n;
    const u64 t = e->t;
    Scratch buf;
    if (buf.alloc((size_t)n * batch, st)) return -1;
    RowMap rt;
    if (make_rowmap(e->T, LGPU_RING_Q, 0, rt)) return -1;
    const Span B{buf.p, (size_t)n, (size_t)n};
    if (launch_vecop(&e->T, rt, LGPU_OP_MULSCALARMONTGOMERY, CSpan{pT, (size_t)n, pT_bs}, CSpan{nullptr, 0, 0}, B, batch, nullptr, nullptr,
                     h_mform(h_powmod(scale % t, t - 2, t), t), 0, n, st)) return -1;
    if (launch_ntt(&e->T, rt, CSpan{buf.p, (size_t)n, (size_t)n}, B, batch, NTT_CANONICAL, st)) return -1;
    count_launch(1);
    bgv_dec_store_kernel<<<dim3((n + kBgvThreads - 1) / kBgvThreads, batch), kBgvThreads, 0, st>>>(buf.p, n, e->d_perm, n, 0, t, values, vs);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // namespace lgpu

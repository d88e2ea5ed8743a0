// mp_refresh.cu -- the scheme-level threshold protocols of multiparty/mpbgv and multiparty/mpckks on the device, NTT-domain ciphertexts
// on the Standard ring, paramsIn == paramsOut. mpckks (EncToShare / ShareToEnc / Refresh with big-integer masks): lgpu_mpckks_*, below
// the mpckks marker. mpbgv:
//   EncToShareProtocol.GenShare                  mpbgv/sharing.go:62-71     lgpu_mpbgv_e2s_share (mask from lgpu_mpbgv_sample_mask)
//   EncToShareProtocol.GetShare                  mpbgv/sharing.go:78-91     lgpu_mpbgv_e2s_get_share
//   ShareToEncProtocol.GenShare                  mpbgv/sharing.go:126-143   lgpu_mpbgv_s2e_share
//   MaskedTransformProtocol.Transform, after the transform: RingT2Q, NTT, Add(aggS2E), c1 = crp (mpbgv/transform.go:173-180)
//                                                                            lgpu_mpbgv_recrypt
//   MaskedTransformFunc's DecodeRingT / EncodeRingT (mpbgv/transform.go:83-100)   lgpu_mpbgv_decode_ring_t / lgpu_mpbgv_encode_ring_t
// MaskedTransformProtocol.GenShare and RefreshProtocol are these steps in sequence (lattigo_b200/mpbgv.py). Sampled polynomials are
// inputs, as in multiparty.cu. Every result keeps the reference's words, which need not be canonical: the E2S and S2E shares lie in
// [0, 2q) (a KeySwitch share in [0, 2q) followed by Sub = CRed(a + q - b) or Add = CRed(a + b) of a canonical word), and RingQ2T at a
// level > 0 with gap 1 returns ModUpExact's lazy word in [0, 3t), which GetShare's ring-T Add and Transform's RingT2Q take as it is.
#include <cstring>
#include "../../include/lattigo_b200.h"
#include "bgv_encoder.h"
#include "crt.cuh"
#include "capi_common.h"
#include "composite.h"
#include "modarith.cuh"

namespace lgpu {

// KeySwitchProtocol.GenShare(sk, 0) then Sub(share, m) (E2S), or KeySwitchProtocol.GenShare(0, sk) then Add(share, m) (S2E), NTT domain.
// On entry share = NTT(e) and m = NTT(RingT2Q(mask)): share = CRed(MRedLazy(c1, CRed(s_in + q - s_out)) + share), then CRed(share + q - m)
// or CRed(share + m).
struct MaskShareParams {
    const LimbConst* limbs;
    const u64* c1; size_t c1_bs;
    const u64* sk;
    const u64* m;
    u64* share; size_t share_bs;
    int n;
};
template <bool E2S>
__global__ void __launch_bounds__(256) mpbgv_share_kernel(MaskShareParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int r = blockIdx.y, b = blockIdx.z;
    const LimbConst& L = p.limbs[r];
    const size_t w = (size_t)r * p.n + i;
    const u64 s = p.sk[w];
    const u64 d = E2S ? cred(s + L.q, L.q) : cred(L.q - s, L.q);
    const size_t o = (size_t)b * p.share_bs + w;
    const u64 x = cred(mred_lazy(p.c1[(size_t)b * p.c1_bs + w], d, L.q, L.qinv) + p.share[o], L.q);
    const u64 m = p.m[o];
    p.share[o] = E2S ? cred(x + L.q - m, L.q) : cred(x + m, L.q);
}

// the E2S / S2E share of `batch` ciphertexts at `level` given m = NTT(lifted mask) ([batch][level + 1][N])
template <bool E2S>
static int masked_share(const Ctx* c, int level, const u64* c1, size_t stride, const u64* sk, const long long* e, const u64* m, u64* share,
                        int batch, cudaStream_t st) {
    const size_t N = c->N, nq = (size_t)level + 1, poly = nq * N;
    const RowMap rq = rows_range(0, 0, (int)nq);
    const Span sh{share, N, poly};
    if (small_to_rns(c, rq, e, N, sh, batch, st)) return -1;
    if (launch_ntt(c, rq, CSpan{share, N, poly}, sh, batch, NTT_CANONICAL, st)) return -1;
    MaskShareParams p;
    p.limbs = c->d_limbs; p.c1 = c1; p.c1_bs = stride; p.sk = sk; p.m = m; p.share = share; p.share_bs = poly; p.n = c->N;
    count_launch(1);
    mpbgv_share_kernel<E2S><<<dim3((c->N + 255) / 256, (unsigned)nq, batch), 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

template <bool E2S>
static int mpbgv_share(const lgpu_bgv_encoder* enc, int level, const u64* c1, size_t stride, const u64* sk, const long long* e, const u64* mask,
                       u64* share, int batch, cudaStream_t st) {
    const BgvEncInfo E = bgv_encoder_info(enc);
    const Ctx* c = &E.ctx->c;
    const size_t N = c->N, poly = ((size_t)level + 1) * N;
    const RowMap rq = rows_range(0, 0, level + 1);
    Scratch m;
    if (m.alloc((size_t)batch * poly, st)) return -1;
    if (bgv_ring_t2q(enc, level, mask, E.n, m.p, poly, batch, st)) return -1;
    if (launch_ntt(c, rq, CSpan{m.p, N, poly}, Span{m.p, N, poly}, batch, NTT_CANONICAL, st)) return -1;
    return masked_share<E2S>(c, level, c1, stride, sk, e, m.p, share, batch, st);
}

// ---- mpckks: big-integer masks ----------------------------------------------------------------------------------------------------
// A value is W little-endian two's-complement words (W = 4 or 8, mpckks_words). Lifted values sit at coefficient j << log_gap of rows
// that are zero elsewhere: SetCoefficientsBigint of the dslots values followed by NTTSparseAndMontgomery is the NTT of that spread
// polynomial (rlwe/utils.go:187-240), which the engine's transform computes.

// a <- floor(a / s) for a 128-bit s = (s1:s0) > 0, by restoring division over a 129-bit remainder
template <int NW>
__device__ __forceinline__ void mw_div128(u64 (&a)[NW], u64 s0, u64 s1) {
    u64 r0 = 0, r1 = 0;
#pragma unroll
    for (int w = NW - 1; w >= 0; w--) {
        const u64 x = a[w];
        u64 q = 0;
        for (int b = 63; b >= 0; b--) {
            const u64 top = r1 >> 63;
            r1 = (r1 << 1) | (r0 >> 63);
            r0 = (r0 << 1) | ((x >> b) & 1);
            if (top || r1 > s1 || (r1 == s1 && r0 >= s0)) {
                const u64 br = r0 < s0;
                r0 -= s0;
                r1 = r1 - s1 - br;
                q |= 1ull << b;
            }
        }
        a[w] = q;
    }
}

// the signed value v (W words) -> Quo(Mul(v, d), s) when scaled (big.Int truncation toward zero), then Mod(., q_r) (Euclidean) for rows
// 0..nrows-1, written at coefficient j << log_gap of out
struct BigScale { u64 d0, d1, s0, s1; int on; };
template <int W>
__device__ __forceinline__ void lift_signed(const u64 (&v)[W], const BigScale& S, const LimbConst* __restrict__ limbs, int nrows, u64* out,
                                            size_t rs, size_t col) {
    constexpr int NW = W + 2;
    const bool neg = (long long)v[W - 1] < 0;
    u64 a[NW];
    u64 c = neg;
#pragma unroll
    for (int w = 0; w < W; w++) {                              // |v|
        const u64 x = neg ? ~v[w] : v[w];
        a[w] = x + c;
        c = c && a[w] == 0;
    }
    a[W] = a[W + 1] = 0;
    if (S.on) {
        u64 p[NW];
#pragma unroll
        for (int w = 0; w < NW; w++) p[w] = 0;
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const u64 dk = k ? S.d1 : S.d0;
            u64 carry = 0;
#pragma unroll
            for (int i = 0; i < W; i++) {
                u64 hi, lo;
                mul128(a[i], dk, hi, lo);
                lo += carry; hi += lo < carry;
                p[i + k] += lo; hi += p[i + k] < lo;
                carry = hi;
            }
            p[W + k] += carry;
        }
        mw_div128<NW>(p, S.s0, S.s1);
#pragma unroll
        for (int w = 0; w < NW; w++) a[w] = p[w];
    }
    for (int r = 0; r < nrows; r++) {
        const LimbConst& L = limbs[r];
        u64 x = 0;
#pragma unroll
        for (int w = NW - 1; w >= 0; w--) x = cred(mform(x, L.q, L.bred_hi, L.bred_lo) + bred_add(a[w], L.q, L.bred_hi), L.q);
        out[(size_t)r * rs + col] = neg && x ? L.q - x : x;
    }
}

// SetCoefficientsBigint (+ the refresh scaling) of `batch` x dslots values: grid (ceil(dslots / 256), batch), out zeroed beforehand
template <int W>
__global__ void __launch_bounds__(256) mpckks_lift_kernel(const u64* __restrict__ words, size_t wbs, int dslots, int log_gap, BigScale S,
                                                          const LimbConst* __restrict__ limbs, int nrows, u64* __restrict__ out, size_t obs, int N) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= dslots) return;
    const size_t b = blockIdx.y;
    u64 v[W];
#pragma unroll
    for (int w = 0; w < W; w++) v[w] = words[b * wbs + (size_t)j * W + w];
    lift_signed<W>(v, S, limbs, nrows, out + b * obs, N, (size_t)j << log_gap);
}

// PolyToBigintCentered at gap (ring.go:469-508) of coefficient-domain rows, plus the secret share (GetShare's Add), written as words;
// with `lift`, the refresh's Mul / Quo by the scales and SetCoefficientsBigint at the output level
template <int W>
__global__ void __launch_bounds__(256) mpckks_decode_kernel(const u64* __restrict__ src, size_t sbs, CrtTab C, int dslots, int log_gap,
                                                            const u64* __restrict__ secret, u64* __restrict__ out, size_t wbs, BigScale S,
                                                            const LimbConst* __restrict__ limbs, int nrows, u64* __restrict__ lift, size_t lbs,
                                                            int N) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= dslots) return;
    const size_t b = blockIdx.y;
    u64 acc[W + 1];
    crt_exact<W>(src + b * sbs + ((size_t)j << log_gap), N, C, acc);
    u64 v[W];
    if (mw_ge<W>(acc, C.Qh)) {                                  // X - Q, as W two's-complement words
        u64 br = 0;
#pragma unroll
        for (int w = 0; w < W; w++) {
            const u64 a = acc[w], q = C.Q[w];
            v[w] = a - q - br;
            br = (a < q) || (a - q < br);
        }
    } else {
#pragma unroll
        for (int w = 0; w < W; w++) v[w] = acc[w];
    }
    if (secret) {
        u64 c = 0;
#pragma unroll
        for (int w = 0; w < W; w++) {
            const u64 s = secret[b * wbs + (size_t)j * W + w];
            const u64 t = v[w] + s;
            const u64 c1 = t < v[w];
            v[w] = t + c;
            c = c1 | (v[w] < t);
        }
    }
    if (out) {
#pragma unroll
        for (int w = 0; w < W; w++) out[b * wbs + (size_t)j * W + w] = v[w];
    }
    if (lift) lift_signed<W>(v, S, limbs, nrows, lift + b * lbs, N, (size_t)j << log_gap);
}

// words per value of the mpckks shares at an E2S level: the smallest of 4 and 8 with room for Q_level plus 16 bits (sums of up to 2^15
// shares stay exact); 0 past 8 words
static int mpckks_words(const Ctx& c, int level) {
    int bits = 0;
    for (int k = 0; k <= level; k++) bits += 64 - __builtin_clzll(c.Q[k]);
    return bits + 16 <= 256 ? 4 : bits + 16 <= 512 ? 8 : 0;
}
static int bitlen_Q(const Ctx& c, int level) {
    std::vector<u64> q{1};
    for (int k = 0; k <= level; k++) mw_mul_small(q, c.Q[k]);
    while (q.size() > 1 && q.back() == 0) q.pop_back();
    return 64 * ((int)q.size() - 1) + 64 - __builtin_clzll(q.back());
}
static int log2_gap(const Ctx& c, int log_slots) {
    int g = 0;
    while (((size_t)2 << (log_slots + g)) < (size_t)c.N) g++;
    return g;
}

static int mpckks_lift(const Ctx* c, int level, int log_slots, int W, const u64* words, const BigScale& S, u64* out, size_t obs, int batch,
                       cudaStream_t st) {
    const int dslots = 2 << log_slots, lg = log2_gap(*c, log_slots);
    LGPU_CUDA_OK(cudaMemset2DAsync(out, obs * 8, 0, (size_t)(level + 1) * c->N * 8, batch, st));
    const dim3 grid((dslots + 255) / 256, batch);
    count_launch(1);
    if (W == 4) mpckks_lift_kernel<4><<<grid, 256, 0, st>>>(words, (size_t)dslots * W, dslots, lg, S, c->d_limbs, level + 1, out, obs, c->N);
    else mpckks_lift_kernel<8><<<grid, 256, 0, st>>>(words, (size_t)dslots * W, dslots, lg, S, c->d_limbs, level + 1, out, obs, c->N);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// Add(agg, ct0), INTT and mpckks_decode_kernel at the E2S level `level`
static int mpckks_decode(const Ctx* c, int level, int log_slots, int W, const u64* ct0, size_t stride, const u64* agg, const u64* secret, u64* out,
                         const BigScale& S, int level_out, u64* lift, size_t lbs, int batch, cudaStream_t st) {
    const size_t N = c->N, poly = (size_t)(level + 1) * N;
    RowMap rq;
    if (make_rowmap(*c, LGPU_RING_Q, level, rq)) return -1;
    Scratch buf, tab;
    if (buf.alloc((size_t)batch * poly, st)) return -1;
    const Span B{buf.p, N, poly};
    if (launch_vecop(c, rq, LGPU_OP_ADD, CSpan{agg, N, poly}, CSpan{ct0, N, stride}, B, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
    if (launch_intt(c, rq, CSpan{buf.p, N, poly}, B, batch, NTT_CANONICAL, st)) return -1;
    std::vector<u64> blob = build_crt(*c, level, W);
    if (tab.alloc(blob.size(), st)) return -1;
    // pageable source: the call returns once `blob` is staged, so it may die with this function
    LGPU_CUDA_OK(cudaMemcpyAsync(tab.p, blob.data(), blob.size() * 8, cudaMemcpyHostToDevice, st));
    const int L = level + 1;
    CrtTab C{};
    C.q = tab.p; C.bhi = tab.p + L; C.blo = tab.p + 2 * L; C.inv = tab.p + 3 * L; C.rq = reinterpret_cast<const double*>(tab.p + 4 * L);
    C.qhat = tab.p + 5 * L; C.Q = C.qhat + (size_t)L * W; C.Qh = C.Q + W; C.L = L;
    const int dslots = 2 << log_slots, lg = log2_gap(*c, log_slots);
    if (lift) LGPU_CUDA_OK(cudaMemset2DAsync(lift, lbs * 8, 0, (size_t)(level_out + 1) * N * 8, batch, st));
    const dim3 grid((dslots + 255) / 256, batch);
    count_launch(1);
    if (W == 4)
        mpckks_decode_kernel<4><<<grid, 256, 0, st>>>(buf.p, poly, C, dslots, lg, secret, out, (size_t)dslots * W, S, c->d_limbs, level_out + 1, lift, lbs, c->N);
    else
        mpckks_decode_kernel<8><<<grid, 256, 0, st>>>(buf.p, poly, C, dslots, lg, secret, out, (size_t)dslots * W, S, c->d_limbs, level_out + 1, lift, lbs, c->N);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

static int check_ckks(lgpu_ctx* ctx, int level, int log_slots, int W, int batch) {
    if (!ctx) { set_error("null context"); return -1; }
    const Ctx& c = ctx->c;
    if (c.ring_type != 0) { set_error("the mpckks protocols are only supported on the Standard ring"); return -1; }
    if (level < 0 || level >= c.nQ) { set_error("level out of range"); return -1; }
    if (batch < 1 || batch > 65535) { set_error("batch out of range"); return -1; }
    if (log_slots < 0 || ((size_t)2 << log_slots) > (size_t)c.N) { set_error("log_slots out of range: 2 * slots must divide N"); return -1; }
    if (W != 4 && W != 8) { set_error("share words W must be 4 or 8"); return -1; }
    return 0;
}
static int get_scale(const uint64_t* scales, BigScale& S) {
    S = BigScale{1, 0, 1, 0, 0};
    if (!scales) return 0;
    if ((scales[0] | scales[1]) == 0 || (scales[2] | scales[3]) == 0) { set_error("scales must be positive integers"); return -1; }
    S = BigScale{scales[0], scales[1], scales[2], scales[3], 1};
    return 0;
}

// the checks every entry point shares: the encoder, the level, the batch
static int check_common(const lgpu_bgv_encoder* enc, int level, int batch, BgvEncInfo& E) {
    if (!enc) { set_error("null encoder"); return -1; }
    E = bgv_encoder_info(enc);
    if (level < 0 || level >= E.ctx->c.nQ) { set_error("level out of range"); return -1; }
    if (batch < 1 || batch > 65535) { set_error("batch out of range"); return -1; }
    return 0;
}

}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_mpbgv_sample_mask(lgpu_bgv_encoder* enc, uint64_t seed, uint64_t stream_id, uint64_t* mask, int batch, void* stream) {
    BgvEncInfo E;
    if (check_common(enc, 0, batch, E)) return -1;
    REQUIRE(mask, "null argument");
    REQUIRE_DEVICE(E.ctx);
    return sample_mask(E.t, E.n, seed, stream_id, (u64*)mask, E.n, batch, (cudaStream_t)stream);
}

int lgpu_mpbgv_e2s_share(lgpu_bgv_encoder* enc, int level, const uint64_t* c1, size_t stride, const uint64_t* sk, const int64_t* e,
                         const uint64_t* mask, uint64_t* share, int batch, void* stream) {
    BgvEncInfo E;
    if (check_common(enc, level, batch, E)) return -1;
    const size_t N = E.ctx->c.N;
    REQUIRE(c1 && sk && e && mask && share, "null argument");
    REQUIRE(stride >= (size_t)(level + 1) * N, "stride below (level + 1) * N");
    const size_t sbytes = (size_t)batch * (level + 1) * N * sizeof(u64), cbytes = ((size_t)(batch - 1) * stride + (size_t)(level + 1) * N) * sizeof(u64);
    REQUIRE(!overlaps(share, sbytes, c1, cbytes), "share overlaps the ciphertexts");
    REQUIRE_DEVICE(E.ctx);
    return mpbgv_share<true>(enc, level, (const u64*)c1, stride, (const u64*)sk, (const long long*)e, (const u64*)mask, (u64*)share, batch,
                             (cudaStream_t)stream);
}

int lgpu_mpbgv_s2e_share(lgpu_bgv_encoder* enc, int level, const uint64_t* crp, const uint64_t* sk, const int64_t* e, const uint64_t* mask,
                         uint64_t* share, int batch, void* stream) {
    BgvEncInfo E;
    if (check_common(enc, level, batch, E)) return -1;
    const size_t poly = (size_t)(level + 1) * E.ctx->c.N;
    REQUIRE(crp && sk && e && mask && share, "null argument");
    REQUIRE(!overlaps(share, batch * poly * sizeof(u64), crp, batch * poly * sizeof(u64)), "share overlaps the crp");
    REQUIRE_DEVICE(E.ctx);
    return mpbgv_share<false>(enc, level, (const u64*)crp, poly, (const u64*)sk, (const long long*)e, (const u64*)mask, (u64*)share, batch,
                              (cudaStream_t)stream);
}

int lgpu_mpbgv_e2s_get_share(lgpu_bgv_encoder* enc, int level, const uint64_t* ct0, size_t stride, const uint64_t* agg, const uint64_t* secret,
                             uint64_t* out, int batch, void* stream) {
    BgvEncInfo E;
    if (check_common(enc, level, batch, E)) return -1;
    const Ctx& c = E.ctx->c;
    const size_t N = c.N, poly = (size_t)(level + 1) * N;
    REQUIRE(ct0 && agg && out, "null argument");
    REQUIRE(stride >= poly, "stride below (level + 1) * N");
    const size_t obytes = (size_t)batch * E.n * sizeof(u64);
    REQUIRE(!overlaps(out, obytes, ct0, ((size_t)(batch - 1) * stride + poly) * sizeof(u64)) && !overlaps(out, obytes, agg, batch * poly * sizeof(u64)),
            "out overlaps the ciphertexts or the share");
    int log_gap = 0;
    while (((size_t)E.n << log_gap) < N) log_gap++;
    if (bgv_q2t_check(enc, level, log_gap)) return -1;
    REQUIRE_DEVICE(E.ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    RowMap rq;
    if (make_rowmap(c, LGPU_RING_Q, level, rq)) return -1;
    Scratch buf;
    if (buf.alloc((size_t)batch * poly, st)) return -1;
    const Span B{buf.p, N, poly};
    // Add(aggregatePublicShare, ct[0]), INTT, RingQ2T (sharing.go:83-85)
    if (launch_vecop(&c, rq, LGPU_OP_ADD, CSpan{(const u64*)agg, N, poly}, CSpan{(const u64*)ct0, N, stride}, B, batch, nullptr, nullptr, 0, 0,
                     c.N, st)) return -1;
    if (launch_intt(&c, rq, CSpan{buf.p, N, poly}, B, batch, NTT_CANONICAL, st)) return -1;
    if (bgv_ring_q2t(enc, level, buf.p, poly, (u64*)out, E.n, batch, st)) return -1;
    if (!secret) return 0;
    // RingT().Add(secretShare, buffT) (:87)
    RowMap rt;
    if (make_rowmap(*E.T, LGPU_RING_Q, 0, rt)) return -1;
    const size_t n = E.n;
    return launch_vecop(E.T, rt, LGPU_OP_ADD, CSpan{(const u64*)secret, n, n}, CSpan{(const u64*)out, n, n}, Span{(u64*)out, n, n}, batch, nullptr,
                        nullptr, 0, 0, E.n, st);
}

int lgpu_mpbgv_recrypt(lgpu_bgv_encoder* enc, int level, const uint64_t* mask, const uint64_t* agg, const uint64_t* crp, uint64_t* ct_out, int batch,
                       void* stream) {
    BgvEncInfo E;
    if (check_common(enc, level, batch, E)) return -1;
    const Ctx& c = E.ctx->c;
    const size_t N = c.N, poly = (size_t)(level + 1) * N;
    REQUIRE(mask && agg && crp && ct_out, "null argument");
    const size_t obytes = (size_t)batch * 2 * poly * sizeof(u64), ibytes = (size_t)batch * poly * sizeof(u64);
    REQUIRE(!overlaps(ct_out, obytes, agg, ibytes) && !overlaps(ct_out, obytes, crp, ibytes), "ct_out overlaps the share or the crp");
    REQUIRE_DEVICE(E.ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    RowMap rq;
    if (make_rowmap(c, LGPU_RING_Q, level, rq)) return -1;
    u64* c0 = (u64*)ct_out;
    const Span C0{c0, N, 2 * poly};
    // RingT2Q(maxLevel, true, mask), NTT, Add(tmpPt, ShareToEncShare) (transform.go:175-178); GetEncryption's c1 = crp
    if (bgv_ring_t2q(enc, level, (const u64*)mask, E.n, c0, 2 * poly, batch, st)) return -1;
    if (launch_ntt(&c, rq, CSpan{c0, N, 2 * poly}, C0, batch, NTT_CANONICAL, st)) return -1;
    if (launch_vecop(&c, rq, LGPU_OP_ADD, CSpan{c0, N, 2 * poly}, CSpan{(const u64*)agg, N, poly}, C0, batch, nullptr, nullptr, 0, 0, c.N, st))
        return -1;
    LGPU_CUDA_OK(cudaMemcpy2DAsync(c0 + poly, 2 * poly * sizeof(u64), crp, poly * sizeof(u64), poly * sizeof(u64), batch, cudaMemcpyDeviceToDevice,
                                   st));
    return 0;
}

int lgpu_mpbgv_encode_ring_t(lgpu_bgv_encoder* enc, const uint64_t* values, uint64_t scale, uint64_t* pt, int batch, void* stream) {
    BgvEncInfo E;
    if (check_common(enc, 0, batch, E)) return -1;
    REQUIRE(values && pt, "null argument");
    REQUIRE_DEVICE(E.ctx);
    return bgv_encode_ring_t(enc, (const u64*)values, E.n, scale, (u64*)pt, batch, (cudaStream_t)stream);
}

int lgpu_mpbgv_decode_ring_t(lgpu_bgv_encoder* enc, const uint64_t* pt, uint64_t scale, uint64_t* values, int batch, void* stream) {
    BgvEncInfo E;
    if (check_common(enc, 0, batch, E)) return -1;
    REQUIRE(pt && values, "null argument");
    REQUIRE_DEVICE(E.ctx);
    return bgv_decode_ring_t(enc, (const u64*)pt, E.n, scale, (u64*)values, E.n, batch, (cudaStream_t)stream);
}

int lgpu_mpckks_sample_mask(lgpu_ctx* ctx, int log_slots, int log_bound, int W, uint64_t seed, uint64_t stream_id, uint64_t* mask, int batch,
                            void* stream) {
    if (check_ckks(ctx, 0, log_slots, W, batch)) return -1;
    REQUIRE(log_bound >= 1 && log_bound < 64 * W, "log_bound out of [1, 64 W)");
    REQUIRE(mask, "null argument");
    REQUIRE_DEVICE(ctx);
    const int dslots = 2 << log_slots;
    return sample_big_mask(dslots, W, log_bound, seed, stream_id, (u64*)mask, (size_t)dslots * W, batch, (cudaStream_t)stream);
}

int lgpu_mpckks_e2s_share(lgpu_ctx* ctx, int level, int log_slots, int log_bound, const uint64_t* c1, size_t stride, const uint64_t* sk,
                          const int64_t* e, const uint64_t* mask, int W, uint64_t* share, int batch, void* stream) {
    if (check_ckks(ctx, level, log_slots, W, batch)) return -1;
    const Ctx& c = ctx->c;
    const size_t N = c.N, poly = (size_t)(level + 1) * N;
    REQUIRE(c1 && sk && e && mask && share, "null argument");
    REQUIRE(stride >= poly, "stride below (level + 1) * N");
    REQUIRE(mpckks_words(c, level) != 0 && W >= mpckks_words(c, level), "share words W below what Q at the E2S level needs (4 or 8 words)");
    REQUIRE(log_bound >= 1 && bitlen_Q(c, level) > log_bound, "cannot GenShare: ciphertext level is not large enough for refresh correctness");
    const size_t cbytes = ((size_t)(batch - 1) * stride + poly) * sizeof(u64);
    REQUIRE(!overlaps(share, batch * poly * sizeof(u64), c1, cbytes), "share overlaps the ciphertexts");
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    Scratch m;
    if (m.alloc((size_t)batch * poly, st)) return -1;
    if (mpckks_lift(&c, level, log_slots, W, (const u64*)mask, BigScale{1, 0, 1, 0, 0}, m.p, poly, batch, st)) return -1;
    const RowMap rq = rows_range(0, 0, level + 1);
    if (launch_ntt(&c, rq, CSpan{m.p, N, poly}, Span{m.p, N, poly}, batch, NTT_CANONICAL, st)) return -1;
    return masked_share<true>(&c, level, (const u64*)c1, stride, (const u64*)sk, (const long long*)e, m.p, (u64*)share, batch, st);
}

int lgpu_mpckks_s2e_share(lgpu_ctx* ctx, int level, int log_slots, const uint64_t* crp, const uint64_t* sk, const int64_t* e, const uint64_t* secret,
                          int W, const uint64_t* scales, uint64_t* share, int batch, void* stream) {
    if (check_ckks(ctx, level, log_slots, W, batch)) return -1;
    const Ctx& c = ctx->c;
    const size_t N = c.N, poly = (size_t)(level + 1) * N;
    REQUIRE(crp && sk && e && secret && share, "null argument");
    REQUIRE(!overlaps(share, batch * poly * sizeof(u64), crp, batch * poly * sizeof(u64)), "share overlaps the crp");
    BigScale S;
    if (get_scale(scales, S)) return -1;
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    Scratch m;
    if (m.alloc((size_t)batch * poly, st)) return -1;
    if (mpckks_lift(&c, level, log_slots, W, (const u64*)secret, S, m.p, poly, batch, st)) return -1;
    const RowMap rq = rows_range(0, 0, level + 1);
    if (launch_ntt(&c, rq, CSpan{m.p, N, poly}, Span{m.p, N, poly}, batch, NTT_CANONICAL, st)) return -1;
    return masked_share<false>(&c, level, (const u64*)crp, poly, (const u64*)sk, (const long long*)e, m.p, (u64*)share, batch, st);
}

int lgpu_mpckks_e2s_get_share(lgpu_ctx* ctx, int level, int log_slots, const uint64_t* ct0, size_t stride, const uint64_t* agg, const uint64_t* secret,
                              int W, uint64_t* out, int batch, void* stream) {
    if (check_ckks(ctx, level, log_slots, W, batch)) return -1;
    const Ctx& c = ctx->c;
    const size_t poly = (size_t)(level + 1) * c.N;
    REQUIRE(ct0 && agg && out, "null argument");
    REQUIRE(stride >= poly, "stride below (level + 1) * N");
    REQUIRE(mpckks_words(c, level) != 0 && W >= mpckks_words(c, level), "share words W below what Q at the E2S level needs (4 or 8 words)");
    const size_t obytes = (size_t)batch * (2 << log_slots) * W * sizeof(u64);
    REQUIRE(!overlaps(out, obytes, ct0, ((size_t)(batch - 1) * stride + poly) * sizeof(u64)) && !overlaps(out, obytes, agg, batch * poly * sizeof(u64)),
            "out overlaps the ciphertexts or the share");
    REQUIRE_DEVICE(ctx);
    return mpckks_decode(&c, level, log_slots, W, (const u64*)ct0, stride, (const u64*)agg, (const u64*)secret, (u64*)out, BigScale{1, 0, 1, 0, 0}, 0,
                         nullptr, 0, batch, (cudaStream_t)stream);
}

int lgpu_mpckks_refresh_finalize(lgpu_ctx* ctx, int level_in, int log_slots, const uint64_t* ct0, size_t stride, const uint64_t* agg_e2s,
                                 int level_out, const uint64_t* agg_s2e, const uint64_t* crp, int W, const uint64_t* scales, uint64_t* ct_out,
                                 int batch, void* stream) {
    if (check_ckks(ctx, level_in, log_slots, W, batch)) return -1;
    const Ctx& c = ctx->c;
    REQUIRE(level_out >= 0 && level_out < c.nQ, "level out of range");
    const size_t N = c.N, pin = (size_t)(level_in + 1) * N, pout = (size_t)(level_out + 1) * N;
    REQUIRE(ct0 && agg_e2s && agg_s2e && crp && ct_out && scales, "null argument");
    REQUIRE(stride >= pin, "stride below (level + 1) * N");
    REQUIRE(mpckks_words(c, level_in) != 0 && W >= mpckks_words(c, level_in), "share words W below what Q at the E2S level needs (4 or 8 words)");
    BigScale S;
    if (get_scale(scales, S)) return -1;
    const size_t obytes = (size_t)batch * 2 * pout * sizeof(u64);
    REQUIRE(!overlaps(ct_out, obytes, ct0, ((size_t)(batch - 1) * stride + pin) * sizeof(u64)) &&
                !overlaps(ct_out, obytes, agg_e2s, batch * pin * sizeof(u64)) && !overlaps(ct_out, obytes, agg_s2e, batch * pout * sizeof(u64)) &&
                !overlaps(ct_out, obytes, crp, batch * pout * sizeof(u64)),
            "ct_out overlaps an input");
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    u64* c0 = (u64*)ct_out;
    // GetShare(nil), Mul / Quo by the scales, SetCoefficientsBigint at the output level (transform.go:215-247), then NTT, Add(aggS2E), c1 = crp
    if (mpckks_decode(&c, level_in, log_slots, W, (const u64*)ct0, stride, (const u64*)agg_e2s, nullptr, nullptr, S, level_out, c0, 2 * pout, batch, st))
        return -1;
    RowMap rq;
    if (make_rowmap(c, LGPU_RING_Q, level_out, rq)) return -1;
    const Span C0{c0, N, 2 * pout};
    if (launch_ntt(&c, rq, CSpan{c0, N, 2 * pout}, C0, batch, NTT_CANONICAL, st)) return -1;
    if (launch_vecop(&c, rq, LGPU_OP_ADD, CSpan{c0, N, 2 * pout}, CSpan{(const u64*)agg_s2e, N, pout}, C0, batch, nullptr, nullptr, 0, 0, c.N, st))
        return -1;
    LGPU_CUDA_OK(cudaMemcpy2DAsync(c0 + pout, 2 * pout * sizeof(u64), crp, pout * sizeof(u64), pout * sizeof(u64), batch, cudaMemcpyDeviceToDevice, st));
    return 0;
}

}  // extern "C"

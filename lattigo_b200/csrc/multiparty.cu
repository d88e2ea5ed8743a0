// multiparty.cu -- the coefficient loops of the threshold protocols of multiparty/ on the device (SURVEY L5).
//
//   AggregateShares (every protocol)                      e.g. multiparty/keyswitch_sk.go:123-130, keygen_cpk.go:86-89
//   KeySwitchProtocol.GenShare, ct.IsNTT branch           multiparty/keyswitch_sk.go:85-118
//   PublicKeySwitchProtocol.GenShare, ct.IsNTT branch     multiparty/keyswitch_pk.go:69-105
//   EvaluationKeyGenProtocol.GenShare                     multiparty/keygen_evk.go:86-183 (gadget_encrypt, encrypt.cu)
//   GaloisKeyGenProtocol.GenShare                         multiparty/keygen_gal.go:48-70
//   RelinearizationKeyGenProtocol.GenShareRoundOne / Two  multiparty/keygen_relin.go:91-234
//   Thresholdizer.GenShamirSecretShare, many recipients   multiparty/threshold.go:102-104
// PublicKeyGenProtocol.GenShare is Encryptor.encryptZeroSkFromC1QP with c1 = crp (encrypt.cu), so it has no entry point here.
// Sampled polynomials are inputs, as in encrypt.cu. Every result keeps the reference's representative, which need not be canonical:
// a KeySwitch share lies in [0, 2q), and a left fold of K shares by Add = CRed(a + b) grows by up to q per share.
#include <cstring>
#include "../../include/lattigo_b200.h"
#include "capi_common.h"
#include "composite.h"
#include "modarith.cuh"

namespace lgpu {

// Source pointers per aggregation launch. The first launch folds shares[0..kAggPtrs); every further one starts from `out` and adds the
// next kAggPtrs - 1 shares, so K shares take 1 + ceil(max(0, K - kAggPtrs) / (kAggPtrs - 1)) launches per 65535 polynomials.
constexpr int kAggPtrs = 32;
struct AggParams {
    const u64* src[kAggPtrs];
    u64* out;
    u64 q[kMaxRows];           // modulus of every row of a block
    size_t poly_words;         // words per block: rows * N
    unsigned z0;               // index of the first block of this launch
    int k, n;
};

// out = (((src0 + src1) mod' q) + src2) mod' q ..., mod' = CRed (one conditional subtract) on the wrapping 64-bit sum: ring.Add applied
// as the reference's left fold. VEC: every pointer is 16-byte aligned, two words per thread through 128-bit accesses.
template <bool VEC>
__global__ void __launch_bounds__(256) mp_aggregate_kernel(const __grid_constant__ AggParams p) {
    constexpr int W = VEC ? 2 : 1;
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) * W;
    if (i >= p.n) return;
    const u64 q = p.q[blockIdx.y];
    const size_t off = (size_t)(p.z0 + blockIdx.z) * p.poly_words + (size_t)blockIdx.y * p.n + i;
    if (VEC) {
        ulonglong2 a = *reinterpret_cast<const ulonglong2*>(p.src[0] + off);
#pragma unroll
        for (int k = 1; k < kAggPtrs; k++) {
            if (k >= p.k) break;
            const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(p.src[k] + off);
            a.x = cred(a.x + b.x, q);
            a.y = cred(a.y + b.y, q);
        }
        *reinterpret_cast<ulonglong2*>(p.out + off) = a;
    } else {
        u64 a = p.src[0][off];
#pragma unroll
        for (int k = 1; k < kAggPtrs; k++) {
            if (k >= p.k) break;
            a = cred(a + p.src[k][off], q);
        }
        p.out[off] = a;
    }
}

int mp_aggregate(const Ctx* c, int levelQ, int levelP, const u64* const* shares, int n_shares, u64* out, size_t n_polys, cudaStream_t st) {
    const int nq = levelQ + 1, np = levelP + 1, rows = nq + np;
    if (n_shares == 1 && out == shares[0]) return 0;
    AggParams p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < nq; r++) p.q[r] = c->Q[r];
    for (int r = 0; r < np; r++) p.q[nq + r] = c->P[r];
    p.poly_words = (size_t)rows * c->N;
    p.out = out;
    p.n = c->N;
    bool vec = AL(out);
    for (int k = 0; k < n_shares; k++) vec = vec && AL(shares[k]);
    const int W = vec ? 2 : 1;
    for (size_t z0 = 0; z0 < n_polys; z0 += 65535) {
        const unsigned nz = (unsigned)(n_polys - z0 < 65535 ? n_polys - z0 : 65535);
        p.z0 = (unsigned)z0;
        for (int next = 0; next < n_shares;) {
            int k = 0;
            if (next > 0) p.src[k++] = out;                  // the fold so far
            while (k < kAggPtrs && next < n_shares) p.src[k++] = shares[next++];
            p.k = k;
            const dim3 grid((c->N / W + 255) / 256, rows, nz);
            count_launch(1);
            if (vec) mp_aggregate_kernel<true><<<grid, 256, 0, st>>>(p);
            else mp_aggregate_kernel<false><<<grid, 256, 0, st>>>(p);
            LGPU_CUDA_OK(cudaGetLastError());
        }
    }
    return 0;
}

// KeySwitchProtocol.GenShare, NTT domain: on entry share = NTT(e); share = CRed(MRedLazy(c1, CRed(s_in + q - s_out)) + share)
struct CksParams {
    const LimbConst* limbs;
    const u64* c1; size_t c1_bs;
    const u64* s_in; const u64* s_out;
    u64* share; size_t share_bs;
    int n;
};
__global__ void __launch_bounds__(256) mp_cks_share_kernel(CksParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int r = blockIdx.y, b = blockIdx.z;
    const LimbConst& L = p.limbs[r];
    const size_t w = (size_t)r * p.n + i;
    const u64 d = cred(p.s_in[w] + L.q - p.s_out[w], L.q);
    u64* o = p.share + (size_t)b * p.share_bs + w;
    *o = cred(mred_lazy(p.c1[(size_t)b * p.c1_bs + w], d, L.q, L.qinv) + *o, L.q);
}

// PublicKeySwitchProtocol.GenShare, NTT domain: on entry share0 = EncryptZero(pk)[0], e = NTT(e_flood);
// share0 = CRed(CRed(share0 + MRed(c1, s)) + e)
struct PcksParams {
    const LimbConst* limbs;
    const u64* c1; size_t c1_bs;
    const u64* s;
    const u64* e; size_t e_bs;
    u64* share0; size_t share_bs;
    int n;
};
__global__ void __launch_bounds__(256) mp_pcks_share_kernel(PcksParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int r = blockIdx.y, b = blockIdx.z;
    const LimbConst& L = p.limbs[r];
    const size_t w = (size_t)r * p.n + i;
    u64* o = p.share0 + (size_t)b * p.share_bs + w;
    const u64 t = cred(*o + mred(p.c1[(size_t)b * p.c1_bs + w], p.s[w], L.q, L.qinv), L.q);
    *o = cred(t + p.e[(size_t)b * p.e_bs + w], L.q);
}

int mp_key_switch_share(const Ctx* c, int level, const u64* c1, size_t stride, const u64* s_in, const u64* s_out, const long long* e, u64* share,
                        int batch, cudaStream_t st) {
    const size_t N = c->N, nq = (size_t)level + 1;
    const RowMap rq = rows_range(0, 0, (int)nq);
    const Span sh{share, N, nq * N};
    if (small_to_rns(c, rq, e, N, sh, batch, st)) return -1;
    if (launch_ntt(c, rq, CSpan{share, N, nq * N}, sh, batch, NTT_CANONICAL, st)) return -1;
    CksParams p;
    p.limbs = c->d_limbs; p.c1 = c1; p.c1_bs = stride; p.s_in = s_in; p.s_out = s_out; p.share = share; p.share_bs = nq * N; p.n = c->N;
    count_launch(1);
    mp_cks_share_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, batch), 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int mp_public_key_switch_share(const Ctx* c, int level, const u64* c1, size_t stride, const u64* s, const u64* pk, const long long* u,
                               const long long* e0, const long long* e1, const long long* e_flood, u64* share, int batch, cudaStream_t st) {
    const size_t N = c->N, nq = (size_t)level + 1;
    if (encrypt_zero_pk(c, level, pk, u, e0, e1, share, true, false, batch, st)) return -1;
    const RowMap rq = rows_range(0, 0, (int)nq);
    Scratch buf;
    if (buf.alloc((size_t)batch * nq * N, st)) return -1;
    const Span E{buf.p, N, nq * N};
    if (small_to_rns(c, rq, e_flood, N, E, batch, st)) return -1;
    if (launch_ntt(c, rq, CSpan{buf.p, N, nq * N}, E, batch, NTT_CANONICAL, st)) return -1;
    PcksParams p;
    p.limbs = c->d_limbs; p.c1 = c1; p.c1_bs = stride; p.s = s; p.e = buf.p; p.e_bs = nq * N; p.share0 = share; p.share_bs = 2 * nq * N; p.n = c->N;
    count_launch(1);
    mp_pcks_share_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, batch), 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// RelinearizationKeyGenProtocol.GenShareRoundTwo, one gadget entry per blockIdx.z: on entry share = NTT(e2);
// share = CRed(CRed(MRedLazy(r0, s) + share) + MRed(CRed(u + q - s), r1)) over the QP rows
struct RkgTwoParams {
    const LimbConst* limbs;
    const u64* r1; size_t r1_es;     // round-one share: component 0 at r1, component 1 at r1 + rows * N
    const u64* u; const u64* s;
    u64* share; size_t share_es;
    int n, rows;
};
__global__ void __launch_bounds__(256) mp_rkg_round_two_kernel(RkgTwoParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int r = blockIdx.y;
    const LimbConst& L = p.limbs[r];
    const size_t w = (size_t)r * p.n + i;
    const u64* r0 = p.r1 + (size_t)blockIdx.z * p.r1_es;
    const u64 s = p.s[w];
    u64* o = p.share + (size_t)blockIdx.z * p.share_es + w;
    const u64 t = cred(mred_lazy(r0[w], s, L.q, L.qinv) + *o, L.q);
    const u64 d = cred(p.u[w] + L.q - s, L.q);
    *o = cred(t + mred(d, r0[(size_t)p.rows * p.n + w], L.q, L.qinv), L.q);
}

// Thresholdizer.GenShamirSecretShare for a list of recipients (multiparty/threshold.go:102-104 -> ringqp.Ring.EvalPolyScalar,
// ring/ringqp/operations.go:92-102 and ring/operations.go:269-275): share_k = EvalPolyScalar(poly, points[k]) on every Q and P row.
// Horner's rule from acc = poly[t-1]: acc = CRed(MRed(acc, MForm(x)) + poly[i-1]), the wrapping 64-bit sum of the reference's
// MulScalar then Add, with MForm the Barrett form of the unreduced point. A thread keeps the accumulators of kShamirPts points in
// registers and reads each coefficient word once for them, so n points cost ceil(n / kShamirPts) t + n share-sizes of traffic instead
// of the 2 + 5 (t - 1) per point of the MulScalar / Add chain. blockIdx.z is the chunk of points.
constexpr int kShamirPts = 8;
struct ShamirParams {
    const u64* poly;             // [t][rows][N]
    u64* shares;                 // [n_points][rows][N]
    const u64* points;           // [n_points], device
    const LimbConst* limbs;
    unsigned char limb[kMaxRows];   // global limb of every row
    size_t poly_words;           // rows * N: the stride of a coefficient and of a share
    int t, n_points, n;
};

template <bool VEC>
__global__ void __launch_bounds__(256) mp_shamir_share_kernel(const __grid_constant__ ShamirParams p) {
    constexpr int W = VEC ? 2 : 1;
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) * W;
    if (i >= p.n) return;
    const LimbConst& L = p.limbs[p.limb[blockIdx.y]];
    const u64 q = L.q, qinv = L.qinv;
    const int k0 = blockIdx.z * kShamirPts;
    u64 x[kShamirPts];
#pragma unroll
    for (int k = 0; k < kShamirPts; k++)     // a chunk's tail repeats its last point; those results are not stored
        x[k] = mform(p.points[min(k0 + k, p.n_points - 1)], q, L.bred_hi, L.bred_lo);
    const size_t off = (size_t)blockIdx.y * p.n + i;
    const u64* c = p.poly + (size_t)(p.t - 1) * p.poly_words + off;
    u64 a[W], acc[kShamirPts][W];
    if (VEC) { const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(c); a[0] = v.x; a[W - 1] = v.y; }
    else a[0] = *c;
#pragma unroll
    for (int k = 0; k < kShamirPts; k++)
#pragma unroll
        for (int w = 0; w < W; w++) acc[k][w] = a[w];
    for (int j = p.t - 1; j > 0; j--) {
        c -= p.poly_words;
        if (VEC) { const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(c); a[0] = v.x; a[W - 1] = v.y; }
        else a[0] = *c;
#pragma unroll
        for (int k = 0; k < kShamirPts; k++)
#pragma unroll
            for (int w = 0; w < W; w++) acc[k][w] = cred(mred(acc[k][w], x[k], q, qinv) + a[w], q);
    }
    u64* o = p.shares + (size_t)k0 * p.poly_words + off;
#pragma unroll
    for (int k = 0; k < kShamirPts; k++) {
        if (k0 + k >= p.n_points) break;
        if (VEC) *reinterpret_cast<ulonglong2*>(o) = make_ulonglong2(acc[k][0], acc[k][W - 1]);
        else *o = acc[k][0];
        o += p.poly_words;
    }
}

int mp_shamir_share(const Ctx* c, int levelQ, int levelP, const u64* poly, int t, const u64* points, int n_points, u64* shares, cudaStream_t st) {
    const int nq = levelQ + 1, np = levelP + 1;
    ShamirParams p;
    memset(&p, 0, sizeof(p));
    for (int r = 0; r < nq; r++) p.limb[r] = (unsigned char)r;
    for (int r = 0; r < np; r++) p.limb[nq + r] = (unsigned char)(c->nQ + r);
    Scratch pts;
    if (pts.alloc((size_t)n_points, st)) return -1;
    LGPU_CUDA_OK(cudaMemcpyAsync(pts.p, points, (size_t)n_points * sizeof(u64), cudaMemcpyHostToDevice, st));
    p.poly = poly; p.shares = shares; p.points = pts.p; p.limbs = c->d_limbs;
    p.poly_words = (size_t)(nq + np) * c->N;
    p.t = t; p.n_points = n_points; p.n = c->N;
    const bool vec = AL(poly) && AL(shares);
    const int W = vec ? 2 : 1;
    const dim3 grid((c->N / W + 255) / 256, nq + np, (n_points + kShamirPts - 1) / kShamirPts);
    count_launch(1);
    if (vec) mp_shamir_share_kernel<true><<<grid, 256, 0, st>>>(p);
    else mp_shamir_share_kernel<false><<<grid, 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// the gadget layout of a key-generation share at the context's maximum levels
static int check_share_layout(const Ctx& c, const lgpu_gadget_ct* g, GadgetCt& out) {
    if (to_gadget_ct(g, out, "null share")) return -1;
    if (out.levelQ != c.nQ - 1 || out.levelP != c.nP - 1) { set_error("key-generation shares are at the maximum levels"); return -1; }
    const int nd = out.levelP >= 0 ? base_rns_decomposition_vector_size(out.levelQ, out.levelP) : out.levelQ + 1;
    if (out.ndigits != nd) { set_error("share: n_digits != BaseRNSDecompositionVectorSize(levelQ, levelP)"); return -1; }
    if (out.npw2max < 1 || out.npw2max > 64) { set_error("share: n_pw2_max out of [1, 64]"); return -1; }
    if (out.pw2 < 0 || out.pw2 > 62) { set_error("share: BaseTwoDecomposition out of [0, 62]"); return -1; }
    for (int i = 0; out.pw2_sizes && i < nd; i++)
        if (out.pw2_sizes[i] < 1 || out.pw2_sizes[i] > out.npw2max) { set_error("share: pw2_sizes[i] out of [1, n_pw2_max]"); return -1; }
    return 0;
}

}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_mp_aggregate(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* const* shares, int n_shares, uint64_t* out, size_t n_polys,
                      void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(level_q >= 0 && level_q < c.nQ && level_p >= -1 && level_p < c.nP, "level out of range");
    REQUIRE(n_shares >= 1 && n_shares <= 65535, "n_shares out of [1, 65535]");
    REQUIRE(n_polys >= 1, "n_polys must be at least 1");
    REQUIRE(shares && out, "null argument");
    const size_t bytes = n_polys * (size_t)(level_q + 1 + level_p + 1) * c.N * sizeof(u64);
    for (int k = 0; k < n_shares; k++) {
        REQUIRE(shares[k], "null share");
        REQUIRE((k == 0 && shares[k] == out) || !overlaps(shares[k], bytes, out, bytes), "out overlaps a share (only out == shares[0] is allowed)");
    }
    REQUIRE_DEVICE(ctx);
    return mp_aggregate(&c, level_q, level_p, (const u64* const*)shares, n_shares, (u64*)out, n_polys, (cudaStream_t)stream);
}

int lgpu_mp_shamir_share(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* poly, int threshold, const uint64_t* points, int n_points,
                         uint64_t* shares, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(level_q >= 0 && level_q < c.nQ && level_p >= -1 && level_p < c.nP, "level out of range");
    REQUIRE(threshold >= 1 && threshold <= 65535, "threshold out of [1, 65535]");
    REQUIRE(n_points >= 1 && n_points <= 65535, "n_points out of [1, 65535]");
    REQUIRE(poly && points && shares, "null argument");
    const size_t bytes = (size_t)(level_q + 1 + level_p + 1) * c.N * sizeof(u64);
    REQUIRE(!overlaps(shares, (size_t)n_points * bytes, poly, (size_t)threshold * bytes), "shares overlap the Shamir polynomial");
    REQUIRE_DEVICE(ctx);
    return mp_shamir_share(&c, level_q, level_p, (const u64*)poly, threshold, (const u64*)points, n_points, (u64*)shares, (cudaStream_t)stream);
}

int lgpu_mp_key_switch_share(lgpu_ctx* ctx, int level, const uint64_t* c1, size_t stride, const uint64_t* sk_in, const uint64_t* sk_out,
                             const int64_t* e, uint64_t* share, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(c1 && sk_in && sk_out && e && share, "null argument");
    REQUIRE(stride >= (size_t)(level + 1) * c.N, "stride below (level + 1) * N");
    const size_t sbytes = (size_t)batch * (level + 1) * c.N * sizeof(u64), cbytes = ((size_t)(batch - 1) * stride + (size_t)(level + 1) * c.N) * sizeof(u64);
    REQUIRE(!overlaps(share, sbytes, c1, cbytes), "share overlaps the ciphertexts");
    REQUIRE_DEVICE(ctx);
    return mp_key_switch_share(&c, level, (const u64*)c1, stride, (const u64*)sk_in, (const u64*)sk_out, (const long long*)e, (u64*)share, batch,
                               (cudaStream_t)stream);
}

int lgpu_mp_public_key_switch_share(lgpu_ctx* ctx, int level, const uint64_t* c1, size_t stride, const uint64_t* sk, const uint64_t* pk,
                                    const int64_t* u, const int64_t* e0, const int64_t* e1, const int64_t* e_flood, uint64_t* share, int batch,
                                    void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(c1 && sk && pk && u && e0 && e1 && e_flood && share, "null argument");
    REQUIRE(stride >= (size_t)(level + 1) * c.N, "stride below (level + 1) * N");
    const size_t sbytes = (size_t)batch * 2 * (level + 1) * c.N * sizeof(u64), cbytes = ((size_t)(batch - 1) * stride + (size_t)(level + 1) * c.N) * sizeof(u64);
    REQUIRE(!overlaps(share, sbytes, c1, cbytes), "share overlaps the ciphertexts");
    REQUIRE_DEVICE(ctx);
    return mp_public_key_switch_share(&c, level, (const u64*)c1, stride, (const u64*)sk, (const u64*)pk, (const long long*)u, (const long long*)e0,
                                      (const long long*)e1, (const long long*)e_flood, (u64*)share, batch, (cudaStream_t)stream);
}

int lgpu_mp_evaluation_key_gen_share(lgpu_ctx* ctx, const uint64_t* sk_in, const uint64_t* sk_out, const uint64_t* gal_els, int n_keys,
                                     const uint64_t* crp, const int64_t* e, const lgpu_gadget_ct* share, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    GadgetCt g;
    if (check_share_layout(c, share, g)) return -1;
    REQUIRE(n_keys >= 1 && n_keys <= 65535, "n_keys out of [1, 65535]");
    REQUIRE(gal_els || n_keys == 1, "without Galois elements there is one key");
    REQUIRE(sk_in && (sk_out || gal_els) && crp && e, "null argument");
    for (int k = 0; gal_els && k < n_keys; k++)
        REQUIRE((gal_els[k] & 1) && gal_els[k] < (uint64_t)c.nthroot, "Galois elements are odd and below 2N");
    REQUIRE(c.ring_type == 0, "multiparty key generation is not supported on the ConjugateInvariant ring");
    REQUIRE_DEVICE(ctx);
    const size_t N = c.N, rows = (size_t)c.nQ + c.nP, entries = (size_t)g.ndigits * g.npw2max, key_words = entries * rows * N;
    // sk_out = AutomorphismNTT(sk_in, galEl^-1 mod 2N) on Q and P for a Galois key (keygen_gal.go:56-63)
    std::vector<GadgetEncCt> cts((size_t)n_keys);
    for (int k = 0; k < n_keys; k++)
        cts[k] = GadgetEncCt{(u64*)share->data + k * key_words, (const u64*)crp + k * key_words, nullptr, gal_els ? (const u64*)sk_in : (const u64*)sk_out,
                             gal_els ? gal_els[k] : 0, (const u64*)sk_in, 0};
    const GadgetEncLayout lay{g.levelQ, g.levelP, g.pw2, g.ndigits, g.npw2max, g.pw2_sizes, rows * N, rows * N, true};
    return gadget_encrypt(&c, lay, cts.data(), n_keys, (const long long*)e, nullptr, (cudaStream_t)stream);
}

int lgpu_mp_rkg_share_round_one(lgpu_ctx* ctx, const uint64_t* sk, const int64_t* u_small, const uint64_t* crp, const int64_t* e0,
                                const int64_t* e1, uint64_t* eph_sk_out, const lgpu_gadget_ct* share, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    GadgetCt g;
    if (check_share_layout(c, share, g)) return -1;
    REQUIRE(sk && u_small && crp && e0 && e1 && eph_sk_out, "null argument");
    REQUIRE(c.ring_type == 0, "multiparty key generation is not supported on the ConjugateInvariant ring");
    REQUIRE_DEVICE(ctx);
    const size_t N = c.N, rows = (size_t)c.nQ + c.nP;
    const int entries = g.ndigits * g.npw2max;
    cudaStream_t st = (cudaStream_t)stream;
    const RowMap rqp = rows_range(0, 0, (int)rows);      // at the maximum levels the P rows' limb indices are nQ + j
    // ephemeral u: ternary -> QP -> NTT -> MForm (keygen_relin.go:116-121)
    u64* eph = (u64*)eph_sk_out;
    if (small_to_rns(&c, rqp, (const long long*)u_small, N, Span{eph, N, 0}, 1, st)) return -1;
    if (launch_ntt(&c, rqp, CSpan{eph, N, 0}, Span{eph, N, 0}, 1, NTT_CANONICAL, st)) return -1;
    if (launch_vecop(&c, rqp, LGPU_OP_MFORM, CSpan{eph, N, 0}, CSpan{nullptr, 0, 0}, Span{eph, N, 0}, 1, nullptr, nullptr, 0, 0, c.N, st)) return -1;
    // component 0: e0 + P 2^(w j) s - u crp, plain form
    u64* data = (u64*)share->data;
    const size_t es = 2 * rows * N;
    const GadgetEncLayout lay{g.levelQ, g.levelP, g.pw2, g.ndigits, g.npw2max, g.pw2_sizes, es, rows * N, false};
    const GadgetEncCt ct{data, (const u64*)crp, nullptr, eph, 0, (const u64*)sk, 0};
    if (gadget_encrypt(&c, lay, &ct, 1, (const long long*)e0, nullptr, st)) return -1;
    // component 1: NTT(e1) + s crp (MulCoeffsMontgomeryThenAdd)
    const Span c1{data + rows * N, N, es};
    if (small_to_rns(&c, rqp, (const long long*)e1, N, c1, entries, st)) return -1;
    if (launch_ntt(&c, rqp, CSpan{c1.p, N, es}, c1, entries, NTT_CANONICAL, st)) return -1;
    return launch_vecop(&c, rqp, LGPU_OP_MULCOEFFSMONTGOMERYTHENADD, CSpan{(const u64*)crp, N, rows * N}, CSpan{(const u64*)sk, N, 0}, c1, entries,
                        nullptr, nullptr, 0, 0, c.N, st);
}

int lgpu_mp_rkg_share_round_two(lgpu_ctx* ctx, const uint64_t* eph_sk, const uint64_t* sk, const lgpu_gadget_ct* round1, const int64_t* e2,
                                const lgpu_gadget_ct* share, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    GadgetCt g1, g2;
    if (check_share_layout(c, round1, g1) || check_share_layout(c, share, g2)) return -1;
    REQUIRE(g1.ndigits == g2.ndigits && g1.npw2max == g2.npw2max && g1.pw2 == g2.pw2, "round-one and round-two shares differ in their gadget layout");
    REQUIRE(eph_sk && sk && e2, "null argument");
    REQUIRE(c.ring_type == 0, "multiparty key generation is not supported on the ConjugateInvariant ring");
    REQUIRE_DEVICE(ctx);
    const size_t N = c.N, rows = (size_t)c.nQ + c.nP;
    const int entries = g2.ndigits * g2.npw2max;
    cudaStream_t st = (cudaStream_t)stream;
    const RowMap rqp = rows_range(0, 0, (int)rows);
    u64* out = (u64*)share->data;
    const Span sh{out, N, rows * N};
    if (small_to_rns(&c, rqp, (const long long*)e2, N, sh, entries, st)) return -1;
    if (launch_ntt(&c, rqp, CSpan{out, N, rows * N}, sh, entries, NTT_CANONICAL, st)) return -1;
    RkgTwoParams p;
    p.limbs = c.d_limbs; p.r1 = (const u64*)round1->data; p.r1_es = 2 * rows * N; p.u = (const u64*)eph_sk; p.s = (const u64*)sk;
    p.share = out; p.share_es = rows * N; p.n = c.N; p.rows = (int)rows;
    count_launch(1);
    mp_rkg_round_two_kernel<<<dim3((c.N + 255) / 256, (unsigned)rows, entries), 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

}  // extern "C"

// encrypt.cu -- the encryptor / key-generator inner loops and the samplers on the device (SURVEY 8(f) rank 3).
//
// Deterministic part (bit-exact with the reference given the same sampled polynomials; restated for tests in oracle/encryptor.py):
//   Encryptor.encryptZeroPk (Element[ring.Poly])          core/rlwe/encryptor.go:204-299
//   Encryptor.encryptZeroPkNoP                            :301-341
//   Encryptor.encryptZeroSkFromC1QP / encryptZeroSk       :346-430
//   KeyGenerator.genEvaluationKey                         core/rlwe/keygenerator.go:287-330
//   AddPolyTimesGadgetVectorToGadgetCiphertext            core/rlwe/gadgetciphertext.go:171-241
//   rgsw.Encryptor.Encrypt / EncryptZero                  core/rgsw/encryptor.go:25-121 (gadget_encrypt, one routine for every
//                                                         batched gadget encryption; its C ABI is keygen.cu)
//   ringqp.Ring.ExtendBasisSmallNormAndCenter             ring/ringqp/operations.go:325-351 (folded into small_to_rns)
// Samplers (ring/sampler_uniform.go, sampler_ternary.go, sampler_gaussian.go): same DISTRIBUTIONS, own random streams -- the
// reference reads a blake2b XOF sequentially (sampling/prng.go), which has no parallel form; here every coefficient owns a
// Philox4x32-10 counter (sampler kind, seed, stream, polynomial, coefficient, attempt), so a batch of polynomials is sampled in
// one launch and the result does not depend on the launch geometry. The layout is restated bit for bit in oracle/philox.py.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>
#include "../../include/lattigo_b200.h"
#include "capi_common.h"
#include "composite.h"
#include "modarith.cuh"

namespace lgpu {

// ---------------------------------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11): counter-based, 128-bit counter, 64-bit key
// ---------------------------------------------------------------------------------------------------------------------
struct Ph4 { unsigned x, y, z, w; };
__device__ __forceinline__ Ph4 philox4x32_10(Ph4 c, unsigned k0, unsigned k1) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = Ph4{hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0};
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c;
}
struct SampleKey { unsigned k0, k1, stream; };
// Which sampler drew a block: bits 30..31 of the counter's polynomial word. The polynomial index itself stays below 2^23, so two
// samplers of different kinds never share a Philox input, whatever the seed and stream id.
enum SampleKind : unsigned { kKindUniform = 0, kKindTernaryP = 1, kKindTernaryH = 2, kKindGaussian = 3 };
constexpr unsigned kKindShift = 30;
static_assert(65535ull * kMaxRows + kMaxRows <= (1ull << kKindShift), "the polynomial index reaches the sampler-kind field");
// The multiparty masks (sample_mask) are uniform draws whose polynomial word also carries kMaskDomain. Every other draw's polynomial
// index stays below it, so the mask streams share no Philox input with any other stream, and the four kinds keep their streams.
constexpr unsigned kMaskDomain = 1u << 29;
static_assert(65535ull * kMaxRows + kMaxRows <= kMaskDomain, "the polynomial index reaches the mask domain bit");
// The mpckks masks (sample_big_mask) add kBigMaskDomain, so they share no Philox input with the mpbgv masks either.
constexpr unsigned kBigMaskDomain = 1u << 28;
static_assert(65535ull * kMaxRows + kMaxRows <= kBigMaskDomain, "the polynomial index reaches the big-mask domain bit");
// counter words: (coefficient, polynomial | kind << 30, stream_id mod 2^32, attempt); key: make_key(seed, stream_id)
__device__ __forceinline__ Ph4 draw(const SampleKey& k, SampleKind kind, unsigned poly, unsigned coeff, unsigned attempt) {
    return philox4x32_10(Ph4{coeff, poly | (unsigned)kind << kKindShift, k.stream, attempt}, k.k0, k.k1);
}

// uniform in [0, q) per row: masked 64-bit words, rejected until below q (ring/sampler_uniform.go:48-100). The polynomial index is
// batch * kMaxRows + global limb index (P limbs are nQ + j), so the Q and P rows of one ringqp.Poly drawn on one stream id differ.
__host__ __device__ inline SampleKey make_key(u64 seed, u64 stream) {
    SampleKey k;
    k.k0 = (unsigned)seed; k.k1 = (unsigned)(seed >> 32) ^ (unsigned)(stream >> 32) * 0x85EBCA6Bu; k.stream = (unsigned)stream;
    return k;
}
// per_stream > 0: batch element b is element b % per_stream of stream id stream0 + b / per_stream, so one launch draws what one call
// per stream id would (the batched key generators); per_stream = 0: every element on `key`
struct StreamSplit { u64 seed, stream0; int per_stream; };
__device__ __forceinline__ void split_stream(const StreamSplit& s, SampleKey& key, unsigned& b) {
    if (s.per_stream > 0) { key = make_key(s.seed, s.stream0 + b / (unsigned)s.per_stream); b %= (unsigned)s.per_stream; }
}
struct UniformParams {
    const LimbConst* limbs; RowMap rm;
    u64* out; size_t rs, bs;
    SampleKey key; int n;
    StreamSplit split;
};
__global__ void __launch_bounds__(256) sample_uniform_kernel(UniformParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int r = blockIdx.y, b = blockIdx.z;
    const u64 q = p.limbs[p.rm.limb[r]].q;
    const u64 mask = ~0ull >> __clzll((long long)(q - 1));
    SampleKey key = p.key;
    unsigned bb = (unsigned)b;
    split_stream(p.split, key, bb);
    const unsigned poly = bb * kMaxRows + (unsigned)p.rm.limb[r];
    u64 v = 0;
    for (unsigned a = 0;; a++) {
        const Ph4 d = draw(key, kKindUniform, poly, (unsigned)i, a);
        v = (((u64)d.x << 32) | d.y) & mask;
        if (v < q) break;
        v = (((u64)d.z << 32) | d.w) & mask;
        if (v < q) break;
    }
    p.out[(size_t)b * p.bs + (size_t)p.rm.drow[r] * p.rs + i] = v;
}

// uniform in [0, m) per word, m >= 2: ring.UniformSampler over a one-modulus ring (the masks of mpbgv over ring T), with the uniform
// kernel's rejection; polynomial word = entry | kMaskDomain
__global__ void __launch_bounds__(256) sample_mask_kernel(u64* out, size_t bs, int n, u64 m, SampleKey key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u64 mask = ~0ull >> __clzll((long long)(m - 1));
    const unsigned poly = blockIdx.y | kMaskDomain;
    u64 v = 0;
    for (unsigned a = 0;; a++) {
        const Ph4 d = draw(key, kKindUniform, poly, (unsigned)i, a);
        v = (((u64)d.x << 32) | d.y) & mask;
        if (v < m) break;
        v = (((u64)d.z << 32) | d.w) & mask;
        if (v < m) break;
    }
    out[(size_t)blockIdx.y * bs + i] = v;
}

// bignum.RandInt(prng, 2^log_bound) mapped to [-2^(log_bound-1), 2^(log_bound-1)) (value >= 2^(log_bound-1) minus 2^log_bound), as W
// little-endian two's-complement words per value: attempt a of value i gives words 2a = (x:y) and 2a + 1 = (z:w), bits from log_bound up
// are the sign extension of bit log_bound - 1. The bound is a power of two, so no draw is rejected. Polynomial word = entry | kMaskDomain
// | kBigMaskDomain.
__global__ void __launch_bounds__(256) sample_big_mask_kernel(u64* out, size_t bs, int n, int W, int log_bound, SampleKey key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned poly = blockIdx.y | kMaskDomain | kBigMaskDomain;
    u64* o = out + (size_t)blockIdx.y * bs + (size_t)i * W;
    const int top = (log_bound - 1) >> 6;                      // word holding the sign bit
    u64 neg = 0;
    for (int a = 0; 2 * a <= top; a++) {
        const Ph4 d = draw(key, kKindUniform, poly, (unsigned)i, (unsigned)a);
        const u64 v[2] = {((u64)d.x << 32) | d.y, ((u64)d.z << 32) | d.w};
        for (int h = 0; h < 2 && 2 * a + h <= top; h++) {
            u64 x = v[h];
            if (2 * a + h == top) {
                const int b = (log_bound - 1) & 63;            // sign bit position in this word
                neg = (x >> b) & 1;
                const u64 low = b == 63 ? ~0ull : ((1ull << (b + 1)) - 1);
                x = neg ? (x | ~low) : (x & low);
            }
            o[2 * a + h] = x;
        }
    }
    for (int w = top + 1; w < W; w++) o[w] = neg ? ~0ull : 0;
}

// ternary with P(+-1) = prob / 2 each (ring.Ternary{P}, ring/sampler_ternary.go:136-201). u takes 53 bits, so it is exact and
// below 1: P(non-zero) = ceil(prob * 2^53) / 2^53, and prob = 1 leaves no zero.
__global__ void __launch_bounds__(256) sample_ternary_p_kernel(long long* out, int n, double prob, SampleKey key) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Ph4 d = draw(key, kKindTernaryP, blockIdx.y, (unsigned)i, 0);
    const double u = (double)(((u64)d.x << 21) | (d.y >> 11)) * (1.0 / 9007199254740992.0);   // [0, 1)
    out[(size_t)blockIdx.y * n + i] = u < prob ? ((d.z & 1u) ? 1 : -1) : 0;
}
// ternary with exactly h non-zero coefficients, uniform positions and signs (ring.Ternary{H}, :203-260): one CTA per polynomial,
// positions drawn by rejection against a bitmap in shared memory. Block a gives the candidates (d.x, sign d.y) then (d.z, sign d.w);
// the polynomial's coefficients are the first h distinct positions of that sequence.
__global__ void __launch_bounds__(256) sample_ternary_h_kernel(long long* out, int n, int h, SampleKey key) {
    extern __shared__ unsigned bitmap[];
    long long* o = out + (size_t)blockIdx.x * n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) o[i] = 0;
    for (int i = threadIdx.x; i < (n + 31) / 32; i += blockDim.x) bitmap[i] = 0;
    __syncthreads();
    if (threadIdx.x != 0) return;
    int placed = 0;
    for (unsigned a = 0; placed < h; a++) {
        const Ph4 d = draw(key, kKindTernaryH, blockIdx.x, a, 0);
        const unsigned cand[2] = {d.x & (unsigned)(n - 1), d.z & (unsigned)(n - 1)};
        const unsigned sgn[2] = {d.y & 1u, d.w & 1u};
        for (int t = 0; t < 2 && placed < h; t++) {
            const unsigned pos = cand[t];
            if (bitmap[pos >> 5] & (1u << (pos & 31))) continue;
            bitmap[pos >> 5] |= 1u << (pos & 31);
            o[pos] = sgn[t] ? 1 : -1;
            placed++;
        }
    }
}
// truncated discrete Gaussian: round(|N(0,1)| * sigma) with a random sign, redrawn while |N(0,1)| * sigma > bound
// (ring/sampler_gaussian.go:160-182); the normal deviate comes from Box-Muller on two 53-bit uniforms
__global__ void __launch_bounds__(256) sample_gaussian_kernel(long long* out, int n, double sigma, double bound, SampleKey key, StreamSplit split) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned poly = blockIdx.y;
    split_stream(split, key, poly);
    long long v = 0;
    for (unsigned a = 0;; a++) {
        const Ph4 d = draw(key, kKindGaussian, poly, (unsigned)i, a);
        const double u1 = ((double)(((u64)d.x << 21) | (d.y >> 11)) + 1.0) * (1.0 / 9007199254740992.0);   // (0, 1]
        const double u2 = (double)(((u64)d.z << 21) | (d.w >> 11)) * (1.0 / 9007199254740992.0);            // [0, 1)
        const double z = sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
        const double m = fabs(z) * sigma;
        if (m <= bound) {
            v = (long long)(m + 0.5);
            if (d.w & 1u) v = -v;      // bit 0 of d.w is not part of u2
            break;
        }
    }
    out[(size_t)blockIdx.y * n + i] = v;
}

// signed small coefficients -> residues on the launch rows: Sampler.Read on the Q rows followed by ExtendBasisSmallNormAndCenter on
// the P rows leaves exactly v mod q_i / v mod p_j (|v| < q_0 / 2); the kernel's v mod q is exact for |v| < q
struct SmallParams {
    const LimbConst* limbs; RowMap rm;
    const long long* in; size_t in_bs;
    u64* out; size_t rs, bs;
    int n;
};
__global__ void __launch_bounds__(256) small_to_rns_kernel(SmallParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const int r = blockIdx.y, b = blockIdx.z;
    const u64 q = p.limbs[p.rm.limb[r]].q;
    const long long v = p.in[(size_t)b * p.in_bs + i];
    p.out[(size_t)b * p.bs + (size_t)p.rm.drow[r] * p.rs + i] = v < 0 ? q - (u64)(-v) : (u64)v;
}

// The epilogue of a batched gadget encryption (encryptZeroSkFromC1QP after its NTT, then AddPolyTimesGadgetVectorToGadgetCiphertext),
// one word per thread pair, every row of every entry of every ciphertext of a chunk in one launch:
//   c0 = MForm(NTT(e)) - c1 s_out   (+ f_j pt on the Q rows of digit i when the target is 0)
//   c1 += f_j pt                    (on the Q rows of digit i when the target is 1)
// with the word operations of the passes it replaces (LGPU_OP_MFORM, LGPU_OP_MULCOEFFSMONTGOMERYTHENSUB, CRed(c + MRed(pt, f))), so
// its words are theirs. c0 is computed from the c1 read before the add, as the reference encrypts zero before adding the plaintext.
struct GadgetEncDev {         // one ciphertext of the chunk (device copy of the host descriptors)
    u64* c0;                  // entry (i, j) at c0 + (i n_pw2_max + j) c0_es
    const u64* c1;            // entry at c1 + (.) c1_es: the uniform polynomial
    size_t c1_es;
    u64* c1_out;              // entry at c1_out + (.) c1_out_es; nullptr: component 1 is not written
    const u64* s;             // [nQ + nP][N] secret of the encryption
    const u64* pt;            // rows 0..levelQ, or nullptr
    int target;
};
struct GadgetEpiParams {
    const LimbConst* limbs;
    const GadgetEncDev* cts;  // the chunk's first ciphertext
    const u64* E;             // NTT(e) of unit u (ciphertext u / entries, entry u % entries) at E + u rows N, QP-stacked rows
    const u64* f;             // [nq][n_pw2_max]: P_levelP 2^(pw2 j) mod q_r (Montgomery form when mont)
    size_t c0_es, c1_out_es;
    int nq, rows, nQ, k, n, npw2, entries, mont;
    unsigned char npw2_of_digit[kMaxRows];
};
template <int VEC>
__global__ void __launch_bounds__(256) gadget_enc_epilogue_kernel(GadgetEpiParams p) {
    using V = typename std::conditional<VEC == 2, ulonglong2, u64>::type;
    const int u = blockIdx.z, r = blockIdx.y;
    const int b = u / p.entries, ent = u - b * p.entries;
    const int i = ent / p.npw2, j = ent - i * p.npw2;
    const GadgetEncDev d = p.cts[b];
    const int limb = r < p.nq ? r : p.nQ + (r - p.nq);
    const u64 q = p.limbs[limb].q, qinv = p.limbs[limb].qinv, bh = p.limbs[limb].bred_hi, bl = p.limbs[limb].bred_lo;
    const size_t row = (size_t)r * p.n;
    const V* E = reinterpret_cast<const V*>(p.E + (size_t)u * p.rows * p.n + row);
    const V* c1 = reinterpret_cast<const V*>(d.c1 + ent * d.c1_es + row);
    const V* s = reinterpret_cast<const V*>(d.s + (size_t)limb * p.n);
    V* c0 = reinterpret_cast<V*>(d.c0 + ent * p.c0_es + row);
    const bool add = d.pt && r < p.nq && r / p.k == i && j < p.npw2_of_digit[i];
    const u64 f = add ? p.f[r * p.npw2 + j] : 0;
    const V* pt = add ? reinterpret_cast<const V*>(d.pt + row) : nullptr;
    const bool add0 = add && d.target == 0, add1 = add && d.target == 1;
    V* c1o = d.c1_out ? reinterpret_cast<V*>(d.c1_out + ent * p.c1_out_es + row) : nullptr;
    if (c1o && (const void*)c1o == (const void*)c1 && !add1) c1o = nullptr;      // component 1 unchanged in place
    auto word = [&](u64 e, u64 a, u64 sk, u64 m, u64& o0, u64& o1) {
        if (p.mont) e = mform(e, q, bh, bl);
        o0 = cred(e + (q - mred(a, sk, q, qinv)), q);
        o1 = a;
        if (add) {
            const u64 t = mred(m, f, q, qinv);
            if (add0) o0 = cred(o0 + t, q);
            else o1 = cred(a + t, q);
        }
    };
    const int nv = p.n / VEC;
    for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nv; w += gridDim.x * blockDim.x) {
        if constexpr (VEC == 2) {
            const ulonglong2 e = E[w], a = c1[w], sk = s[w], m = pt ? pt[w] : make_ulonglong2(0, 0);
            ulonglong2 o0, o1;
            word(e.x, a.x, sk.x, m.x, o0.x, o1.x);
            word(e.y, a.y, sk.y, m.y, o0.y, o1.y);
            c0[w] = o0;
            if (c1o) c1o[w] = o1;
        } else {
            u64 o0, o1;
            word(E[w], c1[w], s[w], pt ? pt[w] : 0, o0, o1);
            c0[w] = o0;
            if (c1o) c1o[w] = o1;
        }
    }
}

int sample_mask(u64 m, int n, u64 seed, u64 stream_id, u64* out, size_t bs, int batch, cudaStream_t st) {
    count_launch(1);
    sample_mask_kernel<<<dim3((n + 255) / 256, batch), 256, 0, st>>>(out, bs, n, m, make_key(seed, stream_id));
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int sample_big_mask(int n, int W, int log_bound, u64 seed, u64 stream_id, u64* out, size_t bs, int batch, cudaStream_t st) {
    count_launch(1);
    sample_big_mask_kernel<<<dim3((n + 255) / 256, batch), 256, 0, st>>>(out, bs, n, W, log_bound, make_key(seed, stream_id));
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int small_to_rns(const Ctx* c, const RowMap& rm, const long long* in, size_t in_bs, Span out, int batch, cudaStream_t st) {
    SmallParams p;
    p.limbs = c->d_limbs; p.rm = rm; p.in = in; p.in_bs = in_bs; p.out = out.p; p.rs = out.row_stride; p.bs = out.batch_stride; p.n = c->N;
    count_launch(1);
    small_to_rns_kernel<<<dim3((c->N + 255) / 256, rm.nrows, batch), 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}
static RowMap one_row(int limb) { RowMap r; r.nrows = 1; r.limb[0] = (unsigned char)limb; r.drow[0] = 0; return r; }

// encryptZeroSkFromC1QP (:404-430). sk: rows of the secret key at the context's maximum levels ([nQ + nP][N], NTT + Montgomery).
// c1 / c0: QP-stacked blocks ([levelQ+1 + levelP+1][N]) with the given batch strides; c1 is only rewritten when !is_ntt.
int encrypt_zero_sk(const Ctx* c, int levelQ, int levelP, const u64* sk, u64* c1, size_t c1_bs, const long long* e, u64* c0, size_t c0_bs,
                    bool is_ntt, bool is_mont, int batch, cudaStream_t st) {
    if (levelQ < 0 || levelQ >= c->nQ || levelP < -1 || levelP >= c->nP) { set_error("level out of range"); return -1; }
    const size_t N = c->N;
    const int nq = levelQ + 1, np = levelP + 1;
    const RowMap rqp = rows_qp(c, nq, np);
    Span s0{c0, N, c0_bs};
    if (small_to_rns(c, rqp, e, N, s0, batch, st)) return -1;
    if (launch_ntt(c, rqp, CSpan{c0, N, c0_bs}, s0, batch, NTT_CANONICAL, st)) return -1;
    if (is_mont && launch_vecop(c, rqp, LGPU_OP_MFORM, CSpan{c0, N, c0_bs}, CSpan{nullptr, 0, 0}, s0, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
    // c0 -= c1 * sk: Q rows, then P rows (the key's P rows start at row nQ)
    if (launch_vecop(c, rows_range(0, 0, nq), LGPU_OP_MULCOEFFSMONTGOMERYTHENSUB, CSpan{c1, N, c1_bs}, CSpan{sk, N, 0}, s0, batch, nullptr, nullptr, 0, 0,
                     c->N, st)) return -1;
    if (np > 0 && launch_vecop(c, rows_range(c->nQ, 0, np), LGPU_OP_MULCOEFFSMONTGOMERYTHENSUB, CSpan{c1 + (size_t)nq * N, N, c1_bs},
                               CSpan{sk + (size_t)c->nQ * N, N, 0}, Span{c0 + (size_t)nq * N, N, c0_bs}, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
    if (!is_ntt) {
        if (launch_intt(c, rqp, CSpan{c0, N, c0_bs}, s0, batch, NTT_CANONICAL, st)) return -1;
        if (launch_intt(c, rqp, CSpan{c1, N, c1_bs}, Span{c1, N, c1_bs}, batch, NTT_CANONICAL, st)) return -1;
    }
    return 0;
}

// encryptZeroPk for an Element[ring.Poly] (:204-299; levelP = 0 there) and encryptZeroPkNoP (:301-341) when the context has no P.
// pk: [2][nQ + nP][N] (rlwe.PublicKey.Value at the maximum levels); u, e0, e1: [batch][N] signed; ct_out: [batch][2][levelQ+1][N].
int encrypt_zero_pk(const Ctx* c, int levelQ, const u64* pk, const long long* u, const long long* e0, const long long* e1, u64* ct_out,
                    bool is_ntt, bool is_mont, int batch, cudaStream_t st) {
    if (levelQ < 0 || levelQ >= c->nQ) { set_error("level out of range"); return -1; }
    const size_t N = c->N;
    const int nq = levelQ + 1;
    const size_t key_rows = (size_t)c->nQ + c->nP, ct_bs = (size_t)2 * nq * N;
    const RowMap rq = rows_range(0, 0, nq);
    const long long* es[2] = {e0, e1};
    if (c->nP == 0) {
        if (is_mont) { set_error("encryptZeroPkNoP has no Montgomery-form output"); return -1; }
        Scratch buf;
        if (buf.alloc((size_t)2 * batch * nq * N, st)) return -1;
        u64* U = buf.p; u64* E = buf.p + (size_t)batch * nq * N;
        if (small_to_rns(c, rq, u, N, Span{U, N, nq * N}, batch, st)) return -1;
        if (launch_ntt(c, rq, CSpan{U, N, nq * N}, Span{U, N, nq * N}, batch, NTT_CANONICAL, st)) return -1;
        for (int k = 0; k < 2; k++) {
            Span o{ct_out + (size_t)k * nq * N, N, ct_bs};
            if (launch_vecop(c, rq, LGPU_OP_MULCOEFFSMONTGOMERY, CSpan{U, N, nq * N}, CSpan{pk + (size_t)k * key_rows * N, N, 0}, o, batch, nullptr, nullptr, 0, 0,
                             c->N, st)) return -1;
            if (small_to_rns(c, rq, es[k], N, Span{E, N, nq * N}, batch, st)) return -1;
            if (is_ntt) { if (launch_ntt(c, rq, CSpan{E, N, nq * N}, Span{E, N, nq * N}, batch, NTT_CANONICAL, st)) return -1; }
            else if (launch_intt(c, rq, CSpan{o.p, N, ct_bs}, o, batch, NTT_CANONICAL, st)) return -1;
            if (launch_vecop(c, rq, LGPU_OP_ADD, CSpan{o.p, N, ct_bs}, CSpan{E, N, nq * N}, o, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
        }
        return 0;
    }
    const int levelP = 0, np = 1;
    const RowMap rqp = rows_qp(c, nq, np);
    const size_t qp = (size_t)(nq + np) * N;
    Scratch buf;
    if (buf.alloc((size_t)3 * batch * qp, st)) return -1;
    u64* U = buf.p; u64* C = U + (size_t)batch * qp; u64* E = C + (size_t)batch * qp;
    if (small_to_rns(c, rqp, u, N, Span{U, N, qp}, batch, st)) return -1;
    if (launch_ntt(c, rqp, CSpan{U, N, qp}, Span{U, N, qp}, batch, NTT_CANONICAL, st)) return -1;
    for (int k = 0; k < 2; k++) {
        const u64* pkk = pk + (size_t)k * key_rows * N;
        if (launch_vecop(c, rq, LGPU_OP_MULCOEFFSMONTGOMERY, CSpan{U, N, qp}, CSpan{pkk, N, 0}, Span{C, N, qp}, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
        if (launch_vecop(c, one_row(c->nQ), LGPU_OP_MULCOEFFSMONTGOMERY, CSpan{U + (size_t)nq * N, N, qp}, CSpan{pkk + (size_t)c->nQ * N, N, 0},
                         Span{C + (size_t)nq * N, N, qp}, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
        if (launch_intt(c, rqp, CSpan{C, N, qp}, Span{C, N, qp}, batch, NTT_CANONICAL, st)) return -1;
        if (small_to_rns(c, rqp, es[k], N, Span{E, N, qp}, batch, st)) return -1;
        if (launch_vecop(c, rqp, LGPU_OP_ADD, CSpan{C, N, qp}, CSpan{E, N, qp}, Span{C, N, qp}, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
        Span o{ct_out + (size_t)k * nq * N, N, ct_bs};
        if (moddown_qp_to_q(c, levelQ, levelP, CSpan{C, N, qp}, CSpan{C + (size_t)nq * N, N, qp}, o, batch, st)) return -1;
        if (is_ntt && launch_ntt(c, rq, CSpan{o.p, N, ct_bs}, o, batch, NTT_CANONICAL, st)) return -1;
        if (is_mont && launch_vecop(c, rq, LGPU_OP_MFORM, CSpan{o.p, N, ct_bs}, CSpan{nullptr, 0, 0}, o, batch, nullptr, nullptr, 0, 0, c->N, st)) return -1;
    }
    return 0;
}

// BaseTwoDecompositionVectorSize (core/rlwe/params.go:520-540) of digit i: ceil(round(log2 q_i) / pw2), or 1 when pw2 = 0 or levelP > 0
int base_two_decomposition_size(const Ctx* c, int levelP, int pw2, int i) {
    if (pw2 == 0 || levelP > 0) return 1;
    const int logq = (int)std::round(std::log2((double)c->Q[i]));
    return (logq + pw2 - 1) / pw2;
}

// Ciphertexts per chunk: LGPU_KEYGEN_CHUNK if set (read on every call), else as many as keep the chunk's scratch under 2^25 words; at
// most 65535 entries per launch either way.
static int keygen_chunk(size_t words_per_ct, int entries) {
    const char* env = getenv("LGPU_KEYGEN_CHUNK");
    long long ch = env && atoi(env) > 0 ? atoi(env) : (long long)((1ull << 25) / (words_per_ct ? words_per_ct : 1));
    if (ch < 1) ch = 1;
    if (ch > 65535 / entries) ch = 65535 / entries;
    return (int)(ch < 1 ? 1 : ch);
}

int gadget_encrypt(const Ctx* c, const GadgetEncLayout& g, const GadgetEncCt* cts, int n_cts, const long long* e, const GadgetEncDraw* draw,
                   cudaStream_t st) {
    const size_t N = c->N;
    const int nq = g.levelQ + 1, np = g.levelP + 1, rows = nq + np, entries = g.n_digits * g.n_pw2_max;
    const size_t rowsN = (size_t)rows * N, key_rows = (size_t)c->nQ + c->nP;
    const RowMap rqp = rows_qp(c, nq, np);
    bool any_gal = false;
    for (int b = 0; b < n_cts; b++) any_gal |= cts[b].gal_el != 0;
    const size_t per_ct = (size_t)entries * rowsN * (draw ? 2 : 1) + (draw ? (size_t)entries * N : 0) + (any_gal ? key_rows * N : 0);
    const int ch = keygen_chunk(per_ct, entries);
    const int C = ch < n_cts ? ch : n_cts;
    // f_j on the Q rows: P_levelP 2^(pw2 j) mod q (the reference's MulScalarBigint by P, then MulScalar by 2^pw2 per j)
    std::vector<u64> hf((size_t)nq * g.n_pw2_max);
    for (int r = 0; r < nq; r++) {
        const u64 q = c->Q[r];
        u64 f = 1;
        for (int j = 0; j <= g.levelP; j++) f = h_mulmod(f, c->P[j] % q, q);
        for (int j = 0; j < g.n_pw2_max; j++) {
            hf[(size_t)r * g.n_pw2_max + j] = g.mont ? h_mform(f, q) : f;
            f = h_mulmod(f, (1ull << g.pw2) % q, q);
        }
    }
    Scratch E, U, G, S, idx, fbuf, dbuf;
    if (E.alloc((size_t)C * entries * rowsN, st)) return -1;
    if (draw && (U.alloc((size_t)C * entries * rowsN, st) || G.alloc((size_t)C * entries * N, st))) return -1;
    if (any_gal && (S.alloc((size_t)C * key_rows * N, st) || idx.alloc(N, st))) return -1;
    if (fbuf.alloc(hf.size(), st)) return -1;
    // host descriptors: a drawn c1 lives in U, an automorphed secret in S, at the ciphertext's place in its chunk
    std::vector<GadgetEncDev> hd((size_t)n_cts);
    for (int b = 0; b < n_cts; b++) {
        const GadgetEncCt& x = cts[b];
        GadgetEncDev& dv = hd[b];
        dv.c0 = x.c0; dv.pt = x.pt; dv.target = x.target; dv.c1_out = x.c1_out;
        if (draw) { dv.c1 = U.p + (size_t)(b % C) * entries * rowsN; dv.c1_es = rowsN; }
        else { dv.c1 = x.c1; dv.c1_es = g.c1_es; }
        dv.s = x.gal_el ? S.p + (size_t)(b % C) * key_rows * N : x.s_out;
    }
    const size_t dwords = (hd.size() * sizeof(GadgetEncDev) + 7) / 8;
    if (dbuf.alloc(dwords, st)) return -1;
    // pageable sources: both copies are staged before they return
    LGPU_CUDA_OK(cudaMemcpyAsync(fbuf.p, hf.data(), hf.size() * sizeof(u64), cudaMemcpyHostToDevice, st));
    LGPU_CUDA_OK(cudaMemcpyAsync(dbuf.p, hd.data(), hd.size() * sizeof(GadgetEncDev), cudaMemcpyHostToDevice, st));
    const GadgetEncDev* d_cts = reinterpret_cast<const GadgetEncDev*>(dbuf.p);
    GadgetEpiParams p;
    memset(&p, 0, sizeof(p));
    p.limbs = c->d_limbs; p.E = E.p; p.f = fbuf.p; p.c0_es = g.c0_es; p.c1_out_es = g.c1_es;
    p.nq = nq; p.rows = rows; p.nQ = c->nQ; p.k = g.levelP >= 0 ? g.levelP + 1 : 1; p.n = c->N; p.npw2 = g.n_pw2_max; p.entries = entries;
    p.mont = g.mont ? 1 : 0;
    for (int i = 0; i < g.n_digits; i++) p.npw2_of_digit[i] = (unsigned char)(g.pw2_sizes ? g.pw2_sizes[i] : g.n_pw2_max);
    // 16-byte accesses when every pointer and stride allows them
    bool vec = AL(E.p) && g.c0_es % 2 == 0 && g.c1_es % 2 == 0 && N % 2 == 0;
    for (int b = 0; b < n_cts && vec; b++)
        vec = AL(hd[b].c0) && AL(hd[b].c1) && hd[b].c1_es % 2 == 0 && AL(hd[b].s) && (!hd[b].pt || AL(hd[b].pt)) && (!hd[b].c1_out || AL(hd[b].c1_out));
    const int W = vec ? 2 : 1;
    for (int b0 = 0; b0 < n_cts; b0 += C) {
        const int nb = n_cts - b0 < C ? n_cts - b0 : C, units = nb * entries;
        const long long* ec = e ? e + (size_t)b0 * entries * N : (const long long*)G.p;
        if (draw) {     // ciphertext m draws on stream id stream0 + m: the uniform c1 of entry t as batch element t, its error likewise
            UniformParams up;
            up.limbs = c->d_limbs; up.rm = rqp; up.out = U.p; up.rs = N; up.bs = rowsN; up.key = make_key(draw->seed, 0); up.n = c->N;
            up.split = StreamSplit{draw->seed, draw->stream0 + (u64)b0, entries};
            count_launch(2);
            sample_uniform_kernel<<<dim3((c->N + 255) / 256, rows, units), 256, 0, st>>>(up);
            sample_gaussian_kernel<<<dim3((c->N + 255) / 256, units), 256, 0, st>>>((long long*)G.p, c->N, draw->sigma, draw->bound, make_key(draw->seed, 0),
                                                                                   StreamSplit{draw->seed, draw->stream0 + (u64)b0, entries});
            LGPU_CUDA_OK(cudaGetLastError());
        }
        if (small_to_rns(c, rqp, ec, N, Span{E.p, N, rowsN}, units, st)) return -1;
        if (launch_ntt(c, rqp, CSpan{E.p, N, rowsN}, Span{E.p, N, rowsN}, units, NTT_CANONICAL, st)) return -1;
        for (int b = b0; b < b0 + nb; b++) {     // s_out = AutomorphismNTT(sk, galEl^-1 mod 2N) on Q and P (keygenerator.go:153-175)
            if (!cts[b].gal_el) continue;
            const u64 inv = h_powmod(cts[b].gal_el, (u64)c->nthroot - 1, (u64)c->nthroot);
            if (automorphism_ntt_index(c, inv, idx.p, st)) return -1;
            if (automorphism_ntt_with_index(c, (int)key_rows, CSpan{cts[b].s_out, N, 0}, idx.p, Span{S.p + (size_t)(b - b0) * key_rows * N, N, 0}, false, 1,
                                            st)) return -1;
        }
        p.cts = d_cts + b0;
        count_launch(1);
        const dim3 grid((unsigned)((N / W + 255) / 256), (unsigned)rows, (unsigned)units);
        if (vec) gadget_enc_epilogue_kernel<2><<<grid, 256, 0, st>>>(p);
        else gadget_enc_epilogue_kernel<1><<<grid, 256, 0, st>>>(p);
        LGPU_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_sample_uniform(lgpu_ctx* ctx, int ring, int level, uint64_t seed, uint64_t stream_id, uint64_t* out, int batch, size_t batch_stride, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(out && batch >= 1 && batch <= 65535, "bad argument");
    UniformParams p;
    if (make_rowmap(ctx->c, ring, level, p.rm)) return -1;
    p.limbs = ctx->c.d_limbs; p.out = (u64*)out; p.rs = ctx->c.N; p.bs = batch_stride; p.key = make_key(seed, stream_id); p.n = ctx->c.N;
    p.split = StreamSplit{0, 0, 0};
    count_launch(1);
    sample_uniform_kernel<<<dim3((ctx->c.N + 255) / 256, p.rm.nrows, batch), 256, 0, (cudaStream_t)stream>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int lgpu_sample_ternary(lgpu_ctx* ctx, double p, int hamming_weight, uint64_t seed, uint64_t stream_id, int64_t* out, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(out && batch >= 1 && batch <= 65535, "bad argument");
    const int N = ctx->c.N;
    count_launch(1);
    if (hamming_weight > 0) {
        if (hamming_weight > N) hamming_weight = N;      // as the reference does (ring/sampler_ternary.go:202-204)
        const size_t smem = (size_t)((N + 31) / 32) * sizeof(unsigned);
        sample_ternary_h_kernel<<<batch, 256, smem, (cudaStream_t)stream>>>((long long*)out, N, hamming_weight, make_key(seed, stream_id));
    } else {
        REQUIRE(p > 0.0 && p <= 1.0, "ternary sampler: P must be in (0, 1]");
        sample_ternary_p_kernel<<<dim3((N + 255) / 256, batch), 256, 0, (cudaStream_t)stream>>>((long long*)out, N, p, make_key(seed, stream_id));
    }
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int lgpu_sample_gaussian(lgpu_ctx* ctx, double sigma, double bound, uint64_t seed, uint64_t stream_id, int64_t* out, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(out && batch >= 1 && batch <= 65535, "bad argument");
    REQUIRE(sigma > 0.0 && bound >= 1.0 && bound < 9.0e18, "gaussian sampler: sigma / bound out of range");
    const int N = ctx->c.N;
    count_launch(1);
    sample_gaussian_kernel<<<dim3((N + 255) / 256, batch), 256, 0, (cudaStream_t)stream>>>((long long*)out, N, sigma, bound, make_key(seed, stream_id),
                                                                                         StreamSplit{0, 0, 0});
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

int lgpu_small_poly_to_rns(lgpu_ctx* ctx, int level_q, int level_p, const int64_t* small, uint64_t* out_q, uint64_t* out_p, int batch, size_t stride_q,
                           size_t stride_p, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(small && (out_q || out_p) && batch >= 1 && batch <= 65535, "bad argument");
    const Ctx& c = ctx->c;
    RowMap rm;
    if (out_q) {
        if (make_rowmap(c, LGPU_RING_Q, level_q, rm)) return -1;
        if (small_to_rns(&c, rm, (const long long*)small, c.N, Span{(u64*)out_q, (size_t)c.N, stride_q}, batch, (cudaStream_t)stream)) return -1;
    }
    if (out_p && level_p >= 0) {
        if (make_rowmap(c, LGPU_RING_P, level_p, rm)) return -1;
        if (small_to_rns(&c, rm, (const long long*)small, c.N, Span{(u64*)out_p, (size_t)c.N, stride_p}, batch, (cudaStream_t)stream)) return -1;
    }
    return 0;
}

int lgpu_encrypt_zero_pk(lgpu_ctx* ctx, int level_q, const uint64_t* pk, const int64_t* u, const int64_t* e0, const int64_t* e1, uint64_t* ct_out,
                         int is_ntt, int is_montgomery, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(pk && u && e0 && e1 && ct_out, "null argument");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    return encrypt_zero_pk(&ctx->c, level_q, (const u64*)pk, (const long long*)u, (const long long*)e0, (const long long*)e1, (u64*)ct_out, is_ntt != 0,
                           is_montgomery != 0, batch, (cudaStream_t)stream);
}

int lgpu_encrypt_zero_sk(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* sk, uint64_t* c1, const int64_t* e, uint64_t* c0, int is_ntt,
                         int is_montgomery, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(sk && c1 && e && c0, "null argument");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    const size_t bs = (size_t)(level_q + 1 + level_p + 1) * ctx->c.N;
    return encrypt_zero_sk(&ctx->c, level_q, level_p, (const u64*)sk, (u64*)c1, bs, (const long long*)e, (u64*)c0, bs, is_ntt != 0, is_montgomery != 0, batch,
                           (cudaStream_t)stream);
}

int lgpu_gen_evaluation_key(lgpu_ctx* ctx, const uint64_t* sk_in, const uint64_t* sk_out, lgpu_gadget_ct* evk, const int64_t* e, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(sk_in && sk_out && evk && evk->data && e, "null argument");
    GadgetCt g;
    if (to_gadget_ct(evk, g)) return -1;
    REQUIRE(g.levelQ == ctx->c.nQ - 1 && g.levelP == ctx->c.nP - 1, "evaluation keys are generated at the maximum levels");
    const size_t ebs = (size_t)2 * (ctx->c.nQ + ctx->c.nP) * ctx->c.N;     // component 1 of every entry holds the uniform polynomial
    u64* data = (u64*)evk->data;
    const int nd = g.levelP >= 0 ? base_rns_decomposition_vector_size(g.levelQ, g.levelP) : g.levelQ + 1;
    REQUIRE(g.ndigits == nd, "evaluation key: n_digits != BaseRNSDecompositionVectorSize(levelQ, levelP)");
    REQUIRE(g.npw2max >= 1 && g.npw2max <= 64, "evaluation key: n_pw2_max out of [1, 64]");
    REQUIRE(g.pw2 >= 0 && g.pw2 <= 62, "evaluation key: BaseTwoDecomposition out of [0, 62]");
    for (int i = 0; g.pw2_sizes && i < g.ndigits; i++)
        REQUIRE(g.pw2_sizes[i] >= 1 && g.pw2_sizes[i] <= g.npw2max, "evaluation key: pw2_sizes[i] out of [1, n_pw2_max]");
    const GadgetEncLayout lay{g.levelQ, g.levelP, g.pw2, g.ndigits, g.npw2max, g.pw2_sizes, ebs, ebs, true};
    const GadgetEncCt ct{data, data + ebs / 2, nullptr, (const u64*)sk_out, 0, (const u64*)sk_in, 0};
    return gadget_encrypt(&ctx->c, lay, &ct, 1, (const long long*)e, nullptr, (cudaStream_t)stream);
}

}  // extern "C"

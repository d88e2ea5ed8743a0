// blindrot.cu -- blindrot.Evaluator.Evaluate (core/rgsw/blindrot/evaluator.go:49-132) for a BATCH of LWE-ring ciphertexts and a set of
// slots, on the device:
//   br_modswitch_kernel  modSwitchRLWETo2NLvl of both components (:80-94, :254-283 of the same file): round(x 2N / q_LWE), ties away
//                        from zero, the mask made odd; after an INTT in the LWE ring when the input is in the NTT domain.
//   (host)               per (batch entry, slot): the mask a_0, -a_{N-1}, ..., -a_1 rotated by X^slot, its discrete-log sets and the
//                        op schedule of Algorithm 3 (eprint 2022/198) with the window logic of BlindRotateCore (:144-229), as
//                        lgpu_blind_rotate_core walks it. The schedules and the key pointer tables go up in one copy.
//   br_fused_kernel      one CTA per accumulator: acc = (AutomorphismNTT(f * X^b, 2N - 5), 0) from the forward root table, then the
//                        schedule (EXT j: rgsw ExternalProduct with RGSW(X^{s_j}); AUTO: Evaluator.Automorphism), then the optional
//                        INTT, entirely in shared memory. No CTA waits on another one.
// The fused kernel serves level 0 (one Q modulus), keys without P and with BaseTwoDecomposition >= 1, and 2^8 <= N <= 2^12: its working
// set is six polynomials (the accumulator, two key-switch accumulators and two digits in flight), 48 N bytes of shared memory, 192 KB at
// N = 2^12 against the 227 KB a CTA can have on sm_90. Every other input takes the reference loop: each slot through lgpu_blind_rotate_core.
//
// Arithmetic, bit for bit with the reference:
//   - transforms are radix-2 stage loops over shared memory. The forward one is the reference's lazy Montgomery butterfly with its
//     4q-correction schedule (fwd_bfly / fwd_reduce_flag, as the FAST = 0 kernels of ntt.cu), so every decomposed digit carries
//     NTTLazy's own representative in [0, 6q).
//   - q < 2^29 (externalProduct32Bit, core/rgsw/evaluator.go:90-128): the products key * NTTLazy(digit) are summed in a wrapping 64-bit
//     word and IMForm is applied once at the end, which is the reference's word even where the sum wraps (small BaseTwoDecomposition
//     and q near 2^29).
//   - q >= 2^29 (externalProductInPlaceSinglePAndBitDecomp) and every automorphism key switch (gadgetProductSinglePAndBitDecompLazy with
//     periodic Reduce, no P): the reference's outputs are canonical residues, so canonical Montgomery sums give the same words.
//   - GaloisElement(v) = 1 (v a multiple of N/2 inside the window) is a copy without a key, as in evaluator_automorphism.go:19-24.
#include <algorithm>
#include <string>
#include <vector>
#include "capi_common.h"
#include "composite.h"
#include "modarith.cuh"
#include "ntt_arith.cuh"
#include "xpow.cuh"

namespace lgpu {

static constexpr int kFusedMinLogN = 8, kFusedMaxLogN = 12;

struct KeyDesc {          // digit 0 of a GadgetCiphertext without P: entry (j, comp) at p + (2 j + comp) * stride
    const u64* p;
    u64 gal_el;           // automorphism keys only
    unsigned stride;      // (levelQ + 1) * N
    int nj;               // BaseTwoDecompositionVectorSize()[0]
    int pw2;
    int pad;
};
struct CtaDesc {          // the schedule of one (batch entry, slot) accumulator and its b modulo 2N
    unsigned long long off;
    unsigned len, bval;
};

struct FusedParams {
    const LimbConst* limbs;
    const KeyDesc* brk;           // [2][n_lwe]
    const KeyDesc* gk;
    const u64* const* tp;         // per slot
    const CtaDesc* cta;           // [batch][n_slots]
    const int* ops;               // j >= 0: EXT j; -(g + 1): AUTO with gk[g]
    u64* out;                     // [batch][n_slots][2][N]
    int n_lwe, n_slots, logN, ntt_out, small_q;
};

__device__ __forceinline__ u64 br_mask(u64 x, int j, int pw2) { return (x >> (j * pw2)) & ((1ull << pw2) - 1); }

// NTTLazy of up to two polynomials in shared memory (ring/ntt.go:155-161 butterflies, reference correction schedule)
static __device__ void br_ntt_lazy(u64* p0, u64* p1, bool act1, const LimbConst& L, int logN) {
    const int N = 1 << logN, T = blockDim.x;
    const int nb = act1 ? N : N >> 1;
    for (int s = 0; s < logN; s++) {
        const int ts = logN - 1 - s;
        const bool red = fwd_reduce_flag(s, logN);
        for (int u = threadIdx.x; u < nb; u += T) {
            u64* p = (u >> (logN - 1)) ? p1 : p0;
            const int bf = u & ((N >> 1) - 1), grp = bf >> ts;
            const int j1 = (grp << (ts + 1)) + (bf & ((1 << ts) - 1));
            fwd_bfly(p[j1], p[j1 + (1 << ts)], __ldg(L.roots_fwd + (1 << s) + grp), L.q, L.qinv, red);
        }
        __syncthreads();
    }
}

// INTT of up to two polynomials in shared memory, canonical outputs (ring/ntt.go:164-171, 185-206)
static __device__ void br_intt(u64* p0, u64* p1, bool act1, const LimbConst& L, int logN) {
    const int N = 1 << logN, T = blockDim.x;
    const int nb = act1 ? N : N >> 1;
    for (int s = logN - 1; s >= 0; s--) {
        const int ts = logN - 1 - s;
        for (int u = threadIdx.x; u < nb; u += T) {
            u64* p = (u >> (logN - 1)) ? p1 : p0;
            const int bf = u & ((N >> 1) - 1), grp = bf >> ts;
            const int j1 = (grp << (ts + 1)) + (bf & ((1 << ts) - 1));
            inv_bfly(p[j1], p[j1 + (1 << ts)], __ldg(L.roots_bwd + (1 << s) + grp), L.q, L.qinv);
        }
        __syncthreads();
    }
    for (int u = threadIdx.x; u < 2 * nb; u += T) {
        u64* p = (u >> logN) ? p1 : p0;
        const int i = u & (N - 1);
        p[i] = mred(p[i], L.ninv, L.q, L.qinv);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(512) br_fused_kernel(FusedParams p) {
    extern __shared__ u64 sm[];
    const int logN = p.logN, N = 1 << logN, T = blockDim.x, tid = threadIdx.x;
    u64* A0 = sm;
    u64* A1 = A0 + N;
    u64* T0 = A1 + N;
    u64* T1 = T0 + N;
    u64* W0 = T1 + N;
    u64* W1 = W0 + N;
    const LimbConst L = p.limbs[0];
    const u64 q = L.q, qinv = L.qinv, mask2n = 2 * (u64)N - 1;
    const CtaDesc cd = p.cta[blockIdx.x];
    // acc = (AutomorphismNTT(testPoly * MForm(NTT(X^b)), 2N - 5), 0)   (evaluator.go:103-111)
    {
        const u64* tp = p.tp[blockIdx.x % p.n_slots];
        for (int i = tid; i < N; i += T) {
            const int idx = (int)auto_index(i, mask2n - 4, mask2n, logN);
            const u64 odd = 2 * (__brevll((u64)idx) >> (64 - logN)) + 1;
            A0[i] = mul_xpow(tp[idx], cd.bval, odd, L, logN, mask2n);
            A1[i] = 0;
        }
        __syncthreads();
    }
    const int* ops = p.ops + cd.off;
    for (unsigned o = 0; o < cd.len; o++) {
        const int op = ops[o];
        if (op >= 0) {
            // rgsw ExternalProduct(acc, RGSW(X^{s_j}), acc), levelQ = 0, no P (core/rgsw/evaluator.go:39-208)
            const KeyDesc K0 = p.brk[op], K1 = p.brk[p.n_lwe + op];
            br_intt(A0, A1, true, L, logN);
            const int nj = max(K0.nj, K1.nj);
            for (int j = 0; j < nj; j++) {
                const bool a0 = j < K0.nj, a1 = j < K1.nj;
                for (int i = tid; i < N; i += T) {
                    if (a0) W0[i] = br_mask(A0[i], j, K0.pw2);
                    if (a1) W1[i] = br_mask(A1[i], j, K1.pw2);
                }
                __syncthreads();
                if (a0) br_ntt_lazy(W0, W1, a1, L, logN);
                else br_ntt_lazy(W1, nullptr, false, L, logN);
                const u64* k00 = K0.p + (size_t)(2 * j) * K0.stride;
                const u64* k01 = k00 + K0.stride;
                const u64* k10 = K1.p + (size_t)(2 * j) * K1.stride;
                const u64* k11 = k10 + K1.stride;
                for (int i = tid; i < N; i += T) {
                    u64 t0 = j ? T0[i] : 0, t1 = j ? T1[i] : 0;
                    if (p.small_q) {
                        if (a0) { const u64 w = W0[i]; t0 += __ldg(k00 + i) * w; t1 += __ldg(k01 + i) * w; }
                        if (a1) { const u64 w = W1[i]; t0 += __ldg(k10 + i) * w; t1 += __ldg(k11 + i) * w; }
                    } else {
                        if (a0) { const u64 w = W0[i]; t0 = cred(t0 + mred(__ldg(k00 + i), w, q, qinv), q); t1 = cred(t1 + mred(__ldg(k01 + i), w, q, qinv), q); }
                        if (a1) { const u64 w = W1[i]; t0 = cred(t0 + mred(__ldg(k10 + i), w, q, qinv), q); t1 = cred(t1 + mred(__ldg(k11 + i), w, q, qinv), q); }
                    }
                    T0[i] = t0; T1[i] = t1;
                }
            }
            for (int i = tid; i < N; i += T) {
                A0[i] = p.small_q ? imform(T0[i], q, qinv) : T0[i];
                A1[i] = p.small_q ? imform(T1[i], q, qinv) : T1[i];
            }
            __syncthreads();
        } else {
            // Evaluator.Automorphism(acc, galEl, acc): GadgetProduct(acc[1], gk) + (acc[0], 0), then AutomorphismNTT (core/rlwe/evaluator_automorphism.go:13-57)
            const KeyDesc K = p.gk[-op - 1];
            br_intt(A1, nullptr, false, L, logN);
            for (int j = 0; j < K.nj; j += 2) {
                const bool a1 = j + 1 < K.nj;
                for (int i = tid; i < N; i += T) {
                    W0[i] = br_mask(A1[i], j, K.pw2);
                    if (a1) W1[i] = br_mask(A1[i], j + 1, K.pw2);
                }
                __syncthreads();
                br_ntt_lazy(W0, W1, a1, L, logN);
                const u64* k0 = K.p + (size_t)(2 * j) * K.stride;
                const u64* k1 = k0 + K.stride;
                for (int i = tid; i < N; i += T) {
                    u64 t0 = j ? T0[i] : 0, t1 = j ? T1[i] : 0;
                    u64 w = W0[i];
                    t0 = cred(t0 + mred(__ldg(k0 + i), w, q, qinv), q); t1 = cred(t1 + mred(__ldg(k1 + i), w, q, qinv), q);
                    if (a1) {
                        w = W1[i];
                        t0 = cred(t0 + mred(__ldg(k0 + 2 * (size_t)K.stride + i), w, q, qinv), q);
                        t1 = cred(t1 + mred(__ldg(k1 + 2 * (size_t)K.stride + i), w, q, qinv), q);
                    }
                    T0[i] = t0; T1[i] = t1;
                }
            }
            for (int i = tid; i < N; i += T) T0[i] = cred(T0[i] + A0[i], q);
            __syncthreads();
            for (int i = tid; i < N; i += T) {
                const int idx = (int)auto_index(i, K.gal_el, mask2n, logN);
                A0[i] = T0[idx];
                A1[i] = T1[idx];
            }
            __syncthreads();
        }
    }
    if (!p.ntt_out) br_intt(A0, A1, true, L, logN);        // !NTTFlag (evaluator.go:123-127)
    u64* out = p.out + (size_t)blockIdx.x * 2 * N;
    for (int i = tid; i < N; i += T) { out[i] = A0[i]; out[N + i] = A1[i]; }
}

// modSwitchRLWETo2NLvl (evaluator.go:254-283) at level 0: ct [batch][2][n] coefficient domain; a2n / b2n: [batch][n]
__global__ void __launch_bounds__(256) br_modswitch_kernel(const u64* ct, u64 q, int n, u64 twoN, u64* a2n, u64* b2n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t b = blockIdx.y;
    const u64* c = ct + b * 2 * n;
    for (int comp = 0; comp < 2; comp++) {
        const unsigned __int128 v = (unsigned __int128)(c[comp * n + i] % q) * twoN;
        u64 r = (u64)(v / q);
        const u64 rem = (u64)(v - (unsigned __int128)r * q);
        if ((unsigned __int128)rem * 2 >= q) r++;           // bignum.DivRound: ties away from zero
        r &= twoN - 1;
        if (comp == 1) {
            if ((r & 1) == 0 && r != 0) r ^= 1;
            a2n[b * n + i] = r;
        } else {
            b2n[b * n + i] = r;
        }
    }
}

// the initial accumulators of the reference loop, every limb: [batch][n_slots][2][level+1][N]
__global__ void __launch_bounds__(256) br_init_kernel(const LimbConst* limbs, const u64* const* tp, const CtaDesc* cta, int n_slots, int logN,
                                                      size_t cs, size_t e0, u64* out) {
    const int N = 1 << logN;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int r = blockIdx.y;
    const size_t e = e0 + blockIdx.z;
    const LimbConst L = limbs[r];
    const u64 mask2n = 2 * (u64)N - 1;
    const int idx = (int)auto_index(i, mask2n - 4, mask2n, logN);
    const u64 odd = 2 * (__brevll((u64)idx) >> (64 - logN)) + 1;
    u64* o = out + e * 2 * cs + (size_t)r * N;
    o[i] = mul_xpow(tp[e % n_slots][(size_t)r * N + idx], cta[e].bval, odd, L, logN, mask2n);
    o[cs + i] = 0;
}

static KeyDesc key_desc(const Ctx& c, const GadgetCt& g, u64 gal_el) {
    return KeyDesc{g.data, gal_el, (unsigned)((g.levelQ + 1 + g.levelP + 1) * (size_t)c.N), g.pw2_sizes ? g.pw2_sizes[0] : 1, g.pw2, 0};
}

static size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

}  // namespace lgpu

using namespace lgpu;

extern "C" int lgpu_blind_rotation_evaluate(lgpu_ctx* ctx, lgpu_ctx* ctx_lwe, const uint64_t* ct_lwe, int level_lwe, int is_ntt, const int* slots,
                                            int n_slots, const uint64_t* const* test_polys, const lgpu_gadget_ct* brk0, const lgpu_gadget_ct* brk1,
                                            int n_brk, const lgpu_galois_keys* gks, int window_size, int ntt_out, uint64_t* ct_out, int batch,
                                            void* stream) {
    REQUIRE(ctx && ctx_lwe, "null context");
    REQUIRE(ct_lwe && slots && test_polys && brk0 && brk1 && gks && ct_out, "null argument");
    const Ctx& c = ctx->c;
    const Ctx& cl = ctx_lwe->c;
    REQUIRE(c.ring_type == 0 && cl.ring_type == 0, "blind rotation is defined on the standard ring");
    REQUIRE(cl.N <= c.N, "blind rotation: the LWE ring degree is larger than the blind-rotation ring degree");
    REQUIRE(level_lwe == 0, "blind rotation: LWE ciphertexts above level 0 are not supported (the reference switches them to 2N with big integers)");
    REQUIRE(is_ntt == 0 || is_ntt == 1, "is_ntt must be 0 or 1");
    REQUIRE(ntt_out == 0 || ntt_out == 1, "ntt_out must be 0 or 1");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(window_size >= 1, "window size must be positive");
    const int n_lwe = cl.N;
    REQUIRE(n_brk >= n_lwe, "blind rotation: fewer blind-rotation keys than LWE coefficients");
    REQUIRE(n_slots >= 1, "no slot to evaluate");
    {
        std::vector<char> seen((size_t)n_lwe, 0);
        for (int k = 0; k < n_slots; k++) {
            REQUIRE(slots[k] >= 0 && slots[k] < n_lwe, "blind rotation: slot index out of range [0, N_LWE)");
            REQUIRE(!seen[slots[k]], "blind rotation: duplicate slot index");
            seen[slots[k]] = 1;
            REQUIRE(test_polys[k], "null test polynomial");
            REQUIRE_ALIGNED(AL(test_polys[k]));
        }
    }
    REQUIRE_ALIGNED(AL(ct_lwe) && AL(ct_out));
    GadgetCt g0;
    if (to_gadget_ct(&brk0[0], g0)) return -1;
    const int level = g0.levelQ;
    REQUIRE(level >= 0 && level < c.nQ, "blind-rotation key level out of range");
    std::vector<KeyDesc> kd(2 * (size_t)n_lwe);
    for (int comp = 0; comp < 2; comp++) {
        for (int j = 0; j < n_lwe; j++) {
            GadgetCt g;
            if (to_gadget_ct(comp ? &brk1[j] : &brk0[j], g)) return -1;
            REQUIRE(g.levelQ == g0.levelQ && g.levelP == g0.levelP && g.pw2 == g0.pw2,
                    "blind-rotation keys must share their levels and BaseTwoDecomposition");
            if (check_evk(&c, level, g)) return -1;
            kd[(size_t)comp * n_lwe + j] = key_desc(c, g, 0);
        }
    }
    bool fused = level == 0 && g0.levelP == -1 && g0.pw2 >= 1 && g0.pw2 <= 62 && c.logN >= kFusedMinLogN && c.logN <= kFusedMaxLogN;
    // the automorphism keys Algorithm 3 can reach: GaloisElement(1..window) and NthRoot - GaloisGen (keys.go:94-101)
    GaloisKeySet ks;
    if (to_galois_keys(gks, ks)) return -1;
    std::vector<u64> need;
    for (int v = 1; v <= window_size && v <= c.N; v++) {
        const u64 g = galois_element(&c, v);
        if (g != 1 && std::find(need.begin(), need.end(), g) == need.end()) need.push_back(g);
    }
    need.push_back(c.nthroot - 5);
    std::vector<KeyDesc> gd;
    for (u64 g : need) {
        const GadgetCt* gk = ks.find(g);
        if (!gk) return -1;
        if (check_evk(&c, level, *gk)) return -1;
        fused = fused && gk->levelP == -1 && gk->pw2 >= 1 && gk->pw2 <= 62;
        gd.push_back(key_desc(c, *gk, g));
    }
    REQUIRE_DEVICE(ctx);
    REQUIRE(cl.device == c.device, "the two contexts must be on the same device");
    LGPU_CUDA_OK(cudaSetDevice(c.device));
    cudaStream_t st = (cudaStream_t)stream;
    const size_t N = c.N, nl = (size_t)n_lwe, twoN = 2 * N, ncta = (size_t)batch * n_slots;

    // 1. LWE -> coefficient domain -> modulo 2N (evaluator.go:65-94)
    Scratch pre;
    if (pre.alloc((size_t)batch * 4 * nl, st)) return -1;
    const u64* coef = (const u64*)ct_lwe;
    if (is_ntt) {
        for (size_t e0 = 0; e0 < 2 * (size_t)batch; e0 += 65535) {
            const int nb = (int)std::min<size_t>(65535, 2 * (size_t)batch - e0);
            if (launch_intt(&cl, rows_range(0, 0, 1), CSpan{coef + e0 * nl, nl, nl}, Span{pre.p + e0 * nl, nl, nl}, nb, NTT_CANONICAL, st)) return -1;
        }
        coef = pre.p;
    }
    u64* a2n = pre.p + (size_t)batch * 2 * nl;
    u64* b2n = a2n + (size_t)batch * nl;
    {
        ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * 4 * nl * batch, 1);
        br_modswitch_kernel<<<dim3((unsigned)((nl + 255) / 256), batch), 256, 0, st>>>(coef, cl.Q[0], n_lwe, twoN, a2n, b2n);
        LGPU_CUDA_OK(cudaGetLastError());
    }
    std::vector<u64> h_ab((size_t)batch * 2 * nl);
    LGPU_CUDA_OK(cudaMemcpyAsync(h_ab.data(), a2n, h_ab.size() * 8, cudaMemcpyDeviceToHost, st));
    LGPU_CUDA_OK(cudaStreamSynchronize(st));

    // 2. per accumulator: the rotated mask (the cumulative mulBySmallMonomialMod2N of :100-104 is the rotation by X^slot) and b
    std::vector<CtaDesc> cta(ncta);
    std::vector<std::vector<u64>> masks(fused ? 0 : ncta);
    std::vector<int> ops;
    const long long Nhalf = (long long)N >> 1;
    std::vector<long long> dlog(twoN, 0);
    std::vector<char> has(twoN, 0);
    {
        unsigned long long pw = 1;
        for (long long i = 0; i < Nhalf; i++) {
            dlog[pw] = i; has[pw] = 1;
            dlog[twoN - pw] = -i; has[twoN - pw] = 1;
            pw = pw * 5 & (twoN - 1);
        }
    }
    auto key_index = [&](u64 g) { for (size_t i = 0; i < gd.size(); i++) if (gd[i].gal_el == g) return (int)i; return -1; };
    std::vector<u64> a(nl);
    std::vector<int> head((size_t)N), cnt((size_t)N), order(nl);
    for (int b = 0; b < batch; b++) {
        const u64* ab = h_ab.data() + (size_t)b * nl;
        const u64* bb = h_ab.data() + (size_t)batch * nl + (size_t)b * nl;
        for (int k = 0; k < n_slots; k++) {
            const size_t e = (size_t)b * n_slots + k;
            const int s = slots[k];
            // a' = a_0, -a_{n-1}, ..., -a_1 (mod 2N), times X^s: a'[j] for j >= s is a'_{j - s}, -a'_{n + j - s} below
            auto ext = [&](size_t j) -> u64 { return j == 0 ? ab[0] : (twoN - ab[nl - j]) & (twoN - 1); };
            for (size_t j = 0; j < nl; j++) a[j] = j >= (size_t)s ? ext(j - s) : (twoN - ext(nl + j - s)) & (twoN - 1);
            cta[e].bval = (unsigned)bb[s];
            cta[e].off = ops.size();
            if (!fused) { masks[e] = a; cta[e].len = 0; continue; }
            // discrete-log sets (getDiscreteLogSets, :261-283): bucket k + N/2, members in increasing j
            std::fill(cnt.begin(), cnt.end(), 0);
            for (size_t j = 0; j < nl; j++) cnt[(size_t)((has[a[j]] ? dlog[a[j]] : 0) + Nhalf)]++;
            int acc = 0;
            for (size_t t = 0; t < N; t++) { head[t] = acc; acc += cnt[t]; }
            {
                std::vector<int> pos(head);
                for (size_t j = 0; j < nl; j++) order[pos[(size_t)((has[a[j]] ? dlog[a[j]] : 0) + Nhalf)]++] = (int)j;
            }
            auto automorph = [&](long long v) {
                const u64 g = galois_element(&c, v);
                if (g != 1) ops.push_back(-key_index(g) - 1);
            };
            auto from_sets = [&](long long kk, int v) -> int {      // evaluateFromDiscreteLogSets (:206-229)
                if (kk > -Nhalf && kk < Nhalf && cnt[(size_t)(kk + Nhalf)] > 0) {
                    if (v != 0) { automorph(v); v = 0; }
                    const size_t t = (size_t)(kk + Nhalf);
                    for (int m = 0; m < cnt[t]; m++) ops.push_back(order[(size_t)head[t] + m]);
                }
                v++;
                if (v == window_size || kk == 1) { automorph(v); v = 0; }
                return v;
            };
            int v = 0;
            for (long long i = Nhalf - 1; i > 0; i--) v = from_sets(-i, v);
            from_sets((long long)twoN, 0);
            ops.push_back(-key_index(c.nthroot - 5) - 1);
            for (long long i = Nhalf - 1; i > 0; i--) v = from_sets(i, v);
            from_sets(0, 0);
            cta[e].len = (unsigned)(ops.size() - cta[e].off);
        }
    }

    // 3. one upload: key tables, test-polynomial pointers, CTA descriptors, schedules
    const size_t o_brk = 0, o_gk = align16(o_brk + kd.size() * sizeof(KeyDesc)), o_tp = align16(o_gk + gd.size() * sizeof(KeyDesc)),
                 o_cta = align16(o_tp + (size_t)n_slots * sizeof(u64)), o_ops = align16(o_cta + ncta * sizeof(CtaDesc)),
                 total = align16(o_ops + std::max<size_t>(1, ops.size()) * sizeof(int));
    std::vector<unsigned char> up(total, 0);
    memcpy(up.data() + o_brk, kd.data(), kd.size() * sizeof(KeyDesc));
    memcpy(up.data() + o_gk, gd.data(), gd.size() * sizeof(KeyDesc));
    memcpy(up.data() + o_tp, test_polys, (size_t)n_slots * sizeof(u64));
    memcpy(up.data() + o_cta, cta.data(), ncta * sizeof(CtaDesc));
    if (!ops.empty()) memcpy(up.data() + o_ops, ops.data(), ops.size() * sizeof(int));
    Scratch dev;
    if (dev.alloc(total / 8, st)) return -1;
    unsigned char* d = (unsigned char*)dev.p;
    LGPU_CUDA_OK(cudaMemcpyAsync(d, up.data(), total, cudaMemcpyHostToDevice, st));
    u64* out = (u64*)ct_out;

    if (fused) {
        FusedParams p;
        p.limbs = c.d_limbs; p.brk = (const KeyDesc*)(d + o_brk); p.gk = (const KeyDesc*)(d + o_gk); p.tp = (const u64* const*)(d + o_tp);
        p.cta = (const CtaDesc*)(d + o_cta); p.ops = (const int*)(d + o_ops); p.out = out;
        p.n_lwe = n_lwe; p.n_slots = n_slots; p.logN = c.logN; p.ntt_out = ntt_out; p.small_q = (c.Q[0] >> 29) == 0;
        const size_t smem = 6 * N * sizeof(u64);
        LGPU_CUDA_OK(cudaFuncSetAttribute(br_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(6 * sizeof(u64) << kFusedMaxLogN)));
        ProfScope ps(LGPU_KCLASS_MAC, st, 8.0 * ncta * (2 * N + (double)2 * n_lwe * 4 * N), 1);
        br_fused_kernel<<<(unsigned)ncta, (unsigned)std::min<size_t>(N, 512), smem, st>>>(p);
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }

    // the reference loop: every accumulator through lgpu_blind_rotate_core, in place in ct_out
    const size_t cs = (size_t)(level + 1) * N;
    for (size_t e0 = 0; e0 < ncta; e0 += 65535) {
        const unsigned nb = (unsigned)std::min<size_t>(65535, ncta - e0);
        ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * 3 * cs * nb, 1);
        br_init_kernel<<<dim3((unsigned)((N + 255) / 256), level + 1, nb), 256, 0, st>>>(
            c.d_limbs, (const u64* const*)(d + o_tp), (const CtaDesc*)(d + o_cta), n_slots, c.logN, cs, e0, out);
        LGPU_CUDA_OK(cudaGetLastError());
    }
    for (size_t e = 0; e < ncta; e++)
        if (lgpu_blind_rotate_core(ctx, (const uint64_t*)masks[e].data(), n_lwe, (uint64_t*)(out + e * 2 * cs), level, brk0, brk1, gks, window_size, stream)) return -1;
    if (!ntt_out) {
        for (size_t e0 = 0; e0 < 2 * ncta; e0 += 65535) {
            const int nb = (int)std::min<size_t>(65535, 2 * ncta - e0);
            if (launch_intt(&c, rows_range(0, 0, level + 1), CSpan{out + e0 * cs, N, cs}, Span{out + e0 * cs, N, cs}, nb, NTT_CANONICAL, st)) return -1;
        }
    }
    return 0;
}

// keygen.cu -- the C ABI of the batched gadget encryptions (gadget_encrypt, encrypt.cu):
//   rgsw.Encryptor.Encrypt / EncryptZero                  core/rgsw/encryptor.go:25-121
//   KeyGenerator.GenGaloisKeysNew                         core/rlwe/keygenerator.go:123-209
//   blindrot.GenEvaluationKeyNew                          core/rgsw/blindrot/keys.go:52-108
// Every argument check runs before any launch, also on a host-only context.
#include <algorithm>
#include <cmath>
#include <utility>
#include <vector>
#include "../../include/lattigo_b200.h"
#include "capi_common.h"
#include "composite.h"

namespace lgpu {

// the layout rgsw.NewCiphertext / NewGadgetCiphertext give a key at its levels and base (core/rlwe/gadgetciphertext.go:27-45)
static int check_layout(const Ctx& c, const GadgetCt& g) {
    if (g.levelQ < 0 || g.levelQ >= c.nQ || g.levelP < -1 || g.levelP >= c.nP) { set_error("gadget ciphertext: level out of range"); return -1; }
    if (g.pw2 < 0 || g.pw2 > 62) { set_error("gadget ciphertext: BaseTwoDecomposition out of [0, 62]"); return -1; }
    const int nd = g.levelP >= 0 ? base_rns_decomposition_vector_size(g.levelQ, g.levelP) : g.levelQ + 1;
    if (g.ndigits != nd) { set_error("gadget ciphertext: n_digits != BaseRNSDecompositionVectorSize(levelQ, levelP)"); return -1; }
    int mx = 1;
    for (int i = 0; i < nd; i++) {
        const int want = base_two_decomposition_size(&c, g.levelP, g.pw2, i);
        mx = std::max(mx, want);
        if ((g.pw2_sizes ? g.pw2_sizes[i] : 1) != want) {
            set_error("gadget ciphertext: pw2_sizes != BaseTwoDecompositionVectorSize(levelQ, levelP, BaseTwoDecomposition)");
            return -1;
        }
    }
    if (g.npw2max != mx) { set_error("gadget ciphertext: n_pw2_max != max(BaseTwoDecompositionVectorSize)"); return -1; }
    return 0;
}

static bool same_layout(const GadgetCt& a, const GadgetCt& b) {
    if (a.levelQ != b.levelQ || a.levelP != b.levelP || a.pw2 != b.pw2 || a.ndigits != b.ndigits || a.npw2max != b.npw2max) return false;
    for (int i = 0; i < a.ndigits; i++)
        if ((a.pw2_sizes ? a.pw2_sizes[i] : 1) != (b.pw2_sizes ? b.pw2_sizes[i] : 1)) return false;
    return true;
}

static size_t key_bytes(const GadgetCt& g, size_t N) {
    return (size_t)g.ndigits * g.npw2max * 2 * (size_t)(g.levelQ + 1 + g.levelP + 1) * N * sizeof(u64);
}

// n arrays of keys -> GadgetCt, every key with the layout of the first and checked against its levels and base; the keys' data blocks
// may not overlap one another or any of the `inputs` ranges
static int check_keys(const Ctx& c, const lgpu_gadget_ct* const* arrays, int n_arrays, int n, std::vector<GadgetCt>& out,
                      const std::vector<std::pair<const void*, size_t>>& inputs) {
    out.resize((size_t)n_arrays * n);
    for (int a = 0; a < n_arrays; a++) {
        if (!arrays[a]) { set_error("null argument"); return -1; }
        for (int k = 0; k < n; k++)
            if (to_gadget_ct(&arrays[a][k], out[(size_t)a * n + k], "null gadget ciphertext")) return -1;
    }
    if (check_layout(c, out[0])) return -1;
    for (const GadgetCt& g : out)
        if (!same_layout(g, out[0])) { set_error("gadget ciphertexts of one call differ in levels or digit layout"); return -1; }
    const size_t kb = key_bytes(out[0], c.N);
    std::vector<const u64*> d;
    for (const GadgetCt& g : out) d.push_back(g.data);
    std::sort(d.begin(), d.end());
    for (size_t k = 1; k < d.size(); k++)
        if (overlaps(d[k - 1], kb, d[k], kb)) { set_error("gadget ciphertexts overlap one another"); return -1; }
    for (const u64* p : d)
        for (const auto& in : inputs)
            if (in.first && overlaps(p, kb, in.first, in.second)) { set_error("a gadget ciphertext overlaps an input"); return -1; }
    return 0;
}

static GadgetEncLayout layout_of(const GadgetCt& g, size_t N) {
    const size_t es = (size_t)2 * (g.levelQ + 1 + g.levelP + 1) * N;
    return GadgetEncLayout{g.levelQ, g.levelP, g.pw2, g.ndigits, g.npw2max, g.pw2_sizes, es, es, true};
}

// components 0 and 1 of a key written in place (component 1 holds the uniform polynomial on entry, or is drawn)
static GadgetEncCt in_place(const GadgetCt& g, size_t N, const u64* s, u64 gal_el, const u64* pt, int target) {
    u64* d = const_cast<u64*>(g.data);
    u64* c1 = d + (size_t)(g.levelQ + 1 + g.levelP + 1) * N;
    return GadgetEncCt{d, c1, c1, s, gal_el, pt, target};
}

}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_rgsw_encrypt(lgpu_ctx* ctx, const uint64_t* sk, const uint64_t* pts, int n_pt, const int* pt_index, int is_ntt, int is_montgomery,
                      const int64_t* e, const lgpu_gadget_ct* value0, const lgpu_gadget_ct* value1, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "RGSW encryption is not supported on the ConjugateInvariant ring");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of [1, 65535]");
    REQUIRE(sk && e && value0 && value1, "null argument");
    REQUIRE(!pts || (n_pt >= 1 && n_pt <= 65535 && pt_index), "plaintexts need n_pt in [1, 65535] and a plaintext index per ciphertext");
    for (int b = 0; pts && b < batch; b++) REQUIRE(pt_index[b] >= 0 && pt_index[b] < n_pt, "pt_index out of [0, n_pt)");
    const size_t N = c.N, sk_bytes = ((size_t)c.nQ + c.nP) * N * 8;
    const lgpu_gadget_ct* arrays[2] = {value0, value1};
    std::vector<GadgetCt> g;
    // the error size needs the layout, so the overlap check against e follows it
    if (check_keys(c, arrays, 2, batch, g, {{sk, sk_bytes}})) return -1;
    const int nq = g[0].levelQ + 1;
    const size_t entries = (size_t)g[0].ndigits * g[0].npw2max, e_bytes = (size_t)batch * 2 * entries * N * 8,
                 pt_bytes = pts ? (size_t)n_pt * nq * N * 8 : 0, kb = key_bytes(g[0], N);
    for (const GadgetCt& k : g)
        REQUIRE(!overlaps(k.data, kb, e, e_bytes) && (!pts || !overlaps(k.data, kb, pts, pt_bytes)), "a gadget ciphertext overlaps an input");
    REQUIRE_DEVICE(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    // the plaintexts in the NTT domain and Montgomery form (encryptor.go:47-60)
    Scratch buf;
    const u64* pt = (const u64*)pts;
    if (pts && !(is_ntt && is_montgomery)) {
        if (buf.alloc((size_t)n_pt * nq * N, st)) return -1;
        const RowMap rq = rows_range(0, 0, nq);
        CSpan src{(const u64*)pts, N, (size_t)nq * N};
        if (!is_ntt) {
            if (launch_ntt(&c, rq, src, Span{buf.p, N, (size_t)nq * N}, n_pt, NTT_CANONICAL, st)) return -1;
            src = CSpan{buf.p, N, (size_t)nq * N};
        }
        if (!is_montgomery && launch_vecop(&c, rq, LGPU_OP_MFORM, src, CSpan{nullptr, 0, 0}, Span{buf.p, N, (size_t)nq * N}, n_pt, nullptr, nullptr, 0, 0,
                                           c.N, st)) return -1;
        pt = buf.p;
    }
    std::vector<GadgetEncCt> cts((size_t)2 * batch);
    for (int b = 0; b < batch; b++)
        for (int v = 0; v < 2; v++)
            cts[(size_t)2 * b + v] = in_place(g[(size_t)v * batch + b], N, (const u64*)sk, 0, pts ? pt + (size_t)pt_index[b] * nq * N : nullptr, v);
    return gadget_encrypt(&c, layout_of(g[0], N), cts.data(), 2 * batch, (const long long*)e, nullptr, st);
}

int lgpu_gen_galois_keys(lgpu_ctx* ctx, const uint64_t* sk, const uint64_t* gal_els, int n_keys, const int64_t* e, const lgpu_gadget_ct* keys,
                         void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "Galois key generation is not supported on the ConjugateInvariant ring");
    REQUIRE(n_keys >= 1 && n_keys <= 65535, "n_keys out of [1, 65535]");
    REQUIRE(sk && gal_els && e && keys, "null argument");
    for (int k = 0; k < n_keys; k++) REQUIRE((gal_els[k] & 1) && gal_els[k] < (uint64_t)c.nthroot, "Galois elements are odd and below 2N");
    const size_t N = c.N;
    std::vector<GadgetCt> g;
    if (check_keys(c, &keys, 1, n_keys, g, {{sk, ((size_t)c.nQ + c.nP) * N * 8}})) return -1;
    const size_t entries = (size_t)g[0].ndigits * g[0].npw2max, kb = key_bytes(g[0], N);
    for (const GadgetCt& k : g) REQUIRE(!overlaps(k.data, kb, e, (size_t)n_keys * entries * N * 8), "a gadget ciphertext overlaps an input");
    REQUIRE_DEVICE(ctx);
    std::vector<GadgetEncCt> cts((size_t)n_keys);
    for (int k = 0; k < n_keys; k++) {
        cts[k] = in_place(g[k], N, (const u64*)sk, gal_els[k], (const u64*)sk, 0);
        cts[k].c1_out = nullptr;        // component 1 stays the uniform polynomial
    }
    return gadget_encrypt(&c, layout_of(g[0], N), cts.data(), n_keys, (const long long*)e, nullptr, (cudaStream_t)stream);
}

int lgpu_blind_rotation_gen_evaluation_key(lgpu_ctx* ctx, const uint64_t* sk, const int64_t* s_lwe, int n_lwe, int window_size, double sigma,
                                           double bound, uint64_t seed, const lgpu_gadget_ct* brk0, const lgpu_gadget_ct* brk1,
                                           const lgpu_gadget_ct* gks, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "blind-rotation keys are not supported on the ConjugateInvariant ring");
    REQUIRE(n_lwe >= 1 && n_lwe <= 32767, "n_lwe out of [1, 32767]");
    REQUIRE(window_size >= 1 && (uint64_t)window_size < c.nthroot / 4, "window_size out of [1, N/2)");
    REQUIRE(sigma > 0.0 && bound >= 1.0 && bound < 9.0e18, "gaussian sampler: sigma / bound out of range");
    REQUIRE(sk && s_lwe && brk0 && brk1 && gks, "null argument");
    const size_t N = c.N;
    const lgpu_gadget_ct* arrays[2] = {brk0, brk1};
    std::vector<GadgetCt> g, gk;
    const std::vector<std::pair<const void*, size_t>> in{{sk, ((size_t)c.nQ + c.nP) * N * 8}};
    if (check_keys(c, arrays, 2, n_lwe, g, in) || check_keys(c, &gks, 1, window_size + 1, gk, in)) return -1;
    REQUIRE(same_layout(g[0], gk[0]), "Galois keys and RGSW ciphertexts differ in levels or digit layout");
    const size_t kb = key_bytes(g[0], N);
    {
        std::vector<const u64*> d;
        for (const GadgetCt& k : g) d.push_back(k.data);
        for (const GadgetCt& k : gk) d.push_back(k.data);
        std::sort(d.begin(), d.end());
        for (size_t k = 1; k < d.size(); k++) REQUIRE(!overlaps(d[k - 1], kb, d[k], kb), "gadget ciphertexts overlap one another");
    }
    REQUIRE_DEVICE(ctx);
    cudaStream_t st = (cudaStream_t)stream;
    const int nq = g[0].levelQ + 1;
    // the distinct monomials X^{s_i} (ring.NewMonomialXi, ring/ring.go:374-396), NTT, MForm
    std::vector<long long> vals(s_lwe, s_lwe + n_lwe);
    std::sort(vals.begin(), vals.end());
    vals.erase(std::unique(vals.begin(), vals.end()), vals.end());
    const int n_pt = (int)vals.size();
    std::vector<u64> hm((size_t)n_pt * nq * N, 0);
    const long long twoN = 2 * (long long)N;
    for (int t = 0; t < n_pt; t++) {
        long long k = vals[t] & (twoN - 1);
        if (k >= (long long)N) k -= twoN;
        for (int r = 0; r < nq; r++) {
            if (k < 0) hm[((size_t)t * nq + r) * N + (size_t)(N + k)] = c.Q[r] - 1;
            else hm[((size_t)t * nq + r) * N + (size_t)k] = 1;
        }
    }
    Scratch mono;
    if (mono.alloc(hm.size(), st)) return -1;
    LGPU_CUDA_OK(cudaMemcpyAsync(mono.p, hm.data(), hm.size() * sizeof(u64), cudaMemcpyHostToDevice, st));   // pageable: staged before return
    const RowMap rq = rows_range(0, 0, nq);
    const Span ms{mono.p, N, (size_t)nq * N};
    if (launch_ntt(&c, rq, CSpan{mono.p, N, (size_t)nq * N}, ms, n_pt, NTT_CANONICAL, st)) return -1;
    if (launch_vecop(&c, rq, LGPU_OP_MFORM, CSpan{mono.p, N, (size_t)nq * N}, CSpan{nullptr, 0, 0}, ms, n_pt, nullptr, nullptr, 0, 0, c.N, st)) return -1;
    // ciphertext m = 2 i + v is Value[v] of RGSW i, ciphertext 2 n_lwe + t the Galois key of galEls[t]; m draws on stream id m
    std::vector<GadgetEncCt> cts;
    cts.reserve((size_t)2 * n_lwe + window_size + 1);
    for (int i = 0; i < n_lwe; i++) {
        const size_t t = (size_t)(std::lower_bound(vals.begin(), vals.end(), (long long)s_lwe[i]) - vals.begin());
        for (int v = 0; v < 2; v++) cts.push_back(in_place(g[(size_t)v * n_lwe + i], N, (const u64*)sk, 0, mono.p + t * nq * N, v));
    }
    for (int t = 0; t <= window_size; t++) {       // GaloisElement(1..window), then NthRoot - GaloisGen (keys.go:91-97)
        const u64 gal = t < window_size ? galois_element(&c, t + 1) : c.nthroot - 5;
        cts.push_back(in_place(gk[t], N, (const u64*)sk, gal, (const u64*)sk, 0));
    }
    const GadgetEncDraw draw{seed, 0, sigma, bound};
    return gadget_encrypt(&c, layout_of(g[0], N), cts.data(), (int)cts.size(), nullptr, &draw, st);
}

}  // extern "C"

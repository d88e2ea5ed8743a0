// capi3.cu -- extern "C" entry points of the rows that sit right above the key-switch path (SURVEY 8(f)): hoisted linear
// transformations (lintrans.cu).
#include <map>
#include <vector>
#include "capi_common.h"
#include "composite.h"
#include "lintrans.h"

using namespace lgpu;

static inline cudaStream_t S(void* stream) { return (cudaStream_t)stream; }

extern "C" {

uint64_t lgpu_galois_element(lgpu_ctx* ctx, long long k) {
    if (!ctx) return 0;
    return galois_element(&ctx->c, k);
}

int lgpu_lintrans_evaluate_many(lgpu_ctx* ctx, int level_in, const uint64_t* ct_in, const lgpu_lintrans* mats, int n_mats,
                                const lgpu_galois_keys* gks, uint64_t* const* ct_outs, int* out_levels, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct_in && mats && ct_outs && out_levels, "null argument");
    REQUIRE(n_mats >= 1, "output *rlwe.Ciphertext slice is too small");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE_ALIGNED(AL(ct_in));
    GaloisKeySet ks;
    if (gks) {
        if (to_galois_keys(gks, ks)) return -1;
        for (const GadgetCt& k : ks.keys) REQUIRE(k.pw2 == 0, "hoisted linear transformations need keys with BaseTwoDecomposition = 0");
    }
    std::vector<LinTransView> mv(n_mats);
    for (int i = 0; i < n_mats; i++) {
        const lgpu_lintrans& m = mats[i];
        mv[i] = LinTransView{m.level_q, m.level_p, m.log_slots, m.n1, m.n_diags, m.diag_index, (const u64* const*)m.diag};
        REQUIRE(ct_outs[i], "output slice contains unallocated ciphertext");
        REQUIRE_ALIGNED(AL(ct_outs[i]));
        for (int d = 0; d < m.n_diags; d++) {
            REQUIRE(m.diag && m.diag[d], "null diagonal");
            REQUIRE_ALIGNED(AL(m.diag[d]));
        }
    }
    return lintrans_evaluate_many(&ctx->c, level_in, (const u64*)ct_in, mv.data(), n_mats, ks, (u64* const*)ct_outs, out_levels, batch, S(stream));
}

int lgpu_rgsw_external_product(lgpu_ctx* ctx, const uint64_t* ct_in, int level_in, const lgpu_gadget_ct* rgsw0, const lgpu_gadget_ct* rgsw1,
                               uint64_t* ct_out, int level_out, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    GadgetCt g0, g1;
    if (to_gadget_ct(rgsw0, g0) || to_gadget_ct(rgsw1, g1)) return -1;
    REQUIRE(g0.levelQ >= 0 && g0.levelQ <= level_in && g0.levelQ <= level_out, "RGSW ciphertext level above the RLWE ciphertexts' level");
    const size_t N = ctx->c.N, ci = (size_t)(level_in + 1) * N, co = (size_t)(level_out + 1) * N;
    const u64* in = (const u64*)ct_in;
    u64* out = (u64*)ct_out;
    return rgsw_external_product(&ctx->c, g0, g1, CSpan{in, N, 2 * ci}, CSpan{in + ci, N, 2 * ci}, Span{out, N, 2 * co}, Span{out + co, N, 2 * co}, batch,
                                 S(stream));
}

// blindrot.Evaluator.BlindRotateCore (core/rgsw/blindrot/evaluator.go:144-203) + evaluateFromDiscreteLogSets (:206-229) +
// getGaloisElementInverseMap / getDiscreteLogSets (:232-283): Algorithm 3 of eprint 2022/198 on one accumulator. The control flow is driven by the
// LWE mask `a` (HOST, values modulo 2N, odd or zero); every step is an evaluator call that is already on the device (Evaluator.Automorphism with the
// window keys, rgsw ExternalProduct with RGSW(X^{s_j})), in place on `acc`.
int lgpu_blind_rotate_core(lgpu_ctx* ctx, const uint64_t* a_host, int n_lwe, uint64_t* acc, int level, const lgpu_gadget_ct* brk0, const lgpu_gadget_ct* brk1,
                           const lgpu_galois_keys* gks, int window_size, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(a_host && acc && brk0 && brk1 && gks && n_lwe >= 1, "null argument");
    REQUIRE_ALIGNED(AL(acc));
    REQUIRE(window_size >= 1, "window size must be positive");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "blind rotation is defined on the standard ring");
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    const long long N = c.N, twoN = 2 * N, Nhalf = N >> 1;
    // map[(+/-) g^k mod 2N] = +/- k   (:232-258)
    std::vector<long long> dlog((size_t)twoN, 0);
    std::vector<char> has((size_t)twoN, 0);
    {
        unsigned long long pw = 1;
        for (long long i = 0; i < Nhalf; i++) {
            dlog[pw] = i; has[pw] = 1;
            dlog[(size_t)(twoN - (long long)pw)] = -i; has[(size_t)(twoN - (long long)pw)] = 1;
            pw = pw * 5 & (unsigned long long)(twoN - 1);
        }
    }
    // discrete-log sets of a (:261-283); Go's map lookup of a[i] = 0 yields the zero value 0
    std::map<long long, std::vector<int>> sets;
    for (int i = 0; i < n_lwe; i++) {
        const unsigned long long ai = a_host[i];
        REQUIRE(ai < (unsigned long long)twoN, "blind rotation: a[i] is not reduced modulo 2N");
        REQUIRE((ai & 1) == 1 || ai == 0, "getDiscreteLogSets: a[i] is not odd and thus not an element of Z_{2N}^{*} -> a[i] = (+/- 1) * g^{k} does not exist.");
        sets[has[ai] ? dlog[ai] : 0].push_back(i);
    }
    GaloisKeySet ks;
    if (to_galois_keys(gks, ks)) return -1;
    const size_t nq = level + 1, cs = nq * (size_t)N;
    u64* A = (u64*)acc;
    cudaStream_t st = S(stream);
    auto automorph = [&](long long k) -> int {     // eval.Automorphism(acc, GaloisElement(k), acc)
        const u64 g = galois_element(&c, k);
        const GadgetCt* gk = ks.find(g);
        if (!gk) return -1;
        return evaluator_automorphism(&c, level, CSpan{A, (size_t)N, 2 * cs}, CSpan{A + cs, (size_t)N, 2 * cs}, g, *gk, Span{A, (size_t)N, 2 * cs},
                                      Span{A + cs, (size_t)N, 2 * cs}, nullptr, 1, st);
    };
    auto from_sets = [&](long long k, int v, int& vout) -> int {
        auto it = sets.find(k);
        if (it != sets.end()) {
            if (v != 0) { if (automorph(v)) return -1; v = 0; }
            for (int j : it->second) {
                GadgetCt g0, g1;
                if (to_gadget_ct(&brk0[j], g0) || to_gadget_ct(&brk1[j], g1)) return -1;
                if (rgsw_external_product(&c, g0, g1, CSpan{A, (size_t)N, 2 * cs}, CSpan{A + cs, (size_t)N, 2 * cs}, Span{A, (size_t)N, 2 * cs},
                                          Span{A + cs, (size_t)N, 2 * cs}, 1, st)) return -1;
            }
        }
        v++;
        if (v == window_size || k == 1) { if (automorph(v)) return -1; v = 0; }
        vout = v;
        return 0;
    };
    int v = 0, dummy = 0;
    for (long long i = Nhalf - 1; i > 0; i--) if (from_sets(-i, v, v)) return -1;          // lines 3-9
    if (from_sets(twoN, 0, dummy)) return -1;                                              // line 10 (never in the sets: 2N is not a residue)
    {                                                                                      // line 12: acc = acc(X^{-g})
        const u64 g = c.nthroot - 5;
        const GadgetCt* gk = ks.find(g);
        if (!gk) return -1;
        if (evaluator_automorphism(&c, level, CSpan{A, (size_t)N, 2 * cs}, CSpan{A + cs, (size_t)N, 2 * cs}, g, *gk, Span{A, (size_t)N, 2 * cs},
                                   Span{A + cs, (size_t)N, 2 * cs}, nullptr, 1, st)) return -1;
    }
    for (long long i = Nhalf - 1; i > 0; i--) if (from_sets(i, v, v)) return -1;           // lines 13-19
    if (from_sets(0, 0, dummy)) return -1;                                                 // lines 20-21
    return 0;
}

int lgpu_evaluator_automorphism_hoisted_lazy(lgpu_ctx* ctx, int level_q, const uint64_t* ct0, const uint64_t* decomp, int decomp_level_q,
                                             uint64_t gal_el, const lgpu_gadget_ct* gk, uint64_t* out0q, uint64_t* out0p, uint64_t* out1q,
                                             uint64_t* out1p, int batch, size_t stride_ct, size_t stride_q, size_t stride_p, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct0 && decomp && out0q && out0p && out1q && out1p, "null polynomial");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE_ALIGNED(AL(ct0) && AL(decomp) && AL(out0q) && AL(out0p) && AL(out1q) && AL(out1p) && ((stride_ct | stride_q | stride_p) & 1) == 0);
    GadgetCt g;
    if (to_gadget_ct(gk, g)) return -1;
    const Ctx& c = ctx->c;
    REQUIRE(level_q >= 0 && level_q < c.nQ && level_q <= g.levelQ, "levelQ out of range");
    REQUIRE(g.levelP >= 0 && g.levelP < c.nP, "AutomorphismHoistedLazy requires a P ring");
    if (decomp_level_q < 0) decomp_level_q = level_q;
    const size_t N = c.N, nq = level_q + 1;
    // ctIn.Value[0] * P (ringQ.MulScalarBigint, evaluator_automorphism.go:150-156)
    const std::vector<u64> pq = p_mod_q_mont(&c, level_q, g.levelP);
    Scratch buf;
    if (buf.alloc((size_t)batch * nq * N, S(stream))) return -1;
    if (launch_vecop(&c, rows_range(0, 0, (int)nq), LGPU_OP_MULSCALARMONTGOMERY, CSpan{(const u64*)ct0, N, stride_ct}, CSpan{nullptr, 0, 0},
                     Span{buf.p, N, nq * N}, batch, pq.data(), nullptr, 0, 0, c.N, S(stream))) return -1;
    AccSpans out;
    out.q[0] = Span{(u64*)out0q, N, stride_q}; out.q[1] = Span{(u64*)out1q, N, stride_q};
    out.p[0] = Span{(u64*)out0p, N, stride_p}; out.p[1] = Span{(u64*)out1p, N, stride_p};
    return automorphism_hoisted_lazy(&c, level_q, CSpan{buf.p, N, nq * N}, (const u64*)decomp, decomp_level_q, gal_el, g, out, batch, S(stream));
}

}  // extern "C"

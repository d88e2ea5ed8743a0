// innersum.cu -- slot aggregation on the device, for a BATCH of ciphertexts sharing one set of Galois keys:
//   rlwe.Evaluator.PartialTracesSum   core/rlwe/inner_sum.go:147-292   (InnerSum / RotateAndAdd / Replicate / Average)
//   rlwe.Evaluator.Trace              core/rlwe/inner_sum.go:36-116
// Same key-switch schedule as the reference (log2(n) + HW(n) - 1 key switches, one DecomposeNTT per doubling step, the
// non-power-of-two terms accumulated mod QP and divided by P once). Two epilogues are fused:
//   - each doubling / Trace step (Add + 2 x AutomorphismNTTWithIndex + 2 x Add) is ONE auto_add_kernel pass;
//   - each non-first lazy term (AutomorphismHoistedLazy + 2 x ringQP.Add) is one lt_hoisted_auto_kernel<Acc = true> pass.
// Every output is a canonical residue that depends on its inputs only through residue classes, so the results equal the
// reference bit for bit (DESIGN 3.4; tests/test_gpu_innersum.py vs oracle/innersum.py).
#include <algorithm>
#include <cstring>
#include <vector>
#include "capi_common.h"
#include "composite.h"
#include "lintrans.h"
#include "modarith.cuh"

namespace lgpu {

// ---------------------------------------------------------------------------------------------------------------------
// kernel
// ---------------------------------------------------------------------------------------------------------------------
struct AutoAddParams {
    const LimbConst* limbs;
    const u64* in; size_t in_cs;           // X: [batch][2][.][N], component stride in_cs, batch stride 2 * in_cs
    const u64* t; size_t t_cs, t_bs;       // GadgetProduct(X[1]) after ModDown: [2][batch][nq][N]
    u64* out; size_t out_cs;               // same layout as X, must not alias it (the gather reads X at other positions)
    u64 galEl, mask;                       // Galois element, NthRoot - 1
    int lg, n;                             // log2(NthRoot / 2), N
};
// X + phi(X) with phi = Automorphism(., galEl) of the key-switched X (Evaluator.Automorphism[Hoisted] + ringQ.Add, inner_sum.go:277-281,
// :85-90):   out0[j] = X0[j] + (t0 + X0)[idx j],   out1[j] = X1[j] + t1[idx j],   idx = AutomorphismNTTIndex(galEl)[j] (computed in place)
__global__ void __launch_bounds__(256) auto_add_kernel(AutoAddParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const int r = blockIdx.y;
    const u64 q = p.limbs[r].q;
    const u64 tmp1 = 2 * (__brevll((u64)j) >> (64 - p.lg)) + 1;           // ring/automorphism.go:12-34
    const size_t idx = (size_t)(__brevll(((p.galEl * tmp1 & p.mask) - 1) >> 1) >> (64 - p.lg));
    const size_t b = blockIdx.z, ro = (size_t)r * p.n;
    const u64* x0 = p.in + b * 2 * p.in_cs + ro;
    const u64* x1 = x0 + p.in_cs;
    const u64* t0 = p.t + b * p.t_bs + ro;
    const u64* t1 = t0 + p.t_cs;
    u64* o0 = p.out + b * 2 * p.out_cs + ro;
    u64* o1 = o0 + p.out_cs;
    o0[j] = cred(x0[j] + cred(t0[idx] + x0[idx], q), q);
    o1[j] = cred(x1[j] + t1[idx], q);
}

namespace {

// Every Block below is a batch of degree-1 ciphertexts, [batch][2][.][N]: bs = 2 * cs.
int auto_add(const Ctx* c, int nq, Block in, const u64* t, int nb, Block out, u64 galEl, cudaStream_t st) {
    if (in.p == out.p) { set_error("auto_add: the output must not alias the input"); return -1; }
    AutoAddParams p;
    int lg = 0;
    while ((1ull << (lg + 1)) < c->nthroot) lg++;
    p.limbs = c->d_limbs; p.in = in.p; p.in_cs = in.cs;
    p.t = t; p.t_bs = (size_t)nq * c->N; p.t_cs = (size_t)nb * nq * c->N;
    p.out = out.p; p.out_cs = out.cs; p.galEl = galEl; p.mask = c->nthroot - 1; p.lg = lg; p.n = c->N;
    ProfScope ps(LGPU_KCLASS_AUTOMORPHISM, st, 8.0 * c->N * nq * nb * 6, 1);
    auto_add_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, (unsigned)nb), 256, 0, st>>>(p);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// rows 0..nq-1 of both components, nb ciphertexts (2 * nb row blocks): NTT / INTT / copy between two ciphertext layouts
int ntt_ct(const Ctx* c, bool inverse, int nq, Block in, Block out, int nb, cudaStream_t st) {
    const RowMap rm = rows_range(0, 0, nq);
    const CSpan i{in.p, (size_t)c->N, in.cs};
    const Span o{out.p, (size_t)c->N, out.cs};
    return inverse ? launch_intt(c, rm, i, o, 2 * nb, NTT_CANONICAL, st) : launch_ntt(c, rm, i, o, 2 * nb, NTT_CANONICAL, st);
}
int copy_ct(const Ctx* c, int nq, Block in, Block out, int nb, cudaStream_t st) {
    if (in.p == out.p) return 0;
    LGPU_CUDA_OK(cudaMemcpy2DAsync(out.p, out.cs * 8, in.p, in.cs * 8, (size_t)nq * c->N * 8, (size_t)2 * nb, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// The schedule of PartialTracesSum (inner_sum.go:217-283) for n >= 2: per iteration i < top bit of n, the optional lazy term
// (k = (n - (n mod 2^(i+1))) * offset, when bit i of n is set) and the doubling rotation 2^i * offset.
struct PtsStep { bool lazy; long long k; long long dbl; };
std::vector<PtsStep> pts_schedule(int offset, int n) {
    std::vector<PtsStep> s;
    for (int i = 0, j = n; j > 1; i++, j >>= 1) {
        PtsStep st;
        st.lazy = (j & 1) != 0;
        st.k = (long long)(n - (n & ((2 << i) - 1))) * offset;
        st.dbl = (1ll << i) * offset;
        s.push_back(st);
    }
    return s;
}

// Trace's Galois elements in order (inner_sum.go:83-101); empty when gap <= 1 (a copy)
std::vector<u64> trace_elements(const Ctx* c, int log_n) {
    std::vector<u64> g;
    const int gap_log = c->logN - log_n - 1 + (log_n == 0 ? 1 : 0);
    if (gap_log <= 0) return g;
    for (int i = log_n; i < c->logN - 1; i++) g.push_back(galois_element(c, 1ll << i));
    if (log_n == 0) g.push_back(c->nthroot - 1);
    return g;
}

int pts_chunk(const Ctx* c, int level, Block in, bool is_ntt, int offset, int n, const std::vector<const GadgetCt*>& lazy_keys,
              const std::vector<const GadgetCt*>& dbl_keys, Block out, int nb, cudaStream_t st) {
    const int nq = level + 1;
    const size_t N = c->N, ctw = (size_t)2 * nb * nq * N;
    if (n == 1) {
        // opOut is a copy of ctIn in its own domain; for a coefficient-domain input the trailing INTT still runs on it (:179-183, :286-289)
        if (is_ntt) return copy_ct(c, nq, in, out, nb, st);
        return ntt_ct(c, true, nq, in, out, nb, st);
    }
    const int levelP = c->nP - 1, np = levelP + 1;
    const std::vector<PtsStep> sched = pts_schedule(offset, n);
    const int d = (int)sched.size();
    bool any_lazy = false;
    for (const PtsStep& s : sched) any_lazy |= s.lazy;
    const int nd = base_rns_decomposition_vector_size(level, levelP);
    const size_t dec_w = (size_t)nd * nb * (nq + np) * N, acc_w = any_lazy ? (size_t)2 * nb * (nq + np) * N : 0, c0p_w = any_lazy ? (size_t)nb * nq * N : 0;
    // ping-pong: X_d lands in `out`; every step reads X_i and writes X_{i+1} != X_i. Buffers: out, B0, and B1 only when an in-place
    // call with an odd number of steps >= 3 needs a third one. X_0 is the input itself for an NTT-domain input (copied only when
    // in == out and one step would write over it), or the NTT of the input.
    enum { OUT, IN, B0, B1 };
    auto same = [&](int a, int b) { return a == b || (((a == OUT && b == IN) || (a == IN && b == OUT)) && in.p == out.p); };
    std::vector<int> tag(d + 1);
    tag[d] = OUT;
    for (int s = d - 1; s >= 1; s--)
        for (int x : {OUT, B0, B1})
            if (!same(x, tag[s + 1]) && !(s == 1 && is_ntt && same(x, IN))) { tag[s] = x; break; }
    bool copy_in = false;
    if (is_ntt) {
        tag[0] = IN;
        if (same(tag[1], IN)) { tag[0] = B0; copy_in = true; }
    } else {
        for (int x : {OUT, B0, B1}) if (!same(x, tag[1])) { tag[0] = x; break; }
    }
    const int nbuf = std::find(tag.begin(), tag.end(), (int)B1) != tag.end() ? 2 : std::find(tag.begin(), tag.end(), (int)B0) != tag.end() ? 1 : 0;
    Scratch buf;
    if (buf.alloc(dec_w + acc_w + c0p_w + ctw /* t */ + nbuf * ctw /* B0, B1 */, st)) return -1;
    u64* decomp = buf.p; u64* accb = decomp + dec_w; u64* c0p = accb + acc_w; u64* t = c0p + c0p_w;
    const Block bufs[4] = {out, in, Block{t + ctw, (size_t)nq * N, (size_t)2 * nq * N}, Block{t + 2 * ctw, (size_t)nq * N, (size_t)2 * nq * N}};
    std::vector<Block> X(d + 1);
    for (int s = 0; s <= d; s++) X[s] = bufs[tag[s]];
    if (copy_in && copy_ct(c, nq, in, X[0], nb, st)) return -1;
    if (!is_ntt && ntt_ct(c, false, nq, in, X[0], nb, st)) return -1;
    const AccSpans acc = stacked_acc(accb, nq, np, N, nb);
    const std::vector<u64> pq = p_mod_q_mont(c, level, levelP);
    bool first = true;
    for (int i = 0; i < d; i++) {
        const Block x = X[i];
        // DecomposeNTT(ctInNTT[1]) once per doubling step; the reference also decomposes in the last iteration, whose result it never reads
        if (decompose_ntt(c, level, levelP, levelP + 1, CSpan{x.p + x.cs, N, x.bs}, true, decomp, nb, st)) return -1;
        if (sched[i].lazy) {
            // accQP (+)= AutomorphismHoistedLazy(ctInNTT, k); P * ctInNTT[0] is its Q-row addend (evaluator_automorphism.go:150-156)
            if (launch_vecop(c, rows_range(0, 0, nq), LGPU_OP_MULSCALARMONTGOMERY, CSpan{x.p, N, x.bs}, CSpan{nullptr, 0, 0}, Span{c0p, N, (size_t)nq * N},
                             nb, pq.data(), nullptr, 0, 0, c->N, st)) return -1;
            if (automorphism_hoisted_lazy(c, level, CSpan{c0p, N, (size_t)nq * N}, decomp, level, galois_element(c, sched[i].k), *lazy_keys[i], acc, nb, st, !first))
                return -1;
            first = false;
        }
        // ctInNTT = ctInNTT + AutomorphismHoisted(ctInNTT, 2^i * offset)
        if (gadget_product_hoisted(c, level, decomp, *dbl_keys[i], Span{t, N, (size_t)nq * N}, Span{t + (size_t)nb * nq * N, N, (size_t)nq * N}, nb, st))
            return -1;
        if (auto_add(c, nq, x, t, nb, X[i + 1], galois_element(c, sched[i].dbl), st)) return -1;
    }
    if (n & (n - 1)) {
        // opOut = ModDown(accQP) + ctInNTT (:256-263); X[d] is `out`, so the addend is read and written in place
        if (moddown_ntt(c, level, levelP, CBlock{accb, (size_t)nb * (nq + np) * N, (nq + np) * N}, out, out, 2, nb, st)) return -1;
    }
    if (!is_ntt) return ntt_ct(c, true, nq, out, out, nb, st);
    return 0;
}

int trace_chunk(const Ctx* c, int level, Block in, bool is_ntt, int log_n, const std::vector<const GadgetCt*>& keys, const std::vector<u64>& els,
                Block out, int nb, cudaStream_t st) {
    const int nq = level + 1;
    const size_t N = c->N;
    const int S = (int)els.size();
    if (S == 0) return copy_ct(c, nq, in, out, nb, st);        // gap <= 1: opOut.Copy(ctIn)
    Scratch buf;
    if (buf.alloc((size_t)4 * nb * nq * N, st)) return -1;
    u64* t = buf.p;
    const Block B{buf.p + (size_t)2 * nb * nq * N, (size_t)nq * N, (size_t)2 * nq * N};
    auto X = [&](int s) { return ((S - s) & 1) ? B : out; };    // X_S = out
    // pre-multiplication by gap^-1 mod Q_level (ringQ.MulScalarBigint, canonical per limb), then NTT for a coefficient-domain input
    const int gap_log = c->logN - log_n - 1 + (log_n == 0 ? 1 : 0);
    std::vector<u64> sc(nq);
    for (int i = 0; i < nq; i++) sc[i] = h_mform(h_invmod(((u64)1 << gap_log) % c->Q[i], c->Q[i]), c->Q[i]);
    const Block x0 = X(0);
    if (launch_vecop(c, rows_range(0, 0, nq), LGPU_OP_MULSCALARMONTGOMERY, CSpan{in.p, N, in.cs}, CSpan{nullptr, 0, 0}, Span{x0.p, N, x0.cs}, 2 * nb, sc.data(),
                     nullptr, 0, 0, c->N, st)) return -1;
    if (!is_ntt && ntt_ct(c, false, nq, x0, x0, nb, st)) return -1;
    for (int s = 1; s <= S; s++) {
        const Block x = X(s - 1);
        // opOut += Automorphism(opOut, g) (:85-101)
        if (gadget_product(c, level, CSpan{x.p + x.cs, N, x.bs}, *keys[s - 1], Span{t, N, (size_t)nq * N}, Span{t + (size_t)nb * nq * N, N, (size_t)nq * N},
                           nb, st)) return -1;
        if (auto_add(c, nq, x, t, nb, X(s), els[s - 1], st)) return -1;
    }
    if (!is_ntt) return ntt_ct(c, true, nq, out, out, nb, st);
    return 0;
}

// every key the call will use, looked up and checked before any device work (the reference fails at the first missing key instead)
int lookup(const Ctx* c, const GaloisKeySet& ks, int level, u64 g, bool max_levelP, const GadgetCt*& out) {
    out = ks.find(g);
    if (!out) return -1;
    if (check_gk(c, level, *out)) return -1;
    if (max_levelP && out->levelP != c->nP - 1) {
        set_error("PartialTracesSum: Galois key levelP must be the parameters' MaxLevelP (the decomposition uses PCount() - 1)");
        return -1;
    }
    return 0;
}

}  // namespace
}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_evaluator_partial_traces_sum(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int is_ntt, int offset, int n, const lgpu_galois_keys* gks,
                                      uint64_t* ct_out, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    REQUIRE(n > 0 && offset != 0, "partialtrace: invalid parameter (n = 0 or batchSize = 0)");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "PartialTracesSum is not supported on the ConjugateInvariant ring");
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(is_ntt == 0 || is_ntt == 1, "is_ntt must be 0 or 1");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    const size_t bytes = (size_t)batch * 2 * (level + 1) * c.N * 8;
    REQUIRE(ct_out == ct_in || !overlaps(ct_out, bytes, ct_in, bytes), "ct_out overlaps ct_in (only ct_out == ct_in is allowed)");
    std::vector<const GadgetCt*> lazy_keys, dbl_keys;
    GaloisKeySet ks;
    if (n >= 2) {
        REQUIRE(c.nP >= 1, "PartialTracesSum requires a P ring");
        if (to_galois_keys(gks, ks)) return -1;
        for (const PtsStep& s : pts_schedule(offset, n)) {
            const GadgetCt* g = nullptr;
            if (s.lazy && lookup(&c, ks, level, galois_element(&c, s.k), true, g)) return -1;
            lazy_keys.push_back(g);
            if (lookup(&c, ks, level, galois_element(&c, s.dbl), true, g)) return -1;
            dbl_keys.push_back(g);
        }
    }
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    const size_t cs = (size_t)(level + 1) * c.N;
    const int ch = batch_chunk();
    for (int k = 0; k < batch; k += ch) {
        const int nb = std::min(ch, batch - k);
        const Block in{(u64*)ct_in + (size_t)k * 2 * cs, cs, 2 * cs}, out{(u64*)ct_out + (size_t)k * 2 * cs, cs, 2 * cs};
        if (pts_chunk(&c, level, in, is_ntt != 0, offset, n, lazy_keys, dbl_keys, out, nb, st)) return -1;
    }
    return 0;
}

int lgpu_evaluator_trace(lgpu_ctx* ctx, int level_in, const uint64_t* ct_in, int is_ntt, int log_n, const lgpu_galois_keys* gks, uint64_t* ct_out,
                         int level_out, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(log_n >= 0 && log_n <= c.logN - 1, "Trace: logN out of range [0, LogN - 1]");
    REQUIRE(c.ring_type == 0, "Trace is not supported on the ConjugateInvariant ring");
    REQUIRE(level_in >= 0 && level_in < c.nQ && level_out >= 0 && level_out < c.nQ, "level out of range");
    REQUIRE(is_ntt == 0 || is_ntt == 1, "is_ntt must be 0 or 1");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    const size_t ib = (size_t)batch * 2 * (level_in + 1) * c.N * 8, ob = (size_t)batch * 2 * (level_out + 1) * c.N * 8;
    if (ct_out == ct_in) REQUIRE(level_in == level_out, "in-place Trace needs level_out == level_in");
    else REQUIRE(!overlaps(ct_out, ob, ct_in, ib), "ct_out overlaps ct_in (only ct_out == ct_in is allowed)");
    const int level = std::min(level_in, level_out);
    const std::vector<u64> els = trace_elements(&c, log_n);
    std::vector<const GadgetCt*> keys;
    GaloisKeySet ks;
    if (!els.empty()) {
        REQUIRE(c.nP >= 1, "Trace requires a P ring");
        if (to_galois_keys(gks, ks)) return -1;
        for (u64 g : els) {
            const GadgetCt* k = nullptr;
            if (lookup(&c, ks, level, g, false, k)) return -1;
            keys.push_back(k);
        }
    }
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    const size_t ci = (size_t)(level_in + 1) * c.N, co = (size_t)(level_out + 1) * c.N;
    const int ch = batch_chunk();
    for (int k = 0; k < batch; k += ch) {
        const int nb = std::min(ch, batch - k);
        const Block in{(u64*)ct_in + (size_t)k * 2 * ci, ci, 2 * ci}, out{(u64*)ct_out + (size_t)k * 2 * co, co, 2 * co};
        if (trace_chunk(&c, level, in, is_ntt != 0, log_n, keys, els, out, nb, st)) return -1;
    }
    return 0;
}

}  // extern "C"

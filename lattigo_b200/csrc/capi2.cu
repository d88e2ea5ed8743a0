// capi2.cu -- extern "C" entry points for automorphisms, basis extension, rescaling, the rlwe.Evaluator
// key-switch family and the fused CKKS batch ops (include/lattigo_b200.h).
#include <algorithm>
#include <mutex>
#include <cstring>
#include "capi_common.h"
#include "composite.h"

using namespace lgpu;



static inline cudaStream_t S(void* stream) { return (cudaStream_t)stream; }

static int check_levels(const Ctx& c, int lq, int lp, bool needP) {
    REQUIRE(lq >= 0 && lq < c.nQ, "levelQ out of range");
    if (needP) REQUIRE(lp >= 0 && lp < c.nP, "levelP out of range");
    return 0;
}

extern "C" {

int lgpu_automorphism_ntt_index(lgpu_ctx* ctx, uint64_t gal_el, uint64_t* index_out, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(index_out, "null index");
    return automorphism_ntt_index(&ctx->c, gal_el, (u64*)index_out, S(stream));
}
int lgpu_automorphism_ntt_with_index(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, const uint64_t* index, uint64_t* out,
                                     int accumulate, int batch, size_t bs, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(in && out && index, "null argument");
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    const size_t N = ctx->c.N;
    return automorphism_ntt_with_index(&ctx->c, level + 1, CSpan{(const u64*)in, N, bs}, (const u64*)index, Span{(u64*)out, N, bs},
                                       accumulate != 0, batch, S(stream));
}
int lgpu_automorphism_ntt(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t gal_el, uint64_t* out, int batch, size_t bs, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(in && out, "null argument");
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    const size_t N = ctx->c.N;
    u64* idx = nullptr;
    LGPU_CUDA_OK(cudaMallocAsync((void**)&idx, N * sizeof(u64), S(stream)));
    int rc = automorphism_ntt_index(&ctx->c, gal_el, idx, S(stream));
    if (!rc) rc = automorphism_ntt_with_index(&ctx->c, level + 1, CSpan{(const u64*)in, N, bs}, idx, Span{(u64*)out, N, bs}, false, batch, S(stream));
    cudaFreeAsync(idx, S(stream));
    return rc;
}
int lgpu_automorphism(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t gal_el, uint64_t* out, int batch, size_t bs, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(in && out, "null argument");
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    const size_t N = ctx->c.N;
    return automorphism_coeff(&ctx->c, rm, CSpan{(const u64*)in, N, bs}, gal_el, Span{(u64*)out, N, bs}, batch, S(stream));
}

int lgpu_modup_qtop(lgpu_ctx* ctx, int lq, int lp, const uint64_t* pq, uint64_t* pp, int batch, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(pq && pp, "null polynomial");
    const size_t N = ctx->c.N;
    return launch_modup_qp(&ctx->c, true, lq, lp, CSpan{(const u64*)pq, N, sq}, Span{(u64*)pp, N, sp}, batch, S(stream));
}
int lgpu_modup_ptoq(lgpu_ctx* ctx, int lp, int lq, const uint64_t* pp, uint64_t* pq, int batch, size_t sp, size_t sq, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(pq && pp, "null polynomial");
    const size_t N = ctx->c.N;
    return launch_modup_qp(&ctx->c, false, lq, lp, CSpan{(const u64*)pp, N, sp}, Span{(u64*)pq, N, sq}, batch, S(stream));
}
int lgpu_moddown_qp_to_q(lgpu_ctx* ctx, int lq, int lp, const uint64_t* p1q, const uint64_t* p1p, uint64_t* p2q, int batch, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(p1q && p1p && p2q, "null polynomial");
    if (check_levels(ctx->c, lq, lp, true)) return -1;
    const size_t N = ctx->c.N;
    return moddown_qp_to_q(&ctx->c, lq, lp, CSpan{(const u64*)p1q, N, sq}, CSpan{(const u64*)p1p, N, sp}, Span{(u64*)p2q, N, sq}, batch, S(stream));
}
int lgpu_moddown_qp_to_q_ntt(lgpu_ctx* ctx, int lq, int lp, const uint64_t* p1q, const uint64_t* p1p, uint64_t* p2q, int batch, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(p1q && p1p && p2q, "null polynomial");
    if (check_levels(ctx->c, lq, lp, true)) return -1;
    const size_t N = ctx->c.N;
    return moddown_qp_to_q_ntt(&ctx->c, lq, lp, CSpan{(const u64*)p1q, N, sq}, CSpan{(const u64*)p1p, N, sp}, Span{(u64*)p2q, N, sq}, batch, S(stream));
}
int lgpu_moddown_qp_to_p(lgpu_ctx* ctx, int lq, int lp, const uint64_t* p1q, const uint64_t* p1p, uint64_t* p2p, int batch, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(p1q && p1p && p2p, "null polynomial");
    if (check_levels(ctx->c, lq, lp, true)) return -1;
    const size_t N = ctx->c.N;
    return moddown_qp_to_p(&ctx->c, lq, lp, CSpan{(const u64*)p1q, N, sq}, CSpan{(const u64*)p1p, N, sp}, Span{(u64*)p2p, N, sp}, batch, S(stream));
}
int lgpu_decompose_and_split(lgpu_ctx* ctx, int lq, int lp, int nb_pi, int digit, const uint64_t* p0q, uint64_t* p1q, uint64_t* p1p,
                             int batch, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(p0q && p1q && (p1p || lp < 0), "null polynomial");
    const size_t N = ctx->c.N;
    return launch_decompose_and_split(&ctx->c, lq, lp, nb_pi, digit, CSpan{(const u64*)p0q, N, sq}, Span{(u64*)p1q, N, sq}, Span{(u64*)p1p, N, sp},
                                      batch, S(stream));
}

int lgpu_div_by_last_modulus_many(lgpu_ctx* ctx, int ring, int level, int flags, int nb, const uint64_t* p0, uint64_t* p1, int batch,
                                  size_t si, size_t so, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(p0 && p1, "null polynomial");
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    const size_t N = ctx->c.N;
    return div_by_last_modulus_many(&ctx->c, ring, level, (flags & LGPU_DIV_ROUND) != 0, (flags & LGPU_DIV_NTT) != 0, nb,
                                    CSpan{(const u64*)p0, N, si}, Span{(u64*)p1, N, so}, batch, S(stream));
}

static AccSpans make_acc(u64* a0q, u64* a0p, u64* a1q, u64* a1p, size_t N, size_t sq, size_t sp) {
    AccSpans a;
    a.q[0] = Span{a0q, N, sq}; a.q[1] = Span{a1q, N, sq};
    a.p[0] = Span{a0p, N, sp}; a.p[1] = Span{a1p, N, sp};
    return a;
}

int lgpu_gadget_product(lgpu_ctx* ctx, int lq, const uint64_t* cx, const lgpu_gadget_ct* evk, uint64_t* ct0, uint64_t* ct1, int batch,
                        size_t scx, size_t sct, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(cx && ct0 && ct1, "null polynomial");
    REQUIRE_ALIGNED(AL(cx) && AL(ct0) && AL(ct1) && ((scx | sct) & 1) == 0);
    GadgetCt g;
    if (to_gadget_ct(evk, g)) return -1;
    lq = std::min(lq, g.levelQ);   // core/rlwe/evaluator_gadget_product.go:18
    const size_t N = ctx->c.N;
    return gadget_product(&ctx->c, lq, CSpan{(const u64*)cx, N, scx}, g, Span{(u64*)ct0, N, sct}, Span{(u64*)ct1, N, sct}, batch, S(stream));
}
int lgpu_gadget_product_lazy(lgpu_ctx* ctx, int lq, const uint64_t* cx, const lgpu_gadget_ct* evk, uint64_t* a0q, uint64_t* a0p, uint64_t* a1q,
                             uint64_t* a1p, int batch, size_t scx, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(cx && a0q && a1q, "null polynomial");
    REQUIRE_ALIGNED(AL(cx) && AL(a0q) && AL(a0p) && AL(a1q) && AL(a1p) && ((scx | sq | sp) & 1) == 0);
    GadgetCt g;
    if (to_gadget_ct(evk, g)) return -1;
    REQUIRE(g.levelP < 0 || (a0p && a1p), "null P accumulator");
    const size_t N = ctx->c.N;
    return gadget_product_lazy(&ctx->c, lq, CSpan{(const u64*)cx, N, scx}, g, make_acc((u64*)a0q, (u64*)a0p, (u64*)a1q, (u64*)a1p, N, sq, sp), batch, S(stream));
}
int lgpu_evaluator_moddown(lgpu_ctx* ctx, int lq, int lp, const uint64_t* a0q, const uint64_t* a0p, const uint64_t* a1q, const uint64_t* a1p,
                           uint64_t* ct0, uint64_t* ct1, int batch, size_t sq, size_t sp, size_t sct, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(a0q && a1q && ct0 && ct1, "null polynomial");
    REQUIRE_ALIGNED(AL(a0q) && AL(a0p) && AL(a1q) && AL(a1p) && AL(ct0) && AL(ct1) && ((sq | sp | sct) & 1) == 0);
    if (check_levels(ctx->c, lq, lp, lp >= 0)) return -1;
    const size_t N = ctx->c.N;
    return evaluator_moddown_ntt(&ctx->c, lq, lp, make_acc((u64*)a0q, (u64*)a0p, (u64*)a1q, (u64*)a1p, N, sq, sp), Span{(u64*)ct0, N, sct},
                                 Span{(u64*)ct1, N, sct}, batch, S(stream));
}
int lgpu_decompose_single_ntt(lgpu_ctx* ctx, int lq, int lp, int nb_pi, int digit, const uint64_t* c2ntt, const uint64_t* c2inv, uint64_t* c2q,
                              uint64_t* c2p, int batch, size_t si, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(c2ntt && c2inv && c2q && (c2p || lp < 0), "null polynomial");
    if (check_levels(ctx->c, lq, lp, lp >= 0)) return -1;
    const size_t N = ctx->c.N;
    return decompose_single_ntt(&ctx->c, lq, lp, nb_pi, digit, CSpan{(const u64*)c2ntt, N, si}, CSpan{(const u64*)c2inv, N, si}, Span{(u64*)c2q, N, sq},
                                Span{(u64*)c2p, N, sp}, true, batch, S(stream));
}
int lgpu_decompose_ntt(lgpu_ctx* ctx, int lq, int lp, int nb_pi, const uint64_t* c2, int is_ntt, uint64_t* decomp, int batch, size_t si, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(c2 && decomp, "null polynomial");
    if (check_levels(ctx->c, lq, lp, true)) return -1;
    const size_t N = ctx->c.N;
    return decompose_ntt(&ctx->c, lq, lp, nb_pi, CSpan{(const u64*)c2, N, si}, is_ntt != 0, (u64*)decomp, batch, S(stream));
}
int lgpu_gadget_product_hoisted(lgpu_ctx* ctx, int lq, const uint64_t* decomp, const lgpu_gadget_ct* evk, uint64_t* ct0, uint64_t* ct1, int batch,
                                size_t sct, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(decomp && ct0 && ct1, "null polynomial");
    REQUIRE_ALIGNED(AL(decomp) && AL(ct0) && AL(ct1) && (sct & 1) == 0);
    GadgetCt g;
    if (to_gadget_ct(evk, g)) return -1;
    const size_t N = ctx->c.N;
    return gadget_product_hoisted(&ctx->c, lq, (const u64*)decomp, g, Span{(u64*)ct0, N, sct}, Span{(u64*)ct1, N, sct}, batch, S(stream));
}
int lgpu_gadget_product_hoisted_lazy(lgpu_ctx* ctx, int lq, const uint64_t* decomp, const lgpu_gadget_ct* evk, uint64_t* a0q, uint64_t* a0p,
                                     uint64_t* a1q, uint64_t* a1p, int batch, size_t sq, size_t sp, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(decomp && a0q && a0p && a1q && a1p, "null polynomial");
    REQUIRE_ALIGNED(AL(decomp) && AL(a0q) && AL(a0p) && AL(a1q) && AL(a1p) && ((sq | sp) & 1) == 0);
    GadgetCt g;
    if (to_gadget_ct(evk, g)) return -1;
    const size_t N = ctx->c.N;
    return gadget_product_hoisted_lazy(&ctx->c, lq, (const u64*)decomp, g, make_acc((u64*)a0q, (u64*)a0p, (u64*)a1q, (u64*)a1p, N, sq, sp), batch, S(stream));
}
int lgpu_evaluator_automorphism(lgpu_ctx* ctx, int level, const uint64_t* ct_in, uint64_t gal_el, const lgpu_gadget_ct* gk, const uint64_t* decomp,
                                uint64_t* ct_out, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    GadgetCt g;
    if (to_gadget_ct(gk, g)) return -1;
    REQUIRE(level >= 0 && level <= g.levelQ && level < ctx->c.nQ, "level out of range");
    const size_t N = ctx->c.N, nq = level + 1, cs = 2 * nq * N;
    const u64* in = (const u64*)ct_in;
    u64* out = (u64*)ct_out;
    return evaluator_automorphism(&ctx->c, level, CSpan{in, N, cs}, CSpan{in + nq * N, N, cs}, gal_el, g, Span{out, N, cs}, Span{out + nq * N, N, cs},
                                  (const u64*)decomp, batch, S(stream));
}
int lgpu_evaluator_relinearize(lgpu_ctx* ctx, int level, const uint64_t* ct_in, const lgpu_gadget_ct* rlk, uint64_t* ct_out, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    GadgetCt g;
    if (to_gadget_ct(rlk, g)) return -1;
    REQUIRE(level >= 0 && level <= g.levelQ && level < ctx->c.nQ, "level out of range");
    const size_t N = ctx->c.N, nq = level + 1;
    const u64* in = (const u64*)ct_in;
    u64* out = (u64*)ct_out;
    return evaluator_relinearize(&ctx->c, level, CSpan{in, N, 3 * nq * N}, CSpan{in + nq * N, N, 3 * nq * N}, CSpan{in + 2 * nq * N, N, 3 * nq * N}, g,
                                 Span{out, N, 2 * nq * N}, Span{out + nq * N, N, 2 * nq * N}, batch, S(stream));
}

int lgpu_ckks_mulrelin_rescale_batch(lgpu_ctx* ctx, int level, const uint64_t* ct_a, const uint64_t* ct_b, const lgpu_gadget_ct* rlk, int nb_rescales,
                                     uint64_t* ct_out, int batch, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct_a && ct_b && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_a) && AL(ct_b) && AL(ct_out));
    REQUIRE(batch >= 1, "batch must be >= 1");
    GadgetCt g;
    if (to_gadget_ct(rlk, g)) return -1;
    return ckks_mulrelin_rescale(&ctx->c, level, (const u64*)ct_a, (const u64*)ct_b, g, nb_rescales, (u64*)ct_out, batch, S(stream));
}

// Host-buffer variant: H2D / compute / D2H pipelined over chunks on three streams with double buffering.
int lgpu_ckks_mulrelin_rescale_batch_host(lgpu_ctx* ctx, int level, const uint64_t* ct_a_host, const uint64_t* ct_b_host, const lgpu_gadget_ct* rlk,
                                          int nb_rescales, uint64_t* ct_out_host, int batch, int chunk) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(ct_a_host && ct_b_host && ct_out_host, "null ciphertext");
    REQUIRE(batch >= 1, "batch must be >= 1");
    GadgetCt g;
    if (to_gadget_ct(rlk, g)) return -1;
    const Ctx& c = ctx->c;
    REQUIRE(level >= 0 && level < c.nQ && nb_rescales >= 0 && nb_rescales <= level, "level out of range");
    if (chunk <= 0) chunk = 2;   // short chunks shrink the pipeline's head and tail (H100: profiles/h100_switch_ab.md)
    if (chunk > batch) chunk = batch;
    const size_t N = c.N, nq = level + 1, nqo = nq - nb_rescales;
    const size_t in_words = 2 * nq * N, out_words = 2 * nqo * N;
    LGPU_CUDA_OK(cudaSetDevice(c.device));
    // Independent streams, each doing H2D -> compute -> D2H for every kStreams-th chunk: the copies of one chunk overlap the compute of the
    // others (copy engines run concurrently with the SMs). Streams and staging buffers live in the
    // context; one host-pipeline call at a time per context.
    Ctx::HostPipe& hp = ctx->c.host_pipe;
    std::lock_guard<std::mutex> lock(hp.mu);
    int rc = 0;
    const size_t need[3] = {chunk * in_words, chunk * in_words, chunk * out_words};
    constexpr int NS = Ctx::HostPipe::kStreams;
    // two streams by default: one chunk's copies overlap the other's compute. A third (LGPU_HOST_STREAMS=3) has not shown a gain beyond the
    // run-to-run spread of this path on the H100 (profiles/h100_switch_ab.md)
    static const int ns_env = [] { const char* e = getenv("LGPU_HOST_STREAMS"); int v = e ? atoi(e) : 2; return v >= 1 && v <= NS ? v : 2; }();
    const int ns = ns_env;
    for (int i = 0; i < ns && !rc; i++) {
        if (!hp.st[i] && cudaStreamCreateWithFlags(&hp.st[i], cudaStreamNonBlocking) != cudaSuccess) rc = -1;
        for (int k = 0; k < 3 && !rc; k++) {
            if (hp.buf[i][k] && hp.cap[k] >= need[k]) continue;
            if (hp.buf[i][k]) { cudaStreamSynchronize(hp.st[i]); cudaFree(hp.buf[i][k]); hp.buf[i][k] = nullptr; }
            if (cudaMalloc(&hp.buf[i][k], need[k] * 8) != cudaSuccess) rc = -1;
        }
    }
    if (rc) lgpu::set_error("allocation failed in mulrelin_rescale_batch_host");
    else for (int k = 0; k < 3; k++) hp.cap[k] = std::max(hp.cap[k], need[k]);
    cudaStream_t* st = hp.st;
    for (int k = 0, i = 0; !rc && k < batch; k += chunk, i = (i + 1) % ns) {
        const int nb = std::min(chunk, batch - k);
        u64 *dA = hp.buf[i][0], *dB = hp.buf[i][1], *dO = hp.buf[i][2];
        if (cudaMemcpyAsync(dA, ct_a_host + (size_t)k * in_words, nb * in_words * 8, cudaMemcpyHostToDevice, st[i]) != cudaSuccess ||
            cudaMemcpyAsync(dB, ct_b_host + (size_t)k * in_words, nb * in_words * 8, cudaMemcpyHostToDevice, st[i]) != cudaSuccess) {
            lgpu::set_error("H2D copy failed"); rc = -1; break;
        }
        rc = ckks_mulrelin_rescale(&c, level, dA, dB, g, nb_rescales, dO, nb, st[i]);
        if (rc) break;
        if (cudaMemcpyAsync(ct_out_host + (size_t)k * out_words, dO, nb * out_words * 8, cudaMemcpyDeviceToHost, st[i]) != cudaSuccess) {
            lgpu::set_error("D2H copy failed"); rc = -1; break;
        }
    }
    for (int i = 0; i < ns; i++) {
        if (st[i]) cudaStreamSynchronize(st[i]);
    }
    if (!rc) {
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { lgpu::set_error(cudaGetErrorString(e)); rc = -1; }
    }
    return rc;
}

}  // extern "C"

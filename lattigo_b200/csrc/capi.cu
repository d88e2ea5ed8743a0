// capi.cu -- extern "C" entry points declared in include/lattigo_b200.h (context, memory, NTT, vec ops).
#include <cstring>
#include "capi_common.h"

using namespace lgpu;


// NULL means the CUDA default stream (same convention as the runtime API), so that callers which pass their
// framework's current stream (0 for torch's default stream) stay ordered with their own work.
static inline cudaStream_t pick_stream(lgpu_ctx* ctx, void* stream) { (void)ctx; return (cudaStream_t)stream; }


namespace lgpu {
// rows 0..level of ring Q or P -> global limb indices
int make_rowmap(const Ctx& c, int ring, int level, RowMap& rm) {
    const int n = ring == LGPU_RING_Q ? c.nQ : c.nP;
    if (ring != LGPU_RING_Q && ring != LGPU_RING_P) { set_error("invalid ring selector"); return -1; }
    if (level < 0) { set_error("level cannot be negative"); return -1; }
    if (level >= n) { set_error("level cannot be larger than max level"); return -1; }
    rm.nrows = level + 1;
    const int off = ring == LGPU_RING_Q ? 0 : c.nQ;
    for (int i = 0; i <= level; i++) { rm.limb[i] = (unsigned char)(off + i); rm.drow[i] = (unsigned char)i; }
    return 0;
}
int make_rowmap_single(const Ctx& c, int ring, int limb, RowMap& rm) {
    const int n = ring == LGPU_RING_Q ? c.nQ : c.nP;
    if (ring != LGPU_RING_Q && ring != LGPU_RING_P) { set_error("invalid ring selector"); return -1; }
    if (limb < 0 || limb >= n) { set_error("limb index out of range"); return -1; }
    rm.nrows = 1;
    rm.limb[0] = (unsigned char)((ring == LGPU_RING_Q ? 0 : c.nQ) + limb);
    rm.drow[0] = 0;
    return 0;
}

int to_gadget_ct(const lgpu_gadget_ct* e, GadgetCt& g, const char* null_msg) {
    REQUIRE(e && e->data, null_msg);
    REQUIRE_ALIGNED(AL(e->data));
    g.data = (const u64*)e->data; g.levelQ = e->level_q; g.levelP = e->level_p; g.pw2 = e->base_two_decomposition;
    g.ndigits = e->n_digits; g.npw2max = e->n_pw2_max > 0 ? e->n_pw2_max : 1; g.pw2_sizes = e->pw2_sizes;
    return 0;
}

int to_galois_keys(const lgpu_galois_keys* gks, GaloisKeySet& ks) {
    REQUIRE(gks, "null Galois key set");
    REQUIRE(gks->n_keys >= 0 && (gks->n_keys == 0 || (gks->gal_els && gks->keys)), "null Galois key arrays");
    ks.n = gks->n_keys; ks.gal_els = (const u64*)gks->gal_els;
    ks.keys.resize(ks.n);
    for (int i = 0; i < ks.n; i++)
        if (to_gadget_ct(&gks->keys[i], ks.keys[i])) return -1;
    return 0;
}

bool overlaps(const void* a, size_t abytes, const void* b, size_t bbytes) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return x < y + bbytes && y < x + abytes;
}
}  // namespace lgpu

extern "C" {

const char* lgpu_version(void) { return "lattigo_b200 0.2 (sm_90a)"; }
const char* lgpu_last_error(void) { return lgpu::last_error(); }

int lgpu_create(lgpu_ctx** out, int device, int logN, int ring_type, const uint64_t* q, int nq, const uint64_t* p, int np) {
    REQUIRE(out, "null output handle");
    lgpu_ctx* h = new lgpu_ctx();
    int rc;
    if (device < 0) {
        // host-only context: tables are generated, nothing is uploaded (used by CPU-only tests of the host logic)
        h->c.device = -1;
        rc = build_context(&h->c, -1, logN, ring_type, (const u64*)q, nq, (const u64*)p, np);
    } else {
        rc = build_context(&h->c, device, logN, ring_type, (const u64*)q, nq, (const u64*)p, np);
    }
    if (rc) { destroy_context(&h->c); delete h; return rc; }
    *out = h;
    return 0;
}

void lgpu_destroy(lgpu_ctx* ctx) {
    if (!ctx) return;
    destroy_context(&ctx->c);
    delete ctx;
}

int lgpu_sync(lgpu_ctx* ctx, void* stream) {
    REQUIRE_DEVICE(ctx);
    LGPU_CUDA_OK(cudaStreamSynchronize(pick_stream(ctx, stream)));
    return 0;
}

int lgpu_ring_get_table(lgpu_ctx* ctx, int ring, int limb, int kind, uint64_t* host_out, size_t nwords) {
    REQUIRE(ctx && host_out, "null argument");
    const Ctx& c = ctx->c;
    const int n = ring == LGPU_RING_Q ? c.nQ : c.nP;
    REQUIRE(ring == LGPU_RING_Q || ring == LGPU_RING_P, "invalid ring selector");
    REQUIRE(limb >= 0 && limb < n, "limb index out of range");
    const HostSubRing& s = c.sub[(ring == LGPU_RING_Q ? 0 : c.nQ) + limb];
    switch (kind) {
        case 0: {
            REQUIRE(nwords >= 6, "buffer too small");
            const u64 v[6] = {s.q, s.qinv, s.bred_hi, s.bred_lo, s.ninv, s.primitive_root};
            memcpy(host_out, v, sizeof(v));
            return 0;
        }
        case 1:
        case 2: {
            const std::vector<u64>& r = kind == 1 ? s.roots_fwd : s.roots_bwd;
            REQUIRE(nwords >= r.size(), "buffer too small");
            memcpy(host_out, r.data(), r.size() * sizeof(u64));
            return 0;
        }
        case 3: {
            REQUIRE(limb >= 1, "RescaleConstants start at limb 1");
            REQUIRE(nwords >= (size_t)limb, "buffer too small");
            const std::vector<u64>& rc = ring == LGPU_RING_Q ? c.rescaleQ : c.rescaleP;
            memcpy(host_out, rc.data() + (size_t)(limb - 1) * n, (size_t)limb * sizeof(u64));
            return 0;
        }
    }
    lgpu::set_error("unknown table kind");
    return -1;
}

int lgpu_ring_set_roots(lgpu_ctx* ctx, int ring, int limb, const uint64_t* roots_fwd, const uint64_t* roots_bwd, uint64_t ninv) {
    REQUIRE(ctx && roots_fwd && roots_bwd, "null argument");
    Ctx& c = ctx->c;
    const int n = ring == LGPU_RING_Q ? c.nQ : c.nP;
    REQUIRE(ring == LGPU_RING_Q || ring == LGPU_RING_P, "invalid ring selector");
    REQUIRE(limb >= 0 && limb < n, "limb index out of range");
    const int g = (ring == LGPU_RING_Q ? 0 : c.nQ) + limb;
    const size_t half = (size_t)(c.nthroot >> 1);
    HostSubRing& s = c.sub[g];
    s.roots_fwd.assign((const u64*)roots_fwd, (const u64*)roots_fwd + half);
    s.roots_bwd.assign((const u64*)roots_bwd, (const u64*)roots_bwd + half);
    s.ninv = ninv;
    if (c.device >= 0) {
        LGPU_CUDA_OK(cudaSetDevice(c.device));
        LGPU_CUDA_OK(cudaDeviceSynchronize());
        if (upload_limb_tables(&c, g)) return -1;
        LGPU_CUDA_OK(cudaMemcpy(c.d_limbs + g, &c.h_limbs[g], sizeof(LimbConst), cudaMemcpyHostToDevice));
    }
    return 0;
}

int lgpu_malloc(lgpu_ctx* ctx, void** dptr, size_t bytes) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(dptr, "null argument");
    LGPU_CUDA_OK(cudaSetDevice(ctx->c.device));
    LGPU_CUDA_OK(cudaMalloc(dptr, bytes));
    return 0;
}
int lgpu_free(lgpu_ctx* ctx, void* dptr) {
    REQUIRE_DEVICE(ctx);
    LGPU_CUDA_OK(cudaSetDevice(ctx->c.device));
    LGPU_CUDA_OK(cudaFree(dptr));
    return 0;
}
int lgpu_memcpy_h2d(lgpu_ctx* ctx, void* dst, const void* src, size_t bytes, void* stream) {
    REQUIRE_DEVICE(ctx);
    LGPU_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, pick_stream(ctx, stream)));
    return 0;
}
int lgpu_memcpy_d2h(lgpu_ctx* ctx, void* dst, const void* src, size_t bytes, void* stream) {
    REQUIRE_DEVICE(ctx);
    LGPU_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, pick_stream(ctx, stream)));
    return 0;
}

// ---- NTT ---------------------------------------------------------------------------------------------
static int ntt_common(lgpu_ctx* ctx, bool inverse, const RowMap& rm, const uint64_t* in, uint64_t* out, int lazy,
                      int batch, size_t batch_stride, void* stream) {
    REQUIRE(in && out, "null polynomial");
    REQUIRE(batch >= 1, "batch must be >= 1");
    const Ctx& c = ctx->c;
    CSpan i{(const u64*)in, (size_t)c.N, batch_stride};
    Span o{(u64*)out, (size_t)c.N, batch_stride};
    const int mode = lazy ? NTT_EXACT_LAZY : NTT_CANONICAL;
    return inverse ? launch_intt(&c, rm, i, o, batch, mode, pick_stream(ctx, stream))
                   : launch_ntt(&c, rm, i, o, batch, mode, pick_stream(ctx, stream));
}

int lgpu_ntt(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t* out, int lazy, int batch, size_t batch_stride, void* stream) {
    REQUIRE_DEVICE(ctx);
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    return ntt_common(ctx, false, rm, in, out, lazy, batch, batch_stride, stream);
}
int lgpu_ntt_then_mul_coeffs_montgomery(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, const uint64_t* other, uint64_t* out, int batch,
                                        size_t batch_stride, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(in && other && out, "null polynomial");
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    const size_t N = ctx->c.N;
    return launch_ntt_mul_montgomery(&ctx->c, rm, CSpan{(const u64*)in, N, batch_stride}, CSpan{(const u64*)other, N, batch_stride},
                                     Span{(u64*)out, N, batch_stride}, batch, (cudaStream_t)stream);
}
int lgpu_intt(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t* out, int lazy, int batch, size_t batch_stride, void* stream) {
    REQUIRE_DEVICE(ctx);
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    return ntt_common(ctx, true, rm, in, out, lazy, batch, batch_stride, stream);
}
int lgpu_subring_ntt(lgpu_ctx* ctx, int ring, int limb, const uint64_t* in, uint64_t* out, int lazy, void* stream) {
    REQUIRE_DEVICE(ctx);
    RowMap rm;
    if (make_rowmap_single(ctx->c, ring, limb, rm)) return -1;
    return ntt_common(ctx, false, rm, in, out, lazy, 1, 0, stream);
}
int lgpu_subring_intt(lgpu_ctx* ctx, int ring, int limb, const uint64_t* in, uint64_t* out, int lazy, void* stream) {
    REQUIRE_DEVICE(ctx);
    RowMap rm;
    if (make_rowmap_single(ctx->c, ring, limb, rm)) return -1;
    return ntt_common(ctx, true, rm, in, out, lazy, 1, 0, stream);
}

// ---- vec ops -----------------------------------------------------------------------------------------
int lgpu_vecop(lgpu_ctx* ctx, int ring, int level, int opcode, const uint64_t* p1, const uint64_t* p2, uint64_t* p3,
               const uint64_t* scalars0, const uint64_t* scalars1, int batch, size_t batch_stride, void* stream) {
    REQUIRE_DEVICE(ctx);
    RowMap rm;
    if (make_rowmap(ctx->c, ring, level, rm)) return -1;
    const size_t N = (size_t)ctx->c.N;
    return launch_vecop(&ctx->c, rm, opcode, CSpan{(const u64*)p1, N, batch_stride}, CSpan{(const u64*)p2, N, batch_stride},
                        Span{(u64*)p3, N, batch_stride}, batch, (const u64*)scalars0, (const u64*)scalars1, 0, 0,
                        ctx->c.N, pick_stream(ctx, stream));
}
int lgpu_subring_vecop(lgpu_ctx* ctx, int ring, int limb, int opcode, const uint64_t* p1, const uint64_t* p2, uint64_t* p3,
                       uint64_t s0, uint64_t s1, int n, void* stream) {
    REQUIRE_DEVICE(ctx);
    REQUIRE(n >= 0 && n <= ctx->c.N, "n out of range");
    RowMap rm;
    if (make_rowmap_single(ctx->c, ring, limb, rm)) return -1;
    return launch_vecop(&ctx->c, rm, opcode, CSpan{(const u64*)p1, 0, 0}, CSpan{(const u64*)p2, 0, 0}, Span{(u64*)p3, 0, 0},
                        1, nullptr, nullptr, s0, s1, n, pick_stream(ctx, stream));
}

}  // extern "C"

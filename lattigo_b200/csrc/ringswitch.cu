// ringswitch.cu -- rlwe.Evaluator.ApplyEvaluationKey (core/rlwe/evaluator_evaluationkey.go:36-107) on the device, for a BATCH of
// ciphertexts sharing one evaluation key, including the ring-degree switches of SwitchCiphertextRingDegree[NTT]
// (core/rlwe/element.go:250-312). The context is the evaluator's (large) degree N; n is the small degree, gap = N / n.
//   same degree   ct_out = (c0 + ks0, ks1), ks = GadgetProduct(c1)
//   up   n -> N   ring_up_ntt_kernel (NTT: large[i gap + w] = small[i]) or ring_stride_coeff_kernel (coefficients: every gap-th
//                 output coefficient written, the others keep their contents), then the same-degree key switch in place on ct_out
//   down N -> n   key switch, then ring_down_ntt_kernel (NTT: the block average below) or ring_stride_coeff_kernel (coefficients:
//                 out[w] = (c0 + ks0)[w gap]); c0 is added inside that pass, so the degree-N (c0 + ks0) is never stored
// The reference's downward NTT switch is, per row, an INTT at N, every gap-th coefficient, and NTTStandard at n with the LARGE ring's
// RootsForward (psi_n = psi_N^gap). In the bit-reversed evaluation order that is the block average
//     out[j] = gap^-1 * sum_{u < gap} A[j gap + u]   (mod q)
// (DESIGN 3.4), one streaming pass. Every output is a canonical residue, so the results equal the reference bit for bit
// (tests/test_gpu_ringswitch.py vs oracle/ringswitch.py). One gadget product runs per batch_chunk() ciphertexts: the key is read once
// per sub-batch.
#include <algorithm>
#include <string>
#include "capi_common.h"
#include "composite.h"
#include "modarith.cuh"

namespace lgpu {

// ---------------------------------------------------------------------------------------------------------------------
// kernels: x = output coefficient, y = row (limb), z = 2 * batch entry + component
// ---------------------------------------------------------------------------------------------------------------------
struct RingDownParams {
    const LimbConst* limbs;
    const u64* src; size_t src_cs, src_bs;   // component c of entry b: src + c * src_cs + b * src_bs, rows of N words
    const u64* add; size_t add_bs;           // component 0 addend, same row layout (nullptr: none)
    u64* out; size_t out_cs, out_bs;         // rows of n words
    int n, lg_gap, m;                        // output degree, log2(N / n), batch entries
    u64 ginv[kMaxRows], ginv_sh[kMaxRows];   // gap^-1 mod q_r and its Shoup constant
};
// out[j] = gap^-1 * sum_u (src + add)[j gap + u], reduced after every add (canonical inputs below 2^63: no wrap at any gap).
// G = min(gap, 32) consecutive lanes share one output: lane l of a group sums u = l, l + G, ..., so each load instruction of a warp
// reads 32 consecutive words at every gap; the G partial sums are then added with shuffles.
__global__ void __launch_bounds__(256) ring_down_ntt_kernel(RingDownParams p) {
    const int lgG = p.lg_gap < 5 ? p.lg_gap : 5;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int j = tid >> lgG, l = tid & ((1 << lgG) - 1);
    const bool valid = j < p.n;                   // every lane stays for the shuffles
    const int r = blockIdx.y;
    const u64 q = p.limbs[r].q;
    const size_t N = (size_t)p.n << p.lg_gap, gap = (size_t)1 << p.lg_gap, G = (size_t)1 << lgG;
    const size_t ri = (size_t)r * N + ((size_t)j << p.lg_gap);
    for (int z = blockIdx.z; z < 2 * p.m; z += gridDim.z) {
        const size_t b = (size_t)(z >> 1), comp = (size_t)(z & 1);
        u64 acc = 0;
        if (valid) {
            const u64* s = p.src + comp * p.src_cs + b * p.src_bs + ri;
            const u64* a = (comp == 0 && p.add) ? p.add + b * p.add_bs + ri : nullptr;
            for (size_t u = l; u < gap; u += G) {
                u64 x = s[u];
                if (a) x = cred(x + a[u], q);
                acc = cred(acc + x, q);
            }
        }
        for (int o = (int)G >> 1; o > 0; o >>= 1) acc = cred(acc + __shfl_xor_sync(0xffffffffu, acc, o), q);
        if (valid && l == 0)
            p.out[comp * p.out_cs + b * p.out_bs + (size_t)r * p.n + j] = cred(acc * p.ginv[r] - __umul64hi(acc, p.ginv_sh[r]) * q, q);
    }
}

struct RingUpParams {
    const u64* src; size_t src_cs, src_bs;   // rows of n words
    u64* out; size_t out_cs, out_bs;         // rows of N words
    int N, lg_gap, m;
};
// MapSmallDimensionToLargerDimensionNTT (ring/operations.go:380-392): out[k] = src[k / gap]
__global__ void __launch_bounds__(256) ring_up_ntt_kernel(RingUpParams p) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= p.N) return;
    const size_t r = blockIdx.y, n = (size_t)p.N >> p.lg_gap;
    for (int z = blockIdx.z; z < 2 * p.m; z += gridDim.z) {
        const size_t b = (size_t)(z >> 1), comp = (size_t)(z & 1);
        p.out[comp * p.out_cs + b * p.out_bs + r * p.N + k] = p.src[comp * p.src_cs + b * p.src_bs + r * n + (k >> p.lg_gap)];
    }
}

struct RingStrideParams {
    const LimbConst* limbs;
    const u64* src; size_t src_cs, src_bs, src_rs, src_step;
    const u64* add; size_t add_bs;           // component 0 addend in src's layout (nullptr: none)
    u64* out; size_t out_cs, out_bs, out_rs, out_step;
    int n, m;                                // small degree (coefficients moved per row), batch entries
};
// SwitchCiphertextRingDegree (element.go:293-312): out[w out_step] = (src + add)[w src_step] for w < n
__global__ void __launch_bounds__(256) ring_stride_coeff_kernel(RingStrideParams p) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= p.n) return;
    const size_t r = blockIdx.y;
    const u64 q = p.limbs[r].q;
    const size_t si = r * p.src_rs + (size_t)w * p.src_step;
    for (int z = blockIdx.z; z < 2 * p.m; z += gridDim.z) {
        const size_t b = (size_t)(z >> 1), comp = (size_t)(z & 1);
        u64 x = p.src[comp * p.src_cs + b * p.src_bs + si];
        if (comp == 0 && p.add) x = cred(x + p.add[b * p.add_bs + si], q);
        p.out[comp * p.out_cs + b * p.out_bs + r * p.out_rs + (size_t)w * p.out_step] = x;
    }
}

namespace {

constexpr unsigned kMaxGridZ = 65535;

int log2_exact(int v) {
    int l = 0;
    while ((1 << l) < v) l++;
    return (1 << l) == v ? l : -1;
}

dim3 grid_of(int width, int rows, int m) {
    return dim3((unsigned)((width + 255) / 256), (unsigned)rows, (unsigned)std::min(2 * m, (int)kMaxGridZ));
}

// ks = GadgetProduct(c1) for nb ciphertexts, in the domain of the input: ks0 at ks, ks1 at ks + nb * cs, entry stride cs.
// Coefficient domain: the NTT of c1 (staged in t), the product, and its INTT. The reference's coefficient-domain GadgetProduct
// (NTT inside, ModDownQPtoQ on the INTT of the accumulators) leaves the same residues: ModDown is linear per coefficient.
int keyswitch_c1(const Ctx* c, int level, bool ntt, CSpan c1, const GadgetCt& key, u64* ks, u64* t, int nb, cudaStream_t st) {
    const size_t N = c->N, cs = (size_t)(level + 1) * N;
    const RowMap rm = rows_range(0, 0, level + 1);
    if (!ntt) {
        if (launch_ntt(c, rm, c1, Span{t, N, cs}, nb, NTT_CANONICAL, st)) return -1;
        c1 = CSpan{t, N, cs};
    }
    if (gadget_product(c, level, c1, key, Span{ks, N, cs}, Span{ks + (size_t)nb * cs, N, cs}, nb, st)) return -1;
    if (!ntt && launch_intt(c, rm, CSpan{ks, N, cs}, Span{ks, N, cs}, 2 * nb, NTT_CANONICAL, st)) return -1;
    return 0;
}

// same-degree applyEvaluationKey (:99-107) on nb ciphertexts ([batch][2][level + 1][N] blocks): out = (c0 + ks0, ks1). `in` and `out` may be
// the same block (the key switch reads all of c1 before writing, the addition is element-wise).
int apply_same(const Ctx* c, int level, bool ntt, CBlock in, Block out, const GadgetCt& key, u64* ks, u64* t, int nb, cudaStream_t st) {
    const size_t N = c->N, cs = (size_t)(level + 1) * N;
    if (ntt) {
        // one ModDown per component: out[0] = ModDown(acc[0]) + c0, out[1] = ModDown(acc[1]); the fused ModDown adds c0 in its epilogue
        const size_t nq = level + 1, np = key.levelP + 1, qp = (nq + np) * N;
        Scratch acc_buf;
        if (acc_buf.alloc((size_t)2 * nb * qp, st)) return -1;
        const AccSpans acc = stacked_acc(acc_buf.p, nq, np, N, nb);
        if (gadget_product_lazy(c, level, CSpan{in.p + in.cs, N, in.bs}, key, acc, nb, st)) return -1;
        if (moddown_ntt(c, level, key.levelP, CBlock{acc_buf.p, 0, qp}, CBlock{in.p, 0, in.bs}, Block{out.p, 0, out.bs}, 1, nb, st)) return -1;
        return moddown_ntt(c, level, key.levelP, CBlock{acc_buf.p + (size_t)nb * qp, 0, qp}, CBlock{nullptr, 0, 0}, Block{out.p + out.cs, 0, out.bs}, 1,
                           nb, st);
    }
    if (keyswitch_c1(c, level, false, CSpan{in.p + in.cs, N, in.bs}, key, ks, t, nb, st)) return -1;
    LGPU_CUDA_OK(cudaMemcpy2DAsync(out.p + out.cs, out.bs * 8, ks + (size_t)nb * cs, cs * 8, cs * 8, nb, cudaMemcpyDeviceToDevice, st));
    return launch_vecop(c, rows_range(0, 0, level + 1), LGPU_OP_ADD, CSpan{in.p, N, in.bs}, CSpan{ks, N, cs}, Span{out.p, N, out.bs}, nb, nullptr,
                        nullptr, 0, 0, c->N, st);
}

int apply_run(const Ctx* c, const u64* in, int n_in, int level_in, bool ntt, const GadgetCt& key, u64* out, int n_out, int level_out, int B,
              cudaStream_t st) {
    const int level = std::min(level_in, level_out), nq = level + 1;
    const size_t N = c->N, cs = (size_t)nq * N;
    const size_t in_cs = (size_t)(level_in + 1) * n_in, out_cs = (size_t)(level_out + 1) * n_out;
    const int ch = std::min(batch_chunk(), B);
    Scratch buf;
    if (buf.alloc((size_t)ch * cs * (ntt ? 2 : 3), st)) return -1;
    u64* ks = buf.p;
    u64* t = buf.p + (size_t)2 * ch * cs;
    if (n_in < n_out) {
        // up: map every ciphertext of the batch to X^(N/n) in ct_out, then key-switch ct_out in place
        const int lg = log2_exact(n_out / n_in);
        if (ntt) {
            RingUpParams p;
            p.src = in; p.src_cs = in_cs; p.src_bs = 2 * in_cs; p.out = out; p.out_cs = out_cs; p.out_bs = 2 * out_cs; p.N = n_out; p.lg_gap = lg;
            p.m = B;
            ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * (n_in + n_out) * nq * 2 * B, 1);
            ring_up_ntt_kernel<<<grid_of(n_out, nq, B), 256, 0, st>>>(p);
        } else {
            RingStrideParams p;
            p.limbs = c->d_limbs; p.src = in; p.src_cs = in_cs; p.src_bs = 2 * in_cs; p.src_rs = n_in; p.src_step = 1; p.add = nullptr; p.add_bs = 0;
            p.out = out; p.out_cs = out_cs; p.out_bs = 2 * out_cs; p.out_rs = n_out; p.out_step = (size_t)1 << lg; p.n = n_in; p.m = B;
            ProfScope ps(LGPU_KCLASS_VECOP, st, 16.0 * n_in * nq * 2 * B, 1);
            ring_stride_coeff_kernel<<<grid_of(n_in, nq, B), 256, 0, st>>>(p);
        }
        LGPU_CUDA_OK(cudaGetLastError());
        for (int e0 = 0; e0 < B; e0 += ch) {
            const int nb = std::min(ch, B - e0);
            const Block o{out + (size_t)e0 * 2 * out_cs, out_cs, 2 * out_cs};
            if (apply_same(c, level, ntt, o, o, key, ks, t, nb, st)) return -1;
        }
        return 0;
    }
    if (n_in == n_out) {
        for (int e0 = 0; e0 < B; e0 += ch) {
            const int nb = std::min(ch, B - e0);
            if (apply_same(c, level, ntt, CBlock{in + (size_t)e0 * 2 * in_cs, in_cs, 2 * in_cs}, Block{out + (size_t)e0 * 2 * out_cs, out_cs, 2 * out_cs}, key,
                           ks, t, nb, st)) return -1;
        }
        return 0;
    }
    // down: key switch at N, then the block average / strided copy with c0 added on the fly
    const int lg = log2_exact(n_in / n_out);
    RingDownParams dp;
    if (ntt) {
        for (int r = 0; r < nq; r++) {
            const u64 q = c->Q[r];
            dp.ginv[r] = h_invmod(((u64)1 << lg) % q, q);
            dp.ginv_sh[r] = (u64)(((unsigned __int128)dp.ginv[r] << 64) / q);
        }
    }
    for (int e0 = 0; e0 < B; e0 += ch) {
        const int nb = std::min(ch, B - e0);
        const u64* i0 = in + (size_t)e0 * 2 * in_cs;
        u64* o = out + (size_t)e0 * 2 * out_cs;
        if (keyswitch_c1(c, level, ntt, CSpan{i0 + in_cs, N, 2 * in_cs}, key, ks, t, nb, st)) return -1;
        if (ntt) {
            dp.limbs = c->d_limbs; dp.src = ks; dp.src_cs = (size_t)nb * cs; dp.src_bs = cs; dp.add = i0; dp.add_bs = 2 * in_cs;
            dp.out = o; dp.out_cs = out_cs; dp.out_bs = 2 * out_cs; dp.n = n_out; dp.lg_gap = lg; dp.m = nb;
            ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * (3 * (size_t)n_in + 2 * (size_t)n_out) * nq * nb, 1);
            ring_down_ntt_kernel<<<grid_of(n_out << std::min(lg, 5), nq, nb), 256, 0, st>>>(dp);
        } else {
            RingStrideParams p;
            p.limbs = c->d_limbs; p.src = ks; p.src_cs = (size_t)nb * cs; p.src_bs = cs; p.src_rs = N; p.src_step = (size_t)1 << lg;
            p.add = i0; p.add_bs = 2 * in_cs; p.out = o; p.out_cs = out_cs; p.out_bs = 2 * out_cs; p.out_rs = n_out; p.out_step = 1;
            p.n = n_out; p.m = nb;
            ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * 5 * (size_t)n_out * nq * nb, 1);
            ring_stride_coeff_kernel<<<grid_of(n_out, nq, nb), 256, 0, st>>>(p);
        }
        LGPU_CUDA_OK(cudaGetLastError());
    }
    return 0;
}

}  // namespace
}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_evaluator_apply_evaluation_key(lgpu_ctx* ctx, const uint64_t* ct_in, int log_n_in, int level_in, int is_ntt, const lgpu_gadget_ct* evk,
                                        uint64_t* ct_out, int log_n_out, int level_out, int batch, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(log_n_in >= 4 && log_n_out >= 4 && log_n_in <= 17 && log_n_out <= 17, "ApplyEvaluationKey: ring degrees must be powers of two in [2^4, 2^17]");
    const int n_in = 1 << log_n_in, n_out = 1 << log_n_out;
    if (n_in < n_out) REQUIRE(n_out == c.N, "cannot ApplyEvaluationKey: opOut ring degree does not match evaluator params ring degree");
    else if (n_in > n_out) REQUIRE(n_in == c.N, "cannot ApplyEvaluationKey: ctIn ring degree does not match evaluator params ring degree");
    else REQUIRE(n_in == c.N, "cannot ApplyEvaluationKey: ctIn and opOut ring degree does not match evaluator params ring degree");
    REQUIRE(n_in == n_out || c.ring_type == 0, "ApplyEvaluationKey: ring-degree switching is only supported for ring.Type = ring.Standard");
    REQUIRE(level_in >= 0 && level_in < c.nQ && level_out >= 0 && level_out < c.nQ, "level out of range");
    REQUIRE(is_ntt == 0 || is_ntt == 1, "is_ntt must be 0 or 1");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    const size_t in_b = (size_t)2 * (level_in + 1) * n_in * 8 * batch, out_b = (size_t)2 * (level_out + 1) * n_out * 8 * batch;
    if (!(n_in == n_out && ct_in == ct_out && level_in == level_out))
        REQUIRE(!overlaps(ct_in, in_b, ct_out, out_b), "ct_out overlaps ct_in (only ct_out == ct_in at the same degree and level is allowed)");
    GadgetCt key;
    if (to_gadget_ct(evk, key)) return -1;
    const int level = std::min(level_in, level_out);
    if (check_evk(&c, level, key)) return -1;
    REQUIRE(key.levelP <= 0 || key.pw2 == 0, "BaseTwoDecomposition != 0 requires levelP <= 0");
    REQUIRE_DEVICE(ctx);
    return apply_run(&c, (const u64*)ct_in, n_in, level_in, is_ntt != 0, key, (u64*)ct_out, n_out, level_out, batch, (cudaStream_t)stream);
}

}  // extern "C"

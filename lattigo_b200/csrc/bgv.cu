// bgv.cu -- bgv.Evaluator.MulRelin (BGV, tensorStandard) and MulRelinScaleInvariant (BFV, tensorScaleInvariant) for batches of
// degree-1 NTT-domain ciphertexts (schemes/bgv/evaluator.go:529-556, :592-667, :806-864, :898-1070), + Rescale (:1363-1393).
//
// lgpu_bgv holds what bgv.NewParameters / newEvaluatorPrecomp add to the rlwe parameters (params.go:98-109, evaluator.go:38-70): t,
// tMontgomery, levelQMul[] and a second context over (Q, QMul). That context's "P ring" is ringQMul, so its muc_QtoP / muc_PtoQ /
// mdc_QtoP tables are basisExtenderQ1toQ2's constants and the NTT / basis-extension launchers run on QMul unchanged.
//
// Per sub-batch (batch_chunk() ciphertexts):
//   BGV  rns_tensor_kernel<MRed by tMontgomery> over the Q rows -> mulrelin_tail (relinearize, rescale), as for CKKS.
//   BFV  modUpAndNTT: INTT(Q) -> ModUpQtoP -> NTT(QMul) per operand (2 polynomials each, one launch per step and operand);
//        rns_tensor_kernel<MForm> over the Q rows and the QMul rows in one launch; INTT of the three products in Q and in QMul;
//        bfv_quantize_kernel (ModDownQPtoP -> ModUpPtoQ -> x t per coefficient, the QMul value stays in registers); NTT(Q);
//        mulrelin_tail.
// Canonical transforms stand in for the reference's NTTLazy / INTTLazy: DESIGN.md §3.4 gives the argument.
#include <algorithm>
#include <cstring>
#include <vector>
#include "bgv.h"
#include "composite.h"
#include "modarith.cuh"

namespace lgpu {

// ---------------------------------------------------------------------------------------------------------
// Tensor
// ---------------------------------------------------------------------------------------------------------
struct TensorSeg {            // one RNS basis: operands [batch][2][rows][N], products [3][batch][rows][N]
    const u64* a; const u64* b; size_t in_cs, in_bs;
    u64* d; size_t out_cs, out_bs;
};
struct RnsTensorParams {
    const LimbConst* limbs;
    RowMap rm;                // launch row -> global limb, data row within its segment
    int nq;                   // launch rows [0, nq) read / write seg[0], the rest seg[1]
    TensorSeg seg[2];
    const u64* pre;           // kTMul: per launch row, tMontgomery of its limb
    int n;
};
// c00 = Pre(a0), c01 = Pre(a1); d0 = MRed(c00, b0), d2 = MRed(c01, b1), d1 = MRed(c00, b1) + MRed(c01, b0) (squaring: 2 MRed(c00, a1)),
// all canonical. Pre = MForm (BFV, tensorLowDeg :1013-1022) or MRed(., tMontgomery_i) (BGV, MulRNSScalarMontgomery :634-635).
template <bool kTMul, bool kSquare>
__global__ void __launch_bounds__(256) rns_tensor_kernel(RnsTensorParams p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i * 2 >= p.n) return;
    const int r = blockIdx.y;
    const TensorSeg& S = p.seg[r < p.nq ? 0 : 1];
    const LimbConst& L = p.limbs[p.rm.limb[r]];
    const u64 q = L.q, qinv = L.qinv;
    const size_t off = (size_t)blockIdx.z * S.in_bs + (size_t)p.rm.drow[r] * p.n;
    const size_t ooff = (size_t)blockIdx.z * S.out_bs + (size_t)p.rm.drow[r] * p.n;
    const ulonglong2 a0 = reinterpret_cast<const ulonglong2*>(S.a + off)[i];
    const ulonglong2 a1 = reinterpret_cast<const ulonglong2*>(S.a + off + S.in_cs)[i];
    ulonglong2 b0 = a0, b1 = a1;
    if (!kSquare) {
        b0 = reinterpret_cast<const ulonglong2*>(S.b + off)[i];
        b1 = reinterpret_cast<const ulonglong2*>(S.b + off + S.in_cs)[i];
    }
    const u64 tm = kTMul ? p.pre[r] : 0;
    auto pre = [&](u64 x) { return kTMul ? mred(x, tm, q, qinv) : mform(x, q, L.bred_hi, L.bred_lo); };
    ulonglong2 d0, d1, d2;
    {
        const u64 m0 = pre(a0.x), m1 = pre(a1.x);
        d0.x = mred(m0, b0.x, q, qinv); d2.x = mred(m1, b1.x, q, qinv);
        const u64 x = mred(m0, b1.x, q, qinv);
        d1.x = cred(x + (kSquare ? x : mred(m1, b0.x, q, qinv)), q);
    }
    {
        const u64 m0 = pre(a0.y), m1 = pre(a1.y);
        d0.y = mred(m0, b0.y, q, qinv); d2.y = mred(m1, b1.y, q, qinv);
        const u64 x = mred(m0, b1.y, q, qinv);
        d1.y = cred(x + (kSquare ? x : mred(m1, b0.y, q, qinv)), q);
    }
    reinterpret_cast<ulonglong2*>(S.d + ooff)[i] = d0;
    reinterpret_cast<ulonglong2*>(S.d + ooff + S.out_cs)[i] = d1;
    reinterpret_cast<ulonglong2*>(S.d + ooff + 2 * S.out_cs)[i] = d2;
}

static int launch_rns_tensor(const RnsTensorParams& p, bool tmul, bool square, int batch, cudaStream_t st) {
    ProfScope ps(LGPU_KCLASS_TENSOR, st, 8.0 * p.n * p.rm.nrows * batch * (square ? 5 : 7), 1);
    dim3 grid((p.n / 2 + 255) / 256, p.rm.nrows, batch);
    if (tmul) {
        if (square) rns_tensor_kernel<true, true><<<grid, 256, 0, st>>>(p);
        else        rns_tensor_kernel<true, false><<<grid, 256, 0, st>>>(p);
    } else {
        if (square) rns_tensor_kernel<false, true><<<grid, 256, 0, st>>>(p);
        else        rns_tensor_kernel<false, false><<<grid, 256, 0, st>>>(p);
    }
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Quantize (evaluator.go:1050-1070 between its INTTLazy and its NTT), one thread per coefficient:
//   stage 1  ModDownQPtoP(level, lm, xQ, xQMul, .) (ring/basis_extension.go:262-278): ext_j = ModUpQtoP(xQ)_j (the reference's exact
//            representative: reconstructRNS + multSum + SubScalarBigint, as basisext.cu), z_j = MRed(ext_j + 2 p_j - xQMul_j, p_j - mdc_j)
//   stage 2  ModUpPtoQ(lm, level, z, .) (:195-209), then MulScalar(t): out_i = MRed(ModUpPtoQ(z)_i, MForm(t mod q_i))
// The float-v sums run over the sources in limb order with IEEE double division and no FMA, like modup_kernel.
// ---------------------------------------------------------------------------------------------------------
struct QuantParams {
    const LimbConst* limbs;   // of the (Q, QMul) context
    const u64* blob;
    const u64* lvl;           // this level's block of d_const
    const u64* tmul;          // MForm(t mod q_i)
    const u64* xq; size_t xq_bs;     // INTT of the Q products, nq rows N apart
    const u64* xm; size_t xm_bs;     // INTT of the QMul products, nm rows
    u64* out; size_t out_bs;         // nq rows (may alias xq: each thread reads its coefficient before writing it)
    int nq, nm, nQ, n;
    size_t c1_cinv, c1_c, c1_v;      // ModUpConstants Q[:nq] -> QMul (muc_QtoP[level]); target row j, ld nq / nq + 1
    size_t c2_cinv, c2_c, c2_v;      // ModUpConstants QMul[:nm] -> Q (muc_PtoQ[lm]); target row i, ld nm / nm + 1
};

static size_t quant_smem_words(int nq, int nm) {
    return (size_t)4 * nq + (size_t)nm * (4 + 2 * nq + 1) + (size_t)2 * nm + (size_t)nq * (4 + 2 * nm + 1);
}

template <int NM>
__global__ void __launch_bounds__(128) bfv_quantize_kernel(QuantParams p) {
    extern __shared__ u64 sm[];
    const int nq = p.nq, nm = p.nm;
    const int rec1 = 4 + 2 * nq + 1, rec2 = 4 + 2 * nm + 1;
    u64* S1 = sm;                       // [nq][4]  q, qinv, floor(Q/2) mod q, (Q/q_i)^-1 mont
    u64* T1 = S1 + 4 * nq;              // [nm][rec1]  p, pinv, floor(Q/2) mod p, p - mdc, c[nq], vtimes[nq + 1]
    u64* S2 = T1 + (size_t)nm * rec1;   // [nm][2]  floor(QMul/2) mod p, (QMul/p_j)^-1 mont
    u64* T2 = S2 + 2 * nm;              // [nq][rec2]  q, qinv, floor(QMul/2) mod q, MForm(t), c[nm], vtimes[nm + 1]
    const u64* half1_s = p.lvl;
    const u64* half2_t = half1_s + nq;
    const u64* half1_t = half2_t + nq;
    const u64* mdcs = half1_t + nm;
    const u64* half2_s = mdcs + nm;
    for (int k = threadIdx.x; k < 4 * nq; k += blockDim.x) {
        const int i = k >> 2, f = k & 3;
        S1[k] = f == 0 ? p.limbs[i].q : f == 1 ? p.limbs[i].qinv : f == 2 ? half1_s[i] : p.blob[p.c1_cinv + i];
    }
    for (int k = threadIdx.x; k < nm * rec1; k += blockDim.x) {
        const int j = k / rec1, f = k - j * rec1;
        const LimbConst& L = p.limbs[p.nQ + j];
        T1[k] = f == 0 ? L.q : f == 1 ? L.qinv : f == 2 ? half1_t[j] : f == 3 ? mdcs[j]
              : f < 4 + nq ? p.blob[p.c1_c + (size_t)j * nq + (f - 4)] : p.blob[p.c1_v + (size_t)j * (nq + 1) + (f - 4 - nq)];
    }
    for (int k = threadIdx.x; k < 2 * nm; k += blockDim.x) {
        const int j = k >> 1;
        S2[k] = (k & 1) ? p.blob[p.c2_cinv + j] : half2_s[j];
    }
    for (int k = threadIdx.x; k < nq * rec2; k += blockDim.x) {
        const int i = k / rec2, f = k - i * rec2;
        T2[k] = f == 0 ? p.limbs[i].q : f == 1 ? p.limbs[i].qinv : f == 2 ? half2_t[i] : f == 3 ? p.tmul[i]
              : f < 4 + nm ? p.blob[p.c2_c + (size_t)i * nm + (f - 4)] : p.blob[p.c2_v + (size_t)i * (nm + 1) + (f - 4 - nm)];
    }
    __syncthreads();
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= p.n) return;
    const size_t b = blockIdx.z;
    // stage 1: sum_i y_i * (Q/q_i mod p_j) accumulated per target while the sources stream by
    u64 hi[NM], lo[NM];
#pragma unroll
    for (int j = 0; j < NM; j++) { hi[j] = 0; lo[j] = 0; }
    double vs = 0.0;
    const u64* xq = p.xq + b * p.xq_bs + x;
    for (int i = 0; i < nq; i++) {
        const u64* R = S1 + 4 * i;
        const u64 yi = mred(xq[(size_t)i * p.n] + R[2], R[3], R[0], R[1]);
        vs = __dadd_rn(vs, __ddiv_rn(__ull2double_rn(yi), __ull2double_rn(R[0])));
#pragma unroll
        for (int j = 0; j < NM; j++) {
            if (j < nm) {
                u64 mhi, mlo;
                mul128(yi, T1[(size_t)j * rec1 + 4 + i], mhi, mlo);
                lo[j] += mlo;
                hi[j] += mhi + (lo[j] < mlo);
            }
        }
    }
    int v = (int)__double2ull_rz(vs);
    const u64* xm = p.xm + b * p.xm_bs + x;
    u64 z[NM];
    double vs2 = 0.0;
#pragma unroll
    for (int j = 0; j < NM; j++) {
        z[j] = 0;
        if (j < nm) {
            const u64* R = T1 + (size_t)j * rec1;
            const u64 pj = R[0], pinv = R[1];
            u64 r = hi[j] - mulhi64(lo[j] * pinv, pj) + pj + R[4 + nq + v];   // multSum
            r = cred(r + pj - R[2], pj);                                      // SubScalarBigint(Q/2)
            const u64 zj = mred(r + 2 * pj - xm[(size_t)j * p.n], R[3], pj, pinv);   // SubThenMulScalarMontgomeryTwoModulus
            // stage 2 source: y_j = MRed(z_j + floor(QMul/2), (QMul/p_j)^-1 mont)
            z[j] = mred(zj + S2[2 * j], S2[2 * j + 1], pj, pinv);
            vs2 = __dadd_rn(vs2, __ddiv_rn(__ull2double_rn(z[j]), __ull2double_rn(pj)));
        }
    }
    v = (int)__double2ull_rz(vs2);
    u64* out = p.out + b * p.out_bs + x;
    for (int i = 0; i < nq; i++) {
        const u64* R = T2 + (size_t)i * rec2;
        const u64 q = R[0], qinv = R[1];
        u64 rhi = 0, rlo = 0;
#pragma unroll
        for (int j = 0; j < NM; j++) {
            if (j < nm) {
                u64 mhi, mlo;
                mul128(z[j], R[4 + j], mhi, mlo);
                rlo += mlo;
                rhi += mhi + (rlo < mlo);
            }
        }
        u64 r = rhi - mulhi64(rlo * qinv, q) + q + R[4 + nm + v];   // multSum
        r = cred(r + q - R[2], q);                                  // SubScalarBigint(QMul/2)
        out[(size_t)i * p.n] = mred(r, R[3], q, qinv);              // MulScalar(t)
    }
}

static int launch_quantize(const QuantParams& p, int batch, cudaStream_t st) {
    ProfScope ps(LGPU_KCLASS_MODUP, st, 8.0 * p.n * batch * (2 * p.nq + p.nm), 1);
    const size_t smem = quant_smem_words(p.nq, p.nm) * sizeof(u64);
    if (smem > 200 * 1024) { set_error("quantize: constant set too large for shared memory"); return -1; }
    dim3 grid((p.n + 127) / 128, 1, batch);
    auto go = [&](auto kern) {
        if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        kern<<<grid, 128, smem, st>>>(p);
    };
    if (p.nm <= 4)       go(bfv_quantize_kernel<4>);
    else if (p.nm <= 8)  go(bfv_quantize_kernel<8>);
    else if (p.nm <= 16) go(bfv_quantize_kernel<16>);
    else                 go(bfv_quantize_kernel<32>);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------------------------------------
// Sub-batches
// ---------------------------------------------------------------------------------------------------------
static RnsTensorParams tensor_params(const LimbConst* limbs, int n) {
    RnsTensorParams p;
    memset(&p, 0, sizeof(p));
    p.limbs = limbs; p.n = n;
    return p;
}

// tensorStandard with relinearization (+ Rescale)
static int bgv_chunk(const Ctx* c, const BgvState& s, int level, const u64* A, const u64* B, const GadgetCt& rlk, int nb_rescales, u64* out,
                     int batch, cudaStream_t st) {
    const size_t N = c->N, nq = level + 1;
    Scratch buf;
    if (buf.alloc((size_t)batch * 5 * nq * N, st)) return -1;   // d0, d1, d2, t0, t1
    RnsTensorParams p = tensor_params(c->d_limbs, c->N);
    p.rm = rows_range(0, 0, (int)nq); p.nq = (int)nq;
    p.seg[0] = TensorSeg{A, B, nq * N, 2 * nq * N, buf.p, (size_t)batch * nq * N, nq * N};
    p.pre = s.tmont();
    if (launch_rns_tensor(p, true, A == B, batch, st)) return -1;
    return mulrelin_tail(c, level, buf.p, rlk, nb_rescales, out, batch, st);
}

// tensorScaleInvariant up to the degree-2 product (bgv.h)
int bfv_tensor(const Ctx* c, const BgvState& s, int level, const u64* A, const u64* B, u64* d, int batch, cudaStream_t st) {
    const Ctx* m = &s.qm;
    const int lm = s.levelQMul[level];
    const size_t N = c->N, nq = level + 1, nm = lm + 1;
    const bool square = A == B;
    Scratch mbuf;
    if (mbuf.alloc((size_t)batch * 7 * nm * N, st)) return -1;            // QMul: extA [2], extB [2], products [3]
    u64* tmp = d + (size_t)3 * batch * nq * N;                             // INTT of one operand
    u64* ext[2] = {mbuf.p, mbuf.p + (size_t)2 * batch * nm * N};
    u64* dm = mbuf.p + (size_t)4 * batch * nm * N;
    const RowMap rq = rows_range(0, 0, (int)nq), rmul = rows_range(m->nQ, 0, (int)nm);
    // modUpAndNTT (:991-1001): both polynomials of an operand per launch
    for (int k = 0; k < (square ? 1 : 2); k++) {
        const u64* src = k == 0 ? A : B;
        if (launch_intt(c, rq, CSpan{src, N, nq * N}, Span{tmp, N, nq * N}, 2 * batch, NTT_CANONICAL, st)) return -1;
        if (launch_modup_qp(m, true, level, lm, CSpan{tmp, N, nq * N}, Span{ext[k], N, nm * N}, 2 * batch, st)) return -1;
        if (launch_ntt(m, rmul, CSpan{ext[k], N, nm * N}, Span{ext[k], N, nm * N}, 2 * batch, NTT_CANONICAL, st)) return -1;
    }
    // tensorLowDeg (:1003-1048): Q rows then QMul rows in one launch
    RnsTensorParams p = tensor_params(m->d_limbs, c->N);
    p.rm.nrows = (int)(nq + nm); p.nq = (int)nq;
    for (size_t i = 0; i < nq; i++) { p.rm.limb[i] = (unsigned char)i; p.rm.drow[i] = (unsigned char)i; }
    for (size_t j = 0; j < nm; j++) { p.rm.limb[nq + j] = (unsigned char)(m->nQ + j); p.rm.drow[nq + j] = (unsigned char)j; }
    p.seg[0] = TensorSeg{A, B, nq * N, 2 * nq * N, d, (size_t)batch * nq * N, nq * N};
    p.seg[1] = TensorSeg{ext[0], square ? ext[0] : ext[1], nm * N, 2 * nm * N, dm, (size_t)batch * nm * N, nm * N};
    if (launch_rns_tensor(p, false, square, batch, st)) return -1;
    // quantize (:1050-1070) on the three products
    if (launch_intt(c, rq, CSpan{d, N, nq * N}, Span{d, N, nq * N}, 3 * batch, NTT_CANONICAL, st)) return -1;
    if (launch_intt(m, rmul, CSpan{dm, N, nm * N}, Span{dm, N, nm * N}, 3 * batch, NTT_CANONICAL, st)) return -1;
    QuantParams q;
    memset(&q, 0, sizeof(q));
    q.limbs = m->d_limbs; q.blob = m->d_blob; q.lvl = s.d_const + s.lvl_off[level]; q.tmul = s.d_const;
    q.xq = d; q.xq_bs = nq * N; q.xm = dm; q.xm_bs = nm * N; q.out = d; q.out_bs = nq * N;
    q.nq = (int)nq; q.nm = (int)nm; q.nQ = m->nQ; q.n = c->N;
    const ModUpSet& u1 = m->muc_QtoP[level];
    const ModUpSet& u2 = m->muc_PtoQ[lm];
    q.c1_cinv = u1.off_qoverqiinvqi; q.c1_c = u1.off_qoverqimodp; q.c1_v = u1.off_vtimesqmodp;
    q.c2_cinv = u2.off_qoverqiinvqi; q.c2_c = u2.off_qoverqimodp; q.c2_v = u2.off_vtimesqmodp;
    if (launch_quantize(q, 3 * batch, st)) return -1;
    return launch_ntt(c, rq, CSpan{d, N, nq * N}, Span{d, N, nq * N}, 3 * batch, NTT_CANONICAL, st);
}

// tensorScaleInvariant with relinearization
static int bfv_chunk(const Ctx* c, const BgvState& s, int level, const u64* A, const u64* B, const GadgetCt& rlk, u64* out, int batch,
                     cudaStream_t st) {
    Scratch buf;
    if (buf.alloc((size_t)batch * 5 * (level + 1) * c->N, st)) return -1;   // d0, d1, d2, t0, t1
    if (bfv_tensor(c, s, level, A, B, buf.p, batch, st)) return -1;
    return mulrelin_tail(c, level, buf.p, rlk, 0, out, batch, st);
}

// number of bits of prod(mods[0..n)), as big.Int.BitLen
static int prod_bitlen(const u64* mods, int n) {
    std::vector<u64> w(1, 1);
    for (int i = 0; i < n; i++) {
        unsigned __int128 carry = 0;
        for (auto& x : w) {
            const unsigned __int128 t = (unsigned __int128)x * mods[i] + carry;
            x = (u64)t;
            carry = t >> 64;
        }
        if (carry) w.push_back((u64)carry);
    }
    return 64 * (int)(w.size() - 1) + (64 - __builtin_clzll(w.back()));
}

}  // namespace lgpu

using namespace lgpu;

extern "C" {

int lgpu_bgv_create(lgpu_ctx* ctx, uint64_t t, const uint64_t* qmul, int nqmul, lgpu_bgv** out) {
    REQUIRE(ctx && out, "null argument");
    REQUIRE(qmul && nqmul > 0, "empty QMul chain");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "BGV / BFV multiplication requires the Standard ring");
    REQUIRE(t >= 2, "plaintext modulus t must be >= 2");
    REQUIRE(t < c.Q[0], "plaintext modulus t must be smaller than Q[0]");
    for (int i = 0; i < c.nQ; i++) REQUIRE(c.Q[i] != t, "insecure parameters: t|Q");
    for (int j = 0; j < nqmul; j++)
        for (int i = 0; i < c.nQ; i++) REQUIRE(c.Q[i] != qmul[j], "a QMul modulus is also a modulus of Q");
    std::vector<int> lq(c.nQ);
    for (int l = 0; l < c.nQ; l++) lq[l] = (prod_bitlen(c.Q.data(), l + 1) + c.logN + 60) / 61 - 1;   // evaluator.go:43-48
    REQUIRE(nqmul >= lq[c.nQ - 1] + 1, "QMul has fewer moduli than levelQMul[MaxLevel] + 1");
    REQUIRE(lq[c.nQ - 1] + 1 <= 32, "more than 32 QMul moduli per level are not supported");
    lgpu_bgv* ev = new lgpu_bgv;
    ev->ctx = ctx;
    BgvState& s = ev->s;
    if (build_context(&s.qm, c.device, c.logN, 0, c.Q.data(), c.nQ, (const u64*)qmul, nqmul, false)) {
        destroy_context(&s.qm);
        delete ev;
        return -1;
    }
    s.t = t;
    s.levelQMul = lq;
    const Ctx& m = s.qm;
    std::vector<u64>& h = s.h_const;
    for (int i = 0; i < c.nQ; i++) h.push_back(h_mform(t % c.Q[i], c.Q[i]));
    for (int i = 0; i < c.nQ; i++) h.push_back(h_mform(h[i], c.Q[i]));
    s.lvl_off.resize(c.nQ);
    for (int l = 0; l < c.nQ; l++) {
        const int nq = l + 1, nm = lq[l] + 1;
        const u64* Q = c.Q.data();
        const u64* PM = m.P.data();
        s.lvl_off[l] = h.size();
        for (int i = 0; i < nq; i++) h.push_back(h_half_prod_mod(Q, nq, Q[i]));
        for (int i = 0; i < nq; i++) h.push_back(h_half_prod_mod(PM, nm, Q[i]));
        for (int j = 0; j < nm; j++) h.push_back(h_half_prod_mod(Q, nq, PM[j]));
        for (int j = 0; j < nm; j++) h.push_back(PM[j] - m.mdc_QtoP[(size_t)l * m.nP + j]);
        for (int j = 0; j < nm; j++) h.push_back(h_half_prod_mod(PM, nm, PM[j]));
    }
    if (c.device >= 0) {
        int rc = 0;
        if (cudaMalloc(&s.d_const, h.size() * sizeof(u64)) != cudaSuccess ||
            cudaMemcpy(s.d_const, h.data(), h.size() * sizeof(u64), cudaMemcpyHostToDevice) != cudaSuccess) {
            set_error("BGV evaluator: device allocation failed");
            rc = -1;
        }
        if (rc) { lgpu_bgv_destroy(ev); return -1; }
    }
    *out = ev;
    return 0;
}

void lgpu_bgv_destroy(lgpu_bgv* ev) {
    if (!ev) return;
    if (ev->s.qm.device >= 0) {
        cudaSetDevice(ev->s.qm.device);
        cudaFree(ev->s.d_const);
    }
    destroy_context(&ev->s.qm);
    delete ev;
}

int lgpu_bgv_mulrelin_batch(lgpu_bgv* ev, int level, const uint64_t* ct_a, const uint64_t* ct_b, const lgpu_gadget_ct* rlk,
                            int scale_invariant, int nb_rescales, uint64_t* ct_out, int batch, void* stream) {
    REQUIRE(ev, "null BGV evaluator");
    REQUIRE_DEVICE(ev->ctx);
    REQUIRE(ct_a && ct_b && ct_out, "null ciphertext");
    REQUIRE_ALIGNED(AL(ct_a) && AL(ct_b) && AL(ct_out));
    REQUIRE(batch >= 1, "batch must be >= 1");
    REQUIRE(scale_invariant == 0 || scale_invariant == 1, "scale_invariant must be 0 or 1");
    const Ctx& c = ev->ctx->c;
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(!scale_invariant || nb_rescales == 0, "the scale-invariant (BFV) multiplication does not rescale: nb_rescales must be 0");
    REQUIRE(!scale_invariant || level + 1 <= kMaxSrc, "the scale-invariant (BFV) multiplication supports at most 64 Q moduli");
    REQUIRE(nb_rescales >= 0 && nb_rescales <= level, "cannot Rescale: input Ciphertext level is too low");
    const size_t N = c.N, nq = level + 1, nqo = nq - nb_rescales;
    const size_t in_bytes = (size_t)batch * 2 * nq * N * 8, out_bytes = (size_t)batch * 2 * nqo * N * 8;
    const bool out_is_a = (const void*)ct_out == (const void*)ct_a && nb_rescales == 0;
    REQUIRE(out_is_a || !overlaps(ct_out, out_bytes, ct_a, in_bytes), "ct_out overlaps ct_a (only ct_out == ct_a without rescale is allowed)");
    REQUIRE((out_is_a && ct_a == ct_b) || !overlaps(ct_out, out_bytes, ct_b, in_bytes), "ct_out overlaps ct_b");
    GadgetCt g;
    if (to_gadget_ct(rlk, g, "null relinearization key")) return -1;
    if (check_evk(&c, level, g)) return -1;
    const cudaStream_t st = (cudaStream_t)stream;
    const u64* A = (const u64*)ct_a;
    const u64* B = (const u64*)ct_b;
    u64* O = (u64*)ct_out;
    const int ch = batch_chunk();
    for (int k = 0; k < batch; k += ch) {
        const int nb = std::min(ch, batch - k);
        const size_t ia = (size_t)k * 2 * nq * N, io = (size_t)k * 2 * nqo * N;
        // a squaring stays a squaring in every sub-batch
        const u64* Bk = A == B ? A + ia : B + ia;
        const int rc = scale_invariant ? bfv_chunk(&c, ev->s, level, A + ia, Bk, g, O + io, nb, st)
                                       : bgv_chunk(&c, ev->s, level, A + ia, Bk, g, nb_rescales, O + io, nb, st);
        if (rc) return -1;
    }
    return 0;
}

}  // extern "C"

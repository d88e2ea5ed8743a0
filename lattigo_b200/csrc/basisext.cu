// basisext.cu -- RNS basis extension kernels.
//
// One per-coefficient kernel implements the reference's fast basis conversion
//     reconstructRNS / reconstructRNSCentered + multSum   (ring/basis_extension.go:504-673)
// for both of its users:
//     BasisExtender.ModUpQtoP / ModUpPtoQ -> ModUpExact    (:177-209, :282-308)
//     Decomposer.DecomposeAndSplit, reconstruction branch   (:438-501)
// Per coefficient:  y_i = MRed(x_i + half_i, (S/s_i)^-1 mont);   v = uint64(sum_i float64(y_i)/float64(s_i))
// (IEEE double, true division, sequential in limb order, no FMA -- a different v is a different answer);
// per target t_j:   out_j = CRed( [sum_i y_i * (S/s_i mod t_j) as uint128 -> one lazy Montgomery reduction]
//                                 + t_j + vtimesqmodp[j][v]  + t_j - (half mod t_j), t_j )
// which reproduces the reference's specific (non-canonical) representative bit for bit.
// Layout: thread = coefficient (coalesced row reads/writes), blockIdx.y = group of targets, blockIdx.z = batch.
#include "../../include/lattigo_b200.h"
#include "engine.h"
#include "modarith.cuh"

namespace lgpu {

struct ModUpParams {
    const LimbConst* limbs;
    const u64* blob;
    // source rows
    const u64* src; size_t src_rs, src_bs;
    int nS;
    unsigned char src_limb[kMaxSrc];
    u64 half_src[kMaxSrc];
    size_t off_qoverqiinvqi;
    // target segment A: rows [0, nA) of outA except [exlo, exhi); global limb = limbA0 + j; constant row = j
    u64* outA; size_t outA_rs, outA_bs; int nA, exlo, exhi, limbA0;
    // target segment B: rows [0, nB) of outB; global limb = limbB0 + j; constant row = crowB0 + j
    u64* outB; size_t outB_rs, outB_bs; int nB, limbB0, crowB0;
    size_t off_qoverqimodp; int ldc;
    size_t off_vtimesqmodp; int ldv;
    u64 half_t[kMaxRows];  // (half mod target), indexed by target ordinal
    int n;                 // coefficients per row
    int tg;                // targets per blockIdx.y
};

// Constants of every target (q, qinv, half, the c_ji row and the vtimesqmodp row) are staged once per CTA in shared
// memory; a thread owns one coefficient, computes y_i and v once and then streams through ALL targets (coalesced
// row stores), so the fp64 divisions and the source loads are not repeated per target group.
template <int NSMAX>
__global__ void __launch_bounds__(256) modup_kernel(ModUpParams p) {
    extern __shared__ u64 sm[];
    const int nT = p.nA + p.nB;
    const int nS = p.nS;
    // per target t: [0] q, [1] qinv, [2] half_t, [3 .. 3+nS) c_ji, [3+nS .. 3+2nS+1) vtimesqmodp row
    const int rec = 3 + 2 * nS + 1;
    for (int idx = threadIdx.x; idx < nT * rec; idx += blockDim.x) {
        const int t = idx / rec, f = idx - t * rec;
        int limb, crow;
        if (t < p.nA) { limb = p.limbA0 + t; crow = t; } else { limb = p.limbB0 + (t - p.nA); crow = p.crowB0 + (t - p.nA); }
        u64 v;
        if (f == 0) v = p.limbs[limb].q;
        else if (f == 1) v = p.limbs[limb].qinv;
        else if (f == 2) v = p.half_t[t];
        else if (f < 3 + nS) v = p.blob[p.off_qoverqimodp + (size_t)crow * p.ldc + (f - 3)];
        else v = p.blob[p.off_vtimesqmodp + (size_t)crow * p.ldv + (f - 3 - nS)];
        sm[idx] = v;
    }
    __syncthreads();
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= p.n) return;
    const int b = blockIdx.z;
    u64 y[NSMAX];
    double vi = 0.0;
    const u64* src = p.src + (size_t)b * p.src_bs + x;
    const u64* cinv = p.blob + p.off_qoverqiinvqi;
#pragma unroll
    for (int i = 0; i < NSMAX; i++) {
        if (i < nS) {
            const LimbConst& L = p.limbs[p.src_limb[i]];
            const u64 q = L.q;
            const u64 xi = src[(size_t)i * p.src_rs];
            const u64 yi = mred(xi + p.half_src[i], cinv[i], q, L.qinv);
            y[i] = yi;
            vi = __dadd_rn(vi, __ddiv_rn(__ull2double_rn(yi), __ull2double_rn(q)));
        } else {
            y[i] = 0;
        }
    }
    const int v = (int)__double2ull_rz(vi);
    const int t0 = blockIdx.y * p.tg;
    const int t1 = min(t0 + p.tg, nT);
#pragma unroll 2
    for (int t = t0; t < t1; t++) {
        u64* dst;
        if (t < p.nA) {
            if (t >= p.exlo && t < p.exhi) continue;
            dst = p.outA + (size_t)b * p.outA_bs + (size_t)t * p.outA_rs + x;
        } else {
            dst = p.outB + (size_t)b * p.outB_bs + (size_t)(t - p.nA) * p.outB_rs + x;
        }
        const u64* R = sm + t * rec;
        const u64 tq = R[0];
        u64 rhi = 0, rlo = 0;
#pragma unroll
        for (int i = 0; i < NSMAX; i++) {
            if (i < nS) {
                u64 mhi, mlo;
                mul128(y[i], R[3 + i], mhi, mlo);
                rlo += mlo;
                rhi += mhi + (rlo < mlo);
            }
        }
        const u64 hhi = mulhi64(rlo * R[1], tq);
        u64 r = rhi - hhi + tq + R[3 + nS + v];     // multSum, ring/basis_extension.go:651
        r = cred(r + tq - R[2], tq);                 // SubScalarBigint
        *dst = r;
    }
}

// Single-limb digit: Decomposer.DecomposeAndSplit fast path, ring/basis_extension.go:402-436.
struct DecompSingleParams {
    const LimbConst* limbs;
    const u64* src; size_t src_bs;   // the digit's single row
    u64 qsrc;
    u64* outA; size_t outA_rs, outA_bs; int nA, limbA0;
    u64* outB; size_t outB_rs, outB_bs; int nB, limbB0;
    int n;
};
__global__ void __launch_bounds__(256) decomp_single_kernel(DecompSingleParams p) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= p.n) return;
    const int b = blockIdx.z;
    u64 coeff = p.src[(size_t)b * p.src_bs + x];
    bool neg = false;
    if (coeff >= (p.qsrc >> 1)) { coeff = p.qsrc - coeff; neg = true; }
    const int nT = p.nA + p.nB;
    for (int t = blockIdx.y; t < nT; t += gridDim.y) {
        int limb; u64* dst;
        if (t < p.nA) { limb = p.limbA0 + t; dst = p.outA + (size_t)b * p.outA_bs + (size_t)t * p.outA_rs + x; }
        else { const int j = t - p.nA; limb = p.limbB0 + j; dst = p.outB + (size_t)b * p.outB_bs + (size_t)j * p.outB_rs + x; }
        const LimbConst& L = p.limbs[limb];
        const u64 tmp = bred_add(coeff, L.q, L.bred_hi);
        *dst = neg ? (L.q - tmp) : tmp;     // tmp*pos + (q - tmp)*neg
    }
}

// all targets in one group (y_i and v computed once per coefficient) as soon as coefficients x batch fill the GPU
static int target_group(const Ctx* c, int nT, int batch) {
    const long ctas = (long)((c->N + 255) / 256) * batch;
    const long want = 4L * c->sms;
    if (ctas >= want) return nT;
    int groups = (int)((want + ctas - 1) / ctas);
    int tg = (nT + groups - 1) / groups;
    return tg < 1 ? 1 : tg;
}

static int launch_modup(const ModUpParams& p, int batch, cudaStream_t st) {
    const int nT = p.nA + p.nB;
    ProfScope ps(LGPU_KCLASS_MODUP, st, 8.0 * p.n * batch * (p.nS + nT - (p.exhi - p.exlo)), 1);
    dim3 grid((p.n + 255) / 256, (nT + p.tg - 1) / p.tg, batch);
    const size_t smem = (size_t)nT * (3 + 2 * p.nS + 1) * sizeof(u64);
    if (smem > 200 * 1024) { set_error("basis extension: constant set too large for shared memory"); return -1; }
    auto go = [&](auto kern) {
        if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        kern<<<grid, 256, smem, st>>>(p);
    };
    if (p.nS <= 4)       go(modup_kernel<4>);
    else if (p.nS <= 8)  go(modup_kernel<8>);
    else if (p.nS <= 16) go(modup_kernel<16>);
    else                 go(modup_kernel<kMaxSrc>);
    LGPU_CUDA_OK(cudaGetLastError());
    return 0;
}

// ---- public launchers ------------------------------------------------------------------------------------

// ModUpQtoP (toP = true): polQ rows 0..levelQ -> polP rows 0..levelP ; ModUpPtoQ (toP = false): the converse.
int launch_modup_qp(const Ctx* c, bool toP, int levelQ, int levelP, CSpan in, Span out, int batch, cudaStream_t st) {
    if (c->nP == 0) { set_error("basis extension requires a P ring"); return -1; }
    if (levelQ < 0 || levelQ >= c->nQ || levelP < 0 || levelP >= c->nP) { set_error("level out of range"); return -1; }
    ModUpParams p;
    memset(&p, 0, sizeof(p));
    p.limbs = c->d_limbs; p.blob = c->d_blob; p.n = c->N;
    p.src = in.p; p.src_rs = in.row_stride; p.src_bs = in.batch_stride;
    const ModUpSet& m = toP ? c->muc_QtoP[levelQ] : c->muc_PtoQ[levelP];
    const std::vector<u64>& S = toP ? c->Q : c->P;
    const std::vector<u64>& T = toP ? c->P : c->Q;
    p.nS = (toP ? levelQ : levelP) + 1;
    if (p.nS > kMaxSrc) { set_error("too many source limbs"); return -1; }
    const int nT = (toP ? levelP : levelQ) + 1;
    for (int i = 0; i < p.nS; i++) {
        p.src_limb[i] = (unsigned char)((toP ? 0 : c->nQ) + i);
        p.half_src[i] = h_half_prod_mod(S.data(), p.nS, S[i]);
    }
    for (int j = 0; j < nT; j++) p.half_t[j] = h_half_prod_mod(S.data(), p.nS, T[j]);
    p.off_qoverqiinvqi = m.off_qoverqiinvqi; p.off_qoverqimodp = m.off_qoverqimodp; p.ldc = m.nS;
    p.off_vtimesqmodp = m.off_vtimesqmodp; p.ldv = m.nS + 1;
    if (toP) {
        p.nA = 0; p.exlo = p.exhi = 0;
        p.outB = out.p; p.outB_rs = out.row_stride; p.outB_bs = out.batch_stride; p.nB = nT; p.limbB0 = c->nQ; p.crowB0 = 0;
    } else {
        p.outA = out.p; p.outA_rs = out.row_stride; p.outA_bs = out.batch_stride; p.nA = nT; p.limbA0 = 0; p.exlo = p.exhi = 0;
        p.nB = 0;
    }
    p.tg = target_group(c, nT, batch);
    return launch_modup(p, batch, st);
}

// Decomposer.DecomposeAndSplit (ring/basis_extension.go:381-502). p0Q: coefficient-domain input (levelQ+1 rows);
// p1Q (levelQ+1 rows) / p1P (levelP+1 rows): outputs. The digit's own rows of p1Q are left untouched in the
// reconstruction branch except for the reference's trailing SubScalarBigint -- callers (DecomposeSingleNTT)
// overwrite them; we simply do not write them.
int launch_decompose_and_split(const Ctx* c, int levelQ, int levelP, int nbPi, int digit, CSpan p0Q, Span p1Q, Span p1P,
                               int batch, cudaStream_t st) {
    if (levelQ < 0 || levelQ >= c->nQ || levelP < -1 || levelP >= c->nP) { set_error("level out of range"); return -1; }
    const int lvlQStart = digit * nbPi;
    int decompLvl;
    if (levelQ > nbPi * (digit + 1) - 1) decompLvl = nbPi - 2;
    else decompLvl = (nbPi > 0 ? (levelQ % nbPi) : 0) - 1;
    if (lvlQStart > levelQ || lvlQStart < 0) { set_error("decomposition digit out of range"); return -1; }
    if (decompLvl < 0) {
        DecompSingleParams p;
        memset(&p, 0, sizeof(p));
        p.limbs = c->d_limbs; p.n = c->N;
        p.src = p0Q.p + (size_t)lvlQStart * p0Q.row_stride; p.src_bs = p0Q.batch_stride;
        p.qsrc = c->Q[lvlQStart];
        p.outA = p1Q.p; p.outA_rs = p1Q.row_stride; p.outA_bs = p1Q.batch_stride; p.nA = levelQ + 1; p.limbA0 = 0;
        p.outB = p1P.p; p.outB_rs = p1P.row_stride; p.outB_bs = p1P.batch_stride; p.nB = levelP + 1; p.limbB0 = c->nQ;
        const int nT = p.nA + p.nB;
        ProfScope ps(LGPU_KCLASS_MODUP, st, 8.0 * p.n * batch * (1 + nT), 1);
        dim3 grid((p.n + 255) / 256, nT < 8 ? nT : 8, batch);
        decomp_single_kernel<<<grid, 256, 0, st>>>(p);
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }
    if (nbPi < 2 || nbPi - 2 >= (int)c->muc_dec.size() || digit >= (int)c->muc_dec[nbPi - 2].size() ||
        decompLvl >= (int)c->muc_dec[nbPi - 2][digit].size()) { set_error("no decomposer constants for this (nbPi, digit, level)"); return -1; }
    const ModUpSet& m = c->muc_dec[nbPi - 2][digit][decompLvl];
    const int p0idxst = lvlQStart;
    int p0idxed = p0idxst + nbPi;
    if (p0idxed > levelQ + 1) p0idxed = levelQ + 1;
    ModUpParams p;
    memset(&p, 0, sizeof(p));
    p.limbs = c->d_limbs; p.blob = c->d_blob; p.n = c->N;
    p.src = p0Q.p + (size_t)p0idxst * p0Q.row_stride; p.src_rs = p0Q.row_stride; p.src_bs = p0Q.batch_stride;
    p.nS = p0idxed - p0idxst;
    const u64* D = c->Q.data() + p0idxst;
    for (int i = 0; i < p.nS; i++) {
        p.src_limb[i] = (unsigned char)(p0idxst + i);
        p.half_src[i] = h_half_prod_mod(D, p.nS, D[i]);
    }
    p.off_qoverqiinvqi = m.off_qoverqiinvqi; p.off_qoverqimodp = m.off_qoverqimodp; p.ldc = m.nS;
    p.off_vtimesqmodp = m.off_vtimesqmodp; p.ldv = m.nS + 1;
    p.outA = p1Q.p; p.outA_rs = p1Q.row_stride; p.outA_bs = p1Q.batch_stride; p.nA = levelQ + 1; p.limbA0 = 0;
    p.exlo = p0idxst; p.exhi = p0idxed;
    p.outB = p1P.p; p.outB_rs = p1P.row_stride; p.outB_bs = p1P.batch_stride; p.nB = levelP + 1; p.limbB0 = c->nQ; p.crowB0 = c->nQ;
    for (int j = 0; j <= levelQ; j++) p.half_t[j] = h_half_prod_mod(D, p.nS, c->Q[j]);
    for (int j = 0; j <= levelP; j++) p.half_t[p.nA + j] = h_half_prod_mod(D, p.nS, c->P[j]);
    p.tg = target_group(c, p.nA + p.nB, batch);
    return launch_modup(p, batch, st);
}

}  // namespace lgpu

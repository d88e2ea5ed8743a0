// lintrans.cu -- hoisted linear transformations on the device (SURVEY 8(f) rank 1: the caller right above the key-switch
// path). Restates, for a BATCH of ciphertexts sharing one plaintext matrix,
//   lintrans.Evaluator.EvaluateMany                                        circuits/common/lintrans/lintrans_evaluator.go:28-79
//   PreRotatedCiphertextForDiagonalMatrixMultiplication                     :82-114
//   MultiplyByDiagMatrix      (single hoisting, one key per diagonal)       :141-274
//   MultiplyByDiagMatrixBSGS  (double hoisting, baby-step giant-step)       :280-470
//   rlwe.Evaluator.AutomorphismHoistedLazy                                  core/rlwe/evaluator_automorphism.go:107-165
//   lintrans.BSGSIndex                                                      circuits/common/lintrans/lintrans.go:344-367
//
// Every output of these methods is a canonical residue vector that depends on its inputs only through residue classes
// (the reference's lazy accumulations never overflow by construction: QiOverflowMargin / PiOverflowMargin), so the device
// code is free to fuse: the inner baby-step sum is ONE kernel over all (diagonal, pre-rotated ciphertext) pairs of a giant
// step instead of 4 MulCoeffsMontgomeryLazyThenAddLazy passes per pair, and the naive evaluator folds the automorphism
// gather into its multiply-accumulate. Results equal the reference bit for bit (tests/test_gpu_lintrans.py vs
// oracle/lintrans.py).
#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <vector>
#include "../../include/lattigo_b200.h"
#include "composite.h"
#include "lintrans.h"
#include "modarith.cuh"

namespace lgpu {

// ---------------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kLtMaxTerms = 20;
struct LtTerm {
    const u64* ptQ; const u64* ptP;       // diagonal rows (NTT + Montgomery), no batch dimension
    const u64* s0Q; const u64* s0P;       // component 0 of the source (P pointer null: the term has no P part)
    const u64* s1Q; const u64* s1P;
    size_t bs;                            // batch stride of the source (words)
};
struct LtInnerParams {
    const LimbConst* limbs;
    LtTerm t[kLtMaxTerms];
    u64* out0; u64* out1; size_t out_bs;  // QP-stacked [batch][nq + np][N]
    int nterms, first, nq, np, nQfull, n, batch;
};
// (t0, t1) (+)= sum_i pt_i (.) src_i, rows = Q limbs then P limbs, canonical result: the inner loop of
// MultiplyByDiagMatrixBSGS (lintrans_evaluator.go:349-407) for one giant step.
__global__ void __launch_bounds__(256) lt_inner_kernel(LtInnerParams p) {
    const int r = blockIdx.y;
    const bool isP = r >= p.nq;
    const int j = isP ? r - p.nq : r;
    const LimbConst L = p.limbs[isP ? p.nQfull + j : j];
    const u64 q = L.q, qinv = L.qinv, twoq = q << 1;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;      // 2-word vector index
    if (i * 2 >= p.n) return;
    const size_t roff = (size_t)j * p.n;
    for (int b = blockIdx.z; b < p.batch; b += gridDim.z) {
        ulonglong2* o0 = reinterpret_cast<ulonglong2*>(p.out0 + (size_t)b * p.out_bs + (size_t)r * p.n);
        ulonglong2* o1 = reinterpret_cast<ulonglong2*>(p.out1 + (size_t)b * p.out_bs + (size_t)r * p.n);
        ulonglong2 a0 = make_ulonglong2(0, 0), a1 = a0;
        if (!p.first) { a0 = o0[i]; a1 = o1[i]; }
        for (int t = 0; t < p.nterms; t++) {
            const LtTerm& T = p.t[t];
            const u64* s0 = isP ? T.s0P : T.s0Q;
            if (!s0) continue;
            const u64* s1 = isP ? T.s1P : T.s1Q;
            const ulonglong2 e = reinterpret_cast<const ulonglong2*>((isP ? T.ptP : T.ptQ) + roff)[i];
            const ulonglong2 x0 = reinterpret_cast<const ulonglong2*>(s0 + (size_t)b * T.bs + roff)[i];
            const ulonglong2 x1 = reinterpret_cast<const ulonglong2*>(s1 + (size_t)b * T.bs + roff)[i];
            a0.x += mred_lazy(e.x, x0.x, q, qinv); a0.y += mred_lazy(e.y, x0.y, q, qinv);
            a1.x += mred_lazy(e.x, x1.x, q, qinv); a1.y += mred_lazy(e.y, x1.y, q, qinv);
            a0.x = a0.x >= twoq ? a0.x - twoq : a0.x; a0.y = a0.y >= twoq ? a0.y - twoq : a0.y;
            a1.x = a1.x >= twoq ? a1.x - twoq : a1.x; a1.y = a1.y >= twoq ? a1.y - twoq : a1.y;
        }
        a0.x = cred(a0.x, q); a0.y = cred(a0.y, q); a1.x = cred(a1.x, q); a1.y = cred(a1.y, q);
        o0[i] = a0; o1[i] = a1;
    }
}

struct LtPermMacParams {
    const LimbConst* limbs;
    const u64* ptQ; const u64* ptP;
    const u64* src0; const u64* src1; size_t src_bs;   // QP-stacked accumulators of the hoisted gadget product
    u64* out0; u64* out1; size_t out_bs;
    const u64* index;
    int first, nq, np, nQfull, n;
};
// c[k][j] (+)= pt[j] * a[k][index[j]]: AutomorphismNTTWithIndex + MulCoeffsMontgomery[ThenAdd] of the naive evaluator
// (lintrans_evaluator.go:222-246) in one pass.
__global__ void __launch_bounds__(256) lt_perm_mac_kernel(LtPermMacParams p) {
    const int r = blockIdx.y;
    const bool isP = r >= p.nq;
    const int jr = isP ? r - p.nq : r;
    const LimbConst L = p.limbs[isP ? p.nQfull + jr : jr];
    const u64 q = L.q, qinv = L.qinv;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const size_t src = p.index ? (size_t)__ldg(p.index + j) : (size_t)j;
    const u64 e = (isP ? p.ptP : p.ptQ)[(size_t)jr * p.n + j];
    const size_t so = (size_t)blockIdx.z * p.src_bs + (size_t)r * p.n, oo = (size_t)blockIdx.z * p.out_bs + (size_t)r * p.n;
    u64 v0 = mred(e, p.src0[so + src], q, qinv), v1 = mred(e, p.src1[so + src], q, qinv);
    if (!p.first) { v0 = cred(v0 + p.out0[oo + j], q); v1 = cred(v1 + p.out1[oo + j], q); }
    p.out0[oo + j] = v0; p.out1[oo + j] = v1;
}

// AutomorphismHoistedLazy in ONE pass (core/rlwe/evaluator_automorphism.go:107-165 = gadgetProductMultiplePLazyHoisted :401-453 + the P * ct0 term +
// AutomorphismNTTWithIndex on the four polynomials): the thread of OUTPUT coefficient j evaluates the whole digit sum at source position
// index[j]. In the bit-reversed NTT layout an automorphism maps every aligned block of 2^k coefficients onto an aligned block (multiplication by
// an odd Galois element preserves the low bits that select the block), so a warp's 32 gathered 8-byte reads cover exactly one 256-byte block:
// the gather costs no extra sectors, and the separate MAC passes (accumulators re-read and re-written per digit) and permutation passes go away.
// index == nullptr: no permutation (the plain hoisted product). Acc: accumulate into the outputs, out = CRed(out + v) on every row (the
// ringqp.Ring.Add that follows AutomorphismHoistedLazy in PartialTracesSum, core/rlwe/inner_sum.go:243-247).
struct HoistParams {
    const LimbConst* limbs;
    const u64* decomp; size_t d_ds, d_bs; int d_pshift;   // [digit][batch][nqd + np][N]; P rows start d_pshift rows after row nq
    const u64* evk; size_t e_ds, e_cs; int nQk;          // digit stride, component stride; the key's P rows start at row nQk
    const u64* ct0P; size_t c_bs;                        // P * ct0 on the Q rows (nullptr: none)
    u64* out0; u64* out1; size_t o_bs;                   // QP-stacked [batch][nq + np][N]
    const u64* index;
    int nq, np, nQfull, nd, n, batch;
};
constexpr int kHoistB = 4;   // batch elements per thread: the key words are loaded once for all of them
template <bool Acc>
__global__ void __launch_bounds__(256) lt_hoisted_auto_kernel(HoistParams p) {
    const int r = blockIdx.y;
    const bool isP = r >= p.nq;
    const int jr = isP ? r - p.nq : r;
    const LimbConst L = p.limbs[isP ? p.nQfull + jr : jr];
    const u64 q = L.q, qinv = L.qinv, twoq = q << 1;
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const size_t src = p.index ? (size_t)__ldg(p.index + j) : (size_t)j;
    const size_t drow = (size_t)(isP ? r + p.d_pshift : r) * p.n + src;
    const size_t erow = (size_t)(isP ? p.nQk + jr : jr) * p.n + src;
    for (int b0 = blockIdx.z * kHoistB; b0 < p.batch; b0 += gridDim.z * kHoistB) {
        u64 a0[kHoistB], a1[kHoistB];
#pragma unroll
        for (int t = 0; t < kHoistB; t++) { a0[t] = 0; a1[t] = 0; }
        // DRAM traffic = decomposition once + key once per group + outputs (the gather costs no extra sectors). Kept rolled: unrolling it
        // by 3 needs 78 registers, which the launch bounds squeeze to 64.
        for (int d = 0; d < p.nd; d++) {
            const u64 e0 = __ldg(p.evk + (size_t)d * p.e_ds + erow), e1 = __ldg(p.evk + (size_t)d * p.e_ds + p.e_cs + erow);
            const u64* x = p.decomp + (size_t)d * p.d_ds + drow;
#pragma unroll
            for (int t = 0; t < kHoistB; t++) {
                if (b0 + t < p.batch) {
                    const u64 xv = x[(size_t)(b0 + t) * p.d_bs];
                    u64 v0 = a0[t] + mred_lazy(e0, xv, q, qinv), v1 = a1[t] + mred_lazy(e1, xv, q, qinv);
                    a0[t] = v0 >= twoq ? v0 - twoq : v0;
                    a1[t] = v1 >= twoq ? v1 - twoq : v1;
                }
            }
        }
#pragma unroll
        for (int t = 0; t < kHoistB; t++) {
            if (b0 + t < p.batch) {
                u64 v0 = cred(a0[t], q);
                if (p.ct0P && !isP) v0 = cred(v0 + p.ct0P[(size_t)(b0 + t) * p.c_bs + (size_t)r * p.n + src], q);
                const size_t o = (size_t)(b0 + t) * p.o_bs + (size_t)r * p.n + j;
                u64 v1 = cred(a1[t], q);
                if (Acc) { v0 = cred(p.out0[o] + v0, q); v1 = cred(p.out1[o] + v1, q); }
                p.out0[o] = v0;
                p.out1[o] = v1;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host helpers
// ---------------------------------------------------------------------------------------------------------------------
// Evaluator.AutomorphismHoistedLazy (core/rlwe/evaluator_automorphism.go:107-165), NTT-domain branch: out = pi_galEl(
// <decomp, gk> + (P * ct0, 0)) mod QP. ct0P = P * ct0 (rows [0, levelQ], canonical).
int check_gk(const Ctx* c, int levelQ, const GadgetCt& gk) {
    if (!gk.data || gk.levelQ < levelQ || gk.levelQ >= c->nQ || gk.levelP < 0 || gk.levelP >= c->nP) { set_error("Galois key levels out of range"); return -1; }
    if (gk.pw2 != 0) { set_error("method is unsupported for BaseTwoDecomposition != 0"); return -1; }
    if (gk.ndigits < base_rns_decomposition_vector_size(levelQ, gk.levelP)) { set_error("Galois key has too few digits"); return -1; }
    return 0;
}

int automorphism_hoisted_lazy(const Ctx* c, int levelQ, CSpan ct0P, const u64* decomp, int decomp_levelQ, u64 galEl, const GadgetCt& gk,
                              const AccSpans& out, int batch, cudaStream_t st, bool accumulate) {
    const int levelP = gk.levelP;
    if (levelP < 0) { set_error("AutomorphismHoistedLazy requires a P ring"); return -1; }
    if (check_gk(c, levelQ, gk)) return -1;
    if (decomp_levelQ < 0) decomp_levelQ = levelQ;
    const size_t N = c->N, nq = levelQ + 1, np = levelP + 1, nqd = decomp_levelQ + 1;
    const bool stacked = out.q[0].row_stride == N && out.p[0].p == out.q[0].p + nq * N && out.p[1].p == out.q[1].p + nq * N &&
                         out.q[0].batch_stride == out.q[1].batch_stride && out.p[0].batch_stride == out.q[0].batch_stride &&
                         out.p[1].batch_stride == out.q[0].batch_stride && out.p[0].row_stride == N && ct0P.row_stride == N;
    if (stacked) {
        Scratch ib;
        if (ib.alloc(N, st)) return -1;
        if (automorphism_ntt_index(c, galEl, ib.p, st)) return -1;
        HoistParams p;
        p.limbs = c->d_limbs; p.decomp = decomp; p.d_ds = (size_t)batch * (nqd + np) * N; p.d_bs = (nqd + np) * N; p.d_pshift = (int)(nqd - nq);
        const size_t key_rows = (size_t)(gk.levelQ + 1) + (size_t)(gk.levelP + 1);
        p.evk = gk.data; p.e_cs = key_rows * N; p.e_ds = (size_t)gk.npw2max * 2 * key_rows * N; p.nQk = gk.levelQ + 1;
        p.ct0P = ct0P.p; p.c_bs = ct0P.batch_stride;
        p.out0 = out.q[0].p; p.out1 = out.q[1].p; p.o_bs = out.q[0].batch_stride;
        p.index = ib.p; p.nq = (int)nq; p.np = (int)np; p.nQfull = c->nQ; p.nd = base_rns_decomposition_vector_size(levelQ, levelP); p.n = c->N; p.batch = batch;
        // decomposition once, key once per group of kHoistB ciphertexts, P * ct0 on the Q rows, two outputs (read back too when accumulating)
        ProfScope ps(LGPU_KCLASS_MAC, st, 8.0 * N * ((double)(nq + np) * (p.nd * (batch + 2.0 * ((batch + kHoistB - 1) / kHoistB)) + (accumulate ? 4.0 : 2.0) * batch) +
                                                     (double)nq * batch), 1);
        const int zb = std::max(1, std::min(16, (batch + kHoistB - 1) / kHoistB));
        const dim3 grid((c->N + 255) / 256, (unsigned)(nq + np), zb);
        if (accumulate) lt_hoisted_auto_kernel<true><<<grid, 256, 0, st>>>(p);
        else lt_hoisted_auto_kernel<false><<<grid, 256, 0, st>>>(p);
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }
    if (accumulate) { set_error("AutomorphismHoistedLazy: accumulation needs QP-stacked outputs"); return -1; }
    Scratch buf;
    if (buf.alloc((size_t)2 * batch * (nq + np) * N + N, st)) return -1;
    AccSpans acc = stacked_acc(buf.p, nq, np, N, batch);
    u64* index = buf.p + (size_t)2 * batch * (nq + np) * N;
    if (gadget_product_hoisted_lazy(c, levelQ, decomp, gk, acc, batch, st, decomp_levelQ)) return -1;
    if (launch_vecop(c, rows_range(0, 0, (int)nq), LGPU_OP_ADD, CSpan{acc.q[0].p, N, (nq + np) * N}, ct0P, acc.q[0], batch, nullptr, nullptr, 0, 0,
                     c->N, st)) return -1;
    if (automorphism_ntt_index(c, galEl, index, st)) return -1;
    for (int k = 0; k < 2; k++) {
        if (automorphism_ntt_with_index(c, (int)nq, CSpan{acc.q[k].p, N, (nq + np) * N}, index, out.q[k], false, batch, st)) return -1;
        if (automorphism_ntt_with_index(c, (int)np, CSpan{acc.p[k].p, N, (nq + np) * N}, index, out.p[k], false, batch, st)) return -1;
    }
    return 0;
}

void bsgs_index(const LinTransView& m, std::map<int, std::vector<int>>& index, std::vector<int>& rotN1, std::vector<int>& rotN2) {
    const int slots = 1 << m.log_slots;
    std::map<int, bool> n1, n2;
    for (int d = 0; d < m.n_diags; d++) {
        const int rot = m.diag_index[d] & (slots - 1);
        const int idxN1 = ((rot / m.n1) * m.n1) & (slots - 1), idxN2 = rot & (m.n1 - 1);
        index[idxN1].push_back(idxN2);
        n1[idxN1] = true; n2[idxN2] = true;
    }
    for (auto& kv : index) std::sort(kv.second.begin(), kv.second.end());
    for (auto& kv : n1) rotN1.push_back(kv.first);
    for (auto& kv : n2) rotN2.push_back(kv.first);
}

namespace {

typedef std::map<int, std::unique_ptr<Scratch>> PreRot;   // baby step -> [comp][batch][nqd + np][N]

struct LtState {
    const Ctx* c; cudaStream_t st; int batch;
    int level_in, levelQd, levelP;
    size_t N, nqd, np;
    const u64* ctc;      // private copy of the input: [comp][batch][nqd][N]
    const u64* ctP;      // P * ct, same layout
    const u64* decomp;   // DecomposeNTT(ct[1]) at (levelQd, levelP)
    const GaloisKeySet* gks;
};

// the key-level check of MultiplyByDiagMatrix[BSGS] (lintrans_evaluator.go:218-220, :410-412), with the reference's message
static int check_key_level_p(int levelP, u64 galEl, const GadgetCt& gk) {
    if (gk.levelP == levelP) return 0;
    set_error("LinearTransformation.LevelP = " + std::to_string(levelP) + " != GaloiKey[" + std::to_string(galEl) + "].LevelP() = " +
              std::to_string(gk.levelP) + ": ensure that the levelP of the linear transformation is the same as the levelP of the GaloisKeys");
    return -1;
}

static const u64* diag_of(const LinTransView& m, int key) {
    for (int d = 0; d < m.n_diags; d++) if (m.diag_index[d] == key) return m.diag[d];
    return nullptr;
}

static int max_lazy_terms(const Ctx* c, int levelQ, int levelP) {   // min(QiOverflowMargin, PiOverflowMargin) >> 1 (:298-299)
    u64 mx = 0;
    for (int i = 0; i <= levelQ; i++) mx = std::max(mx, c->Q[i]);
    for (int j = 0; j <= levelP; j++) mx = std::max(mx, c->P[j]);
    const int m = (int)std::min<u64>(~0ull / mx, 1u << 20) >> 1;
    return m < 1 ? 1 : m;
}

// PreRotatedCiphertextForDiagonalMatrixMultiplication (:82-114)
static int prerotate(const LtState& s, const std::vector<int>& rots, PreRot& pre) {
    for (auto it = pre.begin(); it != pre.end();) {
        if (std::find(rots.begin(), rots.end(), it->first) == rots.end()) it = pre.erase(it);
        else ++it;
    }
    const size_t per = (size_t)2 * s.batch * (s.nqd + s.np) * s.N;
    for (int i : rots) {
        if (i == 0 || pre.count(i)) continue;
        const u64 galEl = galois_element(s.c, i);
        const GadgetCt* gk = s.gks->find(galEl);
        if (!gk) return -1;
        if (check_key_level_p(s.levelP, galEl, *gk)) return -1;
        std::unique_ptr<Scratch> b(new Scratch);
        if (b->alloc(per, s.st)) return -1;
        AccSpans out = stacked_acc(b->p, s.nqd, s.np, s.N, s.batch);
        if (automorphism_hoisted_lazy(s.c, s.levelQd, CSpan{s.ctP, s.N, s.nqd * s.N}, s.decomp, s.levelQd, galEl, *gk, out, s.batch, s.st)) return -1;
        pre[i] = std::move(b);
    }
    return 0;
}

// final ModDown of a QP-stacked accumulator pair into rows [0, levelQ] of the output ciphertexts
static int moddown_out(const LtState& s, int levelQ, u64* cbuf, u64* out, int out_level) {
    const size_t nq = levelQ + 1, N = s.N;
    AccSpans acc = stacked_acc(cbuf, nq, s.np, N, s.batch);
    const size_t cs = (size_t)(out_level + 1) * N;
    return evaluator_moddown_ntt(s.c, levelQ, s.levelP, acc, Span{out, N, 2 * cs}, Span{out + cs, N, 2 * cs}, s.batch, s.st);
}

// MultiplyByDiagMatrix (:141-274)
static int multiply_naive(const LtState& s, const LinTransView& m, int levelQ, u64* out, int out_level) {
    const Ctx* c = s.c;
    const size_t N = s.N, nq = levelQ + 1, np = s.np;
    const int slots = 1 << m.log_slots;
    std::vector<int> keys(m.diag_index, m.diag_index + m.n_diags);
    std::sort(keys.begin(), keys.end());
    bool state = false;
    if (!keys.empty() && keys[0] == 0) { state = true; keys.erase(keys.begin()); }
    const size_t per = (size_t)2 * s.batch * (nq + np) * N;
    Scratch buf;
    if (buf.alloc(2 * per, s.st)) return -1;
    u64* cb = buf.p; u64* ab = buf.p + per;
    AccSpans acc = stacked_acc(ab, nq, np, N, s.batch);
    const size_t cs = (size_t)(out_level + 1) * N;
    for (size_t i = 0; i < keys.size(); i++) {
        const int k = keys[i] & (slots - 1);
        const u64 galEl = galois_element(c, k);
        const GadgetCt* gk = s.gks->find(galEl);
        if (!gk) return -1;
        if (check_key_level_p(s.levelP, galEl, *gk)) return -1;
        // rotated hoisted product in one pass (the permutation is folded into it), then the diagonal multiply-accumulate without gather
        if (automorphism_hoisted_lazy(c, levelQ, CSpan{s.ctP, N, s.nqd * N}, s.decomp, s.levelQd, galEl, *gk, acc, s.batch, s.st)) return -1;
        const u64* pt = diag_of(m, keys[i]);
        LtPermMacParams p;
        p.limbs = c->d_limbs; p.ptQ = pt; p.ptP = pt + (size_t)(m.level_q + 1) * N;
        p.src0 = ab; p.src1 = ab + per / 2; p.src_bs = (nq + np) * N;
        p.out0 = cb; p.out1 = cb + per / 2; p.out_bs = (nq + np) * N;
        p.index = nullptr; p.first = (i == 0); p.nq = (int)nq; p.np = (int)np; p.nQfull = c->nQ; p.n = c->N;
        ProfScope ps(LGPU_KCLASS_MAC, s.st, 8.0 * N * (nq + np) * (1.0 + s.batch * (p.first ? 4.0 : 6.0)), 1);
        dim3 grid((c->N + 255) / 256, (unsigned)(nq + np), s.batch);
        lt_perm_mac_kernel<<<grid, 256, 0, s.st>>>(p);
        LGPU_CUDA_OK(cudaGetLastError());
    }
    if (!keys.empty()) {
        if (moddown_out(s, levelQ, cb, out, out_level)) return -1;
    } else {
        // only the 0-th diagonal: the reference would ModDown whatever its pooled buffers hold; defined here as zero
        for (int k = 0; k < 2; k++)
            LGPU_CUDA_OK(cudaMemset2DAsync(out + k * cs, 2 * cs * 8, 0, nq * N * 8, s.batch, s.st));
    }
    if (state) {
        const u64* pt = diag_of(m, 0);
        for (int k = 0; k < 2; k++)
            if (launch_vecop(c, rows_range(0, 0, (int)nq), LGPU_OP_MULCOEFFSMONTGOMERYTHENADD, CSpan{pt, N, 0},
                             CSpan{s.ctc + (size_t)k * s.batch * s.nqd * N, N, s.nqd * N}, Span{out + k * cs, N, 2 * cs}, s.batch, nullptr, nullptr, 0, 0,
                             c->N, s.st)) return -1;
    }
    return 0;
}

// MultiplyByDiagMatrixBSGS (:280-470)
static int multiply_bsgs(const LtState& s, const LinTransView& m, const PreRot& pre, int levelQ, u64* out, int out_level) {
    const Ctx* c = s.c;
    const size_t N = s.N, nq = levelQ + 1, np = s.np, nqd = s.nqd;
    std::map<int, std::vector<int>> index;
    std::vector<int> rotN1, rotN2;
    bsgs_index(m, index, rotN1, rotN2);
    const size_t per = (size_t)2 * s.batch * (nq + np) * N;
    Scratch buf;
    if (buf.alloc(3 * per + (size_t)s.batch * nq * N + N, s.st)) return -1;
    u64* cb = buf.p; u64* tb = cb + per; u64* gb = tb + per; u64* t1d = gb + per; u64* d_index = t1d + (size_t)s.batch * nq * N;
    const RowMap rqp = rows_qp(c, (int)nq, (int)np);
    const size_t sbs = (nq + np) * N;
    const int margin = max_lazy_terms(c, levelQ, s.levelP);
    int cnt0 = 0, lazy = 0;
    for (auto& kv : index) {
        const int j = kv.first;
        // inner sum over the baby steps of this giant step
        std::vector<LtTerm> terms;
        for (int i : kv.second) {
            const u64* pt = diag_of(m, j + i);
            if (!pt) { set_error("LinearTransformation: diagonal " + std::to_string(j + i) + " is missing"); return -1; }
            LtTerm T;
            T.ptQ = pt; T.ptP = pt + (size_t)(m.level_q + 1) * N;
            if (i == 0) {
                T.s0Q = s.ctP; T.s1Q = s.ctP + (size_t)s.batch * nqd * N; T.s0P = T.s1P = nullptr; T.bs = nqd * N;
            } else {
                auto it = pre.find(i);
                if (it == pre.end()) { set_error("pre-rotated ciphertext " + std::to_string(i) + " is missing"); return -1; }
                const u64* b0 = it->second->p; const u64* b1 = b0 + (size_t)s.batch * (nqd + np) * N;
                T.s0Q = b0; T.s0P = b0 + nqd * N; T.s1Q = b1; T.s1P = b1 + nqd * N; T.bs = (nqd + np) * N;
            }
            terms.push_back(T);
        }
        for (size_t off = 0; off < terms.size(); off += kLtMaxTerms) {
            LtInnerParams p;
            p.limbs = c->d_limbs;
            p.nterms = (int)std::min<size_t>(kLtMaxTerms, terms.size() - off);
            for (int t = 0; t < p.nterms; t++) p.t[t] = terms[off + t];
            p.out0 = tb; p.out1 = tb + per / 2; p.out_bs = sbs;
            p.first = (off == 0); p.nq = (int)nq; p.np = (int)np; p.nQfull = c->nQ; p.n = c->N; p.batch = s.batch;
            ProfScope ps(LGPU_KCLASS_MAC, s.st, 8.0 * N * (nq + np) * (p.nterms * (1.0 + 2.0 * s.batch) + 2.0 * s.batch), 1);
            dim3 grid((c->N / 2 + 255) / 256, (unsigned)(nq + np), std::min(s.batch, 8));
            lt_inner_kernel<<<grid, 256, 0, s.st>>>(p);
            LGPU_CUDA_OK(cudaGetLastError());
        }
        if (j != 0) {
            // hoisted ModDown of the c1 part, key-switch to the giant-step rotation, rotate, accumulate (:409-436)
            u64* t1 = tb + per / 2;
            if (moddown_ntt(c, levelQ, s.levelP, CBlock{t1, 0, sbs}, CBlock{nullptr, 0, 0}, Block{t1d, 0, nq * N}, 1, s.batch, s.st)) return -1;
            const u64 galEl = galois_element(c, j);
            const GadgetCt* gk = s.gks->find(galEl);
            if (!gk) return -1;
            if (check_key_level_p(s.levelP, galEl, *gk)) return -1;
            AccSpans g = stacked_acc(gb, nq, np, N, s.batch);
            if (gadget_product_lazy(c, levelQ, CSpan{t1d, N, nq * N}, *gk, g, s.batch, s.st)) return -1;
            if (launch_vecop(c, rqp, LGPU_OP_ADD, CSpan{gb, N, sbs}, CSpan{tb, N, sbs}, Span{gb, N, sbs}, s.batch, nullptr, nullptr, 0, 0, c->N, s.st)) return -1;
            if (automorphism_ntt_index(c, galEl, d_index, s.st)) return -1;
            for (int k = 0; k < 2; k++)
                if (automorphism_ntt_with_index(c, (int)(nq + np), CSpan{gb + k * (per / 2), N, sbs}, d_index, Span{cb + k * (per / 2), N, sbs}, cnt0 != 0,
                                                s.batch, s.st)) return -1;
        } else if (cnt0 == 0) {
            LGPU_CUDA_OK(cudaMemcpyAsync(cb, tb, per * sizeof(u64), cudaMemcpyDeviceToDevice, s.st));
        } else {
            for (int k = 0; k < 2; k++)
                if (launch_vecop(c, rqp, LGPU_OP_ADDLAZY, CSpan{cb + k * (per / 2), N, sbs}, CSpan{tb + k * (per / 2), N, sbs}, Span{cb + k * (per / 2), N, sbs},
                                 s.batch, nullptr, nullptr, 0, 0, c->N, s.st)) return -1;
        }
        lazy = cnt0 == 0 ? 0 : lazy + 1;
        if (lazy >= margin - 1 && lazy > 0) {
            for (int k = 0; k < 2; k++)
                if (launch_vecop(c, rqp, LGPU_OP_REDUCE, CSpan{cb + k * (per / 2), N, sbs}, CSpan{nullptr, 0, 0}, Span{cb + k * (per / 2), N, sbs}, s.batch,
                                 nullptr, nullptr, 0, 0, c->N, s.st)) return -1;
            lazy = 0;
        }
        cnt0++;
    }
    if (lazy > 0)
        for (int k = 0; k < 2; k++)
            if (launch_vecop(c, rqp, LGPU_OP_REDUCE, CSpan{cb + k * (per / 2), N, sbs}, CSpan{nullptr, 0, 0}, Span{cb + k * (per / 2), N, sbs}, s.batch,
                             nullptr, nullptr, 0, 0, c->N, s.st)) return -1;
    if (cnt0 == 0) { set_error("LinearTransformation has no diagonal"); return -1; }
    return moddown_out(s, levelQ, cb, out, out_level);
}

}  // namespace

// lintrans.Evaluator.EvaluateMany (:28-79). ct_in: [batch][2][level_in + 1][N] (NTT domain); outs[i]: [batch][2][out_levels[i] + 1][N],
// out_levels[i] is updated to the level of the result (the reference resizes opOut to min(opOut, ctIn, matrix levels)); rows above it are
// left untouched. In-place (outs[i] == ct_in) is allowed, like EvaluateSequential uses it.
int lintrans_evaluate_many(const Ctx* c, int level_in, const u64* ct_in, const LinTransView* mats, int n_mats, const GaloisKeySet& gks,
                           u64* const* outs, int* out_levels, int batch, cudaStream_t st) {
    if (n_mats < 1) { set_error("no linear transformation"); return -1; }
    if (level_in < 0 || level_in >= c->nQ) { set_error("ciphertext level out of range"); return -1; }
    int levelQd = 0;
    const int levelP = mats[0].level_p;
    for (int i = 0; i < n_mats; i++) {
        levelQd = std::max(levelQd, mats[i].level_q);
        if (mats[i].level_p != levelP) { set_error("all linearTransformations must have the same levelP"); return -1; }
        if (mats[i].level_q < 0 || mats[i].level_q >= c->nQ) { set_error("LinearTransformation.LevelQ out of range"); return -1; }
        if (mats[i].n_diags < 1 || !mats[i].diag_index || !mats[i].diag) { set_error("LinearTransformation has no diagonal"); return -1; }
        if (mats[i].log_slots < 0 || mats[i].log_slots >= c->logN + (c->ring_type ? 1 : 0)) { set_error("LinearTransformation.LogSlots out of range"); return -1; }
        if (!outs[i]) { set_error("output slice contains unallocated ciphertext"); return -1; }
    }
    if (levelP < 0 || levelP >= c->nP) { set_error("LinearTransformation.LevelP out of range (hoisting needs the P ring)"); return -1; }
    levelQd = std::min(levelQd, level_in);
    LtState s;
    s.c = c; s.st = st; s.batch = batch; s.level_in = level_in; s.levelQd = levelQd; s.levelP = levelP;
    s.N = c->N; s.nqd = levelQd + 1; s.np = levelP + 1; s.gks = &gks;
    const size_t N = s.N, nqd = s.nqd, np = s.np, cin = (size_t)(level_in + 1) * N;
    const int nd = base_rns_decomposition_vector_size(levelQd, levelP);
    Scratch buf;
    const size_t ctw = (size_t)2 * batch * nqd * N;
    if (buf.alloc(2 * ctw + (size_t)nd * batch * (nqd + np) * N, st)) return -1;
    u64* ctc = buf.p; u64* ctP = ctc + ctw; u64* decomp = ctP + ctw;
    for (int k = 0; k < 2; k++)
        LGPU_CUDA_OK(cudaMemcpy2DAsync(ctc + (size_t)k * batch * nqd * N, nqd * N * 8, ct_in + k * cin, 2 * cin * 8, nqd * N * 8, batch,
                                       cudaMemcpyDeviceToDevice, st));
    const std::vector<u64> pq = p_mod_q_mont(c, levelQd, levelP);
    if (launch_vecop(c, rows_range(0, 0, (int)nqd), LGPU_OP_MULSCALARMONTGOMERY, CSpan{ctc, N, nqd * N}, CSpan{nullptr, 0, 0}, Span{ctP, N, nqd * N}, 2 * batch,
                     pq.data(), nullptr, 0, 0, c->N, st)) return -1;
    if (decompose_ntt(c, levelQd, levelP, levelP + 1, CSpan{ctc + (size_t)batch * nqd * N, N, nqd * N}, true, decomp, batch, st)) return -1;
    s.ctc = ctc; s.ctP = ctP; s.decomp = decomp;
    PreRot pre;
    for (int i = 0; i < n_mats; i++) {
        const LinTransView& m = mats[i];
        const int levelQ = std::min(std::min(out_levels[i], level_in), m.level_q);
        if (levelQ < 0) { set_error("output level out of range"); return -1; }
        if (m.n1 == 0) {
            if (multiply_naive(s, m, levelQ, outs[i], out_levels[i])) return -1;
        } else {
            if (m.n1 < 0 || (m.n1 & (m.n1 - 1))) { set_error("LinearTransformation.N1 must be a power of two"); return -1; }
            std::map<int, std::vector<int>> index;
            std::vector<int> rotN1, rotN2;
            bsgs_index(m, index, rotN1, rotN2);
            if (prerotate(s, rotN2, pre)) return -1;
            if (multiply_bsgs(s, m, pre, levelQ, outs[i], out_levels[i])) return -1;
        }
        // NB the result occupies rows [0, levelQ] of a buffer laid out for out_levels[i] (a Go Resize re-slices, it does not move rows)
        out_levels[i] = levelQ;
    }
    return 0;
}

}  // namespace lgpu

// polyeval.cu -- ckks and bgv polynomial.Evaluator.Evaluate (circuits/ckks/polynomial/polynomial_evaluator.go:42-57,
// circuits/bgv/polynomial/polynomial_evaluator.go:38-51) for a BATCH of ciphertexts, running a program planned on the host
// (lattigo_b200/polyeval.py, lattigo_b200/bgv_polyeval.py): MULRELIN / TENSOR / RELIN / RESCALE / LINCOMB ops over
// single-assignment slots (include/lattigo_b200.h). The kernels:
//   poly_lincomb_kernel     every baby step of a call (or one Chebyshev power combine) in one pass that reads each power once;
//   poly_tensor_kernel      EvaluateMonomial's Mul(b, X^k) + Add(.., a) with the scale ratios, in one pass (also the tensor of
//                           MULRELIN); TMUL pre-multiplies b by tMontgomery (BGV tensorStandard) instead of MForm (CKKS);
//   poly_tensor_add_kernel  the same Add on a product that is already in memory (BFV: the scale-invariant tensor of bgv.cu).
// Only MULRELIN and TENSOR depend on the scheme (Runner::mulrelin / Runner::tensor_op). Relinearization, the key switch of
// MulRelinNew and Rescale use the existing launchers. Every op's output is the canonical residue of a linear combination of canonical
// inputs, so the results equal the reference's op-by-op sequence bit for bit (DESIGN 3.4; tests/test_gpu_polyeval.py vs
// oracle/polyeval.py, tests/test_gpu_bgv_polyeval.py vs tests/bgv_polyeval_oracle.py).
#include <algorithm>
#include <cstring>
#include <vector>
#include "bgv.h"
#include "composite.h"
#include "modarith.cuh"

namespace lgpu {

constexpr int kPolyMaxTerms = LGPU_POLY_MAX_TERMS;
constexpr int kPolyMaxOut = LGPU_POLY_MAX_OUTPUTS;

struct LincombParams {
    const LimbConst* limbs;
    const u64* w;                        // [limb][n_out][n_terms + 1][2]: MForm(W) for the terms, the plain constant last
    int n_out, n_terms, n;
    const u64* in[kPolyMaxTerms];        // degree-1 terms: component c of batch entry b at in[k] + b * in_bs[k] + c * in_cs[k]
    unsigned in_cs[kPolyMaxTerms], in_bs[kPolyMaxTerms];
    int in_level[kPolyMaxTerms];         // rows above a term's level read as 0 (its weights there are 0)
    u64* out[kPolyMaxOut];
    unsigned out_cs[kPolyMaxOut], out_bs[kPolyMaxOut];
    int out_level[kPolyMaxOut];
};

// out_i[c][j] = sum_k W[i,k,half(j)] X_k[c][j] (+ W[i,K,half(j)] on c = 0), rows r <= out_level[i]. One thread per (row, coefficient, batch entry)
// holds its K terms of both components in registers and writes every output once. Each product is reduced to [0, q) (MRed by the
// Montgomery-form weight) before it is added, and every add is followed by a conditional subtraction, so the running sum is < 2q < 2^63
// for any K and any q < 2^62: no wide accumulator and no bound on K is needed (a lazy 128-bit sum of K products < q^2 would need
// K q^2 < q 2^64 for one final Montgomery reduction, which fails for K > 8 at q ~ 2^61).
__global__ void __launch_bounds__(256) poly_lincomb_kernel(LincombParams p) {
    extern __shared__ u64 ws[];
    const int r = blockIdx.y;
    const int wn = p.n_out * (p.n_terms + 1) * 2;
    for (int t = threadIdx.x; t < wn; t += blockDim.x) ws[t] = p.w[(size_t)r * wn + t];
    __syncthreads();
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const LimbConst L = p.limbs[r];
    const u64 q = L.q, qinv = L.qinv;
    const int h = j >= (p.n >> 1) ? 1 : 0;
    const size_t b = blockIdx.z, ro = (size_t)r * p.n + j;
    u64 x0[kPolyMaxTerms], x1[kPolyMaxTerms];
#pragma unroll
    for (int k = 0; k < kPolyMaxTerms; k++) {
        if (k < p.n_terms) {
            x0[k] = x1[k] = 0;
            if (r <= p.in_level[k]) {
                const u64* s = p.in[k] + b * p.in_bs[k] + ro;
                x0[k] = s[0];
                x1[k] = s[p.in_cs[k]];
            }
        }
    }
    for (int i = 0; i < p.n_out; i++) {
        if (r > p.out_level[i]) continue;
        const u64* w = ws + i * (p.n_terms + 1) * 2;
        u64 a0 = w[p.n_terms * 2 + h], a1 = 0;
#pragma unroll
        for (int k = 0; k < kPolyMaxTerms; k++) {
            if (k < p.n_terms) {
                const u64 wk = w[k * 2 + h];
                a0 = cred(a0 + mred(x0[k], wk, q, qinv), q);
                a1 = cred(a1 + mred(x1[k], wk, q, qinv), q);
            }
        }
        u64* o = p.out[i] + b * p.out_bs[i] + ro;
        o[0] = a0;
        o[p.out_cs[i]] = a1;
    }
}

struct PtLincombParams {
    const LimbConst* limbs;
    const u64* w;                        // [limb][n_out][n_terms + 1]: Montgomery factors of the scalars (see validate)
    const u64* idx;                      // [n_out][n_terms + 1]: plaintext index, or ~0 for a missing weight
    const u64* pt;                       // plaintext j: pt + j * pt_stride, row r at + r * n
    size_t pt_stride;
    int n_out, n_terms, n, nb;
    const u64* in[kPolyMaxTerms];
    unsigned in_cs[kPolyMaxTerms], in_bs[kPolyMaxTerms];
    int in_level[kPolyMaxTerms];
    u64* out[kPolyMaxOut];
    unsigned out_cs[kPolyMaxOut], out_bs[kPolyMaxOut];
    int out_level[kPolyMaxOut];
};

// out_i[c][j] = sum_k s_ik PT_ik[j] X_k[c][j] (+ s_iK PT_iK[j] on c = 0), rows r <= out_level[i]. A CTA covers 256 / BT coefficients of
// one row for BT consecutive batch entries (one warp per entry and 32 coefficients); each thread holds the K terms of its entry in
// registers, as poly_lincomb_kernel does. Per output, the CTA stages m_ik = MRed(PT_ik, S_ik) for its coefficients in shared memory once
// (S_ik = s_ik 2^128 mod q for a term, so MRed(X, m) = s PT X; S_iK = s_iK 2^64 for the constant), so each plaintext word is read once
// per BT ciphertexts and each power once per batch entry. Every product is reduced to [0, q) and every add is followed by a conditional
// subtraction, so outputs are canonical for any K.
template <int BT>
__global__ void __launch_bounds__(256) poly_pt_lincomb_kernel(PtLincombParams p) {
    constexpr int CJ = 256 / BT;
    extern __shared__ u64 sm[];
    const int r = blockIdx.y;
    const int K1 = p.n_terms + 1, wn = p.n_out * K1;
    u64* ws = sm;                        // [n_out][K1] factors of row r
    u64* mp = sm + wn;                   // [K1][CJ] the staged m_ik of the current output
    for (int t = threadIdx.x; t < wn; t += blockDim.x) ws[t] = p.w[(size_t)r * wn + t];
    const LimbConst L = p.limbs[r];
    const u64 q = L.q, qinv = L.qinv;
    const int jl = threadIdx.x % CJ, j0 = blockIdx.x * CJ, j = j0 + jl;
    const int b = blockIdx.z * BT + threadIdx.x / CJ;
    const bool act = b < p.nb && j < p.n;
    const size_t ro = (size_t)r * p.n + j;
    u64 x0[kPolyMaxTerms], x1[kPolyMaxTerms];
#pragma unroll
    for (int k = 0; k < kPolyMaxTerms; k++) {
        if (k < p.n_terms) {
            x0[k] = x1[k] = 0;
            if (act && r <= p.in_level[k]) {
                const u64* s = p.in[k] + (size_t)b * p.in_bs[k] + ro;
                x0[k] = s[0];
                x1[k] = s[p.in_cs[k]];
            }
        }
    }
    for (int i = 0; i < p.n_out; i++) {
        if (r > p.out_level[i]) continue;            // uniform over the CTA
        __syncthreads();                             // ws is loaded; the previous output's mp is consumed
        for (int t = threadIdx.x; t < K1 * CJ; t += blockDim.x) {
            const int k = t / CJ, jj = j0 + t % CJ;
            const u64 id = p.idx[i * K1 + k];
            u64 v = 0;
            if (id != ~0ull && jj < p.n) v = mred(p.pt[id * p.pt_stride + (size_t)r * p.n + jj], ws[i * K1 + k], q, qinv);
            mp[t] = v;
        }
        __syncthreads();
        if (!act) continue;
        u64 a0 = mp[p.n_terms * CJ + jl], a1 = 0;
#pragma unroll
        for (int k = 0; k < kPolyMaxTerms; k++) {
            if (k < p.n_terms) {
                const u64 m = mp[k * CJ + jl];
                a0 = cred(a0 + mred(x0[k], m, q, qinv), q);
                a1 = cred(a1 + mred(x1[k], m, q, qinv), q);
            }
        }
        u64* o = p.out[i] + (size_t)b * p.out_bs[i] + ro;
        o[0] = a0;
        o[p.out_cs[i]] = a1;
    }
}

struct PolyTensorParams {
    const LimbConst* limbs;
    const u64* b; size_t b_cs, b_bs;     // degree 1
    const u64* x; size_t x_cs, x_bs;     // degree 1
    const u64* a; size_t a_cs, a_bs;     // addend, degree a_deg (ADD only)
    int a_deg;
    const u64* wb; const u64* wa;        // MForm(r_b), MForm(r_a) per limb (ADD only)
    u64* d; size_t d_cs, d_bs;           // degree 2
    int n;
    const u64* tmont;                    // TMUL: tMontgomery per limb
};

// d_c = MRed(x_c, MForm(r_b)) (+) MRed(a_c, MForm(r_a)) for c = 0..2, the addend's components up to a_deg
__device__ __forceinline__ void poly_add_epilogue(const PolyTensorParams& p, const u64 (&x)[3], int r, size_t b, size_t ro, u64 q, u64 qinv) {
    const u64 wb = p.wb[r], wa = p.wa[r];
    const u64* A = p.a + b * p.a_bs + ro;
    u64* D = p.d + b * p.d_bs + ro;
#pragma unroll
    for (int c = 0; c < 3; c++) {
        u64 v = mred(x[c], wb, q, qinv);
        if (c <= p.a_deg) v = cred(v + mred(A[c * p.a_cs], wa, q, qinv), q);
        D[c * p.d_cs] = v;
    }
}
// schemes/ckks/evaluator.go:807-820 (c00 = MForm(b0), c01 = MForm(b1); d0 = MRed(c00, x0), d2 = MRed(c01, x1),
// d1 = MRed(c00, x1) (+) MRed(c01, x0)), then, with ADD, d_c = MRed(d_c, MForm(r_b)) (+) MRed(a_c, MForm(r_a)) (the Mul by the
// truncated scale ratio and the Add of EvaluateMonomial, :238-246 and evaluateInPlace :221-408). All canonical.
// TMUL: c00 = MRed(b0, tMontgomery), c01 = MRed(b1, tMontgomery) (schemes/bgv/evaluator.go:634-635), then the same products and Add
// (r_b, r_a: 1 or matchScalesBinary's r0, r1, :210-227).
template <bool ADD, bool TMUL>
__global__ void __launch_bounds__(256) poly_tensor_kernel(PolyTensorParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const int r = blockIdx.y;
    const LimbConst L = p.limbs[r];
    const u64 q = L.q, qinv = L.qinv;
    const size_t b = blockIdx.z, ro = (size_t)r * p.n + j;
    const u64* B = p.b + b * p.b_bs + ro;
    const u64* X = p.x + b * p.x_bs + ro;
    u64 m0, m1;
    if (TMUL) {
        const u64 tm = p.tmont[r];
        m0 = mred(B[0], tm, q, qinv); m1 = mred(B[p.b_cs], tm, q, qinv);
    } else {
        m0 = mform(B[0], q, L.bred_hi, L.bred_lo); m1 = mform(B[p.b_cs], q, L.bred_hi, L.bred_lo);
    }
    const u64 x0 = X[0], x1 = X[p.x_cs];
    u64 d[3];
    d[0] = mred(m0, x0, q, qinv);
    d[2] = mred(m1, x1, q, qinv);
    d[1] = cred(mred(m0, x1, q, qinv) + mred(m1, x0, q, qinv), q);
    if (ADD) {
        poly_add_epilogue(p, d, r, b, ro, q, qinv);
    } else {
        u64* D = p.d + b * p.d_bs + ro;
#pragma unroll
        for (int c = 0; c < 3; c++) D[c * p.d_cs] = d[c];
    }
}

// The Add of EvaluateMonomial on a degree-2 product x already in memory (p.b, components b_cs apart): BFV, whose scale-invariant
// tensor (bfv_tensor) ends with an NTT pass and so cannot carry the epilogue.
__global__ void __launch_bounds__(256) poly_tensor_add_kernel(PolyTensorParams p) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n) return;
    const int r = blockIdx.y;
    const LimbConst L = p.limbs[r];
    const size_t b = blockIdx.z, ro = (size_t)r * p.n + j;
    const u64* X = p.b + b * p.b_bs + ro;
    const u64 x[3] = {X[0], X[p.b_cs], X[2 * p.b_cs]};
    poly_add_epilogue(p, x, r, b, ro, L.q, L.qinv);
}

namespace {

struct Slot {           // one single-assignment ciphertext of the program for the current sub-batch: [batch][deg+1][level+1][N]
    u64* p = nullptr;
    int deg = 0, level = -1;
    bool owned = false;
};

struct Plan {           // what validation derives from the program
    std::vector<int> deg, level, last_use;
    std::vector<std::vector<u64>> w;      // per op: device-ready weights (LINCOMB: [limb][out][term+1][2]; TENSOR: [2][level+1] MForm)
};

// vw: the plaintext table of the vector entry points; null for the scalar ones, where PTLINCOMB stays an unknown op
int validate(const Ctx& c, int level, const lgpu_poly_program* pg, Plan& pl, const lgpu_poly_pt_weights* vw) {
    REQUIRE(pg && pg->n_ops >= 1 && pg->ops, "empty polynomial program");
    REQUIRE(pg->n_slots >= 2 && pg->n_slots <= (1 << 16), "program slot count out of range");
    REQUIRE(pg->levels_per_rescale >= 1, "levels_per_rescale must be >= 1");
    const int ns = pg->n_slots;
    pl.deg.assign(ns, 0); pl.level.assign(ns, -1); pl.last_use.assign(ns, -1); pl.w.assign(pg->n_ops, {});
    pl.deg[0] = 1; pl.level[0] = level;
    auto slot_ok = [&](int s) { return s >= 0 && s < ns; };
    auto readable = [&](int s) { return slot_ok(s) && pl.level[s] >= 0; };
    auto w_ok = [&](const uint64_t* w, size_t n, int rows, int per_row) {      // w[.][row][per_row] < q_row
        for (size_t i = 0; i < n; i++) {
            const int row = (int)((i / per_row) % rows);
            if (w[i] >= c.Q[row]) return false;
        }
        return true;
    };
    // single assignment: slot d is written once, and never slot 0 (the input)
    auto write = [&](int d, int deg, int lv) {
        REQUIRE(slot_ok(d) && pl.level[d] < 0 && d != 0, "program writes a slot twice (or slot 0)");
        pl.deg[d] = deg; pl.level[d] = lv;
        return 0;
    };
    // what LINCOMB and PTLINCOMB (op i, named `name` in the messages) share: output and term counts, the arrays, output levels whose
    // maximum is the op's level, degree-1 terms
    auto lin_shape = [&](const lgpu_poly_op& o, int i, const std::string& name) {
        const bool lin = o.kind == LGPU_POLY_LINCOMB;
        REQUIRE(o.n_out >= 1 && o.n_out <= kPolyMaxOut, name + " output count out of range");
        REQUIRE(o.n_terms >= 0 && o.n_terms <= kPolyMaxTerms, name + " term count out of range (at most LGPU_POLY_MAX_TERMS)");
        REQUIRE(o.outs && o.out_levels && (!lin || o.weights) && (o.n_terms == 0 || o.terms),
                name + (lin ? " needs outs, out_levels, terms and weights" : " needs outs, out_levels and terms"));
        int mx = -1;
        for (int k = 0; k < o.n_out; k++) {
            REQUIRE(o.out_levels[k] >= 0 && o.out_levels[k] <= o.level, name + " output level out of range");
            mx = std::max(mx, o.out_levels[k]);
        }
        REQUIRE(mx == o.level, name + " level must be the maximum of its output levels");
        for (int k = 0; k < o.n_terms; k++) {
            REQUIRE(readable(o.terms[k]), "program reads a slot before it is written");
            REQUIRE(pl.deg[o.terms[k]] == 1, name + " terms must have degree 1");
            pl.last_use[o.terms[k]] = i;
        }
        return 0;
    };
    int n_pt_ops = 0;
    for (int i = 0; i < pg->n_ops; i++) {
        const lgpu_poly_op& o = pg->ops[i];
        REQUIRE(o.level >= 0 && o.level <= level, "program op level out of range");
        switch (o.kind) {
        case LGPU_POLY_MULRELIN:
        case LGPU_POLY_TENSOR: {
            REQUIRE(readable(o.src0) && readable(o.src1), "program reads a slot before it is written");
            REQUIRE(pl.deg[o.src0] == 1 && pl.deg[o.src1] == 1, "MULRELIN / TENSOR operands must have degree 1");
            int lv = std::min(pl.level[o.src0], pl.level[o.src1]);
            if (o.kind == LGPU_POLY_TENSOR && o.addend >= 0) {
                REQUIRE(readable(o.addend), "program reads a slot before it is written");
                lv = std::min(lv, pl.level[o.addend]);
            }
            REQUIRE(o.level == lv, "MULRELIN / TENSOR level must be the minimum level of its operands");
            if (o.kind == LGPU_POLY_TENSOR) {
                REQUIRE(o.weights, "TENSOR needs its weights");
                REQUIRE(w_ok(o.weights, (size_t)2 * (o.level + 1), o.level + 1, 1), "TENSOR weight not below its modulus");
                std::vector<u64>& w = pl.w[i];
                for (int k = 0; k < 2 * (o.level + 1); k++) w.push_back(h_mform(o.weights[k], c.Q[k % (o.level + 1)]));
            }
            if (write(o.dst, o.kind == LGPU_POLY_MULRELIN ? 1 : 2, o.level)) return -1;
            pl.last_use[o.src0] = pl.last_use[o.src1] = i;
            if (o.kind == LGPU_POLY_TENSOR && o.addend >= 0) pl.last_use[o.addend] = i;
            break;
        }
        case LGPU_POLY_RELIN:
        case LGPU_POLY_RESCALE: {
            REQUIRE(readable(o.src0), "program reads a slot before it is written");
            if (o.kind == LGPU_POLY_RELIN) {
                REQUIRE(pl.deg[o.src0] == 2, "RELIN operand must have degree 2");
                REQUIRE(o.level == pl.level[o.src0], "RELIN keeps the level");
            } else {
                REQUIRE(o.level == pl.level[o.src0] - pg->levels_per_rescale, "cannot Rescale: RESCALE level must be its operand's minus levels_per_rescale");
            }
            if (write(o.dst, o.kind == LGPU_POLY_RELIN ? 1 : pl.deg[o.src0], o.level)) return -1;
            pl.last_use[o.src0] = i;
            break;
        }
        case LGPU_POLY_LINCOMB: {
            if (lin_shape(o, i, "LINCOMB")) return -1;
            const int K = o.n_terms + 1, R = o.level + 1;
            REQUIRE(w_ok(o.weights, (size_t)o.n_out * K * R * 2, R, 2), "LINCOMB weight not below its modulus");
            for (int k = 0; k < o.n_out; k++)            // an output may not use a term above the term's level
                for (int t = 0; t < o.n_terms; t++)
                    for (int r = pl.level[o.terms[t]] + 1; r <= o.out_levels[k]; r++)
                        REQUIRE(o.weights[(((size_t)k * K + t) * R + r) * 2] == 0 && o.weights[(((size_t)k * K + t) * R + r) * 2 + 1] == 0,
                                "LINCOMB output uses a term above the term's level");
            for (int k = 0; k < o.n_out; k++)
                if (write(o.outs[k], 1, o.out_levels[k])) return -1;
            // device layout [limb][out][term][half], Montgomery form for the terms, the constant as is
            std::vector<u64>& w = pl.w[i];
            w.resize((size_t)R * o.n_out * K * 2);
            for (int r = 0; r < R; r++)
                for (int k = 0; k < o.n_out; k++)
                    for (int t = 0; t < K; t++)
                        for (int h = 0; h < 2; h++) {
                            const u64 v = o.weights[(((size_t)k * K + t) * R + r) * 2 + h];
                            w[(((size_t)r * o.n_out + k) * K + t) * 2 + h] = t < o.n_terms ? h_mform(v, c.Q[r]) : v;
                        }
            break;
        }
        case LGPU_POLY_PTLINCOMB: {
            REQUIRE(vw, "unknown polynomial program op");          // to the scalar entry points
            REQUIRE(++n_pt_ops == 1, "a vector program has exactly one PTLINCOMB op");
            if (lin_shape(o, i, "PTLINCOMB")) return -1;
            REQUIRE(vw->n_pt >= 1 && vw->n_pt <= (1 << 20), "plaintext count out of range");
            REQUIRE(vw->pt && vw->pt_levels && vw->index && vw->scalars, "null plaintext table");
            REQUIRE_ALIGNED(AL(vw->pt) && vw->pt_stride % 2 == 0);
            int ptmax = 0;
            for (int j = 0; j < vw->n_pt; j++) {
                REQUIRE(vw->pt_levels[j] >= 0 && vw->pt_levels[j] < c.nQ, "plaintext level out of range");
                ptmax = std::max(ptmax, vw->pt_levels[j]);
            }
            REQUIRE(vw->pt_stride >= (size_t)(ptmax + 1) * c.N, "plaintext stride below the rows of its plaintexts");
            const int K = o.n_terms + 1, R = o.level + 1;
            for (int k = 0; k < o.n_out; k++)
                for (int t = 0; t < K; t++) {
                    const int id = vw->index[k * K + t];
                    REQUIRE(id >= -1 && id < vw->n_pt, "plaintext index out of range");
                    if (id < 0) continue;
                    REQUIRE(vw->pt_levels[id] >= o.out_levels[k], "PTLINCOMB output uses a plaintext below its level");
                    REQUIRE(t == o.n_terms || pl.level[o.terms[t]] >= o.out_levels[k], "PTLINCOMB output uses a term below its level");
                }
            REQUIRE(w_ok(vw->scalars, (size_t)o.n_out * K * R, R, 1), "PTLINCOMB scalar not below its modulus");
            for (int k = 0; k < o.n_out; k++)
                if (write(o.outs[k], 1, o.out_levels[k])) return -1;
            // device layout: [limb][out][term] Montgomery factors (s 2^128 for a term, s 2^64 for the constant), then [out][term] indices
            std::vector<u64>& w = pl.w[i];
            w.resize((size_t)R * o.n_out * K + (size_t)o.n_out * K);
            for (int r = 0; r < R; r++)
                for (int k = 0; k < o.n_out; k++)
                    for (int t = 0; t < K; t++) {
                        const u64 v = h_mform(vw->scalars[((size_t)k * K + t) * R + r], c.Q[r]);
                        w[((size_t)r * o.n_out + k) * K + t] = t < o.n_terms ? h_mform(v, c.Q[r]) : v;
                    }
            for (int k = 0; k < o.n_out * K; k++) w[(size_t)R * o.n_out * K + k] = vw->index[k] < 0 ? ~0ull : (u64)vw->index[k];
            break;
        }
        default:
            REQUIRE(false, "unknown polynomial program op");
        }
    }
    REQUIRE(!vw || n_pt_ops == 1, "a vector program has exactly one PTLINCOMB op");
    REQUIRE(slot_ok(pg->out_slot) && pl.level[pg->out_slot] >= 0 && pl.deg[pg->out_slot] == 1, "program output slot must be a written degree-1 slot");
    const lgpu_poly_op& last = pg->ops[pg->n_ops - 1];
    const bool last_writes_out = last.kind == LGPU_POLY_LINCOMB || last.kind == LGPU_POLY_PTLINCOMB ? std::find(last.outs, last.outs + last.n_out, pg->out_slot) != last.outs + last.n_out
                                                                : last.dst == pg->out_slot;
    REQUIRE(last_writes_out, "the program's last op must write its output slot");
    return 0;
}

struct Runner {
    const Ctx* c;
    const lgpu_poly_program* pg;
    const Plan& pl;
    const GadgetCt& rlk;
    cudaStream_t st;
    int nb;
    std::vector<Slot> s;
    const u64* d_w;                       // all op weights, uploaded once
    std::vector<size_t> w_off;
    const BgvState* bgv = nullptr;        // BGV / BFV: the evaluator state; null for CKKS
    bool si = false;                      // BFV: scale-invariant tensoring
    const lgpu_poly_pt_weights* vw = nullptr;   // the vector entry points' plaintexts
    u64* out_chunk = nullptr;             // the sub-batch's output ciphertexts: the program's output slot is written there

    size_t cs(int i) const { return (size_t)(s[i].level + 1) * c->N; }
    size_t bs(int i) const { return (size_t)(s[i].deg + 1) * cs(i); }

    // slot i: out_chunk if it is the program's output, else a new sub-batch block
    int make(int i) {
        s[i].deg = pl.deg[i]; s[i].level = pl.level[i];
        if (i == pg->out_slot) { s[i].p = out_chunk; return 0; }
        LGPU_CUDA_OK(cudaMallocAsync((void**)&s[i].p, (size_t)nb * bs(i) * 8, st));
        s[i].owned = true;
        return 0;
    }
    void release(int i) {
        if (s[i].owned && s[i].p) cudaFreeAsync(s[i].p, st);
        s[i].p = nullptr; s[i].owned = false;
    }
    ~Runner() { for (size_t i = 0; i < s.size(); i++) release((int)i); }

    int tensor(int bsl, int xsl, int asl, const u64* w, int level, u64* d, size_t d_cs, size_t d_bs) {
        PolyTensorParams p;
        p.limbs = c->d_limbs;
        p.b = s[bsl].p; p.b_cs = cs(bsl); p.b_bs = bs(bsl);
        p.x = s[xsl].p; p.x_cs = cs(xsl); p.x_bs = bs(xsl);
        p.a = asl >= 0 ? s[asl].p : nullptr; p.a_cs = asl >= 0 ? cs(asl) : 0; p.a_bs = asl >= 0 ? bs(asl) : 0; p.a_deg = asl >= 0 ? s[asl].deg : -1;
        p.wb = w; p.wa = w ? w + (level + 1) : nullptr;
        p.d = d; p.d_cs = d_cs; p.d_bs = d_bs; p.n = c->N;
        p.tmont = bgv ? bgv->tmont() : nullptr;
        ProfScope ps(LGPU_KCLASS_TENSOR, st, 8.0 * c->N * (level + 1) * nb * (w ? 7 + (p.a_deg + 1) : 7), 1);
        const dim3 grid((c->N + 255) / 256, (unsigned)(level + 1), (unsigned)nb);
        if (bgv) {
            if (w) poly_tensor_kernel<true, true><<<grid, 256, 0, st>>>(p);
            else poly_tensor_kernel<false, true><<<grid, 256, 0, st>>>(p);
        } else {
            if (w) poly_tensor_kernel<true, false><<<grid, 256, 0, st>>>(p);
            else poly_tensor_kernel<false, false><<<grid, 256, 0, st>>>(p);
        }
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }

    // MulRelinNew of two degree-1 slots into the degree-1 slot dst (made by the caller): the scheme's tensor, then mulrelin_tail
    int mulrelin(const lgpu_poly_op& o) {
        const size_t N = c->N, nq = o.level + 1;
        Scratch buf;                                   // d0, d1, d2, t0, t1: [5][nb][nq][N] (mulrelin_tail's layout)
        if (buf.alloc((size_t)nb * 5 * nq * N, st)) return -1;
        if (si) {
            if (bfv_tensor(c, *bgv, o.level, s[o.src0].p, s[o.src1].p, buf.p, nb, st)) return -1;
        } else if (tensor(o.src0, o.src1, -1, nullptr, o.level, buf.p, (size_t)nb * nq * N, nq * N)) {
            return -1;
        }
        return mulrelin_tail(c, o.level, buf.p, rlk, 0, s[o.dst].p, nb, st);
    }

    // TENSOR of op i into its degree-2 slot dst (made by the caller)
    int tensor_op(int i) {
        const lgpu_poly_op& o = pg->ops[i];
        const u64* w = d_w + w_off[i];
        if (!si) return tensor(o.src0, o.src1, o.addend, w, o.level, s[o.dst].p, cs(o.dst), bs(o.dst));
        const size_t N = c->N, nq = o.level + 1;
        Scratch buf;                                   // the product [3][nb][nq][N] and bfv_tensor's scratch
        if (buf.alloc((size_t)nb * 5 * nq * N, st)) return -1;
        if (bfv_tensor(c, *bgv, o.level, s[o.src0].p, s[o.src1].p, buf.p, nb, st)) return -1;
        const int a = o.addend;
        PolyTensorParams p;
        memset(&p, 0, sizeof(p));
        p.limbs = c->d_limbs;
        p.b = buf.p; p.b_cs = (size_t)nb * nq * N; p.b_bs = nq * N;
        p.a = a >= 0 ? s[a].p : nullptr; p.a_cs = a >= 0 ? cs(a) : 0; p.a_bs = a >= 0 ? bs(a) : 0; p.a_deg = a >= 0 ? s[a].deg : -1;
        p.wb = w; p.wa = w + nq;
        p.d = s[o.dst].p; p.d_cs = cs(o.dst); p.d_bs = bs(o.dst); p.n = c->N;
        ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * N * nq * nb * (6 + (p.a_deg + 1)), 1);
        poly_tensor_add_kernel<<<dim3((c->N + 255) / 256, (unsigned)nq, (unsigned)nb), 256, 0, st>>>(p);
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }

    // the term and output arrays of a LINCOMB / PTLINCOMB launch; makes the output slots
    template <class P>
    int lin_io(const lgpu_poly_op& o, P& p) {
        for (int k = 0; k < o.n_terms; k++) {
            const int t = o.terms[k];
            p.in[k] = s[t].p; p.in_cs[k] = (unsigned)cs(t); p.in_bs[k] = (unsigned)bs(t); p.in_level[k] = s[t].level;
        }
        for (int k = 0; k < o.n_out; k++) {
            const int d = o.outs[k];
            if (make(d)) return -1;
            p.out[k] = s[d].p; p.out_cs[k] = (unsigned)cs(d); p.out_bs[k] = (unsigned)bs(d); p.out_level[k] = o.out_levels[k];
        }
        return 0;
    }

    // PTLINCOMB: batch tiles of BT = min(8, nb) rounded up to a power of two (1, 2, 4, 8), so a sub-batch of up to 8 ciphertexts is
    // one tile and reads each plaintext word once; larger sub-batches read it once per 8 ciphertexts
    int pt_lincomb(int i) {
        const lgpu_poly_op& o = pg->ops[i];
        const size_t N = c->N;
        const int K1 = o.n_terms + 1;
        PtLincombParams p;
        p.limbs = c->d_limbs; p.w = d_w + w_off[i]; p.idx = p.w + (size_t)(o.level + 1) * o.n_out * K1;
        p.pt = (const u64*)vw->pt; p.pt_stride = vw->pt_stride;
        p.n_out = o.n_out; p.n_terms = o.n_terms; p.n = c->N; p.nb = nb;
        if (lin_io(o, p)) return -1;
        const int bt = nb > 4 ? 8 : nb > 2 ? 4 : nb, cj = 256 / bt, tiles = (nb + bt - 1) / bt;
        // bytes: powers once per entry, plaintexts once per tile (every (output, term) pair with a plaintext), outputs once
        double pts = 0;
        for (int k = 0; k < o.n_out; k++)
            for (int t = 0; t < K1; t++) pts += vw->index[k * K1 + t] >= 0 ? o.out_levels[k] + 1 : 0;
        ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * N * ((o.level + 1) * 2.0 * nb * o.n_terms + pts * tiles + 2.0 * nb * (o.level + 1) * o.n_out), 1);
        const dim3 grid((unsigned)((N + cj - 1) / cj), (unsigned)(o.level + 1), (unsigned)tiles);
        const size_t smem = ((size_t)o.n_out * K1 + (size_t)K1 * cj) * 8;
        switch (bt) {
        case 8: poly_pt_lincomb_kernel<8><<<grid, 256, smem, st>>>(p); break;
        case 4: poly_pt_lincomb_kernel<4><<<grid, 256, smem, st>>>(p); break;
        case 2: poly_pt_lincomb_kernel<2><<<grid, 256, smem, st>>>(p); break;
        default: poly_pt_lincomb_kernel<1><<<grid, 256, smem, st>>>(p); break;
        }
        LGPU_CUDA_OK(cudaGetLastError());
        return 0;
    }

    int op(int i) {
        const lgpu_poly_op& o = pg->ops[i];
        const size_t N = c->N;
        switch (o.kind) {
        case LGPU_POLY_MULRELIN:
            if (make(o.dst)) return -1;
            return mulrelin(o);
        case LGPU_POLY_TENSOR:
            if (make(o.dst)) return -1;
            return tensor_op(i);
        case LGPU_POLY_RELIN: {
            if (make(o.dst)) return -1;
            const int a = o.src0, d = o.dst;
            return evaluator_relinearize(c, o.level, CSpan{s[a].p, N, bs(a)}, CSpan{s[a].p + cs(a), N, bs(a)}, CSpan{s[a].p + 2 * cs(a), N, bs(a)}, rlk,
                                         Span{s[d].p, N, bs(d)}, Span{s[d].p + cs(d), N, bs(d)}, nb, st);
        }
        case LGPU_POLY_RESCALE: {
            if (make(o.dst)) return -1;
            const int a = o.src0, d = o.dst;
            // every polynomial of the sub-batch is one (level+1) x N block at a constant stride: one call for all of them
            return div_by_last_modulus_many(c, LGPU_RING_Q, s[a].level, true, true, pg->levels_per_rescale, CSpan{s[a].p, N, cs(a)}, Span{s[d].p, N, cs(d)},
                                            nb * (s[a].deg + 1), st);
        }
        case LGPU_POLY_LINCOMB: {
            LincombParams p;
            p.limbs = c->d_limbs; p.w = d_w + w_off[i]; p.n_out = o.n_out; p.n_terms = o.n_terms; p.n = c->N;
            if (lin_io(o, p)) return -1;
            const size_t smem = (size_t)o.n_out * (o.n_terms + 1) * 2 * 8;
            ProfScope ps(LGPU_KCLASS_VECOP, st, 8.0 * N * (o.level + 1) * nb * 2 * (o.n_terms + o.n_out), 1);
            poly_lincomb_kernel<<<dim3((c->N + 255) / 256, (unsigned)(o.level + 1), (unsigned)nb), 256, smem, st>>>(p);
            LGPU_CUDA_OK(cudaGetLastError());
            return 0;
        }
        case LGPU_POLY_PTLINCOMB:
            return pt_lincomb(i);
        }
        return 0;
    }
};


// what the BGV / BFV evaluators add to validate(): one modulus per rescale, and for BFV no RESCALE and operands at the op's level
int bgv_program_checks(const lgpu_poly_program& prog, const Plan& pl, int scale_invariant) {
    REQUIRE(prog.levels_per_rescale == 1, "levels_per_rescale must be 1 for BGV / BFV (Rescale drops one modulus)");
    if (!scale_invariant) return 0;
    for (int i = 0; i < prog.n_ops; i++) {
        const lgpu_poly_op& o = prog.ops[i];
        REQUIRE(o.kind != LGPU_POLY_RESCALE, "the scale-invariant (BFV) evaluator does not rescale: RESCALE in a scale_invariant program");
        // the scale-invariant tensor reads both operands as [batch][2][level+1][N]
        REQUIRE(!(o.kind == LGPU_POLY_MULRELIN || o.kind == LGPU_POLY_TENSOR) || (pl.level[o.src0] == o.level && pl.level[o.src1] == o.level),
                "scale-invariant MULRELIN / TENSOR operands must be at the op's level");
        // its operand ModUp Q -> QMul extends from all level + 1 Q moduli at once
        REQUIRE(!(o.kind == LGPU_POLY_MULRELIN || o.kind == LGPU_POLY_TENSOR) || o.level + 1 <= kMaxSrc,
                "the scale-invariant (BFV) multiplication supports at most 64 Q moduli");
    }
    return 0;
}

// the relinearization key, checked at every level a MULRELIN / RELIN uses it
int program_rlk(const Ctx& c, const lgpu_poly_program* prog, const lgpu_gadget_ct* rlk, GadgetCt& g) {
    bool needs_rlk = false;
    for (int i = 0; i < prog->n_ops; i++) needs_rlk |= prog->ops[i].kind == LGPU_POLY_MULRELIN || prog->ops[i].kind == LGPU_POLY_RELIN;
    if (!needs_rlk) return 0;
    if (to_gadget_ct(rlk, g, "null relinearization key")) return -1;
    for (int i = 0; i < prog->n_ops; i++)
        if ((prog->ops[i].kind == LGPU_POLY_MULRELIN || prog->ops[i].kind == LGPU_POLY_RELIN) && check_evk(&c, prog->ops[i].level, g)) return -1;
    return 0;
}

// runs a validated program over the batch, one batch_chunk() sub-batch at a time
int run_program(const Ctx& c, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog, const Plan& pl, const GadgetCt& g,
                const BgvState* bgv, bool si, uint64_t* ct_out, cudaStream_t st, const lgpu_poly_pt_weights* vw) {
    std::vector<u64> hw;
    std::vector<size_t> off(prog->n_ops, 0);
    for (int i = 0; i < prog->n_ops; i++) { off[i] = hw.size(); hw.insert(hw.end(), pl.w[i].begin(), pl.w[i].end()); }
    Scratch dw;
    if (!hw.empty()) {
        if (dw.alloc(hw.size(), st)) return -1;
        // pageable source: the call returns once `hw` is staged, so it may die with this function
        LGPU_CUDA_OK(cudaMemcpyAsync(dw.p, hw.data(), hw.size() * 8, cudaMemcpyHostToDevice, st));
    }
    const size_t N = c.N, ci = (size_t)2 * (level + 1) * N, co = (size_t)2 * (pl.level[prog->out_slot] + 1) * N;
    const int ch = batch_chunk();
    for (int k = 0; k < batch; k += ch) {
        const int nb = std::min(ch, batch - k);
        Runner R{&c, prog, pl, g, st, nb, std::vector<Slot>(prog->n_slots), dw.p, off, bgv, si, vw, (u64*)ct_out + (size_t)k * co};
        R.s[0].p = (u64*)ct_in + (size_t)k * ci; R.s[0].deg = 1; R.s[0].level = level;
        for (int i = 0; i < prog->n_ops; i++) {
            if (R.op(i)) return -1;
            for (int sl = 1; sl < prog->n_slots; sl++)
                if (pl.last_use[sl] == i && sl != prog->out_slot) R.release(sl);
        }
    }
    return 0;
}

// the four entry points after their handle checks (fn: the entry point's name, for its NVTX range). bgv: the BGV / BFV evaluator
// state, null for CKKS; vector: a vector entry point, whose plaintext table vw may not be null (vw is null for the scalar ones)
int evaluate(const char* fn, lgpu_ctx* ctx, const BgvState* bgv, int scale_invariant, int level, const uint64_t* ct_in, int batch,
             const lgpu_poly_program* prog, bool vector, const lgpu_poly_pt_weights* vw, const lgpu_gadget_ct* rlk, uint64_t* ct_out,
             void* stream) {
    const Ctx& c = ctx->c;
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(ct_in && ct_out, "null ciphertext");
    REQUIRE(!vector || vw, "null plaintext table");
    REQUIRE_ALIGNED(AL(ct_in) && AL(ct_out));
    Plan pl;
    if (validate(c, level, prog, pl, vw)) return -1;
    if (bgv && bgv_program_checks(*prog, pl, scale_invariant)) return -1;
    if (vw) {                                          // the plaintext block may not overlap the input or the output ciphertexts
        int ptmax = 0;
        for (int j = 0; j < vw->n_pt; j++) ptmax = std::max(ptmax, vw->pt_levels[j]);
        const size_t ptb = ((size_t)(vw->n_pt - 1) * vw->pt_stride + (size_t)(ptmax + 1) * c.N) * 8;
        const size_t inb = (size_t)batch * 2 * (level + 1) * c.N * 8, outb = (size_t)batch * 2 * (pl.level[prog->out_slot] + 1) * c.N * 8;
        REQUIRE(!overlaps(vw->pt, ptb, ct_in, inb) && !overlaps(vw->pt, ptb, ct_out, outb), "the plaintext block overlaps the input or the output");
    }
    GadgetCt g{};
    if (program_rlk(c, prog, rlk, g)) return -1;
    REQUIRE_DEVICE_AS(ctx, fn);
    return run_program(c, level, ct_in, batch, prog, pl, g, bgv, scale_invariant == 1, ct_out, (cudaStream_t)stream, vw);
}

}  // namespace
}  // namespace lgpu

using namespace lgpu;

extern "C" int lgpu_ckks_polynomial_evaluate(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                             const lgpu_gadget_ct* rlk, uint64_t* ct_out, void* stream) {
    REQUIRE(ctx, "null context");
    REQUIRE(ctx->c.ring_type == 0, "polynomial evaluation is not supported on the ConjugateInvariant ring");
    return evaluate(__func__, ctx, nullptr, 0, level, ct_in, batch, prog, false, nullptr, rlk, ct_out, stream);
}

extern "C" int lgpu_bgv_polynomial_evaluate(lgpu_bgv* ev, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                            const lgpu_gadget_ct* rlk, int scale_invariant, uint64_t* ct_out, void* stream) {
    REQUIRE(ev, "null BGV evaluator");
    REQUIRE(scale_invariant == 0 || scale_invariant == 1, "scale_invariant must be 0 or 1");
    return evaluate(__func__, ev->ctx, &ev->s, scale_invariant, level, ct_in, batch, prog, false, nullptr, rlk, ct_out, stream);
}

extern "C" int lgpu_ckks_polynomial_vector_evaluate(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                                    const lgpu_poly_pt_weights* pts, const lgpu_gadget_ct* rlk, uint64_t* ct_out, void* stream) {
    REQUIRE(ctx, "null context");
    REQUIRE(ctx->c.ring_type == 0, "polynomial evaluation is not supported on the ConjugateInvariant ring");
    return evaluate(__func__, ctx, nullptr, 0, level, ct_in, batch, prog, true, pts, rlk, ct_out, stream);
}

extern "C" int lgpu_bgv_polynomial_vector_evaluate(lgpu_bgv* ev, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                                   const lgpu_poly_pt_weights* pts, const lgpu_gadget_ct* rlk, int scale_invariant, uint64_t* ct_out,
                                                   void* stream) {
    REQUIRE(ev, "null BGV evaluator");
    REQUIRE(scale_invariant == 0 || scale_invariant == 1, "scale_invariant must be 0 or 1");
    return evaluate(__func__, ev->ctx, &ev->s, scale_invariant, level, ct_in, batch, prog, true, pts, rlk, ct_out, stream);
}

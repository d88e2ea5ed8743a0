// bgv.h -- the BGV / BFV evaluator state (lgpu_bgv) and the two tensor products that bgv.cu and polyeval.cu share.
#pragma once
#include <vector>
#include "capi_common.h"

namespace lgpu {

struct BgvState {
    Ctx qm;                          // (Q, QMul): Q limbs 0..nQ-1, QMul limbs nQ..nQ+nQMul-1
    u64 t = 0;
    std::vector<int> levelQMul;      // [level of Q]
    std::vector<size_t> lvl_off;     // [level of Q]: offset (words) of that level's quantize block in d_const
    // d_const: tmul[nQ] = MForm(t mod q_i) | tmont[nQ] = MForm(t 2^64 mod q_i) (tMontgomery) | per-level blocks:
    //   half1_s[nq]: floor(Q_l/2) mod q_i   half2_t[nq]: floor(QMul_lm/2) mod q_i   half1_t[nm]: floor(Q_l/2) mod p_j
    //   mdcs[nm]: p_j - modDownConstantsQtoP[l][j]   half2_s[nm]: floor(QMul_lm/2) mod p_j          (nm = levelQMul[l] + 1)
    std::vector<u64> h_const;
    u64* d_const = nullptr;

    const u64* tmont() const { return d_const + qm.nQ; }
};

// tensorScaleInvariant without relinearization (evaluator.go:898-1070 up to the quantize's NTT): the degree-2 product of the degree-1
// operands A, B ([batch][2][level+1][N], NTT domain; A == B is the squaring case) into d = [3][batch][level+1][N]. buf holds 2 more
// such blocks of scratch right after d (mulrelin_tail's [5][batch][level+1][N] layout).
int bfv_tensor(const Ctx* c, const BgvState& s, int level, const u64* A, const u64* B, u64* d, int batch, cudaStream_t st);

}  // namespace lgpu

struct lgpu_bgv {
    lgpu_ctx* ctx = nullptr;
    lgpu::BgvState s;
};

// lintrans.h -- host-side view used by lintrans.cu (mirror of lgpu_lintrans of the public header).
#pragma once
#include <map>
#include <vector>
#include "composite.h"

namespace lgpu {

struct LinTransView {        // lintrans.LinearTransformation, circuits/common/lintrans/lintrans.go:150-160
    int level_q, level_p, log_slots, n1, n_diags;
    const int* diag_index;   // host: keys of Vec
    const u64* const* diag;  // host array of device pointers: (level_q+1) Q rows then (level_p+1) P rows, NTT + Montgomery
};

void bsgs_index(const LinTransView& m, std::map<int, std::vector<int>>& index, std::vector<int>& rotN1, std::vector<int>& rotN2);
// accumulate: out = CRed(out + result) (needs QP-stacked outputs: out.p[k] right after the nq rows of out.q[k], one batch stride)
int automorphism_hoisted_lazy(const Ctx* c, int levelQ, CSpan ct0P, const u64* decomp, int decomp_levelQ, u64 galEl, const GadgetCt& gk,
                              const AccSpans& out, int batch, cudaStream_t st, bool accumulate = false);
// Galois key usable by the hoisted products at levelQ: levels in range, BaseTwoDecomposition = 0, enough digits (error set otherwise)
int check_gk(const Ctx* c, int levelQ, const GadgetCt& gk);
int lintrans_evaluate_many(const Ctx* c, int level_in, const u64* ct_in, const LinTransView* mats, int n_mats, const GaloisKeySet& gks,
                           u64* const* outs, int* out_levels, int batch, cudaStream_t st);

}  // namespace lgpu

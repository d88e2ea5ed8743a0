// composite.h -- prototypes of composite.cu (multi-kernel operations of the hot path).
#pragma once
#include <vector>
#include "engine.h"

namespace lgpu {

struct GadgetCt {          // device-side view of a rlwe.GadgetCiphertext (mirror of lgpu_gadget_ct)
    const u64* data;       // [digit][pw2][2][nQk + nPk][N], NTT + Montgomery (core/rlwe/gadgetciphertext.go:19-45)
    int levelQ, levelP;    // of the key
    int pw2;               // BaseTwoDecomposition
    int ndigits, npw2max;
    const int* pw2_sizes;  // host, per digit (nullptr => all 1)
    const u64* at(int d, int j, int comp, size_t N) const {
        const size_t rows = (size_t)(levelQ + 1) + (size_t)(levelP + 1);
        return data + ((((size_t)d * npw2max + j) * 2 + comp) * rows) * N;
    }
};
struct AccSpans {  // the four accumulator polynomials of a ctQP: [comp].Q (levelQ+1 rows) and [comp].P (levelP+1 rows)
    Span q[2];
    Span p[2];
};
// ncomp components x batch elements with rows of N words: component k of element b starts at p + k * cs + b * bs
struct CBlock {
    const u64* p;
    size_t cs, bs;
};
struct Block {
    u64* p;
    size_t cs, bs;
    operator CBlock() const { return CBlock{p, cs, bs}; }
};
struct GaloisKeySet {        // the GaloisKeys map of rlwe.MemEvaluationKeySet, core/rlwe/evaluationkeyset.go
    int n = 0;
    const u64* gal_els = nullptr;
    std::vector<GadgetCt> keys;
    const GadgetCt* find(u64 galEl) const;   // nullptr + error "GaloisKey[..] is missing"
};

struct Scratch {
    u64* p = nullptr;
    cudaStream_t st = nullptr;
    int alloc(size_t words, cudaStream_t s) {
        st = s;
        LGPU_CUDA_OK(cudaMallocAsync((void**)&p, words * sizeof(u64), s));
        return 0;
    }
    ~Scratch() { if (p) cudaFreeAsync(p, st); }
};

inline RowMap rows_range(int limb0, int drow0, int count) {
    RowMap rm;
    rm.nrows = count;
    for (int i = 0; i < count; i++) { rm.limb[i] = (unsigned char)(limb0 + i); rm.drow[i] = (unsigned char)(drow0 + i); }
    return rm;
}
// QP-stacked buffer: data rows [0, nq) are Q limbs 0.., rows [nq, nq+np) are P limbs 0..
inline RowMap rows_qp(const Ctx* c, int nq, int np) {
    RowMap rm;
    rm.nrows = nq + np;
    for (int i = 0; i < nq; i++) { rm.limb[i] = (unsigned char)i; rm.drow[i] = (unsigned char)i; }
    for (int j = 0; j < np; j++) { rm.limb[nq + j] = (unsigned char)(c->nQ + j); rm.drow[nq + j] = (unsigned char)(nq + j); }
    return rm;
}
// the accumulators of a [comp][batch][nq + np][N] block: each element's np P rows right after its nq Q rows
inline AccSpans stacked_acc(u64* base, size_t nq, size_t np, size_t N, int batch) {
    AccSpans a;
    for (int k = 0; k < 2; k++) {
        u64* b = base + (size_t)k * batch * (nq + np) * N;
        a.q[k] = Span{b, N, (nq + np) * N};
        a.p[k] = Span{b + nq * N, N, (nq + np) * N};
    }
    return a;
}

u64 galois_element(const Ctx* c, long long k);
// p * P_levelP mod q_i in Montgomery form, i <= levelQ: the per-limb scalars of ringQ.MulScalarBigint(., P, .)
std::vector<u64> p_mod_q_mont(const Ctx* c, int levelQ, int levelP);

int base_rns_decomposition_vector_size(int levelQ, int levelP);
int moddown_qp_to_q(const Ctx* c, int levelQ, int levelP, CSpan p1Q, CSpan p1P, Span p2Q, int batch, cudaStream_t st);
int moddown_qp_to_q_ntt(const Ctx* c, int levelQ, int levelP, CSpan p1Q, CSpan p1P, Span p2Q, int batch, cudaStream_t st);
int moddown_qp_to_p(const Ctx* c, int levelQ, int levelP, CSpan p1Q, CSpan p1P, Span p2P, int batch, cudaStream_t st);
int div_by_last_modulus_ntt(const Ctx* c, int ring, int level, bool round, CSpan p0, Span p1, int batch, cudaStream_t st);
int div_by_last_modulus(const Ctx* c, int ring, int level, bool round, CSpan p0, Span p1, int batch, cudaStream_t st);
int div_by_last_modulus_many(const Ctx* c, int ring, int level, bool round, bool ntt, int nb, CSpan p0, Span p1, int batch, cudaStream_t st);
int automorphism_ntt_index(const Ctx* c, u64 galEl, u64* d_index, cudaStream_t st);
int automorphism_ntt_with_index(const Ctx* c, int rows, CSpan in, const u64* d_index, Span out, bool accumulate, int batch, cudaStream_t st);
int automorphism_coeff(const Ctx* c, const RowMap& rm, CSpan in, u64 gen, Span out, int batch, cudaStream_t st);
int decompose_single_ntt(const Ctx* c, int levelQ, int levelP, int nbPi, int digit, CSpan c2NTT, CSpan c2Inv, Span c2Q, Span c2P,
                         bool copy_digit_rows, int batch, cudaStream_t st);
int decompose_ntt(const Ctx* c, int levelQ, int levelP, int nbPi, CSpan c2, bool c2IsNTT, u64* decomp, int batch, cudaStream_t st);
int gadget_product_lazy(const Ctx* c, int levelQ, CSpan cx, const GadgetCt& evk, const AccSpans& acc, int batch, cudaStream_t st);
int evaluator_moddown_ntt(const Ctx* c, int levelQ, int levelP, const AccSpans& acc, Span ct0, Span ct1, int batch, cudaStream_t st);
// out = ModDown(acc) (+ add) for ncomp x batch QP-stacked accumulators (nq Q rows, then the P rows), NTT domain; add.p == nullptr: no
// addend; add may alias out
int moddown_ntt(const Ctx* c, int levelQ, int levelP, CBlock acc, CBlock add, Block out, int ncomp, int batch, cudaStream_t st);
int gadget_product(const Ctx* c, int levelQ, CSpan cx, const GadgetCt& evk, Span ct0, Span ct1, int batch, cudaStream_t st);
int rgsw_external_product(const Ctx* c, const GadgetCt& rg0, const GadgetCt& rg1, CSpan ct0, CSpan ct1, Span out0, Span out1, int batch, cudaStream_t st);
// decomp_levelQ: level the DecomposeNTT buffer was laid out for (>= levelQ; -1 = levelQ) -- lintrans uses one decomposition for matrices of lower levels
int gadget_product_hoisted_lazy(const Ctx* c, int levelQ, const u64* decomp, const GadgetCt& evk, const AccSpans& acc, int batch, cudaStream_t st,
                                int decomp_levelQ = -1);
int gadget_product_hoisted(const Ctx* c, int levelQ, const u64* decomp, const GadgetCt& evk, Span ct0, Span ct1, int batch, cudaStream_t st);
int evaluator_automorphism(const Ctx* c, int level, CSpan in0, CSpan in1, u64 galEl, const GadgetCt& gk, Span out0, Span out1,
                           const u64* decomp_hoisted, int batch, cudaStream_t st);
int evaluator_relinearize(const Ctx* c, int level, CSpan c0, CSpan c1, CSpan c2, const GadgetCt& rlk, Span out0, Span out1, int batch, cudaStream_t st);
// keyswitch_fused.cu
bool ks_fused_applicable(const Ctx* c, int levelQ, const GadgetCt& evk);
int gadget_product_multiple_p_fused(const Ctx* c, int levelQ, CSpan cx, CSpan cxInv, const GadgetCt& evk, Block acc, int batch, cudaStream_t st);

bool fz_applicable(const Ctx* c, int levelQ, int levelP);
int moddown_ntt_fused(const Ctx* c, int levelQ, int levelP, CBlock acc, CBlock D, Block out, int ncomp, int batch, cudaStream_t st);
int div_round_last_ntt_fused(const Ctx* c, int level, CBlock X, Block out, int ncomp, int batch, cudaStream_t st);
// moddown_ntt_fused with addend D followed by div_round_last_ntt_fused (D is overwritten), in fewer passes when Q[levelQ] is an FP64-pipe prime
bool moddown_rescale_applicable(const Ctx* c, int level);
int moddown_rescale_ntt_fused(const Ctx* c, int levelQ, int levelP, CBlock acc, Block D, Block out, int ncomp, int batch, cudaStream_t st);

int ckks_mulrelin_rescale(const Ctx* c, int level, const u64* ctA, const u64* ctB, const GadgetCt& rlk, int nb_rescales, u64* out, int batch,
                          cudaStream_t st);
// shared by the CKKS and BGV/BFV multiplications (composite.cu, bgv.cu)
int check_evk(const Ctx* c, int levelQ, const GadgetCt& evk);
int batch_chunk();
int mulrelin_tail(const Ctx* c, int level, u64* d, const GadgetCt& rlk, int nb_rescales, u64* out, int batch, cudaStream_t st);

// encrypt.cu, shared with the multiparty shares (multiparty.cu)
int small_to_rns(const Ctx* c, const RowMap& rm, const long long* in, size_t in_bs, Span out, int batch, cudaStream_t st);
// batch entries of n words uniform in [0, m) on the mask domain of the Philox counter (the mpbgv masks, mp_refresh.cu)
int sample_mask(u64 m, int n, u64 seed, u64 stream_id, u64* out, size_t bs, int batch, cudaStream_t st);
// batch entries of n values uniform in [-2^(log_bound-1), 2^(log_bound-1)), W two's-complement words each (the mpckks masks)
int sample_big_mask(int n, int W, int log_bound, u64 seed, u64 stream_id, u64* out, size_t bs, int batch, cudaStream_t st);
int encrypt_zero_pk(const Ctx* c, int levelQ, const u64* pk, const long long* u, const long long* e0, const long long* e1, u64* ct_out,
                    bool is_ntt, bool is_mont, int batch, cudaStream_t st);
// A batch of gadget ciphertexts sharing levels and digit layout (KeyGenerator.genEvaluationKey, keygenerator.go:287-330; rgsw.Encryptor,
// core/rgsw/encryptor.go:25-121; the multiparty key-generation shares): per ciphertext, every entry (i, j) gets
//   component 0 = e_ij - c1_ij s_out (+ f_j pt on the Q limbs of digit i when target == 0), component 1 = c1_ij (+ f_j pt when target == 1)
// with f_j = P_levelP 2^(pw2 j) (Montgomery form and e taken to Montgomery form when mont). Entries with j >= pw2_sizes[i] get only the
// encryption of zero.
struct GadgetEncLayout {
    int levelQ, levelP, pw2, n_digits, n_pw2_max;
    const int* pw2_sizes;     // host, per digit; nullptr = all n_pw2_max
    size_t c0_es, c1_es;      // entry strides (words) of component 0 and of component 1 (input c1 and c1_out alike)
    bool mont;
};
struct GadgetEncCt {
    u64* c0;                  // entry (i, j) at c0 + (i n_pw2_max + j) c0_es: level_q+1 Q rows then level_p+1 P rows
    const u64* c1;            // uniform component 1 (NTT domain), ignored when gadget_encrypt draws it
    u64* c1_out;              // component 1 output (may equal c1); nullptr when it is neither drawn nor the target
    const u64* s_out;         // [nQ + nP][N] secret key, NTT + Montgomery
    u64 gal_el;               // != 0: encrypt under AutomorphismNTT(s_out, gal_el^-1 mod 2N) instead (a Galois key)
    const u64* pt;            // rows 0..levelQ (stride N), NTT + Montgomery, or nullptr (an encryption of zero)
    int target;               // 0 or 1
};
struct GadgetEncDraw { u64 seed, stream0; double sigma, bound; };   // ciphertext m draws c1 and e on stream id stream0 + m
// e: [n_cts][n_digits][n_pw2_max][N] signed errors, or nullptr with draw != nullptr
int gadget_encrypt(const Ctx* c, const GadgetEncLayout& g, const GadgetEncCt* cts, int n_cts, const long long* e, const GadgetEncDraw* draw,
                   cudaStream_t st);
int base_two_decomposition_size(const Ctx* c, int levelP, int pw2, int i);
}  // namespace lgpu

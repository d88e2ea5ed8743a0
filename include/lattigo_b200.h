/*
 * lattigo_b200.h -- C ABI of the H100-native RNS polynomial-ring engine.
 *
 * Drop-in boundary for ONE hot path of tuneinsight/lattigo v6.2.0: the `ring` package's NTT /
 * coefficient-wise / basis-extension / rescale / automorphism loops and core/rlwe.Evaluator's
 * GadgetProduct key-switch family. The reference has no FFI of its own (pure Go); each entry point
 * below names the Go method it replaces (file:line relative to the upstream tree) and is what a thin
 * cgo shim in forked `ring`, `ring/ringqp` and `core/rlwe` packages binds (see INTEGRATION.md).
 *
 * Conventions
 *   - Polynomials are `uint64_t*` DEVICE-ACCESSIBLE pointers (cudaMalloc / managed / lgpu_malloc) to a
 *     contiguous (limb, coeff) row-major block: row i = residues mod the i-th modulus, N words per row.
 *     ring.Poly{Coeffs [][]uint64} (ring/poly.go:13-15) maps onto it with Coeffs[i] = row i.
 *   - Alignment: lgpu_malloc / cudaMalloc blocks are always fine. The ring-level entry points accept any
 *     8-byte aligned pointer (odd word offsets take 64-bit kernels); the rlwe-level ones (gadget products,
 *     evaluator_*, ckks_*) and evaluation keys require 16-byte aligned blocks and even strides, and return
 *     an error otherwise (their kernels move 128 bits per access, the widest global access on sm_90).
 *   - `ring` selects the moduli chain: LGPU_RING_Q or LGPU_RING_P (ringqp.Ring{RingQ,RingP},
 *     ring/ringqp/ring.go:15-17). `level` is the reference's level (number of limbs - 1).
 *   - All calls are asynchronous on `stream` (a cudaStream_t cast to void*; NULL = the CUDA default
 *     stream); lgpu_sync() before host access. Entry points ending in _host take HOST pointers and
 *     include the copies.
 *   - Return 0 on success, non-zero on error with lgpu_last_error() (thread-local) describing it.
 *     The shim maps ring-level errors to panic and evaluator-level errors to `error` like the
 *     reference (ring/ntt.go:212, core/rlwe/evaluator_gadget_product.go:110-112).
 *   - Outputs are bit-identical to the reference on identical inputs: canonical residues for the
 *     non-Lazy methods, the reference's exact representative for the *Lazy ones.
 */
#ifndef LATTIGO_B200_H
#define LATTIGO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lgpu_ctx lgpu_ctx;

#define LGPU_RING_Q 0
#define LGPU_RING_P 1

#define LGPU_RING_STANDARD 0           /* ring.Standard            (ring/ring.go:27-31) */
#define LGPU_RING_CONJUGATE_INVARIANT 1 /* ring.ConjugateInvariant  */

/* Opcodes of lgpu_vecop / lgpu_subring_vecop: one per kernel of ring/vec_ops.go, named after the
 * SubRing method that wraps it (ring/subring_ops.go:6-273). */
enum lgpu_vecop_code {
    LGPU_OP_ADD = 0,                             /* SubRing.Add                              vec_ops.go:7   */
    LGPU_OP_ADDLAZY,                             /* AddLazy                                  :31  */
    LGPU_OP_SUB,                                 /* Sub                                      :55  */
    LGPU_OP_SUBLAZY,                             /* SubLazy                                  :79  */
    LGPU_OP_NEG,                                 /* Neg                                      :103 */
    LGPU_OP_REDUCE,                              /* Reduce                                   :125 */
    LGPU_OP_REDUCELAZY,                          /* ReduceLazy                               :147 */
    LGPU_OP_MULCOEFFSLAZY,                       /* MulCoeffsLazy                            :169 */
    LGPU_OP_MULCOEFFSLAZYTHENADDLAZY,            /* MulCoeffsLazyThenAddLazy                 :193 */
    LGPU_OP_MULCOEFFSBARRETT,                    /* MulCoeffsBarrett                         :217 */
    LGPU_OP_MULCOEFFSBARRETTLAZY,                /* MulCoeffsBarrettLazy                     :241 */
    LGPU_OP_MULCOEFFSBARRETTTHENADD,             /* MulCoeffsBarrettThenAdd                  :265 */
    LGPU_OP_MULCOEFFSBARRETTTHENADDLAZY,         /* MulCoeffsBarrettThenAddLazy              :289 */
    LGPU_OP_MULCOEFFSMONTGOMERY,                 /* MulCoeffsMontgomery                      :313 */
    LGPU_OP_MULCOEFFSMONTGOMERYLAZY,             /* MulCoeffsMontgomeryLazy                  :336 */
    LGPU_OP_MULCOEFFSMONTGOMERYTHENADD,          /* MulCoeffsMontgomeryThenAdd               :360 */
    LGPU_OP_MULCOEFFSMONTGOMERYTHENADDLAZY,      /* MulCoeffsMontgomeryThenAddLazy           :383 */
    LGPU_OP_MULCOEFFSMONTGOMERYLAZYTHENADDLAZY,  /* MulCoeffsMontgomeryLazyThenAddLazy       :407 */
    LGPU_OP_MULCOEFFSMONTGOMERYTHENSUB,          /* MulCoeffsMontgomeryThenSub               :431 */
    LGPU_OP_MULCOEFFSMONTGOMERYTHENSUBLAZY,      /* MulCoeffsMontgomeryThenSubLazy           :455 */
    LGPU_OP_MULCOEFFSMONTGOMERYLAZYTHENSUBLAZY,  /* MulCoeffsMontgomeryLazyThenSubLazy       :479 */
    LGPU_OP_MULCOEFFSMONTGOMERYLAZYTHENNEG,      /* MulCoeffsMontgomeryLazyThenNeg           :504 */
    LGPU_OP_ADDLAZYTHENMULSCALARMONTGOMERY,      /* AddLazyThenMulScalarMontgomery (s0)      :529 */
    LGPU_OP_ADDSCALARLAZYTHENMULSCALARMONTGOMERY,/* AddScalarLazyThenMulScalarMontgomery(s0,s1) :553 */
    LGPU_OP_ADDSCALAR,                           /* AddScalar (s0)                           :575 */
    LGPU_OP_ADDSCALARLAZY,                       /* AddScalarLazy (s0)                       :597 */
    LGPU_OP_ADDSCALARLAZYTHENNEGTWOMODULUSLAZY,  /* AddScalarLazyThenNegTwoModulusLazy (s0)  :619 */
    LGPU_OP_SUBSCALAR,                           /* SubScalar (s0)                           :642 */
    LGPU_OP_MULSCALARMONTGOMERY,                 /* MulScalarMontgomery (s0)                 :664 */
    LGPU_OP_MULSCALARMONTGOMERYLAZY,             /* MulScalarMontgomeryLazy (s0)             :686 */
    LGPU_OP_MULSCALARMONTGOMERYTHENADD,          /* MulScalarMontgomeryThenAdd (s0)          :708 */
    LGPU_OP_MULSCALARMONTGOMERYTHENADDSCALAR,    /* MulScalarMontgomeryThenAddScalar (s0,s1=scalarMont) :730 */
    LGPU_OP_SUBTHENMULSCALARMONTGOMERYTWOMODULUS,/* SubThenMulScalarMontgomeryTwoModulus (s0): (p1 - p2 + 2q) * s0  :752 */
    LGPU_OP_MFORM,                               /* MForm                                    :778 */
    LGPU_OP_MFORMLAZY,                           /* MFormLazy                                :800 */
    LGPU_OP_IMFORM,                              /* IMForm                                   :822 */
    LGPU_OP_ZERO,                                /* ZeroVec                                  :847 */
    LGPU_OP_MASK,                                /* MaskVec (w = s0, mask = s1)              :870 */
    LGPU_OP_COUNT
};

/* ---- context ------------------------------------------------------------------------------------ */
/* ring.NewRing x2 + ring.NewBasisExtender + ring.NewDecomposer (ring/ring.go:258-322,
 * ring/basis_extension.go:52-87,318-377): builds every per-prime constant (BRed/MRed constants, NInv,
 * RootsForward/RootsBackward with the reference's primitive-root choice ring/subring.go:161-194,
 * RescaleConstants ring/ring.go:329-346, ModUp/ModDown/Decomposer constants) and uploads them.
 * `p` may be NULL / np = 0 (ring-only use). N = 2^logN, 16 <= N <= 2^17. */
int lgpu_create(lgpu_ctx** out, int device, int logN, int ring_type,
                const uint64_t* q, int nq, const uint64_t* p, int np);
void lgpu_destroy(lgpu_ctx* ctx);
const char* lgpu_last_error(void);
const char* lgpu_version(void);
int lgpu_sync(lgpu_ctx* ctx, void* stream);

/* Table read-back (host buffers) so the Go shim / tests can check the constants against the
 * reference's exported fields (SubRing.Modulus/MRedConstant/BRedConstant/NInv/RootsForward/
 * RootsBackward, ring/subring.go:15-35, ring/ntt.go:38-44). kind: 0 = {q, qinv, bred_hi, bred_lo, ninv,
 * primitive_root} (6 words), 1 = RootsForward (NthRoot/2 words), 2 = RootsBackward,
 * 3 = RescaleConstants row `limb-1` (limb words; Q or P ring). */
int lgpu_ring_get_table(lgpu_ctx* ctx, int ring, int limb, int kind, uint64_t* host_out, size_t nwords);
/* Replaces the generated root tables of one limb by caller-supplied ones (the Go structs' own tables),
 * so constants are identical by construction. */
int lgpu_ring_set_roots(lgpu_ctx* ctx, int ring, int limb, const uint64_t* roots_fwd, const uint64_t* roots_bwd,
                        uint64_t ninv);

/* ---- device memory (mirrors BufferPool.Get / Recycle, ring/pool.go:40-61) ---------------------------- */
int lgpu_malloc(lgpu_ctx* ctx, void** dptr, size_t bytes);
int lgpu_free(lgpu_ctx* ctx, void* dptr);
int lgpu_memcpy_h2d(lgpu_ctx* ctx, void* dst, const void* src, size_t bytes, void* stream);
int lgpu_memcpy_d2h(lgpu_ctx* ctx, void* dst, const void* src, size_t bytes, void* stream);

/* ---- NTT ----------------------------------------------------------------------------------------------
 * Ring.NTT / NTTLazy / INTT / INTTLazy (ring/ntt.go:127-152). In-place (in == out) allowed.
 * lazy != 0 returns NTTLazy's representative in [0, 6q) (exact reference schedule); INTTLazy is fully
 * reduced for N >= 16 like the reference (ring/ntt.go:197-206). `batch` polynomials, `batch_stride`
 * words apart (use batch = 1, batch_stride = 0 for a single polynomial). */
int lgpu_ntt(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t* out, int lazy,
             int batch, size_t batch_stride, void* stream);
int lgpu_intt(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t* out, int lazy,
              int batch, size_t batch_stride, void* stream);
/* Ring.NTT(in, out) followed by Ring.MulCoeffsMontgomery(out, other, out) (ring/ntt.go:127-131 + ring/operations.go:88-92) as
 * one pass over HBM: the product is applied in the transform's last pass (N = 2^13..2^16; two launches otherwise).
 * `other` must not alias `out`; in == out is allowed. */
int lgpu_ntt_then_mul_coeffs_montgomery(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, const uint64_t* other,
                                        uint64_t* out, int batch, size_t batch_stride, void* stream);
/* SubRing.NTT / NTTLazy / INTT / INTTLazy on one row (ring/subring_ops.go:235-253) */
int lgpu_subring_ntt(lgpu_ctx* ctx, int ring, int limb, const uint64_t* in, uint64_t* out, int lazy, void* stream);
int lgpu_subring_intt(lgpu_ctx* ctx, int ring, int limb, const uint64_t* in, uint64_t* out, int lazy, void* stream);

/* ---- coefficient-wise ops -------------------------------------------------------------------------------
 * Ring-level (ring/operations.go:11-392): loops over limbs 0..level. `scalars0/1` are HOST arrays with
 * one value per limb (NULL when the op takes none), e.g. AddScalar passes scalar mod q_i, MulScalar passes
 * MForm(scalar mod q_i). p1/p2 may be NULL for ops that do not read them. */
int lgpu_vecop(lgpu_ctx* ctx, int ring, int level, int opcode, const uint64_t* p1, const uint64_t* p2,
               uint64_t* p3, const uint64_t* scalars0, const uint64_t* scalars1,
               int batch, size_t batch_stride, void* stream);
/* SubRing-level (ring/subring_ops.go:6-273): one row of n words (n <= N) with immediate scalars. */
int lgpu_subring_vecop(lgpu_ctx* ctx, int ring, int limb, int opcode, const uint64_t* p1, const uint64_t* p2,
                       uint64_t* p3, uint64_t s0, uint64_t s1, int n, void* stream);


/* ---- automorphisms (ring/automorphism.go) --------------------------------------------------------------- */
/* AutomorphismNTTIndex (:12-34): writes the N-entry uint64 look-up table to DEVICE memory `index_out`. */
int lgpu_automorphism_ntt_index(lgpu_ctx* ctx, uint64_t gal_el, uint64_t* index_out, void* stream);
/* Ring.AutomorphismNTTWithIndex (:50-77) and ...ThenAddLazy (:82-109, accumulate != 0). Cannot be in-place. */
int lgpu_automorphism_ntt_with_index(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, const uint64_t* index,
                                     uint64_t* out, int accumulate, int batch, size_t batch_stride, void* stream);
/* Ring.AutomorphismNTT (:38-45): index computed on the fly. */
int lgpu_automorphism_ntt(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t gal_el, uint64_t* out,
                          int batch, size_t batch_stride, void* stream);
/* Ring.Automorphism (:113-176), coefficient domain, Standard ring. Cannot be in-place. */
int lgpu_automorphism(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, uint64_t gal_el, uint64_t* out,
                      int batch, size_t batch_stride, void* stream);

/* Ring.Shift (ring/operations.go:278-282): out[i] = in[(i + k) mod N] on rows 0..level. In-place allowed. */
int lgpu_shift(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, int k, uint64_t* out,
               int batch, size_t batch_stride, void* stream);
/* Ring.MultByMonomial (ring/operations.go:306-363): out = in * X^k, k > -2N, with the reference's literal
 * `q - x` negation (a wrapped zero coefficient becomes q). In-place allowed. */
int lgpu_mult_by_monomial(lgpu_ctx* ctx, int ring, int level, const uint64_t* in, int k, uint64_t* out,
                          int batch, size_t batch_stride, void* stream);
/* MapSmallDimensionToLargerDimensionNTT (ring/operations.go:380-392): large[r][i*gap + w] = small[r][i],
 * `rows` contiguous rows of n_small resp. n_large words. */
int lgpu_map_small_dimension_to_larger_dimension_ntt(lgpu_ctx* ctx, const uint64_t* pol_small, int n_small,
                                                     uint64_t* pol_large, int n_large, int rows, void* stream);
/* ringqp.Ring.ExtendBasisSmallNormAndCenter (ring/ringqp/operations.go:325-351): reads row 0 of poly_in_q,
 * writes level_p+1 rows of poly_out_p (the copy polyOutQ = polyInQ is the caller's). */
int lgpu_extend_basis_small_norm_and_center(lgpu_ctx* ctx, const uint64_t* poly_in_q, int level_p, uint64_t* poly_out_p,
                                            int batch, size_t stride_q, size_t stride_p, void* stream);

/* bootstrapping.Evaluator.ModUp's coefficient loops (circuits/ckks/bootstrapping/evaluator.go:652-699, :729-741): the value of row 0 (mod q_0,
 * coefficient domain) centred around q_0 and written modulo q_i on rows first_q..level_q of out_q and modulo p_j on rows 0..level_p of out_p
 * (level_p = -1: none). strict = 0 uses the reference's `coeff >= q/2` test (ctIn.Value[0], and Value[1] without ephemeral key), strict = 1
 * its `coeff > q/2` (Value[1] on the sparse-key path). Literal: a negative multiple of a modulus is written as that modulus. */
int lgpu_modup_centered(lgpu_ctx* ctx, const uint64_t* row0, int first_q, int level_q, int level_p, int strict, uint64_t* out_q,
                        uint64_t* out_p, int batch, size_t stride_in, size_t stride_q, size_t stride_p, void* stream);

/* ---- RNS basis extension (ring/basis_extension.go) -------------------------------------------------------
 * polQ has levelQ+1 rows, polP has levelP+1 rows; `batch` polynomials with the given strides (words).
 * One basis extension takes at most 64 source limbs (ModUpQtoP up to level_q = 63, ModUpPtoQ up to level_p = 63, and
 * DecomposeAndSplit digits of up to 64 limbs); more returns an error. The reference's reconstructRNS stops at 32 source
 * limbs; from 33 to 64 the result is its formula (same float64 `v`, same representative) applied to more limbs. */
/* BasisExtender.ModUpQtoP (:177-190) / ModUpPtoQ (:195-209): outputs are the reference's exact (non-canonical,
 * < 2p) representatives. */
int lgpu_modup_qtop(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* pol_q, uint64_t* pol_p,
                    int batch, size_t stride_q, size_t stride_p, void* stream);
int lgpu_modup_ptoq(lgpu_ctx* ctx, int level_p, int level_q, const uint64_t* pol_p, uint64_t* pol_q,
                    int batch, size_t stride_p, size_t stride_q, void* stream);
/* BasisExtender.ModDownQPtoQ (:215-228), ModDownQPtoQNTT (:235-256), ModDownQPtoP (:262-278) */
int lgpu_moddown_qp_to_q(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* p1q, const uint64_t* p1p, uint64_t* p2q,
                         int batch, size_t stride_q, size_t stride_p, void* stream);
int lgpu_moddown_qp_to_q_ntt(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* p1q, const uint64_t* p1p, uint64_t* p2q,
                             int batch, size_t stride_q, size_t stride_p, void* stream);
int lgpu_moddown_qp_to_p(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* p1q, const uint64_t* p1p, uint64_t* p2p,
                         int batch, size_t stride_q, size_t stride_p, void* stream);
/* Decomposer.DecomposeAndSplit (:381-502). p0q: coefficient domain. In the reconstruction branch the rows of
 * p1q that belong to the digit itself are left untouched (the reference leaves unspecified values there and its
 * only caller, DecomposeSingleNTT, overwrites them). */
int lgpu_decompose_and_split(lgpu_ctx* ctx, int level_q, int level_p, int nb_pi, int digit, const uint64_t* p0q,
                             uint64_t* p1q, uint64_t* p1p, int batch, size_t stride_q, size_t stride_p, void* stream);

/* ---- rescaling (ring/scaling.go) ---------------------------------------------------------------------------
 * Ring.DivRoundByLastModulus[NTT] (:101-144), DivFloorByLastModulus[NTT] (:6-33) and the *Many forms
 * (:37-97, :148-212). `level` = input level; the output has level - nb_rescales + 1 rows. flags: bit0 = round
 * (else floor), bit1 = NTT domain. In-place allowed. Strides in words. */
#define LGPU_DIV_ROUND 1
#define LGPU_DIV_NTT 2
int lgpu_div_by_last_modulus_many(lgpu_ctx* ctx, int ring, int level, int flags, int nb_rescales, const uint64_t* p0,
                                  uint64_t* p1, int batch, size_t stride_in, size_t stride_out, void* stream);

/* ---- rlwe.Evaluator key-switch family (core/rlwe/evaluator_gadget_product.go) --------------------------------
 * Evaluation keys are uploaded once as a device array in the layout of rlwe.GadgetCiphertext.Value
 * (core/rlwe/gadgetciphertext.go:19-45): data[digit][pw2][component][limb][coeff] with the (level_q+1) Q limbs
 * first, then the (level_p+1) P limbs; always NTT + Montgomery form (core/rlwe/keygenerator.go:309-318). */
typedef struct {
    const uint64_t* data;         /* device pointer */
    int level_q, level_p;         /* levels of the key (level_p = -1: no P) */
    int base_two_decomposition;   /* GadgetCiphertext.BaseTwoDecomposition */
    int n_digits;                 /* len(Value) */
    int n_pw2_max;                /* max_i len(Value[i]) (second array dimension) */
    const int* pw2_sizes;         /* HOST array, len(Value[i]) per digit; NULL = all 1 */
} lgpu_gadget_ct;

/* Evaluator.GadgetProduct (:16-36): ct = ModDown(<decomp(cx), evk>), cx and ct in the NTT domain.
 * cx: level_q+1 rows; ct0/ct1: level_q+1 rows each. batch with strides in words. */
int lgpu_gadget_product(lgpu_ctx* ctx, int level_q, const uint64_t* cx, const lgpu_gadget_ct* evk,
                        uint64_t* ct0, uint64_t* ct1, int batch, size_t stride_cx, size_t stride_ct, void* stream);
/* Evaluator.GadgetProductLazy (:108-127): result mod QP, not divided by P. acc{0,1}q: level_q+1 rows,
 * acc{0,1}p: level_p+1 rows (canonical residues, as the reference's trailing Reduce leaves them). */
int lgpu_gadget_product_lazy(lgpu_ctx* ctx, int level_q, const uint64_t* cx, const lgpu_gadget_ct* evk,
                             uint64_t* acc0q, uint64_t* acc0p, uint64_t* acc1q, uint64_t* acc1p,
                             int batch, size_t stride_cx, size_t stride_q, size_t stride_p, void* stream);
/* Evaluator.ModDown (:39-97), NTT -> NTT case: ct[k] = ModDownQPtoQNTT(acc[k]). */
int lgpu_evaluator_moddown(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* acc0q, const uint64_t* acc0p,
                           const uint64_t* acc1q, const uint64_t* acc1p, uint64_t* ct0, uint64_t* ct1,
                           int batch, size_t stride_q, size_t stride_p, size_t stride_ct, void* stream);
/* Evaluator.DecomposeSingleNTT (:487-510). c2ntt / c2inv: the input in and out of the NTT domain. */
int lgpu_decompose_single_ntt(lgpu_ctx* ctx, int level_q, int level_p, int nb_pi, int digit, const uint64_t* c2ntt,
                              const uint64_t* c2inv, uint64_t* c2q, uint64_t* c2p, int batch, size_t stride_in,
                              size_t stride_q, size_t stride_p, void* stream);
/* Evaluator.DecomposeNTT (:459-483). decomp: device array [digit][batch][level_q+1 + level_p+1][N]
 * (BuffDecompQP[digit].Q rows then .P rows). */
int lgpu_decompose_ntt(lgpu_ctx* ctx, int level_q, int level_p, int nb_pi, const uint64_t* c2, int c2_is_ntt,
                       uint64_t* decomp, int batch, size_t stride_in, void* stream);
/* Evaluator.GadgetProductHoisted (:348-368) / GadgetProductHoistedLazy (:381-399) on a DecomposeNTT result. */
int lgpu_gadget_product_hoisted(lgpu_ctx* ctx, int level_q, const uint64_t* decomp, const lgpu_gadget_ct* evk,
                                uint64_t* ct0, uint64_t* ct1, int batch, size_t stride_ct, void* stream);
int lgpu_gadget_product_hoisted_lazy(lgpu_ctx* ctx, int level_q, const uint64_t* decomp, const lgpu_gadget_ct* evk,
                                     uint64_t* acc0q, uint64_t* acc0p, uint64_t* acc1q, uint64_t* acc1p,
                                     int batch, size_t stride_q, size_t stride_p, void* stream);
/* Evaluator.Automorphism (core/rlwe/evaluator_automorphism.go:13-57) and AutomorphismHoisted (:63-102,
 * decomp != NULL), degree-1 NTT-domain ciphertexts stored as [batch][2][level+1][N]. */
int lgpu_evaluator_automorphism(lgpu_ctx* ctx, int level, const uint64_t* ct_in, uint64_t gal_el,
                                const lgpu_gadget_ct* gk, const uint64_t* decomp, uint64_t* ct_out, int batch, void* stream);
/* Evaluator.Relinearize (core/rlwe/evaluator_evaluationkey.go:121-148): ct_in [batch][3][level+1][N] ->
 * ct_out [batch][2][level+1][N]. */
int lgpu_evaluator_relinearize(lgpu_ctx* ctx, int level, const uint64_t* ct_in, const lgpu_gadget_ct* rlk,
                               uint64_t* ct_out, int batch, void* stream);

/* ---- hoisted linear transformations (circuits/common/lintrans/lintrans_evaluator.go) -------------------------------
 * lintrans.LinearTransformation (lintrans.go:150-160) with its diagonals resident on the device. */
typedef struct {
    int level_q, level_p;          /* LinearTransformation.LevelQ / LevelP */
    int log_slots;                 /* LogDimensions.Cols: rotations are taken modulo 2^log_slots */
    int n1;                        /* N1: 0 = naive evaluator (one key per diagonal), else the BSGS baby-step count (power of two) */
    int n_diags;                   /* len(Vec) */
    const int* diag_index;         /* HOST: the keys of Vec */
    const uint64_t* const* diag;   /* HOST array of DEVICE pointers; diag[i] = Vec[diag_index[i]] as a ringqp.Poly block:
                                      (level_q+1) Q rows then (level_p+1) P rows, NTT + Montgomery form */
} lgpu_lintrans;
/* The GaloisKeys of an rlwe.EvaluationKeySet (core/rlwe/evaluationkeyset.go): gal_els[i] -> keys[i]. HOST arrays. */
typedef struct {
    int n_keys;
    const uint64_t* gal_els;
    const lgpu_gadget_ct* keys;
} lgpu_galois_keys;
/* rlwe.Parameters.GaloisElement (core/rlwe/params.go:580-583): GaloisGen^k mod NthRoot, k may be negative. */
uint64_t lgpu_galois_element(lgpu_ctx* ctx, long long k);
/* lintrans.Evaluator.EvaluateMany (:28-79; Evaluate / EvaluateNew are the one-matrix calls): decomposes ct_in[1] once,
 * pre-rotates the baby steps once for all BSGS matrices (AutomorphismHoistedLazy, :82-114), then MultiplyByDiagMatrix
 * (:141-274) or MultiplyByDiagMatrixBSGS (:280-470) per matrix. ct_in: [batch][2][level_in+1][N], NTT domain.
 * ct_outs: HOST array of n_mats device pointers, ct_outs[i]: [batch][2][out_levels[i]+1][N]; on return out_levels[i] is the
 * level of the result = min(out_levels[i], level_in, mats[i].level_q) (the reference Resizes opOut): rows 0..that level of
 * each component are written, the block keeps its layout. ct_outs[i] == ct_in is allowed (EvaluateSequential, :117-139).
 * A missing Galois key is an error ("GaloisKey[g] is missing"), like CheckAndGetGaloisKey. */
int lgpu_lintrans_evaluate_many(lgpu_ctx* ctx, int level_in, const uint64_t* ct_in, const lgpu_lintrans* mats, int n_mats,
                                const lgpu_galois_keys* gks, uint64_t* const* ct_outs, int* out_levels, int batch, void* stream);
/* Evaluator.AutomorphismHoistedLazy (core/rlwe/evaluator_automorphism.go:107-165), NTT-domain ciphertexts: the result stays
 * modulo QP, scaled by P. ct0: ctIn.Value[0] (level_q+1 rows used); decomp: lgpu_decompose_ntt output laid out for
 * decomp_level_q >= level_q. Outputs as in lgpu_gadget_product_lazy. */
int lgpu_evaluator_automorphism_hoisted_lazy(lgpu_ctx* ctx, int level_q, const uint64_t* ct0, const uint64_t* decomp, int decomp_level_q,
                                             uint64_t gal_el, const lgpu_gadget_ct* gk, uint64_t* out0q, uint64_t* out0p, uint64_t* out1q,
                                             uint64_t* out1p, int batch, size_t stride_ct, size_t stride_q, size_t stride_p, void* stream);

/* ---- slot aggregation (core/rlwe/inner_sum.go), Standard ring only -------------------------------------------------------
 * Evaluator.PartialTracesSum (:147-292): ct_out = sum_{i<n} phi(i * offset)(ct_in), phi(k) = Automorphism by GaloisElement(k), with
 * the reference's schedule: log2(n) + HW(n) - 1 key switches, one DecomposeNTT per doubling step, the terms of the non-power-of-two
 * bits accumulated mod QP and divided by P once. InnerSum / RotateAndAdd: offset = batchSize; Replicate: offset = -batchSize.
 * ct_in, ct_out: [batch][2][level+1][N]; is_ntt = 0: coefficient domain in and out (with n = 1 the output is INTT(ct_in), as the
 * reference's copy followed by its trailing INTT). ct_out == ct_in allowed, no other overlap.
 * Errors: n <= 0 or offset == 0 ("partialtrace: invalid parameter (n = 0 or batchSize = 0)"), a ConjugateInvariant ctx, n >= 2
 * without a P ring, a key with levelP != MaxLevelP or BaseTwoDecomposition != 0, a missing key ("GaloisKey[g] is missing").
 * Unlike the reference, which fails at the first missing key after part of the work, every key is checked before any device work;
 * the argument checks also run on a host-only ctx. */
int lgpu_evaluator_partial_traces_sum(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int is_ntt, int offset, int n,
                                      const lgpu_galois_keys* gks, uint64_t* ct_out, int batch, void* stream);
/* Evaluator.Trace (:36-116), 0 <= log_n <= LogN - 1: keeps the plaintext coefficients whose index is a multiple of
 * gap = 2^(LogN - log_n - 1) (gap = N for log_n = 0) and zeroes the others; gap = 1 is a copy. ct_in: [batch][2][level_in+1][N],
 * ct_out: [batch][2][level_out+1][N]; the result is at level min(level_in, level_out) and rows 0..that level of each component are
 * written, the block keeps its layout (as in lgpu_lintrans_evaluate_many). ct_out == ct_in allowed (with level_out == level_in).
 * Keys: GaloisElement(2^i) for log_n <= i < LogN - 1, and NthRoot - 1 for log_n = 0, with a P ring and BaseTwoDecomposition = 0;
 * errors as for lgpu_evaluator_partial_traces_sum, checked before any device work. */
int lgpu_evaluator_trace(lgpu_ctx* ctx, int level_in, const uint64_t* ct_in, int is_ntt, int log_n, const lgpu_galois_keys* gks,
                         uint64_t* ct_out, int level_out, int batch, void* stream);

/* ---- ring packing (core/rlwe/ring_packing.go), Standard ring only -------------------------------------------------------------
 * RingPackingEvaluator.Expand / Pack on a single ring degree (the evaluator's MinLogN == MaxLogN == ctx LogN; with MinLogN < MaxLogN
 * the caller keeps Split / Merge and calls these at MinLogN). At every step of either tree all key switches use one Galois element:
 * they go through one gadget product per step per batch_chunk() ciphertexts (key read once per sub-batch). Keys are whatever
 * lgpu_gadget_product accepts (multiple P, single P, BaseTwoDecomposition, levelP < MaxLevelP); only the steps that key-switch look
 * theirs up, all of them before any device work (the reference fails at the first missing key after part of the work). The argument
 * checks also run on a host-only ctx. Results equal the reference bit for bit.
 * Errors common to both: a ConjugateInvariant ctx (the reference's messages), a missing key ("GaloisKey[g] is missing") or one that
 * lgpu_gadget_product rejects, overlapping input and output, misalignment. */
/* RingPackingEvaluator.Expand (:457-571). ct_in: [batch][2][level+1][N], is_ntt its domain. ct_out: [batch][N >> log_gap][2][level+1][N];
 * element k of a batch entry is the reference's cts[k << log_gap]. Outputs are ALWAYS in the NTT domain: for a coefficient-domain
 * input the reference marks cts[0] as NTT after transforming it, so its trailing INTT loop (:563-569) never fires. 0 <= log_gap <=
 * LogN ("Expand: logGap out of range [0, LogN]"; the reference does not check it). Keys: N / 2^i + 1 for 0 <= i < LogN
 * (GaloisElementsForExpand(LogN)). Scratch: max(1, S / 2) * batch ciphertexts (S = N >> log_gap) + min(batch_chunk(), S / 2 * batch)
 * key-switch outputs + the gadget product's own; ct_out itself also serves as a scratch block before the last step writes it. */
int lgpu_ring_packing_expand(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int is_ntt, int log_gap,
                             const lgpu_galois_keys* gks, uint64_t* ct_out, int batch, void* stream);
/* RingPackingEvaluator.Pack (:600-770). cts_in: [batch][n_cts][2][level+1][N], all at one level, is_ntt their domain; idx: HOST array
 * of the n_cts map keys, sorted (the reference sorts them; here every consecutive pair is checked, with getMinimumGap's messages
 * "getMinimumGap: invalid index list: element must be sorted from smallest to largest" / "...: contains duplicated elements").
 * Keys >= 2^input_log_gap (or < 0) take part in the gap only, as in the reference. ct_out: [batch][2][level+1][N], NTT domain.
 * cts_in is NOT modified (the reference NTTs and rescales its inputs in place). 0 <= input_log_gap <= LogN
 * ("Pack: inputLogGap out of range [0, LogN]"; unchecked in the reference). Errors: n_cts <= 0 ("len(cts) = 0"), logStart >= logEnd
 * ("gaps between ciphertexts is smaller than inputLogGap > N"), and no input reaching slot 0 ("Pack: no input ciphertext reaches
 * slot 0 ..."): the reference returns a nil ciphertext with a nil error there. Keys: NthRoot - 1 at tree level 0 (reached only with
 * input_log_gap = LogN) and GaloisElement(2^(i-1)) at level i >= 1 (GaloisElementsForPack). Scratch: (pairs of the first step) *
 * batch ciphertexts + 2 * min(batch_chunk(), that) for the key-switch input and output of one sub-batch (+ batch ciphertexts
 * per index in [0, 2^input_log_gap) for a coefficient-domain input: the NTT of the inputs the tree reads) + the gadget product's own. */
int lgpu_ring_packing_pack(lgpu_ctx* ctx, int level, const uint64_t* cts_in, int is_ntt, const int* idx, int n_cts,
                           int input_log_gap, int zero_garbage_slots, const lgpu_galois_keys* gks, uint64_t* ct_out,
                           int batch, void* stream);

/* ---- generic key switch with ring-degree switching (core/rlwe/evaluator_evaluationkey.go, core/rlwe/element.go) --------------
 * Evaluator.ApplyEvaluationKey (:36-107) for a batch of degree-1 ciphertexts sharing one evaluation key. ctx is the evaluator,
 * i.e. the LARGE ring degree N. ct_in: [batch][2][level_in+1][2^log_n_in], ct_out: [batch][2][level_out+1][2^log_n_out], both in
 * the domain is_ntt gives. Rows 0..min(level_in, level_out) of each component of ct_out are written; the block keeps its layout.
 *   n_in == n_out == N   ct_out = (c0 + ks0, ks1), ks = GadgetProduct(c1); ct_out == ct_in is allowed (with level_out == level_in)
 *   n_in <  n_out == N   SwitchCiphertextRingDegree[NTT] to X^(N/n_in) into ct_out, then the key switch in place. In the coefficient
 *                        domain only every gap-th coefficient of ct_out is written by the map, as in the reference
 *   n_in == N >  n_out   key switch at N, then SwitchCiphertextRingDegree[NTT] down to n_out (the NTT case as one block-average
 *                        pass, DESIGN 3.4)
 * Any other overlap of ct_in and ct_out is rejected. One gadget product runs per batch_chunk() ciphertexts (the key is read once per
 * sub-batch). The evaluation key is whatever lgpu_gadget_product accepts at level min(level_in, level_out).
 * Errors, all checked before any device work (also on a host-only ctx): "cannot ApplyEvaluationKey: opOut ring degree does not match
 * evaluator params ring degree" and the ctIn variant (the reference's messages), equal degrees other than N, a degree below 2^4,
 * a degree switch on a ConjugateInvariant ctx (the reference supports it; here only the same-degree case runs on that ring), a
 * key level below min(level_in, level_out) (the reference adds rows the gadget product did not write there), and any key
 * lgpu_gadget_product rejects. Where the reference panics because ct_out has more rows than ct_in (both directions in the
 * coefficient domain, downward in the NTT domain), the rows above min(level_in, level_out) are left as they were. */
int lgpu_evaluator_apply_evaluation_key(lgpu_ctx* ctx, const uint64_t* ct_in, int log_n_in, int level_in, int is_ntt,
                                        const lgpu_gadget_ct* evk, uint64_t* ct_out, int log_n_out, int level_out,
                                        int batch, void* stream);

/* ---- RGSW (core/rgsw) --------------------------------------------------------------------------------------------------
 * rgsw.Evaluator.ExternalProduct (core/rgsw/evaluator.go:39-88): RLWE x RGSW -> RLWE at the RGSW ciphertext's levels.
 * rgsw0 / rgsw1 = rgsw.Ciphertext.Value[0] / Value[1] (core/rgsw/elements.go:11-13). ct_in: [batch][2][level_in+1][N], NTT domain;
 * ct_out: [batch][2][level_out+1][N], rows 0..rgsw level written; ct_out == ct_in allowed (how the reference's callers use it).
 * All three reference paths (multiple P :210-283, single P / bit decomposition :130-208, 32-bit :90-128) are covered. */
int lgpu_rgsw_external_product(lgpu_ctx* ctx, const uint64_t* ct_in, int level_in, const lgpu_gadget_ct* rgsw0,
                               const lgpu_gadget_ct* rgsw1, uint64_t* ct_out, int level_out, int batch, void* stream);

/* ---- encryptor / key-generator inner loops and device samplers (core/rlwe/encryptor.go, keygenerator.go, ring/sampler_*.go) ----
 * Samplers: the reference's distributions on Philox4x32-10 counter streams keyed by (seed, stream_id) -- NOT the reference's
 * blake2b-XOF byte stream (sampling/prng.go), which is inherently sequential. Small polynomials are int64 vectors [batch][N].
 * Every block is philox4x32_10(counter, key) with key = (seed mod 2^32, (seed >> 32) ^ (stream_id >> 32) * 0x85EBCA6B mod 2^32)
 * and counter = (c, poly | kind << 30, stream_id mod 2^32, attempt), kind = 0 uniform, 1 ternary {P}, 2 ternary {H}, 3 Gaussian:
 *   uniform      c = coefficient, poly = batch index * 128 + global limb index (P limbs are nQ + j), one block per attempt;
 *   ternary {P}  c = coefficient, poly = batch index, attempt = 0;
 *   ternary {H}  c = attempt, poly = batch index, last word 0;
 *   Gaussian     c = coefficient, poly = batch index, one block per attempt.
 * Draws of different kinds therefore never share a block, and neither do the Q and P rows of one ringqp.Poly. Two calls of the
 * same kind on the same (seed, stream_id) do: give every call its own stream_id (lattigo_b200.encryptor.Samplers does). This
 * layout replaced one without the kind field, so output for a given (seed, stream_id) differs from builds before it. */
/* ringqp.UniformSampler.Read (ring/sampler_uniform.go:48-100): rows 0..level uniform in [0, q_i). */
int lgpu_sample_uniform(lgpu_ctx* ctx, int ring, int level, uint64_t seed, uint64_t stream_id, uint64_t* out, int batch,
                        size_t batch_stride, void* stream);
/* ring.TernarySampler (ring/sampler_ternary.go): hamming_weight > 0 selects ring.Ternary{H} (exactly min(H, N) non-zero
 * coefficients), otherwise ring.Ternary{P = p} (P(+1) = P(-1) = ceil(p 2^53) / 2^54), p in (0, 1]. */
int lgpu_sample_ternary(lgpu_ctx* ctx, double p, int hamming_weight, uint64_t seed, uint64_t stream_id, int64_t* out, int batch,
                        void* stream);
/* ring.GaussianSampler (ring/sampler_gaussian.go:160-182): round(|N(0,1)| sigma) with a random sign, |.| <= bound. */
int lgpu_sample_gaussian(lgpu_ctx* ctx, double sigma, double bound, uint64_t seed, uint64_t stream_id, int64_t* out, int batch,
                         void* stream);
/* What Sampler.Read + ringqp.Ring.ExtendBasisSmallNormAndCenter (ring/ringqp/operations.go:325-351) leave in a ringqp.Poly:
 * the signed value modulo every q_i (out_q, level_q+1 rows) and p_j (out_p, level_p+1 rows); either output may be NULL.
 * Precondition: |v| < q_0 / 2, where the reference's centring is exact (and |v| below every modulus written). */
int lgpu_small_poly_to_rns(lgpu_ctx* ctx, int level_q, int level_p, const int64_t* small, uint64_t* out_q, uint64_t* out_p,
                           int batch, size_t stride_q, size_t stride_p, void* stream);
/* Encryptor.encryptZeroPk for a plain rlwe.Ciphertext (core/rlwe/encryptor.go:204-299: one special prime, ModDownQPtoQ) or, when
 * the context has no P, encryptZeroPkNoP (:301-341). pk: rlwe.PublicKey.Value = [2][nQ + nP][N] at the maximum levels (NTT +
 * Montgomery); u (xs sample), e0, e1 (xe samples): [batch][N]; ct_out: [batch][2][level_q+1][N]. */
int lgpu_encrypt_zero_pk(lgpu_ctx* ctx, int level_q, const uint64_t* pk, const int64_t* u, const int64_t* e0, const int64_t* e1,
                         uint64_t* ct_out, int is_ntt, int is_montgomery, int batch, void* stream);
/* Encryptor.encryptZeroSkFromC1QP (:404-430; level_p = -1 for a plain ciphertext): c0 = e - c1 * sk. sk: [nQ + nP][N]; c1, c0:
 * [batch][level_q+1 + level_p+1][N] (Q rows then P rows); c1 is the uniform polynomial in the NTT domain (rewritten by INTT only
 * when !is_ntt, like the reference). */
int lgpu_encrypt_zero_sk(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* sk, uint64_t* c1, const int64_t* e, uint64_t* c0,
                         int is_ntt, int is_montgomery, int batch, void* stream);
/* KeyGenerator.genEvaluationKey (core/rlwe/keygenerator.go:287-330) + AddPolyTimesGadgetVectorToGadgetCiphertext
 * (core/rlwe/gadgetciphertext.go:171-241) at the maximum levels. On entry component 1 of every evk->data[i][j] holds the uniform
 * polynomial (e.g. from lgpu_sample_uniform; evk->data is written although the struct declares it const); e: [n_digits][n_pw2_max][N]
 * error samples; sk_in: [nQ][N], sk_out: [nQ + nP][N], NTT + Montgomery. */
int lgpu_gen_evaluation_key(lgpu_ctx* ctx, const uint64_t* sk_in, const uint64_t* sk_out, lgpu_gadget_ct* evk, const int64_t* e,
                            void* stream);

/* ---- batched RGSW encryption and key generation at any levels (keygen.cu) -------------------------------------------------------
 * Keys are lgpu_gadget_ct at any level_q <= max and level_p in [-1, max_p], with any BaseTwoDecomposition in [0, 62], laid out as
 * rgsw.NewCiphertext / NewGadgetCiphertext lay them out: n_digits = BaseRNSDecompositionVectorSize(level_q, level_p), pw2_sizes =
 * BaseTwoDecompositionVectorSize(level_q, level_p, base) (NULL when all are 1), n_pw2_max their maximum. Every key of one call has the
 * same layout; no key's data may overlap another key or an input. The gadget factor of entry (i, j) is P_level_p 2^(base j) with
 * P_level_p = p_0 ... p_level_p (1 when level_p = -1). sk: [nQ + nP][N] at the maximum levels, NTT + Montgomery. Secret-key
 * encryption only, Standard ring only. Every argument check runs before any launch, also on a host-only ctx; batch and n_keys are in
 * [1, 65535]. */
/* rgsw.Encryptor.Encrypt (core/rgsw/encryptor.go:25-70) of batch plaintexts, or EncryptZero (:74-121) when pts == NULL. value0 /
 * value1: HOST arrays of batch keys, Value[0] and Value[1] of each RGSW ciphertext; on entry component 1 of every entry holds its
 * uniform polynomial (NTT domain). e: [batch][2][n_digits][n_pw2_max][N] error samples, [b][v] for Value[v] of ciphertext b.
 * pts: [n_pt][level_q+1][N] distinct plaintexts, ciphertext b encrypting pts[pt_index[b]] (pt_index: HOST array); is_ntt /
 * is_montgomery describe all of them and are handled as encryptor.go:47-60 does (NTT, then MForm, as needed). */
int lgpu_rgsw_encrypt(lgpu_ctx* ctx, const uint64_t* sk, const uint64_t* pts, int n_pt, const int* pt_index, int is_ntt, int is_montgomery,
                      const int64_t* e, const lgpu_gadget_ct* value0, const lgpu_gadget_ct* value1, int batch, void* stream);
/* KeyGenerator.GenGaloisKeysNew(gal_els, sk, evkParams) (core/rlwe/keygenerator.go:123-209): key k encrypts sk under
 * AutomorphismNTT(sk, gal_els[k]^-1 mod 2N). gal_els: HOST, odd and below 2N. keys: HOST array of n_keys keys, component 1 of every
 * entry holding its uniform polynomial on entry; e: [n_keys][n_digits][n_pw2_max][N]. */
int lgpu_gen_galois_keys(lgpu_ctx* ctx, const uint64_t* sk, const uint64_t* gal_els, int n_keys, const int64_t* e, const lgpu_gadget_ct* keys,
                         void* stream);
/* blindrot.GenEvaluationKeyNew (core/rgsw/blindrot/keys.go:52-108): brk0[i] / brk1[i] = Value[0] / Value[1] of RGSW(X^{s_lwe[i]}) and
 * gks[t] the Galois key of GaloisElement(t + 1) for t < window_size, gks[window_size] that of NthRoot - GaloisGen. s_lwe: HOST array of
 * the n_lwe (<= 32767) centred LWE-key coefficients (what the Go computes with INTT, IMForm and PolyToBigintCentered at level 0).
 * All keys share one layout; their data is written whole. The samples are drawn here, from (seed, stream id m) for the m-th gadget
 * ciphertext, m = 2 i + v for Value[v] of RGSW i and m = 2 n_lwe + t for gks[t]: component 1 of entry (d, j) is batch element
 * d n_pw2_max + j of lgpu_sample_uniform(RING_Q, level_q) followed by lgpu_sample_uniform(RING_P, level_p) on that stream id, and its
 * error is batch element d n_pw2_max + j of lgpu_sample_gaussian(sigma, bound) on it. */
int lgpu_blind_rotation_gen_evaluation_key(lgpu_ctx* ctx, const uint64_t* sk, const int64_t* s_lwe, int n_lwe, int window_size, double sigma,
                                           double bound, uint64_t seed, const lgpu_gadget_ct* brk0, const lgpu_gadget_ct* brk1,
                                           const lgpu_gadget_ct* gks, void* stream);

/* ---- threshold protocols (multiparty/), Standard ring, NTT domain ------------------------------------------------------------
 * Sampled polynomials are inputs, as for the encryptor above; every protocol's common reference polynomial comes from the same
 * samplers keyed by a seed all parties share. PublicKeyGenProtocol.GenShare (multiparty/keygen_cpk.go:70-83) is
 * lgpu_encrypt_zero_sk at the maximum levels with c1 = crp, is_ntt = is_montgomery = 1. Results keep the reference's
 * representatives, which need not be canonical (see lgpu_mp_aggregate). Every argument check runs before any launch, also on a
 * host-only ctx; batch and n_shares are in [1, 65535].
 *
 * AggregateShares of any protocol (e.g. keyswitch_sk.go:123-130): out = the left fold agg = shares[0]; agg = Add(agg, shares[k]) in
 * share order, Add = CRed(a + b) on the wrapping 64-bit sum, exactly as the reference's pairwise calls chain; no final reduction, so
 * K shares in [0, 2q) give a result in [0, (K + 1) q). shares: HOST array of n_shares device pointers; each share and out are n_polys
 * blocks of (level_q + 1) Q rows then (level_p + 1) P rows of N words (level_p = -1: Q only). out == shares[0] is allowed, any other
 * overlap of out and a share is not. One read of every share and one write of out per chunk of 32 pointers. */
int lgpu_mp_aggregate(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* const* shares, int n_shares, uint64_t* out, size_t n_polys,
                      void* stream);
/* KeySwitchProtocol.GenShare (multiparty/keyswitch_sk.go:85-118), ct.IsNTT: share = MRedLazy(c1, s_in - s_out) + NTT(e), in [0, 2q).
 * c1: ct.Value[1] of `batch` ciphertexts, level + 1 rows each, batch stride `stride` words; sk_in, sk_out: [nQ (+ nP)][N] NTT +
 * Montgomery (rows 0..level are read); e: [batch][N] smudging samples (sigma' = sqrt(NoiseFreshSK^2 + sigma_flood^2), bound 6 sigma',
 * :45-52); share: [batch][level + 1][N]. */
int lgpu_mp_key_switch_share(lgpu_ctx* ctx, int level, const uint64_t* c1, size_t stride, const uint64_t* sk_in, const uint64_t* sk_out,
                             const int64_t* e, uint64_t* share, int batch, void* stream);
/* PublicKeySwitchProtocol.GenShare (multiparty/keyswitch_pk.go:69-105), ct.IsNTT: share = EncryptZero(pk) with (u, e0, e1) as in
 * lgpu_encrypt_zero_pk (NTT, not Montgomery), then share[0] = CRed(share[0] + MRed(c1, sk)) + NTT(e_flood). c1 as above; sk: [nQ (+ nP)][N];
 * pk: [2][nQ + nP][N]; u, e0, e1, e_flood: [batch][N]; share: [batch][2][level + 1][N]. */
int lgpu_mp_public_key_switch_share(lgpu_ctx* ctx, int level, const uint64_t* c1, size_t stride, const uint64_t* sk, const uint64_t* pk,
                                    const int64_t* u, const int64_t* e0, const int64_t* e1, const int64_t* e_flood, uint64_t* share, int batch,
                                    void* stream);
/* Key-generation shares, at the context's maximum levels, for any BaseTwoDecomposition, with or without P. `share` (and `round1`) describe
 * a gadget layout as for lgpu_gadget_ct (levels, base_two_decomposition, n_digits, n_pw2_max, pw2_sizes); their data is written although
 * the struct declares it const. A share entry (i, j) is a QP block of nQ + nP rows; a CRP is [n_digits][n_pw2_max][nQ + nP][N] uniform
 * rows (NTT domain); error samples are [n_digits][n_pw2_max][N]. Entries with j >= pw2_sizes[i] hold unspecified values. Secret keys are
 * [nQ + nP][N], NTT + Montgomery.
 *
 * EvaluationKeyGenProtocol.GenShare (multiparty/keygen_evk.go:86-183): share data [n_digits][n_pw2_max][nQ + nP][N] (one component, like
 * NewGadgetCiphertext(params, 0, ...)), entry (i, j) = -crp_ij sk_out + e_ij + P 2^(w j) sk_in on the limbs of digit i, NTT + Montgomery.
 * With gal_els != NULL it is GaloisKeyGenProtocol.GenShare (keygen_gal.go:48-70) for n_keys Galois elements (odd, below 2N) in one call:
 * key k uses sk_out = AutomorphismNTT(sk_in, gal_els[k]^-1 mod 2N) on Q and P (sk_out is not read), and crp, e and share data carry a
 * leading key index. gal_els == NULL requires n_keys = 1. */
int lgpu_mp_evaluation_key_gen_share(lgpu_ctx* ctx, const uint64_t* sk_in, const uint64_t* sk_out, const uint64_t* gal_els, int n_keys,
                                     const uint64_t* crp, const int64_t* e, const lgpu_gadget_ct* share, void* stream);
/* RelinearizationKeyGenProtocol.GenShareRoundOne (multiparty/keygen_relin.go:91-184), plain (not Montgomery) form: share data
 * [n_digits][n_pw2_max][2][nQ + nP][N], entry (i, j) = (e0_ij + P 2^(w j) s - u crp_ij on the limbs of digit i, NTT(e1_ij) + s crp_ij);
 * eph_sk_out: the ephemeral secret u (u_small: [N] ternary) as [nQ + nP][N] NTT + Montgomery rows. */
int lgpu_mp_rkg_share_round_one(lgpu_ctx* ctx, const uint64_t* sk, const int64_t* u_small, const uint64_t* crp, const int64_t* e0,
                                const int64_t* e1, uint64_t* eph_sk_out, const lgpu_gadget_ct* share, void* stream);
/* RelinearizationKeyGenProtocol.GenShareRoundTwo (:193-234): round1 is the aggregated round-one share (two components), share data
 * [n_digits][n_pw2_max][nQ + nP][N] (one component), entry (i, j) = CRed(CRed(MRedLazy(r0_ij, s) + NTT(e2_ij)) + MRed(u - s, r1_ij)), in
 * [0, 2q). GenRelinearizationKey (:261-276) is MForm of the aggregated round-two share and of round-one component 1. */
int lgpu_mp_rkg_share_round_two(lgpu_ctx* ctx, const uint64_t* eph_sk, const uint64_t* sk, const lgpu_gadget_ct* round1, const int64_t* e2,
                                const lgpu_gadget_ct* share, void* stream);
/* Thresholdizer.GenShamirSecretShare (multiparty/threshold.go:102-104) for n_points recipients in one pass: share k is
 * ringqp.Ring.EvalPolyScalar(poly, points[k]) (ring/ringqp/operations.go:92-102) on the Q rows and on the P rows, by Horner's rule
 * acc = poly[t-1]; acc = CRed(MRed(acc, MForm(points[k])) + poly[i-1]) for i = t-1 .. 1, with the wrapping 64-bit sum and MForm the
 * Barrett form of the unreduced point, so any 64-bit input word gives the reference's word. poly: [threshold][(level_q + 1) Q rows then
 * (level_p + 1) P rows][N], coefficient 0 the secret (ShamirPolynomial.Value); points: HOST array of n_points 64-bit points;
 * shares: [n_points][rows][N], which must not overlap poly. level_p = -1: Q only; threshold and n_points are in [1, 65535]. Reads every
 * coefficient once per chunk of 8 points: ceil(n_points / 8) threshold + n_points polynomial sizes of traffic. */
int lgpu_mp_shamir_share(lgpu_ctx* ctx, int level_q, int level_p, const uint64_t* poly, int threshold, const uint64_t* points, int n_points,
                         uint64_t* shares, void* stream);
/* blindrot.Evaluator.BlindRotateCore (core/rgsw/blindrot/evaluator.go:144-229; Algorithm 3 of eprint 2022/198) on one accumulator, in place.
 * a_host: the LWE mask modulo 2N (HOST, n_lwe odd-or-zero words); acc: [2][level+1][N] NTT-domain RLWE accumulator; brk0[j] / brk1[j]:
 * Value[0] / Value[1] of RGSW(X^{s_j}) (HOST arrays of n_lwe key descriptors); gks: the automorphism keys of the window
 * (GaloisElement(1..window_size) and NthRoot - GaloisGen; a missing one is an error). window_size = 10 in the reference (keys.go:14). */
int lgpu_blind_rotate_core(lgpu_ctx* ctx, const uint64_t* a_host, int n_lwe, uint64_t* acc, int level, const lgpu_gadget_ct* brk0,
                           const lgpu_gadget_ct* brk1, const lgpu_galois_keys* gks, int window_size, void* stream);
/* blindrot.Evaluator.Evaluate (core/rgsw/blindrot/evaluator.go:49-132) for a batch of LWE-ring ciphertexts: every listed slot of every
 * ciphertext is blind-rotated in one call. ctx: the blind-rotation ring (N, Q); ctx_lwe: the LWE ring (N_LWE <= N, q_LWE; may be ctx).
 * ct_lwe: [batch][2][level_lwe+1][N_LWE] in the domain is_ntt gives (the INTT runs in ctx_lwe); only level_lwe = 0 is supported (the
 * reference switches higher levels to 2N with big integers). slots: HOST list of n_slots distinct indices in [0, N_LWE); test_polys[k]:
 * the device rows (level+1 of them, stride N) of slot slots[k]'s test polynomial, NTT domain; slots may share a pointer. brk0[j] / brk1[j]
 * (j < N_LWE <= n_brk): RGSW(X^{s_j}), all at the same levels and base; level = brk0[0].level_q. gks: the keys of GaloisElement(1..window_size)
 * (except GaloisElement(v) = 1, which is a copy) and NthRoot - GaloisGen, all required before any device work. ct_out:
 * [batch][n_slots][2][level+1][N], NTT domain, or coefficient domain when ntt_out = 0 (the reference's !NTTFlag branch).
 * With level = 0, keys without P, BaseTwoDecomposition >= 1 and 2^8 <= N <= 2^12, every accumulator runs its whole Algorithm 3 in
 * one CTA (csrc/blindrot.cu: at most three launches per call whatever batch, n_slots and N_LWE); otherwise each slot goes through
 * lgpu_blind_rotate_core. Bit-identical to the reference in both cases. */
int lgpu_blind_rotation_evaluate(lgpu_ctx* ctx, lgpu_ctx* ctx_lwe, const uint64_t* ct_lwe, int level_lwe, int is_ntt, const int* slots,
                                 int n_slots, const uint64_t* const* test_polys, const lgpu_gadget_ct* brk0, const lgpu_gadget_ct* brk1,
                                 int n_brk, const lgpu_galois_keys* gks, int window_size, int ntt_out, uint64_t* ct_out, int batch,
                                 void* stream);
/* ckks.SpecialFFTDouble / SpecialIFFTDouble (schemes/ckks/ckks_vector_ops.go:18-77; Encoder.FFT / IFFT, schemes/ckks/encoder.go:764-816), in
 * place on `batch` vectors of n complex128 values (device, interleaved re / im, batch_stride in complex values). rot_group (n int64 values)
 * and roots (m + 1 complex128 values) are the encoder's own tables (encoder.go:83-112), device resident. Same operations in the same order
 * as the Go code and no fused multiply-add: results are bit-identical on identical tables. */
int lgpu_ckks_special_fft(lgpu_ctx* ctx, double* values, int n, int m, const int64_t* rot_group, const double* roots, int inverse,
                          int batch, size_t batch_stride, void* stream);
/* ckks.Encoder on the prec <= 53 path, ring.Standard only (csrc/encoder.cu), bit-identical to the reference on identical rot_group / roots.
 * flags: LGPU_ENC_NTT = MetaData.IsNTT, LGPU_ENC_MONTGOMERY = MetaData.IsMontgomery (encode; ignored by the non-batched Encode and by
 * Decode, as in the reference), LGPU_ENC_COEFFS = IsBatched false. scale = MetaData.Scale.Float64(), finite and > 0. Strides are in
 * elements (complex128 values, float64 values, or uint64 words); batch <= 65535. Every check runs before any launch, also on a
 * host-only context; inputs are never written; scratch is stream-ordered (cudaMallocAsync on `stream`).
 *
 * Encode: Encoder.Embed / Encode with IsBatched (schemes/ckks/encoder.go:208-337): `values` holds n_values <= 2^log_slots complex128
 * values per entry (16-byte aligned), zero-padded to the slots, 0 <= log_slots <= LogN - 1; IFFT, Complex128ToFixedPointCRT and
 * rlwe.NTTSparseAndMontgomery into out_q (level_q + 1 rows) and, when level_p >= 0, out_p (level_p + 1 rows; the ringqp.Poly of a
 * linear-transformation diagonal). Without LGPU_ENC_NTT the words are the reference's literal ones (possibly q, or an unreduced
 * c < 2^61); the coefficient-domain case with slots < N/2 is rejected (the reference's spreading loop, core/rlwe/utils.go:234-241,
 * has no defined output). With LGPU_ENC_COEFFS (encoder.go:156-189): n_values <= N float64 values, Float64ToFixedPointCRT, NTT when
 * LGPU_ENC_NTT, level_p = -1; log_slots, rot_group and roots are unused. Values must be finite.
 *
 * Decode: Encoder.DecodePublic (encoder.go:497-762) of `batch` plaintexts pt [level + 1][N]: INTT when LGPU_ENC_NTT (NTT-domain words
 * canonical), then polyToComplexNoCRT (level 0) / polyToComplexCRT, the forward special FFT and, for logprec != 0 (an integer in
 * [-1022, 1023]), math.Round(x 2^logprec) / 2^logprec per part; `values` receives 2^log_slots complex128 per entry (16-byte aligned).
 * With LGPU_ENC_COEFFS: polyToFloatNoCRT / polyToFloatCRT into N float64 per entry, no FFT, logprec unused. At level >= 1 the bit
 * lengths of q_0..q_level must sum to at most 4096 (the CRT accumulator has 16, 32 or 64 words of 64 bits, chosen from that sum);
 * past it the call is refused before any launch, even where Q_level itself has fewer than 4096 bits. */
#define LGPU_ENC_NTT 1
#define LGPU_ENC_MONTGOMERY 2
#define LGPU_ENC_COEFFS 4
int lgpu_ckks_encode(lgpu_ctx* ctx, const double* values, int n_values, int log_slots, double scale, int flags, const int64_t* rot_group,
                     const double* roots, int level_q, uint64_t* out_q, int level_p, uint64_t* out_p, int batch, size_t values_stride,
                     size_t out_q_stride, size_t out_p_stride, void* stream);
int lgpu_ckks_decode(lgpu_ctx* ctx, const uint64_t* pt, int level, int log_slots, double scale, int flags, double logprec,
                     const int64_t* rot_group, const double* roots, double* values, int batch, size_t pt_stride, size_t values_stride,
                     void* stream);

/* ---- wire format -> device (the reference's WriteTo / ReadFrom byte streams, little-endian uint64 words) ------------------
 * ring.Poly (ring/poly.go:132-179): rows, then per row {len, len words}. */
int lgpu_poly_load(lgpu_ctx* ctx, const void* bytes, size_t nbytes, uint64_t* dst, int rows_cap, int* rows_out, size_t* consumed,
                   void* stream);
/* ring.Poly.WriteTo of `rows` device rows into `bytes` (8 + rows * (8 + 8 N) bytes); synchronises `stream`. */
int lgpu_poly_store(lgpu_ctx* ctx, const uint64_t* src, int rows, void* bytes, size_t cap, size_t* written, void* stream);
#define LGPU_MAX_DIGITS 128
typedef struct {
    int level_q, level_p, base_two_decomposition, n_digits, n_pw2_max;
    int pw2_sizes[LGPU_MAX_DIGITS];   /* len(Value[i]); usable as lgpu_gadget_ct.pw2_sizes */
    size_t device_bytes;              /* size of the device block in the lgpu_gadget_ct layout */
    size_t consumed;                  /* bytes of the stream that belong to this object */
} lgpu_evk_info;
/* rlwe.GadgetCiphertext.ReadFrom / UnmarshalBinary (core/rlwe/gadgetciphertext.go:101-167; also EvaluationKey and
 * RelinearizationKey, which are GadgetCiphertexts): BaseTwoDecomposition, then structs.Matrix[VectorQP]
 * (utils/structs/matrix.go:80-140). With dst == NULL only *info is filled (no device work); with a 16-byte aligned device
 * block of info->device_bytes bytes the rows are copied straight from the byte stream into the lgpu_gadget_ct layout. */
int lgpu_gadget_ct_load(lgpu_ctx* ctx, const void* bytes, size_t nbytes, uint64_t* dst, size_t dst_bytes, lgpu_evk_info* info,
                        void* stream);
/* rlwe.GaloisKey.ReadFrom (core/rlwe/keys.go:628-700): GaloisElement, NthRoot, EvaluationKey. */
int lgpu_galois_key_load(lgpu_ctx* ctx, const void* bytes, size_t nbytes, uint64_t* gal_el, uint64_t* nth_root, uint64_t* dst,
                         size_t dst_bytes, lgpu_evk_info* info, void* stream);

/* ---- fused batch entry points for the measured op sequences ---------------------------------------------------
 * ckks.Evaluator.MulRelinNew(ct_a, ct_b) followed by Rescale (schemes/ckks/evaluator.go:719-872, :477-515;
 * nb_rescales = Parameters.LevelsConsumedPerRescaling(), 0 = no rescale). ct_a, ct_b: [batch][2][level+1][N]
 * (NTT domain); ct_out: [batch][2][level+1-nb_rescales][N]. _host: pinned or pageable HOST buffers, copies
 * included and pipelined in chunks of `chunk` ciphertext pairs (0 = default). */
int lgpu_ckks_mulrelin_rescale_batch(lgpu_ctx* ctx, int level, const uint64_t* ct_a, const uint64_t* ct_b,
                                     const lgpu_gadget_ct* rlk, int nb_rescales, uint64_t* ct_out, int batch, void* stream);
int lgpu_ckks_mulrelin_rescale_batch_host(lgpu_ctx* ctx, int level, const uint64_t* ct_a_host, const uint64_t* ct_b_host,
                                          const lgpu_gadget_ct* rlk, int nb_rescales, uint64_t* ct_out_host, int batch, int chunk);

/* ---- CKKS polynomial evaluation (circuits/ckks/polynomial.Evaluator.Evaluate) ---------------------------------------
 * A program planned on the host (lattigo_b200/polyeval.py restates the reference's power basis, Paterson-Stockmeyer split and
 * scale bookkeeping) and run on a batch. Slots are single-assignment ciphertexts: slot 0 is the input (degree 1, `level`), every
 * op writes one new slot (LINCOMB: n_out new slots) from slots written before it. The ops, one per rounding boundary:
 *   MULRELIN dst = MulRelinNew(src0, src1)                 degree 1 x 1 -> 1, level = min(levels)
 *   TENSOR   dst = r_b (src0 (x) src1) + r_a addend         degree 2; addend of degree 1 or 2 (-1: none, r_a unused);
 *                                                           weights [2][level+1] = r_b, r_a per limb
 *   RELIN    dst = Relinearize(src0)                        degree 2 -> 1
 *   RESCALE  dst = Rescale(src0)                            levels_per_rescale x DivRoundByLastModulusNTT, degree kept
 *   LINCOMB  outs[i] = sum_k W[i][k] terms[k] + W[i][n_terms] on component 0, rows 0..out_levels[i], per limb and NTT half
 *            (slots < N/2 use half 0); weights [n_out][n_terms+1][level+1][2], level = max(out_levels); terms are degree 1,
 *            and an output's weights of a term are 0 on rows above the term's level; n_terms <= LGPU_POLY_MAX_TERMS, n_out <= LGPU_POLY_MAX_OUTPUTS.
 * `level` of every op is the level of what it writes; every weight is a canonical residue (< q_i). */
#define LGPU_POLY_MULRELIN 0
#define LGPU_POLY_TENSOR 1
#define LGPU_POLY_RELIN 2
#define LGPU_POLY_RESCALE 3
#define LGPU_POLY_LINCOMB 4
#define LGPU_POLY_MAX_TERMS 16
#define LGPU_POLY_MAX_OUTPUTS 64
typedef struct {
    int kind;
    int dst, src0, src1, addend;
    int level;
    int n_out, n_terms;
    const int* outs;
    const int* out_levels;
    const int* terms;
    const uint64_t* weights;   /* HOST */
} lgpu_poly_op;
typedef struct {
    int n_slots;
    int n_ops;
    const lgpu_poly_op* ops;   /* HOST */
    int out_slot;              /* degree 1, written by the last op */
    int levels_per_rescale;
} lgpu_poly_program;
/* Runs `prog` on ct_in [batch][2][level+1][N] (NTT domain) into ct_out [batch][2][level_out+1][N], level_out the level of
 * prog->out_slot. Equal bit for bit to the reference's op sequence when prog is what the planner emits for it. The whole program
 * is checked before any launch, also on a host-only context: slot indices and single assignment, degrees and level arithmetic,
 * term / output counts, every weight below its modulus, the relinearization key at every level it is used. Scratch: the slots are
 * allocated when written and freed after their last read, per sub-batch of batch_chunk() ciphertexts; per ciphertext the peak is
 * at most sum over slots of (degree+1)(level+1) N words plus the key-switch scratch of one MulRelinNew at `level`. */
int lgpu_ckks_polynomial_evaluate(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                  const lgpu_gadget_ct* rlk, uint64_t* ct_out, void* stream);

/* ---- BGV / BFV ciphertext multiplication (schemes/bgv) ---------------------------------------------------------
 * State of bgv.NewParameters' ringQMul + newEvaluatorPrecomp (schemes/bgv/params.go:98-109, evaluator.go:38-70) for the
 * context's Q: the plaintext modulus t, tMontgomery, levelQMul[] and the Q <-> QMul basis extender.
 * qmul: the caller's RingQMul moduli (as lgpu_create takes Q and P), in the reference's
 * NextDownstreamPrimes(61, NthRoot) order. Errors: t < 2, t >= q_0, t in Q, a QMul prime in Q,
 * nqmul < levelQMul[MaxLevel] + 1, a ConjugateInvariant ctx. A host-only ctx (device < 0) gives a host-only handle (argument
 * checks, no device execution). Destroy before ctx. */
typedef struct lgpu_bgv lgpu_bgv;
int lgpu_bgv_create(lgpu_ctx* ctx, uint64_t t, const uint64_t* qmul, int nqmul, lgpu_bgv** out);
void lgpu_bgv_destroy(lgpu_bgv* ev);
/* bgv.Evaluator.MulRelin of two degree-1 ciphertexts followed by nb_rescales x Rescale (scale_invariant = 0;
 * evaluator.go:529-556, tensorStandard :592-667, Rescale :1363-1393), or MulRelinScaleInvariant (scale_invariant = 1, BFV;
 * :806-864, tensorScaleInvariant :898-1070; nb_rescales must be 0). ct_a, ct_b: [batch][2][level+1][N], NTT domain;
 * ct_out: [batch][2][level+1-nb_rescales][N]. ct_a == ct_b is the squaring case. ct_out == ct_a is allowed when
 * nb_rescales == 0; no other overlap. rlk: the relinearization key of ctx's (Q, P). The scale-invariant product extends its
 * operands from all level+1 Q moduli to QMul in one basis extension, which takes at most 64 sources: level + 1 <= 64 (BGV has no limit).
 * Scale bookkeeping stays with the caller: the reference sets the output scale to s_a * s_b (BGV), divided by q_level for
 * each Rescale, and to MulScaleInvariant(s_a, s_b, level) = s_a * s_b / (-Q_level mod t) for BFV (:983-989). */
int lgpu_bgv_mulrelin_batch(lgpu_bgv* ev, int level, const uint64_t* ct_a, const uint64_t* ct_b, const lgpu_gadget_ct* rlk,
                            int scale_invariant, int nb_rescales, uint64_t* ct_out, int batch, void* stream);
/* bgv polynomial.Evaluator.Evaluate (circuits/bgv/polynomial/polynomial_evaluator.go:38-51) of one polynomial on a batch: the program
 * format of lgpu_ckks_polynomial_evaluate, planned by lattigo_b200/bgv_polyeval.py (power basis, Paterson-Stockmeyer split, the BGV
 * simEvaluator, and the schemes/bgv Add / MulThenAdd / Mul scale rules mod t folded into the weights). The ops, for the BGV evaluator
 * (scale_invariant = 0, tensorStandard) or the BFV one (scale_invariant = 1, tensorScaleInvariant: the evaluator's ScaleInvariant):
 *   MULRELIN dst = MulRelinNew(src0, src1)                 tensorStandard or tensorScaleInvariant, then relinearization
 *   TENSOR   dst = r_b Mul(src0, src1) + r_a addend        Mul without relinearization (same tensor), then Add: r_b = r_a = 1, or
 *                                                           matchScalesBinary's (r0, r1) when the scales differ
 *   RELIN    dst = Relinearize(src0)
 *   RESCALE  dst = Rescale(src0)                            DivRoundByLastModulusNTT; levels_per_rescale must be 1
 *   LINCOMB  as for CKKS; the planner gives both NTT halves the same weights
 * ct_in [batch][2][level+1][N] (NTT domain) -> ct_out [batch][2][level_out+1][N]. Checked before any launch, also on a host-only
 * handle: everything lgpu_ckks_polynomial_evaluate checks, a non-null ev, scale_invariant 0 or 1, levels_per_rescale == 1, no RESCALE
 * when scale_invariant, scale-invariant MULRELIN / TENSOR operands at the op's level and at most 64 Q moduli (level + 1 <= 64, as for
 * lgpu_bgv_mulrelin_batch), and rlk at every MULRELIN / RELIN level. The
 * output scale and level are the planner's. Scratch as lgpu_ckks_polynomial_evaluate, plus the QMul buffers of one
 * tensorScaleInvariant for BFV. */
int lgpu_bgv_polynomial_evaluate(lgpu_bgv* ev, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                 const lgpu_gadget_ct* rlk, int scale_invariant, uint64_t* ct_out, void* stream);

/* ---- polynomial-vector evaluation (Evaluate with a polynomial.PolynomialVector and a Mapping, CKKS and BGV / BFV) ----------------
 * The program format above plus one op that only these two entry points accept (the scalar entry points refuse it as an unknown op):
 *   PTLINCOMB outs[i] = sum_k s[i][k] PT[i][k] terms[k] + s[i][n_terms] PT[i][n_terms] on component 0, rows 0..out_levels[i]
 *            PT[i][k] = plaintext index[i][k] of `pts` (NTT domain, canonical words), or nothing when the index is -1 (the term is
 *            skipped: odd / even polynomials); s: [n_out][n_terms+1][level+1] per-limb scalars (< q_r), in which the planner folds
 *            MForm and the reference's scalar multiplications of the baby step (CKKS: the equal-scale q_level products and the ratio
 *            >= 2 Mul of MulThenAdd; BGV: tMontgomery and matchScalesBinary's r0 / r1); level = max(out_levels); terms are degree 1 at
 *            or above every output level that uses them; a used plaintext's level is at least its output's level; n_terms <=
 *            LGPU_POLY_MAX_TERMS, n_out <= LGPU_POLY_MAX_OUTPUTS; the op's `weights` are unused. Outputs are canonical residues, so
 *            the result equals the reference's Add(res, vector) / MulThenAdd(X^k, vector, res) sequence bit for bit.
 * A vector program has exactly one PTLINCOMB (every baby step of the call). The kernel holds each power of a batch entry in
 * registers and stages the plaintext words of a tile of batch entries in shared memory: each power is read once per batch entry and
 * each plaintext word once per tile; a sub-batch of up to 8 ciphertexts is one tile, larger ones are tiles of 8. Checked before any launch, also on a host-only context or handle: everything the
 * scalar entry point checks, the plaintext count (1..2^20), every index (-1..n_pt-1) and plaintext level, the stride, every scalar
 * below its modulus, and no overlap of the plaintext block with ct_in or ct_out. */
#define LGPU_POLY_PTLINCOMB 5
typedef struct {
    const uint64_t* pt;        /* DEVICE, 16-byte aligned: plaintext j at pt + j * pt_stride, rows 0..pt_levels[j] of N words */
    size_t pt_stride;          /* words, even, >= (max pt_levels + 1) N */
    int n_pt;
    const int* pt_levels;      /* HOST [n_pt] */
    const int* index;          /* HOST [n_out][n_terms + 1]: plaintext of term k of output i (k = n_terms: the constant), or -1 */
    const uint64_t* scalars;   /* HOST [n_out][n_terms + 1][level + 1] */
} lgpu_poly_pt_weights;
int lgpu_ckks_polynomial_vector_evaluate(lgpu_ctx* ctx, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                         const lgpu_poly_pt_weights* pts, const lgpu_gadget_ct* rlk, uint64_t* ct_out, void* stream);
int lgpu_bgv_polynomial_vector_evaluate(lgpu_bgv* ev, int level, const uint64_t* ct_in, int batch, const lgpu_poly_program* prog,
                                        const lgpu_poly_pt_weights* pts, const lgpu_gadget_ct* rlk, int scale_invariant, uint64_t* ct_out,
                                        void* stream);


/* ---- BGV / BFV encoder (schemes/bgv/encoder.go; BFV uses the same bgv.Encoder) ---------------------------------------
 * lgpu_bgv_encoder_create: the plaintext ring T of bgv.NewParameters (params.go:76-135) and the tables of NewEncoder (encoder.go:49-133)
 * for ctx's Q and plaintext modulus t. Checks, in the reference's terms: t >= 2, t < Q[0], t not in Q, `order` (the largest power of
 * two with t = 1 mod order) >= 16, t prime with t = 1 mod 2n for n = min(N, order / 2). One deliberate difference: n < 16 (t = 1 mod 16
 * but not mod 32, e.g. t = 17) is rejected, since the engine's transforms start at 16 points. Standard ring only. A host-only ctx gives
 * a host-only handle (argument checks, no device execution). Independent of lgpu_bgv; destroy before ctx.
 *
 * flags: LGPU_ENC_NTT = MetaData.IsNTT, LGPU_ENC_MONTGOMERY = MetaData.IsMontgomery (ignored by the coefficient Encode and by Decode, as in
 * the reference), LGPU_ENC_COEFFS = IsBatched false, LGPU_ENC_SIGNED: the values are int64 rather than uint64, LGPU_ENC_SCALE_UP:
 * multiply by t^-1 mod Q (Encode; without it the call is Embed). scale = MetaData.Scale.Uint64(), any value. `values` are device arrays
 * of 64-bit words; strides are in words; batch <= 65535. Every check runs before any launch, also on a host-only handle; inputs are never
 * written; scratch is stream-ordered (cudaMallocAsync on `stream`).
 *
 * Encode: EncodeRingT + EmbedScale (encoder.go:201-333) of n_values <= n (MaxSlots) values per entry, the unmapped slots zero, into out_q
 * (level_q + 1 rows) and, for Embed only (no LGPU_ENC_SCALE_UP), out_p (level_p + 1 rows of a ringqp.Poly; level_p = -1: none). Words
 * are canonical, except that Embed without NTT or Montgomery keeps the reference's literal ring-T word on a row whose q_i < t. With
 * LGPU_ENC_COEFFS (Encode with IsBatched false, encoder.go:148-199; LGPU_ENC_SCALE_UP required, level_p = -1): n_values <= N words as
 * coefficients, uint64 words unreduced, MulScalar(scale) mod t, RingT2Q(scaleUp), NTT when LGPU_ENC_NTT.
 *
 * Decode: Decode (encoder.go:471-521) of `batch` plaintexts pt [level + 1][N] (INTT first when LGPU_ENC_NTT; coefficient-domain words may
 * be any 64-bit value): RingQ2T(scaleDown), then MulScalar(scale^-1 mod t); batched: ring-T NTT and the n slots into `values`; with
 * LGPU_ENC_COEFFS: uint64 gives N words, int64 (LGPU_ENC_SIGNED) centres only the first n words and leaves the rest of the entry
 * untouched, as the reference does. Signed words are v - t for v >= t >> 1. At level > 0 with n < N (gap > 1), the bit lengths of
 * q_0..q_level must sum to at most 4096 (the CRT accumulator has 16, 32 or 64 words of 64 bits, chosen from that sum); past it the
 * call is refused before any launch, even where Q_level itself has fewer than 4096 bits. */
#define LGPU_ENC_SIGNED 8
#define LGPU_ENC_SCALE_UP 16
typedef struct lgpu_bgv_encoder lgpu_bgv_encoder;
int lgpu_bgv_encoder_create(lgpu_ctx* ctx, uint64_t t, lgpu_bgv_encoder** out);
void lgpu_bgv_encoder_destroy(lgpu_bgv_encoder* enc);
int lgpu_bgv_encode(lgpu_bgv_encoder* enc, const uint64_t* values, int n_values, int flags, uint64_t scale, int level_q, uint64_t* out_q,
                    int level_p, uint64_t* out_p, int batch, size_t values_stride, size_t out_q_stride, size_t out_p_stride, void* stream);
int lgpu_bgv_decode(lgpu_bgv_encoder* enc, const uint64_t* pt, int level, int flags, uint64_t scale, uint64_t* values, int batch,
                    size_t pt_stride, size_t values_stride, void* stream);


/* ---- multiparty BGV / BFV: collective refresh, encryption-to-shares, shares-to-encryption (multiparty/mpbgv) ----------------------
 * NTT-domain ciphertexts on the Standard ring, paramsIn == paramsOut, through the encoder handle (t, t^-1 mod q_i, floor(Q/2) and the slot
 * permutation). An AdditiveShare is n = RingT().N() words per entry ([batch][n], dense); KeySwitch shares, CRPs and aggregates are
 * [batch][level + 1][N]; sk is [nQ + nP][N] (NTT + Montgomery, rows 0..level used); e is [batch][N] signed. batch <= 65535. Every check
 * runs before any launch, also on a host-only handle. Results keep the reference's words:
 *   - E2S and S2E shares lie in [0, 2q) (a KeySwitch share in [0, 2q), then Sub = CRed(a + q - b) or Add = CRed(a + b));
 *   - RingQ2T at level > 0 with n = N returns ModUpExact's lazy word in [0, 3t); the other branches are canonical. GetShare's
 *     ring-T Add and the RingT2Q of recrypt take such words as the integers they are, as the reference does.
 *
 * lgpu_mpbgv_sample_mask: the mask of EncToShareProtocol.GenShare, ring.UniformSampler over ring T: every word uniform in [0, t), with
 * the rejection of lgpu_sample_uniform, on the mask domain of the Philox counter (bit 29 of the polynomial word, which no other sampler
 * sets), so mask streams are disjoint from every other stream of the same seed and id.
 * lgpu_mpbgv_e2s_share: EncToShareProtocol.GenShare (mpbgv/sharing.go:62-71) at `level` = min(ct level, share level): c1 rows 0..level
 * at batch stride `stride`; share = Sub(KeySwitch(sk, 0) share, NTT(RingT2Q(level, true, mask))).
 * lgpu_mpbgv_s2e_share: ShareToEncProtocol.GenShare (:126-143): share = Add(KeySwitch(0, sk) share on the crp, NTT(RingT2Q(mask))).
 * lgpu_mpbgv_e2s_get_share: EncToShareProtocol.GetShare (:78-91): out = RingQ2T(level, true, INTT(Add(agg, ct0))) [+ secret, ring-T
 * Add]; secret may be null. ct0 rows 0..level at batch stride `stride`. Refused past the CRT limit of lgpu_bgv_decode.
 * lgpu_mpbgv_recrypt: the end of MaskedTransformProtocol.Transform (mpbgv/transform.go:173-180): ct_out [batch][2][level + 1][N] gets
 * c0 = Add(NTT(RingT2Q(level, true, mask)), agg) and c1 = crp.
 * lgpu_mpbgv_encode_ring_t / lgpu_mpbgv_decode_ring_t: EncodeRingT / DecodeRingT (encoder.go:203-262, :341-374) of n []uint64 values per
 * entry, the Decode / Encode steps of a MaskedTransformFunc; scale = MetaData.Scale.Uint64(). */
int lgpu_mpbgv_sample_mask(lgpu_bgv_encoder* enc, uint64_t seed, uint64_t stream_id, uint64_t* mask, int batch, void* stream);
int lgpu_mpbgv_e2s_share(lgpu_bgv_encoder* enc, int level, const uint64_t* c1, size_t stride, const uint64_t* sk, const int64_t* e,
                         const uint64_t* mask, uint64_t* share, int batch, void* stream);
int lgpu_mpbgv_s2e_share(lgpu_bgv_encoder* enc, int level, const uint64_t* crp, const uint64_t* sk, const int64_t* e, const uint64_t* mask,
                         uint64_t* share, int batch, void* stream);
int lgpu_mpbgv_e2s_get_share(lgpu_bgv_encoder* enc, int level, const uint64_t* ct0, size_t stride, const uint64_t* agg, const uint64_t* secret,
                             uint64_t* out, int batch, void* stream);
int lgpu_mpbgv_recrypt(lgpu_bgv_encoder* enc, int level, const uint64_t* mask, const uint64_t* agg, const uint64_t* crp, uint64_t* ct_out, int batch,
                       void* stream);
int lgpu_mpbgv_encode_ring_t(lgpu_bgv_encoder* enc, const uint64_t* values, uint64_t scale, uint64_t* pt, int batch, void* stream);
int lgpu_mpbgv_decode_ring_t(lgpu_bgv_encoder* enc, const uint64_t* pt, uint64_t scale, uint64_t* values, int batch, void* stream);


/* ---- multiparty CKKS: collective refresh, encryption-to-shares, shares-to-encryption (multiparty/mpckks) --------------------------
 * NTT-domain ciphertexts on the Standard ring, paramsIn == paramsOut, IsMontgomery false. An AdditiveShareBigint is dslots = 2 slots
 * big integers per entry ([batch][dslots][W], W little-endian two's-complement 64-bit words). W is 4 or 8: the smallest with
 * 64 W >= bits(q_0) + ... + bits(q_level) + 16 at the E2S level, so sums of up to 2^15 shares stay exact; E2S levels needing more are
 * refused. Lifted values go to coefficient j N / dslots (SetCoefficientsBigint followed by NTTSparseAndMontgomery, whose output is
 * the NTT of that spread polynomial). Shares lie in [0, 2q) as for mpbgv. Every check runs before any launch, also on a host-only ctx.
 *
 * lgpu_mpckks_sample_mask: bignum.RandInt(prng, 2^log_bound) mapped to [-2^(log_bound-1), 2^(log_bound-1)) (sharing.go GenShare), on
 * the mask domain of the Philox counter plus bit 28 (disjoint from every other stream, mpbgv masks included); log_bound < 64 W.
 * lgpu_mpckks_e2s_share: EncToShareProtocol.GenShare at `level` = min(ct level, share level): Sub(KeySwitch(sk, 0) share,
 * NTT(SetCoefficientsBigint(mask))). Refused with "cannot GenShare: ciphertext level is not large enough for refresh correctness" when
 * 2^log_bound > Q_level.
 * lgpu_mpckks_s2e_share: ShareToEncProtocol.GenShare: Add(KeySwitch(0, sk) share on the crp, NTT(SetCoefficientsBigint(secret))). With
 * scales = {d_lo, d_hi, s_lo, s_hi} (128-bit d = defaultScale, s = inputScaleInt, both > 0) each value is Quo(Mul(v, d), s) first
 * (RefreshProtocol.GenShare's applyTransformAndScale, truncation toward zero); null: no scaling.
 * lgpu_mpckks_e2s_get_share: EncToShareProtocol.GetShare: PolyToBigintCentered(INTT(Add(agg, ct0)), gap) [+ secret] into out.
 * lgpu_mpckks_refresh_finalize: RefreshProtocol.Finalize: GetShare(nil) at level_in, the scaling above, SetCoefficientsBigint at level_out,
 * NTT, Add(agg_s2e) into c0; c1 = crp. ct_out is [batch][2][level_out + 1][N]. */
int lgpu_mpckks_sample_mask(lgpu_ctx* ctx, int log_slots, int log_bound, int W, uint64_t seed, uint64_t stream_id, uint64_t* mask, int batch,
                            void* stream);
int lgpu_mpckks_e2s_share(lgpu_ctx* ctx, int level, int log_slots, int log_bound, const uint64_t* c1, size_t stride, const uint64_t* sk,
                          const int64_t* e, const uint64_t* mask, int W, uint64_t* share, int batch, void* stream);
int lgpu_mpckks_s2e_share(lgpu_ctx* ctx, int level, int log_slots, const uint64_t* crp, const uint64_t* sk, const int64_t* e, const uint64_t* secret,
                          int W, const uint64_t* scales, uint64_t* share, int batch, void* stream);
int lgpu_mpckks_e2s_get_share(lgpu_ctx* ctx, int level, int log_slots, const uint64_t* ct0, size_t stride, const uint64_t* agg, const uint64_t* secret,
                              int W, uint64_t* out, int batch, void* stream);
int lgpu_mpckks_refresh_finalize(lgpu_ctx* ctx, int level_in, int log_slots, const uint64_t* ct0, size_t stride, const uint64_t* agg_e2s,
                                 int level_out, const uint64_t* agg_s2e, const uint64_t* crp, int W, const uint64_t* scales, uint64_t* ct_out,
                                 int batch, void* stream);


/* ---- launch accounting / profiling (used by bench.py) ------------------------------------------------------- */
enum lgpu_kclass {
    LGPU_KCLASS_NTT_FWD = 0,   /* one forward transform of rows x batch polynomials (1 or 2 kernels) */
    LGPU_KCLASS_NTT_INV,
    LGPU_KCLASS_VECOP,
    LGPU_KCLASS_MODUP,         /* basis extension / decomposition */
    LGPU_KCLASS_MAC,           /* key-switch multiply-accumulate */
    LGPU_KCLASS_TENSOR,
    LGPU_KCLASS_AUTOMORPHISM,
    LGPU_KCLASS_FUSED,         /* K2: basis extension / rescale prologue folded into the strided transform pass */
    LGPU_KCLASS_EPILOGUE,      /* chunk transform pass with the ModDown / Rescale epilogue */
    LGPU_KCLASS_COUNT
};
/* total number of CUDA kernels this library has launched in the process */
unsigned long long lgpu_launch_count(void);
/* When enabled every launch scope is bracketed by CUDA events on its stream. lgpu_profile_read sums (and clears)
 * per class: elapsed ms, algorithmic bytes (compulsory read + write of the operands), scopes and kernels. */
int lgpu_profile_enable(int on);
int lgpu_profile_read(double* ms, double* alg_bytes, unsigned long long* scopes, unsigned long long* kernels);

#ifdef __cplusplus
}
#endif
#endif /* LATTIGO_B200_H */

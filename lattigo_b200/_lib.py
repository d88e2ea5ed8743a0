"""ctypes loader for lattigo_b200/lib/liblattigo_b200.so (the C ABI in include/lattigo_b200.h).

The product path has NO CPU fallback: if the CUDA library is missing this module raises, loudly."""
import ctypes
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
# LGPU_SO_PATH: development override used to A/B kernel variants built into lib/variants/ (never a CPU path)
SO_PATH = os.environ.get("LGPU_SO_PATH") or os.path.join(HERE, "lib", "liblattigo_b200.so")
HEADER = os.path.join(HERE, "..", "include", "lattigo_b200.h")

_lib = None


class LgpuError(RuntimeError):
    pass


def declared_symbols():
    """Every function name declared in include/lattigo_b200.h."""
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lgpu_[a-z0-9_]+)\s*\(", src)))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise LgpuError(
                "liblattigo_b200.so is missing (%s). Build it with `python -m lattigo_b200.build` "
                "(nvcc, sm_90a). There is no CPU fallback." % SO_PATH)
        L = ctypes.CDLL(SO_PATH)
        c = ctypes
        vp, u64, i, z = c.c_void_p, c.c_uint64, c.c_int, c.c_size_t
        L.lgpu_last_error.restype = c.c_char_p
        L.lgpu_version.restype = c.c_char_p
        sig = {
            "lgpu_create": [c.POINTER(vp), i, i, i, vp, i, vp, i],
            "lgpu_destroy": [vp],
            "lgpu_sync": [vp, vp],
            "lgpu_ring_get_table": [vp, i, i, i, vp, z],
            "lgpu_ring_set_roots": [vp, i, i, vp, vp, u64],
            "lgpu_malloc": [vp, c.POINTER(vp), z],
            "lgpu_free": [vp, vp],
            "lgpu_memcpy_h2d": [vp, vp, vp, z, vp],
            "lgpu_memcpy_d2h": [vp, vp, vp, z, vp],
            "lgpu_ntt": [vp, i, i, vp, vp, i, i, z, vp],
            "lgpu_intt": [vp, i, i, vp, vp, i, i, z, vp],
            "lgpu_ntt_then_mul_coeffs_montgomery": [vp, i, i, vp, vp, vp, i, z, vp],
            "lgpu_subring_ntt": [vp, i, i, vp, vp, i, vp],
            "lgpu_subring_intt": [vp, i, i, vp, vp, i, vp],
            "lgpu_vecop": [vp, i, i, i, vp, vp, vp, vp, vp, i, z, vp],
            "lgpu_subring_vecop": [vp, i, i, i, vp, vp, vp, u64, u64, i, vp],
            "lgpu_automorphism_ntt_index": [vp, u64, vp, vp],
            "lgpu_automorphism_ntt_with_index": [vp, i, i, vp, vp, vp, i, i, z, vp],
            "lgpu_automorphism_ntt": [vp, i, i, vp, u64, vp, i, z, vp],
            "lgpu_automorphism": [vp, i, i, vp, u64, vp, i, z, vp],
            "lgpu_shift": [vp, i, i, vp, i, vp, i, z, vp],
            "lgpu_mult_by_monomial": [vp, i, i, vp, i, vp, i, z, vp],
            "lgpu_map_small_dimension_to_larger_dimension_ntt": [vp, vp, i, vp, i, i, vp],
            "lgpu_extend_basis_small_norm_and_center": [vp, vp, i, vp, i, z, z, vp],
            "lgpu_modup_centered": [vp, vp, i, i, i, i, vp, vp, i, z, z, z, vp],
            "lgpu_modup_qtop": [vp, i, i, vp, vp, i, z, z, vp],
            "lgpu_modup_ptoq": [vp, i, i, vp, vp, i, z, z, vp],
            "lgpu_moddown_qp_to_q": [vp, i, i, vp, vp, vp, i, z, z, vp],
            "lgpu_moddown_qp_to_q_ntt": [vp, i, i, vp, vp, vp, i, z, z, vp],
            "lgpu_moddown_qp_to_p": [vp, i, i, vp, vp, vp, i, z, z, vp],
            "lgpu_decompose_and_split": [vp, i, i, i, i, vp, vp, vp, i, z, z, vp],
            "lgpu_div_by_last_modulus_many": [vp, i, i, i, i, vp, vp, i, z, z, vp],
            "lgpu_gadget_product": [vp, i, vp, vp, vp, vp, i, z, z, vp],
            "lgpu_gadget_product_lazy": [vp, i, vp, vp, vp, vp, vp, vp, i, z, z, z, vp],
            "lgpu_evaluator_moddown": [vp, i, i, vp, vp, vp, vp, vp, vp, i, z, z, z, vp],
            "lgpu_decompose_single_ntt": [vp, i, i, i, i, vp, vp, vp, vp, i, z, z, z, vp],
            "lgpu_decompose_ntt": [vp, i, i, i, vp, i, vp, i, z, vp],
            "lgpu_gadget_product_hoisted": [vp, i, vp, vp, vp, vp, i, z, vp],
            "lgpu_gadget_product_hoisted_lazy": [vp, i, vp, vp, vp, vp, vp, vp, i, z, z, vp],
            "lgpu_evaluator_automorphism": [vp, i, vp, u64, vp, vp, vp, i, vp],
            "lgpu_evaluator_relinearize": [vp, i, vp, vp, vp, i, vp],
            "lgpu_ckks_mulrelin_rescale_batch": [vp, i, vp, vp, vp, i, vp, i, vp],
            "lgpu_ckks_mulrelin_rescale_batch_host": [vp, i, vp, vp, vp, i, vp, i, i],
            "lgpu_ckks_polynomial_evaluate": [vp, i, vp, i, vp, vp, vp, vp],
            "lgpu_bgv_create": [vp, u64, vp, i, c.POINTER(vp)],
            "lgpu_bgv_destroy": [vp],
            "lgpu_bgv_mulrelin_batch": [vp, i, vp, vp, vp, i, i, vp, i, vp],
            "lgpu_bgv_polynomial_evaluate": [vp, i, vp, i, vp, vp, i, vp, vp],
            "lgpu_ckks_polynomial_vector_evaluate": [vp, i, vp, i, vp, vp, vp, vp, vp],
            "lgpu_bgv_polynomial_vector_evaluate": [vp, i, vp, i, vp, vp, vp, i, vp, vp],
            "lgpu_lintrans_evaluate_many": [vp, i, vp, vp, i, vp, vp, vp, i, vp],
            "lgpu_evaluator_automorphism_hoisted_lazy": [vp, i, vp, vp, i, u64, vp, vp, vp, vp, vp, i, z, z, z, vp],
            "lgpu_evaluator_partial_traces_sum": [vp, i, vp, i, i, i, vp, vp, i, vp],
            "lgpu_evaluator_trace": [vp, i, vp, i, i, vp, vp, i, i, vp],
            "lgpu_ring_packing_expand": [vp, i, vp, i, i, vp, vp, i, vp],
            "lgpu_ring_packing_pack": [vp, i, vp, i, vp, i, i, i, vp, vp, i, vp],
            "lgpu_evaluator_apply_evaluation_key": [vp, vp, i, i, i, vp, vp, i, i, i, vp],
            "lgpu_rgsw_external_product": [vp, vp, i, vp, vp, vp, i, i, vp],
            "lgpu_sample_uniform": [vp, i, i, u64, u64, vp, i, z, vp],
            "lgpu_sample_ternary": [vp, c.c_double, i, u64, u64, vp, i, vp],
            "lgpu_sample_gaussian": [vp, c.c_double, c.c_double, u64, u64, vp, i, vp],
            "lgpu_small_poly_to_rns": [vp, i, i, vp, vp, vp, i, z, z, vp],
            "lgpu_encrypt_zero_pk": [vp, i, vp, vp, vp, vp, vp, i, i, i, vp],
            "lgpu_encrypt_zero_sk": [vp, i, i, vp, vp, vp, vp, i, i, i, vp],
            "lgpu_gen_evaluation_key": [vp, vp, vp, vp, vp, vp],
            "lgpu_mp_aggregate": [vp, i, i, vp, i, vp, z, vp],
            "lgpu_mp_key_switch_share": [vp, i, vp, z, vp, vp, vp, vp, i, vp],
            "lgpu_mp_public_key_switch_share": [vp, i, vp, z, vp, vp, vp, vp, vp, vp, vp, i, vp],
            "lgpu_mp_evaluation_key_gen_share": [vp, vp, vp, vp, i, vp, vp, vp, vp],
            "lgpu_rgsw_encrypt": [vp, vp, vp, i, vp, i, i, vp, vp, vp, i, vp],
            "lgpu_gen_galois_keys": [vp, vp, vp, i, vp, vp, vp],
            "lgpu_blind_rotation_gen_evaluation_key": [vp, vp, vp, i, i, c.c_double, c.c_double, u64, vp, vp, vp, vp],
            "lgpu_mp_rkg_share_round_one": [vp, vp, vp, vp, vp, vp, vp, vp, vp],
            "lgpu_mp_rkg_share_round_two": [vp, vp, vp, vp, vp, vp, vp],
            "lgpu_mp_shamir_share": [vp, i, i, vp, i, vp, i, vp, vp],
            "lgpu_blind_rotate_core": [vp, vp, i, vp, i, vp, vp, vp, i, vp],
            "lgpu_blind_rotation_evaluate": [vp, vp, vp, i, i, vp, i, vp, vp, vp, i, vp, i, i, vp, i, vp],
            "lgpu_ckks_special_fft": [vp, vp, i, i, vp, vp, i, i, z, vp],
            "lgpu_ckks_encode": [vp, vp, i, i, c.c_double, i, vp, vp, i, vp, i, vp, i, z, z, z, vp],
            "lgpu_ckks_decode": [vp, vp, i, i, c.c_double, i, c.c_double, vp, vp, vp, i, z, z, vp],
            "lgpu_bgv_encoder_create": [vp, u64, c.POINTER(vp)],
            "lgpu_bgv_encoder_destroy": [vp],
            "lgpu_bgv_encode": [vp, vp, i, i, u64, i, vp, i, vp, i, z, z, z, vp],
            "lgpu_bgv_decode": [vp, vp, i, i, u64, vp, i, z, z, vp],
            "lgpu_mpbgv_sample_mask": [vp, u64, u64, vp, i, vp],
            "lgpu_mpbgv_e2s_share": [vp, i, vp, z, vp, vp, vp, vp, i, vp],
            "lgpu_mpbgv_s2e_share": [vp, i, vp, vp, vp, vp, vp, i, vp],
            "lgpu_mpbgv_e2s_get_share": [vp, i, vp, z, vp, vp, vp, i, vp],
            "lgpu_mpbgv_recrypt": [vp, i, vp, vp, vp, vp, i, vp],
            "lgpu_mpbgv_encode_ring_t": [vp, vp, u64, vp, i, vp],
            "lgpu_mpbgv_decode_ring_t": [vp, vp, u64, vp, i, vp],
            "lgpu_mpckks_sample_mask": [vp, i, i, i, u64, u64, vp, i, vp],
            "lgpu_mpckks_e2s_share": [vp, i, i, i, vp, z, vp, vp, vp, i, vp, i, vp],
            "lgpu_mpckks_s2e_share": [vp, i, i, vp, vp, vp, vp, i, vp, vp, i, vp],
            "lgpu_mpckks_e2s_get_share": [vp, i, i, vp, z, vp, vp, i, vp, i, vp],
            "lgpu_mpckks_refresh_finalize": [vp, i, i, vp, z, vp, i, vp, vp, i, vp, vp, i, vp],
            "lgpu_poly_load": [vp, vp, z, vp, i, vp, vp, vp],
            "lgpu_poly_store": [vp, vp, i, vp, z, vp, vp],
            "lgpu_gadget_ct_load": [vp, vp, z, vp, z, vp, vp],
            "lgpu_galois_key_load": [vp, vp, z, vp, vp, vp, z, vp, vp],
            "lgpu_profile_enable": [i],
            "lgpu_profile_read": [vp, vp, vp, vp],
        }
        for name, args in sig.items():
            f = getattr(L, name)
            f.argtypes = args
            if name not in ("lgpu_destroy", "lgpu_bgv_destroy", "lgpu_bgv_encoder_destroy"):
                f.restype = i
        L.lgpu_destroy.restype = None
        L.lgpu_bgv_destroy.restype = None
        L.lgpu_bgv_encoder_destroy.restype = None
        L.lgpu_galois_element.restype = c.c_uint64
        L.lgpu_galois_element.argtypes = [vp, c.c_longlong]
        L.lgpu_launch_count.restype = c.c_ulonglong
        L.lgpu_launch_count.argtypes = []
        _lib = L
    return _lib


class GadgetCtStruct(ctypes.Structure):
    """lgpu_gadget_ct (include/lattigo_b200.h)."""
    _fields_ = [("data", ctypes.c_void_p), ("level_q", ctypes.c_int), ("level_p", ctypes.c_int),
                ("base_two_decomposition", ctypes.c_int), ("n_digits", ctypes.c_int), ("n_pw2_max", ctypes.c_int),
                ("pw2_sizes", ctypes.POINTER(ctypes.c_int))]


class EvkInfoStruct(ctypes.Structure):
    """lgpu_evk_info (include/lattigo_b200.h)."""
    _fields_ = [("level_q", ctypes.c_int), ("level_p", ctypes.c_int), ("base_two_decomposition", ctypes.c_int), ("n_digits", ctypes.c_int),
                ("n_pw2_max", ctypes.c_int), ("pw2_sizes", ctypes.c_int * 128), ("device_bytes", ctypes.c_size_t), ("consumed", ctypes.c_size_t)]


class LinTransStruct(ctypes.Structure):
    """lgpu_lintrans (include/lattigo_b200.h)."""
    _fields_ = [("level_q", ctypes.c_int), ("level_p", ctypes.c_int), ("log_slots", ctypes.c_int), ("n1", ctypes.c_int),
                ("n_diags", ctypes.c_int), ("diag_index", ctypes.POINTER(ctypes.c_int)), ("diag", ctypes.POINTER(ctypes.c_void_p))]


class GaloisKeysStruct(ctypes.Structure):
    """lgpu_galois_keys (include/lattigo_b200.h)."""
    _fields_ = [("n_keys", ctypes.c_int), ("gal_els", ctypes.POINTER(ctypes.c_uint64)), ("keys", ctypes.POINTER(GadgetCtStruct))]


class GaloisKeys:
    """The lgpu_galois_keys view of {galEl: GadgetCiphertext}. gks keeps its two host arrays alive (ctypes holds what a struct field
    points to), but it also points into the keys' device tensors: whoever holds gks holds `keys` for as long."""

    def __init__(self, keys):
        self.keys = dict(keys)
        els = list(self.keys)
        self._els = (ctypes.c_uint64 * max(1, len(els)))(*els)
        self._structs = (GadgetCtStruct * max(1, len(els)))(*[self.keys[g].struct for g in els])
        self.gks = GaloisKeysStruct(len(els), self._els, self._structs)


def check(rc):
    if rc != 0:
        raise LgpuError(lib().lgpu_last_error().decode())

"""The key checks of the C-ABI entry points that check the device first, on a small device context with real ciphertext buffers.
Each entry point reports the same message as the host-only entry points (tests/test_cabi_keys_cpu.py) for the same fault, and
refuses the call before any kernel launch. The misaligned key points 8 bytes into a device buffer one key larger than a key, so a
check that moved behind a launch would show up as a launch count, not as a fault."""
import ctypes

import numpy as np
import pytest

from tests import helpers as H
from tests.test_cabi_keys_cpu import ALIGN, ARRAYS, KEY_FAULTS, NULL_ARG, NULL_KEY, NULL_RLK

pytestmark = pytest.mark.gpu

LOGN, LQ, LP = 10, 3, 1
N = 1 << LOGN
NQ, NP = LQ + 1, LP + 1
ND = (LQ + LP + 1) // (LP + 1)
KEY_WORDS = ND * 2 * (NQ + NP) * N


class Env:
    def __init__(self):
        import torch
        import lattigo_b200 as lb
        self.lb, self.torch = lb, torch
        self.ctx = lb.Context(LOGN, H.Qi60[:NQ], H.Pi60[:NP])
        self.keybuf = self.zeros(2 * KEY_WORDS)           # one key larger than a key: the misaligned key stays inside it
        self.bufs = []

    def zeros(self, words):
        return self.torch.zeros(words, dtype=self.torch.int64, device="cuda")

    def ptr(self, words):
        t = self.zeros(words)
        self.bufs.append(t)
        return ctypes.c_void_p(t.data_ptr())

    def key(self, fault=None, pw2=0):
        addr = self.keybuf.data_ptr() + (8 if fault == "misaligned" else 0)
        return self.lb._lib.GadgetCtStruct(None if fault == "null_data" else ctypes.c_void_p(addr), LQ, LP, pw2, ND, 1, None)

    def key_ref(self, fault, keep):
        if fault == "null":
            return None
        g = self.key(fault)
        keep.append(g)
        return ctypes.byref(g)

    def set_ref(self, els, fault, keep, pw2=()):
        """lgpu_galois_keys over els with `fault` on its last key (or on its arrays); pw2: indices of keys with BaseTwoDecomposition 8."""
        lb = self.lb
        if fault == "null":
            return None
        arr = (ctypes.c_uint64 * len(els))(*els)
        keys = (lb._lib.GadgetCtStruct * len(els))(*[self.key(fault if i == len(els) - 1 and fault in KEY_FAULTS else None, 8 if i in pw2 else 0)
                                                     for i in range(len(els))])
        gks = lb._lib.GaloisKeysStruct(len(els), None if fault == "null_gal_els" else arr, None if fault == "null_keys" else keys)
        keep += [arr, keys, gks]
        return ctypes.byref(gks)

    def refused(self, call):
        """The error message of a refused call, which must not have launched a kernel."""
        self.torch.cuda.synchronize()
        rc = []
        n = H.launch_delta(lambda: rc.append(call()))
        assert rc[0] != 0 and n == 0, (rc, n)
        return self.lb.lib().lgpu_last_error().decode()


@pytest.fixture(scope="module")
def env():
    e = Env()
    yield e
    e.torch.cuda.synchronize()
    e.ctx.close()


KEY_MSG = {"null_data": NULL_KEY, "misaligned": ALIGN, "null": NULL_KEY}
RLK_MSG = {"null_data": NULL_RLK, "misaligned": ALIGN, "null": NULL_RLK}
SET_MSG = {"null_data": NULL_KEY, "misaligned": ALIGN, "null_gal_els": ARRAYS, "null_keys": ARRAYS}


def _gadget_family(e, name, k):
    """One call of a gadget-product-family entry point with key pointer k, on valid buffers."""
    L, h = e.lb.lib(), e.ctx.h
    ct, qp = NQ * N, (NQ + NP) * N
    if name == "gadget_product":
        return L.lgpu_gadget_product(h, LQ, e.ptr(ct), k, e.ptr(ct), e.ptr(ct), 1, ct, ct, None)
    if name == "gadget_product_lazy":
        return L.lgpu_gadget_product_lazy(h, LQ, e.ptr(ct), k, e.ptr(ct), e.ptr(NP * N), e.ptr(ct), e.ptr(NP * N), 1, ct, ct, NP * N, None)
    if name == "gadget_product_hoisted":
        return L.lgpu_gadget_product_hoisted(h, LQ, e.ptr(ND * qp), k, e.ptr(ct), e.ptr(ct), 1, ct, None)
    if name == "gadget_product_hoisted_lazy":
        return L.lgpu_gadget_product_hoisted_lazy(h, LQ, e.ptr(ND * qp), k, e.ptr(ct), e.ptr(NP * N), e.ptr(ct), e.ptr(NP * N), 1, ct, NP * N, None)
    if name == "evaluator_automorphism":
        return L.lgpu_evaluator_automorphism(h, LQ, e.ptr(2 * ct), 5, k, None, e.ptr(2 * ct), 1, None)
    if name == "evaluator_relinearize":
        return L.lgpu_evaluator_relinearize(h, LQ, e.ptr(3 * ct), k, e.ptr(2 * ct), 1, None)
    if name == "ckks_mulrelin_rescale_batch":
        return L.lgpu_ckks_mulrelin_rescale_batch(h, LQ, e.ptr(2 * ct), e.ptr(2 * ct), k, 1, e.ptr(2 * ct), 1, None)
    if name == "ckks_mulrelin_rescale_batch_host":
        a, b, o = (np.zeros(2 * ct, dtype=np.uint64) for _ in range(3))
        return L.lgpu_ckks_mulrelin_rescale_batch_host(h, LQ, a.ctypes.data, b.ctypes.data, k, 1, o.ctypes.data, 1, 1)
    if name == "rgsw_external_product_0":
        return L.lgpu_rgsw_external_product(h, e.ptr(2 * ct), LQ, k, ctypes.byref(e.key()), e.ptr(2 * ct), LQ, 1, None)
    if name == "rgsw_external_product_1":
        return L.lgpu_rgsw_external_product(h, e.ptr(2 * ct), LQ, ctypes.byref(e.key()), k, e.ptr(2 * ct), LQ, 1, None)
    if name == "evaluator_automorphism_hoisted_lazy":
        return L.lgpu_evaluator_automorphism_hoisted_lazy(h, LQ, e.ptr(2 * ct), e.ptr(ND * qp), LQ, 5, k, e.ptr(ct), e.ptr(NP * N), e.ptr(ct),
                                                          e.ptr(NP * N), 1, 2 * ct, ct, NP * N, None)
    raise AssertionError(name)


FAMILY = ("gadget_product", "gadget_product_lazy", "gadget_product_hoisted", "gadget_product_hoisted_lazy", "evaluator_automorphism",
          "evaluator_relinearize", "ckks_mulrelin_rescale_batch", "ckks_mulrelin_rescale_batch_host", "rgsw_external_product_0",
          "rgsw_external_product_1", "evaluator_automorphism_hoisted_lazy")


@pytest.mark.parametrize("name", FAMILY)
@pytest.mark.parametrize("fault", KEY_FAULTS)
def test_gadget_product_family(env, name, fault):
    keep = []
    assert env.refused(lambda: _gadget_family(env, name, env.key_ref(fault, keep))) == KEY_MSG[fault]


def _lintrans(e, gks):
    L = e.lb.lib()
    diag = (ctypes.c_void_p * 1)(e.ptr((NQ + NP) * N))
    mats = (e.lb._lib.LinTransStruct * 1)(e.lb._lib.LinTransStruct(LQ, LP, LOGN - 1, 0, 1, (ctypes.c_int * 1)(1), diag))
    outs = (ctypes.c_void_p * 1)(e.ptr(2 * NQ * N))
    levels = (ctypes.c_int * 1)(LQ)
    return L.lgpu_lintrans_evaluate_many(e.ctx.h, LQ, e.ptr(2 * NQ * N), mats, 1, gks, outs, levels, 1, None)


@pytest.mark.parametrize("fault", tuple(SET_MSG) + ("base_two",))
def test_lintrans_evaluate_many(env, fault):
    keep = []
    if fault == "base_two":
        gks = env.set_ref([5, 25], None, keep, pw2=(0,))
        want = "hoisted linear transformations need keys with BaseTwoDecomposition = 0"
    else:
        gks = env.set_ref([5, 25], fault, keep)
        want = SET_MSG[fault]
    assert env.refused(lambda: _lintrans(env, gks)) == want


def _blind_rotate_core(e, brk0, brk1, gks):
    a = np.zeros(4, dtype=np.uint64)
    return e.lb.lib().lgpu_blind_rotate_core(e.ctx.h, a.ctypes.data, len(a), e.ptr(2 * NQ * N), LQ, brk0, brk1, gks, 1, None)


@pytest.mark.parametrize("fault", tuple(SET_MSG) + ("null", "null_brk0", "null_brk1"))
def test_blind_rotate_core(env, fault):
    keep = []
    brk = (env.lb._lib.GadgetCtStruct * 4)(*[env.key() for _ in range(4)])
    els = [5, 2 * N - 5]
    if fault in ("null_brk0", "null_brk1"):
        gks = env.set_ref(els, None, keep)
        args = (None, brk) if fault == "null_brk0" else (brk, None)
        assert env.refused(lambda: _blind_rotate_core(env, *args, gks)) == NULL_ARG
        return
    gks = env.set_ref(els, fault, keep)
    assert env.refused(lambda: _blind_rotate_core(env, brk, brk, gks)) == (NULL_ARG if fault == "null" else SET_MSG[fault])


@pytest.mark.parametrize("fault", KEY_FAULTS)
def test_bgv_mulrelin_batch(env, fault):
    L = env.lb.lib()
    qmul = np.array(H.Pi60[NP:NP + 6], dtype=np.uint64)
    ev = ctypes.c_void_p()
    env.lb._lib.check(L.lgpu_bgv_create(env.ctx.h, 65537, qmul.ctypes.data, len(qmul), ctypes.byref(ev)))
    try:
        keep = []
        ct = 2 * NQ * N
        msg = env.refused(lambda: L.lgpu_bgv_mulrelin_batch(ev, LQ, env.ptr(ct), env.ptr(ct), env.key_ref(fault, keep), 0, 0, env.ptr(ct), 1, None))
        assert msg == RLK_MSG[fault]
    finally:
        L.lgpu_bgv_destroy(ev)


@pytest.mark.parametrize("fault", KEY_FAULTS)
def test_gen_evaluation_key(env, fault):
    keep = []
    qp = (NQ + NP) * N
    msg = env.refused(lambda: env.lb.lib().lgpu_gen_evaluation_key(env.ctx.h, env.ptr(qp), env.ptr(qp), env.key_ref(fault, keep), env.ptr(ND * qp),
                                                                   None))
    assert msg == (ALIGN if fault == "misaligned" else NULL_ARG)

"""The key checks of every C-ABI entry point that checks its keys before the device, on host-only contexts (no device work: keys
and ciphertexts carry placeholder addresses that are never dereferenced). Each entry point reports the same message for the same
fault: a key with null data, a key 8 but not 16 bytes aligned, a Galois key set with null arrays, a null key or key set; and a
valid call reaches the host-only refusal."""
import ctypes

import pytest

from lattigo_b200 import polyeval as PE
from oracle import innersum as OI
from oracle import oracle as O
from oracle import ringpacking as ORP
from tests.test_innersum_cpu import FAKE, LOGN, _ctx, _params, _pts_elements

NULL_KEY = "null evaluation key"
NULL_RLK = "null relinearization key"
ALIGN = "polynomial buffers and evaluation keys must be 16-byte aligned with even strides (words)"
ARRAYS = "null Galois key arrays"
NULL_SET = "null Galois key set"
NULL_ARG = "null argument"
HOST_ONLY = "host-only"

KEY_FAULTS = ("null_data", "misaligned", "null")
SET_FAULTS = ("null_data", "misaligned", "null_gal_els", "null_keys", "null")


def _key(levelQ=3, levelP=1, pw2=0, nd=None, addr=FAKE):
    import lattigo_b200 as lb
    nd = (levelQ + levelP + 1) // (levelP + 1) if nd is None else nd
    return lb._lib.GadgetCtStruct(ctypes.c_void_p(addr), levelQ, levelP, pw2, nd, 1, None)


def _faulty(g, fault):
    """g with the fault applied to its data address (valid for fault None or a fault of the set itself)."""
    if fault == "null_data":
        g.data = None
    elif fault == "misaligned":
        g.data = FAKE + 8
    return g


def _key_ref(fault, keep, **kw):
    """A pointer to one key descriptor with `fault`, or NULL."""
    if fault == "null":
        return None
    g = _faulty(_key(**kw), fault)
    keep.append(g)
    return ctypes.byref(g)


def _set_ref(els, fault, keep, **kw):
    """A pointer to a lgpu_galois_keys over els with `fault` (on its last key for the key faults), or NULL."""
    import lattigo_b200 as lb
    if fault == "null":
        return None
    els = list(els)
    arr = (ctypes.c_uint64 * max(1, len(els)))(*els)
    keys = (lb._lib.GadgetCtStruct * max(1, len(els)))(*[_key(**kw) for _ in els])
    _faulty(keys[len(els) - 1], fault)
    gks = lb._lib.GaloisKeysStruct(len(els), None if fault == "null_gal_els" else arr, None if fault == "null_keys" else keys)
    keep += [arr, keys, gks]
    return ctypes.byref(gks)


def _err(rc):
    import lattigo_b200 as lb
    assert rc != 0
    return lb.lib().lgpu_last_error().decode()


SET_MSG = {None: HOST_ONLY, "null_data": NULL_KEY, "misaligned": ALIGN, "null_gal_els": ARRAYS, "null_keys": ARRAYS, "null": NULL_SET}


@pytest.fixture(scope="module")
def ctx():
    c = _ctx()
    yield c
    c.close()


# ---- Galois key sets ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fault", (None,) + SET_FAULTS)
def test_partial_traces_sum(ctx, fault):
    import lattigo_b200 as lb
    keep = []
    gks = _set_ref(set(_pts_elements(_params(), 1, 7)), fault, keep)
    msg = _err(lb.lib().lgpu_evaluator_partial_traces_sum(ctx.h, 3, ctypes.c_void_p(FAKE), 1, 1, 7, gks, ctypes.c_void_p(FAKE << 4), 1, None))
    assert HOST_ONLY in msg if fault is None else msg == SET_MSG[fault]


@pytest.mark.parametrize("fault", (None,) + SET_FAULTS)
def test_trace(ctx, fault):
    import lattigo_b200 as lb
    keep = []
    gks = _set_ref(OI.GaloisElementsForTrace(_params(), 0), fault, keep)
    msg = _err(lb.lib().lgpu_evaluator_trace(ctx.h, 3, ctypes.c_void_p(FAKE), 1, 0, gks, ctypes.c_void_p(FAKE << 4), 3, 1, None))
    assert HOST_ONLY in msg if fault is None else msg == SET_MSG[fault]


@pytest.mark.parametrize("fault", (None,) + SET_FAULTS)
def test_ring_packing_expand(ctx, fault):
    import lattigo_b200 as lb
    keep = []
    gks = _set_ref(ORP.GaloisElementsForExpand(_params(), LOGN), fault, keep)
    msg = _err(lb.lib().lgpu_ring_packing_expand(ctx.h, 3, ctypes.c_void_p(FAKE), 1, 4, gks, ctypes.c_void_p(FAKE << 8), 1, None))
    assert HOST_ONLY in msg if fault is None else msg == SET_MSG[fault]


@pytest.mark.parametrize("fault", (None,) + SET_FAULTS)
def test_ring_packing_pack(ctx, fault):
    import lattigo_b200 as lb
    keep = []
    gks = _set_ref(ORP.GaloisElementsForPack(_params(), LOGN), fault, keep)
    idx = (ctypes.c_int * 2)(0, 1)
    msg = _err(lb.lib().lgpu_ring_packing_pack(ctx.h, 3, ctypes.c_void_p(FAKE), 1, idx, 2, LOGN, 1, gks, ctypes.c_void_p(FAKE << 8), 1, None))
    assert HOST_ONLY in msg if fault is None else msg == SET_MSG[fault]


# ---- single keys -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fault", (None,) + KEY_FAULTS)
def test_apply_evaluation_key(ctx, fault):
    import lattigo_b200 as lb
    keep = []
    evk = _key_ref(fault, keep)
    msg = _err(lb.lib().lgpu_evaluator_apply_evaluation_key(ctx.h, ctypes.c_void_p(FAKE), LOGN, 3, 1, evk, ctypes.c_void_p(FAKE << 8), LOGN, 3, 1,
                                                            None))
    assert HOST_ONLY in msg if fault is None else msg == {"null_data": NULL_KEY, "misaligned": ALIGN, "null": NULL_KEY}[fault]


@pytest.mark.parametrize("fault", (None,) + KEY_FAULTS)
def test_ckks_polynomial_evaluate(fault):
    import lattigo_b200 as lb
    q, p = O.gen_moduli(11, [55] + [40] * 8, [55, 55])
    c = lb.Context(10, q, p, device=-1)
    try:
        prog = PE.plan(q, 8, 2 ** 40, [0.1, 0.2, 0.3, 0.4], PE.MONOMIAL, 2 ** 40)
        assert PE.RELIN in prog.kinds()
        keep = []
        rlk = _key_ref(fault, keep, levelQ=8, levelP=1, nd=8)
        msg = _err(lb.lib().lgpu_ckks_polynomial_evaluate(c.h, 8, ctypes.c_void_p(FAKE), 1, ctypes.byref(prog.to_c(1)), rlk, ctypes.c_void_p(FAKE << 8),
                                                          None))
        assert HOST_ONLY in msg if fault is None else msg == {"null_data": NULL_RLK, "misaligned": ALIGN, "null": NULL_RLK}[fault]
    finally:
        c.close()


# ---- blind rotation: brk0, brk1 and the Galois keys ----------------------------------------------------------------------------
BR_LOGN, BR_LOGN_LWE, BR_WINDOW = 8, 5, 4


def _blind_rotation(which, fault):
    import lattigo_b200 as lb
    ctx, lwe = lb.Context(BR_LOGN, [0x7fff801], [], device=-1), lb.Context(BR_LOGN_LWE, [0x3001], [], device=-1)
    try:
        n = 1 << BR_LOGN_LWE
        kw = dict(levelQ=0, levelP=-1, pw2=7, nd=1)
        keep = []

        def brk(comp):
            if which == comp and fault == "null":
                return None
            arr = (lb._lib.GadgetCtStruct * n)(*[_key(**kw) for _ in range(n)])
            if which == comp:
                _faulty(arr[n - 1], fault)
            keep.append(arr)
            return arr
        els = [pow(5, k, 2 * ctx.N) for k in range(1, BR_WINDOW + 1)] + [2 * ctx.N - 5]
        gks = _set_ref(els, fault if which == "gks" else None, keep, **kw)
        slots = (ctypes.c_int * 2)(0, 3)
        polys = (ctypes.c_void_p * 2)(FAKE << 2, FAKE << 2)
        rc = lb.lib().lgpu_blind_rotation_evaluate(ctx.h, lwe.h, ctypes.c_void_p(FAKE), 0, 1, slots, 2, polys, brk(0), brk(1), n, gks, BR_WINDOW, 1,
                                                   ctypes.c_void_p(FAKE << 4), 1, None)
        return _err(rc)
    finally:
        ctx.close(); lwe.close()


@pytest.mark.parametrize("which", (0, 1))
@pytest.mark.parametrize("fault", (None,) + KEY_FAULTS)
def test_blind_rotation_keys(which, fault):
    msg = _blind_rotation(which, fault)
    assert HOST_ONLY in msg if fault is None else msg == {"null_data": NULL_KEY, "misaligned": ALIGN, "null": NULL_ARG}[fault]


@pytest.mark.parametrize("fault", (None,) + SET_FAULTS)
def test_blind_rotation_galois_keys(fault):
    msg = _blind_rotation("gks", fault)
    assert HOST_ONLY in msg if fault is None else msg == dict(SET_MSG, null=NULL_ARG)[fault]

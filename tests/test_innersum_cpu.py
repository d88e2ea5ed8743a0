"""lgpu_evaluator_partial_traces_sum / lgpu_evaluator_trace argument checks on a host-only context (no device work: the key
descriptors carry placeholder addresses that are never dereferenced), and the Python GaloisElementsFor* functions against
oracle/innersum.py."""
import ctypes

import pytest

from oracle import innersum as OI
from oracle import oracle as O
from tests import helpers as H

LOGN = 8
FAKE = 1 << 20          # 16-byte aligned placeholder device address


def _ctx(ring_type=0, P=True):
    import lattigo_b200 as lb
    return lb.Context(LOGN, H.Qi60[:4], H.Pi60[:2] if P else [], device=-1, ring_type=ring_type)


def _keys(els, levelQ=3, levelP=1, pw2=0):
    import lattigo_b200 as lb
    els = list(els)
    arr = (ctypes.c_uint64 * max(1, len(els)))(*els)
    nd = (levelQ + levelP + 1) // (levelP + 1)
    structs = (lb._lib.GadgetCtStruct * max(1, len(els)))(*[lb._lib.GadgetCtStruct(ctypes.c_void_p(FAKE), levelQ, levelP, pw2, nd, 1, None)
                                                             for _ in els])
    gks = lb._lib.GaloisKeysStruct(len(els), arr, structs)
    return gks, (arr, structs)


def _pts(ctx, gks, offset, n, level=3):
    import lattigo_b200 as lb
    rc = lb.lib().lgpu_evaluator_partial_traces_sum(ctx.h, level, ctypes.c_void_p(FAKE), 1, offset, n, ctypes.byref(gks), ctypes.c_void_p(FAKE << 4), 1, None)
    return rc, lb.lib().lgpu_last_error().decode()


def _trace(ctx, gks, log_n, level=3):
    import lattigo_b200 as lb
    rc = lb.lib().lgpu_evaluator_trace(ctx.h, level, ctypes.c_void_p(FAKE), 1, log_n, ctypes.byref(gks), ctypes.c_void_p(FAKE << 4), level, 1, None)
    return rc, lb.lib().lgpu_last_error().decode()


def _params():
    return O.Parameters(LOGN, H.Qi60[:4], H.Pi60[:2])


def _pts_elements(params, offset, n):
    out = []
    i, j = 0, n
    while j > 1:        # the keys PartialTracesSum asks for, in order (inner_sum.go:220-283)
        if j & 1:
            out.append(params.GaloisElement((n - (n & ((2 << i) - 1))) * offset))
        out.append(params.GaloisElement((1 << i) * offset))
        i, j = i + 1, j >> 1
    return out


@pytest.mark.parametrize("offset,n", [(0, 3), (1, 0), (-2, 0), (1, -1)])
def test_partial_traces_sum_rejects_n_and_offset(offset, n):
    ctx = _ctx()
    gks, _keep = _keys([])
    rc, msg = _pts(ctx, gks, offset, n)
    assert rc != 0 and msg == "partialtrace: invalid parameter (n = 0 or batchSize = 0)"
    ctx.close()


def test_all_keys_present_reaches_the_host_only_refusal():
    params = _params()
    ctx = _ctx()
    for offset, n in ((1, 7), (-4, 5), (3, 16), (1, 1)):
        gks, _keep = _keys(set(_pts_elements(params, offset, n)))
        rc, msg = _pts(ctx, gks, offset, n)
        assert rc != 0 and "host-only" in msg, (offset, n, msg)
    for log_n in range(LOGN):
        gks, _keep = _keys(OI.GaloisElementsForTrace(params, log_n))
        rc, msg = _trace(ctx, gks, log_n)
        assert rc != 0 and "host-only" in msg, (log_n, msg)
    ctx.close()


@pytest.mark.parametrize("which", range(5))
def test_missing_key_is_found_before_any_device_work(which):
    """Every key of the schedule is checked up front: dropping any one of them is reported by name."""
    params = _params()
    els = _pts_elements(params, 3, 7)
    need = sorted(set(els))
    drop = need[which % len(need)]
    gks, _keep = _keys([g for g in need if g != drop])
    ctx = _ctx()
    rc, msg = _pts(ctx, gks, 3, 7)
    assert rc != 0 and msg == "GaloisKey[%d] is missing" % drop
    ctx.close()


def test_trace_missing_key_and_log_n_range():
    params = _params()
    ctx = _ctx()
    need = OI.GaloisElementsForTrace(params, 0)
    gks, _keep = _keys(need[:-1])
    rc, msg = _trace(ctx, gks, 0)
    assert rc != 0 and msg == "GaloisKey[%d] is missing" % (2 * params.N() - 1)
    for bad in (-1, LOGN):
        rc, msg = _trace(ctx, gks, bad)
        assert rc != 0 and "out of range" in msg
    gks, _keep = _keys([])
    rc, msg = _trace(ctx, gks, LOGN - 1)          # gap = 1: a copy, no key needed
    assert rc != 0 and "host-only" in msg
    ctx.close()


def test_key_levels_and_base_two_decomposition_are_refused():
    params = _params()
    ctx = _ctx()
    els = set(_pts_elements(params, 1, 3))
    gks, _keep = _keys(els, levelP=0)
    rc, msg = _pts(ctx, gks, 1, 3)
    assert rc != 0 and "MaxLevelP" in msg
    gks, _keep = _keys(els, pw2=8)
    rc, msg = _pts(ctx, gks, 1, 3)
    assert rc != 0 and "BaseTwoDecomposition" in msg
    gks, _keep = _keys(OI.GaloisElementsForTrace(params, 2), pw2=8)
    rc, msg = _trace(ctx, gks, 2)
    assert rc != 0 and "BaseTwoDecomposition" in msg
    gks, _keep = _keys(els, levelQ=2)
    rc, msg = _pts(ctx, gks, 1, 3, level=3)          # key below the ciphertext level
    assert rc != 0 and "levels" in msg
    ctx.close()


def test_ring_type_and_missing_p_ring_are_refused():
    ctx = _ctx(ring_type=1)
    gks, _keep = _keys([])
    rc, msg = _pts(ctx, gks, 1, 2)
    assert rc != 0 and "ConjugateInvariant" in msg
    rc, msg = _trace(ctx, gks, 1)
    assert rc != 0 and "ConjugateInvariant" in msg
    ctx.close()
    ctx = _ctx(P=False)
    rc, msg = _pts(ctx, gks, 1, 2)
    assert rc != 0 and "P ring" in msg
    rc, msg = _pts(ctx, gks, 1, 1)                  # n = 1 is a copy: no key switch, no P ring needed
    assert rc != 0 and "host-only" in msg
    ctx.close()


def test_galois_elements_for_functions_match_the_oracle():
    import lattigo_b200 as lb
    params = _params()
    ctx = _ctx()
    for log_n in range(LOGN):
        assert lb.innersum.GaloisElementsForTrace(ctx, log_n) == OI.GaloisElementsForTrace(params, log_n)
    for batch in (1, 2, 3, 5, 16):
        for n in (1, 2, 3, 4, 5, 7, 8, 9, 16, 33, 128):
            assert lb.innersum.GaloisElementsForInnerSum(ctx, batch, n) == OI.GaloisElementsForInnerSum(params, batch, n)
            assert lb.innersum.GaloisElementsForReplicate(ctx, batch, n) == OI.GaloisElementsForReplicate(params, batch, n)
            # the reference's set holds every key the schedule uses; its extras are GaloisElement(0) (n not a power of two)
            # and GaloisElement(n * batch) (n a power of two)
            used = set(_pts_elements(params, batch, n))
            listed = set(OI.GaloisElementsForInnerSum(params, batch, n))
            assert used <= listed
            extra = {params.GaloisElement(0)} if n & (n - 1) else ({params.GaloisElement(n * batch)} if n > 1 else set())
            assert listed - used <= extra
    ctx.close()

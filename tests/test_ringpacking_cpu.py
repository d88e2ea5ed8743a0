"""lgpu_ring_packing_expand / lgpu_ring_packing_pack argument checks on a host-only context (no device work: the key descriptors
carry placeholder addresses that are never dereferenced), the GaloisElementsFor* sets and getMinimumGap against
oracle/ringpacking.py, and the keys each call looks up against the ones the restatement asks for."""
import ctypes
import gc
import weakref

import numpy as np
import pytest

from oracle import oracle as O
from oracle import ringpacking as ORP
from tests import helpers as H
from tests.test_innersum_cpu import FAKE, LOGN, _ctx, _keys

N = 1 << LOGN


def _expand(ctx, gks, log_gap, level=3, ct_in=FAKE, ct_out=FAKE << 8):
    import lattigo_b200 as lb
    rc = lb.lib().lgpu_ring_packing_expand(ctx.h, level, ctypes.c_void_p(ct_in), 1, log_gap, ctypes.byref(gks), ctypes.c_void_p(ct_out), 1, None)
    return rc, lb.lib().lgpu_last_error().decode()


def _pack(ctx, gks, idx, input_log_gap, zero, level=3, cts_in=FAKE, ct_out=FAKE << 8):
    import lattigo_b200 as lb
    arr = (ctypes.c_int * max(1, len(idx)))(*idx)
    rc = lb.lib().lgpu_ring_packing_pack(ctx.h, level, ctypes.c_void_p(cts_in), 1, arr, len(idx), input_log_gap, 1 if zero else 0, ctypes.byref(gks),
                                         ctypes.c_void_p(ct_out), 1, None)
    return rc, lb.lib().lgpu_last_error().decode()


def _params():
    return O.Parameters(LOGN, H.Qi60[:4], H.Pi60[:2])


def _all_keys(params):
    return sorted(set(ORP.GaloisElementsForExpand(params, LOGN)) | set(ORP.GaloisElementsForPack(params, LOGN)))


def test_error_paths_on_a_host_only_context():
    params = _params()
    ctx = _ctx()
    gks, _keep = _keys(_all_keys(params))
    assert _pack(ctx, gks, [], 8, True)[1] == "len(cts) = 0"
    assert _pack(ctx, gks, [3, 1], 8, True)[1] == "getMinimumGap: invalid index list: element must be sorted from smallest to largest"
    assert _pack(ctx, gks, [0, 1, 0], 8, True)[1] == "getMinimumGap: invalid index list: element must be sorted from smallest to largest"
    assert _pack(ctx, gks, [1, 1], 8, True)[1] == "getMinimumGap: invalid index list: contains duplicated elements"
    msg = "gaps between ciphertexts is smaller than inputLogGap > N"
    assert _pack(ctx, gks, [5], 8, False)[1] == msg              # one input: logGap = LogN, logEnd = 0
    assert _pack(ctx, gks, [0, 2], 0, True)[1] == msg            # inputLogGap = 0: logStart = LogN
    assert _pack(ctx, gks, [0, 4], 2, False)[1] == msg           # logEnd = LogN - 2 = logStart
    assert "slot 0" in _pack(ctx, gks, [1, 3], 8, False)[1]     # the reference returns nil, nil
    assert "slot 0" in _pack(ctx, gks, [300, 400], 8, True)[1]  # every index >= 2^inputLogGap
    for bad in (-1, LOGN + 1):
        assert "inputLogGap out of range" in _pack(ctx, gks, [0, 1], bad, True)[1]
        assert "logGap out of range" in _expand(ctx, gks, bad)[1]
    assert "overlaps" in _expand(ctx, gks, 4, ct_out=FAKE + 8 * 1024)[1]
    assert "overlaps" in _pack(ctx, gks, [0, 1], 8, True, ct_out=FAKE + 2 * 4 * N * 8)[1]
    assert "aligned" in _expand(ctx, gks, 4, ct_out=(FAKE << 8) + 8)[1]
    for g in (params.GaloisElement(1), 2 * N - 1):
        gks2, _k2 = _keys([x for x in _all_keys(params) if x != g])
        assert _pack(ctx, gks2, list(range(N)), 8, True)[1] == "GaloisKey[%d] is missing" % g
    gks2, _k2 = _keys([x for x in _all_keys(params) if x != N + 1])
    assert _expand(ctx, gks2, 8)[1] == "GaloisKey[%d] is missing" % (N + 1)
    gks3, _k3 = _keys(_all_keys(params), pw2=8)
    assert "BaseTwoDecomposition" in _expand(ctx, gks3, 8)[1]
    gks4, _k4 = _keys(_all_keys(params), levelQ=2)
    assert "levelQ out of range" in _pack(ctx, gks4, [0, 1], 8, True, level=3)[1]
    for call in (lambda: _expand(ctx, gks, 8), lambda: _pack(ctx, gks, [0, 1], 8, True)):
        rc, msg = call()
        assert rc != 0 and "host-only" in msg
    ctx.close()
    ci = _ctx(ring_type=1)
    assert "ring.Standard" in _expand(ci, gks, 8)[1]
    assert "ring.Standard" in _pack(ci, gks, [0, 1], 8, True)[1]
    ci.close()


def test_galois_elements_for_functions_match_the_oracle():
    import lattigo_b200 as lb
    params = _params()
    ctx = _ctx()
    for logN in range(LOGN + 1):
        assert lb.ringpacking.GaloisElementsForExpand(ctx, logN) == ORP.GaloisElementsForExpand(params, logN)
        assert lb.ringpacking.GaloisElementsForPack(ctx, logN) == ORP.GaloisElementsForPack(params, logN)
    for bad in (-1, LOGN + 1):
        with pytest.raises(ValueError, match="logGap > logN"):
            lb.ringpacking.GaloisElementsForPack(ctx, bad)
        with pytest.raises(ValueError, match="logGap > logN"):
            ORP.GaloisElementsForPack(params, bad)
    ctx.close()
    ci = _ctx(ring_type=1)
    with pytest.raises(ValueError, match="invalid ring type"):
        lb.ringpacking.GaloisElementsForPack(ci, 2)
    ci.close()


def test_get_minimum_gap_quirks():
    import lattigo_b200 as lb
    for keys, want in (([0, 6, 10], (1, 2)),        # smallest difference 4 -> logGap 2, although gcd(6, 4) = 2
                       ([0, 12, 20], (1, 3)), ([3, 4, 100], (1, 0)), ([0, 5], (5, 0)), ([7], (0x7FFFFFFFFFFFFFFF, 0))):
        assert lb.ringpacking.getMinimumGap(keys) == ORP.getMinimumGap(keys) == want, keys
    for keys, msg in (([2, 1], "sorted"), ([1, 1], "duplicated")):
        with pytest.raises(ValueError, match=msg):
            lb.ringpacking.getMinimumGap(keys)
    # Pack with one key takes gap = N, logGap = LogN instead: without zeroing, logEnd = 0
    ctx = _ctx()
    gks, _keep = _keys(_all_keys(_params()))
    assert "smaller than inputLogGap" in _pack(ctx, gks, [0], LOGN, False)[1]
    assert "host-only" in _pack(ctx, gks, [0], LOGN, True)[1]
    ctx.close()


def _oracle_asked(fn):
    params = O.Parameters(LOGN, H.Qi60[:2], H.Pi60[:1])
    rng = np.random.default_rng(5)
    keys = {g: H.random_gadget_ciphertext(params, 1, 0, rng) for g in _all_keys(params)}
    ev = ORP.RingPackingEvaluator(params, keys, keys)
    ct = [H.rand_poly(params.qi, N, rng) for _ in range(2)]
    fn(ev, ct)
    return sorted(set(ev.asked))


@pytest.mark.parametrize("case", [("expand", 8), ("expand", 5), ("pack", ([1, 3], 8, True)), ("pack", ([0, 5, 6], 3, True)),
                                  ("pack", ([2], 8, True)), ("pack", ([0, 1, 2, 3], 2, False)), ("pack", ([4, 8, 300], 4, False))])
def test_keys_looked_up_equal_the_oracles(case):
    """Every key the restatement asks for is looked up by the call (dropping it is reported by name) and no other one is needed."""
    kind, arg = case
    if kind == "expand":
        asked = _oracle_asked(lambda ev, ct: ev.Expand(ct, arg))
        call = lambda ctx, gks: _expand(ctx, gks, arg, level=1)                                     # noqa: E731
    else:
        idx, ilg, zero = arg
        asked = _oracle_asked(lambda ev, ct: ev.Pack({k: ct for k in idx}, ilg, zero))
        call = lambda ctx, gks: _pack(ctx, gks, idx, ilg, zero, level=1)                            # noqa: E731
    ctx = _ctx()
    gks, _keep = _keys(asked, levelQ=3, levelP=1)
    assert "host-only" in call(ctx, gks)[1]
    for g in asked:
        gks, _keep = _keys([x for x in asked if x != g])
        assert call(ctx, gks)[1] == "GaloisKey[%d] is missing" % g
    ctx.close()


class _FakeKey:
    """Stands in for a GadgetCiphertext: the evaluator only reads .struct, whose pointers the key object owns."""

    def __init__(self, addr):
        self._sizes = (ctypes.c_int * 4)(1, 1, 1, 1)
        import lattigo_b200 as lb
        self.struct = lb._lib.GadgetCtStruct(ctypes.c_void_p(addr), 3, 1, 0, 2, 1, self._sizes)


def test_evaluator_keeps_its_keys_alive():
    """The key structs point into memory the key objects own, so an evaluator built from a temporary dict holds the keys."""
    import lattigo_b200 as lb
    ctx = _ctx()
    keys = {g: _FakeKey(FAKE + 256 * i) for i, g in enumerate(ORP.GaloisElementsForExpand(_params(), LOGN))}
    refs = [weakref.ref(k) for k in keys.values()]
    ev = lb.ringpacking.RingPackingEvaluator(ctx, keys, dict(keys))
    del keys
    gc.collect()
    assert all(r() is not None for r in refs)
    assert "host-only" in _expand(ctx, ev._extract.gks, 8)[1]     # every key found and its descriptor intact
    del ev
    gc.collect()
    assert all(r() is None for r in refs)
    ctx.close()

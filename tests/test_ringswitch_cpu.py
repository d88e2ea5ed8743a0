"""lgpu_evaluator_apply_evaluation_key argument checks on a host-only context (no device work: the key descriptor and the
ciphertexts carry placeholder addresses that are never dereferenced)."""
import ctypes

import pytest

from tests.test_innersum_cpu import FAKE, LOGN, _ctx


def _key(levelQ=3, levelP=1, pw2=0, nd=None, addr=FAKE):
    import lattigo_b200 as lb
    nd = (levelQ + levelP + 1) // (levelP + 1) if nd is None else nd
    return lb._lib.GadgetCtStruct(ctypes.c_void_p(addr), levelQ, levelP, pw2, nd, 1, None)


def _apply(ctx, log_in, log_out, key=None, level_in=3, level_out=3, is_ntt=1, ct_in=FAKE, ct_out=FAKE << 8, batch=1):
    import lattigo_b200 as lb
    key = _key() if key is None else key
    rc = lb.lib().lgpu_evaluator_apply_evaluation_key(ctx.h, ctypes.c_void_p(ct_in), log_in, level_in, is_ntt, ctypes.byref(key),
                                                      ctypes.c_void_p(ct_out), log_out, level_out, batch, None)
    return rc, lb.lib().lgpu_last_error().decode()


def test_error_paths_on_a_host_only_context():
    ctx = _ctx()
    device_only = "host-only"
    # every valid call reaches the device check last
    for log_in, log_out in ((LOGN, LOGN), (LOGN, LOGN - 1), (LOGN - 3, LOGN), (LOGN, 4)):
        for is_ntt in (0, 1):
            rc, msg = _apply(ctx, log_in, log_out, is_ntt=is_ntt)
            assert rc != 0 and device_only in msg, (log_in, log_out, msg)
    assert _apply(ctx, LOGN - 1, LOGN + 1)[1] == "cannot ApplyEvaluationKey: opOut ring degree does not match evaluator params ring degree"
    assert _apply(ctx, LOGN + 1, LOGN - 1)[1] == "cannot ApplyEvaluationKey: ctIn ring degree does not match evaluator params ring degree"
    assert "does not match evaluator params ring degree" in _apply(ctx, LOGN - 1, LOGN - 1)[1]
    assert "powers of two in [2^4" in _apply(ctx, LOGN, 3)[1]
    assert "powers of two in [2^4" in _apply(ctx, 3, LOGN)[1]
    for lv in ((-1, 3), (3, 4), (4, 3)):
        assert _apply(ctx, LOGN, LOGN, level_in=lv[0], level_out=lv[1])[1] == "level out of range"
    assert "is_ntt" in _apply(ctx, LOGN, LOGN, is_ntt=2)[1]
    assert "batch" in _apply(ctx, LOGN, LOGN, batch=0)[1]
    assert "aligned" in _apply(ctx, LOGN, LOGN, ct_out=(FAKE << 8) + 8)[1]
    assert "null ciphertext" in _apply(ctx, LOGN, LOGN, ct_in=0)[1]
    # overlaps: in place only at the same degree and level
    N = 1 << LOGN
    assert device_only in _apply(ctx, LOGN, LOGN, ct_out=FAKE)[1]
    assert "overlaps" in _apply(ctx, LOGN, LOGN, ct_out=FAKE, level_out=2)[1]
    assert "overlaps" in _apply(ctx, LOGN, LOGN, ct_out=FAKE + 2 * 4 * N * 8 - 16)[1]
    assert "overlaps" in _apply(ctx, LOGN, LOGN - 1, ct_out=FAKE)[1]
    assert "overlaps" in _apply(ctx, LOGN - 1, LOGN, ct_out=FAKE + 16)[1]
    assert device_only in _apply(ctx, LOGN, LOGN, ct_out=FAKE + 2 * 4 * N * 8)[1]
    # keys lgpu_gadget_product rejects
    assert "null evaluation key" in _apply(ctx, LOGN, LOGN, key=_key(addr=0))[1]
    assert "levelQ out of range for this evaluation key" in _apply(ctx, LOGN, LOGN, key=_key(levelQ=2))[1]
    assert device_only in _apply(ctx, LOGN, LOGN, key=_key(levelQ=2), level_in=2, level_out=3)[1]
    assert "fewer digits" in _apply(ctx, LOGN, LOGN, key=_key(nd=1))[1]
    assert "BaseTwoDecomposition" in _apply(ctx, LOGN, LOGN, key=_key(pw2=16))[1]
    assert device_only in _apply(ctx, LOGN, LOGN, key=_key(levelP=0, pw2=16, nd=4))[1]
    assert device_only in _apply(ctx, LOGN, LOGN, key=_key(levelP=-1, nd=4))[1]
    assert "evaluation key levels out of range" in _apply(ctx, LOGN, LOGN, key=_key(levelP=2))[1]


def test_conjugate_invariant_context_switches_no_degree():
    ctx = _ctx(ring_type=1)
    assert "host-only" in _apply(ctx, LOGN, LOGN)[1]
    for log_in, log_out in ((LOGN, LOGN - 1), (LOGN - 1, LOGN)):
        assert "only supported for ring.Type = ring.Standard" in _apply(ctx, log_in, log_out)[1]


def test_python_wrapper_checks_shapes():
    import lattigo_b200 as lb
    ctx = _ctx()

    class T:                      # shape-only stand-in: the wrapper rejects it before touching memory
        def __init__(self, *shape):
            self.shape = shape

        def dim(self):
            return len(self.shape)

    ev = lb.Evaluator(ctx)
    with pytest.raises(ValueError, match="not a power of two"):
        ev.ApplyEvaluationKey(T(2, 4, 96), None, T(2, 4, 1 << LOGN))
    with pytest.raises(ValueError, match="batch sizes differ"):
        ev.ApplyEvaluationKey(T(2, 2, 4, 1 << LOGN), None, T(3, 2, 4, 1 << LOGN))

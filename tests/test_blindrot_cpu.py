"""lgpu_blind_rotation_evaluate argument checks on host-only contexts (no device work: keys, test polynomials and ciphertexts carry
placeholder addresses that are never dereferenced)."""
import ctypes

from tests.test_innersum_cpu import FAKE

LOGN, LOGN_LWE, WINDOW = 8, 5, 4
Q = 0x7fff801


def _ctx(logN=LOGN, Qs=(Q,), ring_type=0):
    import lattigo_b200 as lb
    return lb.Context(logN, list(Qs), [], device=-1, ring_type=ring_type)


def _call(ctx, ctx_lwe, slots=(0, 3), n_brk=None, els=None, level_lwe=0, ct=FAKE, brk_level=0, window=WINDOW, is_ntt=1, ntt_out=1, batch=1):
    import lattigo_b200 as lb
    n_lwe = 1 << LOGN_LWE
    n_brk = n_lwe if n_brk is None else n_brk
    N = ctx.N
    if els is None:
        els = [pow(5, k, 2 * N) for k in range(1, window + 1)] + [2 * N - 5]
    key = lambda: lb._lib.GadgetCtStruct(ctypes.c_void_p(FAKE), brk_level, -1, 7, brk_level + 1, 4, None)
    b0 = (lb._lib.GadgetCtStruct * n_brk)(*[key() for _ in range(n_brk)])
    b1 = (lb._lib.GadgetCtStruct * n_brk)(*[key() for _ in range(n_brk)])
    arr = (ctypes.c_uint64 * max(1, len(els)))(*els)
    gk = (lb._lib.GadgetCtStruct * max(1, len(els)))(*[key() for _ in els])
    gks = lb._lib.GaloisKeysStruct(len(els), arr, gk)
    c_slots = (ctypes.c_int * len(slots))(*slots)
    polys = (ctypes.c_void_p * len(slots))(*[FAKE << 2 for _ in slots])
    rc = lb.lib().lgpu_blind_rotation_evaluate(ctx.h, ctx_lwe.h, ctypes.c_void_p(ct), level_lwe, is_ntt, c_slots, len(slots), polys, b0, b1,
                                               n_brk, ctypes.byref(gks), window, ntt_out, ctypes.c_void_p(FAKE << 4), batch, None)
    return rc, lb.lib().lgpu_last_error().decode()


def test_error_paths_on_a_host_only_context():
    ctx, lwe = _ctx(), _ctx(LOGN_LWE, (0x3001,))
    try:
        for is_ntt in (0, 1):
            for ntt_out in (0, 1):
                rc, msg = _call(ctx, lwe, is_ntt=is_ntt, ntt_out=ntt_out)
                assert rc != 0 and "host-only" in msg, msg                # every valid call reaches the device check last
        N = ctx.N
        g3 = pow(5, 3, 2 * N)
        assert _call(ctx, lwe, els=[e for e in [pow(5, k, 2 * N) for k in range(1, WINDOW + 1)] + [2 * N - 5] if e != g3])[1] == \
            "GaloisKey[%d] is missing" % g3
        assert _call(ctx, lwe, els=[pow(5, k, 2 * N) for k in range(1, WINDOW + 1)])[1] == "GaloisKey[%d] is missing" % (2 * N - 5)
        assert "fewer blind-rotation keys" in _call(ctx, lwe, n_brk=(1 << LOGN_LWE) - 1)[1]
        assert "duplicate slot" in _call(ctx, lwe, slots=(1, 2, 1))[1]
        assert "out of range" in _call(ctx, lwe, slots=(0, 1 << LOGN_LWE))[1]
        assert "out of range" in _call(ctx, lwe, slots=(-1,))[1]
        assert "above level 0" in _call(ctx, lwe, level_lwe=1)[1]
        assert "LWE ring degree is larger" in _call(_ctx(LOGN_LWE, (0x3001,)), ctx)[1]
        assert "aligned" in _call(ctx, lwe, ct=FAKE + 8)[1]
        assert "batch" in _call(ctx, lwe, batch=0)[1]
        assert "window" in _call(ctx, lwe, window=0, els=[2 * N - 5])[1]
        assert "no slot" in _call(ctx, lwe, slots=())[1]
        assert "level out of range" in _call(ctx, lwe, brk_level=1)[1]
        ci = _ctx(ring_type=1)
        assert "standard ring" in _call(ci, lwe)[1]
        ci.close()
    finally:
        ctx.close(); lwe.close()


def test_same_context_for_both_rings():
    ctx = _ctx(LOGN_LWE, (Q,))
    try:
        rc, msg = _call(ctx, ctx)
        assert rc != 0 and "host-only" in msg, msg
    finally:
        ctx.close()

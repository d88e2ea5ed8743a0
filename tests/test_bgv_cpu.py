"""lgpu_bgv_create's argument checks on a host-only context (no device work): the plaintext modulus, the QMul chain and the ring
type, as bgv.NewParameters rejects them (schemes/bgv/params.go:80-110), plus what the product adds (QMul disjoint from Q)."""
import pytest

from lattigo_b200 import params as presets
from oracle import oracle as O


def _ctx():
    import lattigo_b200 as lb
    s = presets.PRESETS["BGV_N15QP880"]
    return lb.Context(s["logN"], s["Q"], s["P"], device=-1), s


def _create(ctx, t, qmul):
    import ctypes
    import numpy as np
    import lattigo_b200 as lb
    a = np.array(qmul, dtype=np.uint64)
    h = ctypes.c_void_p()
    lb._lib.check(lb.lib().lgpu_bgv_create(ctx.h, t, a.ctypes.data if len(qmul) else None, len(qmul), ctypes.byref(h)))
    lb.lib().lgpu_bgv_destroy(h)


def test_bgv_create_accepts_the_preset():
    ctx, s = _ctx()
    _create(ctx, s["T"], s["QMul"])
    g = O.NTTFriendlyPrimesGenerator(61, 2 << s["logN"])
    longer = [g.NextDownstreamPrime() for _ in range(13)]
    assert longer[:12] == s["QMul"]
    _create(ctx, 2, longer)   # more QMul moduli than levelQMul needs are fine
    ctx.close()


@pytest.mark.parametrize("case", ["t_lt_2", "t_ge_q0", "t_in_Q", "qmul_in_Q", "qmul_short", "qmul_empty"])
def test_bgv_create_rejects(case):
    import lattigo_b200 as lb
    ctx, s = _ctx()
    t, qmul = s["T"], list(s["QMul"])
    if case == "t_lt_2":
        t = 1
    elif case == "t_ge_q0":
        t = s["Q"][0] + 2
    elif case == "t_in_Q":
        t = s["Q"][1]          # smaller than q_0
    elif case == "qmul_in_Q":
        qmul[3] = s["Q"][5]
    elif case == "qmul_short":
        qmul = qmul[:11]        # levelQMul[19] + 1 = 12
    elif case == "qmul_empty":
        qmul = []
    with pytest.raises(lb.LgpuError):
        _create(ctx, t, qmul)
    ctx.close()


def test_bgv_create_rejects_conjugate_invariant_ring():
    import lattigo_b200 as lb
    ctx = lb.Context(8, presets.QI60[:3], presets.PI60[:1], device=-1, ring_type=1)
    with pytest.raises(lb.LgpuError, match="Standard ring"):
        _create(ctx, 0x10001, presets.PI60[1:4])
    ctx.close()


def test_bgv_mulrelin_refuses_host_only_context():
    import ctypes
    import numpy as np
    import lattigo_b200 as lb
    ctx, s = _ctx()
    a = np.array(s["QMul"], dtype=np.uint64)
    h = ctypes.c_void_p()
    lb._lib.check(lb.lib().lgpu_bgv_create(ctx.h, s["T"], a.ctypes.data, len(a), ctypes.byref(h)))
    rc = lb.lib().lgpu_bgv_mulrelin_batch(h, 0, None, None, None, 0, 0, None, 1, None)
    assert rc != 0 and b"host-only" in lb.lib().lgpu_last_error()
    lb.lib().lgpu_bgv_destroy(h)
    ctx.close()

"""Smoke test of the bootstrapping op-trace replay (lattigo_b200/bootreplay.py, BASELINE config 5) on a reduced literal: every op kind of
the trace runs through the C ABI at N = 2^13 and the per-phase timing covers the four phases. (The replay measures device time on
synthetic operands; the arithmetic of each entry point is covered by its own parity test. For the lintrans ops, that test runs the
replay's own matrices and keys from this literal: tests/test_gpu_lintrans_shapes.py.)"""
import pytest

pytestmark = pytest.mark.gpu


def test_bootstrap_replay_runs_every_op_kind():
    import torch
    import lattigo_b200 as lb
    from lattigo_b200 import boottrace
    from lattigo_b200.bootreplay import BootstrapReplay
    from oracle import oracle as O
    logN = 13
    trace = boottrace.bootstrap_trace(logN=logN, residual_limbs=2, stc_depth=2, evalmod_limbs=9, cts_depth=2)
    top = 2 - 1 + 2 + 9 + 2
    q, p = O.gen_moduli(logN + 1, [60, 40] + [39] * 2 + [60] * 9 + [56] * 2, [61, 61, 61])
    assert len(q) == top + 1
    ctx = lb.Context(logN, q, p)
    try:
        g = torch.Generator(device="cuda"); g.manual_seed(1)
        rep = BootstrapReplay(ctx, 2, g, trace)
        n0 = lb.lib().lgpu_launch_count()
        ms, nops = rep.run()
        assert set(ms) == {"ModUp", "CoeffsToSlots", "EvalMod", "SlotsToCoeffs"} and all(v > 0 for v in ms.values())
        assert nops == len(trace) and {o["op"] for o in trace} >= {"keyswitch", "modup_centered", "gadget_product_hoisted", "lintrans", "rescale", "conjugate",
                                                                  "mulrelin_rescale", "mul_by_i"}
        assert lb.lib().lgpu_launch_count() - n0 > 100
    finally:
        ctx.close()


def test_modup_centered_matches_the_reference_loop():
    """lgpu_modup_centered against a literal numpy restatement of bootstrapping/evaluator.go:652-699."""
    import ctypes
    import numpy as np
    import torch
    import lattigo_b200 as lb
    from lattigo_b200 import _lib
    from oracle import oracle as O
    logN = 10
    q, p = O.gen_moduli(logN + 1, [60, 40, 39, 56], [61, 61])
    ctx = lb.Context(logN, q, p)
    try:
        N = 1 << logN
        rng = np.random.default_rng(3)
        x = rng.integers(0, q[0], (3, N), dtype=np.uint64)
        x[0, :4] = [0, q[0] >> 1, (q[0] >> 1) + 1, q[0] - 1]
        x[1, 0] = q[0] - q[1]                                   # negative multiple of q_1 -> written as q_1 by the reference
        d = ctx.to_device(x)
        for strict in (0, 1):
            oq = torch.zeros((3, 4, N), dtype=torch.int64, device="cuda"); op = torch.zeros((3, 2, N), dtype=torch.int64, device="cuda")
            _lib.check(_lib.lib().lgpu_modup_centered(ctx.h, ctypes.c_void_p(d.data_ptr()), 1, 3, 1, strict, ctypes.c_void_p(oq.data_ptr()),
                                                      ctypes.c_void_p(op.data_ptr()), 3, N, 4 * N, 2 * N, None))
            gq, gp = ctx.to_host(oq), ctx.to_host(op)
            neg = (x > (q[0] >> 1)) if strict else (x >= (q[0] >> 1))
            mag = np.where(neg, np.uint64(q[0]) - x, x)
            for i, m in list(enumerate(q))[1:]:
                t = mag % np.uint64(m)
                assert np.array_equal(gq[:, i], np.where(neg, np.uint64(m) - t, t)), (strict, i)
            assert not gq[:, 0].any()                            # rows below first_q are not written
            for i, m in enumerate(p):
                t = mag % np.uint64(m)
                assert np.array_equal(gp[:, i], np.where(neg, np.uint64(m) - t, t)), (strict, i)
        assert int(ctx.to_host(oq)[1, 1, 0]) == q[1]
    finally:
        ctx.close()

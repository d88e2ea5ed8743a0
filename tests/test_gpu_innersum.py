"""GPU parity of lgpu_evaluator_partial_traces_sum / lgpu_evaluator_trace (lattigo_b200/csrc/innersum.cu) and of the scheme
wrappers of lattigo_b200/innersum.py against oracle/innersum.py = core/rlwe/inner_sum.go, bit for bit. Keys and ciphertexts are
uniform residues (parity is over Z_q identities, as in test_gpu_lintrans.py)."""
import numpy as np
import pytest

from oracle import innersum as OI
from oracle import oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64


class _Env:
    def __init__(self, logN, q, p, seed):
        import lattigo_b200 as lb
        self.lb = lb
        self.params = O.Parameters(logN, q, p)
        self.ctx = lb.Context(logN, q, p)
        self.rng = np.random.default_rng(seed)
        self.keys_o, self.keys_d = {}, {}
        self.level, self.levelP = len(q) - 1, len(p) - 1

    def add_keys(self, els):
        for g in els:
            if g not in self.keys_o:
                gk = H.random_gadget_ciphertext(self.params, self.level, self.levelP, self.rng)
                self.keys_o[g] = gk
                self.keys_d[g] = self.lb.GadgetCiphertext(self.ctx, gk.data, self.level, self.levelP)

    def ct(self, batch, level=None):
        level = self.level if level is None else level
        q = self.params.qi[: level + 1]
        return np.stack([np.stack([H.rand_poly(q, self.params.N(), self.rng) for _ in range(2)]) for _ in range(batch)])

    def ev(self):
        return self.lb.innersum.Evaluator(self.ctx, self.keys_d)

    def oracle(self):
        return OI.Evaluator(self.params, self.keys_o)

    def close(self):
        self.ctx.close()


def _pts_els(params, offset, n):
    out = []
    i, j = 0, n
    while j > 1:
        if j & 1:
            out.append(params.GaloisElement((n - (n & ((2 << i) - 1))) * offset))
        out.append(params.GaloisElement((1 << i) * offset))
        i, j = i + 1, j >> 1
    return out


def _oracle_pts(env, ct, offset, n, is_ntt):
    ev = env.oracle()
    res = np.zeros_like(ct)
    for b in range(ct.shape[0]):
        out = [res[b, 0], res[b, 1]]
        ev.PartialTracesSum([ct[b, 0], ct[b, 1]], offset, n, out, is_ntt)
    return res


@pytest.fixture(scope="module")
def env8():
    e = _Env(8, *O.gen_moduli(9, [55, 45, 45, 45], [55, 55]), 7)
    yield e
    e.close()


@pytest.mark.parametrize("offset", [1, -1, 3, -4])
def test_partial_traces_sum_logN8_every_n(env8, offset):
    e = env8
    N = e.params.N()
    for n in list(range(1, 10)) + [16, N // 2]:
        e.add_keys(_pts_els(e.params, offset, n))
        for is_ntt in (True, False):
            ct = e.ct(1)
            d = e.ctx.to_device(ct)
            out = d.clone().zero_()
            e.ev().PartialTracesSum(d, offset, n, out, is_ntt)
            want = _oracle_pts(e, ct, offset, n, is_ntt)
            assert np.array_equal(e.ctx.to_host(out), want), (offset, n, is_ntt)


def test_partial_traces_sum_batch_inplace_and_lower_level(env8):
    e = env8
    for n, offset, is_ntt in ((7, 3, True), (5, -4, False), (2, 1, True), (3, -1, True), (8, 1, False), (9, 1, True)):
        e.add_keys(_pts_els(e.params, offset, n))
        for level in (e.level, e.level - 2):
            ct = e.ct(3, level)
            d = e.ctx.to_device(ct)
            out = d.clone().zero_()
            e.ev().PartialTracesSum(d, offset, n, out, is_ntt)
            got = e.ctx.to_host(out)
            assert np.array_equal(got, _oracle_pts(e, ct, offset, n, is_ntt)), (n, offset, is_ntt, level)
            for b in range(3):                                    # each element of the batch equals a single call
                one = d[b:b + 1].clone()
                e.ev().PartialTracesSum(one, offset, n, one, is_ntt)
                assert np.array_equal(e.ctx.to_host(one), got[b:b + 1])
            inpl = d.clone()                                      # in place on the whole batch
            e.ev().PartialTracesSum(inpl, offset, n, inpl, is_ntt)
            assert np.array_equal(e.ctx.to_host(inpl), got)


def test_replicate_and_rotate_and_add(env8):
    e = env8
    e.add_keys(_pts_els(e.params, -2, 5) + _pts_els(e.params, 2, 5))
    ct = e.ct(2)
    d = e.ctx.to_device(ct)
    out = d.clone()
    e.ev().Replicate(d, 2, 5, out)
    assert np.array_equal(e.ctx.to_host(out), _oracle_pts(e, ct, -2, 5, True))
    e.ev().RotateAndAdd(d, 2, 5, out)
    assert np.array_equal(e.ctx.to_host(out), _oracle_pts(e, ct, 2, 5, True))


def test_trace_every_log_n(env8):
    e = env8
    logN = e.params.logN
    for log_n in range(logN):
        e.add_keys(OI.GaloisElementsForTrace(e.params, log_n))
        for is_ntt in (True, False):
            ct = e.ct(2)
            d = e.ctx.to_device(ct)
            lvl_out = e.level - 1
            out = e.ctx.to_device(np.zeros((2, 2, lvl_out + 1, e.params.N()), dtype=U64))
            level = e.ev().Trace(d, log_n, out, is_ntt)
            assert level == lvl_out
            ev = e.oracle()
            got = e.ctx.to_host(out)
            for b in range(2):
                w = [np.zeros((lvl_out + 1, e.params.N()), dtype=U64) for _ in range(2)]
                ev.Trace([ct[b, 0], ct[b, 1]], log_n, w, is_ntt)
                assert np.array_equal(got[b, 0], w[0]) and np.array_equal(got[b, 1], w[1]), (log_n, is_ntt, b)
            inpl = d.clone()
            e.ev().Trace(inpl, log_n, inpl, is_ntt)
            ev2 = e.oracle()
            for b in range(2):
                w = [np.zeros((e.level + 1, e.params.N()), dtype=U64) for _ in range(2)]
                ev2.Trace([ct[b, 0], ct[b, 1]], log_n, w, is_ntt)
                g = e.ctx.to_host(inpl[b])
                assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), ("in place", log_n, is_ntt, b)
            tn = e.ev().TraceNew(d, log_n, is_ntt)
            assert np.array_equal(e.ctx.to_host(tn), e.ctx.to_host(inpl))


def test_doubling_step_is_one_fused_launch(env8):
    """n = 2: one doubling step. Its launches are those of DecomposeNTT and of the hoisted gadget product on the same shapes plus
    exactly one auto_add_kernel (the composed tail would be Add + index + 2 AutomorphismNTTWithIndex + 2 Add)."""
    import torch
    e = env8
    lb = e.lb
    e.add_keys(_pts_els(e.params, 1, 2))
    d = e.ctx.to_device(e.ct(3))
    out = torch.empty_like(d)
    ev = e.ev()
    rl = lb.Evaluator(e.ctx)
    total = H.launch_delta(lambda: ev.PartialTracesSum(d, 1, 2, out))
    dec = [None]
    n_dec = H.launch_delta(lambda: dec.__setitem__(0, rl.DecomposeNTT(e.level, e.levelP, e.levelP + 1, d[:, 1].contiguous(), True)))
    t0 = torch.empty((3, e.level + 1, e.params.N()), dtype=torch.int64, device=d.device)
    t1 = torch.empty_like(t0)
    n_gp = H.launch_delta(lambda: rl.GadgetProductHoisted(e.level, dec[0], e.keys_d[e.params.GaloisElement(1)], t0, t1))
    assert total == n_dec + n_gp + 1, (total, n_dec, n_gp)


def test_error_paths_launch_nothing(env8):
    import torch
    e = env8
    lb = e.lb
    d = e.ctx.to_device(e.ct(1))
    out = torch.empty_like(d)
    e.add_keys(_pts_els(e.params, 1, 7))
    keys = {g: k for g, k in e.keys_d.items() if g != e.params.GaloisElement(4)}
    ev = lb.innersum.Evaluator(e.ctx, keys)
    n0 = lb.lib().lgpu_launch_count()
    with pytest.raises(lb.LgpuError, match=r"GaloisKey\[%d\] is missing" % e.params.GaloisElement(4)):
        ev.PartialTracesSum(d, 1, 7, out)        # the key of the last lazy term: found missing before any launch
    for args in ((1, 0), (0, 3)):
        with pytest.raises(lb.LgpuError, match=r"partialtrace: invalid parameter \(n = 0 or batchSize = 0\)"):
            ev.PartialTracesSum(d, args[0], args[1], out)
    with pytest.raises(lb.LgpuError, match="GaloisKey"):
        lb.innersum.Evaluator(e.ctx, {}).Trace(d, 0, out)
    assert lb.lib().lgpu_launch_count() == n0
    ci = lb.Context(8, H.Qi60[:2], H.Pi60[:1], ring_type=1)
    try:
        dc = ci.to_device(np.zeros((1, 2, 2, 256), dtype=U64))
        with pytest.raises(lb.LgpuError, match="ConjugateInvariant"):
            lb.innersum.Evaluator(ci, {}).PartialTracesSum(dc, 1, 2, dc)
        with pytest.raises(lb.LgpuError, match="ConjugateInvariant"):
            lb.innersum.Evaluator(ci, {}).Trace(dc, 1, dc)
    finally:
        ci.close()


def test_logN14_fused_pipeline():
    """N = 2^14 with 8 Q and 3 P limbs: fused key-switch pipeline, persistent transforms and the fused ModDown + add of the
    non-power-of-two tail; batch 2."""
    q, p = O.gen_moduli(15, [56] + [45] * 7, [55] * 3)
    e = _Env(14, q, p, 3)
    try:
        e.add_keys(_pts_els(e.params, 1, 7) + OI.GaloisElementsForTrace(e.params, 11))
        ct = e.ct(2)
        d = e.ctx.to_device(ct)
        out = d.clone()
        e.ev().PartialTracesSum(d, 1, 7, out, False)
        assert np.array_equal(e.ctx.to_host(out), _oracle_pts(e, ct, 1, 7, False))
        e.ev().Trace(d, 11, out, True)
        ev = e.oracle()
        w = [np.zeros_like(ct[0, 0]) for _ in range(2)]
        ev.Trace([ct[0, 0], ct[0, 1]], 11, w, True)
        got = e.ctx.to_host(out)
        assert np.array_equal(got[0, 0], w[0]) and np.array_equal(got[0, 1], w[1])
    finally:
        e.close()


def test_bgv_inner_sum_N15_batch16():
    """BGV_N15QP880 at batch 16: InnerSum(1, N/2) is PartialTracesSum(1, N/2) (Slots() = N for BGV), and InnerSum(1, N) takes the
    RotateRows branch: PartialTracesSum(1, N/2) + Automorphism(NthRoot - 1) + Add. Ciphertext 0 is checked with the oracle
    and every ciphertext against a single-ciphertext call."""
    import torch
    from lattigo_b200 import params as presets
    P = presets.PRESETS["BGV_N15QP880"]
    e = _Env(15, P["Q"], P["P"], 11)
    try:
        N = e.params.N()
        e.add_keys(_pts_els(e.params, 1, N // 2) + [2 * N - 1])
        d = torch.empty((16, 2, e.level + 1, N), dtype=torch.int64, device="cuda:0")
        rows = H.rand_poly(e.params.qi, N, e.rng)
        for b in range(16):                                      # distinct ciphertexts built from a few uniform rows on the device
            d[b, 0] = torch.from_numpy(np.roll(rows, b, axis=1).view(np.int64)).cuda()
            d[b, 1] = torch.from_numpy(np.roll(rows, 3 * b + 1, axis=1).view(np.int64)).cuda()
        ct = e.ctx.to_host(d)
        ev = e.ev()
        half = torch.empty_like(d)
        ev.InnerSum(d, 1, N // 2, half, N, bgv=True)
        full = torch.empty_like(d)
        ev.InnerSum(d, 1, N, full, N, bgv=True)
        ho, fo = e.ctx.to_host(half), e.ctx.to_host(full)
        oe = e.oracle()
        for b in (0,):
            w = [np.zeros_like(ct[b, 0]) for _ in range(2)]
            oe.InnerSum([ct[b, 0], ct[b, 1]], 1, N // 2, w, N, bgv=True)
            assert np.array_equal(ho[b, 0], w[0]) and np.array_equal(ho[b, 1], w[1]), b
            oe.InnerSum([ct[b, 0], ct[b, 1]], 1, N, w, N, bgv=True)
            assert np.array_equal(fo[b, 0], w[0]) and np.array_equal(fo[b, 1], w[1]), b
        for b in range(16):
            one = d[b:b + 1].clone()
            ev.InnerSum(one, 1, N, one, N, bgv=True)
            assert torch.equal(one, full[b:b + 1]), b
    finally:
        e.close()


def test_ckks_average(env8):
    e = env8
    N = e.params.N()
    log_slots = e.params.logN - 1
    for logBatch in (0, 3):
        n = 1 << (log_slots - logBatch)
        e.add_keys(_pts_els(e.params, 1 << logBatch, n))
        ct = e.ct(2)
        d = e.ctx.to_device(ct)
        out = d.clone()
        e.ev().Average(d, logBatch, out, log_slots)
        ev = e.oracle()
        got = e.ctx.to_host(out)
        for b in range(2):
            w = [np.zeros((e.level + 1, N), dtype=U64) for _ in range(2)]
            ev.Average([ct[b, 0], ct[b, 1]], logBatch, w, log_slots)
            assert np.array_equal(got[b, 0], w[0]) and np.array_equal(got[b, 1], w[1]), (logBatch, b)
        with pytest.raises(ValueError):
            e.ev().Average(d, log_slots + 1, out, log_slots)

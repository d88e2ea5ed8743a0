"""GPU parity of lgpu_ring_packing_expand / lgpu_ring_packing_pack (lattigo_b200/csrc/ringpacking.cu) and of
lattigo_b200/ringpacking.py against oracle/ringpacking.py = core/rlwe/ring_packing.go, bit for bit. Keys and ciphertexts are
uniform residues (parity is over Z_q identities, as in test_gpu_innersum.py)."""
import ctypes

import numpy as np
import pytest

from oracle import oracle as O
from oracle import ringpacking as ORP
from tests import helpers as H
from tests.test_gpu_innersum import _Env

pytestmark = pytest.mark.gpu
U64 = np.uint64


class _RP(_Env):
    def __init__(self, logN, q, p, seed, levelP=None, pw2=0):
        super().__init__(logN, q, p, seed)
        self.keyP = self.levelP if levelP is None else levelP
        self.pw2 = pw2
        self.add_keys(ORP.GaloisElementsForExpand(self.params, logN) + ORP.GaloisElementsForPack(self.params, logN))

    def add_keys(self, els):
        for g in els:
            if g not in self.keys_o:
                gk = H.random_gadget_ciphertext(self.params, self.level, self.keyP, self.rng, pw2=self.pw2)
                self.keys_o[g] = gk
                self.keys_d[g] = self.lb.GadgetCiphertext(self.ctx, gk.data, self.level, self.keyP, self.pw2, gk.pw2_sizes)

    def rp(self, keys=None):
        k = self.keys_d if keys is None else keys
        return self.lb.ringpacking.RingPackingEvaluator(self.ctx, k, k)

    def orp(self):
        return ORP.RingPackingEvaluator(self.params, self.keys_o, self.keys_o)


def _check_expand(e, ct, logGap, is_ntt):
    """Device Expand of the batch ct against the oracle on entry 0; every entry against a single call."""
    d = e.ctx.to_device(ct)
    got = e.rp().Expand(d, logGap, is_ntt)
    want = e.orp().Expand([ct[0, 0], ct[0, 1]], logGap, is_ntt)
    assert sorted(got) == sorted(want)
    for j, w in want.items():
        g = e.ctx.to_host(got[j][0].contiguous())
        assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), (logGap, is_ntt, j)
    for b in range(1, ct.shape[0]):
        one = e.rp().Expand(d[b:b + 1].clone(), logGap, is_ntt)
        for j in got:
            assert np.array_equal(e.ctx.to_host(one[j].contiguous()), e.ctx.to_host(got[j][b:b + 1].contiguous())), (b, j)
    return got


def _check_pack(e, idx, ilg, zero, is_ntt, batch=1, level=None):
    """Device Pack against the oracle (entry 0) and single calls (every entry); errors where the oracle fails or returns nil."""
    lb = e.lb
    cts = e.ct(batch * len(idx), level).reshape(batch, len(idx), 2, -1, e.params.N())
    dev = {k: e.ctx.to_device(np.ascontiguousarray(cts[:, n])) for n, k in enumerate(idx)}
    try:
        want = e.orp().Pack({k: [cts[0, n, 0], cts[0, n, 1]] for n, k in enumerate(idx)}, ilg, zero, is_ntt)
    except ValueError:
        want = None
    if want is None:
        n0 = lb.lib().lgpu_launch_count()
        with pytest.raises(lb.LgpuError):
            e.rp().Pack(dev, ilg, zero, is_ntt)
        assert lb.lib().lgpu_launch_count() == n0
        return False
    got = e.rp().Pack(dev, ilg, zero, is_ntt)
    g = e.ctx.to_host(got)
    assert np.array_equal(g[0, 0], want[0]) and np.array_equal(g[0, 1], want[1]), (idx, ilg, zero, is_ntt)
    for b in range(1, batch):
        one = e.rp().Pack({k: v[b:b + 1].clone() for k, v in dev.items()}, ilg, zero, is_ntt)
        assert np.array_equal(e.ctx.to_host(one), g[b:b + 1]), (idx, ilg, zero, b)
    return True


@pytest.fixture(scope="module")
def env8():
    e = _RP(8, *O.gen_moduli(9, [55, 45, 45, 45], [55, 55]), 17)
    yield e
    e.close()


def test_expand_logN8_every_log_gap(env8):
    for logGap in range(9):
        for is_ntt in (True, False):
            _check_expand(env8, env8.ct(1), logGap, is_ntt)


@pytest.mark.parametrize("idx", [list(range(8)), [1, 3], [0, 5, 6], [2], [0], [0, 1, 2, 9, 17, 300], [3, 6, 9, 12, 15, 40], [-7, -1, 2, 4, 5]])
def test_pack_logN8_pair_cases(env8, idx):
    """Every inputLogGap (errors included) and both zeroGarbageSlots: dense sets, holes (a-only and b-only pairs), one index,
    indices >= 2^inputLogGap."""
    ok = 0
    for ilg in range(9):
        for zero in (True, False):
            ok += _check_pack(env8, idx, ilg, zero, is_ntt=(ilg + zero) % 2 == 0)
    assert ok > 0


def test_pack_logN8_dense_full_tree(env8):
    _check_pack(env8, list(range(256)), 8, True, True)
    _check_pack(env8, list(range(0, 256, 4)), 8, False, False)


def test_batches_at_a_lower_level(env8):
    e = env8
    for batch in (1, 3):
        _check_expand(e, e.ct(batch, e.level - 2), 5, True)
        _check_pack(e, [0, 5, 6], 3, True, False, batch=batch, level=e.level - 2)
        _check_pack(e, [1, 2, 7, 30], 8, True, True, batch=batch, level=e.level - 1)
        _check_pack(e, [-5, 0, 3, 6, 40], 3, True, False, batch=batch)        # the tree reads inputs 1..3 only


def test_pack_leaves_cts_in_untouched(env8):
    """lgpu_ring_packing_pack called on a stacked block directly: the block is unchanged after the call in both domains (the
    reference NTTs and rescales its inputs in place), including indices the tree does not read, and the result is the one the
    Python wrapper gives."""
    import torch
    e = env8
    lb = e.lb
    N, nq = e.params.N(), e.level + 1
    ev = e.rp()
    for is_ntt in (True, False):
        for idx, ilg in (([0, 1, 2, 3], 2), ([-1, 2, 5, 300], 3)):
            block = e.ctx.to_device(e.ct(2 * len(idx)).reshape(2, len(idx), 2, nq, N))
            before = block.clone()
            out = torch.empty((2, 2, nq, N), dtype=torch.int64, device=block.device)
            arr = (ctypes.c_int * len(idx))(*idx)
            lb._lib.check(lb.lib().lgpu_ring_packing_pack(e.ctx.h, e.level, ctypes.c_void_p(block.data_ptr()), 1 if is_ntt else 0, arr, len(idx), ilg,
                                                          1, ctypes.byref(ev._repack.gks), ctypes.c_void_p(out.data_ptr()), 2, None))
            torch.cuda.synchronize()
            assert torch.equal(block, before), (is_ntt, idx)
            want = ev.Pack({k: block[:, n] for n, k in enumerate(idx)}, ilg, True, is_ntt)
            assert torch.equal(out, want), (is_ntt, idx)


def test_expand_input_untouched_and_repack_of_extract(env8):
    e = env8
    ct = e.ct(2)
    d = e.ctx.to_device(ct)
    ev = e.rp()
    cts = ev.Extract(d, {i: True for i in range(0, 256, 16)}, is_ntt=False)
    assert np.array_equal(e.ctx.to_host(d), ct)
    out = ev.Repack({k: v.contiguous() for k, v in cts.items()})
    o = e.orp()
    want = o.Repack(o.Extract([ct[1, 0], ct[1, 1]], list(range(0, 256, 16)), is_ntt=False))
    g = e.ctx.to_host(out)
    assert np.array_equal(g[1, 0], want[0]) and np.array_equal(g[1, 1], want[1])


@pytest.mark.parametrize("levelP,pw2", [(0, 0), (0, 20), (0, None)])
def test_other_key_types(levelP, pw2):
    """Single-P keys, BaseTwoDecomposition keys, and (pw2 None) multiple-P keys below MaxLevelP."""
    q, p = O.gen_moduli(9, [55, 45, 45], [55, 55, 55])
    e = _RP(8, q, p, 23, levelP=1 if pw2 is None else levelP, pw2=pw2 or 0)
    try:
        _check_expand(e, e.ct(2), 4, True)
        _check_pack(e, [0, 3, 5, 6], 8, True, False, batch=2)
    finally:
        e.close()


@pytest.mark.parametrize("logN", [13, 14])
def test_fused_pipeline(logN):
    q, p = O.gen_moduli(logN + 1, [56] + [45] * 7, [55] * 3)
    e = _RP(logN, q, p, logN)
    try:
        _check_expand(e, e.ct(2), logN - 2, False)
        _check_pack(e, [0, 1, 2, 3], 2, True, True, batch=2)
        _check_pack(e, [0, 3], logN, False, False)
    finally:
        e.close()


def test_logN16():
    q, p = O.gen_moduli(17, [56, 45, 45], [55, 55])
    e = _RP(16, q, p, 16)
    try:
        _check_expand(e, e.ct(1), 14, True)
        _check_pack(e, [0, 1, 2, 3], 2, True, True)
    finally:
        e.close()


def test_error_paths_launch_nothing(env8):
    e = env8
    lb = e.lb
    d = e.ctx.to_device(e.ct(1))
    g = e.params.GaloisElement(1 << 3)
    keys = {k: v for k, v in e.keys_d.items() if k not in (g, e.params.N() + 1)}
    n0 = lb.lib().lgpu_launch_count()
    with pytest.raises(lb.LgpuError, match=r"GaloisKey\[%d\] is missing" % (e.params.N() + 1)):
        e.rp(keys).Expand(d, 3)
    with pytest.raises(lb.LgpuError, match=r"GaloisKey\[%d\] is missing" % g):
        e.rp(keys).Pack({k: d for k in range(64)}, 8, True)
    with pytest.raises(lb.LgpuError, match="out of range"):
        e.rp().Pack({0: d, 1: d}, 9, True)
    with pytest.raises(lb.LgpuError, match="slot 0"):
        e.rp().Pack({1: d, 3: d}, 8, False)
    assert lb.lib().lgpu_launch_count() == n0


def _mac_scopes(lb, fn):
    import torch
    L = lb.lib()
    nk = 16
    ms, by = (ctypes.c_double * nk)(), (ctypes.c_double * nk)()
    sc, kn = (ctypes.c_ulonglong * nk)(), (ctypes.c_ulonglong * nk)()
    torch.cuda.synchronize()
    L.lgpu_profile_read(ms, by, sc, kn)
    L.lgpu_profile_enable(1)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        L.lgpu_profile_enable(0)
    L.lgpu_profile_read(ms, by, sc, kn)
    return int(sc[4])                                # LGPU_KCLASS_MAC


def test_one_gadget_product_per_step_and_sub_batch(env8):
    """The MAC-class scopes of a call equal those of sum over steps of ceil(pairs * batch / batch_chunk()) gadget products: the
    key of a step is read once per sub-batch of batch_chunk() = 64 ciphertexts, not once per ciphertext."""
    import torch
    e = env8
    lb = e.lb
    N = e.params.N()
    rl = lb.Evaluator(e.ctx)
    key = e.keys_d[N + 1]
    per_gp = _mac_scopes(lb, lambda: rl.GadgetProduct(e.level, torch.zeros((3, e.level + 1, N), dtype=torch.int64, device="cuda:0"), key,
                                                       torch.empty((3, e.level + 1, N), dtype=torch.int64, device="cuda:0"),
                                                       torch.empty((3, e.level + 1, N), dtype=torch.int64, device="cuda:0")))
    assert per_gp > 0
    d = e.ctx.to_device(e.ct(3))
    for logGap in (0, 4):
        gap = 1 << logGap
        steps = [max(1, (1 << i) // gap) for i in range(e.params.logN)]
        want = sum(-(-(c * 3) // 64) for c in steps)
        assert _mac_scopes(lb, lambda: e.rp().Expand(d, logGap)) == want * per_gp, logGap
    cts = {k: d for k in range(0, 256, 2)}             # 128 inputs: steps of 64, 32, ..., 1 pairs (inputLogGap 8, no zeroing)
    want = sum(-(-(p * 3) // 64) for p in (64, 32, 16, 8, 4, 2, 1))
    assert _mac_scopes(lb, lambda: e.rp().Pack(cts, 8, False)) == want * per_gp

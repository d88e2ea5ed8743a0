"""GPU parity of lgpu_evaluator_apply_evaluation_key (lattigo_b200/csrc/ringswitch.cu) and rlwe.Evaluator.ApplyEvaluationKey
against oracle/ringswitch.py = core/rlwe/evaluator_evaluationkey.go + element.go, bit for bit, for every ciphertext of a batch.
Keys and ciphertexts are uniform residues (parity is over Z_q identities, as in test_gpu_ringpacking.py)."""
import ctypes

import numpy as np
import pytest

from oracle import oracle as O
from oracle import ringswitch as ORS
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64


class _Env:
    def __init__(self, logN, q, p, seed, ring_type=0):
        import lattigo_b200 as lb
        self.lb = lb
        self.params = O.Parameters(logN, q, p, "Standard" if ring_type == 0 else "ConjugateInvariant")
        self.ctx = lb.Context(logN, q, p, ring_type=ring_type)
        self.ev_o = O.Evaluator(self.params)
        self.ev_d = lb.Evaluator(self.ctx)
        self.rng = np.random.default_rng(seed)
        self.level, self.levelP = len(q) - 1, len(p) - 1

    def key(self, levelQ=None, levelP=None, pw2=0):
        levelQ = self.level if levelQ is None else levelQ
        levelP = self.levelP if levelP is None else levelP
        gk = H.random_gadget_ciphertext(self.params, levelQ, levelP, self.rng, pw2=pw2)
        return gk, self.lb.GadgetCiphertext(self.ctx, gk.data, levelQ, levelP, pw2, gk.pw2_sizes)

    def ct(self, batch, level, n, fill=None):
        q = self.params.qi[: level + 1]
        if fill == "qm1":
            return np.stack([np.stack([np.stack([np.full(n, x - 1, dtype=U64) for x in q])] * 2)] * batch)
        return np.stack([np.stack([H.rand_poly(q, n, self.rng) for _ in range(2)]) for _ in range(batch)])

    def close(self):
        self.ctx.close()


def _check(e, key, log_in, log_out, level_in, level_out, is_ntt, batch=1, in_place=False, fill=None, out_init="zero"):
    """Device ApplyEvaluationKey of a batch against the oracle on every entry. out_init: the contents of ct_out before the call."""
    lb = e.lb
    ko, kd = key
    n_in, n_out = 1 << log_in, 1 << log_out
    ct = e.ct(batch, level_in, n_in, fill)
    if in_place:
        out0 = ct
    elif out_init == "zero":
        out0 = np.zeros((batch, 2, level_out + 1, n_out), dtype=U64)
    else:
        out0 = e.ct(batch, level_out, n_out)
    want = out0.copy()
    for b in range(batch):
        opOut = [want[b, 0], want[b, 1]]
        ORS.ApplyEvaluationKey(e.ev_o, [ct[b, 0].copy(), ct[b, 1].copy()], ko, opOut, is_ntt)
    d_in = e.ctx.to_device(ct)
    d_out = d_in if in_place else e.ctx.to_device(out0)
    e.ev_d.ApplyEvaluationKey(d_in, kd, d_out, is_ntt)
    got = e.ctx.to_host(d_out)
    for b in range(batch):
        for k in range(2):
            assert np.array_equal(got[b, k], want[b, k]), (log_in, log_out, level_in, level_out, is_ntt, b, k)
    if not in_place:
        assert np.array_equal(e.ctx.to_host(d_in), ct)          # the input is never written
    return got


@pytest.fixture(scope="module")
def env10():
    e = _Env(10, *O.gen_moduli(11, [55, 45, 45, 45], [55, 55]), 10)
    yield e
    e.close()


@pytest.mark.parametrize("is_ntt", [True, False])
def test_logN10_all_directions(env10, is_ntt):
    e = env10
    key = e.key()
    L = e.level
    for batch in (1, 3):
        _check(e, key, 10, 10, L, L, is_ntt, batch)
        _check(e, key, 10, 9, L, L, is_ntt, batch)
        _check(e, key, 9, 10, L, L, is_ntt, batch)
        _check(e, key, 10, 7, L, L, is_ntt, batch)
        _check(e, key, 10, 4, L, L, is_ntt, batch)                 # gap 64: 32 lanes per output, two loads each
        _check(e, key, 6, 10, L, L, is_ntt, batch)
    # lower levels: ct_out below ct_in, and (same degree / NTT up) above it, where the rows above the result keep their contents
    _check(e, key, 10, 10, L, L - 2, is_ntt, 2)
    _check(e, key, 10, 9, L, L - 1, is_ntt, 2)
    _check(e, key, 9, 10, L, L - 1, is_ntt, 2)
    _check(e, key, 10, 10, L - 1, L, is_ntt, 2, out_init="random")
    if is_ntt:
        _check(e, key, 9, 10, L - 2, L, is_ntt, 2, out_init="random")


def test_in_place_and_coefficient_up_into_a_non_zero_output(env10):
    e = env10
    key = e.key()
    for is_ntt in (True, False):
        _check(e, key, 10, 10, e.level, e.level, is_ntt, 3, in_place=True)
        _check(e, key, 10, 10, e.level - 1, e.level - 1, is_ntt, 1, in_place=True)
    # SwitchCiphertextRingDegree upward writes only every gap-th coefficient: the others keep what ct_out held
    got = _check(e, key, 8, 10, e.level, e.level, False, 2, out_init="random")
    assert np.count_nonzero(got) > 0


@pytest.mark.parametrize("levelP,pw2", [(0, 0), (0, 20), (-1, 0), (0, None)])
def test_other_key_types(env10, levelP, pw2):
    """Single-P, BaseTwoDecomposition, no-P keys, and (pw2 None) a multiple-P key below MaxLevelP on a 3-prime P ring."""
    if pw2 is None:
        q, p = O.gen_moduli(11, [55, 45, 45, 45], [55, 55, 55])
        e = _Env(10, q, p, 3)
        key = e.key(levelP=1)
    else:
        e = env10
        key = e.key(levelP=levelP, pw2=pw2)
    try:
        for is_ntt in (True, False):
            _check(e, key, 10, 10, e.level, e.level, is_ntt, 2)
            _check(e, key, 10, 9, e.level, e.level, is_ntt, 2)
            _check(e, key, 9, 10, e.level, e.level, is_ntt, 2)
    finally:
        if e is not env10:
            e.close()


def test_conjugate_invariant_same_degree():
    q, p = O.gen_moduli(12, [55, 45, 45], [55, 55])
    e = _Env(10, q, p, 4, ring_type=1)
    try:
        key = e.key()
        for is_ntt in (True, False):
            _check(e, key, 10, 10, e.level, e.level, is_ntt, 2)
            _check(e, key, 10, 10, e.level, e.level, is_ntt, 1, in_place=True)
        with pytest.raises(e.lb.LgpuError, match="ring.Standard"):
            e.ev_d.ApplyEvaluationKey(e.ctx.to_device(e.ct(1, e.level, 1024)), key[1], e.ctx.to_device(e.ct(1, e.level, 512)))
    finally:
        e.close()


def test_fused_pipeline_logN14():
    """Every direction and domain on the fused key-switch pipeline, and the fused ModDown epilogue in each of them: the same-degree
    NTT case (and so the upward one, which key-switches ct_out in place) runs it once per component with c0 folded in, instead of
    the unfused per-component ModDown."""
    import torch
    e = _Env(14, *O.gen_moduli(15, [56] + [45] * 7, [55] * 3), 14)
    try:
        for key in (e.key(), e.key(levelP=0)):
            for is_ntt in (True, False):
                _check(e, key, 14, 13, e.level, e.level, is_ntt, 2)
                _check(e, key, 13, 14, e.level, e.level, is_ntt, 2)
                _check(e, key, 14, 14, e.level, e.level, is_ntt, 3)
                _check(e, key, 14, 14, e.level, e.level - 2, is_ntt, 1)
            _check(e, key, 14, 14, e.level, e.level, True, 2, in_place=True)
            _check(e, key, 14, 14, e.level, e.level, False, 2, in_place=True)
        kd = e.key()[1]
        nq = e.level + 1
        for log_in, log_out in ((14, 14), (13, 14), (14, 13)):
            d_in = e.ctx.to_device(e.ct(2, e.level, 1 << log_in))
            d_out = torch.zeros((2, 2, nq, 1 << log_out), dtype=torch.int64, device="cuda:0")
            for is_ntt in (True, False):
                assert _mac_scopes(e.lb, lambda: e.ev_d.ApplyEvaluationKey(d_in, kd, d_out, is_ntt), kclass=8) > 0, (log_in, log_out, is_ntt)
    finally:
        e.close()


def test_logN16_to_12_61bit_all_q_minus_1():
    """gap 16 with 61-bit rows and every input q - 1: the block sums exceed 2^64 unless reduced as they go."""
    e = _Env(16, *O.gen_moduli(17, [61, 61], [61]), 16)
    try:
        key = e.key()
        _check(e, key, 16, 12, e.level, e.level, True, 1, fill="qm1")
        _check(e, key, 16, 12, e.level, e.level, False, 1, fill="qm1")
    finally:
        e.close()


def test_error_paths_launch_nothing(env10):
    e = env10
    lb = e.lb
    _, kd = e.key()
    d10 = e.ctx.to_device(e.ct(1, e.level, 1024))
    d9 = e.ctx.to_device(e.ct(1, e.level, 512))
    d8 = e.ctx.to_device(e.ct(1, e.level, 256))
    n0 = lb.lib().lgpu_launch_count()
    with pytest.raises(lb.LgpuError, match="ctIn ring degree does not match"):
        e.ev_d.ApplyEvaluationKey(d9, kd, d8)
    with pytest.raises(lb.LgpuError, match="opOut ring degree does not match"):
        e.ev_d.ApplyEvaluationKey(d8, kd, d9)
    with pytest.raises(lb.LgpuError, match="overlaps"):
        e.ev_d.ApplyEvaluationKey(d10, kd, d10.view(-1)[: 2 * (e.level + 1) * 512].view(1, 2, e.level + 1, 512))   # inside ct_in
    _, low = e.key(levelQ=e.level - 1)
    with pytest.raises(lb.LgpuError, match="levelQ out of range"):
        e.ev_d.ApplyEvaluationKey(d10, low, d9)
    assert lb.lib().lgpu_launch_count() == n0


def _mac_scopes(lb, fn, kclass=4):
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
    return int(sc[kclass])                           # 4: LGPU_KCLASS_MAC, 8: LGPU_KCLASS_EPILOGUE


def test_one_gadget_product_per_sub_batch(env10):
    """The MAC-class scopes of a call are those of ceil(batch / batch_chunk()) gadget products (batch_chunk() = 64)."""
    import torch
    e = env10
    lb = e.lb
    N, nq = 1024, e.level + 1
    _, kd = e.key()
    per_gp = _mac_scopes(lb, lambda: e.ev_d.GadgetProduct(e.level, torch.zeros((3, nq, N), dtype=torch.int64, device="cuda:0"), kd,
                                                          torch.empty((3, nq, N), dtype=torch.int64, device="cuda:0"),
                                                          torch.empty((3, nq, N), dtype=torch.int64, device="cuda:0")))
    assert per_gp > 0
    for batch in (3, 65):
        for log_in, log_out in ((10, 10), (10, 9), (9, 10)):
            d_in = e.ctx.to_device(e.ct(batch, e.level, 1 << log_in))
            d_out = torch.zeros((batch, 2, nq, 1 << log_out), dtype=torch.int64, device="cuda:0")
            for is_ntt in (True, False):
                got = _mac_scopes(lb, lambda: e.ev_d.ApplyEvaluationKey(d_in, kd, d_out, is_ntt))
                assert got == -(-batch // 64) * per_gp, (batch, log_in, log_out, is_ntt)

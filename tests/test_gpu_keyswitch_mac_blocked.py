"""GPU parity of the batch-blocked key-switch MAC pass (K3) on the FP64 rows, `ks_chunk_mac_fp8r_bct_kernel` in
lattigo_b200/csrc/keyswitch_fused.cu: one CTA serves KS_BCT ciphertexts per evaluation-key load.

`gadget_product_multiple_p_fused` gives the first batch - batch % KS_BCT ciphertexts to the blocked kernel and the rest (all of
them below KS_BCT) to the one-ciphertext kernel `ks_chunk_mac_fp8r_kernel<1>`, which LGPU_K3_VARIANT=11 selects for the whole
batch. Every case of test_gpu_keyswitch_fused.py (A, B, C, D) runs its fused GadgetProducts at batch 1, KS_BCT - 1, KS_BCT,
KS_BCT + 1 and 64 at RL = logN - 12 in 1..4, and checks
  * the first and the last ciphertext against the oracle,
  * every ciphertext bit for bit against the one-ciphertext kernel (a subprocess under LGPU_K3_VARIANT=11: the switch is read
    once per process),
  * the MAC scopes and their kernel counts, and the launch count against the one-ciphertext kernel's at the same batch.
Run with -m gpu on an H100."""
import ctypes
import functools
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_keyswitch_fused import CASES, DEFAULT_CONFIG, _classes, _key, chain, product_fused

U64 = np.uint64
HERE = os.path.dirname(os.path.abspath(__file__))
BCT = 2                    # keyswitch_fused.cu: KS_BCT
BATCHES = tuple(sorted({1, BCT - 1, BCT, BCT + 1, 64} - {0}))
KCLASS_MAC = 4             # LGPU_KCLASS_MAC
KCLASSES = 9               # LGPU_KCLASS_COUNT


def _lb():
    import lattigo_b200 as lb
    return lb


# ---- the dispatch of the FP64-row K3, restated ------------------------------------------------------------------------------
def k3_fp_launches(batch):
    """(blocked launches, one-ciphertext launches) of the FP64-row MAC pass in the default configuration."""
    nb, tail = divmod(batch, BCT)
    return int(nb > 0), int(tail > 0)


def k3_cell(batch):
    return {(1, 0): "blocked", (1, 1): "blocked+tail", (0, 1): "unblocked"}[k3_fp_launches(batch)]


def gp_ops(name, logN):
    """The fused GadgetProducts of a case that have FP64 rows (the ones the blocked kernel serves)."""
    Q, P, ops = chain(name, logN)
    out = []
    for op in ops:
        if op[0] != "gp":
            continue
        _, levelQ, keyP, pw2 = op
        if product_fused(logN, levelQ + 1, keyP, pw2) and "fp" in _classes(Q[: levelQ + 1] + P[: keyP + 1], logN):
            out.append(op)
    return out


def predict_mac(logN, Q, P, op, batch):
    """(MAC scopes, MAC kernels) of one fused GadgetProduct: one scope per row class, the FP64 one with its blocked / tail split."""
    _, levelQ, keyP, _ = op
    cls = _classes(Q[: levelQ + 1] + P[: keyP + 1], logN)
    return len(cls), len(cls) - 1 + sum(k3_fp_launches(batch))


def test_dispatch_reaches_every_cell():
    """The batches reach the blocked kernel alone, the blocked kernel with a one-ciphertext tail and the one-ciphertext kernel
    alone, and every case has a fused GadgetProduct with FP64 rows at every RL (no GPU needed)."""
    assert {k3_cell(b) for b in BATCHES} == {"blocked", "blocked+tail", "unblocked"}
    assert k3_cell(1) == "unblocked" and k3_cell(BCT) == "blocked" and k3_cell(BCT + 1) == "blocked+tail"
    assert sum(k3_fp_launches(64)) == 1
    for logN, name in CASES:
        assert gp_ops(name, logN), (logN, name)
    assert {logN - 12 for logN, _ in CASES} == {1, 2, 3, 4}


# ---- device runs ------------------------------------------------------------------------------------------------------------
def _inputs(logN, name, op, batch):
    """Seeded uniform NTT-domain input of one (op, batch); the same words in every process."""
    Q, _, _ = chain(name, logN)
    _, levelQ, keyP, _ = op
    rng = np.random.default_rng([logN, ord(name), levelQ, keyP, batch])
    return np.stack([H.rand_poly(Q[: levelQ + 1], 1 << logN, rng) for _ in range(batch)])


class _Case:
    def __init__(self, logN, name):
        lb = _lb()
        self.logN, self.name = logN, name
        self.Q, self.P, _ = chain(name, logN)
        self.ctx = lb.Context(logN, self.Q, self.P)
        self.params = O.Parameters(logN, self.Q, self.P)
        self.ev = lb.Evaluator(self.ctx)
        self.keys = {}

    def key(self, keyP, pw2):
        if (keyP, pw2) not in self.keys:
            gk = _key(self.params, keyP, pw2, np.random.default_rng([self.logN, ord(self.name), keyP, pw2]))
            self.keys[(keyP, pw2)] = (gk, _lb().GadgetCiphertext(self.ctx, gk.data, gk.LevelQ(), gk.LevelP(), pw2, gk.pw2_sizes))
        return self.keys[(keyP, pw2)]

    def runner(self, op, cx):
        import torch
        _, levelQ, keyP, pw2 = op
        gk = self.key(keyP, pw2)[1]
        dcx = self.ctx.to_device(cx)

        def run():
            out = torch.zeros((2, cx.shape[0], levelQ + 1, 1 << self.logN), dtype=torch.int64, device="cuda")
            self.ev.GadgetProduct(levelQ, dcx, gk, out[0], out[1])
            return out
        return run

    def close(self):
        self.keys.clear()
        self.ctx.close()


def _digest(out):
    return hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()


def _digest_and_launches(run):
    """(sha256 of the output of run(), kernel launches of one call)."""
    return _digest(run()), H.launch_delta(run)


def digests(logN, name):
    """(sha256 of the output, launches) of every (op, batch) of one case, keyed by 'op/batch'."""
    c = _Case(logN, name)
    try:
        return {"%r/%d" % (op, b): _digest_and_launches(c.runner(op, _inputs(logN, name, op, b))) for op in gp_ops(name, logN) for b in BATCHES}
    finally:
        c.close()


@functools.lru_cache(maxsize=None)
def _one_ciphertext_digests():
    """digests() of every case under LGPU_K3_VARIANT=11, in one subprocess."""
    env = dict(os.environ, LGPU_K3_VARIANT="11")
    code = ("import json, sys; from tests.test_gpu_keyswitch_mac_blocked import CASES, digests; "
            "print(json.dumps({'%d-%s' % c: digests(*c) for c in CASES}))")
    r = subprocess.run([sys.executable, "-c", code], cwd=os.path.dirname(HERE), env=env, capture_output=True, text=True, timeout=3600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _mac_scopes(fn):
    """(MAC scopes, MAC kernels) of one call of fn()."""
    import torch
    L = _lb().lib()
    ms, by = (ctypes.c_double * KCLASSES)(), (ctypes.c_double * KCLASSES)()
    sc, kn = (ctypes.c_ulonglong * KCLASSES)(), (ctypes.c_ulonglong * KCLASSES)()
    torch.cuda.synchronize()
    L.lgpu_profile_read(ms, by, sc, kn)
    L.lgpu_profile_enable(1)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        L.lgpu_profile_enable(0)
    L.lgpu_profile_read(ms, by, sc, kn)
    return int(sc[KCLASS_MAC]), int(kn[KCLASS_MAC])


@pytest.mark.gpu
@pytest.mark.parametrize("logN,name", CASES, ids=["%d-%s" % c for c in CASES])
def test_blocked_mac_case(logN, name):
    """Each fused GadgetProduct of one case at every batch: the oracle on chosen ciphertexts, the one-ciphertext kernel on all
    of them (bit for bit), and (default configuration) the MAC scope / kernel counts and the launch count: the one-ciphertext
    kernel's plus the tail launch (batch > KS_BCT, odd)."""
    c = _Case(logN, name)
    try:
        got = {}
        ev_o = O.Evaluator(c.params)
        for op in gp_ops(name, logN):
            _, levelQ, keyP, pw2 = op
            gk_o = c.key(keyP, pw2)[0]
            for b in BATCHES:
                cx = _inputs(logN, name, op, b)
                run = c.runner(op, cx)
                out = run()
                what = "logN=%d %s %r batch %d" % (logN, name, op, b)
                host = c.ctx.to_host(out)
                for i in sorted({0, b - 1}):
                    want = [np.zeros((levelQ + 1, 1 << logN), dtype=U64) for _ in range(2)]
                    ev_o.GadgetProduct(levelQ, cx[i].copy(), gk_o, want)
                    for m in range(2):
                        assert np.array_equal(host[m, i], want[m]), "%s: ciphertext %d component %d differs from the oracle" % (what, i, m)
                got["%r/%d" % (op, b)] = (_digest(out), H.launch_delta(run))
                if DEFAULT_CONFIG:
                    assert _mac_scopes(run) == predict_mac(logN, c.Q, c.P, op, b), what
        ref = _one_ciphertext_digests()["%d-%s" % (logN, name)]
        bad = sorted(k for k in got if got[k][0] != ref[k][0])
        assert not bad, "outputs differ from the one-ciphertext kernel (LGPU_K3_VARIANT=11): %s" % bad
        if DEFAULT_CONFIG:
            for k in got:
                b = int(k.rsplit("/", 1)[1])
                assert got[k][1] - ref[k][1] == sum(k3_fp_launches(b)) - 1, (k, got[k][1], ref[k][1])
    finally:
        c.close()

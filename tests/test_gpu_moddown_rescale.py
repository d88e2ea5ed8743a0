"""GPU parity (bit-exact vs the oracle) of the relinearization tail with one rescale (composite.cu: mulrelin_tail), whose ModDown and
rescale share one K2 and one epilogue pass on the FP64-pipe rows below q_L when q_L itself is an FP64-pipe prime
(keyswitch_fused.cu: moddown_rescale_ntt_fused), and take the two stages otherwise.

Cases, at every ring degree of the fused pipeline (2^13 ... 2^16): q_L an FP64-pipe prime over FP64 rows only, over FP64 rows and an
integer q0, and at level 1 over the integer q0 alone (no merged rows); q_L an integer prime (the two stages); 2, 4 and 6 P primes
(the ModDown's NSMAX groups 4 and 8; one P prime takes no fused key switch). Inputs carry the float-`v` edge words of
test_gpu_keyswitch_fused.py and the key has 0 and q - 1 words in every row. In the default configuration every run also checks the
K2 / epilogue scope counts of the two stages (one per row class of Q[:level + 1] for the ModDown, of Q[:level] for the rescale).
LGPU_FUSED_RESCALE=0 selects the two stages everywhere; the switch test re-runs the file under it and compares the outputs of the
benchmark's ring (CKKS_L44: N = 2^16, 44 + 4 limbs, level 43) between the two configurations. That comparison runs in child
processes next to this one, whose stream-ordered pool keeps what earlier tests allocated, so it takes 4 pairs (about 3 GB) rather than
the benchmark's 64 (about 40 GB); the 64-pair sub-batch itself is checked pair by pair against the oracle by
test_gpu_headline_parity.py. The range of the merged K2 prologue at its edges is pinned by test_moddown_rescale_model_cpu.py. Run
with -m gpu on an H100."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_keyswitch_fused import _lb, _op_mrr
from tests.test_gpu_ntt_persist import fp_ok

HERE = os.path.dirname(os.path.abspath(__file__))
LOGNS = (13, 14, 15, 16)


def chain(name, logN):
    """(Q, P, levels) of one case; every level is a MulRelinRescaleNew with the key at MaxLevelP."""
    if name == "fp":          # FP64 rows only, 4 P primes
        Q, P = O.gen_moduli(logN + 1, [45] * 6, [55] * 4)
        levels = [5, 2]
    elif name == "q0":        # an integer q0 under FP64 rows, 2 P primes; level 1: q_L over q0 alone
        Q, P = O.gen_moduli(logN + 1, [56] + [45] * 5, [55] * 2)
        levels = [5, 1]
    elif name == "p6":        # 60-bit q0 under 40-bit rows, 6 P primes (NSMAX 8)
        Q = O.gen_moduli(logN + 1, [60] + [40] * 7, [])[0]
        P = H.Pi60[:6]
        levels = [7, 3]
    elif name == "intL":      # q_L a 56-bit integer prime (two stages), then an FP64 q_L over it
        Q, P = O.gen_moduli(logN + 1, [45] * 4 + [56, 45], [55] * 3)
        levels = [4, 5]
    else:
        raise ValueError(name)
    return list(Q), list(P), levels


NAMES = ("fp", "q0", "p6", "intL")


def test_cases_reach_both_paths():
    """Every case's levels put q_L on the side the comment says (no GPU needed)."""
    for logN in LOGNS:
        for name in NAMES:
            Q, P, levels = chain(name, logN)
            merged = [fp_ok(Q[lv], logN) for lv in levels]
            below = [[fp_ok(q, logN) for q in Q[:lv]] for lv in levels]
            if name == "intL":
                assert merged == [False, True]
            else:
                assert all(merged)
            if name == "fp":
                assert all(all(b) for b in below)
            if name in ("q0", "p6"):
                assert not below[0][0] and not below[1][0] and all(below[0][1:])
            if name == "q0":
                assert below[1] == [False]          # level 1: no FP64 row below q_L


@pytest.mark.gpu
@pytest.mark.parametrize("logN,name", [(l, n) for l in LOGNS for n in NAMES], ids=["%d-%s" % (l, n) for l in LOGNS for n in NAMES])
def test_mulrelin_rescale_vs_oracle(logN, name):
    """MulRelinRescaleNew on a batch of 2 against the oracle, every element, batch consistency and (default configuration) the scope
    counts of test_gpu_keyswitch_fused.predict."""
    lb = _lb()
    Q, P, levels = chain(name, logN)
    ctx = lb.Context(logN, Q, P)
    params = O.Parameters(logN, Q, P)
    rng = np.random.default_rng(1000 * logN + sum(map(ord, name)))
    keys = {}
    for level in levels:
        _op_mrr(lb, ctx, params, keys, logN, Q, P, ("mrr", level), rng)
    keys.clear()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("logN", (13, 16))
def test_bgv_mulrelin_rescale_vs_oracle(logN):
    """BGV MulRelin + Rescale (the same tail) on the q0 chain against the CPU restatement of schemes/bgv, every element."""
    from tests.test_gpu_bgv import Setup
    Q, P, levels = chain("q0", logN)
    s = Setup(logN, Q, P, 7 + logN)
    for level in levels:
        a, b = s.cts(level, 2), s.cts(level, 2)
        out = s.ctx.to_host(s.gpu(False, s.ctx.to_device(a), s.ctx.to_device(b), 1))
        for k in range(2):
            assert np.array_equal(out[k], s.oracle(False, a[k], b[k], 1)), (logN, level, k)


def _l44_digest(batch):
    """sha256 of MulRelinRescaleNew on the benchmark's ring (CKKS_L44, level 43) for `batch` seeded uniform pairs."""
    import torch
    from lattigo_b200 import params as presets
    from tests.test_gpu_headline_parity import _torch_rand_rows
    lb = _lb()
    s = presets.PRESETS["CKKS_L44"]
    logN, Q, P = s["logN"], list(s["Q"]), list(s["P"])
    N, nq = 1 << logN, len(Q)
    ctx = lb.Context(logN, Q, P)
    nd = O.Parameters(logN, Q, P).BaseRNSDecompositionVectorSize(nq - 1, len(P) - 1)
    g = torch.Generator(device="cuda").manual_seed(44)
    evk = _torch_rand_rows(N, Q + P, (nd, 1, 2), g)
    ev = lb.CKKSEvaluator(ctx, lb.GadgetCiphertext(ctx, evk, nq - 1, len(P) - 1))
    a, b = _torch_rand_rows(N, Q, (batch, 2), g), _torch_rand_rows(N, Q, (batch, 2), g)
    out = ev.MulRelinRescaleNew(a, b)
    return hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()


@pytest.mark.gpu
def test_switch_off_gives_the_same_outputs():
    """LGPU_FUSED_RESCALE=0 (read once per process, hence subprocesses): every case of this file against the oracle again, and the
    benchmark's ring (4 pairs) bit for bit equal to the default configuration's output."""
    env = dict(os.environ, LGPU_FUSED_RESCALE="0")
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_moddown_rescale.py"), "-m", "gpu", "-x", "-q",
                        "-k", "vs_oracle"], cwd=root, env=env, capture_output=True, text=True, timeout=3600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    code = "from tests.test_gpu_moddown_rescale import _l44_digest; print(_l44_digest(4))"
    digests = []
    for e in (dict(os.environ), env):
        r = subprocess.run([sys.executable, "-c", code], cwd=root, env=e, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
        digests.append(r.stdout.split()[-1])
    assert digests[0] == digests[1], digests

"""Kernel choice of every transform entry point (ntt.cu: transform), per row class: NTT, NTTLazy, INTT, INTTLazy and
NTTThenMulCoeffsMontgomery at N = 2^11 (no persistent kernels), 2^13 and 2^16 (persistent kernels) and 2^17 (no persistent
kernels, FP64 rows with a strided pass), on FP64-pipe rows (45-bit primes), integer rows without forward corrections (55-bit)
and with them (61-bit), and mixed rows; 63 and 64 limb-transforms for the whole launch and per row class; 16-byte aligned
buffers and buffers at an odd word offset; ringP (global limbs offset by nQ); and a ConjugateInvariant ring.

Each call runs once to warm up, once for the library's launch count and once under the event profiler for the scopes, kernels
and algorithmic bytes of the transform and coefficient-wise classes (no other class may show up); then its output is compared
with the oracle. tests/golden/ntt_dispatch.json holds what the library measured on an H100 for these calls under the default
setting and under LGPU_NTT_PERSIST=0, LGPU_NTT_PERSIST=1 and LGPU_NO_FP64_NTT=1 (read once per process, hence the
subprocesses of test_switches). The counts depend only on the host code that picks the kernels, so a change to it that
changes any of them must update the file on purpose. Run with -m gpu on an H100."""
import ctypes
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_ntt_persist import assert_same, fp_ok, fwd_mask

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ntt_dispatch.json")
KCLASSES = 9             # LGPU_KCLASS_COUNT
PINNED = (0, 1, 2)       # LGPU_KCLASS_NTT_FWD, NTT_INV, VECOP
SWITCHES = ("LGPU_NTT_PERSIST=0", "LGPU_NTT_PERSIST=1", "LGPU_NO_FP64_NTT=1")
OPS = ("NTT", "NTTLazy", "INTT", "INTTLazy", "NTTThenMulCoeffsMontgomery")
BITS = {"fp": 45, "nocorr": 55, "corr": 61}

# name: (Q row classes, P row classes, ring used (Q or P), batch, odd word offset, ConjugateInvariant)
SHAPES = {
    "fp_64": (["fp"] * 4, [], "Q", 16, False, False),
    "fp_63": (["fp"] * 3, [], "Q", 21, False, False),
    "nocorr_64": (["nocorr"] * 4, [], "Q", 16, False, False),
    "corr_63": (["corr"] * 3, [], "Q", 21, False, False),
    "mixed_64": (["fp"] * 4 + ["corr"] * 4, [], "Q", 8, False, False),       # 64 in all, 32 per class
    "mixed_63": (["fp"] * 3 + ["nocorr"] * 4, [], "Q", 9, False, False),
    "mixed_64_odd": (["fp"] * 4 + ["corr"] * 4, [], "Q", 8, True, False),
    "fp_63_odd": (["fp"] * 3, [], "Q", 21, True, False),
    "ringP_64": (["fp"] * 2, ["fp", "corr", "fp", "nocorr"], "P", 16, False, False),
    "ci_64": (["fp", "fp", "corr", "corr"], [], "Q", 16, False, True),
}
CASES = [(13, s) for s in SHAPES] + [(16, s) for s in SHAPES if s != "ci_64"] + \
        [(logN, s) for logN in (11, 17) for s in ("mixed_64", "mixed_64_odd", "nocorr_64")]


def setting():
    """The column of the golden file this process runs under."""
    on = [s for s in SWITCHES if os.environ.get(s.split("=")[0]) == s.split("=")[1]]
    assert len(on) <= 1, on
    return on[0] if on else "default"


def moduli(logN, classes, ci, skip=()):
    """Distinct NTT-friendly primes of the given classes (1 mod 4N for a ConjugateInvariant ring), none of `skip`."""
    need = {b: sum(BITS[c] == b for c in classes) + len(skip) for b in BITS.values()}
    pool = {b: [q for q in O.gen_moduli(logN + (2 if ci else 1), [b] * n, [])[0] if q not in skip] for b, n in need.items() if n}
    return [pool[BITS[c]].pop(0) for c in classes]


def shape_moduli(logN, name):
    qc, pc, _, _, _, ci = SHAPES[name]
    Q = moduli(logN, qc, ci)
    return Q, moduli(logN, pc, ci, skip=Q)


def classify(q, logN):
    return "fp" if fp_ok(q, logN) else ("corr" if fwd_mask(q, logN) else "nocorr")


class Shape:
    def __init__(self, logN, name):
        import torch
        import lattigo_b200 as lb
        qc, pc, which, self.batch, self.odd, ci = SHAPES[name]
        Q, P = shape_moduli(logN, name)
        self.ctx = lb.Context(logN, Q, P, ring_type=1 if ci else 0)
        self.ring = self.ctx.ringQ if which == "Q" else self.ctx.ringP
        self.mods = Q if which == "Q" else P
        self.oracle = O.Ring(1 << logN, self.mods, "ConjugateInvariant" if ci else "Standard")
        rng = np.random.default_rng(logN * 100 + list(SHAPES).index(name))
        shape = (self.batch, len(self.mods), 1 << logN)
        self.x = np.stack([H.rand_poly(self.mods, 1 << logN, rng) for _ in range(self.batch)])
        self.m = np.stack([H.rand_poly([(1 << 64) - 1] * len(self.mods), 1 << logN, rng) for _ in range(self.batch)])   # any uint64
        self.dx, self.dm, self.out = self.dev(self.x), self.dev(self.m), self.dev(np.zeros(shape, dtype=np.uint64))
        if self.odd:
            assert self.dx.data_ptr() % 16 == 8 and self.out.data_ptr() % 16 == 8
        torch.cuda.synchronize()

    def dev(self, a):
        """a on the device, at a word offset of 1 (8- but not 16-byte aligned) for the odd shapes."""
        import torch
        if not self.odd:
            return self.ctx.to_device(a)
        flat = torch.zeros(a.size + 1, dtype=torch.int64, device="cuda")
        view = flat[1:].view(*a.shape)
        view.copy_(self.ctx.to_device(a))
        return view

    def call(self, op):
        if op == "NTTThenMulCoeffsMontgomery":
            return lambda: self.ring.NTTThenMulCoeffsMontgomery(self.dx, self.dm, self.out)
        return lambda: getattr(self.ring, op)(self.dx, self.out)

    def want(self, op):
        out = np.empty_like(self.x)
        for b in range(self.batch):
            if op == "NTTThenMulCoeffsMontgomery":
                self.oracle.NTT(self.x[b], out[b])
                self.oracle.MulCoeffsMontgomery(out[b], self.m[b], out[b])
            else:
                getattr(self.oracle, op)(self.x[b], out[b])
        return out


def measure(fn):
    """[launches, scopes, kernels, algorithmic bytes] of one call of fn after a warm-up call, the last three per PINNED class."""
    import torch
    import lattigo_b200 as lb
    L = lb.lib()
    ms, by = (ctypes.c_double * KCLASSES)(), (ctypes.c_double * KCLASSES)()
    sc, kn = (ctypes.c_ulonglong * KCLASSES)(), (ctypes.c_ulonglong * KCLASSES)()
    fn()
    torch.cuda.synchronize()
    n0 = L.lgpu_launch_count()
    fn()
    torch.cuda.synchronize()
    launches = L.lgpu_launch_count() - n0
    L.lgpu_profile_read(ms, by, sc, kn)
    L.lgpu_profile_enable(1)
    try:
        fn()
        torch.cuda.synchronize()
    finally:
        L.lgpu_profile_enable(0)
    L.lgpu_profile_read(ms, by, sc, kn)
    assert all(sc[k] == 0 and kn[k] == 0 for k in range(KCLASSES) if k not in PINNED), list(sc)
    return [int(launches), [int(sc[k]) for k in PINNED], [int(kn[k]) for k in PINNED], [int(by[k]) for k in PINNED]]


def key(logN, name, op):
    return "%d/%s/%s" % (logN, name, op)


def observe(logN, name):
    """{key: measurement} of every op on one shape, each output checked against the oracle."""
    s = Shape(logN, name)
    got = {}
    for op in OPS:
        got[key(logN, name, op)] = measure(s.call(op))
        assert_same(s.ctx.to_host(s.out), s.want(op), "logN=%d %s %s" % (logN, name, op))
    s.ctx.close()
    return got


def expected():
    with open(GOLDEN) as f:
        return json.load(f)


def test_golden_covers_every_case():
    """Every (shape, op) has a measurement under every setting, and the shapes reach what they are named for."""
    want = {key(logN, name, op) for logN, name in CASES for op in OPS}
    exp = expected()
    assert set(exp) == {"default"} | set(SWITCHES)
    assert all(set(col) == want for col in exp.values())
    for name, (qc, pc, which, batch, _, _) in SHAPES.items():
        rows = qc if which == "Q" else pc
        assert len(rows) * batch == int(name.split("_")[1])
    for logN, name in CASES:
        Q, P = shape_moduli(logN, name)
        assert len(set(Q + P)) == len(Q + P)
        assert [classify(q, logN) for q in Q + P] == SHAPES[name][0] + SHAPES[name][1], (logN, name)


@pytest.mark.gpu
@pytest.mark.parametrize("logN,name", CASES, ids=["%d-%s" % c for c in CASES])
def test_dispatch(logN, name):
    exp = expected()[setting()]
    got = observe(logN, name)
    bad = {k: (v, exp[k]) for k, v in got.items() if v != exp[k]}
    assert not bad, "%s: (launches, scopes, kernels, bytes) measured vs expected: %r" % (setting(), bad)


@pytest.mark.gpu
@pytest.mark.parametrize("env", SWITCHES)
def test_switches(env):
    """test_dispatch under a switch that changes the kernel choice (read once per process, hence a subprocess)."""
    import subprocess
    import sys
    k, v = env.split("=")
    e = dict(os.environ, **{k: v})
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_ntt_dispatch.py"), "-m", "gpu", "-x", "-q",
                        "-k", "test_dispatch"], cwd=os.path.dirname(HERE), env=e, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]

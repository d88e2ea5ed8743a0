"""Launch mix of every caller of the NTT-domain ModDown (composite.cu: moddown_ntt), at a ring degree where the fused ModDown applies
(N = 2^13) and at one where it does not (N = 2^12): PartialTracesSum with n not a power of two (its ModDown(accQP) + ctInNTT tail),
same-degree ApplyEvaluationKey in the NTT domain with and without P (in place and not), a BSGS linear transformation (the hoisted
ModDown of each giant step), Evaluator.ModDown through the C ABI on one QP-stacked block and on separate tensors, CKKS MulRelin with
0, 1 (q_L an integer prime: two stages; q_L an FP64-pipe prime: merged) and 2 rescales, and BGV MulRelin.

Each call runs once to warm up, once for the library's launch count, and once under the event profiler for the scopes and kernels of
every kernel class (lgpu_kclass). EXPECTED holds what the library measured on an H100 for these calls; the outputs themselves are
checked against the oracle by the callers' own test files. The counts depend only on the host code that picks the kernels, so they
restate its dispatch: a change to it that changes any of them must update EXPECTED on purpose. Run with -m gpu on an H100."""
import ctypes

import pytest

from oracle import oracle as O
from tests import bgv_oracle as B
from tests.test_gpu_bgv import T
from tests.test_gpu_headline_parity import _torch_rand_rows
from tests.test_gpu_keyswitch_fused import _moddown_block

BATCH = 2
LOGNS = (13, 12)       # fused ModDown / unfused ModDown
KCLASSES = 9           # LGPU_KCLASS_COUNT

# (scopes per class, kernels per class, launch count) per (logN, case); classes: NTT_FWD, NTT_INV, VECOP, MODUP, MAC, TENSOR,
# AUTOMORPHISM, FUSED, EPILOGUE
EXPECTED = {
    (13, 'pts_n3'): ((6, 6, 1, 4, 3, 0, 1, 4, 4), (12, 12, 1, 4, 3, 0, 1, 4, 4), 42),
    (13, 'apply_p'): ((0, 4, 0, 3, 2, 0, 0, 6, 4), (0, 8, 0, 3, 2, 0, 0, 6, 4), 23),
    (13, 'apply_p_in_place'): ((0, 4, 0, 3, 2, 0, 0, 6, 4), (0, 8, 0, 3, 2, 0, 0, 6, 4), 23),
    (13, 'apply_no_p'): ((4, 2, 1, 4, 4, 0, 0, 0, 0), (8, 4, 1, 4, 4, 0, 0, 0, 0), 21),
    (13, 'apply_no_p_in_place'): ((4, 2, 1, 4, 4, 0, 0, 0, 0), (8, 4, 1, 4, 4, 0, 0, 0, 0), 21),
    (13, 'lintrans_bsgs'): ((6, 10, 5, 7, 8, 0, 4, 10, 6), (12, 20, 5, 7, 8, 0, 4, 10, 6), 75),
    (13, 'moddown_stacked'): ((0, 2, 0, 1, 0, 0, 0, 2, 2), (0, 4, 0, 1, 0, 0, 0, 2, 2), 9),
    (13, 'moddown_split'): ((2, 2, 2, 2, 0, 0, 0, 0, 0), (4, 4, 2, 2, 0, 0, 0, 0, 0), 12),
    (13, 'ckks_mulrelin'): ((0, 4, 0, 2, 2, 1, 0, 4, 2), (0, 8, 0, 2, 2, 1, 0, 4, 2), 19),
    (13, 'ckks_mulrelin_rescale_int_qL'): ((0, 6, 0, 2, 2, 1, 0, 6, 4), (0, 12, 0, 2, 2, 1, 0, 6, 4), 27),
    (13, 'ckks_mulrelin_rescale_fp_qL'): ((0, 6, 0, 2, 2, 1, 0, 6, 4), (0, 12, 0, 2, 2, 1, 0, 6, 4), 27),
    (13, 'ckks_mulrelin_rescale2'): ((4, 8, 14, 2, 2, 1, 0, 4, 2), (8, 16, 14, 2, 2, 1, 0, 4, 2), 49),
    (13, 'bgv_mulrelin'): ((0, 4, 0, 2, 2, 1, 0, 4, 2), (0, 8, 0, 2, 2, 1, 0, 4, 2), 19),
    (12, 'pts_n3'): ((10, 6, 7, 6, 3, 0, 1, 0, 0), (10, 6, 7, 6, 3, 0, 1, 0, 0), 34),
    (12, 'apply_p'): ((8, 4, 3, 4, 2, 0, 0, 0, 0), (8, 4, 3, 4, 2, 0, 0, 0, 0), 21),
    (12, 'apply_p_in_place'): ((8, 4, 3, 4, 2, 0, 0, 0, 0), (8, 4, 3, 4, 2, 0, 0, 0, 0), 21),
    (12, 'apply_no_p'): ((4, 2, 1, 4, 4, 0, 0, 0, 0), (4, 2, 1, 4, 4, 0, 0, 0, 0), 15),
    (12, 'apply_no_p_in_place'): ((4, 2, 1, 4, 4, 0, 0, 0, 0), (4, 2, 1, 4, 4, 0, 0, 0, 0), 15),
    (12, 'lintrans_bsgs'): ((22, 10, 9, 10, 8, 0, 4, 0, 0), (22, 10, 9, 10, 8, 0, 4, 0, 0), 66),
    (12, 'moddown_stacked'): ((2, 2, 2, 2, 0, 0, 0, 0, 0), (2, 2, 2, 2, 0, 0, 0, 0, 0), 8),
    (12, 'moddown_split'): ((2, 2, 2, 2, 0, 0, 0, 0, 0), (2, 2, 2, 2, 0, 0, 0, 0, 0), 8),
    (12, 'ckks_mulrelin'): ((8, 4, 4, 4, 2, 1, 0, 0, 0), (8, 4, 4, 4, 2, 1, 0, 0, 0), 23),
    (12, 'ckks_mulrelin_rescale_int_qL'): ((10, 6, 10, 4, 2, 1, 0, 0, 0), (10, 6, 10, 4, 2, 1, 0, 0, 0), 33),
    (12, 'ckks_mulrelin_rescale_fp_qL'): ((9, 6, 10, 4, 2, 1, 0, 0, 0), (9, 6, 10, 4, 2, 1, 0, 0, 0), 32),
    (12, 'ckks_mulrelin_rescale2'): ((12, 8, 16, 4, 2, 1, 0, 0, 0), (12, 8, 16, 4, 2, 1, 0, 0, 0), 43),
    (12, 'bgv_mulrelin'): ((8, 4, 4, 4, 2, 1, 0, 0, 0), (8, 4, 4, 4, 2, 1, 0, 0, 0), 23),
}


def _lb():
    import lattigo_b200 as lb
    return lb


def _moduli(logN):
    """4 Q primes (56-bit q0 and q_3, 45-bit between: an integer q_L at level 3, an FP64-pipe q_L at level 2) and 2 P primes."""
    Q, P = O.gen_moduli(logN + 1, [56, 45, 45, 56], [55, 55])
    return list(Q), list(P)


class Shape:
    def __init__(self, logN):
        import torch
        lb = _lb()
        self.logN, self.N = logN, 1 << logN
        self.Q, self.P = _moduli(logN)
        self.ctx = lb.Context(logN, self.Q, self.P)
        self.g = torch.Generator(device="cuda").manual_seed(logN)
        self.levelQ, self.levelP = len(self.Q) - 1, len(self.P) - 1

    def rows(self, mods, lead):
        return _torch_rand_rows(self.N, mods, lead, self.g)

    def key(self, levelP):
        lb = _lb()
        nd = self.levelQ + 1 if levelP < 0 else (self.levelQ + levelP + 1) // (levelP + 1)
        return lb.GadgetCiphertext(self.ctx, self.rows(self.Q + self.P[: levelP + 1], (nd, 1, 2)), self.levelQ, levelP)

    def galois(self, ks):
        lib = _lb().lib()
        return {int(lib.lgpu_galois_element(self.ctx.h, k)): self.key(self.levelP) for k in ks}

    def ct(self, level):
        return self.rows(self.Q[: level + 1], (BATCH, 2))


def _pts(s):
    from lattigo_b200 import innersum
    ev = innersum.Evaluator(s.ctx, s.galois([1, 2]))      # n = 3: the lazy term k = 2 and the doubling step 1
    ct, out = s.ct(s.levelQ), s.ct(s.levelQ)
    return lambda: ev.PartialTracesSum(ct, 1, 3, out)


def _apply(levelP, in_place):
    def make(s):
        ev = _lb().Evaluator(s.ctx)
        evk = s.key(levelP)
        ct = s.ct(s.levelQ)
        out = ct if in_place else s.ct(s.levelQ)
        return lambda: ev.ApplyEvaluationKey(ct, evk, out)
    return make


def _bsgs(s):
    from lattigo_b200 import lintrans
    ev = lintrans.Evaluator(s.ctx, s.galois([1, 2, 4]))    # baby step 1, giant steps 2 and 4
    diags = {k: s.rows(s.Q + s.P, ()) for k in range(6)}
    lt = lintrans.LinearTransformation(diags, s.levelQ, s.levelP, s.logN - 1, N1=2)
    ct, out = s.ct(s.levelQ), s.ct(s.levelQ)
    return lambda: ev.Evaluate(ct, lt, out)


def _moddown_stacked(s):
    import torch
    acc = torch.cat([s.rows(s.Q, (2, BATCH)), s.rows(s.P, (2, BATCH))], dim=2).contiguous()
    out = s.ct(s.levelQ)
    return lambda: _moddown_block(_lb(), s.ctx, s.levelQ, s.levelP, acc, out)


def _moddown_split(s):
    ev = _lb().Evaluator(s.ctx)
    aq = [s.rows(s.Q, (BATCH,)) for _ in range(2)]
    ap = [s.rows(s.P, (BATCH,)) for _ in range(2)]
    ct = [s.rows(s.Q, (BATCH,)) for _ in range(2)]
    return lambda: ev.ModDown(s.levelQ, s.levelP, aq[0], ap[0], aq[1], ap[1], ct[0], ct[1])


def _ckks(level, nb):
    def make(s):
        ev = _lb().CKKSEvaluator(s.ctx, s.key(s.levelP), levels_per_rescale=nb)
        a, b = s.ct(level), s.ct(level)
        return lambda: ev.MulRelinRescaleNew(a, b, rescale=nb > 0)
    return make


def _bgv(s):
    ev = _lb().BGVEvaluator(s.ctx, T, B.qmul_moduli(s.logN, s.Q), s.key(s.levelP))
    a, b = s.ct(s.levelQ), s.ct(s.levelQ)
    return lambda: ev.MulRelinNew(a, b)


CASES = {
    "pts_n3": _pts,
    "apply_p": _apply(1, False),
    "apply_p_in_place": _apply(1, True),
    "apply_no_p": _apply(-1, False),
    "apply_no_p_in_place": _apply(-1, True),
    "lintrans_bsgs": _bsgs,
    "moddown_stacked": _moddown_stacked,
    "moddown_split": _moddown_split,
    "ckks_mulrelin": _ckks(3, 0),
    "ckks_mulrelin_rescale_int_qL": _ckks(3, 1),
    "ckks_mulrelin_rescale_fp_qL": _ckks(2, 1),
    "ckks_mulrelin_rescale2": _ckks(3, 2),
    "bgv_mulrelin": _bgv,
}


def measure(fn):
    """(scopes per class, kernels per class, launch count) of one call of fn after a warm-up call."""
    import torch
    L = _lb().lib()
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
    return tuple(int(x) for x in sc), tuple(int(x) for x in kn), int(launches)


_shapes = {}


def _shape(logN):
    if logN not in _shapes:
        _shapes[logN] = Shape(logN)
    return _shapes[logN]


def observe(logN, name):
    return measure(CASES[name](_shape(logN)))


def test_cases_cover_both_sides():
    """The two ring degrees sit on either side of fz_applicable, and the CKKS cases' q_L on either side of the merged rescale."""
    from tests.test_gpu_keyswitch_fused import moddown_fused
    from tests.test_gpu_ntt_persist import fp_ok
    assert [moddown_fused(logN, 4, 2) for logN in LOGNS] == [True, False]
    Q, _ = _moduli(13)
    assert not fp_ok(Q[3], 13) and fp_ok(Q[2], 13)
    assert set(EXPECTED) == {(logN, name) for logN in LOGNS for name in CASES}


@pytest.mark.gpu
@pytest.mark.parametrize("logN,name", [(l, n) for l in LOGNS for n in CASES], ids=["%d-%s" % (l, n) for l in LOGNS for n in CASES])
def test_launch_mix(logN, name):
    got = observe(logN, name)
    assert got == EXPECTED[(logN, name)], "logN=%d %s: (scopes, kernels, launches) %r, expected %r" % (logN, name, got, EXPECTED[(logN, name)])

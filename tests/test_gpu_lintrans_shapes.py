"""The hoisted linear transformations (lgpu_lintrans_evaluate_many, lattigo_b200/csrc/lintrans.cu) at the shapes the
bootstrapping replay runs and on every branch of their driver, bit for bit against oracle/lintrans.py.

`predict` restates in Python what the host code of lintrans.cu decides for a (matrix, batch, primes) case: the inner
launches per giant step (kLtMaxTerms = 20 terms each, later launches accumulate onto the first), whether lt_inner_kernel
loops over the batch (grid z = min(batch, 8)), the groups of lt_hoisted_auto_kernel (kHoistB = 4 ciphertexts per thread,
grid z = min(16, groups)), where the giant-step loop reduces its lazy sum (max_lazy_terms) and whether the sum would
overflow a u64 without those reductions, the BSGS extremes, the naive evaluator with only the 0-th diagonal, and the fused
or unfused ModDown of the giant steps. `test_dispatch_reaches_every_cell` (no GPU) checks that CASES reach every cell of
REQUIRED and `test_dispatch_removing_a_case_leaves_a_cell` that each case is needed. The small cases run on primes near
2^61 (margin 4 of the lazy sums) with 0 and q - 1 words at fixed positions of every operand; `test_replay_matrices` runs
the matrices of the N = 2^13 replay literal at its batch of 64, and `test_boot16_matrices` one CoeffsToSlots and one
SlotsToCoeffs matrix of the N = 2^16 bootstrapping parameters. Run with -m gpu on an H100."""
import ctypes
import functools
from collections import namedtuple

import numpy as np
import pytest

from oracle import lintrans as LT
from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_keyswitch_fused import moddown_fused
from tests.test_gpu_lintrans import _oracle_many, _rand, _setup

U64 = np.uint64
KMAX_TERMS = 20            # lintrans.cu: kLtMaxTerms
INNER_ZMAX = 8             # lt_inner_kernel grid z = min(batch, 8)
KHOIST_B = 4               # lintrans.cu: kHoistB
HOIST_ZMAX = 16            # lt_hoisted_auto_kernel grid z = min(16, groups)
BATCHES = (1, 5, 9, 17, 64, 67)


# ---- the dispatch of lintrans.cu, restated -----------------------------------------------------------------------------------
def max_lazy_terms(moduli):
    """max_lazy_terms: min(QiOverflowMargin, PiOverflowMargin) >> 1 over the rows of the giant-step sum."""
    m = min((2 ** 64 - 1) // max(moduli), 1 << 20) >> 1
    return max(m, 1)


def reduce_points(n_giant, margin):
    """The giant steps (cnt0) after which multiply_bsgs reduces its lazy accumulator inside the loop."""
    pts, lazy = [], 0
    for cnt0 in range(n_giant):
        lazy = 0 if cnt0 == 0 else lazy + 1
        if lazy >= margin - 1 and lazy > 0:
            pts.append(cnt0)
            lazy = 0
    return pts


def hoist_cells(batch):
    """lt_hoisted_auto_kernel: groups of kHoistB ciphertexts, grid z = min(16, groups), z-loop over the rest."""
    groups = -(-batch // KHOIST_B)
    zb = max(1, min(HOIST_ZMAX, groups))
    cells = set()
    if groups > 1 and batch % KHOIST_B:
        cells.add(("hoist_partial_after_full",))
    if groups > zb:
        cells.add(("hoist_zloop",))
    if zb == HOIST_ZMAX and groups == zb and batch % KHOIST_B == 0:
        cells.add(("hoist_full_grid",))
    return cells


Case = namedtuple("Case", "name logN ring_type log_slots Q P levelP ct_level mats batches")


def predict_matrix(case, rots, N1, levelQ, batch):
    """Cells one matrix of a case reaches at one batch size."""
    logN, slots = case.logN, 1 << case.log_slots
    nq, np_ = min(levelQ, case.ct_level) + 1, case.levelP + 1
    ev = "bsgs" if N1 else "naive"
    cells = {("batch", ev, batch)}
    if not N1:
        keys = sorted(rots)
        rest = [k for k in keys if k & (slots - 1)]
        if keys == [0]:
            cells.add(("naive_diag0_only",))
        if len(rest) >= 16:
            cells.add(("naive_many",))
        if rest:
            cells |= hoist_cells(batch)
        return cells
    index, _, rotN2 = LT.bsgs_index(rots, slots, N1)
    if any(rotN2):
        cells |= hoist_cells(batch)
    if batch > INNER_ZMAX:
        cells.add(("inner_batch_loop",))
    if N1 == 1:
        cells.add(("N1=1",))
    if N1 >= slots:
        cells.add(("N1=slots",))
    cells.add(("j0",) if 0 in index else ("no_j0",))
    for j, babies in index.items():
        n = len(babies)
        if n in (KMAX_TERMS, KMAX_TERMS + 1, 2 * KMAX_TERMS):
            cells.add(("terms", n))
        if n > KMAX_TERMS:
            cells.add(("inner_split",))
        if 0 not in babies:
            cells.add(("no_i0",))
        if j:
            cells.add(("moddown_fused", logN - 12) if moddown_fused(logN, nq, np_) else ("moddown_unfused",))
    mods = list(case.Q[:nq]) + list(case.P[:np_])
    if reduce_points(len(index), max_lazy_terms(mods)):
        cells.add(("mid_reduce",))
    if len(index) * (max(mods) - 1) >= 2 ** 64:
        cells.add(("overflow_without_reduce",))
    return cells


def predict(case):
    cells = set()
    for rots, N1, levelQ in case.mats:
        for b in case.batches:
            cells |= predict_matrix(case, rots, N1, levelQ, b)
        if levelQ > case.ct_level:
            cells.add(("levelQ_above_ct",))
    if case.levelP < len(case.P) - 1:
        cells.add(("levelP_below_max",))
    if case.ring_type:
        cells.add(("conjugate_invariant",))
    elif case.log_slots < case.logN - 1:
        cells.add(("sparse_slots",))
    return cells


REQUIRED = ({("terms", n) for n in (KMAX_TERMS, KMAX_TERMS + 1, 2 * KMAX_TERMS)}
            | {("batch", ev, b) for ev in ("naive", "bsgs") for b in BATCHES}
            | {(c,) for c in ("inner_split", "inner_batch_loop", "hoist_partial_after_full", "hoist_zloop", "hoist_full_grid",
                              "mid_reduce", "overflow_without_reduce", "j0", "no_j0", "N1=1", "N1=slots", "no_i0",
                              "naive_diag0_only", "naive_many", "moddown_unfused", "levelP_below_max", "levelQ_above_ct",
                              "sparse_slots", "conjugate_invariant")}
            | {("moddown_fused", 1), ("moddown_fused", 4)})


# ---- the cases ----------------------------------------------------------------------------------------------------------------
Q61, P61 = H.Qi60, H.Pi60        # near 2^61: max_lazy_terms = 4, and 9 canonical terms overflow a u64
SMALL = [
    # giant steps of 40 (0..39), 21 (64..84) and 20 terms without baby step 0 (129..148): 2, 2 and 1 inner launches
    Case("term_split", 9, 0, 8, Q61[:3], P61[:2], 1, 2,
         [(list(range(40)) + list(range(64, 85)) + list(range(129, 149)), 64, 2)], (9,)),
    Case("bsgs_batches", 8, 0, 7, Q61[:3], P61[:2], 1, 2, [([1, 2, 5, 7, 9, 10, 14], 4, 2)], (1, 5, 17, 64, 67)),
    Case("naive_batches", 8, 0, 7, Q61[:3], P61[:2], 1, 2, [([0, 1, 3, 6, 100], 0, 2)], BATCHES),
    # every diagonal its own giant step: no pre-rotation, 20 giant steps of the i = 0 term P * ct alone
    Case("n1_one", 8, 0, 7, Q61[:3], P61[:2], 1, 2, [(list(range(20)), 1, 2)], (2,)),
    # 64 slots of 256: N1 = slots (one giant step, j = 0) and a naive matrix on masked rotations
    Case("n1_slots_sparse", 9, 0, 6, Q61[:3], P61[:2], 1, 2, [([0, 1, 2, 7, 63], 64, 2), ([3, 60], 0, 2)], (2,)),
    # the first giant step is j = 4: the non-accumulating automorphism at cnt0 = 0
    Case("no_diag0", 8, 0, 7, Q61[:3], P61[:2], 1, 2, [([5, 6, 9, 13, 14, 22], 4, 2)], (3,)),
    # matrix LevelP 1 of 3 P primes (keys at levelP 1), matrices at level 4 above a level-2 ciphertext
    Case("levels", 8, 0, 7, Q61[:5], P61[:3], 1, 2, [([0, 1, 2, 5, 6], 2, 4), ([0, 3, 7], 0, 4)], (2,)),
    Case("conjugate_invariant", 8, 1, 8, Q61[:3], P61[:2], 1, 2, [([0, 1, 2, 9, 17, 255], 8, 2), ([0, 1, 129], 0, 2)], (2,)),
    # naive with the 0-th diagonal alone, and naive with 24 diagonals
    Case("naive_edge", 8, 0, 7, Q61[:3], P61[:2], 1, 2, [([0], 0, 2), (list(range(0, 48, 2)), 0, 2)], (2,)),
]


REPLAY_LOGN = 13


@functools.lru_cache(maxsize=None)
def replay_literal():
    """(Q, P, trace) of the reduced N = 2^13 bootstrapping literal of tests/test_gpu_bootreplay.py."""
    from lattigo_b200 import boottrace
    trace = boottrace.bootstrap_trace(logN=REPLAY_LOGN, residual_limbs=2, stc_depth=2, evalmod_limbs=9, cts_depth=2)
    q, p = O.gen_moduli(REPLAY_LOGN + 1, [60, 40] + [39] * 2 + [60] * 9 + [56] * 2, [61, 61, 61])
    return tuple(q), tuple(p), tuple(o for o in trace if o["op"] == "lintrans")


@functools.lru_cache(maxsize=None)
def boot16():
    """(Q, P, [CoeffsToSlots op, SlotsToCoeffs op]) at N = 2^16 on BOOT_N16QP1767: of each phase, the matrix with the fewest
    rotation keys."""
    from lattigo_b200 import boottrace
    from lattigo_b200.params import PRESETS
    pr = PRESETS["BOOT_N16QP1767"]
    ops = [o for o in boottrace.bootstrap_trace(logN=16) if o["op"] == "lintrans"]

    def nkeys(o):
        _, r1, r2 = LT.bsgs_index(o["diags"], 1 << 15, o["N1"])
        return len({r for r in r1 + r2 if r})
    pick = [min((o for o in ops if o["phase"] == ph), key=nkeys) for ph in ("CoeffsToSlots", "SlotsToCoeffs")]
    return tuple(pr["Q"]), tuple(pr["P"]), tuple(pick)


def replay_case(name):
    if name == "replay13":
        Q, P, ops = replay_literal()
        logN = REPLAY_LOGN
    else:
        Q, P, ops = boot16()
        logN = 16
    mats = [(o["diags"], o["N1"], o["level"]) for o in ops]
    return Case(name, logN, 0, logN - 1, list(Q), list(P), len(P) - 1, max(o["level"] for o in ops), mats,
                (64,) if name == "replay13" else (2,))


CASES = SMALL + [replay_case("replay13"), replay_case("boot16")]


def reached_cells(cases):
    cells = set()
    for c in cases:
        cells |= predict(c)
    return cells


def test_dispatch_reaches_every_cell():
    """CASES reach every branch of the lintrans.cu driver listed in REQUIRED (no GPU needed)."""
    missing = REQUIRED - reached_cells(CASES)
    assert not missing, "cells no case reaches: %s" % sorted(missing, key=str)
    # the replay's own matrices: up to 16 giant steps on 61-bit P primes, which overflow a u64 without the mid-loop reduction
    rep = predict(replay_case("replay13"))
    assert {("mid_reduce",), ("overflow_without_reduce",), ("moddown_fused", 1)} <= rep
    assert max(len(LT.bsgs_index(r, 1 << 12, n1)[0]) for r, n1, _ in replay_case("replay13").mats) == 16
    assert reduce_points(20, 4) == [3, 6, 9, 12, 15, 18]


def test_dispatch_removing_a_case_leaves_a_cell():
    """Every case reaches some cell that no other case reaches, so dropping one fails the check above."""
    for case in CASES:
        rest = [c for c in CASES if c is not case]
        assert REQUIRED - reached_cells(rest), case.name


# ---- device runs --------------------------------------------------------------------------------------------------------------
def _check(ctx, got, want, level, what):
    g = ctx.to_host(got)
    bad = [b for b in range(g.shape[0]) if not all(np.array_equal(g[b, k, : level + 1], want[b][k][: level + 1]) for k in range(2))]
    assert not bad, "%s: batch elements %s differ from the oracle" % (what, bad[:16])


def _fill(shape, device, seed):
    """Receivers pre-filled with non-zero words: every result row must be written."""
    import torch
    g = torch.Generator(device=device); g.manual_seed(seed)
    return torch.randint(1, 1 << 62, shape, generator=g, device=device, dtype=torch.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in SMALL])
def test_branch_case(name):
    """Every small case on the device at each of its batch sizes, each batch element against the oracle. The naive_edge
    case's first matrix has only the 0-th diagonal: the reference ModDowns whatever its pooled buffers hold before adding
    diag0 * ct (lintrans_evaluator.go:254-273); the device defines that sum as zero, which is what the oracle computes from
    its zero-initialised receivers, so the device receivers start with non-zero words here."""
    case = next(c for c in SMALL if c.name == name)
    B = max(case.batches)
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(case.logN, None, None, case.mats, 17, batch=B, primes=(case.Q, case.P),
                                                 ring_type=case.ring_type, log_slots=case.log_slots, levelP=case.levelP,
                                                 edges=True, ct_level=case.ct_level)
    try:
        import torch
        N = params.N()
        ev = lb.lintrans.Evaluator(ctx, kd)
        levels_want = [min(lv, case.ct_level) for _, _, lv in case.mats]
        want = _oracle_many(params, ko, lo, ct, [case.ct_level] * len(case.mats))
        for b in case.batches:
            d_ct = ctx.to_device(ct[:b])
            outs = [_fill((b, 2, case.ct_level + 1, N), d_ct.device, 3 + i) for i in range(len(case.mats))]
            before = [o.clone() for o in outs]
            levels = ev.EvaluateMany(d_ct, ld, outs)
            assert levels == levels_want
            for i, (o, lv) in enumerate(zip(outs, levels)):
                _check(ctx, o, [w[i] for w in want[:b]], lv, "%s matrix %d batch %d" % (name, i, b))
                assert torch.equal(o[:, :, lv + 1:], before[i][:, :, lv + 1:])          # rows above the result level untouched
    finally:
        ctx.close()


def _mac_scopes(fn):
    """Runs fn() with the event profiler on; returns the number of LGPU_KCLASS_MAC scopes it opened."""
    import torch
    import lattigo_b200 as lb
    L = lb.lib()
    nk = 9
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
    return int(sc[4])                     # LGPU_KCLASS_MAC


@pytest.mark.gpu
def test_term_split_launches():
    """One giant step (j = 0) of 20, 21 and 40 baby steps: one MAC scope per pre-rotation (AutomorphismHoistedLazy) and one
    per lt_inner_kernel launch of at most 20 terms. 21 terms = one more pre-rotation and one more launch than 20; 40 terms =
    19 more pre-rotations and the same two launches as 21. Each result matches the oracle."""
    mats = [(list(range(n)), 64, 2) for n in (KMAX_TERMS, KMAX_TERMS + 1, 2 * KMAX_TERMS)]
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(9, None, None, mats, 29, batch=2, primes=(Q61[:3], P61[:2]), edges=True)
    try:
        import torch
        ev = lb.lintrans.Evaluator(ctx, kd)
        d_ct = ctx.to_device(ct)
        want = _oracle_many(params, ko, lo, ct, [2] * 3)
        scopes = []
        for i in range(3):
            out = torch.zeros_like(d_ct)
            scopes.append(_mac_scopes(lambda: ev.Evaluate(d_ct, ld[i], out)))
            _check(ctx, out, [w[i] for w in want], 2, "%d terms" % len(mats[i][0]))
        assert scopes[1] - scopes[0] == 2 and scopes[2] - scopes[1] == 19, scopes
    finally:
        ctx.close()


# ---- the replay's own matrices ------------------------------------------------------------------------------------------------
def _host_matrix(ctx, lt, levelQ):
    vec = {}
    for d, t in lt.Vec.items():
        h = ctx.to_host(t)
        vec[d] = (h[: levelQ + 1].copy(), h[levelQ + 1:].copy())
    return LT.LinearTransformation(vec, lt.LevelQ, lt.LevelP, lt.LogSlots, lt.N1)


def _host_keys(ctx, params, keys, rots, N1, levelP):
    """The Galois keys one BSGS matrix uses, pulled to the host."""
    _, r1, r2 = LT.bsgs_index(rots, params.N() >> 1, N1)
    out = {}
    for r in {x for x in r1 + r2 if x}:
        g = params.GaloisElement(r)
        gk = keys[g]
        out[g] = O.GadgetCiphertext(ctx.to_host(gk.data), gk.levelQ + 1, levelP + 1)
    return out


@pytest.fixture(scope="module")
def replay13():
    import torch
    import lattigo_b200 as lb
    from lattigo_b200.bootreplay import BootstrapReplay
    Q, P, ops = replay_literal()
    ctx = lb.Context(REPLAY_LOGN, list(Q), list(P))
    try:
        g = torch.Generator(device="cuda"); g.manual_seed(11)
        rep = BootstrapReplay(ctx, 64, g, [dict(o) for o in ops])
        yield ctx, rep, O.Parameters(REPLAY_LOGN, list(Q), list(P))
    finally:
        ctx.close()


SAMPLE = (0, 3, 4, 5, 31, 63)      # straddle the hoist groups of 4 and the inner kernel's 8 z-blocks


@pytest.mark.gpu
@pytest.mark.parametrize("op", range(4))
def test_replay_matrices(replay13, op):
    """Each lintrans op of the N = 2^13 replay trace (rep.lts, rep.lt_ev: its own diagonals and Galois keys) at batch 64:
    the SAMPLE elements against the oracle, and every element against the same ciphertext evaluated alone."""
    import torch
    ctx, rep, params = replay13
    ops = replay_literal()[2]
    assert len(ops) == len(rep.lts) == 4
    o, lt = ops[op], rep.lts[op]
    lvl = o["level"]
    rng = np.random.default_rng(40 + op)
    ct = np.stack([np.stack([H.rand_poly(ctx.Q[: lvl + 1], ctx.N, rng) for _ in range(2)]) for _ in range(rep.batch)])
    d_ct = ctx.to_device(ct)
    out = _fill(d_ct.shape, d_ct.device, 5)
    assert rep.lt_ev.Evaluate(d_ct, lt, out) == lvl
    for b in range(rep.batch):
        one = torch.zeros_like(d_ct[b:b + 1])
        rep.lt_ev.Evaluate(d_ct[b:b + 1].contiguous(), lt, one)
        assert torch.equal(one, out[b:b + 1]), (op, b)
    keys = _host_keys(ctx, params, rep.lt_ev.keys, o["diags"], o["N1"], rep.levelP)
    want = _oracle_many(params, keys, [_host_matrix(ctx, lt, lvl)], ct[list(SAMPLE)], [lvl])
    _check(ctx, out[list(SAMPLE)], [w[0] for w in want], lvl, "replay op %d (%s, %d diagonals, N1 = %d)" % (op, o["phase"], len(o["diags"]), o["N1"]))


@pytest.mark.gpu
@pytest.mark.parametrize("which", [0, 1], ids=["CoeffsToSlots", "SlotsToCoeffs"])
def test_boot16_matrices(which):
    """One matrix of each DFT phase of bootstrap_trace(logN = 16) on the BOOT_N16QP1767 primes, batch 2, every element
    against the oracle."""
    import lattigo_b200 as lb
    Q, P, ops = boot16()
    o = ops[which]
    lvl, levelP = o["level"], len(P) - 1
    params = O.Parameters(16, list(Q), list(P))
    ctx = lb.Context(16, list(Q), list(P))
    try:
        import torch
        N = params.N()
        rng = np.random.default_rng(70 + which)
        _, r1, r2 = LT.bsgs_index(o["diags"], N >> 1, o["N1"])
        ko, kd = {}, {}
        for r in sorted({x for x in r1 + r2 if x}):
            g = params.GaloisElement(r)
            ko[g] = H.random_gadget_ciphertext(params, lvl, levelP, rng)
            kd[g] = lb.GadgetCiphertext(ctx, ko[g].data, lvl, levelP)
        vo, vd = {}, {}
        for d in o["diags"]:
            dq, dp = H.rand_poly(Q[: lvl + 1], N, rng), H.rand_poly(P, N, rng)
            vo[d] = (dq, dp)
            vd[d] = ctx.to_device(np.concatenate([dq, dp]))
        lo = LT.LinearTransformation(vo, lvl, levelP, 15, o["N1"])
        ld = lb.lintrans.LinearTransformation(vd, lvl, levelP, 15, o["N1"])
        ct = np.stack([np.stack([H.rand_poly(Q[: lvl + 1], N, rng) for _ in range(2)]) for _ in range(2)])
        d_ct = ctx.to_device(ct)
        out = torch.zeros_like(d_ct)
        assert lb.lintrans.Evaluator(ctx, kd).Evaluate(d_ct, ld, out) == lvl
        _check(ctx, out, [w[0] for w in _oracle_many(params, ko, [lo], ct, [lvl])], lvl, o["phase"])
    finally:
        ctx.close()


# ---- argument errors ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_argument_errors_leave_the_context_usable():
    """Each argument error raises LgpuError with its message; a correct evaluation afterwards matches the oracle."""
    logN, slots = 8, 128
    mats = [([0, 1, 2, 5], 2, 2), ([1, 3], 0, 2)]
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(logN, None, None, mats, 41, batch=2, primes=(Q61[:3], P61[:2]), edges=True)
    try:
        import torch
        N = params.N()
        ev = lb.lintrans.Evaluator(ctx, kd)
        d_ct = ctx.to_device(ct)
        want = _oracle_many(params, ko, lo, ct, [2, 2])
        LTd = lb.lintrans.LinearTransformation
        rng = np.random.default_rng(5)

        def diag(levelP):
            return ctx.to_device(np.concatenate([_rand(params.qi, N, rng, True), _rand(params.pi[: levelP + 1], N, rng, True)]))

        def check_usable():
            outs = [torch.zeros_like(d_ct) for _ in mats]
            assert ev.EvaluateMany(d_ct, ld, outs) == [2, 2]
            for i in range(2):
                _check(ctx, outs[i], [w[i] for w in want], 2, "after an error, matrix %d" % i)

        low = LTd({1: diag(0), 3: diag(0)}, 2, 0, logN - 1, 0)
        with pytest.raises(lb.LgpuError, match="all linearTransformations must have the same levelP"):
            ev.EvaluateMany(d_ct, [ld[0], low], [torch.zeros_like(d_ct)] * 2)
        check_usable()
        # keys at levelP 1 for matrices at levelP 0, on both evaluators (pre-rotation / giant step and naive)
        for m in (low, LTd({0: diag(0), 1: diag(0), 2: diag(0), 5: diag(0)}, 2, 0, logN - 1, 2)):
            g = params.GaloisElement(1)
            with pytest.raises(lb.LgpuError, match=r"LinearTransformation\.LevelP = 0 != GaloiKey\[%d\]\.LevelP\(\) = 1: ensure that" % g):
                ev.Evaluate(d_ct, m, torch.zeros_like(d_ct))
            check_usable()
        with pytest.raises(lb.LgpuError, match="LinearTransformation.N1 must be a power of two"):
            ev.Evaluate(d_ct, LTd(ld[0].Vec, 2, 1, logN - 1, 3), torch.zeros_like(d_ct))
        check_usable()
        for ls in (logN, -1):
            with pytest.raises(lb.LgpuError, match="LinearTransformation.LogSlots out of range"):
                ev.Evaluate(d_ct, LTd(ld[0].Vec, 2, 1, ls, 2), torch.zeros_like(d_ct))
            check_usable()
        # a diagonal key >= slots: BSGS places it at its masked index, where no diagonal is stored
        bad = dict(ld[0].Vec)
        bad[slots + 4] = bad.pop(5)
        with pytest.raises(lb.LgpuError, match="LinearTransformation: diagonal 4 is missing"):
            ev.Evaluate(d_ct, LTd(bad, 2, 1, logN - 1, 2), torch.zeros_like(d_ct))
        check_usable()
    finally:
        ctx.close()

"""GPU parity (bit-exact vs the oracle) of the fused key-switch pipeline (lattigo_b200/csrc/keyswitch_fused.cu) at every
template instantiation it selects, with inputs at the edges of its float64 overflow count `v`.

Every key switch at 2^13 <= N <= 2^16 runs the pipeline: K1 `ks_prepare_kernel`, K2 `ks_strided_j4_kernel` /
`ks_strided_kernel` (the `PRO_BCAST` rescale prologue included), K3 `ks_chunk_mac_fp8r_kernel<1>` /
`ks_chunk_mac_int8r_kernel<CORR>`, and the fused ModDown / Rescale epilogues `fz_chunk_epi_{fp8,int8<CORR>}_kernel`.
`predict` restates in Python the host code that picks each of them; `test_dispatch_reaches_every_cell` (no GPU) checks
that CASES reaches every cell of REQUIRED at RL = logN - 12 in {1, 2, 3, 4}, and `test_fused_case` runs the cases on the
device against the oracle and checks the prediction through the profiler's K2 / epilogue scope counts.

Edge inputs (`digit_edges`): K1 computes the reference's `v = uint64(sum_i float64(y_i) / float64(q_i))`, which is not the
exact floor of sum_i y_i / q_i. Near X' = (X + floor(Q_d/2)) mod Q_d = Q_d - j it rounds up to v_exact + 1, and when every
y_i = q_i - 1 with all sources above 2^53 it is nS, which reads the last entry of the `vt` table. Uniform inputs reach
neither. Run with -m gpu on an H100."""
import ctypes
import functools
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_keyswitch import _gadget_case
from tests.test_gpu_ntt_persist import FWD_BOUND, fp_bound, fp_ok, fwd_mask, primes_below, primes_from

U64 = np.uint64
HERE = os.path.dirname(os.path.abspath(__file__))
LOGNS = (13, 14, 15, 16)
KMAX_DIGITS = 32           # keyswitch_fused.cu: kMaxDigits
KMAX_ROWS = 128            # engine.h: kMaxRows
K3 = {"fp": "fp8r<1>", "corr": "int8r<true>", "plain": "int8r<false>"}
FZ = {"fp": "fp8", "corr": "int8<true>", "plain": "int8<false>"}
# the path assertions restate the default configuration; a development switch changes it
DEFAULT_CONFIG = not any(k.startswith("LGPU_") for k in os.environ)


def _lb():
    import lattigo_b200 as lb
    return lb


# ---- the dispatch of keyswitch_fused.cu, restated --------------------------------------------------------------------------
def row_class(q, logN):
    """FP64-pipe row (fp_ok), integer row with the lazy-correction schedule (fwd_mask != 0: CORR) or plain integer row."""
    return "fp" if fp_ok(q, logN) else ("corr" if fwd_mask(q, logN) else "plain")


def product_fused(logN, nq, keyP, pw2):
    """ks_fused_applicable: multiple-P key without BaseTwoDecomposition, at most 64 Q rows, 32 digits and 6 P rows."""
    if not 13 <= logN <= 16 or keyP < 1 or pw2 != 0:
        return False
    k = keyP + 1
    return nq <= 64 and (nq + keyP) // k <= KMAX_DIGITS and k <= 6


def moddown_fused(logN, nq, np_):
    """fz_applicable."""
    return 13 <= logN <= 16 and nq <= KMAX_ROWS and 1 <= np_ <= 6


def digits(nq, k):
    """(first row, number of sources) of each digit: BaseRNSDecompositionVectorSize digits of k rows, the last one ragged."""
    return [(d * k, min(k, nq - d * k)) for d in range((nq + k - 1) // k)]


def _classes(qs, logN):
    return sorted({row_class(q, logN) for q in qs})


def predict_product(logN, Q, P, nq, keyP):
    """Cells of gadget_product_multiple_p_fused and its number of K2 scopes (one K2 + one K3 launch per row class). A K2 cell
    counts only when some (digit, target row) of that class is computed: the digit's own rows are skipped."""
    RL, k = logN - 12, keyP + 1
    dg = digits(nq, k)
    ns = 4 if max(s for _, s in dg) <= 4 else 8
    j4 = all(s > 1 for _, s in dg)          # a single-limb digit anywhere in the launch takes the plain kernel
    rows = [(r, Q[r]) for r in range(nq)] + [(None, p) for p in P[:k]]
    cells = set()
    for cls in _classes([q for _, q in rows], logN):
        cells.add(("k3", RL, K3[cls]))
        for r0, s in dg:
            if not any(row_class(q, logN) == cls and (r is None or not r0 <= r < r0 + s) for r, q in rows):
                continue
            if not j4:
                cells.add(("k2_plain", RL, ns, cls))
            elif cls == "fp" and ns == 4:
                split = s == ns and all(fp_ok(q, logN) for q in Q[r0:r0 + s])
                cells.add(("k2_j4", RL, 4, "fp", split))
            else:
                cells.add(("k2_j4", RL, ns, cls, None))
    return cells, len(_classes([q for _, q in rows], logN))


def predict_moddown(logN, Q, nq, np_, with_d):
    """moddown_ntt_fused: K2 j4 (no single-limb rule, NSMAX from np) and one epilogue per row class of the Q rows."""
    RL = logN - 12
    g = "1" if np_ == 1 else ("2-4" if np_ <= 4 else "5-6")
    cls = _classes(Q[:nq], logN)
    cells = {("k2_moddown", RL, g, c) for c in cls} | {("fz", RL, FZ[c], with_d) for c in cls}
    return cells, len(cls), len(cls)


def predict_rescale(logN, Q, level):
    """div_round_last_ntt_fused: K2 PRO_BCAST (with the reduction when q_last >= 2^50) and the epilogue, per row class."""
    RL = logN - 12
    wide = Q[level] >> 50 != 0
    cls = _classes(Q[:level], logN)
    cells = {("k2_bcast", RL, c, wide) for c in cls} | {("fz", RL, FZ[c], False) for c in cls}
    return cells, len(cls), len(cls)


def predict(logN, Q, P, op):
    """(cells, K2 scopes, epilogue scopes) of one operation of a case in the default configuration."""
    kind = op[0]
    cells, nf, ne = set(), 0, 0
    if kind == "gp":                      # Evaluator.GadgetProduct(levelQ) with a key at levelP = keyP
        _, levelQ, keyP, pw2 = op
        if product_fused(logN, levelQ + 1, keyP, pw2):
            c, f = predict_product(logN, Q, P, levelQ + 1, keyP)
            cells |= c; nf += f
            if (levelQ + 1 + keyP) // (keyP + 1) == KMAX_DIGITS:
                cells.add(("nd_max", logN - 12))
        elif levelQ + 1 > 64 and keyP >= 1 and pw2 == 0:
            cells.add(("product_falls_back", logN - 12))
        if keyP >= 0 and moddown_fused(logN, levelQ + 1, keyP + 1):
            c, f, e = predict_moddown(logN, Q, levelQ + 1, keyP + 1, False)
            cells |= c; nf += f; ne += e
    elif kind == "mrr":                   # CKKSEvaluator.MulRelinRescaleNew at `level`, key at MaxLevelP
        _, level = op
        keyP = len(P) - 1
        assert product_fused(logN, level + 1, keyP, 0) and moddown_fused(logN, level + 1, keyP + 1) and level >= 1
        c, f = predict_product(logN, Q, P, level + 1, keyP)
        c2, f2, e2 = predict_moddown(logN, Q, level + 1, keyP + 1, True)
        c3, f3, e3 = predict_rescale(logN, Q, level)
        cells = c | c2 | c3; nf = f + f2 + f3; ne = e2 + e3
    elif kind == "md":                    # Evaluator.ModDown on one QP-stacked accumulator block
        _, levelQ, levelP = op
        assert moddown_fused(logN, levelQ + 1, levelP + 1)
        cells, nf, ne = predict_moddown(logN, Q, levelQ + 1, levelP + 1, False)
    else:
        raise ValueError(op)
    return cells, nf, ne


def required_cells():
    cells = set()
    for RL in (1, 2, 3, 4):
        cells |= {("k2_j4", RL, 4, "fp", True), ("k2_j4", RL, 4, "fp", False), ("k2_j4", RL, 8, "fp", None)}
        cells |= {("k2_j4", RL, ns, c, None) for ns in (4, 8) for c in ("corr", "plain")}
        cells |= {("k2_plain", RL, ns, c) for ns in (4, 8) for c in ("fp", "corr", "plain")}
        cells |= {("k2_moddown", RL, g, c) for g in ("1", "2-4", "5-6") for c in ("fp", "corr", "plain")}
        cells |= {("k2_bcast", RL, c, w) for c in ("fp", "corr", "plain") for w in (False, True)}
        cells |= {("k3", RL, v) for v in K3.values()}
        cells |= {("fz", RL, v, d) for v in FZ.values() for d in (False, True)}
    # the largest fused product (nd = kMaxDigits, FP64 MAC sums up to 32 q) and the first shape past it
    return cells | {("nd_max", 1), ("product_falls_back", 1)}


# ---- the cases --------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def chain(name, logN):
    """(Q, P, operations) of one case.
    A  CKKS-like, k = 4: [56] + [45] x 8 with [55] x 4. Level 8 = 4 + 4 + 1 (single-limb digit), level 7 = 4 + 4 (digit 1 splits,
       digit 0 holds the 56-bit q0 and does not), level 5 = 4 + 2; a k = 2 key below MaxLevelP.
    B  k = 6 and (key at levelP = 4) k = 5, 61-bit P over 60 / 56 / 40-bit Q: NSMAX = 8, CORR rows, ModDown with 5 and 6 P rows,
       a rescale by a 56-bit modulus over 40-bit rows.
    C  rows on both sides of the fp_ok and 2^58 bounds in one launch, k = 3 (digit 0 and every P row above 2^53), rescales by
       moduli just below and just above 2^50, a levelP = 0 key with and without BaseTwoDecomposition.
    D  (logN 13) 65 Q primes just below fp_bound with k = 2: 64 Q rows give nd = 32 = kMaxDigits (fused); 65 take the unfused
       product and the fused ModDown."""
    m = 2 << logN
    if name == "A":
        Q, P = O.gen_moduli(logN + 1, [56] + [45] * 8, [55] * 4)
        ops = [("gp", 8, 3, 0), ("gp", 7, 3, 0), ("gp", 5, 3, 0), ("gp", 8, 1, 0), ("mrr", 8), ("md", 8, 3)]
    elif name == "B":
        Q = O.gen_moduli(logN + 1, [60, 56, 40, 40, 40, 40, 40, 56], [])[0]
        P = H.Pi60[:6]
        ops = [("gp", 7, 5, 0), ("gp", 6, 5, 0), ("gp", 7, 4, 0), ("gp", 5, 4, 0), ("mrr", 7), ("md", 7, 5), ("md", 7, 4)]
    elif name == "C":
        c, n = primes_from(FWD_BOUND + 1, m, 3), primes_below(FWD_BOUND + 1, m, 3)
        f, a = primes_below(fp_bound(logN), m, 2), primes_from(fp_bound(logN), m, 2)
        Q = [c[0], n[0], c[1], f[0], a[0], f[1], n[1], primes_below(1 << 50, m, 1)[0], primes_from(1 << 50, m, 1)[0]]
        P = [c[2], n[2], a[1]]
        ops = [("gp", 6, 2, 0), ("gp", 5, 2, 0), ("gp", 6, 0, 0), ("mrr", 8), ("mrr", 7), ("md", 8, 2), ("md", 8, 0)]
    elif name == "D":
        Q = primes_below(fp_bound(logN), m, 65)
        P = O.gen_moduli(logN + 1, [], [55, 55])[1]
        ops = [("gp", 63, 1, 0), ("gp", 64, 1, 0)]
    else:
        raise ValueError(name)
    assert len(set(Q + P)) == len(Q) + len(P)
    return list(Q), list(P), ops


CASES = [(logN, name) for logN in LOGNS for name in ("A", "B", "C")] + [(13, "D")]


def reached_cells(cases):
    cells = set()
    for logN, name in cases:
        Q, P, ops = chain(name, logN)
        for op in ops:
            cells |= predict(logN, Q, P, op)[0]
    return cells


def test_dispatch_reaches_every_cell():
    """CASES reach every kernel instantiation of the fused pipeline at every RL (no GPU needed)."""
    missing = required_cells() - reached_cells(CASES)
    assert not missing, "cells no case reaches: %s" % sorted(missing, key=str)
    Q, P, ops = chain("D", 13)
    assert product_fused(13, 64, 1, 0) and (64 + 1) // 2 == KMAX_DIGITS
    assert not product_fused(13, 65, 1, 0) and moddown_fused(13, 65, 2)
    assert predict(13, Q, P, ("gp", 64, 1, 0))[1:] == (1, 1)        # only the ModDown's K2 scope is left


def test_dispatch_removing_a_case_leaves_a_cell():
    """Every case reaches some cell that no other case reaches at its RL, so dropping one fails the check above."""
    for case in CASES:
        rest = [c for c in CASES if c != case]
        assert required_cells() - reached_cells(rest), case


# ---- edge inputs ------------------------------------------------------------------------------------------------------------
def v_float(ys, qs):
    """K1's overflow count, as the reference computes it: sequential float64 divisions and sum, then truncation."""
    acc = np.float64(0.0)
    for y, q in zip(ys, qs):
        acc = acc + np.float64(y) / np.float64(q)
    return int(acc)


@functools.lru_cache(maxsize=None)
def digit_edges(qs):
    """Coefficient residue tuples (one entry per source q_i) at the edges of one digit's basis extension, and the restated v of
    the all-(q_i - 1) tuple. Multi-source digits: X' in {0, 1, floor(Q_d/2)}, X' = Q_d - j for the first j where v_float =
    v_exact + 1 (asserted), and every y_i = q_i - 1. Single-limb digits: c in {0, 1, (q >> 1) - 1, q >> 1, q - 1}."""
    qs = [int(q) for q in qs]
    if len(qs) == 1:
        q = qs[0]
        return [(0,), (1,), ((q >> 1) - 1,), (q >> 1,), (q - 1,)], None
    Qd = 1
    for q in qs:
        Qd *= q
    half = Qd >> 1
    hat = [Qd // q for q in qs]
    inv = [pow(h % q, -1, q) for h, q in zip(hat, qs)]

    def residues(xp):            # x with (x + floor(Q_d/2)) mod Q_d = X'
        x = (xp - half) % Qd
        return tuple(x % q for q in qs)

    out, ups = [residues(0), residues(1), residues(half)], 0
    for j in range(1, 1 << 14):
        xp = Qd - j
        ys = [xp * iv % q for iv, q in zip(inv, qs)]
        exact = (sum(y * h for y, h in zip(ys, hat)) - xp) // Qd
        vf = v_float(ys, qs)
        if vf != exact:
            assert vf == exact + 1, (qs, j)
            out.append(residues(xp))
            ups += 1
            if ups == 3:
                break
    assert ups, "no X' = Q_d - j rounds the float sum up: %r" % qs
    out.append(tuple(((q - 1) * h - half) % q for q, h in zip(qs, hat)))
    vmax = v_float([q - 1 for q in qs], qs)
    if all(q > 1 << 53 for q in qs):
        assert vmax == len(qs), qs          # every term rounds to 1.0: K2 reads vt[nS]
    return out, vmax


def put_edges(coef, moduli, k, rng):
    """Writes the edge tuples of every digit (k sources) of `coef` (coefficient domain, rows = moduli) at random positions."""
    N = coef.shape[-1]
    for r0, s in digits(len(moduli), k):
        tuples, _ = digit_edges(tuple(moduli[r0:r0 + s]))
        pos = rng.choice(N, size=len(tuples), replace=False)
        for t, x in zip(tuples, pos):
            coef[r0:r0 + s, x] = t


def test_edge_inputs_reach_the_float_v_edges():
    """Every digit of every case has X' = Q_d - j inputs with v_float = v_exact + 1 (asserted in digit_edges), and the digits
    whose sources all lie above 2^53 (C's digit 0 at k = 3, the P rows of B's and C's ModDowns) read vt[nS] (no GPU needed)."""
    top = []
    for logN, name in CASES:
        Q, P, ops = chain(name, logN)
        for op in ops:
            if op[0] == "gp" or op[0] == "mrr":
                nq = op[1] + 1
                k = max(op[2] + 1, 1) if op[0] == "gp" else len(P)
                for r0, s in digits(nq, k):
                    _, vmax = digit_edges(tuple(Q[r0:r0 + s]))
                    top.append(vmax == s)
            else:
                _, vmax = digit_edges(tuple(P[:op[2] + 1]))
                top.append(vmax == op[2] + 1)
    assert sum(top) >= 3 * len(LOGNS)


# ---- device runs ------------------------------------------------------------------------------------------------------------
def _scopes(fn, classes=(7, 8)):
    """Runs fn() with the event profiler on: (output, scopes of each of `classes`), by default LGPU_KCLASS_FUSED (K2) and
    LGPU_KCLASS_EPILOGUE. The profiler keeps every chain on the caller's stream."""
    import torch
    lb = _lb()
    L = lb.lib()
    nk = 9
    ms, by = (ctypes.c_double * nk)(), (ctypes.c_double * nk)()
    sc, kn = (ctypes.c_ulonglong * nk)(), (ctypes.c_ulonglong * nk)()
    torch.cuda.synchronize()
    L.lgpu_profile_read(ms, by, sc, kn)
    L.lgpu_profile_enable(1)
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        L.lgpu_profile_enable(0)
    L.lgpu_profile_read(ms, by, sc, kn)
    return (out,) + tuple(int(sc[k]) for k in classes)


def _check(ctx, got, want, what):
    got = ctx.to_host(got) if hasattr(got, "is_cuda") else got
    if not np.array_equal(got, want):
        bad = sorted({tuple(int(i) for i in ix[:-1]) for ix in zip(*np.nonzero(got != want))})
        raise AssertionError("%s: %d polynomials differ from the oracle, e.g. %s" % (what, len(bad), bad[:8]))


def _run(ctx, fn, logN, Q, P, op, want, what):
    """Unprofiled run against the oracle; in the default configuration, a profiled run with the predicted scope counts and
    the same output."""
    out = fn()
    _check(ctx, out, want, what)
    if DEFAULT_CONFIG:
        out2, nf, ne = _scopes(fn)
        _, pf, pe = predict(logN, Q, P, op)
        assert (nf, ne) == (pf, pe), "%s: K2 / epilogue scopes %r, predicted %r" % (what, (nf, ne), (pf, pe))
        _check(ctx, out2, want, what + " (profiled)")
    return out


def _ntt(ring, coef):
    out = np.empty_like(coef)
    for b in range(coef.shape[0]):
        ring.NTT(coef[b], out[b])
    return out


def _key(params, keyP, pw2, rng):
    """Uniform key at MaxLevelQ with words 0 and q - 1 in every row (positions 5 and 6)."""
    gk = H.random_gadget_ciphertext(params, params.MaxLevelQ(), keyP, rng, pw2=pw2)
    mods = np.array(params.qi + params.pi[: keyP + 1], dtype=U64)
    gk.data[..., 5] = 0
    gk.data[..., 6] = mods - U64(1)
    return gk


def _op_gp(lb, ctx, params, keys, logN, Q, P, op, rng, batch=2):
    _, levelQ, keyP, pw2 = op
    nq, N = levelQ + 1, params.N()
    if (keyP, pw2) not in keys:
        gk = _key(params, keyP, pw2, rng)
        keys[(keyP, pw2)] = (gk, lb.GadgetCiphertext(ctx, gk.data, gk.LevelQ(), gk.LevelP(), pw2, gk.pw2_sizes))
    gk_o, gk = keys[(keyP, pw2)]
    coef = np.stack([H.rand_poly(Q[:nq], N, rng) for _ in range(batch)])
    for b in range(batch):
        put_edges(coef[b], Q[:nq], max(keyP + 1, 1), rng)
    cx = _ntt(params.ringQ.AtLevel(levelQ), coef)
    ev_o = O.Evaluator(params)
    want = np.zeros((2, batch, nq, N), dtype=U64)
    for b in range(batch):
        ev_o.GadgetProduct(levelQ, cx[b].copy(), gk_o, [want[0, b], want[1, b]])
    import torch
    ev = lb.Evaluator(ctx)
    dcx = ctx.to_device(cx)

    def run(x=dcx):
        out = torch.zeros((2, x.shape[0], nq, N), dtype=torch.int64, device="cuda")
        ev.GadgetProduct(levelQ, x, gk, out[0], out[1])
        return out

    what = "logN=%d %r GadgetProduct" % (logN, op)
    out = _run(ctx, run, logN, Q, P, op, want, what)
    assert torch.equal(run(dcx[1:2].contiguous())[:, 0], out[:, 1]), what + ": batch consistency"


def _op_mrr(lb, ctx, params, keys, logN, Q, P, op, rng, batch=2):
    import torch
    _, level = op
    keyP, N = len(P) - 1, params.N()
    if (keyP, 0) not in keys:
        gk = _key(params, keyP, 0, rng)
        keys[(keyP, 0)] = (gk, lb.GadgetCiphertext(ctx, gk.data, gk.LevelQ(), gk.LevelP()))
    gk_o, gk = keys[(keyP, 0)]
    a = np.stack([np.stack([H.rand_poly(Q[: level + 1], N, rng) for _ in range(2)]) for _ in range(batch)])
    b = np.stack([np.stack([H.rand_poly(Q[: level + 1], N, rng) for _ in range(2)]) for _ in range(batch)])
    # element 0: op1[1] = 1 (NTT domain), so the relinearised polynomial a1 * b1 is a1 and carries the edge inputs
    coef = H.rand_poly(Q[: level + 1], N, rng)
    put_edges(coef, Q[: level + 1], keyP + 1, rng)
    a[0, 1] = _ntt(params.ringQ.AtLevel(level), coef[None])[0]
    b[0, 1] = 1
    ev_o = O.CKKSEvaluator(params, gk_o)
    want = np.zeros((batch, 2, level, N), dtype=U64)
    for i in range(batch):
        r = ev_o.Rescale(ev_o.MulRelinNew([a[i, 0], a[i, 1]], [b[i, 0], b[i, 1]]))
        want[i, 0], want[i, 1] = r
    ev = lb.CKKSEvaluator(ctx, gk)
    da, db = ctx.to_device(a), ctx.to_device(b)
    what = "logN=%d %r MulRelinRescaleNew" % (logN, op)
    out = _run(ctx, lambda: ev.MulRelinRescaleNew(da, db), logN, Q, P, op, want, what)
    assert torch.equal(ev.MulRelinRescaleNew(da[1:2].contiguous(), db[1:2].contiguous())[0], out[1]), what + ": batch consistency"


def _moddown_block(lb, ctx, levelQ, levelP, acc, out):
    """Evaluator.ModDown through the C ABI on one QP-stacked block acc = (2, batch, Q rows | P rows, N) into out = (batch, 2,
    levelQ + 1, N): the layout the fused ModDown takes (the Python wrapper derives strides from separate tensors)."""
    from lattigo_b200 import _lib
    from lattigo_b200.ring import _stream
    nq, np_, N, batch = levelQ + 1, levelP + 1, ctx.N, acc.shape[1]
    a0q = acc.data_ptr()
    a1q = a0q + batch * (nq + np_) * N * 8
    c0 = out.data_ptr()
    vp = ctypes.c_void_p
    _lib.check(lb.lib().lgpu_evaluator_moddown(ctx.h, levelQ, levelP, vp(a0q), vp(a0q + nq * N * 8), vp(a1q), vp(a1q + nq * N * 8),
                                               vp(c0), vp(c0 + nq * N * 8), batch, (nq + np_) * N, (nq + np_) * N, 2 * nq * N, _stream()))


def _op_md(lb, ctx, params, keys, logN, Q, P, op, rng, batch=2):
    import torch
    _, levelQ, levelP = op
    nq, np_, N = levelQ + 1, levelP + 1, params.N()
    accQ = np.stack([np.stack([H.rand_poly(Q[:nq], N, rng) for _ in range(batch)]) for _ in range(2)])
    coefP = np.stack([H.rand_poly(P[:np_], N, rng) for _ in range(2 * batch)])
    for x in coefP:
        put_edges(x, P[:np_], np_, rng)
    accP = _ntt(params.ringP.AtLevel(levelP), coefP).reshape(2, batch, np_, N)
    ev_o = O.Evaluator(params)
    want = np.zeros((batch, 2, nq, N), dtype=U64)
    for b in range(batch):
        ev_o.ModDown(levelQ, levelP, [accQ[0, b].copy(), accQ[1, b].copy()], [accP[0, b].copy(), accP[1, b].copy()], [want[b, 0], want[b, 1]])
    block = ctx.to_device(np.concatenate([accQ, accP], axis=2))

    def run(blk=block):
        out = torch.zeros((blk.shape[1], 2, nq, N), dtype=torch.int64, device="cuda")
        _moddown_block(lb, ctx, levelQ, levelP, blk, out)
        return out

    what = "logN=%d %r ModDown" % (logN, op)
    out = _run(ctx, run, logN, Q, P, op, want, what)
    assert torch.equal(run(block[:, 1:2].contiguous())[0], out[1]), what + ": batch consistency"


@pytest.mark.gpu
@pytest.mark.parametrize("logN,name", CASES, ids=["%d-%s" % c for c in CASES])
def test_fused_case(logN, name):
    """Every operation of one case: each ciphertext of a batch of 2 against the oracle, batch consistency, and (default
    configuration) the predicted K2 / epilogue scope counts with a profiled run that gives the same output."""
    lb = _lb()
    Q, P, ops = chain(name, logN)
    ctx = lb.Context(logN, Q, P)
    params = O.Parameters(logN, Q, P)
    rng = np.random.default_rng(100 * logN + ord(name))
    keys = {}
    run = {"gp": _op_gp, "mrr": _op_mrr, "md": _op_md}
    for op in ops:
        run[op[0]](lb, ctx, params, keys, logN, Q, P, op, rng)
    keys.clear()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("logN", LOGNS)
def test_fused_case_single_p_bit_decomposition(logN):
    """A context with one P prime and a BaseTwoDecomposition key (levelP = 0, unfused product, fused one-source ModDown), on
    chain C's rows: GadgetProduct, GadgetProductLazy and ModDown against the oracle."""
    Q, P, _ = chain("C", logN)
    _gadget_case(_lb(), logN, Q, P[:1], 30, (6,), seed=logN)


# ---- development switches ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("env", ["LGPU_K3_VARIANT=0", "LGPU_K3_VARIANT=10", "LGPU_K3_VARIANT=12", "LGPU_K3_VARIANT=13",
                                 "LGPU_K3_INT_VARIANT=0", "LGPU_K2_SPLIT=0", "LGPU_K2_J4=0", "LGPU_K2_FPSUM=1 LGPU_K2_J4=0",
                                 "LGPU_FZ_VARIANT=0", "LGPU_NO_FP64_NTT=1", "LGPU_NO_FUSED_KS=1", "LGPU_BATCH_CHUNK=1"])
def test_switches_stay_bit_exact(env):
    """The kernels' development switches (read once per process, hence a subprocess) re-run every fused_case against the
    oracle; the scope-count assertions restate the default configuration and are skipped there. LGPU_K2_FPSUM only reaches
    the plain K2 kernel, hence LGPU_K2_J4=0 with it."""
    import subprocess
    import sys
    e = dict(os.environ, **dict(kv.split("=") for kv in env.split()))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_keyswitch_fused.py"), "-m", "gpu", "-x", "-q",
                        "-k", "fused_case"], cwd=os.path.dirname(HERE), env=e, capture_output=True, text=True, timeout=3600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]

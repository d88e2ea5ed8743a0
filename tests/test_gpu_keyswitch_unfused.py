"""GPU parity (bit-exact vs the oracle) of the unfused key-switch kernels: basis extension and decomposition
(lattigo_b200/csrc/basisext.cu: `modup_kernel<NSMAX>`, `decomp_single_kernel`), the MAC (`mac_kernel`), the unfused ModDown and the
rescale family (composite.cu), at every ring degree and instantiation they serve.

These run whenever the fused pipeline (test_gpu_keyswitch_fused.py) does not: N = 2^4..2^12 and N = 2^17, single-P, BaseTwoDecomposition
and P-less keys, k > 6 P limbs, more than 64 Q rows, every ring-level entry point (ModUp, ModDown, DecomposeAndSplit, DecomposeSingleNTT,
DivBy{Round,Floor}LastModulusMany) and `Evaluator.ModDown` on accumulators that are not one QP-stacked block. `predict` restates the host
dispatch (target group, NSMAX, shared memory, the grids of `decomp_single_kernel` and `mac_kernel`, the single-P mode, and that nothing
takes the fused path); `test_dispatch_reaches_every_cell` (no GPU) checks that CASES reaches every cell of `required_cells()`, and
`test_unfused_case` runs each case on the device against the oracle, checks batch consistency and, in the default configuration, the
predicted MODUP / MAC scope counts with FUSED / EPILOGUE at 0.

Inputs carry the edges of the float `v` of every digit and of every ModDown P block (`digit_edges`), single-limb values
{0, 1, q/2 - 1, q/2, q - 1} and, for single-limb digits, c = q_s - t with t <= q_s/2 a target prime: the single-limb rule then writes t
itself, not 0 (the reference does the same, ring/basis_extension.go:428). Key words include 0 and q - 1. Run with -m gpu on an H100."""
import ctypes
import functools
import math

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_keyswitch_fused import (DEFAULT_CONFIG, KMAX_ROWS, _check, _ntt, _scopes, digit_edges, digits, moddown_fused,
                                            product_fused, put_edges)
from tests.test_gpu_ntt_persist import FWD_BOUND, fp_bound, primes_below, primes_from

U64 = np.uint64
KMAX_SRC = 64                 # basisext.cu: kMaxSrc
SMEM_DEFAULT = 48 * 1024      # dynamic shared memory without the opt-in
RING_LEVEL = ("qtop", "ptoq", "das", "dsn", "mdq", "mdqn", "mdp", "emd", "rs")
KC_MODUP, KC_MAC, KC_FUSED, KC_EPILOGUE = 3, 4, 7, 8      # enum lgpu_kclass
H100_SMS = (114, 132)         # PCIe and SXM5: the CPU-side dispatch checks hold for both


def _lb():
    import lattigo_b200 as lb
    return lb


# ---- the host dispatch of basisext.cu / composite.cu, restated --------------------------------------------------------------
def target_group(N, nT, batch, sms):
    """basisext.cu target_group: all targets in one CTA once (N/256) x batch CTAs reach 4 per SM, else enough groups for 4 per SM."""
    ctas = ((N + 255) // 256) * batch
    want = 4 * sms
    if ctas >= want:
        return nT
    groups = -(-want // ctas)
    return max(-(-nT // groups), 1)


def nsmax(nS):
    assert 1 <= nS <= KMAX_SRC
    return 4 if nS <= 4 else 8 if nS <= 8 else 16 if nS <= 16 else 64


def modup_smem(nS, nT):
    """Bytes of the per-target constant records modup_kernel stages: q, qinv, half, nS c_ij and nS + 1 vt entries."""
    return nT * (2 * nS + 4) * 8


def _modup(src, N, nS, nT, batch, sms):
    tg = target_group(N, nT, batch, sms)
    cells = {("modup", nsmax(nS), src), ("smem", "gt48K" if modup_smem(nS, nT) > SMEM_DEFAULT else "le48K")}
    if nT > 1:
        cells.add(("tg", "1" if tg == 1 else "nT" if tg >= nT else "ragged" if nT % tg else "even"))
    return cells


def _das(N, Q, P, lq, lp, nbPi, digit, batch, sms):
    """Cells of one launch_decompose_and_split: the reconstruction (modup_kernel) or the single-limb kernel, whose grid.y is
    min(nT, 8); its `t += gridDim.y` loop runs when nT > 8."""
    st, ed = digit * nbPi, min(digit * nbPi + nbPi, lq + 1)
    nT = lq + 1 + lp + 1
    if ed - st > 1:
        return _modup("das", N, ed - st, nT, batch, sms)
    cells = {("dsingle", "le8" if nT <= 8 else "gt8")}
    if any(t <= Q[st] // 2 for t in list(Q[: lq + 1]) + list(P[: lp + 1])):
        cells.add(("edge", "single_limb_writes_q"))
    return cells


def _mac(batch, xb=False, pshift=0, nd1=False, key_below=False):
    """mac_kernel: grid.z = min(batch, 4), the `b += gridDim.z` loop covers the rest."""
    zb = min(batch, 4)
    cells = {("mac_batch", "1" if batch == 1 else "4" if batch == 4 else "ragged>4" if batch > zb and batch % zb else "other")}
    for on, name in ((xb, "digit_from_xb"), (pshift > 0, "pshift"), (nd1, "nd1"), (key_below, "key_below_maxlevel")):
        if on:
            cells.add(("mac", name))
    return cells


def pw2_sizes(Q, pw2):
    """BaseTwoDecompositionVectorSize, core/rlwe/params.go:520-540 (levelP <= 0)."""
    return [(int(round(math.log2(float(q)))) + pw2 - 1) // pw2 for q in Q]


def nd_of(lq, keyP):
    return lq + 1 if keyP == -1 else (lq + keyP + 1) // (keyP + 1)


def predict(logN, Q, P, op, sms):
    """(cells, MODUP scopes, MAC scopes) of one operation; the counts are None where the path is not profiled."""
    N, kind = 1 << logN, op[0]
    cells = {("logN", logN), ("entry", kind)}
    if kind in RING_LEVEL:
        cells.add(("entry_at", kind, logN))
    nm = nmac = 0
    if kind == "qtop":
        _, lq, lp, b, lay = op
        cells |= _modup("qtop", N, lq + 1, lp + 1, b, sms); nm = 1
    elif kind == "ptoq":
        _, lp, lq, b, lay = op
        cells |= _modup("ptoq", N, lp + 1, lq + 1, b, sms); nm = 1
    elif kind in ("das", "dsn"):
        _, lq, lp, digit, b, lay = op
        cells |= _das(N, Q, P, lq, lp, lp + 1, digit, b, sms); nm = 1
    elif kind in ("mdq", "mdqn", "mdp"):
        _, lq, lp, b, lay = op
        cells |= _modup("qtop", N, lq + 1, lp + 1, b, sms) if kind == "mdp" else _modup("ptoq", N, lp + 1, lq + 1, b, sms)
        nm = 1
    elif kind == "emd":                     # separate accumulator tensors: one unfused ModDownQPtoQNTT per component
        _, lq, lp, b, lay = op
        cells |= _modup("ptoq", N, lp + 1, lq + 1, b, sms); nm = 2
    elif kind == "rs":
        _, ring, level, rnd, ntt, nb, inplace, b, lay = op
        cells.add(("rescale", ring, rnd, ntt, nb))
        if inplace:
            cells.add(("rescale", "in_place"))
    elif kind == "rs_ci":
        cells.add(("rescale", "ConjugateInvariant"))
        return cells, None, None
    elif kind in ("gp", "gpl", "hoist", "mrr"):
        if kind == "mrr":
            _, level, b = op
            lq, keyP, pw2, klq = level, len(P) - 1, 0, len(Q) - 1
            cells.add(("entry", "mrr", logN))
        elif kind == "gp":
            _, lq, keyP, pw2, klq, b = op
        else:
            _, lq, keyP, b = op
            pw2, klq = 0, len(Q) - 1
        assert not product_fused(logN, lq + 1, keyP, pw2)
        below = klq < len(Q) - 1
        if keyP >= 1:
            assert pw2 == 0
            nd = nd_of(lq, keyP)
            for d in range(nd):
                cells |= _das(N, Q, P, lq, keyP, keyP + 1, d, b, sms)
            cells |= _mac(b, xb=kind != "hoist", nd1=nd == 1, key_below=below)
            nm, nmac = nd, nd
            cells.add(("product", "multiple_p" if keyP + 1 <= 6 else "k>6"))
        elif pw2 == 0:
            assert keyP == 0
            for i in range(lq + 1):
                cells |= _das(N, Q, P, lq, 0, 1, i, b, sms)
            cells |= _mac(b, nd1=lq == 0, key_below=below) | {("singleP", "decomposer")}
            nm, nmac = lq + 1, lq + 1
        else:
            sz = pw2_sizes(Q, pw2)[: lq + 1]
            cells |= _mac(b, nd1=sum(sz) == 1, key_below=below)
            cells.add(("singleP", "pw2", "ragged" if len(set(sz)) > 1 else "even"))
            if keyP == -1:
                cells.add(("singleP", "noP"))
            nmac = sum(sz)
        if keyP >= 0:                       # QP-stacked accumulators (or separate tensors for gpl): unfused ModDown outside 2^13..2^16
            assert kind == "gpl" or not moddown_fused(logN, lq + 1, keyP + 1)
            cells |= _modup("ptoq", N, keyP + 1, lq + 1, b, sms)
            nm += 2
    elif kind == "ahl":                     # DecomposeNTT at dlq (outside the profiled call), then the hoisted MAC at lq < dlq
        _, lq, dlq, keyP, b = op
        for d in range(nd_of(dlq, keyP)):
            cells |= _das(N, Q, P, dlq, keyP, keyP + 1, d, b, sms)
        nd = nd_of(lq, keyP)
        cells |= _mac(b, pshift=dlq - lq, nd1=nd == 1)
        nmac = nd
    elif kind == "rgsw":                    # levelP = 0, pw2 = 0: every digit is the raw limb under the all-ones mask
        _, lq, b = op
        cells |= _mac(b) | {("singleP", "rgsw_all_ones")} | _modup("ptoq", N, 1, lq + 1, b, sms)
        nm, nmac = 2, 2 * (lq + 1)
    elif kind == "err":
        cells.add(("error", op[1]))
        return cells, None, None
    else:
        raise ValueError(op)
    if kind in RING_LEVEL and op[-1] != "dense":
        cells.add(("layout", op[-1]))
    return cells, nm, nmac


def required_cells():
    cells = {("modup", ns, src) for ns in (4, 8, 16, 64) for src in ("qtop", "ptoq", "das")}
    cells |= {("tg", "1"), ("tg", "ragged"), ("tg", "nT"), ("smem", "le48K"), ("smem", "gt48K"), ("dsingle", "le8"), ("dsingle", "gt8")}
    cells |= {("mac_batch", x) for x in ("1", "4", "ragged>4")} | {("mac", x) for x in ("digit_from_xb", "pshift", "nd1", "key_below_maxlevel")}
    cells |= {("singleP", "decomposer"), ("singleP", "pw2", "ragged"), ("singleP", "noP"), ("singleP", "rgsw_all_ones")}
    cells |= {("product", "multiple_p"), ("product", "k>6"), ("edge", "single_limb_writes_q")}
    cells |= {("rescale", r, rnd, ntt, nb) for r in (0, 1) for rnd in (True, False) for ntt in (True, False) for nb in (1, 2, 3)}
    cells |= {("rescale", "in_place"), ("rescale", "ConjugateInvariant"), ("layout", "pad"), ("layout", "odd")}
    cells |= {("logN", n) for n in (4, 5, 8, 11, 12, 17)} | {("entry_at", k, n) for k in RING_LEVEL for n in (13, 16)}
    cells |= {("entry", k) for k in RING_LEVEL + ("gp", "gpl", "hoist", "ahl", "rgsw")} | {("entry", "mrr", 12), ("entry", "mrr", 17)}
    cells |= {("error", e) for e in ("too_many_sources", "no_p_ring", "digit_out_of_range", "decompose_single_null_p")}
    return cells


# ---- the cases -------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def chain(name, logN):
    """(Q, P, operations) of one case.
    M  (every logN but 5) rows of every class in one chain: 61-bit and 58-bit+ rows with the lazy-correction schedule, rows just below
       and above 2^58, FP64-pipe rows (fp_ok, used by the transforms at logN >= 10) next to the first integer rows past fp_bound, and
       rows just below / above 2^50. Q = 10 rows, P = 4 rows; row 9 (61-bit) is the single-limb digit at k = 3 and k = 1.
    W  (logN 5) 66 Q rows (47 / 55-bit alternating) and 56 P rows above 2^58: NSMAX 8 / 16 / 64 from every source, shared memory
       above 48 KB (56 -> 56, 56 -> 66), k = 17 products, 56-source ModDown, and 65 sources refused."""
    m = 2 << logN
    if name == "M":
        c, n = primes_from(FWD_BOUND + 1, m, 3), primes_below(FWD_BOUND + 1, m, 3)
        f, a = primes_below(fp_bound(logN), m, 3), primes_from(fp_bound(logN), m, 2)
        Q = [c[0], f[0], n[0], a[0], f[1], c[1], n[1], primes_below(1 << 50, m, 1)[0], primes_from(1 << 50, m, 1)[0], H.Qi60[0]]
        P = [H.Pi60[0], n[2], a[1], f[2]]
        ops = _ops_m(logN)
    elif name == "W":
        lo, hi = primes_below(1 << 47, m, 33), primes_below(1 << 55, m, 33)
        Q = [x for pair in zip(lo, hi) for x in pair]
        P = primes_from(FWD_BOUND + 1, m, 56)
        ops = [("qtop", 55, 55, 2, "dense"), ("qtop", 12, 55, 2, "dense"), ("qtop", 6, 10, 2, "dense"),
               ("ptoq", 55, 65, 2, "dense"), ("ptoq", 12, 65, 2, "dense"), ("ptoq", 6, 65, 2, "dense"),
               ("das", 65, 16, 1, 2, "dense"), ("das", 65, 10, 2, 2, "dense"), ("das", 65, 5, 3, 2, "dense"),
               ("gp", 65, 16, 0, 65, 2), ("mdqn", 65, 55, 2, "dense"), ("err", "too_many_sources")]
    else:
        raise ValueError(name)
    assert len(set(Q + P)) == len(Q) + len(P) and len(Q) + len(P) <= KMAX_ROWS
    return list(Q), list(P), ops


def _ops_m(logN):
    if logN == 4:
        return [("qtop", 3, 3, 2, "dense"), ("qtop", 9, 3, 2, "dense"), ("ptoq", 3, 9, 2, "dense"), ("das", 9, 2, 1, 2, "dense"),
                ("das", 9, 2, 3, 2, "dense"), ("gp", 9, 2, 0, 9, 2), ("gp", 9, 0, 0, 9, 2), ("rs", 0, 9, True, True, 2, False, 2, "dense")]
    if logN == 8:
        rs = [("rs", ring, level, rnd, ntt, nb, False, 2, "dense") for ring, level in ((0, 9), (1, 3))
              for rnd in (True, False) for ntt in (True, False) for nb in (1, 2, 3)]
        return [("gp", 9, 2, 0, 9, 4), ("gp", 6, 3, 0, 7, 5), ("gp", 2, 3, 0, 9, 2),
                ("gp", 9, 0, 0, 9, 2), ("gp", 9, 0, 20, 9, 2), ("gp", 9, -1, 20, 9, 3), ("rgsw", 9, 2),
                ("gpl", 9, 3, 2), ("hoist", 9, 2, 2), ("ahl", 5, 9, 2, 2), ("dsn", 9, 2, 3, 2, "dense"), ("dsn", 3, 2, 1, 2, "dense"),
                ("rs", 0, 9, True, True, 1, True, 2, "dense"), ("rs", 1, 3, False, False, 2, True, 2, "dense")] + rs + \
               [("err", "no_p_ring"), ("err", "digit_out_of_range"), ("err", "decompose_single_null_p")]
    if logN == 11:
        return [("qtop", 9, 3, 1, "dense"), ("ptoq", 3, 9, 1, "dense"), ("das", 9, 2, 1, 1, "dense"), ("dsn", 9, 2, 3, 1, "dense"),
                ("gp", 9, 2, 0, 9, 1), ("mdq", 9, 3, 1, "dense"), ("emd", 9, 3, 1, "dense"),
                ("rs", 0, 9, False, True, 3, False, 1, "dense")]
    if logN == 12:
        lay = [(k,) + args + (lay,) for lay in ("pad", "odd") for k, args in
               (("qtop", (9, 3, 2)), ("das", (9, 2, 1, 2)), ("mdqn", (9, 3, 2)), ("rs", (0, 9, True, True, 1, False, 2)))]
        return [("das", 9, 2, 1, 3, "dense"), ("mrr", 9, 2), ("rs_ci",)] + lay
    if logN in (13, 16):
        return [("qtop", 9, 3, 2, "dense"), ("ptoq", 3, 9, 2, "dense"), ("das", 9, 2, 1, 2, "dense"), ("das", 9, 2, 3, 2, "dense"),
                ("dsn", 9, 2, 1, 2, "dense"), ("dsn", 9, 2, 3, 2, "dense"), ("mdq", 9, 3, 2, "dense"), ("mdqn", 9, 3, 2, "dense"),
                ("mdp", 9, 3, 2, "dense"), ("emd", 9, 3, 2, "dense"), ("rs", 0, 9, True, True, 1, False, 2, "dense"),
                ("rs", 1, 3, False, False, 2, False, 2, "dense")]
    if logN == 17:
        return [("gp", 9, 3, 0, 9, 2), ("mrr", 9, 1), ("qtop", 9, 3, 1, "dense"), ("das", 9, 2, 3, 1, "dense")]
    raise ValueError(logN)


CASES = [(4, "M"), (5, "W"), (8, "M"), (11, "M"), (12, "M"), (13, "M"), (16, "M"), (17, "M")]


def reached_cells(cases, sms):
    cells = set()
    for logN, name in cases:
        Q, P, ops = chain(name, logN)
        for op in ops:
            cells |= predict(logN, Q, P, op, sms)[0]
    return cells


@pytest.mark.parametrize("sms", H100_SMS)
def test_dispatch_reaches_every_cell(sms):
    """CASES reach every cell of the unfused path (no GPU needed)."""
    missing = required_cells() - reached_cells(CASES, sms)
    assert not missing, "cells no case reaches: %s" % sorted(missing, key=str)


@pytest.mark.parametrize("sms", H100_SMS)
def test_dispatch_removing_a_case_leaves_a_cell(sms):
    """Every case reaches a required cell no other case reaches, so dropping one fails the check above."""
    for case in CASES:
        rest = [c for c in CASES if c != case]
        assert required_cells() - reached_cells(rest, sms), case


def test_dispatch_restatement():
    """Spot checks of the restated dispatch against the numbers it is meant to produce (no GPU needed)."""
    assert target_group(1 << 17, 13, 2, 132) == 13 and target_group(1 << 4, 13, 2, 132) == 1
    assert target_group(1 << 12, 13, 3, 132) == 2 and target_group(1 << 12, 13, 3, 114) == 2
    assert [nsmax(s) for s in (1, 4, 5, 8, 9, 16, 17, 64)] == [4, 4, 8, 8, 16, 16, 64, 64]
    assert modup_smem(56, 56) == 51968 > SMEM_DEFAULT >= modup_smem(55, 52)
    assert pw2_sizes(chain("M", 8)[0], 20) == [3, 3, 3, 3, 3, 3, 3, 3, 3, 4]
    for logN, name in CASES:                # no product and no QP-stacked ModDown of a case is fused
        Q, P, ops = chain(name, logN)
        assert logN not in range(13, 17) or all(op[0] in RING_LEVEL for op in ops)


def test_edge_inputs_exist_for_every_digit():
    """digit_edges finds X' = Q_d - j with v_float = v_exact + 1 for every multi-limb digit of every case, and the P blocks above
    2^53 read vt[nS] (no GPU needed)."""
    top = 0
    for logN, name in CASES:
        Q, P, ops = chain(name, logN)
        for op in ops:
            for mods, k in _edge_digits(Q, P, op):
                for r0, s in digits(len(mods), k):
                    _, vmax = digit_edges(tuple(mods[r0:r0 + s]))
                    top += vmax == s and s > 1
    assert top >= 3


def test_oracle_refuses_more_than_64_sources():
    """The oracle's C restatement holds 64 sources per coefficient; more is refused on the Python side (no GPU needed)."""
    Q, P, _ = chain("W", 5)
    ringQ, ringP = O.Ring(32, Q), O.Ring(32, P)
    x, y = np.zeros((65, 32), dtype=U64), np.zeros((1, 32), dtype=U64)
    with pytest.raises(AssertionError, match="64 source limbs"):
        O.mod_up_exact(x, y, ringQ, ringP, O.ModUpConstants(Q[:65], P[:1]))


def _edge_digits(Q, P, op):
    """(moduli, digit size) of every block whose basis extension an operation runs on inputs the test sets."""
    kind = op[0]
    if kind in ("qtop", "mdp"):
        return [(Q[: op[1] + 1], op[1] + 1)]
    if kind == "ptoq":
        return [(P[: op[1] + 1], op[1] + 1)]
    if kind in ("das", "dsn"):
        return [(Q[: op[1] + 1], op[2] + 1)]
    if kind in ("mdq", "mdqn", "emd"):
        return [(P[: op[2] + 1], op[2] + 1)]
    if kind in ("gp", "gpl", "hoist", "mrr"):
        lq, keyP = (op[1], len(P) - 1) if kind == "mrr" else (op[1], op[2])
        return [(Q[: lq + 1], max(keyP + 1, 1))] + ([(P[: keyP + 1], keyP + 1)] if keyP >= 0 else [])
    if kind == "ahl":
        return [(Q[: op[2] + 1], op[3] + 1)]
    return []


# ---- device runs -----------------------------------------------------------------------------------------------------------
def _vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _place(ctx, arr, lay):
    """Device copy of the batched array `arr` (batch, rows, N): dense, with a padded batch stride, or at an odd word offset
    (8- but not 16-byte aligned)."""
    import torch
    d = ctx.to_device(np.ascontiguousarray(arr))
    if lay == "dense":
        return d
    b, r, N = arr.shape
    if lay == "pad":
        s = torch.zeros((b, r + 3, N), dtype=torch.int64, device=d.device)
        s[:, :r] = d
        return s[:, :r]
    flat = torch.zeros(b * r * N + 1, dtype=torch.int64, device=d.device)
    v = flat[1:].view(b, r, N)
    v.copy_(d)
    assert v.data_ptr() % 16 == 8
    return v


class _Env:
    def __init__(self, logN, name, sms):
        lb = _lb()
        self.lb, self.logN, self.name, self.sms = lb, logN, name, sms
        self.Q, self.P, self.ops = chain(name, logN)
        self.N = 1 << logN
        self.ctx = lb.Context(logN, self.Q, self.P)
        self.params = O.Parameters(logN, self.Q, self.P)
        self.ev_o = O.Evaluator(self.params)
        self.rng = np.random.default_rng(1000 * logN + ord(name))
        self.keys = {}

    def coef(self, mods, b, k, targets=()):
        """b coefficient-domain polynomials over `mods` with the edge inputs of every digit of k rows; single-limb digits also get
        c = q_s - t for the largest target prime t <= q_s/2."""
        x = np.stack([H.rand_poly(mods, self.N, self.rng) for _ in range(b)])
        for xb in x:
            put_edges(xb, mods, k, self.rng)
            for r0, s in digits(len(mods), k):
                ts = [t for t in targets if t <= mods[r0] // 2]
                if s == 1 and ts:
                    used = {int(e[0]) for e in digit_edges((mods[r0],))[0]}
                    free = [j for j in range(self.N) if int(xb[r0, j]) not in used]
                    xb[r0, self.rng.choice(free)] = mods[r0] - max(ts)
        return x

    def ntt(self, ring, level, x):
        return _ntt((self.params.ringQ if ring == 0 else self.params.ringP).AtLevel(level), x)

    def key(self, klq, keyP, pw2):
        """Uniform gadget ciphertext at (klq, keyP) with words 0 and q - 1 in every row, on the oracle and the device."""
        if (klq, keyP, pw2) not in self.keys:
            gk = H.random_gadget_ciphertext(self.params, klq, keyP, self.rng, pw2=pw2)
            mods = np.array(self.Q[: klq + 1] + self.P[: keyP + 1], dtype=U64)
            gk.data[..., 5] = 0
            gk.data[..., 6] = mods - U64(1)
            self.keys[(klq, keyP, pw2)] = (gk, self.lb.GadgetCiphertext(self.ctx, gk.data, klq, keyP, pw2, gk.pw2_sizes))
        return self.keys[(klq, keyP, pw2)]

    def run(self, op, fn, want):
        """fn(None) runs the whole batch, fn(i) element i alone; both against the oracle, then (default configuration) a profiled
        run with the predicted MODUP / MAC scopes and no fused scope."""
        what = "logN=%d %s %r" % (self.logN, self.name, op)
        out = fn(None)
        _check(self.ctx, out, want, what)
        b = want.shape[0]
        if b > 1:
            _check(self.ctx, fn(b - 1), want[b - 1:], what + " (last element alone)")
        _, pm, pmac = predict(self.logN, self.Q, self.P, op, self.sms)
        if DEFAULT_CONFIG and pm is not None:
            out2, m, mac, fz, ep = _scopes(lambda: fn(None), classes=(KC_MODUP, KC_MAC, KC_FUSED, KC_EPILOGUE))
            assert (m, mac, fz, ep) == (pm, pmac, 0, 0), "%s: MODUP / MAC / FUSED / EPILOGUE scopes %r, predicted %r" % (
                what, (m, mac, fz, ep), (pm, pmac, 0, 0))
            _check(self.ctx, out2, want, what + " (profiled)")


def _sl(t, i):
    return t if i is None else t[i:i + 1]


def _zeros(env, b, rows, lay="dense"):
    return _place(env.ctx, np.zeros((b, rows, env.N), dtype=U64), lay)


def _op_modup(env, op):
    from lattigo_b200.ring import _stream
    kind, ls, lt, b, lay = op
    S, T = (env.Q, env.P) if kind == "qtop" else (env.P, env.Q)
    x = env.coef(S[: ls + 1], b, ls + 1)
    want = np.zeros((b, lt + 1, env.N), dtype=U64)
    be = env.ev_o.BasisExtender
    for i in range(b):
        (be.ModUpQtoP if kind == "qtop" else be.ModUpPtoQ)(ls, lt, x[i].copy(), want[i])
    dx = _place(env.ctx, x, lay)
    f = env.lb.lib().lgpu_modup_qtop if kind == "qtop" else env.lb.lib().lgpu_modup_ptoq

    def fn(i):
        xi = _sl(dx, i)
        out = _zeros(env, xi.shape[0], lt + 1, lay)
        env.lb._lib.check(f(env.ctx.h, ls, lt, _vp(xi), _vp(out), xi.shape[0], xi.stride(0), out.stride(0), _stream()))
        return out
    env.run(op, fn, want)


def _op_das(env, op):
    import torch
    from lattigo_b200.ring import _stream
    kind, lq, lp, digit, b, lay = op
    nbPi, N = lp + 1, env.N
    x = env.coef(env.Q[: lq + 1], b, nbPi, targets=env.Q[: lq + 1] + env.P[: lp + 1])
    wq, wp = np.zeros((b, lq + 1, N), dtype=U64), np.zeros((b, lp + 1, N), dtype=U64)
    L = env.lb.lib()
    if kind == "das":
        for i in range(b):
            env.ev_o.Decomposer.DecomposeAndSplit(lq, lp, nbPi, digit, x[i].copy(), wq[i], wp[i])
        st, ed = digit * nbPi, min(digit * nbPi + nbPi, lq + 1)
        if ed - st > 1:
            wq[:, st:ed] = 0                # the reconstruction branch leaves the digit's own rows untouched
        dx = _place(env.ctx, x, lay)
    else:
        xn = env.ntt(0, lq, x)
        for i in range(b):
            env.ev_o.DecomposeSingleNTT(lq, lp, nbPi, digit, xn[i].copy(), x[i].copy(), wq[i], wp[i])
        dx, dn = env.ctx.to_device(x), env.ctx.to_device(xn)

    def fn(i):
        xi = _sl(dx, i)
        oq, op_ = _zeros(env, xi.shape[0], lq + 1, lay), _zeros(env, xi.shape[0], lp + 1, lay)
        if kind == "das":
            env.lb._lib.check(L.lgpu_decompose_and_split(env.ctx.h, lq, lp, nbPi, digit, _vp(xi), _vp(oq), _vp(op_), xi.shape[0],
                                                         xi.stride(0), op_.stride(0), _stream()))
        else:
            env.lb._lib.check(L.lgpu_decompose_single_ntt(env.ctx.h, lq, lp, nbPi, digit, _vp(_sl(dn, i)), _vp(xi), _vp(oq), _vp(op_),
                                                          xi.shape[0], xi.stride(0), oq.stride(0), op_.stride(0), _stream()))
        return torch.cat([oq, op_], dim=1)
    env.run(op, fn, np.concatenate([wq, wp], axis=1))


def _op_md(env, op):
    from lattigo_b200.ring import _stream
    kind, lq, lp, b, lay = op
    N, Q, P = env.N, env.Q, env.P
    if kind == "mdp":
        xq, xp = env.coef(Q[: lq + 1], b, lq + 1), np.stack([H.rand_poly(P[: lp + 1], N, env.rng) for _ in range(b)])
    else:
        xq, xp = np.stack([H.rand_poly(Q[: lq + 1], N, env.rng) for _ in range(b)]), env.coef(P[: lp + 1], b, lp + 1)
        if kind == "mdqn":
            xp = env.ntt(1, lp, xp)
    name = {"mdq": "ModDownQPtoQ", "mdqn": "ModDownQPtoQNTT", "mdp": "ModDownQPtoP"}[kind]
    rows = lp + 1 if kind == "mdp" else lq + 1
    want = np.zeros((b, rows, N), dtype=U64)
    for i in range(b):
        getattr(env.ev_o.BasisExtender, name)(lq, lp, xq[i].copy(), xp[i].copy(), want[i])
    dq, dp = _place(env.ctx, xq, lay), _place(env.ctx, xp, lay)
    f = getattr(env.lb.lib(), {"mdq": "lgpu_moddown_qp_to_q", "mdqn": "lgpu_moddown_qp_to_q_ntt", "mdp": "lgpu_moddown_qp_to_p"}[kind])

    def fn(i):
        qi, pi = _sl(dq, i), _sl(dp, i)
        out = _zeros(env, qi.shape[0], rows, lay)
        env.lb._lib.check(f(env.ctx.h, lq, lp, _vp(qi), _vp(pi), _vp(out), qi.shape[0], qi.stride(0), pi.stride(0), _stream()))
        return out
    env.run(op, fn, want)


def _op_emd(env, op):
    import torch
    _, lq, lp, b, _lay = op
    N, nq, np_ = env.N, lq + 1, lp + 1
    accQ = np.stack([np.stack([H.rand_poly(env.Q[:nq], N, env.rng) for _ in range(b)]) for _ in range(2)])
    accP = np.stack([env.ntt(1, lp, env.coef(env.P[:np_], b, np_)) for _ in range(2)])
    want = np.zeros((b, 2, nq, N), dtype=U64)
    for i in range(b):
        env.ev_o.ModDown(lq, lp, [accQ[0, i].copy(), accQ[1, i].copy()], [accP[0, i].copy(), accP[1, i].copy()], [want[i, 0], want[i, 1]])
    dq, dp = env.ctx.to_device(accQ), env.ctx.to_device(accP)      # two tensors: Q and P rows are not one QP-stacked block
    ev = env.lb.Evaluator(env.ctx)

    def fn(i):
        q0, q1, p0, p1 = (_sl(t, i).contiguous() for t in (dq[0], dq[1], dp[0], dp[1]))
        c = torch.zeros((2, q0.shape[0], nq, N), dtype=torch.int64, device="cuda")
        ev.ModDown(lq, lp, q0, p0, q1, p1, c[0], c[1])
        return c.transpose(0, 1)
    env.run(op, fn, want)


def _oracle_rescale(ring, rnd, ntt, nb, x, out):
    tmp = np.zeros_like(x)
    buff = np.zeros_like(x)
    if rnd and ntt:
        ring.DivRoundByLastModulusManyNTT(nb, x, buff, tmp)
    elif rnd:
        ring.DivRoundByLastModulusMany(nb, x, buff, tmp)
    elif ntt:
        ring.DivFloorByLastModulusManyNTT(nb, x, tmp)
    else:
        ring.DivFloorByLastModulusMany(nb, x, buff, tmp)
    out[...] = tmp[: out.shape[0]]


def _op_rs(env, op):
    from lattigo_b200.ring import _stream
    _, ring, level, rnd, ntt, nb, inplace, b, lay = op
    mods = env.Q if ring == 0 else env.P
    x = np.stack([H.rand_poly(mods[: level + 1], env.N, env.rng) for _ in range(b)])
    r = (env.params.ringQ if ring == 0 else env.params.ringP).AtLevel(level)
    want = np.zeros((b, level + 1 - nb, env.N), dtype=U64)
    for i in range(b):
        _oracle_rescale(r, rnd, ntt, nb, x[i].copy(), want[i])

    def fn(i):
        xi = _place(env.ctx, x if i is None else x[i:i + 1], lay)
        out = xi if inplace else _zeros(env, xi.shape[0], level + 1 - nb, lay)
        env.lb._lib.check(env.lb.lib().lgpu_div_by_last_modulus_many(env.ctx.h, ring, level, (1 if rnd else 0) | (2 if ntt else 0), nb,
                                                                     _vp(xi), _vp(out), xi.shape[0], xi.stride(0), out.stride(0), _stream()))
        return out[:, : level + 1 - nb]
    env.run(op, fn, want)


def _op_rs_ci(env, op):
    """Rescale on a ConjugateInvariant ring (NthRoot = 4N, its own transforms): every variant, nb in 1..3."""
    lb, logN, N = env.lb, env.logN, env.N
    m = 4 * N
    Q = primes_from(FWD_BOUND + 1, m, 2) + primes_below(fp_bound(logN), m, 2)
    ctx = lb.Context(logN, Q, [], ring_type=1)
    ring = O.Ring(N, Q, "ConjugateInvariant")
    x = np.stack([H.rand_poly(Q, N, env.rng) for _ in range(2)])
    dx = ctx.to_device(x)
    for rnd in (True, False):
        for ntt in (True, False):
            for nb in (1, 2, 3):
                want = np.zeros((2, 4 - nb, N), dtype=U64)
                for i in range(2):
                    _oracle_rescale(ring.AtLevel(3), rnd, ntt, nb, x[i].copy(), want[i])
                out = ctx.new_poly(4 - nb, 2)
                lb.div_by_last_modulus_many(ctx, 0, 3, rnd, ntt, nb, dx, out)
                _check(ctx, out, want, "ConjugateInvariant rescale %r" % ((rnd, ntt, nb),))
    ctx.close()


def _op_gp(env, op):
    import torch
    kind, N = op[0], env.N
    if kind == "gp":
        _, lq, keyP, pw2, klq, b = op
    else:
        _, lq, keyP, b = op
        pw2, klq = 0, len(env.Q) - 1
    nq, np_ = lq + 1, keyP + 1
    gk_o, gk = env.key(klq, keyP, pw2)
    coef = env.coef(env.Q[:nq], b, max(keyP + 1, 1), targets=env.Q[:nq] + env.P[: max(np_, 0)])
    cx = env.ntt(0, lq, coef)
    ev_o, ev = env.ev_o, env.lb.Evaluator(env.ctx)
    want = np.zeros((b, 2, nq, N), dtype=U64)
    for i in range(b):
        ev_o.GadgetProduct(lq, cx[i].copy(), gk_o, [want[i, 0], want[i, 1]])
    dcx = env.ctx.to_device(cx)
    if kind == "gp":
        def fn(i):
            x = _sl(dcx, i)
            c = torch.zeros((2, x.shape[0], nq, N), dtype=torch.int64, device="cuda")
            ev.GadgetProduct(lq, x, gk, c[0], c[1])
            return c.transpose(0, 1)
        env.run(op, fn, want)
    elif kind == "gpl":                     # GadgetProductLazy into separate Q / P tensors, then ModDown on them
        lazy = np.zeros((b, 2, nq + np_, N), dtype=U64)
        for i in range(b):
            aq = [np.zeros((nq, N), dtype=U64) for _ in range(2)]
            ap = [np.zeros((np_, N), dtype=U64) for _ in range(2)]
            ev_o.GadgetProductLazy(lq, cx[i].copy(), gk_o, aq, ap)
            for k in range(2):
                lazy[i, k, :nq], lazy[i, k, nq:] = aq[k], ap[k]

        def fn(i):
            x = _sl(dcx, i)
            bb = x.shape[0]
            aq = torch.zeros((2, bb, nq, N), dtype=torch.int64, device="cuda")
            ap = torch.zeros((2, bb, np_, N), dtype=torch.int64, device="cuda")
            ev.GadgetProductLazy(lq, x, gk, aq[0], ap[0], aq[1], ap[1])
            c = torch.zeros((2, bb, nq, N), dtype=torch.int64, device="cuda")
            ev.ModDown(lq, keyP, aq[0], ap[0], aq[1], ap[1], c[0], c[1])
            return torch.cat([aq, ap, c], dim=2).transpose(0, 1)
        env.run(op, fn, np.concatenate([lazy, want], axis=2))
    else:                                   # DecomposeNTT + GadgetProductHoisted
        nd = nd_of(lq, keyP)
        dq = [[np.zeros((nq, N), dtype=U64) for _ in range(nd)] for _ in range(b)]
        dp = [[np.zeros((np_, N), dtype=U64) for _ in range(nd)] for _ in range(b)]
        wh = np.zeros((b, 2, nq, N), dtype=U64)
        for i in range(b):
            ev_o.DecomposeNTT(lq, keyP, np_, cx[i].copy(), True, dq[i], dp[i])
            ev_o.GadgetProductHoisted(lq, dq[i], dp[i], gk_o, [wh[i, 0], wh[i, 1]])
        assert np.array_equal(wh, want)
        dec = env.ctx.to_host(ev.DecomposeNTT(lq, keyP, np_, dcx, True))
        wdec = np.stack([np.stack([np.concatenate([dq[i][d], dp[i][d]]) for i in range(b)]) for d in range(nd)])
        _check(env.ctx, dec, wdec, "logN=%d %r DecomposeNTT" % (env.logN, op))

        def fn(i):
            x = _sl(dcx, i)
            d = ev.DecomposeNTT(lq, keyP, np_, x, True)
            c = torch.zeros((2, x.shape[0], nq, N), dtype=torch.int64, device="cuda")
            ev.GadgetProductHoisted(lq, d, gk, c[0], c[1])
            return c.transpose(0, 1)
        env.run(op, fn, want)


def _op_ahl(env, op):
    """lgpu_evaluator_automorphism_hoisted_lazy into separate Q / P tensors: the unfused hoisted MAC on a decomposition laid out at
    dlq > lq (its P rows start dlq - lq rows later)."""
    import torch
    from lattigo_b200.ring import _stream
    _, lq, dlq, keyP, b = op
    N, nq, np_ = env.N, lq + 1, keyP + 1
    gk_o, gk = env.key(len(env.Q) - 1, keyP, 0)
    c1 = env.ntt(0, dlq, env.coef(env.Q[: dlq + 1], b, np_))
    c0 = np.stack([H.rand_poly(env.Q[:nq], N, env.rng) for _ in range(b)])
    galEl = env.params.GaloisElement(5)
    ndd = nd_of(dlq, keyP)
    want = np.zeros((b, 2, nq + np_, N), dtype=U64)
    for i in range(b):
        dq = [np.zeros((dlq + 1, N), dtype=U64) for _ in range(ndd)]
        dp = [np.zeros((np_, N), dtype=U64) for _ in range(ndd)]
        env.ev_o.DecomposeNTT(dlq, keyP, np_, c1[i].copy(), True, dq, dp)
        oq = [np.zeros((nq, N), dtype=U64) for _ in range(2)]
        opp = [np.zeros((np_, N), dtype=U64) for _ in range(2)]
        env.ev_o.AutomorphismHoistedLazy(lq, [c0[i].copy(), c1[i, :nq].copy()], dq, dp, galEl, gk_o, oq, opp)
        for k in range(2):
            want[i, k, :nq], want[i, k, nq:] = oq[k], opp[k]
    ev = env.lb.Evaluator(env.ctx)
    dec = ev.DecomposeNTT(dlq, keyP, np_, env.ctx.to_device(c1), True)
    d0 = env.ctx.to_device(c0)

    def fn(i):
        x0, d = _sl(d0, i), (dec if i is None else dec[:, i:i + 1].contiguous())
        bb = x0.shape[0]
        oq = torch.zeros((2, bb, nq, N), dtype=torch.int64, device="cuda")
        opp = torch.zeros((2, bb, np_, N), dtype=torch.int64, device="cuda")
        env.lb._lib.check(env.lb.lib().lgpu_evaluator_automorphism_hoisted_lazy(
            env.ctx.h, lq, _vp(x0), _vp(d), dlq, galEl, gk.ref(), _vp(oq[0]), _vp(opp[0]), _vp(oq[1]), _vp(opp[1]), bb, nq * N, nq * N,
            np_ * N, _stream()))
        return torch.cat([oq, opp], dim=2).transpose(0, 1)
    env.run(op, fn, want)


def _op_rgsw(env, op):
    """rgsw.ExternalProduct with a levelP = 0, BaseTwoDecomposition = 0 RGSW ciphertext: the raw limb under the all-ones mask."""
    import torch
    from lattigo_b200 import rgsw as lrgsw
    from oracle import rgsw as ORG
    _, lq, b = op
    N, nq = env.N, lq + 1
    g = [H.random_gadget_ciphertext(env.params, lq, 0, env.rng) for _ in range(2)]
    for gk in g:
        gk.data[..., 5] = 0
        gk.data[..., 6] = np.array(env.Q[:nq] + env.P[:1], dtype=U64) - U64(1)
    rg = lrgsw.Ciphertext(*[env.lb.GadgetCiphertext(env.ctx, gk.data, lq, 0) for gk in g])
    ct = np.stack([env.ntt(0, lq, env.coef(env.Q[:nq], 2, 1)) for _ in range(b)])
    want = np.zeros((b, 2, nq, N), dtype=U64)
    for i in range(b):
        ORG.Evaluator(env.params).ExternalProduct([ct[i, 0].copy(), ct[i, 1].copy()], g, [want[i, 0], want[i, 1]])
    dct = env.ctx.to_device(ct)
    ev = lrgsw.Evaluator(env.ctx)

    def fn(i):
        x = _sl(dct, i)
        out = torch.zeros_like(x)
        ev.ExternalProduct(x, rg, out)
        return out
    env.run(op, fn, want)


def _op_mrr(env, op):
    _, level, b = op
    N, nq = env.N, level + 1
    keyP = len(env.P) - 1
    gk_o, gk = env.key(len(env.Q) - 1, keyP, 0)
    a = np.stack([np.stack([H.rand_poly(env.Q[:nq], N, env.rng) for _ in range(2)]) for _ in range(b)])
    c = np.stack([np.stack([H.rand_poly(env.Q[:nq], N, env.rng) for _ in range(2)]) for _ in range(b)])
    # element 0: op1[1] = 1 (NTT domain), so the relinearised polynomial a1 * b1 is a1 and carries the edge inputs
    a[0, 1] = env.ntt(0, level, env.coef(env.Q[:nq], 1, keyP + 1, targets=env.Q[:nq] + env.P))[0]
    c[0, 1] = 1
    ev_o = O.CKKSEvaluator(env.params, gk_o)
    want = np.zeros((b, 2, level, N), dtype=U64)
    for i in range(b):
        want[i, 0], want[i, 1] = ev_o.Rescale(ev_o.MulRelinNew([a[i, 0], a[i, 1]], [c[i, 0], c[i, 1]]))
    ev = env.lb.CKKSEvaluator(env.ctx, gk)
    da, dc = env.ctx.to_device(a), env.ctx.to_device(c)
    env.run(op, lambda i: ev.MulRelinRescaleNew(_sl(da, i), _sl(dc, i)), want)


def _op_err(env, op):
    """Each error is returned as an error, and a correct call on the same context afterwards still matches the oracle."""
    from lattigo_b200.ring import _stream
    lb, N, what = env.lb, env.N, op[1]
    L = lb.lib()
    if what == "too_many_sources":          # ModUpQtoP at level 64: 65 sources
        x = env.ctx.to_device(np.stack([H.rand_poly(env.Q[:65], N, env.rng)]))
        with pytest.raises(lb.LgpuError, match="too many source limbs"):
            lb.BasisExtender(env.ctx).ModUpQtoP(64, 0, x, env.ctx.new_poly(1, 1))
        _op_modup(env, ("qtop", 55, 55, 1, "dense"))
    elif what == "no_p_ring":
        ctx0 = lb.Context(env.logN, env.Q)
        x = ctx0.to_device(np.stack([H.rand_poly(env.Q[:4], N, env.rng)]))
        with pytest.raises(lb.LgpuError, match="basis extension requires a P ring"):
            lb.BasisExtender(ctx0).ModUpQtoP(3, 0, x, ctx0.new_poly(1, 1))
        y = np.stack([H.rand_poly(env.Q, N, env.rng)])
        want = np.zeros((1, len(env.Q) - 1, N), dtype=U64)
        _oracle_rescale(env.params.ringQ, True, True, 1, y[0].copy(), want[0])
        out = ctx0.new_poly(len(env.Q) - 1, 1)
        lb.div_by_last_modulus_many(ctx0, 0, len(env.Q) - 1, True, True, 1, ctx0.to_device(y), out)
        _check(ctx0, out, want, "rescale after the refused basis extension")
        ctx0.close()
    elif what == "digit_out_of_range":      # digit 4 at nbPi = 3 starts at row 12 > levelQ = 9
        x = env.ctx.to_device(np.stack([H.rand_poly(env.Q, N, env.rng)]))
        with pytest.raises(lb.LgpuError, match="decomposition digit out of range"):
            lb.Decomposer(env.ctx).DecomposeAndSplit(9, 2, 3, 4, x, env.ctx.new_poly(10, 1), env.ctx.new_poly(3, 1))
        _op_das(env, ("das", 9, 2, 2, 2, "dense"))
    elif what == "decompose_single_null_p":  # levelP >= 0 without a P output
        x = env.ctx.to_device(np.stack([H.rand_poly(env.Q, N, env.rng)]))
        out = env.ctx.new_poly(10, 1)
        rc = L.lgpu_decompose_single_ntt(env.ctx.h, 9, 2, 3, 1, _vp(x), _vp(x), _vp(out), None, 1, 10 * N, 10 * N, 3 * N, _stream())
        assert rc != 0 and "null polynomial" in L.lgpu_last_error().decode()
        rc = L.lgpu_decompose_single_ntt(env.ctx.h, 9, 4, 5, 1, _vp(x), _vp(x), _vp(out), _vp(out), 1, 10 * N, 10 * N, 10 * N, _stream())
        assert rc != 0 and "levelP out of range" in L.lgpu_last_error().decode()
        _op_das(env, ("dsn", 9, 2, 1, 2, "dense"))
    else:
        raise ValueError(what)


RUN = {"qtop": _op_modup, "ptoq": _op_modup, "das": _op_das, "dsn": _op_das, "mdq": _op_md, "mdqn": _op_md, "mdp": _op_md,
       "emd": _op_emd, "rs": _op_rs, "rs_ci": _op_rs_ci, "gp": _op_gp, "gpl": _op_gp, "hoist": _op_gp, "ahl": _op_ahl,
       "rgsw": _op_rgsw, "mrr": _op_mrr, "err": _op_err}


@pytest.mark.gpu
@pytest.mark.parametrize("logN,name", CASES, ids=["%d-%s" % c for c in CASES])
def test_unfused_case(logN, name):
    """Every operation of one case: each element of the batch against the oracle, the last element alone, and (default
    configuration) the predicted MODUP / MAC scope counts, with FUSED and EPILOGUE at 0, on a profiled run with the same output."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    env = _Env(logN, name, sms)
    for op in env.ops:
        RUN[op[0]](env, op)
    env.keys.clear()
    env.ctx.close()

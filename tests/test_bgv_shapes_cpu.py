"""Shapes of the BGV / BFV ciphertext product (lattigo_b200/csrc/bgv.cu) that tests/test_gpu_bgv_shapes.py runs, restated and checked
without a GPU.

`predict(logN, Q, level)` restates the host's choices for the scale-invariant (BFV) product at `level`: nq and nm = levelQMul + 1, the
`bfv_quantize_kernel<NM>` instantiation, the `modup_kernel<NSMAX>` of the operand ModUp Q -> QMul, whether the quantize needs more
than 48 KB of shared memory, and the row classes of the Q transforms. `CASES` (the chains and levels the GPU file runs) must reach
every cell: each NM at its lowest and highest nm, each NSMAX at its lowest and highest nq, the > 48 KB branch, and both row classes.

Quantize stage 1 computes the reference's v = uint64(sum_i float64(y_i) / float64(q_i)) over Q[:level+1]. The edge words of
tests/test_gpu_keyswitch_fused.digit_edges, taken over Q[:level+1] as one source set, reach the words where that float sum rounds up
(X' = Q - j) and, on the 61-bit chain B, the word where v = nq reads the last vtimes entry; `test_edge_words_reach_the_float_v_edges`
checks this by exact arithmetic. Stage 2's float v (QMul -> Q) can only differ from the exact one near z = +-QMul/2, which a product
of two ciphertexts never reaches: `test_quantize_stage2_edge_is_unreachable` states the bound.

The BFV product extends its operands from all level + 1 Q moduli to QMul in one basis extension, which takes at most 64 sources;
`test_host_only_refuses_bfv_above_64_moduli` checks that lgpu_bgv_polynomial_evaluate refuses a scale-invariant program above that,
before any launch, on a host-only handle."""
import ctypes
import functools

import numpy as np
import pytest

from lattigo_b200 import params as presets
from oracle import oracle as O
from tests import bgv_oracle as B
from tests import helpers as H
from tests.test_gpu_keyswitch_fused import digit_edges, v_float

LOGN = 10
KMAX_SRC = 64              # engine.h: kMaxSrc
SMEM_DEFAULT = 48 * 1024   # bytes of dynamic shared memory a launch gets without cudaFuncSetAttribute
REFUSAL = "the scale-invariant (BFV) multiplication supports at most 64 Q moduli"


# ---- the host's choices, restated ---------------------------------------------------------------------------------------------
def quant_smem_words(nq, nm):
    """bgv.cu: quant_smem_words."""
    return 4 * nq + nm * (4 + 2 * nq + 1) + 2 * nm + nq * (4 + 2 * nm + 1)


def fp_row(q, logN):
    """Whether the transforms of a Q row run on the FP64 pipe: tables.cu (LimbConst.fp_ok) and ntt_fp64.cu (fp64_ntt_supported)."""
    return 10 <= logN <= 17 and q * (10 + logN) < 1 << 51


def template(n, sizes):
    """The smallest instantiation in `sizes` that holds n (the if / else-if chains of launch_quantize and launch_modup)."""
    return next(s for s in sizes if n <= s)


def predict(logN, Q, level):
    nq = level + 1
    nm = B.level_qmul(logN, Q)[level] + 1                 # bgv.cu: lgpu_bgv_create, lq[l] (evaluator.go:43-48)
    return {
        "nq": nq,
        "nm": nm,
        "NM": template(nm, (4, 8, 16, 32)),               # bgv.cu: launch_quantize
        "NSMAX": template(nq, (4, 8, 16, KMAX_SRC)),       # basisext.cu: launch_modup, via launch_modup_qp in bfv_tensor
        "big_smem": quant_smem_words(nq, nm) * 8 > SMEM_DEFAULT,   # bgv.cu: launch_quantize, cudaFuncSetAttribute branch
        "rows": sorted({"fp" if fp_row(q, logN) else "int" for q in Q[:nq]}),
    }


# ---- the chains and the cases ---------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def chain(name, logN=LOGN):
    """(Q, P) of one chain. P of A and R is 55-bit so that QMul (61-bit primes) stays disjoint from it.
    A  [36] + [30] x 63: 64 FP64-pipe rows; nm runs 1..32 and nq 1..64 with the level; t may exceed q_i for i >= 1.
    B  Qi60[:31]: integer rows, all above 2^53; nm = 32 at the top.
    R  [36] + [29] x 65: 66 rows; level 63 is the largest BFV product (nq = 64), levels 64 and 65 are refused."""
    if name == "A":
        Q, P = O.gen_moduli(logN + 1, [36] + [30] * 63, [55] * 3)
    elif name == "B":
        Q, P = H.Qi60[:31], H.Pi60[:3]
    elif name == "R":
        Q, P = O.gen_moduli(logN + 1, [36] + [29] * 65, [55] * 3)
    else:
        raise ValueError(name)
    Q, P = [int(q) for q in Q], [int(p) for p in P]
    qmul = B.qmul_moduli(logN, Q)
    assert len(set(Q + P + qmul)) == len(Q) + len(P) + len(qmul), name
    return Q, P


def boundary_levels(name, logN=LOGN):
    """Level 0, the top level, and both sides of every level where the NM template, the NSMAX template or the shared-memory
    branch changes."""
    Q = chain(name, logN)[0]
    key = lambda l: tuple(predict(logN, Q, l)[k] for k in ("NM", "NSMAX", "big_smem"))
    out = {0, len(Q) - 1}
    for l in range(1, len(Q)):
        if key(l) != key(l - 1):
            out |= {l - 1, l}
    return sorted(out)


# (chain, logN, level, edge inputs): BFV and BGV products at t = 65537, and for the edge cases the float-v edge words
CASES = ([("A", LOGN, l, True) for l in boundary_levels("A")] + [("B", LOGN, len(chain("B")[0]) - 1, True)]
         + [("A", 14, len(chain("A", 14)[0]) - 1, False), ("R", LOGN, KMAX_SRC - 1, False)])


def required_cells():
    cells = {("NM", 4, 1), ("NM", 4, 4), ("NM", 8, 5), ("NM", 8, 8), ("NM", 16, 9), ("NM", 16, 16), ("NM", 32, 17), ("NM", 32, 32)}
    cells |= {("NSMAX", 4, 1), ("NSMAX", 4, 4), ("NSMAX", 8, 5), ("NSMAX", 8, 8), ("NSMAX", 16, 9), ("NSMAX", 16, 16),
              ("NSMAX", 64, 17), ("NSMAX", 64, 64)}
    return cells | {("big_smem",), ("rows", "fp"), ("rows", "int")}


def reached_cells(cases):
    cells = set()
    for name, logN, level, _ in cases:
        p = predict(logN, chain(name, logN)[0], level)
        cells |= {("NM", p["NM"], p["nm"]), ("NSMAX", p["NSMAX"], p["nq"])} | {("rows", r) for r in p["rows"]}
        if p["big_smem"]:
            cells.add(("big_smem",))
    return cells


def test_cases_reach_every_cell():
    missing = required_cells() - reached_cells(CASES)
    assert not missing, "cells no case reaches: %s" % sorted(missing, key=str)


def test_chains_reach_their_edges():
    Q = chain("A")[0]
    assert predict(LOGN, Q, 51)["big_smem"] is False and predict(LOGN, Q, 52)["big_smem"] is True
    assert all(q < Q[0] - 1 for q in Q[1:])                      # t = Q[0] - 1 exceeds every other modulus of A
    for name in ("A", "B"):
        Q = chain(name)[0]
        p = predict(LOGN, Q, len(Q) - 1)
        assert (p["NM"], p["nm"]) == (32, 32), name
    Q = chain("R")[0]
    assert predict(LOGN, Q, 63)["nq"] == KMAX_SRC and B.level_qmul(LOGN, Q)[-1] + 1 <= 32   # lgpu_bgv_create accepts R
    assert predict(14, chain("A", 14)[0], 63)["NM"] == 32


# ---- float v of quantize stage 1 ------------------------------------------------------------------------------------------------
def v_exact(ys, qs):
    """The exact overflow count: (sum_i y_i (Q/q_i) - X') / Q with X' = sum_i y_i (Q/q_i) mod Q."""
    Qd = 1
    for q in qs:
        Qd *= q
    return sum(y * (Qd // q) for y, q in zip(ys, qs)) // Qd


def stage1_y(word, qs):
    """y_i = (x_i + floor(Q/2)) (Q/q_i)^-1 mod q_i: the stage 1 sources of coefficient x (bgv.cu: bfv_quantize_kernel)."""
    Qd = 1
    for q in qs:
        Qd *= q
    return [(x + (Qd >> 1)) * pow(Qd // q % q, -1, q) % q for x, q in zip(word, qs)]


def edge_cases():
    return [(name, logN, level) for name, logN, level, edges in CASES if edges]


def test_edge_words_reach_the_float_v_edges():
    """At every edge case: some words have v_float = v_exact + 1 (X' = Q - j), none is off by more than one, and on chain B the
    all-(q_i - 1) word has v = nq (every term rounds to 1.0), so stage 1 reads vtimes[nq]."""
    for name, logN, level in edge_cases():
        qs = tuple(chain(name, logN)[0][: level + 1])
        words, vmax = digit_edges(qs)
        ups = 0
        for w in words:
            ys = stage1_y(w, qs)
            vf, ve = v_float(ys, qs), v_exact(ys, qs)
            assert abs(vf - ve) <= 1, (name, level, w)    # X' = 0 (an integer sum) may round down as well
            ups += vf == ve + 1
        if len(qs) > 1:
            assert ups >= 1, (name, level)
        if name == "B":
            assert vmax == len(qs) and any(stage1_y(w, qs) == [q - 1 for q in qs] for w in words), level


# ---- quantize stage 2 ---------------------------------------------------------------------------------------------------------------
def _stage2_chains():
    out = [(name, logN, chain(name, logN)[0]) for name, logN in (("A", LOGN), ("B", LOGN), ("R", LOGN), ("A", 14))]
    out.append(("2^8", 8, O.gen_moduli(9, [55, 40, 40, 40, 50, 50, 58, 58], [60, 60])[0]))
    sp = presets.PRESETS["BGV_N15QP880"]
    return out + [("BGV_N15QP880", sp["logN"], sp["Q"])]


def test_quantize_stage2_edge_is_unreachable():
    """Stage 2 lifts z (|z| <= N Q_level / 4 for a product of two ciphertexts) from QMul_level to Q with a float v that can only
    differ from the exact one near z = +-QMul_level / 2. N Q_level / 2 < QMul_level at every level keeps that edge out of reach."""
    for name, logN, Q in _stage2_chains():
        qmul = B.qmul_moduli(logN, Q)
        lq = B.level_qmul(logN, Q)
        Ql = 1
        for level, q in enumerate(Q):
            Ql *= int(q)
            M = 1
            for m in qmul[: lq[level] + 1]:
                M *= int(m)
            assert (1 << logN) * Ql // 2 < M, (name, logN, level)


# ---- host-only refusal --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_r():
    import lattigo_b200 as lb
    Q, P = chain("R")
    ctx = lb.Context(LOGN, Q, P, device=-1)
    qmul = np.array(B.qmul_moduli(LOGN, Q), dtype=np.uint64)
    h = ctypes.c_void_p()
    lb._lib.check(lb.lib().lgpu_bgv_create(ctx.h, 0x10001, qmul.ctypes.data, len(qmul), ctypes.byref(h)))
    yield Q, h
    lb.lib().lgpu_bgv_destroy(h)
    ctx.close()


def _poly_err(h, level, prog, si):
    """lgpu_bgv_polynomial_evaluate's error on a host-only handle (tests/test_bgv_polyeval_cpu.py: _err)."""
    import lattigo_b200 as lb
    buf = (ctypes.c_uint64 * 4)()
    addr = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    data = (ctypes.c_uint64 * 4)()
    g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), 65, 2, 0, 22, 1, None)   # levelQ 65, levelP 2
    cp = prog.to_c(1)
    rc = lb._lib.lib().lgpu_bgv_polynomial_evaluate(h, level, addr, 1, ctypes.byref(cp), ctypes.byref(g), si, addr, None)
    return None if rc == 0 else lb._lib.lib().lgpu_last_error().decode()


def test_host_only_refuses_bfv_above_64_moduli(host_r):
    from lattigo_b200 import bgv_polyeval as BPE
    from tests import bgv_polyeval_cases as C
    Q, h = host_r
    coeffs = C.cases(0x10001)["d3"][0]
    for level in (KMAX_SRC, KMAX_SRC + 1):
        e = _poly_err(h, level, BPE.plan(Q, 0x10001, level, 1, coeffs, 1, True), 1)
        assert e is not None and REFUSAL in e, (level, e)
    # nq = 64 passes every argument check, and BGV has no such limit
    assert "host-only" in _poly_err(h, KMAX_SRC - 1, BPE.plan(Q, 0x10001, KMAX_SRC - 1, 1, coeffs, 1, True), 1)
    assert "host-only" in _poly_err(h, KMAX_SRC + 1, BPE.plan(Q, 0x10001, KMAX_SRC + 1, 1, coeffs, 1, False), 0)

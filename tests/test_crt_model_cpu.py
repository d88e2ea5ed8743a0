"""The multiword CRT decoders' arithmetic (csrc/crt.cuh crt_exact_load<W>, mw_ge; csrc/encoder.cu words_to_double<W> and the CKKS
centring; csrc/bgv_encoder.cu's Horner reduction mod t), restated in tests/crt_cases.py, against exact integer references on the edge
sets that tests/test_gpu_crt_decode.py sends through the kernels. No GPU: this file shows, on the chains the GPU test uses, that those
inputs reach every branch of the device code, and pins the word-count rule (summed bit lengths) at each width switch."""
import math
import sys

import numpy as np
import pytest

from tests import crt_cases as K

TWO_T = [257, K.t60()]                                            # the GPU test's plaintext moduli
SCALES = [1.0, 2.0 ** 40, 2.0 ** 40 + 1, 1.75 * 2.0 ** 1023]       # the last one: |X| < 4 divides to a rounded subnormal


def _levels():
    out = [("A", lv) for lv, (_, W) in K.BOUNDARY_A.items() if W]
    return out + [("B", lv) for lv in K.BOUNDARY_B]


def _chain(name):
    return {"A": K.chain_a, "B": K.chain_b, "R": K.chain_r}[name]()


def _edges(name, level):
    C = K.Crt(_chain(name), level)
    return C, K.edge_values(C, np.random.default_rng(level))


def test_chain_boundaries_and_widths():
    """Every boundary level: the summed bit lengths, bits(Q_level), crt_words and the width the decoders launch (None = refused)."""
    q = K.chain_a()
    assert len(set(q)) == len(q) == len(K.SPEC_A) and all(x % (2 * K.N) == 1 and x < 1 << 61 for x in q)
    assert [x.bit_length() for x in q] == K.SPEC_A
    for lv, (words, W) in K.BOUNDARY_A.items():
        bits = sum(x.bit_length() for x in q[: lv + 1])
        assert K.crt_words(q, lv) == words and K.crt_width(words) == W, lv
        if lv in K.FULL_A:                                          # the top bit of word W - 1 is set
            assert bits == 64 * words == 64 * W and K.modulus(q, lv).bit_length() == 64 * W, lv
        else:                                                       # one prime past a boundary opens one more word
            assert bits > 64 * (words - 1) and K.crt_words(q, lv - 1) == words - 1, lv
    assert [W for _, W in K.BOUNDARY_A.values()] == [16, 32, 32, 64, 64, None]
    b = K.chain_b()
    for lv, (words, W) in K.BOUNDARY_B.items():
        assert K.crt_words(b, lv) == words and K.crt_width(words) == W
    fp_ok = [x * (10 + K.LOGN) < 1 << 51 for x in b]                # the FP64-pipe transform rows (tables.cu fp_ok)
    assert any(fp_ok[:20]) and not all(fp_ok[:20]) and fp_ok == [x.bit_length() == 45 for x in b]
    r = K.chain_r()                                                 # bits(Q) <= 4096, summed bit lengths past it: refused
    assert sum(x.bit_length() for x in r) == 4148 and K.modulus(r, K.REFUSE_R).bit_length() <= 4096
    assert K.crt_words(r, K.REFUSE_R) == 65 and K.crt_width(65) is None and K.crt_width(K.crt_words(r, K.REFUSE_R - 1)) == 64


@pytest.mark.parametrize("name,level", _levels())
def test_model_matches_exact_reference(name, level):
    """crt_exact rebuilds X; the CKKS value is Float64(centred X) / scale bit for bit; the BGV residue is the Euclidean centred X mod t."""
    C, xs = _edges(name, level)
    xs = K.fill_uniform(xs, len(xs) + 64, C.Q, np.random.default_rng(1000 + level))
    for X in xs:
        assert K.crt_exact(C, X)[0] == X
        c = K.centred(X, C.Q)
        for s in SCALES:
            got = K.ckks_value(C, X, s)[0]
            want = K.to_float64(c) / s
            assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (hex(X), s, got, want)
        for t in TWO_T:
            assert K.bgv_value(C, X, t)[0] == c % t, (hex(X), t)


def _branches(name, level):
    C, xs = _edges(name, level)
    infos = [K.ckks_value(C, X, 1.0) for X in xs]
    return C, [(X, v, i) for X, (v, _, i) in zip(xs, infos)]


@pytest.mark.parametrize("name,level", _levels())
def test_edge_sets_reach_every_crt_branch(name, level):
    """At every launched level: the quotient estimate exact, one too small (the >= Q subtraction, mw_ge true) and one too large (+ Q);
    mw_ge against Q false; the centring comparison both ways; where Q fills its W words, the accumulation carrying into acc[W]."""
    C, rows = _branches(name, level)
    ts = {i["t"] for _, _, i in rows}
    assert ts == {"exact", "under", "over"}, ts
    assert any(i.get("ge_Q") for _, _, i in rows if i["t"] == "under")
    assert any(i.get("ge_Q") is False for _, _, i in rows)
    assert {i["ge"] for _, _, i in rows} == {True, False}
    assert any(i["S_carry"] for _, _, i in rows) == (C.Q.bit_length() == 64 * C.W)


def test_edge_sets_reach_every_rounding_outcome():
    """Over the boundary levels: each words_to_double outcome, with the value that must come out of it."""
    seen = {}
    for name, level in _levels():
        _, rows = _branches(name, level)
        for X, v, i in rows:
            keys = [i["w_path"], "round_" + i.get("w_round", ""), "inf_" + i.get("w_inf", "")]
            keys += ["bs0"] if i.get("w_bs0") else []
            keys += ["carry"] if i.get("w_carry") else []
            keys += ["ws>0"] if i.get("w_ws", 0) > 0 else []
            keys += ["max_finite"] if abs(v) == sys.float_info.max else []
            for k in keys:
                seen.setdefault(k, v)
    for k in ("zero", "u64", "window", "round_down", "round_up", "round_tie_down", "round_tie_up", "round_sticky_low_up", "bs0",
              "carry", "ws>0", "inf_tie", "inf_big", "max_finite"):
        assert k in seen, k
    assert math.isinf(seen["inf_tie"]) and math.isinf(seen["inf_big"])
    # the sticky-only tie break needs both sides of the window rule: rounding the tie to even gives a different double
    for name, level in _levels():
        C, rows = _branches(name, level)
        for X, v, i in rows:
            if i.get("w_round") == "sticky_low_up":
                m = abs(K.centred(X, C.Q))
                assert K.to_float64(m) != K.to_float64(m - 1) and i["w_ws"] > 0


@pytest.mark.parametrize("name,level", [("A", lv) for lv in K.FULL_A])
def test_acc_top_word_after_subtraction_needs_q_within_the_quotient_error_of_2_64w(name, level):
    """After S - t Q, acc[W] != 0 only if t was one too small AND X + Q >= 2^(64 W), i.e. X / Q >= (2^(64 W) - Q) / Q; t is too small
    only if X / Q is below the error of the double quotient. At every full-width level of an NTT chain the first exceeds the second
    by more than 2^10, so the device's `acc[W] != 0 ||` guard is never the deciding term there (it stays for correctness)."""
    C = K.Crt(_chain(name), level)
    gap = ((1 << (64 * C.W)) - C.Q) / C.Q
    assert gap > 2 ** 10 * K.f_error_bound(C)


def _coprime_near(bits, count, taken):
    out, c = [], 1
    while len(out) < count:
        x = (1 << bits) - c
        if all(math.gcd(x, y) == 1 for y in taken + out):
            out.append(x)
        c += 2
    return out


def test_acc_top_word_branch_on_a_synthetic_table():
    """The same model on sixteen coprime 64-bit moduli just below 2^64 (no device context has them: they are neither NTT-friendly nor
    below 2^61), so Q lies within 2^-50 of 2^1024: a value with t one too small and acc[W] = 1 after the subtraction exists, and the
    guard is what makes the result right."""
    q = _coprime_near(64, 16, [])
    C = K.Crt(q, 15)
    assert C.W == 16 and C.Q.bit_length() == 1024 and sum(x.bit_length() for x in q) == 1024
    base = (1 << 1024) - C.Q
    hit = None
    for j in range(1 << 14):
        X = base + j * 977
        acc, info = K.crt_exact(C, X)
        assert acc == X
        if info.get("accW"):
            hit = (X, info)
            break
    assert hit is not None and hit[1]["t"] == "under" and not hit[1]["ge_Q"]  # mw_ge alone would keep X + Q

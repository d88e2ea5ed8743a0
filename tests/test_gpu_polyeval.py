"""lgpu_ckks_polynomial_evaluate against oracle/polyeval.py (the literal op-by-op restatement of ckks polynomial.Evaluator.Evaluate):
bit-for-bit equal ciphertexts, and the planner's output level and scale equal the oracle's. Every CPU case at N = 2^12 (batch 1 and 3),
CKKS_N15QP881 (batch 4, Chebyshev degree 30), BOOT_N16QP1767 at its EvalMod levels (60-bit primes, batch 2, even Chebyshev degree 30),
and one LINCOMB at the maximum term count with all-(q - 1) inputs and weights on 61-bit primes against Python integers."""
from fractions import Fraction

import numpy as np
import pytest

from lattigo_b200 import polyeval as PE
from lattigo_b200.params import PRESETS
from oracle import oracle as O
from oracle import polyeval as OP
from tests import helpers as H
from tests import polyeval_cases as PC

pytestmark = pytest.mark.gpu
U64 = np.uint64


def _run(logN, q, p, level, batch, cases, scale, lpr=1, prec=53, seed=0):
    import lattigo_b200 as lb
    rng = np.random.default_rng(seed)
    params = O.Parameters(logN, q, p)
    rlk = H.random_gadget_ciphertext(params, len(q) - 1, len(p) - 1, rng)
    ctx = lb.Context(logN, q, p, device=0)
    grlk = lb.GadgetCiphertext(ctx, rlk.data, len(q) - 1, len(p) - 1)
    N = 1 << logN
    cts = np.stack([np.stack([H.rand_poly(q[: level + 1], N, rng) for _ in range(2)]) for _ in range(batch)])
    dev = ctx.to_device(cts)
    ev = PE.PolynomialEvaluator(ctx, grlk, lpr, prec)
    oev = OP.PolyEvaluator(params, rlk, lpr, prec)
    for basis, coeffs, odd, even, tmul in cases:
        target = scale * tmul
        out, lv, sc = ev.Evaluate(dev, scale, coeffs, basis, target, odd, even)
        got = ctx.to_host(out)
        for b in range(batch):
            want = oev.Evaluate(OP.Ct([cts[b, 0], cts[b, 1]], scale), OP.new_polynomial(basis, coeffs, odd, even), target)
            assert lv == want.Level() and sc == want.Scale
            assert np.array_equal(got[b, 0], want.Value[0]) and np.array_equal(got[b, 1], want.Value[1]), "batch entry %d differs" % b
    ctx.close()


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("lpr", [1, 2])
def test_every_case_at_n4096(batch, lpr):
    logscale = 40 * lpr
    q, p = O.gen_moduli(13, [55] + [40] * 8, [55, 55])                # lpr = 2 rescales by pairs of 40-bit primes (scale 2^80)
    cases = [(b, c, o, e, t) for (b, c, o, e, l, t) in PC.cases().values() if l == lpr]
    _run(12, q, p, len(q) - 1, batch, cases, Fraction(2) ** logscale, lpr, max(53, logscale))


def test_n15qp881_batch4_chebyshev30():
    pr = PRESETS["CKKS_N15QP881"]
    rng = np.random.default_rng(11)
    coeffs = [float(rng.uniform(-1, 1)) / (k + 1) for k in range(31)]
    _run(pr["logN"], pr["Q"], pr["P"], len(pr["Q"]) - 1, 4, [(PE.CHEBYSHEV, coeffs, True, True, 1)], Fraction(2) ** 40)


def test_boot_n16qp1767_evalmod_levels_even_chebyshev30():
    pr = PRESETS["BOOT_N16QP1767"]
    rng = np.random.default_rng(12)
    coeffs = [0.0 if k & 1 else float(rng.uniform(-1, 1)) / (k + 1) for k in range(31)]
    # EvalMod runs on the 60-bit primes Q[17..25]; its input sits at level 25 (below CoeffsToSlots' four 56-bit primes)
    _run(pr["logN"], pr["Q"], pr["P"], 25, 2, [(PE.CHEBYSHEV, coeffs, False, True, 1)], Fraction(2) ** 60)


def test_lincomb_at_the_maximum_term_count_with_all_q_minus_1():
    import lattigo_b200 as lb
    logN, q = 12, H.Qi60[:3]
    N = 1 << logN
    ctx = lb.Context(logN, q, H.Pi60[:1], device=0)
    L, K = 2, PE.MAX_TERMS
    x = np.stack([np.stack([np.full(N, qi - 1, dtype=U64) for qi in q]) for _ in range(2)])[None]
    prog = PE.Program()
    prog.n_slots = 3
    w = []
    for _ in range(2):                                 # [n_out][K + 1][L + 1][2], every weight q - 1
        for _ in range(K + 1):
            for qi in q:
                w += [qi - 1, qi - 1]
    prog.ops = [dict(kind=PE.LINCOMB, level=L, outs=[1, 2], out_levels=[L, L - 1], terms=[0] * K, weights=w)]
    prog.out_slot, prog.out_level = 1, L
    out = ctx.new_poly(L + 1, 2).reshape(1, 2, L + 1, N)
    ev = PE.PolynomialEvaluator(ctx, None)
    ev.run(prog, ctx.to_device(x), out, 1)
    got = ctx.to_host(out)[0]
    for r, qi in enumerate(q):
        want0 = (K * (qi - 1) * (qi - 1) + (qi - 1)) % qi
        want1 = (K * (qi - 1) * (qi - 1)) % qi
        assert (got[0, r] == want0).all() and (got[1, r] == want1).all()
    ctx.close()

"""Anchors oracle/polyeval.py (the literal restatement of ckks polynomial.Evaluator.Evaluate) by decryption: with a real secret key and
relinearization key, the output decrypts to the polynomial evaluated on the plaintext slots within 2^-20, at the output scale the
restatement reports. Also pins OptimalSplit / SplitDegree and the 128-bit scale rounding on hand-computed values."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import polyeval as OP
from tests import polyeval_cases as PC

PRECISION_BITS = 20


@pytest.fixture(scope="module")
def toys():
    return {1: PC.Toy(lpr=1), 2: PC.Toy(lpr=2, nlevels=4, logscale=80)}


@pytest.mark.parametrize("name", sorted(PC.cases()))
def test_oracle_decrypts_to_the_polynomial(name, toys):
    basis, coeffs, odd, even, lpr, tmul = PC.cases()[name]
    toy = toys[lpr]
    rng = np.random.default_rng(3)
    x = rng.uniform(-1, 1, toy.N // 2)
    ct = OP.Ct(toy.encrypt(x), toy.scale)
    ev = OP.PolyEvaluator(toy.params, toy.rlk, lpr, toy.prec)
    target = toy.scale * tmul
    out = ev.Evaluate(ct, OP.new_polynomial(basis, coeffs, odd, even), target)
    assert OP.in_delta(out.Scale, target, 100), "output scale %s far from the target" % float(out.Scale)
    got = toy.decrypt(out.Value, out.Scale)
    want = PC.expected(basis, coeffs, x)
    err = np.max(np.abs(got - want))
    assert err < 2.0 ** -PRECISION_BITS, "%s: max error 2^%.1f" % (name, np.log2(err))


def test_optimal_split_and_split_degree_tables():
    # OptimalSplit(logDegree), utils/bignum/polynomial.go:14-23, computed by hand for logDegree = 1..8
    assert [OP.optimal_split(k) for k in range(1, 9)] == [1, 1, 2, 2, 3, 3, 4, 4]
    # SplitDegree, power_basis.go:34-52: halves for powers of two, otherwise (2^k - 1, n + 1 - 2^k) with k = bitlen(n-1) - 1
    assert [OP.split_degree(n) for n in (2, 3, 4, 5, 6, 7, 9, 12, 63)] == [(1, 1), (1, 2), (2, 2), (3, 2), (3, 3), (3, 4), (7, 2), (7, 5),
                                                                            (31, 32)]
    with pytest.raises(ValueError):
        OP.split_degree(0)


def test_scale_rounding_is_128_bit_nearest_even():
    # 1/3 = 0.0101...: 2^129 = 3k + 2, so the 128-bit mantissa rounds up to k + 1
    k = (2 ** 129 - 2) // 3
    assert OP.rnd(Fraction(1, 3), 128) == Fraction(k + 1, 2 ** 129)
    # ties go to the even mantissa
    assert OP.rnd(2 ** 128 + 1, 128) == 2 ** 128
    assert OP.rnd(2 ** 128 + 3, 128) == 2 ** 128 + 4
    assert OP.rnd(-(2 ** 128 + 3), 128) == -(2 ** 128 + 4)
    # products of two 61-bit primes are exact, a quotient is rounded
    q0, q1 = 0x1fffffffffe00001, 0x1fffffffffc80001
    assert OP.scale_mul(Fraction(q0), Fraction(q1)) == q0 * q1
    assert OP.scale_div(Fraction(2 ** 80), Fraction(q0)) == OP.rnd(Fraction(2 ** 80, q0), 128) != Fraction(2 ** 80, q0)
    # bigComplexToRNSScalar rounds half away from zero
    half = (OP.BF(Fraction(5, 2), 53), OP.BF(0, 53))
    assert OP.big_complex_to_rns_scalar([97], Fraction(1), half)[0] == [3]
    neg = (OP.BF(Fraction(-5, 2), 53), OP.BF(0, 53))
    assert OP.big_complex_to_rns_scalar([97], Fraction(1), neg)[0] == [97 - 3]


def test_degree_zero_and_too_few_levels_are_errors(toys):
    toy = toys[1]
    ct = OP.Ct(toy.encrypt(np.zeros(toy.N // 2)), toy.scale)
    ev = OP.PolyEvaluator(toy.params, toy.rlk, 1, toy.prec)
    with pytest.raises(ValueError):
        ev.Evaluate(ct, OP.new_polynomial(OP.MONOMIAL, [1.0]), toy.scale)
    low = OP.Ct([v[:3] for v in ct.Value], toy.scale)                  # level 2 < Depth(15) = 4
    with pytest.raises(ValueError):
        ev.Evaluate(low, OP.new_polynomial(OP.MONOMIAL, [0.5] * 16), toy.scale)

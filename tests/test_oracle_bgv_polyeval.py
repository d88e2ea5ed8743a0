"""Anchors the op-by-op BGV / BFV polynomial evaluation oracle (tests/bgv_polyeval_oracle.py) by decryption with real keys and slot
decoding: the reference's own test (bgv.testInsecure, t in {0x101, 0xffc001}, x^2 at MaxLevel), then dense, odd-only, even-only and
sparse polynomials up to degree 63, each decoding to EvalPolyModP of the slots; plus the errors the reference returns."""
import pytest

from oracle import oracle as O
from tests import bgv_polyeval_cases as C
from tests import bgv_polyeval_oracle as BP


@pytest.fixture(scope="module", params=C.INSECURE_T)
def insecure(request):
    return C.Toy(10, C.INSECURE_Q, C.INSECURE_P, request.param)


@pytest.mark.parametrize("invariant", [False, True])
def test_reference_test_x_squared(insecure, invariant):
    toy = insecure
    vals = toy.random_values()
    L = len(toy.q) - 1
    ct = toy.encrypt(vals, L)
    r, _ = C.oracle_eval(toy, invariant, ct, 1, [0, 0, 1], 1)
    assert int(r.Scale) == 1                     # res.Scale.Cmp(DefaultScale()) == 0
    if invariant:
        assert r.Level() == L
    assert toy.decrypt(r.Value, 1) == [v * v % toy.t for v in vals]


@pytest.fixture(scope="module", params=C.INSECURE_T)
def chain(request):
    q, p = O.gen_moduli(11, [55] + [45] * 9, [60, 60])
    return C.Toy(10, q, p, request.param, seed=5)


@pytest.mark.parametrize("invariant", [False, True])
def test_degrees_decode_to_eval_poly_mod_p(chain, invariant):
    toy = chain
    vals = toy.random_values()
    L = len(toy.q) - 1
    ct = toy.encrypt(vals, L)
    for name, (coeffs, odd, even) in C.cases(toy.t).items():
        pe = toy.evaluator(invariant)
        r = pe.Evaluate(BP.P.Ct(ct, 1), BP.new_polynomial(coeffs, odd, even), 1)
        cc = C.parity(coeffs, odd, even)
        assert toy.decrypt(r.Value, int(r.Scale)) == [C.eval_poly_mod(cc, v, toy.t) for v in vals], name
        assert int(r.Scale) == 1, name
        assert pe.counts["matchScalesBinary"] == 0, name           # EvaluateMonomial's InDelta check leaves only equal scales
        if invariant:
            assert r.Level() == L, name


def test_errors(insecure):
    toy = insecure
    ct = toy.encrypt(toy.random_values(), 1)
    for invariant in (False, True):
        with pytest.raises(ValueError, match="cannot evaluate poly"):            # 1 level < Depth(7) = 3, BFV included
            C.oracle_eval(toy, invariant, ct, 1, [1] * 8, 1)
        with pytest.raises(ValueError, match="degree"):
            C.oracle_eval(toy, invariant, ct, 1, [5], 1)
        pe = toy.evaluator(invariant)
        with pytest.raises(ValueError, match="Chebyshev"):
            pe.Evaluate(BP.P.Ct(ct, 1), BP.new_polynomial([1, 2, 3], basis=BP.CHEBYSHEV), 1)
    # BGV: x^2 at level 1 passes the Depth check and then has no level left for the final Rescale
    with pytest.raises(ValueError, match="cannot rescale"):
        C.oracle_eval(toy, False, ct, 1, [0, 0, 1], 1)


def test_match_scales_binary():
    """matchScalesBinary (evaluator.go:1569-1615): r0 s0 = r1 s1 mod t with small centred r0, r1."""
    t = 0x10001
    for s0, s1 in ((3, 5), (12345, 777), (1, t - 1), (2, 65000)):
        r0, r1, _ = BP.match_scales_binary(s0, s1, t)
        assert r0 * s0 % t == r1 * s1 % t
        with pytest.raises(ValueError):
            BP.match_scales_binary(0, s1, t)

"""Anchoring of oracle/ringswitch.py (ApplyEvaluationKey with ring-degree switching) by decryption with real keys, mirroring
core/rlwe/rlwe_test.go:818-894 (same degree, large -> small, small -> large at LogN 10 / 9, the small degree with its own P,
BaseTwoDecomposition 0 and 16) and its noise bound: log2 of the standard deviation of the decryption error <= LogN + bpw2.
Also checks the block-average identity the device uses for the downward NTT-domain switch against the literal
INTT / stride / NTTStandard-with-the-large-table path, at every gap 2 .. 2^12, for 45- and 61-bit primes."""
import numpy as np
import pytest

from oracle import oracle as O
from oracle import ringswitch as ORS
from tests import helpers as H

U64 = np.uint64


class _Sk:
    """A ternary secret of `params`: sn = NTT(s) (Q rows), mont = MForm(sn) (SecretKey.Value.Q)."""

    def __init__(self, params: O.Parameters, rng):
        N = params.N()
        self.params = params
        self.s = rng.integers(-1, 2, N)
        self.sn = np.empty((len(params.qi), N), dtype=U64)
        params.ringQ.NTT(H.small_poly_rns(self.s, params.qi), self.sn)
        self.mont = np.empty_like(self.sn)
        params.ringQ.MForm(self.sn, self.mont)

    def encrypt(self, m, rng, is_ntt=True):
        p = self.params
        N = p.N()
        a = H.rand_poly(p.qi, N, rng)
        me = H.small_poly_rns(np.asarray(m) + np.rint(rng.normal(0, 3.2, N)).astype(np.int64), p.qi)
        p.ringQ.NTT(me, me)
        c0 = np.stack([np.array([(int(x) - int(y) * int(t)) % int(q) for x, y, t in zip(me[l], a[l], self.sn[l])], dtype=U64)
                       for l, q in enumerate(p.qi)])
        ct = [c0, a]
        if not is_ntt:
            for k in range(2):
                p.ringQ.INTT(ct[k], ct[k])
        return ct

    def decrypt(self, ct, is_ntt=True):
        p = self.params
        level = ct[0].shape[0] - 1
        ringQ = p.ringQ.AtLevel(level)
        c = [np.ascontiguousarray(ct[0]).copy(), np.ascontiguousarray(ct[1]).copy()]
        if not is_ntt:
            for k in range(2):
                ringQ.NTT(c[k], c[k])
        acc = np.stack([np.array([(int(x) + int(y) * int(t)) % int(q) for x, y, t in zip(c[0][l], c[1][l], self.sn[l])], dtype=U64)
                        for l, q in enumerate(p.qi[: level + 1])])
        back = np.empty_like(acc)
        ringQ.INTT(acc, back)
        Q = ringQ.ModulusAtLevel[level]
        return [v if v < Q // 2 else v - Q for v in ringQ.PolyToBigint(back)]


def _log2_std(got, want):
    err = np.array([a - b for a, b in zip(got, want)], dtype=np.float64)
    return float(np.log2(np.std(err) + 1e-300))


def _params(bpw2):
    P = H.RLWE_TEST_P if bpw2 == 0 else H.RLWE_TEST_P[:1]      # BaseTwoDecomposition needs levelP <= 0
    big = O.Parameters(10, H.RLWE_TEST_Q, P)
    # the small degree has a P of its own, as rlwe_test.go:818-894 gives it; GenEvaluationKey reads only skOutput.Value.Q
    # (keygenerator.go:268-279), so the key's P rows come from the large parameters whatever the small P is
    small = O.Parameters(9, H.RLWE_TEST_Q, O.gen_moduli(11, [], [52])[1])
    assert set(small.pi).isdisjoint(big.pi)
    return big, small


@pytest.mark.parametrize("bpw2", [0, 16])
@pytest.mark.parametrize("is_ntt", [True, False])
def test_apply_evaluation_key_decrypts(bpw2, is_ntt):
    rng = np.random.default_rng(100 + bpw2 + is_ntt)
    big, small = _params(bpw2)
    N, n = big.N(), small.N()
    gap = N // n
    ev = O.Evaluator(big)
    skA, skB, skS = _Sk(big, rng), _Sk(big, rng), _Sk(small, rng)
    nq = len(big.qi)
    bound = big.logN + bpw2

    # same degree: skA -> skB
    evk = ORS.GenEvaluationKey(big, skA.mont, skB.mont, rng, pw2=bpw2)
    m = rng.integers(-(1 << 20), 1 << 20, N)
    ct = skA.encrypt(m, rng, is_ntt)
    out = [np.zeros((nq, N), dtype=U64) for _ in range(2)]
    ORS.ApplyEvaluationKey(ev, ct, evk, out, is_ntt)
    assert _log2_std(skB.decrypt(out, is_ntt), m) <= bound

    # large -> small: skA (N) -> skS (n); the result encrypts the coefficients at multiples of gap
    evk = ORS.GenEvaluationKey(big, skA.mont, skS.mont, rng, pw2=bpw2)
    ct = skA.encrypt(m, rng, is_ntt)
    out = [np.zeros((nq, n), dtype=U64) for _ in range(2)]
    ORS.ApplyEvaluationKey(ev, ct, evk, out, is_ntt)
    assert _log2_std(skS.decrypt(out, is_ntt), m[::gap]) <= bound

    # small -> large: skS (n) -> skA (N); Y = X^gap
    evk = ORS.GenEvaluationKey(big, skS.mont, skA.mont, rng, pw2=bpw2)
    ms = rng.integers(-(1 << 20), 1 << 20, n)
    ct = skS.encrypt(ms, rng, is_ntt)
    out = [np.zeros((nq, N), dtype=U64) for _ in range(2)]
    ORS.ApplyEvaluationKey(ev, ct, evk, out, is_ntt)
    want = np.zeros(N, dtype=np.int64)
    want[::gap] = ms
    assert _log2_std(skA.decrypt(out, is_ntt), want) <= bound


def test_degree_errors_are_the_references():
    big, _ = _params(0)
    ev = O.Evaluator(big)
    evk = H.random_gadget_ciphertext(big, 4, 1, np.random.default_rng(0))
    a = [np.zeros((5, 256), dtype=U64) for _ in range(2)]
    b = [np.zeros((5, 512), dtype=U64) for _ in range(2)]
    with pytest.raises(ValueError, match="opOut ring degree does not match"):
        ORS.ApplyEvaluationKey(ev, a, evk, b)
    with pytest.raises(ValueError, match="ctIn ring degree does not match"):
        ORS.ApplyEvaluationKey(ev, b, evk, a)


@pytest.mark.parametrize("bits", [45, 61])
def test_block_average_is_the_literal_downward_switch(bits):
    """SwitchCiphertextRingDegreeNTT(large -> small) == gap^-1 * block sums, for gap = 2 .. 2^12 at N = 2^14, on inputs all q - 1,
    all zero and uniform."""
    logN = 14
    q = O.gen_moduli(logN + 1, [bits], [])[0]
    ring = O.Ring(1 << logN, q)
    N = ring.N()
    rng = np.random.default_rng(bits)
    qq = int(q[0])
    inputs = [np.full((1, N), qq - 1, dtype=U64), np.zeros((1, N), dtype=U64), rng.integers(0, qq, (1, N), dtype=U64)]
    for lg in range(1, 13):
        n = N >> lg
        for A in inputs:
            out = [np.zeros((1, n), dtype=U64) for _ in range(2)]
            ORS.SwitchCiphertextRingDegreeNTT([A, A], ring, out)
            assert np.array_equal(out[0][0], ORS.block_average(A[0], n, qq)), (bits, lg)


def test_coefficient_domain_up_switch_keeps_the_other_coefficients():
    """SwitchCiphertextRingDegree upward writes only every gap-th coefficient of opOut (element.go:305-307)."""
    rng = np.random.default_rng(5)
    small = [rng.integers(0, 1 << 40, (2, 64), dtype=U64) for _ in range(2)]
    big = [rng.integers(0, 1 << 40, (2, 256), dtype=U64) for _ in range(2)]
    before = [b.copy() for b in big]
    ORS.SwitchCiphertextRingDegree(small, big)
    for k in range(2):
        assert np.array_equal(big[k][:, ::4], small[k])
        mask = np.ones(256, dtype=bool)
        mask[::4] = False
        assert np.array_equal(big[k][:, mask], before[k][:, mask])

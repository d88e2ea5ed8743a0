"""Anchoring of oracle/blindrot_evaluate.py (blindrot.Evaluator.Evaluate, core/rgsw/blindrot/evaluator.go:49-132) the way the reference's
blindrot_test.go checks it: a sign test polynomial, an RLWE ciphertext of evenly spaced values in [-1, 1), every slot blind-rotated,
decrypted and decoded against sign(x). Plus the host-side identities the device path relies on: the modulus switch to 2N against
Python integers (rounding boundary, ties, the even -> odd flip) and the cumulative mulBySmallMonomialMod2N against a direct rotation."""
import numpy as np
import pytest

from oracle import blindrot_evaluate as BE
from oracle import oracle as O
from tests import helpers as H

U64 = np.uint64
Q_BR = 0x7fff801            # blindrot_test.go: the blind-rotation modulus
Q_LWE = 0x3001              # and the LWE one


def _negacyclic(a, s, q):
    n = len(a)
    out = [0] * n
    for i, x in enumerate(a):
        for j, y in enumerate(s):
            k = i + j
            if k < n: out[k] += int(x) * int(y)
            else: out[k - n] -= int(x) * int(y)
    return [v % q for v in out]


def _auto_int(poly, g, N):
    out = [0] * N
    for i, c in enumerate(poly):
        e = (i * g) % (2 * N)
        if e < N: out[e] += int(c)
        else: out[e - N] -= int(c)
    return out


def make_keys(params, s_br, s_lwe, rng, pw2, window):
    """RGSW(X^{s_j}) per LWE coefficient and the window's automorphism keys, as GenEvaluationKeyNew (keys.go:52-109) lays them out."""
    N = params.N()
    q = params.qi
    brk = []
    for j in range(len(s_lwe)):
        mono = [0] * N
        if s_lwe[j] == 0: mono[0] = 1
        elif s_lwe[j] == 1: mono[1] = 1
        else: mono[N - 1] = -1                                   # X^{-1} = -X^{N-1}
        brk.append(H.gen_rgsw(params, mono, list(s_br), rng, pw2=pw2))
    ring1 = O.Ring(N, [q[0]])
    sp = H.small_poly_rns(s_br, [q[0]])
    gks = {}
    for g in [params.GaloisElement(k) for k in range(1, window + 1)] + [2 * N - 5]:
        ginv = pow(g, -1, 2 * N)
        row = np.empty_like(sp); ring1.Automorphism(sp, ginv, row)
        s_out = [int(v) if int(v) < q[0] // 2 else int(v) - q[0] for v in row[0]]
        gks[g] = H.gen_switching_key(params, s_br, s_out, rng, pw2=pw2)
    return brk, gks


def encrypt_lwe_values(values, n_lwe, s_lwe, rng, q=Q_LWE):
    """blindrot_test.go:104-123: coefficient i = round-toward-zero(values[i] * q/4), encrypted as (-a s + e + m, a), coefficient domain."""
    scale = float(q) / 4.0
    m = [0] * n_lwe
    for i, v in enumerate(values):
        m[i] = q - int(-v * scale) if v < 0 else int(v * scale)
    a = [int(x) for x in rng.integers(0, q, n_lwe)]
    e = [int(x) for x in np.rint(rng.normal(0, 3.2, n_lwe))]
    as_ = _negacyclic(a, s_lwe, q)
    c0 = [(-x + y + z) % q for x, y, z in zip(as_, e, m)]
    return [np.array([c0], dtype=U64), np.array([a], dtype=U64)]


def decrypt_coeff0(params, ct, s_br, ntt=True):
    q = params.qi[0]
    N = params.N()
    ringQ = params.ringQ.AtLevel(0)
    sn = H.small_poly_rns(s_br, [q])
    if ntt:
        ringQ.NTT(sn, sn)
        dec = np.array([[(int(x) + int(y) * int(t)) % q for x, y, t in zip(ct[0][0], ct[1][0], sn[0])]], dtype=U64)
        ringQ.INTT(dec, dec)
        c = int(dec[0, 0])
    else:
        c = (int(ct[0][0][0]) + _negacyclic([int(x) for x in ct[1][0]], list(s_br), q)[0]) % q
    return c if c < q // 2 else c - q


def test_evaluate_decrypts_to_sign():
    """The reference's own test at N = 2^7 (blind-rotation ring) and N_LWE = 2^4, its moduli and BaseTwoDecomposition 7, window 10."""
    logN, n_lwe, pw2, window = 7, 16, 7, 10
    params = O.Parameters(logN, [Q_BR], [])
    params_lwe = O.Parameters(4, [Q_LWE], [])
    N = params.N()
    rng = np.random.default_rng(5)
    s_br = rng.integers(-1, 2, N)
    s_lwe = rng.integers(-1, 2, n_lwe)
    brk, gks = make_keys(params, s_br, s_lwe, rng, pw2, window)
    scale_br = float(Q_BR) / 4.0
    tp = BE.InitTestPolynomial(np.sign, scale_br, params.ringQ, -1.0, 1.0)
    values = [-1 + 2 * i / n_lwe for i in range(n_lwe)]
    ct = encrypt_lwe_values(values, n_lwe, s_lwe, rng)
    ev = BE.Evaluator(params, params_lwe, window)
    for ntt_flag in (True, False):
        res = ev.Evaluate(ct, {i: tp for i in range(n_lwe)}, brk, gks, is_ntt=False, ntt_flag=ntt_flag)
        assert sorted(res) == list(range(n_lwe))
        for i, v in enumerate(values):
            if abs(v) < 0.25:
                continue      # within the 2N modulus switch's rounding of 0 (the reference prints these without a check)
            got = decrypt_coeff0(params, res[i], s_br, ntt=ntt_flag) / scale_br
            assert round(got * 8) / 8 == np.sign(v), (i, v, got)


def test_init_test_polynomial_coefficients():
    """InitTestPolynomial (blindrot.go:12-44) of sign on [-1, 1]: f_i = scaleUp(g(-i 2/N)) for i <= N/2, -g(2 (N - i)/N) above."""
    ring = O.Ring(16, [Q_BR])
    F = BE.InitTestPolynomial(np.sign, Q_BR / 4.0, ring, -1.0, 1.0)
    ring.INTT(F, F)
    s = int(Q_BR / 4.0 + 0.5)
    want = [0] + [Q_BR - s] * 8 + [Q_BR - s] * 7
    assert [int(x) for x in F[0]] == want


def test_mod_switch_against_python_integers():
    q, twoN = Q_LWE, 2048
    xs = [0, 1, q - 1, q // 2, q // 2 + 1]
    # values on both sides of every rounding boundary x 2N / q = k + 1/2
    for k in (0, 1, 5, 1000, twoN - 1):
        x = ((2 * k + 1) * q) // (2 * twoN)
        xs += [x - 1, x, x + 1]
    xs = [x % q for x in xs]
    for odd in (False, True):
        got = BE.mod_switch_to_2n(xs, q, twoN, odd)
        for x, r in zip(xs, got):
            num, den = 2 * x * twoN + q, 2 * q          # round half up == DivRound for x >= 0
            want = (num // den) & (twoN - 1)
            if odd and want % 2 == 0 and want != 0:
                want ^= 1
            assert r == want, (x, odd, r, want)
    # an exact tie rounds away from zero: q even so that x 2N / q hits k + 1/2
    assert BE.mod_switch_to_2n([3], 8, 4, False) == [2]           # 3 * 4 / 8 = 1.5 -> 2
    assert BE.mod_switch_to_2n([1], 8, 4, False) == [1]           # 0.5 -> 1
    assert BE.mod_switch_to_2n([1], 8, 4, True) == [1]
    assert BE.mod_switch_to_2n([3], 8, 4, True) == [3]            # 2 is even and non-zero -> 3
    assert BE.mod_switch_to_2n([0, 7], 8, 4, True) == [0, 0]      # 3.5 -> 4 = 2N -> 0, which stays 0
    assert BE.div_round(-3, 2) == -2 and BE.div_round(3, -2) == -2 and BE.div_round(-5, 4) == -1


@pytest.mark.parametrize("n,twoN", [(16, 64), (512, 2048)])
def test_cumulative_monomial_equals_direct_rotation(n, twoN):
    rng = np.random.default_rng(n)
    mask = twoN - 1
    a0 = [int(x) for x in rng.integers(0, twoN, n)]
    a = list(a0)
    prev = 0
    for idx in sorted(set([0, 1, 2, n // 2, n - 1] + [int(x) for x in rng.integers(0, n, 20)])):
        a = BE.mul_by_small_monomial_mod2n(mask, a, idx - prev)
        prev = idx
        direct = [a0[j - idx] if j >= idx else (-a0[n + j - idx]) & mask for j in range(n)]
        assert a == direct, idx

"""oracle/encoder.py (the CKKS encoder restated) anchored without the device:
- Decode(Encode(v)) = v within the quantisation bound at every log_slots (N = 2^8), at level 0 and above, on Q and on P rows;
- Encode, secret-key encrypt, decrypt, Decode gives v back; an IsMontgomery plaintext times a ciphertext (MulCoeffsMontgomery) decodes to
  u * v at the product scale;
- the sparse-NTT identity (n-point NTT with the N-point table, each output repeated gap times = N-point NTT of the spread polynomial) at
  every gap on 45- and 61-bit primes, also on the non-canonical words quantisation leaves;
- hand-computed words for every SingleFloat64ToFixedPointCRT branch, and the vectorised form equal to the literal one;
- the CRT-to-double rounding at exact ties and at 2^1024, the NoCRT uint64 wrap, math.Round;
- the reference's coefficient-domain spreading loop (core/rlwe/utils.go:234-241) panics or misplaces coefficients at every sparse slot
  count, which is why that case is rejected."""
import math

import numpy as np
import pytest

from oracle import encoder as E
from oracle import encryptor as ENC
from oracle import oracle as O

U64 = np.uint64
LOGN = 8
N = 1 << LOGN


@pytest.fixture(scope="module")
def params():
    q, p = O.gen_moduli(LOGN + 1, [55, 45, 45], [55, 61])
    return O.Parameters(LOGN, q, p)


def _values(rng, n):
    return rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)


@pytest.mark.parametrize("log_slots", list(range(LOGN)))
def test_decode_encode_round_trip(params, log_slots):
    rng = np.random.default_rng(log_slots)
    slots = 1 << log_slots
    scale = 2.0 ** 40
    v = _values(rng, max(1, slots - 1))                     # n_values < slots: zero-padded
    want = np.concatenate([v, np.zeros(slots - v.size)])
    for level in (0, 2):
        pq, pp = E.embed_double(params.ringQ, params.ringP, v, log_slots, scale, True, False, level, 1)
        for ring, pol, lvl in ((params.ringQ, pq, level), (params.ringP, pp, 1)):
            got = np.array(E.decode_public(ring, pol, lvl, log_slots, scale, True))
            assert np.abs(got - want).max() < slots * 2.0 ** -38, (level, lvl)
    if log_slots == LOGN - 1:                                # full slots also in the coefficient domain
        pq, _ = E.embed_double(params.ringQ, None, v, log_slots, scale, False, False, 2)
        got = np.array(E.decode_public(params.ringQ, pq, 2, log_slots, scale, False))
        assert np.abs(got - want).max() < slots * 2.0 ** -38


def test_decode_logprec_rounds(params):
    rng = np.random.default_rng(7)
    v = _values(rng, 16)
    pq, _ = E.embed_double(params.ringQ, None, v, 4, 2.0 ** 40, True, False, 1)
    got = np.array(E.decode_public(params.ringQ, pq, 1, 4, 2.0 ** 40, True, logprec=10))
    assert np.all((got.real * 1024) == np.round(got.real * 1024)) and np.abs(got - v).max() <= 2.0 ** -10


def test_coefficient_encoding_round_trip(params):
    rng = np.random.default_rng(3)
    v = rng.uniform(-100, 100, N - 5)
    for level in (0, 2):
        for ntt in (True, False):
            pol = E.encode_coeffs(params.ringQ, v, level, 2.0 ** 30, ntt)
            got = np.array(E.decode_public(params.ringQ, pol, level, LOGN - 1, 2.0 ** 30, ntt, is_batched=False))
            assert np.abs(got[: v.size] - v).max() < 2.0 ** -30 and np.all(got[v.size:] == 0)


def _sk(params, rng):
    s = rng.integers(-1, 2, N)
    sk = ENC.small_rows(s, params.qi + params.pi)
    nq = len(params.qi)
    params.ringQ.NTT(sk[:nq], sk[:nq]); params.ringQ.MForm(sk[:nq], sk[:nq])
    return sk


def _encrypt(params, rng, sk, pt, level):
    mods = params.qi[: level + 1]
    c1 = np.stack([rng.integers(0, q, N, dtype=U64) for q in mods])
    e = np.rint(rng.normal(0, 3.2, N)).astype(np.int64)
    c0 = ENC.Encryptor(params).encryptZeroSkFromC1QP(level, -1, sk, c1, e, True, False)
    r = params.ringQ.AtLevel(level)
    r.Add(c0, pt, c0)
    return c0, c1


def _decrypt(params, sk, c0, c1, level):
    r = params.ringQ.AtLevel(level)
    out = c0.copy()
    r.MulCoeffsMontgomeryThenAdd(c1, sk[: level + 1], out)
    return out


def test_encrypt_decrypt_and_montgomery_product(params):
    rng = np.random.default_rng(11)
    level, log_slots = 2, 5
    v, u = _values(rng, 32), _values(rng, 32)
    sk = _sk(params, rng)
    pv, _ = E.embed_double(params.ringQ, None, v, log_slots, 2.0 ** 35, True, False, level)
    c0, c1 = _encrypt(params, rng, sk, pv, level)
    got = np.array(E.decode_public(params.ringQ, _decrypt(params, sk, c0, c1, level), level, log_slots, 2.0 ** 35, True))
    assert np.abs(got - v).max() < 2.0 ** -20
    pu, _ = E.embed_double(params.ringQ, None, u, log_slots, 2.0 ** 30, True, True, level)     # IsMontgomery
    r = params.ringQ.AtLevel(level)
    d0, d1 = np.zeros_like(c0), np.zeros_like(c1)
    r.MulCoeffsMontgomery(c0, pu, d0)
    r.MulCoeffsMontgomery(c1, pu, d1)
    got = np.array(E.decode_public(params.ringQ, _decrypt(params, sk, d0, d1, level), level, log_slots, 2.0 ** 65, True))
    assert np.abs(got - u * v).max() < 2.0 ** -15


@pytest.mark.parametrize("bits", [45, 61])
def test_sparse_ntt_identity(bits):
    logN = 10
    (q,), _ = O.gen_moduli(logN + 1, [bits], [])
    s = O.get_subring(1 << logN, q)
    rng = np.random.default_rng(bits)
    for log_slots in range(logN - 1):
        n = 2 << log_slots
        gap = (1 << logN) // n
        for words in (rng.integers(0, q, n, dtype=U64), rng.integers(0, 1 << 61, n, dtype=U64)):   # canonical, then raw < 2^61
            sparse = np.repeat(E._ntt_n(s, words, n), gap)
            spread = np.zeros(1 << logN, dtype=U64)
            spread[::gap] = words % U64(q)
            full = np.empty_like(spread)
            s.NTT(spread, full)
            assert np.array_equal(sparse, full), (log_slots, words.max() >= q)


def test_single_float64_to_fixed_point_branches():
    (q0, q1), _ = O.gen_moduli(LOGN + 1, [45, 61], [])
    r = O.Ring(N, [q0, q1])
    cases = [
        (0.0, 1.0, [0, 0]), (-0.0, 1.0, [0, 0]),
        (1.5, 2.0, [3, 3]),                                        # 3.0 + 0.5 -> uint64 3
        (0.49999999999999994, 1.0, [1, 1]),                        # the sum rounds up to 1.0
        (-0.1, 1.0, [q0, q1]),                                     # c = 0: the word q itself
        (-3.0, 1.0, [q0 - 3, q1 - 3]),
        (-(2.0 ** 50), 1.0, [q0 - (2 ** 50 % q0), q1 - 2 ** 50]),  # c > q0: q - BRedAdd(c); c < q1: q - c
        (2.0 ** 50, 1.0, [2 ** 50, 2 ** 50]),                      # c > q0 left unreduced (<= 2^61 - 1)
        (2.0 ** 62, 1.0, [2 ** 62 % q0, 2 ** 62 % q1]),            # c > 2^61 - 1: BRedAdd
        (3.0, 2.0 ** 70, [3 * 2 ** 70 % q0, 3 * 2 ** 70 % q1]),    # >= 2^64: big.Int residue
        (-3.0, 2.0 ** 70, [q0 - 3 * 2 ** 70 % q0, q1 - 3 * 2 ** 70 % q1]),
        (1.0, 2.0 ** 64, [2 ** 64 % q0, 2 ** 64 % q1]),            # exactly 2^64 takes the big branch
        (math.inf, 1.0, [0, 0]), (-math.inf, 1.0, [q0, q1]),      # Float.Int(+-Inf) leaves xInt = 0
    ]
    for value, scale, want in cases:
        coeffs = [[None], [None]]
        E.SingleFloat64ToFixedPointCRT(r, 0, value, scale, coeffs)
        assert [coeffs[0][0], coeffs[1][0]] == want, (value, scale)
        rows = E.fixed_point_rows(r, np.array([value]), scale)
        assert [int(rows[0, 0]), int(rows[1, 0])] == want, (value, scale)
    assert 2 ** 50 > q0 and q0 - (2 ** 50 % q0) != q0


def test_vectorised_quantisation_equals_the_literal_one():
    (q0, q1, q2), _ = O.gen_moduli(LOGN + 1, [45, 55, 61], [])
    r = O.Ring(N, [q0, q1, q2])
    rng = np.random.default_rng(5)
    vals = np.concatenate([rng.normal(0, 1, 200), rng.normal(0, 2.0 ** 30, 50), [0.0, -0.0, 0.3, -0.3, 2.0 ** 20, -(2.0 ** 22)]])
    for scale in (2.0 ** 30, 2.0 ** 45, 2.0 ** 62):
        rows = E.fixed_point_rows(r, vals, scale)
        coeffs = [[0] * vals.size for _ in range(3)]
        for i, v in enumerate(vals):
            E.SingleFloat64ToFixedPointCRT(r, i, float(v), scale, coeffs)
        assert np.array_equal(rows, np.array(coeffs, dtype=U64))


def test_crt_to_double_ties_and_overflow():
    t = 2 ** 53
    assert E.to_float64(t + 1) == float(t) and E.to_float64(t + 3) == float(t + 4)           # ties to even
    assert E.to_float64(-(t + 1)) == -float(t) and E.to_float64(-(t + 3)) == -float(t + 4)
    big = 2 ** 1024
    assert E.to_float64(big) == math.inf and E.to_float64(-big) == -math.inf
    assert E.to_float64(big - 2 ** 970) == math.inf                                            # tie between DBL_MAX and 2^1024: even
    assert E.to_float64(big - 2 ** 970 - 1) == 1.7976931348623157e308
    # through polyToFloatCRT: centred X = 2^53 + 1 and Q - (2^53 + 1) on a two-limb ring
    q = O.gen_moduli(LOGN + 1, [40, 40], [])[0]
    r = O.Ring(N, q)
    Q = q[0] * q[1]
    p = np.zeros((2, N), dtype=U64)
    coeffs = [0] * N
    coeffs[0], coeffs[1], coeffs[2] = t + 1, Q - (t + 1), Q >> 1
    r.SetCoefficientsBigint(coeffs, p)
    got = E.polyToFloatCRT(r, p, 2.0)
    assert got[0] == float(t) / 2 and got[1] == -float(t) / 2 and got[2] == E.to_float64((Q >> 1) - Q) / 2
    assert got[3] == 0.0 and math.copysign(1, got[3]) == 1


def test_nocrt_wrap_is_pinned():
    (q,), _ = O.gen_moduli(LOGN + 1, [45], [])
    coeffs = np.array([q + 5, q, q - 1, 5, q >> 1], dtype=U64)
    got = E.polyToFloatNoCRT(coeffs, 4.0, q)
    assert got[0] == -float(2 ** 64 - 5) / 4.0                # Q - c wraps modulo 2^64
    assert got[1] == 0.0 and math.copysign(1, got[1]) == -1   # -float64(0) / s = -0
    assert got[2] == -0.25 and got[3] == 1.25 and got[4] == -float(q - (q >> 1)) / 4.0
    # complex form: -0 becomes +0 through values[i] += complex(0, .)
    row = np.zeros(N, dtype=U64)
    row[0] = q
    row[N // 2] = q
    vals = E.polyToComplexNoCRT(row, LOGN - 1, 2.0, N, q)
    assert math.copysign(1, vals[0].real) == 1 and math.copysign(1, vals[0].imag) == 1


def test_go_round():
    for x, want in ((2.5, 3.0), (-2.5, -3.0), (0.49999999999999994, 0.0), (1.5, 2.0), (2.0 ** 60 + 2.0 ** 8, 2.0 ** 60 + 2.0 ** 8)):
        assert E.go_round(x) == want
    assert math.copysign(1, E.go_round(-0.2)) == -1 and math.isnan(E.go_round(math.nan)) and E.go_round(-math.inf) == -math.inf


@pytest.mark.parametrize("logN", [4, 6, 8, 12])
def test_literal_spreading_loop_panics_or_misplaces(logN):
    n_full = 1 << logN
    for log_slots in range(logN - 1):
        n = 2 << log_slots
        gap = n_full // n
        coeffs = np.zeros(n_full, dtype=np.int64)
        coeffs[:n] = np.arange(1, n + 1)
        want = np.zeros(n_full, dtype=np.int64)
        want[::gap] = np.arange(1, n + 1)
        try:
            E.sparse_spread_literal(coeffs, n, gap)
        except IndexError:
            continue
        assert not np.array_equal(coeffs, want), (logN, log_slots)


def test_roots_table_symmetries():
    m = 2 * N
    rt = E.get_roots_complex128(m)
    assert rt[0] == 1 and rt[m // 4] == 1j and rt[m] == rt[0] and rt[m // 2] == -1
    for k in range(m):
        assert abs(rt[k] - complex(math.cos(2 * math.pi * k / m), math.sin(2 * math.pi * k / m))) < 1e-15

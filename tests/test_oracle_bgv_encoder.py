"""Anchors oracle/bgv_encoder.py without trusting its own restatement: round trips at levels 0, 1 and max for n = N, N/2, N/8 and 16 (signed
and unsigned, batched and coefficient mode, scale != 1); the slot-wise product is the decode of the negacyclic product mod t of the two
ring-T encodings; AutomorphismNTT by 5^k rotates both rows of n/2 slots left by k and 2N - 1 swaps them, at gap 1 and gap > 1 (this pins
permuteMatrix independently); coefficient-mode Encode equals the hand encoding of tests/test_oracle_bgv.py."""
import numpy as np
import pytest

from oracle import bgv_encoder as BE
from oracle import oracle as O

U64 = np.uint64
LOGN = 8


def _prime(m, bits):
    x = ((1 << bits) - 1) // m * m + 1
    while not O.is_prime(x):
        x -= m
    return x


# (t, slots) at N = 2^8: t = 1 mod 2^k exactly for k = 9 (n = N), 8 (N/2), 6 (N/8), 5 (16)
T_CASES = [(_prime(512, 30), 256), (257, 128), (193, 32), (97, 16)]


@pytest.fixture(scope="module")
def params():
    q, p = O.gen_moduli(LOGN + 1, [55, 45, 45], [61])
    return O.Parameters(LOGN, q, p)


def _enc(params, t):
    return BE.BGVEncoder(params.ringQ, t, params.ringP)


def _negacyclic(a, b, t):
    N = len(a)
    full = np.convolve(np.asarray(a, dtype=object), np.asarray(b, dtype=object))
    out = list(full[:N])
    for i in range(N - 1):
        out[i] -= full[N + i]
    return [int(x) % t for x in out]


@pytest.mark.parametrize("t,n", T_CASES)
def test_slot_counts_and_permutation(params, t, n):
    e = _enc(params, t)
    assert e.MaxSlots() == n and BE.plaintext_order(t) >= 2 * n
    assert sorted(e.indexMatrix) == list(range(n))


@pytest.mark.parametrize("t,n", T_CASES)
@pytest.mark.parametrize("signed", [False, True])
def test_round_trip(params, t, n, signed):
    e = _enc(params, t)
    rng = np.random.default_rng(t)
    N = params.N()
    for level in (0, 1, 2):
        for scale in (1, 12345, (1 << 64) - 3):
            if signed:
                v = [int(x) for x in rng.integers(-(1 << 63), (1 << 63) - 1, n)]
                v[:3] = [-(1 << 63), -t, 0]
                want = [x % t - t if x % t >= t >> 1 else x % t for x in v]
            else:
                v = [int(x) for x in rng.integers(0, (1 << 64) - 1, n, dtype=U64)]
                v[:3] = [(1 << 64) - 1, t, 0]
                want = [x % t for x in v]
            if scale % t == 0:
                continue
            pt = e.Encode(v, signed, scale, True, False, level)
            assert e.Decode(pt, level, scale, True, True, signed) == want
            coeffs = (v * (N // n))[:N]
            pt = e.Encode(coeffs, signed, scale, False, False, level, batched=False)
            got = e.Decode(pt, level, scale, False, False, signed)
            if signed:
                cw = [x % t - t if x % t >= t >> 1 else x % t for x in coeffs]
                assert got[:n] == cw[:n] and got[n:] == [0] * (N - n)      # only RingT().N() entries are written
            else:
                assert got == [x % t for x in coeffs]


@pytest.mark.parametrize("t,n", T_CASES)
def test_slotwise_product_is_the_negacyclic_product(params, t, n):
    e = _enc(params, t)
    rng = np.random.default_rng(n)
    a = [int(x) for x in rng.integers(0, t, n)]
    b = [int(x) for x in rng.integers(0, t, n)]
    pa = [int(x) for x in e.EncodeRingT(a, False, 1)[0]]
    pb = [int(x) for x in e.EncodeRingT(b, False, 1)[0]]
    prod = np.array([_negacyclic(pa, pb, t)], dtype=U64)
    assert e.DecodeRingT(prod, 1, False) == [x * y % t for x, y in zip(a, b)]


@pytest.mark.parametrize("t,n", [(_prime(512, 30), 256), (257, 128), (193, 32)])
def test_rotations(params, t, n):
    e = _enc(params, t)
    N = params.N()
    rng = np.random.default_rng(3)
    v = [int(x) for x in rng.integers(0, t, n)]
    h = n // 2
    ring = params.ringQ.AtLevel(1)
    pt = e.Encode(v, False, 1, True, False, 1)
    for k in (1, 2, 5):
        out = np.empty_like(pt)
        ring.AutomorphismNTT(pt, pow(5, k, 2 * N), out)
        assert e.Decode(out, 1, 1, True) == v[k:h] + v[:k] + v[h + k:] + v[h:h + k]
    out = np.empty_like(pt)
    ring.AutomorphismNTT(pt, 2 * N - 1, out)
    assert e.Decode(out, 1, 1, True) == v[h:] + v[:h]


def test_coefficient_encode_is_the_hand_encoding(params):
    """tests/test_oracle_bgv.py encodes m as (m t^-1 mod Q_level) per row, then NTT."""
    t, level = 65537, 2
    e = _enc(params, t)
    rng = np.random.default_rng(5)
    m = [int(x) for x in rng.integers(0, t, params.N())]
    mods = params.qi[: level + 1]
    Ql = 1
    for q in mods:
        Ql *= q
    tinv = pow(t, -1, Ql)
    hand = np.stack([np.array([x * (tinv % q) % q for x in m], dtype=U64) for q in mods])
    params.ringQ.AtLevel(level).NTT(hand, hand)
    assert np.array_equal(e.Encode(m, False, 1, True, False, level, batched=False), hand)

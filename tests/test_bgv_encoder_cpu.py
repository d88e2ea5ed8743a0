"""lgpu_bgv_encoder_create / lgpu_bgv_encode / lgpu_bgv_decode argument checks on a host-only context (device = -1): every rejection happens
before any device work, so the host-only handle reports the argument error, not the missing device. Pointers are never dereferenced by
the checks; fake device addresses stand in for buffers."""
import ctypes

import pytest

import lattigo_b200 as lb
from lattigo_b200 import _lib
from lattigo_b200.bgv_encoder import ENC_COEFFS, ENC_MONTGOMERY, ENC_NTT, ENC_SCALE_UP, ENC_SIGNED, plaintext_slots
from oracle import oracle as O

LOGN = 8
T = 65537
BUF = ctypes.c_void_p(1 << 20)          # aligned fake address
BAD = ctypes.c_void_p((1 << 20) + 4)    # not 8-byte aligned


def _create(ctx, t):
    h = ctypes.c_void_p()
    rc = _lib.lib().lgpu_bgv_encoder_create(ctx.h, t, ctypes.byref(h))
    return rc, _lib.lib().lgpu_last_error().decode(), h


@pytest.fixture(scope="module")
def ctx():
    q, p = O.gen_moduli(LOGN + 1, [55, 45, 45], [55])
    c = lb.Context(LOGN, q, p, device=-1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def enc(ctx):
    rc, msg, h = _create(ctx, T)
    assert rc == 0, msg
    yield h
    _lib.lib().lgpu_bgv_encoder_destroy(h)


def encode(enc, n_values=4, flags=ENC_NTT | ENC_SCALE_UP, scale=1, level_q=1, out_q=BUF, level_p=-1, out_p=BUF, batch=1, values=BUF, vs=0,
           qs=0, ps=0):
    rc = _lib.lib().lgpu_bgv_encode(enc, values, n_values, flags, scale, level_q, out_q, level_p, out_p, batch, vs, qs, ps, None)
    return rc, _lib.lib().lgpu_last_error().decode()


def decode(enc, level=1, flags=ENC_NTT, scale=1, values=BUF, batch=1, pt=BUF, ps=0, vs=0):
    rc = _lib.lib().lgpu_bgv_decode(enc, pt, level, flags, scale, values, batch, ps, vs, None)
    return rc, _lib.lib().lgpu_last_error().decode()


def test_valid_calls_reach_the_device_check(enc):
    for kw in ({}, {"flags": ENC_NTT}, {"flags": 0, "level_p": 0}, {"flags": ENC_NTT | ENC_MONTGOMERY, "level_p": 0},
               {"flags": ENC_COEFFS | ENC_SCALE_UP | ENC_SIGNED, "n_values": 1 << LOGN}, {"scale": 2 ** 64 - 1}, {"n_values": 0, "values": None}):
        rc, msg = encode(enc, **kw)
        assert rc != 0 and "host-only" in msg, (kw, msg)
    for kw in ({}, {"level": 0, "flags": 0}, {"flags": ENC_COEFFS | ENC_SIGNED}, {"flags": ENC_MONTGOMERY}, {"level": 2}):
        rc, msg = decode(enc, **kw)
        assert rc != 0 and "host-only" in msg, (kw, msg)


@pytest.mark.parametrize("t,word", [(0, ">= 2"), (1, ">= 2"), (None, "t|Q"), (1 << 56, "smaller than Q[0]"), (65536, "order < 16"),
                                    (17, "fewer than 16 slots"), (7, "order < 16"), (161, "not prime")])
def test_plaintext_modulus_conditions(ctx, t, word):
    t = ctx.Q[1] if t is None else t
    rc, msg, _ = _create(ctx, t)
    assert rc != 0 and word in msg, (t, msg)


def test_plaintext_ring_degree():
    assert plaintext_slots(1 << 8, 65537) == 1 << 8
    assert plaintext_slots(1 << 16, 65537) == 1 << 15
    assert plaintext_slots(1 << 12, 257) == 128
    assert plaintext_slots(1 << 12, 17) == 8                   # rejected by the encoder (n < 16)


def test_conjugate_invariant_ring_is_rejected():
    q, _ = O.gen_moduli(LOGN + 2, [55, 45], [])
    c = lb.Context(LOGN, q, [], device=-1, ring_type=1)
    try:
        rc, msg, _ = _create(c, T)
        assert rc != 0 and "Standard ring" in msg
    finally:
        c.close()


def test_value_counts(enc):
    slots = 1 << LOGN
    assert "slots" in encode(enc, n_values=slots + 1)[1]
    assert "slots" in encode(enc, n_values=-1)[1]
    assert "host-only" in encode(enc, n_values=slots)[1]
    assert "> N" in encode(enc, n_values=slots + 1, flags=ENC_COEFFS | ENC_SCALE_UP)[1]


def test_levels_out_of_range(enc):
    for lq in (-1, 3):
        assert "level_q out of range" in encode(enc, level_q=lq)[1]
        assert "level out of range" in decode(enc, level=lq)[1]
    assert "level_p out of range" in encode(enc, flags=0, level_p=1)[1]
    assert "level_p out of range" in encode(enc, level_p=-2)[1]


def test_no_p_rows_on_a_context_without_p():
    q, _ = O.gen_moduli(LOGN + 1, [55, 45], [])
    c = lb.Context(LOGN, q, [], device=-1)
    rc, msg, h = _create(c, T)
    try:
        assert rc == 0, msg
        assert "no P moduli" in encode(h, flags=0, level_p=0)[1]
    finally:
        _lib.lib().lgpu_bgv_encoder_destroy(h)
        c.close()


def test_mode_combinations(enc):
    assert "level_p must be -1" in encode(enc, level_p=0, flags=ENC_COEFFS | ENC_SCALE_UP)[1]
    assert "LGPU_ENC_SCALE_UP is required" in encode(enc, flags=ENC_COEFFS)[1]
    assert "Q moduli" in encode(enc, level_p=0, flags=ENC_SCALE_UP)[1]                 # Encode into a ringqp.Poly
    assert "flags" in encode(enc, flags=32)[1]
    assert "flags" in decode(enc, flags=ENC_SCALE_UP)[1]


def test_null_and_misaligned_pointers(enc):
    assert "null values" in encode(enc, values=None)[1]
    assert "aligned" in encode(enc, values=BAD)[1]
    assert "out_q" in encode(enc, out_q=None)[1]
    assert "out_q" in encode(enc, out_q=BAD)[1]
    assert "out_p" in encode(enc, flags=0, level_p=0, out_p=None)[1]
    assert "out_p" in encode(enc, flags=0, level_p=0, out_p=BAD)[1]
    assert "plaintext" in decode(enc, pt=None)[1]
    assert "plaintext" in decode(enc, pt=BAD)[1]
    assert "values" in decode(enc, values=None)[1]
    assert "values" in decode(enc, values=BAD)[1]
    assert "null encoder" in encode(None)[1]
    assert "null encoder" in decode(None)[1]
    h = ctypes.c_void_p()
    assert _lib.lib().lgpu_bgv_encoder_create(None, T, ctypes.byref(h)) != 0


def test_batch_and_strides(enc):
    for b in (0, 65536):
        assert "batch" in encode(enc, batch=b)[1]
        assert "batch" in decode(enc, batch=b)[1]
    assert "strides" in encode(enc, batch=2, vs=3, qs=2 << LOGN)[1]
    assert "strides" in encode(enc, batch=2, vs=4, qs=(2 << LOGN) - 1)[1]
    assert "strides" in encode(enc, flags=0, level_p=0, batch=2, vs=4, qs=2 << LOGN, ps=(1 << LOGN) - 1)[1]
    assert "host-only" in encode(enc, batch=2, vs=4, qs=2 << LOGN)[1]
    assert "strides" in decode(enc, batch=2, ps=(2 << LOGN) - 1, vs=1 << LOGN)[1]
    assert "strides" in decode(enc, batch=2, ps=2 << LOGN, vs=(1 << LOGN) - 1)[1]
    assert "host-only" in decode(enc, batch=2, ps=2 << LOGN, vs=1 << LOGN)[1]

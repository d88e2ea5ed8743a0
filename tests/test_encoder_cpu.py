"""lgpu_ckks_encode / lgpu_ckks_decode argument checks on a host-only context (device = -1): every rejection happens before any device
work, so the host-only context reports the argument error, not the missing device. Pointers are never dereferenced by the checks; fake
device addresses stand in for buffers."""
import ctypes

import pytest

import lattigo_b200 as lb
from lattigo_b200 import _lib
from lattigo_b200.encoder import ENC_COEFFS, ENC_MONTGOMERY, ENC_NTT
from oracle import oracle as O

LOGN = 8
BUF = ctypes.c_void_p(1 << 20)          # 16-byte aligned fake address
ODD = ctypes.c_void_p((1 << 20) + 8)    # 8-byte but not 16-byte aligned
BAD = ctypes.c_void_p((1 << 20) + 4)    # not 8-byte aligned


@pytest.fixture(scope="module")
def ctx():
    q, p = O.gen_moduli(LOGN + 1, [55, 45, 45], [55])
    c = lb.Context(LOGN, q, p, device=-1)
    yield c
    c.close()


@pytest.fixture(scope="module")
def ctx_nop():
    q, _ = O.gen_moduli(LOGN + 1, [55, 45], [])
    c = lb.Context(LOGN, q, [], device=-1)
    yield c
    c.close()


def encode(ctx, n_values=4, log_slots=LOGN - 1, scale=2.0 ** 40, flags=ENC_NTT, rot=BUF, roots=BUF, level_q=1, out_q=BUF, level_p=-1,
           out_p=BUF, batch=1, values=BUF, vs=0, qs=0, ps=0):
    rc = _lib.lib().lgpu_ckks_encode(ctx.h, values, n_values, log_slots, scale, flags, rot, roots, level_q, out_q, level_p, out_p, batch, vs, qs, ps,
                                     None)
    return rc, _lib.lib().lgpu_last_error().decode()


def decode(ctx, level=1, log_slots=LOGN - 1, scale=2.0 ** 40, flags=ENC_NTT, logprec=0.0, rot=BUF, roots=BUF, values=BUF, batch=1, pt=BUF,
           ps=0, vs=0):
    rc = _lib.lib().lgpu_ckks_decode(ctx.h, pt, level, log_slots, scale, flags, logprec, rot, roots, values, batch, ps, vs, None)
    return rc, _lib.lib().lgpu_last_error().decode()


def test_valid_calls_reach_the_device_check(ctx):
    for kw in ({}, {"level_p": 0}, {"flags": ENC_COEFFS, "n_values": 1 << LOGN, "rot": None, "roots": None}, {"flags": ENC_NTT | ENC_MONTGOMERY}):
        rc, msg = encode(ctx, **kw)
        assert rc != 0 and "host-only" in msg, (kw, msg)
    for kw in ({}, {"level": 0, "flags": 0}, {"flags": ENC_COEFFS, "rot": None, "roots": None}, {"logprec": 20.0}):
        rc, msg = decode(ctx, **kw)
        assert rc != 0 and "host-only" in msg, (kw, msg)


def test_conjugate_invariant_ring_is_rejected():
    q, _ = O.gen_moduli(LOGN + 2, [55, 45], [])
    c = lb.Context(LOGN, q, [], device=-1, ring_type=1)
    try:
        assert "Standard ring" in encode(c)[1]
        assert "Standard ring" in decode(c)[1]
    finally:
        c.close()


@pytest.mark.parametrize("log_slots", [-1, LOGN, LOGN + 3])
def test_log_slots_out_of_range(ctx, log_slots):
    assert "logSlots" in encode(ctx, log_slots=log_slots)[1]
    assert "logSlots" in decode(ctx, log_slots=log_slots)[1]
    assert "logSlots" in decode(ctx, log_slots=log_slots, flags=ENC_COEFFS)[1]     # decodePublic checks it before the type switch


def test_value_counts(ctx):
    assert "#values" in encode(ctx, n_values=5, log_slots=2)[1]
    assert "#values" in encode(ctx, n_values=-1)[1]
    assert "maximum number of values" in encode(ctx, n_values=(1 << LOGN) + 1, flags=ENC_COEFFS)[1]


def test_levels_out_of_range(ctx, ctx_nop):
    for lq in (-1, 3):
        assert "level_q out of range" in encode(ctx, level_q=lq)[1]
        assert "level out of range" in decode(ctx, level=lq)[1]
    assert "level_p out of range" in encode(ctx, level_p=1)[1]
    assert "level_p out of range" in encode(ctx, level_p=-2)[1]
    assert "no P moduli" in encode(ctx_nop, level_p=0)[1]
    assert "level_p must be -1" in encode(ctx, level_p=0, flags=ENC_COEFFS)[1]


@pytest.mark.parametrize("log_slots", list(range(LOGN - 1)))
def test_coefficient_domain_sparse_encoding_is_rejected(ctx, log_slots):
    for flags in (0, ENC_MONTGOMERY):
        rc, msg = encode(ctx, n_values=1, log_slots=log_slots, flags=flags)
        assert rc != 0 and "core/rlwe/utils.go:234-241" in msg
    assert "host-only" in encode(ctx, n_values=1, log_slots=LOGN - 1, flags=0)[1]      # full slots in the coefficient domain are fine
    assert "host-only" in encode(ctx, n_values=1, log_slots=log_slots, flags=ENC_NTT)[1]


def test_null_and_misaligned_pointers(ctx):
    assert "null values" in encode(ctx, values=None)[1]
    assert "host-only" in encode(ctx, values=None, n_values=0)[1]
    assert "aligned" in encode(ctx, values=ODD)[1]                                    # complex128 input
    assert "host-only" in encode(ctx, values=ODD, flags=ENC_COEFFS, rot=None, roots=None)[1]
    assert "aligned" in encode(ctx, values=BAD, flags=ENC_COEFFS)[1]
    assert "null rot_group" in encode(ctx, rot=None)[1]
    assert "null rot_group" in encode(ctx, roots=None)[1]
    assert "aligned" in encode(ctx, roots=ODD)[1]
    assert "aligned" in encode(ctx, rot=BAD)[1]
    assert "out_q" in encode(ctx, out_q=None)[1]
    assert "out_q" in encode(ctx, out_q=BAD)[1]
    assert "out_p" in encode(ctx, level_p=0, out_p=None)[1]
    assert "out_p" in encode(ctx, level_p=0, out_p=BAD)[1]
    assert "plaintext" in decode(ctx, pt=None)[1]
    assert "plaintext" in decode(ctx, pt=BAD)[1]
    assert "values" in decode(ctx, values=None)[1]
    assert "values" in decode(ctx, values=ODD)[1]
    assert "host-only" in decode(ctx, values=ODD, flags=ENC_COEFFS)[1]
    assert "null rot_group" in decode(ctx, roots=None)[1]
    assert "aligned" in decode(ctx, roots=ODD)[1]


def test_scalar_arguments(ctx):
    for s in (0.0, -1.0, float("inf"), float("nan")):
        assert "scale" in encode(ctx, scale=s)[1]
        assert "scale" in decode(ctx, scale=s)[1]
    for lp in (0.5, 1024.0, -1023.0, float("nan")):
        assert "logprec" in decode(ctx, logprec=lp)[1]
    assert "host-only" in decode(ctx, logprec=0.5, flags=ENC_COEFFS)[1]               # unused without the FFT
    assert "flags" in encode(ctx, flags=8)[1]
    assert "flags" in decode(ctx, flags=8)[1]
    for b in (0, 65536):
        assert "batch" in encode(ctx, batch=b)[1]
        assert "batch" in decode(ctx, batch=b)[1]
    assert "strides" in encode(ctx, batch=2, vs=3, qs=2 << LOGN)[1]
    assert "strides" in encode(ctx, batch=2, vs=4, qs=(2 << LOGN) - 1)[1]
    assert "host-only" in encode(ctx, batch=2, vs=4, qs=2 << LOGN)[1]
    assert "strides" in decode(ctx, batch=2, ps=(2 << LOGN) - 1, vs=1 << (LOGN - 1))[1]
    assert "strides" in decode(ctx, batch=2, ps=2 << LOGN, vs=(1 << (LOGN - 1)) - 1)[1]
    assert "host-only" in decode(ctx, batch=2, ps=2 << LOGN, vs=1 << (LOGN - 1))[1]

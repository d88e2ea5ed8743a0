"""Host logic of the mpbgv protocols (include/lattigo_b200.h lgpu_mpbgv_*, lattigo_b200/mpbgv.py) without a GPU: every argument check of
the entry points runs before any launch, so also on a host-only context; the reference's GenShare / AggregateShares / Transform errors;
and the restated mask stream (tests/mp_refresh_oracle.py): its range, that it reaches the top bit of t, and that its Philox inputs are
disjoint from every other sampler's."""
import ctypes

import numpy as np
import pytest

from oracle import philox as PH
from tests import mp_refresh_oracle as R

QI = [0x3fffffa8001, 0x1000090001, 0x10000c8001, 0x10000f0001, 0xffff00001]
PJ = [0x7fffffd8001]
FAKE = ctypes.c_void_p(1 << 20)          # never dereferenced: every case fails its checks first
N = 1 << 10


@pytest.fixture(scope="module")
def env():
    import lattigo_b200 as lb
    c = lb.Context(10, QI, PJ, device=-1)
    enc = lb.BGVEncoder(c, 0x101)
    yield c, enc
    enc.close()
    c.close()


def _err(rc):
    import lattigo_b200 as lb
    assert rc == -1
    return lb.lib().lgpu_last_error().decode()


def _addr(k):
    return ctypes.c_void_p(k << 24)


def test_entry_points_refuse_bad_arguments_before_any_launch(env):
    import lattigo_b200 as lb
    L = lb.lib()
    ctx, enc = env
    h = enc.h
    big = (4 + 1) * N
    assert "null encoder" in _err(L.lgpu_mpbgv_sample_mask(None, 1, 1, FAKE, 1, None))
    assert "batch out of range" in _err(L.lgpu_mpbgv_sample_mask(h, 1, 1, FAKE, 0, None))
    assert "batch out of range" in _err(L.lgpu_mpbgv_sample_mask(h, 1, 1, FAKE, 65536, None))
    assert "null argument" in _err(L.lgpu_mpbgv_sample_mask(h, 1, 1, None, 1, None))
    for lvl in (-1, 5):
        assert "level out of range" in _err(L.lgpu_mpbgv_e2s_share(h, lvl, FAKE, big, FAKE, FAKE, FAKE, _addr(2), 1, None))
        assert "level out of range" in _err(L.lgpu_mpbgv_s2e_share(h, lvl, FAKE, FAKE, FAKE, FAKE, _addr(2), 1, None))
        assert "level out of range" in _err(L.lgpu_mpbgv_e2s_get_share(h, lvl, FAKE, big, FAKE, None, _addr(2), 1, None))
        assert "level out of range" in _err(L.lgpu_mpbgv_recrypt(h, lvl, FAKE, FAKE, FAKE, _addr(2), 1, None))
    assert "null argument" in _err(L.lgpu_mpbgv_e2s_share(h, 4, FAKE, big, None, FAKE, FAKE, _addr(2), 1, None))
    assert "stride below" in _err(L.lgpu_mpbgv_e2s_share(h, 4, FAKE, big - 1, FAKE, FAKE, FAKE, _addr(2), 1, None))
    assert "overlaps" in _err(L.lgpu_mpbgv_e2s_share(h, 4, FAKE, big, FAKE, FAKE, FAKE, ctypes.c_void_p((1 << 20) + 8), 1, None))
    assert "null argument" in _err(L.lgpu_mpbgv_s2e_share(h, 4, FAKE, FAKE, None, FAKE, _addr(2), 1, None))
    assert "overlaps" in _err(L.lgpu_mpbgv_s2e_share(h, 4, FAKE, FAKE, FAKE, FAKE, FAKE, 1, None))
    assert "null argument" in _err(L.lgpu_mpbgv_e2s_get_share(h, 4, FAKE, big, None, None, _addr(2), 1, None))
    assert "stride below" in _err(L.lgpu_mpbgv_e2s_get_share(h, 4, FAKE, big - N, FAKE, None, _addr(2), 1, None))
    assert "overlaps" in _err(L.lgpu_mpbgv_e2s_get_share(h, 4, FAKE, big, _addr(2), None, ctypes.c_void_p((1 << 20) + 8), 1, None))
    assert "overlaps" in _err(L.lgpu_mpbgv_e2s_get_share(h, 4, FAKE, big, _addr(2), None, _addr(2), 1, None))
    assert "null argument" in _err(L.lgpu_mpbgv_recrypt(h, 4, FAKE, FAKE, None, _addr(2), 1, None))
    assert "overlaps" in _err(L.lgpu_mpbgv_recrypt(h, 4, FAKE, FAKE, _addr(2), _addr(2), 1, None))
    assert "null argument" in _err(L.lgpu_mpbgv_encode_ring_t(h, None, 1, FAKE, 1, None))
    assert "null argument" in _err(L.lgpu_mpbgv_decode_ring_t(h, FAKE, 1, None, 1, None))
    assert "batch out of range" in _err(L.lgpu_mpbgv_decode_ring_t(h, FAKE, 1, FAKE, 0, None))
    # valid arguments reach the device check of the host-only context
    assert "host-only" in _err(L.lgpu_mpbgv_e2s_share(h, 4, FAKE, big, FAKE, FAKE, FAKE, _addr(2), 1, None))
    assert "host-only" in _err(L.lgpu_mpbgv_s2e_share(h, 4, FAKE, FAKE, FAKE, FAKE, _addr(2), 1, None))
    assert "host-only" in _err(L.lgpu_mpbgv_e2s_get_share(h, 4, FAKE, big, FAKE, FAKE, _addr(2), 1, None))
    assert "host-only" in _err(L.lgpu_mpbgv_recrypt(h, 4, FAKE, FAKE, FAKE, _addr(2), 1, None))
    assert "host-only" in _err(L.lgpu_mpbgv_sample_mask(h, 1, 1, FAKE, 1, None))
    assert "host-only" in _err(L.lgpu_mpbgv_encode_ring_t(h, FAKE, 1, FAKE, 1, None))
    assert "host-only" in _err(L.lgpu_mpbgv_decode_ring_t(h, FAKE, 1, FAKE, 1, None))


def _zeros(*shape):
    import torch
    return torch.zeros(shape, dtype=torch.int64)


def test_protocol_errors_carry_the_reference_messages(env):
    import lattigo_b200 as lb
    from lattigo_b200 import mpbgv
    ctx, enc = env
    S = lb.encryptor.Samplers(ctx, 1)
    p = mpbgv.RefreshProtocol(enc, S, 3.2)
    ct = _zeros(2, 2, 2, N)
    with pytest.raises(lb.LgpuError, match="cannot GenShare: ct\\[1\\] level must be at least equal to EncToShareShare level"):
        p.GenShare(None, ct, _zeros(2, 5, N), level=3)
    with pytest.raises(lb.LgpuError, match="cannot GenShare: crp and c0ShareOut level must be equal"):
        p.s2e.GenShare(None, _zeros(2, 5, N), _zeros(2, enc.n), level=3)
    a = mpbgv.RefreshShare(_zeros(2, 2, N), _zeros(2, 5, N), mpbgv.MetaData(3))
    b = mpbgv.RefreshShare(_zeros(2, 1, N), _zeros(2, 5, N), mpbgv.MetaData(3))
    c = mpbgv.RefreshShare(_zeros(2, 2, N), _zeros(2, 4, N), mpbgv.MetaData(3))
    with pytest.raises(lb.LgpuError, match="cannot AggregateShares: all e2s shares must be at the same level"):
        p.AggregateShares(a, b)
    with pytest.raises(lb.LgpuError, match="cannot AggregateShares: all s2e shares must be at the same level"):
        p.AggregateShares([a, c])
    with pytest.raises(lb.LgpuError, match="cannot Transform: input ct.MetaData != share.MetaData"):
        p.Finalize(ct, _zeros(2, 5, N), a, scale=2)
    with pytest.raises(lb.LgpuError, match="cannot Transform: input ciphertext level must be at least equal to e2s level"):
        p.Finalize(_zeros(2, 2, 1, N), _zeros(2, 5, N), a, scale=3)
    with pytest.raises(lb.LgpuError, match="cannot Transform: crs level and s2e level must be the same"):
        p.Finalize(ct, _zeros(2, 4, N), a, scale=3)
    with pytest.raises(lb.LgpuError, match="cannot GetEncryption"):
        p.s2e.GetEncryption(_zeros(2, 5, N), _zeros(2, 4, N))


@pytest.mark.parametrize("t", [0x101, 0xffc001, (3 << 40) + 1])
def test_mask_stream_is_uniform_below_t_and_reaches_the_top_bit(t):
    n, batch = 4096, 3
    m = R.sample_mask(0xABCDEF, 7, t, n, batch)
    assert int(m.max()) < t
    top = 1 << (t.bit_length() - 1)
    assert (m >= np.uint64(top)).any()          # values with t's top bit set occur
    assert (m < np.uint64(top)).any()
    # the entries of a batch and the streams of two ids differ
    assert not np.array_equal(m[0], m[1])
    assert not np.array_equal(m, R.sample_mask(0xABCDEF, 8, t, n, batch))
    # mean of a uniform draw in [0, t): within 6 standard errors
    sd = t / np.sqrt(12 * m.size)
    assert abs(float(m.astype(np.float64).mean()) - (t - 1) / 2) < 6 * sd


def test_mask_counters_are_disjoint_from_every_other_sampler():
    """The mask's polynomial word has bit 29 set; the uniform's is batch * 128 + limb < 2^23 and the other kinds' is the batch index,
    each with its kind in bits 30..31. So no (kind, polynomial) word of another sampler equals a mask's, whatever the seed and id."""
    mask_words = {PH.KIND_UNIFORM << PH.KIND_SHIFT | b | R.MASK_DOMAIN for b in (0, 1, 65534)}
    other = {PH.KIND_UNIFORM << PH.KIND_SHIFT | (65534 * PH.MAX_ROWS + PH.MAX_ROWS - 1)}
    other |= {k << PH.KIND_SHIFT | b for k in (PH.KIND_TERNARY_P, PH.KIND_TERNARY_H, PH.KIND_GAUSSIAN) for b in (0, 65534)}
    assert 65535 * PH.MAX_ROWS + PH.MAX_ROWS <= R.MASK_DOMAIN
    assert not mask_words & other
    for w in mask_words:
        assert (w >> PH.KIND_SHIFT) == PH.KIND_UNIFORM and w & R.MASK_DOMAIN

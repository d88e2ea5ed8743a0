"""Host logic of the mpckks protocols (lgpu_mpckks_*, lattigo_b200/mpckks.py) without a GPU: GetMinimumLevelForRefresh against the
reference's formula on both test sets for K = 1..8, the scale rounding (defaultScale, inputScaleInt) and big.Int.Quo's truncation of
negative masks, the share word rule, the big-mask stream's range and sign split, every argument refusal on a host-only context, and an
oracle anchor: on testInsecurePrec45 and testInsecurePrec90 (checked as integers) the E2S shares of K parties sum to the centred
decryption within the smudging noise, and a refresh decrypts to the input times defaultScale / inputScaleInt within its bound."""
import ctypes
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests import mp_refresh_oracle as R
from tests import multiparty_oracle as M

P45 = [0x80000000080001, 0x2000000a0001, 0x2000000e0001, 0x2000001d0001, 0x1fffffcf0001, 0x1fffffc20001, 0x200000440001]
P90 = [0x80000000080001, 0x80000000440001, 0x2000000a0001, 0x2000000e0001, 0x1fffffc20001, 0x200000440001, 0x200000500001,
       0x200000620001, 0x1fffff980001, 0x2000006a0001, 0x1fffff7e0001, 0x200000860001]
FAKE = ctypes.c_void_p(1 << 20)


@pytest.mark.parametrize("moduli,log_scale", [(P45, 45), (P90, 90)])
@pytest.mark.parametrize("K", range(1, 9))
def test_minimum_level_for_refresh_matches_the_reference_formula(moduli, log_scale, K):
    from lattigo_b200 import mpckks
    lvl, log_bound, ok = mpckks.GetMinimumLevelForRefresh(128, 2.0 ** log_scale, K, moduli)
    assert ok and log_bound == 128 + log_scale
    need = math.ceil(log_bound + math.log2(K))
    logq = [sum(math.log2(q) for q in moduli[: i + 1]) for i in range(len(moduli))]
    assert logq[lvl] >= need and (lvl == 0 or logq[lvl - 1] < need)
    Q = math.prod(moduli[: lvl + 1])
    assert Q > 1 << log_bound                               # GenShare's bound check passes at that level


def test_scale_rounding_and_truncation():
    from lattigo_b200 import mpckks
    assert mpckks.input_scale_int(Fraction(2) ** 45) == 1 << 45
    assert mpckks.input_scale_int(Fraction(2) ** 45 * Fraction(5, 3)) == -(-(5 << 45) // 3)          # ceiling
    assert mpckks.input_scale_int(2.5) == 3
    assert mpckks.default_scale_int(Fraction(2) ** 90) == 1 << 90
    assert mpckks.default_scale_int((1 << 60) + 1, 53) == 1 << 60                                      # rounded to 53 bits first
    assert mpckks.default_scale_int(Fraction(7, 2), 53) == 3                                            # then truncated
    assert R.quo(-7, 2) == -3 and R.quo(7, 2) == 3 and R.quo(-1, 3) == 0 and R.quo(-6, 3) == -2
    d, s = 1 << 90, -(-(5 << 90) // 3)
    for v in (-(1 << 217), -12345, -1, 0, 1, (1 << 217) - 1):
        assert R.quo(v * d, s) == int(Fraction(v * d, s))                                                 # toward zero


def test_share_words_rule():
    import lattigo_b200 as lb
    ctx = lb.Context(10, P90, [0xffffffffffc0001], device=-1)
    try:
        assert lb.mpckks.share_words(ctx, 0) == 4
        bits = [sum(q.bit_length() for q in P90[: i + 1]) + 16 for i in range(len(P90))]
        for lvl, b in enumerate(bits):
            if b <= 256:
                assert lb.mpckks.share_words(ctx, lvl) == 4
            elif b <= 512:
                assert lb.mpckks.share_words(ctx, lvl) == 8
    finally:
        ctx.close()


@pytest.mark.parametrize("log_bound", [45, 64, 173, 218])
def test_big_mask_stream_range_and_sign_split(log_bound):
    vals = R.sample_big_mask(0xBEEF, 3, log_bound, 2048, 2)
    flat = [v for row in vals for v in row]
    half = 1 << (log_bound - 1)
    assert all(-half <= v < half for v in flat)
    neg = sum(v < 0 for v in flat)
    assert 0.45 < neg / len(flat) < 0.55
    assert max(abs(v) for v in flat) >= half >> 4                          # the top bits are reached
    assert vals[0] != vals[1] and vals != R.sample_big_mask(0xBEEF, 4, log_bound, 2048, 2)
    assert R.BIG_MASK_DOMAIN | R.MASK_DOMAIN > 65535 * 128 + 128 and R.BIG_MASK_DOMAIN != R.MASK_DOMAIN


def test_entry_points_refuse_bad_arguments_before_any_launch():
    import lattigo_b200 as lb
    L = lb.lib()
    ctx = lb.Context(10, P45, [0x80000000130001], device=-1)
    h = ctx.h
    err = lambda rc: (rc == -1) and L.lgpu_last_error().decode()
    big = 7 * 1024
    try:
        assert "null context" in err(L.lgpu_mpckks_sample_mask(None, 9, 173, 4, 1, 1, FAKE, 1, None))
        assert "log_slots out of range" in err(L.lgpu_mpckks_sample_mask(h, 10, 173, 4, 1, 1, FAKE, 1, None))
        assert "W must be 4 or 8" in err(L.lgpu_mpckks_sample_mask(h, 9, 173, 5, 1, 1, FAKE, 1, None))
        assert "log_bound out of" in err(L.lgpu_mpckks_sample_mask(h, 9, 256, 4, 1, 1, FAKE, 1, None))
        assert "batch out of range" in err(L.lgpu_mpckks_sample_mask(h, 9, 173, 4, 1, 1, FAKE, 0, None))
        assert "not large enough for refresh correctness" in err(
            L.lgpu_mpckks_e2s_share(h, 2, 9, 173, FAKE, big, FAKE, FAKE, FAKE, 4, ctypes.c_void_p(1 << 30), 1, None))
        assert "level out of range" in err(L.lgpu_mpckks_e2s_share(h, 7, 9, 173, FAKE, big, FAKE, FAKE, FAKE, 4, ctypes.c_void_p(1 << 30), 1, None))
        assert "stride below" in err(L.lgpu_mpckks_e2s_share(h, 3, 9, 173, FAKE, 10, FAKE, FAKE, FAKE, 4, ctypes.c_void_p(1 << 30), 1, None))
        assert "overlaps" in err(L.lgpu_mpckks_e2s_share(h, 3, 9, 173, FAKE, big, FAKE, FAKE, FAKE, 4, FAKE, 1, None))
        sc = (ctypes.c_uint64 * 4)(0, 0, 1, 0)
        assert "positive" in err(L.lgpu_mpckks_s2e_share(h, 6, 9, FAKE, FAKE, FAKE, FAKE, 4, sc, ctypes.c_void_p(1 << 30), 1, None))
        assert "overlaps" in err(L.lgpu_mpckks_e2s_get_share(h, 3, 9, FAKE, big, ctypes.c_void_p(1 << 30), None, 4, FAKE, 1, None))
        ok = (ctypes.c_uint64 * 4)(1, 0, 1, 0)
        assert "null argument" in err(L.lgpu_mpckks_refresh_finalize(h, 3, 9, FAKE, big, FAKE, 6, FAKE, FAKE, 4, None, ctypes.c_void_p(1 << 30), 1, None))
        assert "host-only" in err(L.lgpu_mpckks_e2s_share(h, 3, 9, 173, FAKE, big, FAKE, FAKE, FAKE, 4, ctypes.c_void_p(1 << 30), 1, None))
        assert "host-only" in err(L.lgpu_mpckks_refresh_finalize(h, 3, 9, FAKE, big, FAKE, 6, ctypes.c_void_p(1 << 31), ctypes.c_void_p(1 << 32), 4, ok,
                                                                 ctypes.c_void_p(1 << 33), 1, None))
    finally:
        ctx.close()


def test_protocol_errors_carry_the_reference_messages():
    import torch
    import lattigo_b200 as lb
    ctx = lb.Context(10, P45, [0x80000000130001], device=-1)
    try:
        p = lb.mpckks.RefreshProtocol(ctx, lb.encryptor.Samplers(ctx, 1), 3.2, 2.0 ** 45)
        z = lambda *s: torch.zeros(s, dtype=torch.int64)
        a = lb.mpckks.RefreshShare(z(1, 4, 1024), z(1, 7, 1024), lb.mpckks.MetaData(Fraction(2) ** 45, 9))
        with pytest.raises(lb.LgpuError, match="ct\\[1\\] level must be at least equal to EncToShareShare level"):
            p.GenShare(None, 173, z(1, 2, 3, 1024), z(1, 7, 1024), 2.0 ** 45, 9, level=3)
        with pytest.raises(lb.LgpuError, match="input ciphertext MetaData is not equal to share.MetaData"):
            p.Finalize(z(1, 2, 4, 1024), z(1, 7, 1024), a, 2.0 ** 44, 9)
        with pytest.raises(lb.LgpuError, match="input ciphertext level must be at least equal to e2s level"):
            p.Finalize(z(1, 2, 3, 1024), z(1, 7, 1024), a, 2.0 ** 45, 9)
        with pytest.raises(lb.LgpuError, match="crs level and s2e level must be the same"):
            p.Finalize(z(1, 2, 4, 1024), z(1, 6, 1024), a, 2.0 ** 45, 9)
        with pytest.raises(lb.LgpuError, match="all e2s shares must be at the same level"):
            p.AggregateShares(a, lb.mpckks.RefreshShare(z(1, 3, 1024), z(1, 7, 1024), a.MetaData))
        with pytest.raises(lb.LgpuError, match="below 2\\^128"):
            lb.mpckks._scales(1 << 128, 1)
    finally:
        ctx.close()


@pytest.mark.parametrize("moduli,log_scale,K", [(P45, 45, 3), (P90, 90, 2)])
def test_oracle_refresh_decrypts_and_shares_recombine(moduli, log_scale, K):
    from lattigo_b200 import mpckks
    params = O.Parameters(10, moduli, [])
    P = R.MPCKKS(params)
    rng = np.random.default_rng(log_scale + K)
    N = params.N()
    s = [rng.integers(-1, 2, N) for _ in range(K)]
    sk = [M.sk_rows(params, si) for si in s]
    ideal = M.sk_rows(params, sum(s))
    lvl, log_bound, _ = mpckks.GetMinimumLevelForRefresh(128, 2.0 ** log_scale, K, moduli)
    log_slots, top = 7, len(moduli) - 1
    dslots, gap = 2 << log_slots, N // (2 << 7)
    m = [0] * N
    for j in range(0, N, gap):
        m[j] = int(rng.integers(-(1 << 40), 1 << 40)) << (log_scale - 41)
    ct = P.encrypt_coeffs(ideal, m, lvl + 1, H.rand_poly(moduli[: lvl + 2], N, rng), np.rint(rng.normal(0, 3.2, N)).astype(np.int64))
    scale = Fraction(2) ** log_scale * Fraction(7, 5)
    d, sc = mpckks.default_scale_int(Fraction(2) ** log_scale), mpckks.input_scale_int(scale)
    e = lambda: np.clip(np.rint(rng.normal(0, 4.6, N)), -27, 27).astype(np.int64)
    masks = [[int(v) for v in R.sample_big_mask(99 + i, 1, log_bound, dslots, 1)[0]] for i in range(K)]
    crp = H.rand_poly(moduli, N, rng)
    e2s = [P.e2s_share(lvl, sk[i], ct[1], e(), masks[i]) for i in range(K)]
    s2e = [P.s2e_share(top, sk[i], crp, e(), P.scale(masks[i], d, sc)) for i in range(K)]
    agg_e2s, agg_s2e = M.aggregate(e2s, moduli[: lvl + 1]), M.aggregate(s2e, moduli)
    rec = P.get_share(lvl, ct[0], agg_e2s, dslots, masks[0])
    for i in range(1, K):
        rec = [a + b for a, b in zip(rec, masks[i])]
    assert max(abs(rec[i] - m[i * gap]) for i in range(dslots)) <= K * 27 + 20
    out = P.finalize(lvl, ct, agg_e2s, agg_s2e, crp, dslots, d, sc)
    dec = P.decrypt_coeffs(ideal, out)
    assert max(abs(dec[j] - R.quo(m[j] * d, sc)) for j in range(0, N, gap)) <= 2 * K * 27 + 20 + K + 1

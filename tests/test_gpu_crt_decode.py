"""The multiword CRT decoders on the device (dec_crt_kernel<W> under lgpu_ckks_decode, bgv_dec_crt_kernel<W> under lgpu_bgv_decode,
both on csrc/crt.cuh) at W = 16, 32 and 64, tolerance ZERO, at the chains and edge sets of tests/crt_cases.py (N = 2^10):

- the levels where the summed bit lengths fill 16, 32 and 64 words exactly (Q has its top bit in word W - 1) and the levels one prime
  later, which switch 16 -> 32 and 32 -> 64 words; a second chain puts 45-bit (FP64-pipe) rows inside the W = 32 and W = 64 prefixes;
- CKKS: DecodeCoeffs at scales 1, 2^40, 2^40 + 1 and one that makes small results subnormal, against Float64(centred X) / scale and
  oracle.encoder.decode_public; Decode through the special FFT at full and sparse slots; batch 3 at a padded stride with rows above the
  level holding a sentinel; the plaintext never written;
- BGV at gap > 1 (t = 257 and a 60-bit t): signed and unsigned, scale 1 and random, against oracle.bgv_encoder.Decode;
- the 4096-bit limit: 65 words refused by both decoders before any launch, also where Q itself has fewer than 4096 bits, 64 accepted.

tests/test_crt_model_cpu.py shows that these edge sets reach every branch of the kernels' arithmetic."""
import ctypes
import functools

import numpy as np
import pytest

from oracle import bgv_encoder as BE
from oracle import encoder as E
from oracle import oracle as O
from tests import crt_cases as K
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64
M64 = (1 << 64) - 1
T60 = K.t60()                                  # 512 slots at gap 2
SENTINEL = 0xDEADBEEFDEADBEEF
E_NTT, E_COEFFS, E_SIGNED = 1, 4, 8             # LGPU_ENC_* flags of the direct C ABI calls

LEVELS = [("A", lv) for lv, (_, W) in K.BOUNDARY_A.items() if W] + [("B", lv) for lv in K.BOUNDARY_B]


@functools.lru_cache(None)
def _chain(name):
    import lattigo_b200 as lb
    q = {"A": K.chain_a, "B": K.chain_b, "R": K.chain_r}[name]()
    return q, lb.Context(K.LOGN, q, []), O.Parameters(K.LOGN, q, [])


@functools.lru_cache(None)
def _bgv(name, t):
    import lattigo_b200 as lb
    q, ctx, params = _chain(name)
    return lb.BGVEncoder(ctx, t), BE.BGVEncoder(params.ringQ, t)


def _same_doubles(got, want):
    g, w = np.asarray(got).view(np.float64), np.asarray(want).view(np.float64)
    gn, wn = np.isnan(g), np.isnan(w)
    assert np.array_equal(gn, wn), "NaN positions differ"
    bad = np.nonzero(g[~gn].view(U64) != w[~wn].view(U64))[0]
    assert bad.size == 0, (bad[:8], g[~gn][bad[:8]], w[~wn][bad[:8]])


def _placed(C, xs, gap, seed):
    """N coefficients: the edge values at j * gap (the coefficients the decoder reads), uniform values of [0, Q) everywhere else."""
    rng = np.random.default_rng(seed)
    X = K.fill_uniform([], K.N, C.Q, rng)
    used = K.fill_uniform(xs, K.N // gap, C.Q, rng)
    X[::gap] = used
    return X


def _ntt(params, level, rows):
    out = np.array(rows, dtype=U64)
    params.ringQ.AtLevel(level).NTT(out, out)
    return out


def _edges(name, level):
    q, ctx, params = _chain(name)
    C = K.Crt(q, level)
    assert C.W == K.crt_width(K.crt_words(q, level))
    return q, ctx, params, C, K.edge_values(C, np.random.default_rng(level))


@pytest.mark.parametrize("name,level", LEVELS)
def test_ckks_decode_coeffs_and_slots(name, level):
    import lattigo_b200 as lb
    q, ctx, params, C, xs = _edges(name, level)
    enc = lb.Encoder(ctx)
    X = _placed(C, xs, 1, level)
    pt = K.rows_of(X, q, level)
    d = ctx.to_device(pt)
    for s in (1.0, 2.0 ** 40, 2.0 ** 40 + 1, 1.75 * 2.0 ** 1023):
        got = enc.DecodeCoeffs(d, s, ntt=False).cpu().numpy()
        _same_doubles(got, np.array([K.to_float64(K.centred(x, C.Q)) / s for x in X]))
        _same_doubles(got, np.array(E.decode_public(params.ringQ, pt, level, 0, s, False, is_batched=False)))
    assert np.array_equal(ctx.to_host(d), pt)
    ptn = _ntt(params, level, pt)
    got = enc.DecodeCoeffs(ctx.to_device(ptn), 2.0 ** 40, ntt=True).cpu().numpy()
    _same_doubles(got, np.array([K.to_float64(K.centred(x, C.Q)) / 2.0 ** 40 for x in X]))
    # slots: full (gap 1, every coefficient) and 64 slots (gap 8: the edge values sit on the 128 coefficients read)
    for log_slots in (K.LOGN - 1, 6):
        gap = (K.N // 2) >> log_slots
        Xs = _placed(C, xs, gap, level + log_slots)
        ptn = _ntt(params, level, K.rows_of(Xs, q, level))
        dn = ctx.to_device(ptn)
        got = enc.Decode(dn, 2.0 ** 40, log_slots, ntt=True).cpu().numpy()
        _same_doubles(got, np.array(E.decode_public(params.ringQ, ptn, level, log_slots, 2.0 ** 40, True), dtype=np.complex128))
        assert np.array_equal(ctx.to_host(dn), ptn)


def _padded(ctx, entries, level, extra_rows=2, pad=37):
    """Batch entries at a stride of (level + 1 + extra_rows) N + pad words, rows past `level` and the padding set to SENTINEL."""
    import torch
    stride = (level + 1 + extra_rows) * K.N + pad
    buf = np.full(len(entries) * stride, SENTINEL, dtype=U64)
    for b, rows in enumerate(entries):
        buf[b * stride: b * stride + (level + 1) * K.N] = np.asarray(rows, dtype=U64).reshape(-1)
    return torch.from_numpy(buf.view(np.int64)).to("cuda:%d" % ctx.device), buf, stride


@pytest.mark.parametrize("name,level", LEVELS)
def test_ckks_batch_at_padded_stride_with_sentinel_rows(name, level):
    import torch
    import lattigo_b200 as lb
    from lattigo_b200 import _lib
    q, ctx, params, C, xs = _edges(name, level)
    enc = lb.Encoder(ctx)
    entries = [_ntt(params, level, K.rows_of(_placed(C, xs[b:] + xs[:b], 1, 7 * level + b), q, level)) for b in range(3)]
    d, host, stride = _padded(ctx, entries, level)
    for coeffs, log_slots in ((True, K.LOGN - 1), (False, 5)):
        n = K.N if coeffs else 1 << log_slots
        vstride = n + 3
        out = torch.full((3 * vstride,), -7.0, dtype=torch.float64 if coeffs else torch.complex128, device=d.device)
        flags = E_NTT | (E_COEFFS if coeffs else 0)
        _lib.check(_lib.lib().lgpu_ckks_decode(ctx.h, ctypes.c_void_p(d.data_ptr()), level, log_slots, 2.0 ** 40, flags, 0.0,
                                               ctypes.c_void_p(enc.rot_group.data_ptr()), ctypes.c_void_p(enc.roots.data_ptr()),
                                               ctypes.c_void_p(out.data_ptr()), 3, stride, vstride, None))
        got = out.cpu().numpy()
        for b in range(3):
            want = E.decode_public(params.ringQ, entries[b], level, log_slots, 2.0 ** 40, True, is_batched=not coeffs)
            _same_doubles(got[b * vstride: b * vstride + n], np.array(want, dtype=np.float64 if coeffs else np.complex128))
            if b < 2:                                                # the gap between entries is not written
                assert np.all(got[b * vstride + n: (b + 1) * vstride] == -7.0)
    assert np.array_equal(d.cpu().numpy().view(U64), host)         # neither the plaintext nor the sentinel rows are written


def _bgv_rows(C, q, level, t, xs, gap, seed):
    """Rows whose value after RingQ2T's MulScalar(t) is X: X t^-1 mod Q, the edge values on the decoder's coefficients j * gap."""
    X = _placed(C, xs, gap, seed)
    return K.rows_of(X, q, level, mul=pow(t, -1, C.Q))


@pytest.mark.parametrize("t", [257, T60])
@pytest.mark.parametrize("name,level", LEVELS)
def test_bgv_decode_gap_above_one(name, level, t):
    q, ctx, params, C, xs = _edges(name, level)
    enc, oenc = _bgv(name, t)
    n = enc.MaxSlots()
    gap = K.N // n
    assert gap > 1 and n == (128 if t == 257 else 512)
    rng = np.random.default_rng(level)
    pt = _bgv_rows(C, q, level, t, xs, gap, level)
    ptn = _ntt(params, level, pt)
    scale = int(rng.integers(2, M64, dtype=U64))
    for rows, ntt in ((pt, False), (ptn, True)):
        d = ctx.to_device(rows)
        for signed in (False, True):
            for s in (1, scale):
                got = enc.Decode(d, s, ntt=ntt, signed=signed).cpu().numpy()
                want = oenc.Decode(rows, level, s, ntt, True, signed)
                assert np.array_equal(got.view(U64), np.array([x & M64 for x in want], dtype=U64)), (ntt, signed, s)
        assert np.array_equal(ctx.to_host(d), rows)
    # batch 3 at a padded stride, rows past the level holding a sentinel
    import torch
    from lattigo_b200 import _lib
    entries = [_bgv_rows(C, q, level, t, xs[b:] + xs[:b], gap, 11 * level + b) for b in range(3)]
    d, host, stride = _padded(ctx, entries, level)
    vstride = n + 5
    out = torch.full((3 * vstride,), -7, dtype=torch.int64, device=d.device)
    _lib.check(_lib.lib().lgpu_bgv_decode(enc.h, ctypes.c_void_p(d.data_ptr()), level, E_SIGNED, scale, ctypes.c_void_p(out.data_ptr()), 3,
                                          stride, vstride, None))
    got = out.cpu().numpy()
    for b in range(3):
        assert np.array_equal(got[b * vstride: b * vstride + n], np.array(oenc.Decode(entries[b], level, scale, False, True, True)))
        if b < 2:
            assert np.all(got[b * vstride + n: (b + 1) * vstride] == -7)
    assert np.array_equal(d.cpu().numpy().view(U64), host)


@pytest.mark.parametrize("name,level,words", [("A", 68, 65), ("R", K.REFUSE_R, 65)])
def test_refused_past_64_words_before_any_launch(name, level, words):
    """65 words: refused by both decoders before anything runs, including chain R, whose Q has only 4081 bits (the rule is the
    summed bit lengths of q_0..q_level). One level below: 64 words, accepted and launched."""
    import lattigo_b200 as lb
    q, ctx, params = _chain(name)
    assert K.crt_words(q, level) == words and K.crt_words(q, level - 1) == 64
    enc, benc = lb.Encoder(ctx), _bgv(name, 257)[0]
    rng = np.random.default_rng(level)
    pt = ctx.to_device(H.rand_poly(q[: level + 1], K.N, rng))
    calls = [lambda p: enc.DecodeCoeffs(p, 2.0 ** 40, ntt=False), lambda p: enc.Decode(p, 2.0 ** 40, 6, ntt=True),
             lambda p: benc.Decode(p, 3, ntt=False), lambda p: benc.Decode(p, 3, ntt=True, signed=True)]
    for call in calls:
        def refused():
            with pytest.raises(lb.LgpuError, match="exceeds 4096 bits"):
                call(pt)
        assert H.launch_delta(refused) == 0
        assert H.launch_delta(lambda: call(pt[:level].contiguous())) > 0

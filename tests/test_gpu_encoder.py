"""lgpu_ckks_encode / lgpu_ckks_decode (csrc/encoder.cu) against oracle/encoder.py with tolerance ZERO: plaintext words compared as uint64,
decoded doubles through their 64-bit patterns, NaN positions required to match. Covers N = 2^8 .. 2^12 at every log_slots (NTT, NTT +
Montgomery, and the coefficient domain at full slots; with and without P rows; batch 1 and 3; fewer values than slots), scales up to
2^62 so that every quantisation branch is reached, PN16QP1761 at level 33 with 4 P rows and BOOT_N16QP1767 with its 61-bit P rows,
decoding at level 0 and above (level 33 on uniform residues, where the CRT value passes 2^1024 and the FFT meets Inf and NaN), logprec
rounding, coefficient mode, a device encrypt / decrypt round trip and a Montgomery plaintext-ciphertext product."""
import numpy as np
import pytest

from lattigo_b200.params import PRESETS
from oracle import encoder as E
from oracle import encryptor as ENC
from oracle import oracle as O

pytestmark = pytest.mark.gpu
U64 = np.uint64


def _same_doubles(got, want):
    g, w = np.asarray(got).view(np.float64), np.asarray(want).view(np.float64)
    gn, wn = np.isnan(g), np.isnan(w)
    assert np.array_equal(gn, wn), "NaN positions differ"
    assert np.array_equal(g[~gn].view(U64), w[~wn].view(U64)), float(np.nanmax(np.abs(g - w)))


def _values(rng, batch, n):
    mag = 10.0 ** rng.uniform(-13, 1, (batch, n))            # from below one unit at scale 2^40 to past 2^64 / 2^62
    v = mag * (rng.normal(size=(batch, n)) + 1j * rng.normal(size=(batch, n)))
    v[:, ::7] = 0
    return v


def _setup(logN, logQ, logP):
    import lattigo_b200 as lb
    q, p = O.gen_moduli(logN + 1, logQ, logP)
    ctx = lb.Context(logN, q, p)
    return ctx, O.Parameters(logN, q, p), lb.Encoder(ctx)


def _check_tables(enc, m):
    assert np.array_equal(enc.rot_group.cpu().numpy(), np.array(E.rot_group(m)))
    assert np.array_equal(enc.roots.cpu().numpy().view(U64), np.array(E.get_roots_complex128(m), dtype=np.complex128).view(U64))


def _encode_and_compare(ctx, params, enc, v, log_slots, scale, ntt, mont, level_q, level_p):
    got = ctx.to_host(enc.Encode(v, level_q, scale, ntt=ntt, montgomery=mont, level_p=level_p, log_slots=log_slots))
    for b in range(v.shape[0]):
        pq, pp = E.embed_double(params.ringQ, params.ringP, v[b], log_slots, scale, ntt, mont, level_q, level_p)
        want = pq if pp is None else np.concatenate([pq, pp])
        assert np.array_equal(got[b], want), (log_slots, ntt, mont, level_q, level_p, b)
    return got


@pytest.mark.parametrize("logN", [8, 9, 10, 11, 12])
def test_encode_matches_oracle(logN):
    ctx, params, enc = _setup(logN, [55, 45, 45], [61, 55])
    try:
        _check_tables(enc, 2 << logN)
        rng = np.random.default_rng(logN)
        k = 0
        for log_slots in range(logN):
            slots = 1 << log_slots
            full = log_slots == logN - 1
            for ntt, mont in ((True, False), (True, True)) + (((False, False), (False, True)) if full else ()):
                batch = 3 if k % 2 else 1
                level_p = (k // 2) % 3 - 1                         # -1, 0, 1
                n = max(1, slots - (k % 3))
                scale = (2.0 ** 40, 2.0 ** 62, 2.0 ** 21)[k % 3]
                _encode_and_compare(ctx, params, enc, _values(rng, batch, n), log_slots, scale, ntt, mont, 2 - k % 2, level_p)
                k += 1
        # IsBatched = false
        for ntt in (True, False):
            v = _values(rng, 3, ctx.N - 3).real
            got = ctx.to_host(enc.EncodeCoeffs(v, 2, 2.0 ** 62, ntt=ntt))
            for b in range(3):
                assert np.array_equal(got[b], E.encode_coeffs(params.ringQ, v[b], 2, 2.0 ** 62, ntt))
    finally:
        ctx.close()


def test_quantisation_reaches_every_branch():
    """The words the coefficient-domain output keeps: 0, q, q - c, unreduced c > q, BRedAdd(c) past 2^61 - 1, big.Int residues."""
    logN = 8
    ctx, params, enc = _setup(logN, [45, 61], [])
    try:
        q0, q1 = params.qi
        N = ctx.N
        v = np.zeros(N)
        v[:12] = [0.0, -0.0, 1.5, 0.49999999999999994, -0.1, -3.0, -(2.0 ** 50), 2.0 ** 50, 2.0 ** 62, 3 * 2.0 ** 70, -3 * 2.0 ** 70, 2.0 ** 64]
        got = ctx.to_host(enc.EncodeCoeffs(v, 1, 1.0, ntt=False))
        want = E.encode_coeffs(params.ringQ, v, 1, 1.0, False)
        assert np.array_equal(got, want)
        assert int(got[0, 4]) == q0 and int(got[1, 4]) == q1 and int(got[0, 7]) == 2 ** 50 > q0
    finally:
        ctx.close()


def _preset_ctx(name):
    import lattigo_b200 as lb
    pr = PRESETS[name]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    return ctx, O.Parameters(pr["logN"], pr["Q"], pr["P"]), lb.Encoder(ctx)


@pytest.mark.parametrize("name,level_p,batch,log_slots", [("CKKS_PN16QP1761", 3, 4, 15), ("BOOT_N16QP1767", 5, 2, 12)])
def test_encode_large_presets(name, level_p, batch, log_slots):
    ctx, params, enc = _preset_ctx(name)
    try:
        rng = np.random.default_rng(len(name))
        v = _values(rng, batch, 1 << log_slots)
        _encode_and_compare(ctx, params, enc, v, log_slots, 2.0 ** 45, True, True, len(params.qi) - 1, level_p)
    finally:
        ctx.close()


def _decode_and_compare(ctx, params, enc, pt, level, log_slots, scale, ntt, logprec=0, coeffs=False):
    d = ctx.to_device(pt)
    got = (enc.DecodeCoeffs(d, scale, ntt=ntt) if coeffs else enc.Decode(d, scale, log_slots, ntt=ntt, logprec=logprec)).cpu().numpy()
    for b in range(pt.shape[0]):
        want = np.array(E.decode_public(params.ringQ, pt[b], level, log_slots, scale, ntt, logprec, is_batched=not coeffs),
                        dtype=np.float64 if coeffs else np.complex128)
        _same_doubles(got[b], want)
    assert np.array_equal(ctx.to_host(d), pt)                  # the plaintext is not written


def _uniform(params, level, batch, rng, N):
    return np.stack([np.stack([rng.integers(0, q, N, dtype=U64) for q in params.qi[: level + 1]]) for _ in range(batch)])


@pytest.mark.parametrize("logN", [8, 10, 12])
def test_decode_matches_oracle(logN):
    ctx, params, enc = _setup(logN, [55, 45, 45, 45], [])
    try:
        rng = np.random.default_rng(100 + logN)
        N = ctx.N
        for level in (0, 1, 3):
            for log_slots in range(logN):
                batch = 3 if log_slots % 2 else 1
                v = _values(rng, batch, 1 << log_slots) * 1e-9
                pt = ctx.to_host(enc.Encode(v, level, 2.0 ** 40, log_slots=log_slots))
                _decode_and_compare(ctx, params, enc, pt, level, log_slots, 2.0 ** 40, True, logprec=(0, 20, -3)[log_slots % 3])
            # uniform residues (huge centred values), NTT and coefficient domain, and non-canonical words (>= q, the q itself)
            pt = _uniform(params, level, 2, rng, N)
            pt[:, 0, :4] = [params.qi[0], params.qi[0] + 5, (1 << 61) - 1, params.qi[0] >> 1]
            for ntt in (False, True):
                if ntt:
                    pt = pt % np.array(params.qi[: level + 1], dtype=U64)[None, :, None]
                _decode_and_compare(ctx, params, enc, pt, level, logN - 1, 2.0 ** 40, ntt)
                _decode_and_compare(ctx, params, enc, pt, level, 3, 2.0 ** 30, ntt, logprec=8)
                _decode_and_compare(ctx, params, enc, pt, level, 0, 2.0 ** 30, ntt, coeffs=True)
    finally:
        ctx.close()


def test_decode_pn16_level33_uniform_inf_nan():
    ctx, params, enc = _preset_ctx("CKKS_PN16QP1761")
    try:
        rng = np.random.default_rng(33)
        level = 33
        pt = _uniform(params, level, 2, rng, ctx.N)
        _decode_and_compare(ctx, params, enc, pt, level, 15, 2.0 ** 45, True)
        got = enc.Decode(ctx.to_device(pt), 2.0 ** 45, 15).cpu().numpy()
        assert np.isnan(got.real).any()                          # the Inf / NaN path is exercised
        _decode_and_compare(ctx, params, enc, pt[:1], level, 0, 2.0 ** 45, False, coeffs=True)
        v = _values(rng, 2, 1 << 15) * 1e-12
        _decode_and_compare(ctx, params, enc, ctx.to_host(enc.Encode(v, level, 2.0 ** 45)), level, 15, 2.0 ** 45, True, logprec=30)
    finally:
        ctx.close()


def test_device_round_trip_and_montgomery_product():
    import torch
    import lattigo_b200 as lb
    logN, level, log_slots, batch = 12, 2, 11, 3
    ctx, params, enc = _setup(logN, [55, 45, 45], [])
    try:
        N = ctx.N
        rng = np.random.default_rng(9)
        s = rng.integers(-1, 2, N)
        sk = ENC.small_rows(s, params.qi)
        params.ringQ.NTT(sk, sk); params.ringQ.MForm(sk, sk)
        d_sk = ctx.to_device(sk)
        skb = d_sk[: level + 1].unsqueeze(0).expand(batch, -1, -1).contiguous()
        v = rng.uniform(-1, 1, (batch, 1 << log_slots)) + 1j * rng.uniform(-1, 1, (batch, 1 << log_slots))
        u = rng.uniform(-1, 1, (batch, 1 << log_slots)) + 1j * rng.uniform(-1, 1, (batch, 1 << log_slots))
        pv = enc.Encode(v, level, 2.0 ** 35)
        c1 = ctx.to_device(_uniform(params, level, batch, rng, N))
        e = torch.from_numpy(np.rint(rng.normal(0, 3.2, (batch, N))).astype(np.int64)).cuda()
        c0 = lb.encryptor.Encryptor(ctx).EncryptZeroSk(level, -1, d_sk, c1, e, True, False)
        r = ctx.ringQ.AtLevel(level)
        r.Add(c0, pv, c0)

        def decrypt(a0, a1):
            out = a0.clone()
            r.MulCoeffsMontgomeryThenAdd(a1, skb, out)
            return out

        got = enc.Decode(decrypt(c0, c1), 2.0 ** 35, log_slots).cpu().numpy()
        assert np.abs(got - v).max() < 2.0 ** -20
        pu = enc.Encode(u, level, 2.0 ** 30, montgomery=True)
        d0, d1 = torch.empty_like(c0), torch.empty_like(c1)
        r.MulCoeffsMontgomery(c0, pu, d0)
        r.MulCoeffsMontgomery(c1, pu, d1)
        dec = decrypt(d0, d1)
        got = enc.Decode(dec, 2.0 ** 65, log_slots).cpu().numpy()
        assert np.abs(got - u * v).max() < 2.0 ** -15
        _decode_and_compare(ctx, params, enc, ctx.to_host(dec), level, log_slots, 2.0 ** 65, True)
    finally:
        ctx.close()

"""lgpu_bgv_encode / lgpu_bgv_decode (csrc/bgv_encoder.cu) against oracle/bgv_encoder.py with tolerance ZERO (every word as uint64):

- N = 2^8 .. 2^12 with t = 65537 (gap 1 up to 2^15 slots), t = 257 (gap > 1) and a 60-bit t under a 61-bit Q[0] (integer-pipe ring-T
  transforms); every flag combination of Encode / Embed, Q-only and Q + P output, edge values (0, t - 1, t, multiples of t, 2^64 - 1,
  INT64_MIN, negative multiples of t), fewer values than slots, batch 1 and 3, scale 1 and random;
- Decode of uniform residues at level 0 and above through all three RingQ2T branches, coefficients at the edges of the float v
  ([t x]_Q in {0, 1, Q/2 - 1, Q/2, Q/2 + 1, Q - 1}), coefficient mode and its signed quirk;
- BGV_N15QP880 (t = 0x10001, level 19, batch 16) and N = 2^16 with gap 2 decoded through the multiword CRT;
- a device round trip: encode, encrypt, MulRelinNew (BGV and BFV) and Rescale, decrypt with ring ops, decode to the slot-wise product;
  and an automorphism by 5^k decoding to the rotated rows."""
import numpy as np
import pytest

from lattigo_b200.params import PRESETS
from oracle import bgv_encoder as BE
from oracle import encryptor as ENC
from oracle import oracle as O

pytestmark = pytest.mark.gpu
U64 = np.uint64
M64 = (1 << 64) - 1


def _setup(logN, logQ, logP, t):
    import lattigo_b200 as lb
    q, p = O.gen_moduli(logN + 1, logQ, logP)
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    return ctx, params, lb.BGVEncoder(ctx, t), BE.BGVEncoder(params.ringQ, t, params.ringP)


def _ntt_prime(bits, m, below=None):
    x = ((below or (1 << bits)) - 1) // m * m + 1
    while not O.is_prime(x):
        x -= m
    return x


def _values(rng, t, batch, n, signed):
    if signed:
        v = rng.integers(-(1 << 62), 1 << 62, (batch, n), dtype=np.int64)
        edge = [0, t - 1, t, -t, 3 * t, -5 * t, -(1 << 63), (1 << 63) - 1, -1, 1]
        v[:, : min(n, len(edge))] = np.array(edge[:n], dtype=np.int64)
    else:
        v = rng.integers(0, M64, (batch, n), dtype=U64, endpoint=True)
        edge = [0, t - 1, t, 2 * t, M64, (1 << 63), 7 * t, 1]
        v[:, : min(n, len(edge))] = np.array(edge[:n], dtype=U64)
    return v


def _cmp_encode(ctx, enc, oenc, v, level, scale, ntt, mont, level_p, scale_up, batched=True):
    signed = v.dtype == np.int64
    if scale_up:
        got = ctx.to_host(enc.Encode(v, level, scale, ntt=ntt, montgomery=mont, batched=batched))
    else:
        got = ctx.to_host(enc.Embed(v, level, scale, ntt=ntt, montgomery=mont, level_p=level_p))
    for b in range(v.shape[0]):
        if scale_up:
            want = oenc.Encode(list(v[b]), signed, scale, ntt, mont, level, batched)
        else:
            pq, pp = oenc.Embed(list(v[b]), signed, scale, ntt, mont, level, level_p)
            want = pq if pp is None else np.concatenate([pq, pp])
        assert np.array_equal(got[b], want), (level, scale, ntt, mont, level_p, scale_up, batched, b)


def _cmp_decode(ctx, enc, oenc, pt, level, scale, ntt, batched=True, signed=False):
    import torch
    d = ctx.to_device(pt)
    n = enc.MaxSlots() if batched else ctx.N
    out = torch.full((pt.shape[0], n), -7, dtype=torch.int64, device=d.device)
    got = enc.Decode(d, scale, ntt=ntt, batched=batched, signed=signed, out=out).cpu().numpy()
    for b in range(pt.shape[0]):
        want = oenc.Decode(pt[b], level, scale, ntt, batched, signed, values=[-7] * n)
        assert np.array_equal(got[b].view(U64), np.array([x & M64 for x in want], dtype=U64)), (level, scale, ntt, batched, signed, b)
    assert np.array_equal(ctx.to_host(d), pt)                  # the plaintext is not written


def _uniform(params, level, batch, rng, N):
    return np.stack([np.stack([rng.integers(0, q, N, dtype=U64) for q in params.qi[: level + 1]]) for _ in range(batch)])


def _float_v_edges(params, level, t, N, rng):
    """Coefficient domain rows whose [t x]_Q is 0, 1, Q/2 - 1, Q/2, Q/2 + 1, Q - 1 (then uniform)."""
    Q = 1
    for q in params.qi[: level + 1]:
        Q *= q
    tinv = pow(t, -1, Q)
    targets = [0, 1, Q // 2 - 1, Q // 2, Q // 2 + 1, Q - 1]
    xs = [y * tinv % Q for y in targets] + [int(rng.integers(0, 1 << 62)) * int(rng.integers(0, 1 << 62)) % Q for _ in range(N - len(targets))]
    return np.stack([np.array([x % q for x in xs], dtype=U64) for q in params.qi[: level + 1]])


CASES = [(8, 65537), (9, 257), (10, 65537), (11, 257), (12, 65537)]


@pytest.mark.parametrize("logN,t", CASES)
def test_encode_matches_oracle(logN, t):
    ctx, params, enc, oenc = _setup(logN, [55, 45, 45], [61, 55], t)
    try:
        rng = np.random.default_rng(logN)
        n = enc.MaxSlots()
        assert n == oenc.MaxSlots() == min(ctx.N, 128 if t == 257 else 1 << 15)
        k = 0
        for scale_up in (True, False):
            for ntt in (True, False):
                for mont in (False, True):
                    for signed in (False, True):
                        batch = 3 if k % 2 else 1
                        level_p = -1 if scale_up else (k // 2) % 3 - 1
                        nv = max(1, n - (k % 3) * 5)
                        scale = 1 if k % 3 == 0 else int(rng.integers(0, M64, dtype=U64, endpoint=True))
                        v = _values(rng, t, batch, nv, signed)
                        _cmp_encode(ctx, enc, oenc, v, 2 - k % 2, scale, ntt, mont, level_p, scale_up)
                        k += 1
        for ntt in (True, False):                                # IsBatched = false (IsMontgomery ignored)
            for signed in (False, True):
                v = _values(rng, t, 3, ctx.N - 3, signed)
                _cmp_encode(ctx, enc, oenc, v, 2, 12345, ntt, True, -1, True, batched=False)
    finally:
        enc.close(); ctx.close()


def test_encode_60bit_t_integer_pipe():
    """t of 60 bits below a 61-bit Q[0]: the ring-T transforms take the integer pipe, and Q rows below t keep the literal Embed words."""
    logN = 10
    q0 = _ntt_prime(61, 2 << logN)
    t = _ntt_prime(60, 1 << 17)
    import lattigo_b200 as lb
    q1 = _ntt_prime(45, 2 << logN)
    p0 = _ntt_prime(55, 2 << logN)
    ctx = lb.Context(logN, [q0, q1], [p0])
    params = O.Parameters(logN, [q0, q1], [p0])
    enc, oenc = lb.BGVEncoder(ctx, t), BE.BGVEncoder(params.ringQ, t, params.ringP)
    try:
        assert enc.MaxSlots() == ctx.N
        rng = np.random.default_rng(60)
        for ntt, mont in ((False, False), (True, False), (False, True), (True, True)):
            for signed in (False, True):
                v = _values(rng, t, 2, ctx.N - 1, signed)
                _cmp_encode(ctx, enc, oenc, v, 1, 3, ntt, mont, 0, False)
                _cmp_encode(ctx, enc, oenc, v, 1, 3, ntt, mont, -1, True)
        pt = _uniform(params, 1, 2, rng, ctx.N)
        for lvl in (0, 1):
            _cmp_decode(ctx, enc, oenc, pt[:, : lvl + 1].copy(), lvl, 5, True, signed=True)
            _cmp_decode(ctx, enc, oenc, pt[:, : lvl + 1].copy(), lvl, 5, False)
    finally:
        enc.close(); ctx.close()


@pytest.mark.parametrize("logN,t", CASES)
def test_decode_matches_oracle(logN, t):
    ctx, params, enc, oenc = _setup(logN, [55, 45, 45, 45], [], t)
    try:
        rng = np.random.default_rng(200 + logN)
        N = ctx.N
        for level in (0, 1, 3):
            v = _values(rng, t, 2, enc.MaxSlots(), True)
            pt = ctx.to_host(enc.Encode(v, level, 3))
            _cmp_decode(ctx, enc, oenc, pt, level, 3, True, signed=True)
            pt = _uniform(params, level, 2, rng, N)
            pt[1] = _float_v_edges(params, level, t, N, rng)
            scale = int(rng.integers(1, M64, dtype=U64))
            for ntt in (True, False):
                _cmp_decode(ctx, enc, oenc, pt, level, scale, ntt)
                _cmp_decode(ctx, enc, oenc, pt, level, 1, ntt, signed=True)
                _cmp_decode(ctx, enc, oenc, pt, level, scale, ntt, batched=False)
                _cmp_decode(ctx, enc, oenc, pt, level, scale, ntt, batched=False, signed=True)   # only the first n words written
            raw = pt.copy()
            raw[:, 0, :3] = [params.qi[0], M64, (1 << 61) - 1]                  # non-canonical coefficient-domain words
            _cmp_decode(ctx, enc, oenc, raw, level, scale, False)
    finally:
        enc.close(); ctx.close()


def _preset(name):
    import lattigo_b200 as lb
    pr = PRESETS[name]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    params = O.Parameters(pr["logN"], pr["Q"], pr["P"])
    return ctx, params


def test_bgv_n15qp880():
    import lattigo_b200 as lb
    ctx, params = _preset("BGV_N15QP880")
    t = PRESETS["BGV_N15QP880"]["T"]
    enc, oenc = lb.BGVEncoder(ctx, t), BE.BGVEncoder(params.ringQ, t, params.ringP)
    try:
        rng = np.random.default_rng(15)
        batch, level = 16, 19
        v = _values(rng, t, batch, enc.MaxSlots(), False)
        got = ctx.to_host(enc.Encode(v, level, 1))
        for b in (0, batch - 1):
            assert np.array_equal(got[b], oenc.Encode(list(v[b]), False, 1, True, False, level))
        e = ctx.to_host(enc.Embed(v[:2], level, 7, ntt=True, montgomery=True, level_p=3))
        pq, pp = oenc.Embed(list(v[1]), False, 7, True, True, level, 3)
        assert np.array_equal(e[1], np.concatenate([pq, pp]))
        d = enc.Decode(ctx.to_device(got), 1).cpu().numpy()
        assert np.array_equal(d.view(U64), v % U64(t))
        for lvl in (0, 19):
            pt = _uniform(params, lvl, 2, rng, ctx.N)
            _cmp_decode(ctx, enc, oenc, pt, lvl, 3, True, signed=True)
    finally:
        enc.close(); ctx.close()


def test_gap2_multiword_crt_at_2_16():
    """N = 2^16, t = 65537: 2^15 slots at gap 2; level 30 of 45-bit primes needs the 32-word CRT, level 10 the 16-word one."""
    import lattigo_b200 as lb
    logN, t = 16, 65537
    q, _ = O.gen_moduli(logN + 1, [55] + [45] * 30, [])
    ctx = lb.Context(logN, q, [])
    params = O.Parameters(logN, q, [])
    enc, oenc = lb.BGVEncoder(ctx, t), BE.BGVEncoder(params.ringQ, t)
    try:
        assert enc.MaxSlots() == 1 << 15
        rng = np.random.default_rng(16)
        for level in (10, 30):
            pt = _uniform(params, level, 1, rng, ctx.N)
            pt[0, :, :6] = _float_v_edges(params, level, t, 6, rng)[:, :6]
            d = ctx.to_device(pt)
            got = enc.Decode(d, 3, ntt=False, signed=True).cpu().numpy()
            want = oenc.Decode(pt[0], level, 3, False, True, True)
            assert np.array_equal(got[0], np.array(want, dtype=np.int64)), level
    finally:
        enc.close(); ctx.close()


def _negacyclic(a, b, t):
    N = len(a)
    full = np.convolve(np.asarray(a, dtype=object), np.asarray(b, dtype=object))
    out = list(full[:N])
    for i in range(N - 1):
        out[i] -= full[N + i]
    return [int(x) % t for x in out]


def test_device_end_to_end_product_and_rotation():
    """Encode, encrypt (EncryptZeroSk + Add), MulRelinNew (BGV and BFV) + Rescale, decrypt with ring ops, Decode = slot-wise product
    times the output scale; an automorphism by 5^k decodes to both rows rotated by k."""
    import torch
    import lattigo_b200 as lb
    from tests import bgv_oracle as B
    from tests import helpers as H
    logN, t, level, batch = 11, 65537, 3, 2
    q, p = O.gen_moduli(logN + 1, [55, 45, 45, 45], [60])
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    enc = lb.BGVEncoder(ctx, t)
    try:
        N, n = ctx.N, enc.MaxSlots()
        rng = np.random.default_rng(11)
        s = rng.integers(-1, 2, N)
        s2 = _negacyclic(s, s, 1 << 62)
        s2 = [x - (1 << 62) if x >= 1 << 61 else x for x in s2]
        rlk = lb.GadgetCiphertext(ctx, H.gen_switching_key(params, s2, s, rng).data, len(q) - 1, len(p) - 1)
        sk = ENC.small_rows(s, params.qi)
        params.ringQ.NTT(sk, sk); params.ringQ.MForm(sk, sk)
        d_sk = ctx.to_device(sk)
        r = ctx.ringQ.AtLevel(level)

        def encrypt(pt):
            c1 = ctx.to_device(_uniform(params, level, batch, rng, N))
            e = torch.from_numpy(np.rint(rng.normal(0, 3.2, (batch, N))).astype(np.int64)).cuda()
            c0 = lb.encryptor.Encryptor(ctx).EncryptZeroSk(level, -1, d_sk, c1, e, True, False)
            r.Add(c0, pt, c0)
            return torch.stack([c0, c1], dim=1).contiguous()

        def decrypt(ct):
            lv = ct.shape[-2] - 1
            rl = ctx.ringQ.AtLevel(lv)
            skb = d_sk[: lv + 1].unsqueeze(0).expand(ct.shape[0], -1, -1).contiguous()
            out = ct[:, 0].clone()
            rl.MulCoeffsMontgomeryThenAdd(ct[:, 1].contiguous(), skb, out)
            return out

        m0 = rng.integers(-(t // 2), t // 2, (batch, n), dtype=np.int64)
        m1 = rng.integers(-(t // 2), t // 2, (batch, n), dtype=np.int64)
        ct0, ct1 = encrypt(enc.Encode(m0, level)), encrypt(enc.Encode(m1, level))
        assert np.array_equal(enc.Decode(decrypt(ct0), signed=True).cpu().numpy(), m0)
        prod = (m0 * m1) % t                                     # int64 products of |x| < 2^15 are exact
        qmul = B.qmul_moduli(logN, q)
        Ql = params.ringQ.ModulusAtLevel[level]
        for si in (False, True):
            ev = lb.BGVEvaluator(ctx, t, qmul, rlk, scale_invariant=si)
            out = ev.MulRelinNew(ct0, ct1)
            scale = pow((-Ql) % t, -1, t) if si else 1          # MulScaleInvariant / the BGV product scale
            got = enc.Decode(decrypt(out), scale).cpu().numpy()
            assert np.array_equal(got, prod), si
            if not si:
                res = ev.Rescale(out)
                got = enc.Decode(decrypt(res), pow(q[level], -1, t)).cpu().numpy()
                assert np.array_equal(got, prod)
            ev.close()
        # rotations: 5^k rotates both rows of n/2 slots left by k, 2N - 1 swaps the rows
        pt0 = decrypt(ct0)
        h = n // 2
        for k, gal in ((1, 5), (3, pow(5, 3, 2 * N)), (None, 2 * N - 1)):
            rot = torch.empty_like(pt0)
            r.AutomorphismNTT(pt0, gal, rot)
            got = enc.Decode(rot, signed=True).cpu().numpy()
            if k is None:
                want = np.concatenate([m0[:, h:], m0[:, :h]], axis=1)
            else:
                want = np.concatenate([np.roll(m0[:, :h], -k, axis=1), np.roll(m0[:, h:], -k, axis=1)], axis=1)
            assert np.array_equal(got, want), gal
    finally:
        enc.close(); ctx.close()

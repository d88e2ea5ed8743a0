"""GPU parity of the batched RGSW encryption and key generation (lgpu_rgsw_encrypt, lgpu_gen_galois_keys,
lgpu_blind_rotation_gen_evaluation_key) with oracle/rgsw_keygen.py and oracle/blindrot_keys.py, bit for bit given the same samples; and
blind rotation end to end under keys made on the device, decrypted to sign(x)."""
import ctypes

import numpy as np
import pytest

from oracle import blindrot_evaluate as BE
from oracle import blindrot_keys as BK
from oracle import rgsw_keygen as E
from oracle import oracle as O
from tests import helpers as H
from tests.test_oracle_blindrot_evaluate import Q_BR, Q_LWE, encrypt_lwe_values
from tests.test_rgsw_keygen_cpu import sk_rows
from lattigo_b200.ring import RING_P, RING_Q

pytestmark = pytest.mark.gpu
U64 = np.uint64

# the blind-rotation ring of examples/singleparty/ckks_scheme_switching: N = 2^12, two Q limbs, one P limb, BaseTwoDecomposition 12,
# and its LWE ring N = 2^11 over Q[:1]
SS_Q, SS_P, SS_Q_LWE, SS_P_LWE = [0x800004001, 0x40002001], [0x4000026001], [0x800004001], [0x42001]


def _samples(params, n, levelQ, levelP, pw2, rng):
    """a (n, digits, pw2, rows, N) uniform and e (n, digits, pw2, N) Gaussian, zero on the padding entries."""
    nd, sizes = E.gadget_layout(params, levelQ, levelP, pw2)
    mods = params.qi[: levelQ + 1] + params.pi[: levelP + 1]
    N = params.N()
    a = np.zeros((n, nd, max(sizes), len(mods), N), dtype=U64)
    e = np.zeros((n, nd, max(sizes), N), dtype=np.int64)
    for k in range(n):
        for i in range(nd):
            for j in range(sizes[i]):
                a[k, i, j] = H.rand_poly(mods, N, rng)
                e[k, i, j] = np.rint(rng.normal(0, 3.2, N)).astype(np.int64)
    return a, e, sizes


def _as_lists(a, e, sizes):
    return [[a[i][j] for j in range(sizes[i])] for i in range(len(sizes))], [[e[i][j] for j in range(sizes[i])] for i in range(len(sizes))]


def _same(got, want, sizes):
    for i in range(len(sizes)):
        for j in range(sizes[i]):
            assert np.array_equal(got[i, j], want.data[i, j]), (i, j)


RGSW_CASES = [
    # logN, Q bits, P bits, levelQ, levelP, pw2, batch, n_pt, flags (is_ntt, is_montgomery), chunk
    (7, [30], [], 0, -1, 7, 3, 2, (False, False), None),
    (8, [50, 40], [55], 1, 0, 12, 5, 3, (True, False), "2"),          # batches crossing two chunk boundaries
    (9, [50, 40, 40], [55, 55], 1, 1, 0, 2, 1, (False, True), None),   # levelQ < max
    (10, [50, 40, 40], [55, 55], 2, 0, 7, 2, 2, (True, True), None),   # levelP < max
    (11, [50, 40], [55], 1, -1, 0, 2, 1, (False, False), None),        # P in the context, none in the key
    (12, [55, 45], [56], 1, 0, 12, 2, 2, (True, False), "1"),
    (8, [50, 40], [55], 1, 0, 7, 3, 0, None, None),                    # EncryptZero
]


@pytest.mark.parametrize("case", RGSW_CASES, ids=lambda c: "N2^%d-lq%d-lp%d-pw%d-%s" % (c[0], c[3], c[4], c[5], "zero" if c[8] is None else
                                                                                         "ntt%dmont%d" % c[8]))
def test_rgsw_encrypt_matches_the_oracle(case, monkeypatch):
    import torch
    import lattigo_b200 as lb
    logN, qb, pb, levelQ, levelP, pw2, batch, n_pt, flags, chunk = case
    if chunk:
        monkeypatch.setenv("LGPU_KEYGEN_CHUNK", chunk)
    q, p = O.gen_moduli(logN + 1, qb, pb)
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(logN * 7 + levelQ + levelP + pw2)
    sk = sk_rows(params, rng.integers(-1, 2, N))
    a, e, sizes = _samples(params, 2 * batch, levelQ, levelP, pw2, rng)
    pts = np.stack([H.rand_poly(q[: levelQ + 1], N, rng) for _ in range(n_pt)]) if n_pt else None
    idx = [int(x) for x in rng.integers(0, n_pt, batch)] if n_pt else None
    ctx = lb.Context(logN, q, p)
    try:
        enc = lb.rgsw.Encryptor(ctx, ctx.to_device(sk))
        da = ctx.to_device(a).view((batch, 2) + a.shape[1:])
        de = torch.from_numpy(e).cuda().view((batch, 2) + e.shape[1:])
        if n_pt:
            cts = enc.Encrypt(ctx.to_device(pts), levelQ, levelP, pw2, idx, flags[0], flags[1], a=da, e=de)
        else:
            cts = enc.EncryptZero(batch, levelQ, levelP, pw2, a=da, e=de)
        assert len(cts) == batch
        for b in range(batch):
            al = [_as_lists(a[2 * b + v], e[2 * b + v], sizes) for v in range(2)]
            want = E.rgsw_encrypt(params, sk, pts[idx[b]] if n_pt else None, [x[0] for x in al], [x[1] for x in al], levelQ, levelP, pw2,
                                  *(flags or (True, True)))
            for v in range(2):
                assert cts[b].Value[v].LevelQ() == levelQ and cts[b].Value[v].LevelP() == levelP
                _same(ctx.to_host(cts[b].Value[v].data), want[v], sizes)
    finally:
        ctx.close()


@pytest.mark.parametrize("levelQ,levelP,pw2", [(2, 1, 0), (1, 0, 7), (2, -1, 12), (0, 0, 0)])
def test_gen_galois_keys_matches_the_oracle(levelQ, levelP, pw2, monkeypatch):
    import torch
    import lattigo_b200 as lb
    logN = 10
    q, p = O.gen_moduli(logN + 1, [50, 40, 40], [55, 55])
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(levelQ + 3 * levelP + pw2)
    sk = sk_rows(params, rng.integers(-1, 2, N))
    gals = [params.GaloisElement(k) for k in (1, 2, 5)] + [2 * N - 5, 2 * N - 1]
    a, e, sizes = _samples(params, len(gals), levelQ, levelP, pw2, rng)
    monkeypatch.setenv("LGPU_KEYGEN_CHUNK", "2")
    ctx = lb.Context(logN, q, p)
    try:
        keys = lb.encryptor.KeyGenerator(ctx).GenGaloisKeysNew(gals, ctx.to_device(sk), levelQ, levelP, pw2, a=ctx.to_device(a),
                                                               e=torch.from_numpy(e).cuda())
        for k, g in enumerate(gals):
            want = E.gen_galois_key(params, g, sk, *_as_lists(a[k], e[k], sizes), pw2, levelQ, levelP)
            _same(ctx.to_host(keys[k].data), want, sizes)
    finally:
        ctx.close()


def _redraw(ctx, seed, m, levelQ, levelP, sizes, sigma, bound):
    """The samples of gadget ciphertext m of lgpu_blind_rotation_gen_evaluation_key, redrawn from the header's stream layout."""
    import torch
    import lattigo_b200 as lb
    N, rows, nd, npw2 = ctx.N, levelQ + 1 + levelP + 1, len(sizes), max(sizes)
    ent = nd * npw2
    a = ctx.new_poly(rows, ent)
    L = lb.lib()
    lb._lib.check(L.lgpu_sample_uniform(ctx.h, RING_Q, levelQ, seed, m, ctypes.c_void_p(a.data_ptr()), ent, rows * N, None))
    if levelP >= 0:
        lb._lib.check(L.lgpu_sample_uniform(ctx.h, RING_P, levelP, seed, m, ctypes.c_void_p(a.data_ptr() + 8 * (levelQ + 1) * N), ent, rows * N, None))
    e = torch.empty((ent, N), dtype=torch.int64, device="cuda")
    lb._lib.check(L.lgpu_sample_gaussian(ctx.h, sigma, bound, seed, m, ctypes.c_void_p(e.data_ptr()), ent, None))
    a = ctx.to_host(a).reshape(nd, npw2, rows, N)
    e = e.cpu().numpy().reshape(nd, npw2, N)
    return _as_lists(a, e, sizes)


def _lwe_key(params_lwe, s, ctx_lwe):
    return ctx_lwe.to_device(sk_rows(params_lwe, s))


def test_blind_rotation_keys_scheme_switching_shape_subset():
    """All 2048 RGSW ciphertexts and 11 Galois keys at the scheme-switching shape in one call (chunked), a seeded subset of them
    recomputed by the oracle from samples redrawn on the documented streams."""
    import lattigo_b200 as lb
    params = O.Parameters(12, SS_Q, SS_P)
    params_lwe = O.Parameters(11, SS_Q_LWE, SS_P_LWE)
    rng = np.random.default_rng(2048)
    s_br = rng.integers(-1, 2, params.N())
    s_lwe = rng.integers(-1, 2, params_lwe.N())
    sk = sk_rows(params, s_br)
    seed, sigma, bound, window = 0x5EED5EED12345678, 3.2, 19.2, 10
    ctx, ctx_lwe = lb.Context(12, SS_Q, SS_P), lb.Context(11, SS_Q_LWE, SS_P_LWE)
    try:
        brk, gks = lb.rgsw.GenEvaluationKeyNew(ctx, ctx.to_device(sk), ctx_lwe, _lwe_key(params_lwe, s_lwe, ctx_lwe), pw2=12, window_size=window,
                                               sigma=sigma, bound=bound, seed=seed)
        assert len(brk) == 2048 and sorted(gks) == sorted(BK.galois_elements(params, window))
        levelQ, levelP = 1, 0
        _, sizes = E.gadget_layout(params, levelQ, levelP, 12)
        assert sizes == [3, 3]
        for i in sorted(set([0, 2047] + [int(x) for x in rng.integers(0, 2048, 4)])):
            pt = BK.monomial(params.ringQ, int(s_lwe[i])); params.ringQ.NTT(pt, pt)
            al = [_redraw(ctx, seed, 2 * i + v, levelQ, levelP, sizes, sigma, bound) for v in range(2)]
            want = E.rgsw_encrypt(params, sk, pt, [x[0] for x in al], [x[1] for x in al], levelQ, levelP, 12, True, False)
            for v in range(2):
                _same(ctx.to_host(brk[i].Value[v].data), want[v], sizes)
        for t in (0, window):
            g = BK.galois_elements(params, window)[t]
            want = E.gen_galois_key(params, g, sk, *_redraw(ctx, seed, 2 * 2048 + t, levelQ, levelP, sizes, sigma, bound), 12, levelQ, levelP)
            _same(ctx.to_host(gks[g].data), want, sizes)
    finally:
        ctx.close(); ctx_lwe.close()


def _sign_check(params, res, slots, values, s_br, delta):
    for i in slots:
        v = values[i]
        assert abs(v) >= 0.25
        r = res[i]
        got = _decrypt(params, [r[0], r[1]], s_br) / delta
        assert round(got * 8) / 8 == np.sign(v), (i, v, got)


def _decrypt(params, ct, s):
    """Coefficient 0 of c0 + c1 s over all the ciphertext's Q limbs, centred (NTT-domain ciphertext)."""
    nq = ct[0].shape[0]
    ringQ = params.ringQ.AtLevel(nq - 1)
    sn = H.small_poly_rns(s, params.qi[:nq]); ringQ.NTT(sn, sn)
    dec = np.stack([np.array([(int(x) + int(y) * int(t)) % m for x, y, t in zip(ct[0][l], ct[1][l], sn[l])], dtype=U64)
                    for l, m in enumerate(params.qi[:nq])])
    ringQ.INTT(dec, dec)
    Q = ringQ.ModulusAtLevel[nq - 1]
    c = ringQ.PolyToBigint(dec)[0]
    return c if c < Q // 2 else c - Q


def test_end_to_end_reference_shape_fused_path():
    """blindrot_test.go's shape: 0x7fff801 / 0x3001, N = 2^10 / 2^9, BaseTwoDecomposition 7, window 10; all 512 RGSW ciphertexts and 11
    Galois keys made on the device; 16 slots through the fused kernel decrypt to sign(x)."""
    import lattigo_b200 as lb
    params = O.Parameters(10, [Q_BR], [])
    params_lwe = O.Parameters(9, [Q_LWE], [])
    n_lwe = params_lwe.N()
    rng = np.random.default_rng(10)
    s_br = rng.integers(-1, 2, params.N())
    s_lwe = rng.integers(-1, 2, n_lwe)
    ctx, ctx_lwe = lb.Context(10, [Q_BR], []), lb.Context(9, [Q_LWE], [])
    try:
        brk, gks = lb.rgsw.GenEvaluationKeyNew(ctx, ctx.to_device(sk_rows(params, s_br)), ctx_lwe, _lwe_key(params_lwe, s_lwe, ctx_lwe), pw2=7,
                                               window_size=10, seed=77)
        assert len(brk) == 512 and len(gks) == 11
        delta = float(Q_BR) / 4.0
        tp = ctx.to_device(BE.InitTestPolynomial(np.sign, delta, params.ringQ, -1.0, 1.0))
        values = [-1 + 2 * i / n_lwe for i in range(n_lwe)]
        ct = encrypt_lwe_values(values, n_lwe, s_lwe, rng)
        d_ct = ctx_lwe.to_device(np.stack([ct[0], ct[1]]))
        slots = [int(i) for i in np.linspace(0, n_lwe - 1, 24).round() if abs(values[int(i)]) >= 0.25][:16]
        assert len(slots) == 16
        ev = lb.rgsw.BlindRotationEvaluator(ctx, brk, gks, 10)
        out = {}
        assert H.launch_delta(lambda: out.update(ev.Evaluate(d_ct, {i: tp for i in slots}, ctx_lwe, is_ntt=False))) == 2   # the fused kernel
        _sign_check(params, {i: ctx.to_host(v) for i, v in out.items()}, slots, values, s_br, delta)
    finally:
        ctx.close(); ctx_lwe.close()


def test_end_to_end_scheme_switching_shape_fallback_path():
    """The scheme-switching shape (keys with P take the per-slot fallback): a few slots decrypt to sign(x)."""
    import lattigo_b200 as lb
    params = O.Parameters(12, SS_Q, SS_P)
    params_lwe = O.Parameters(11, SS_Q_LWE, SS_P_LWE)
    n_lwe = params_lwe.N()
    rng = np.random.default_rng(12)
    s_br = rng.integers(-1, 2, params.N())
    s_lwe = rng.integers(-1, 2, n_lwe)
    ctx, ctx_lwe = lb.Context(12, SS_Q, SS_P), lb.Context(11, SS_Q_LWE, SS_P_LWE)
    try:
        brk, gks = lb.rgsw.GenEvaluationKeyNew(ctx, ctx.to_device(sk_rows(params, s_br)), ctx_lwe, _lwe_key(params_lwe, s_lwe, ctx_lwe), pw2=12,
                                               seed=3)
        Q = SS_Q[0] * SS_Q[1]
        delta = float(Q) / 4.0
        tp = ctx.to_device(BE.InitTestPolynomial(np.sign, delta, params.ringQ, -1.0, 1.0))
        values = [-1 + 2 * i / n_lwe for i in range(n_lwe)]
        ct = encrypt_lwe_values(values, n_lwe, s_lwe, rng, q=SS_Q_LWE[0])
        d_ct = ctx_lwe.to_device(np.stack([ct[0], ct[1]]))
        slots = [3, 700, 1500, 2040]
        ev = lb.rgsw.BlindRotationEvaluator(ctx, brk, gks, 10)
        out = {}
        assert H.launch_delta(lambda: out.update(ev.Evaluate(d_ct, {i: tp for i in slots}, ctx_lwe, is_ntt=False))) > 100   # the fallback
        _sign_check(params, {i: ctx.to_host(v) for i, v in out.items()}, slots, values, s_br, delta)
    finally:
        ctx.close(); ctx_lwe.close()

"""The RGSW encryption and key-generation restatements (oracle/rgsw_keygen.py rgsw_encrypt / gen_evaluation_key at any levels,
oracle/blindrot_keys.py GenEvaluationKeyNew), pinned by decryption as core/rgsw/rgsw_test.go and blindrot_test.go pin the reference:
an RGSW(m) external-producted with an RLWE encryption of m' decrypts to m m' plus small noise, and keys from GenEvaluationKeyNew drive
the blind-rotation restatement to sign(x). Plus every refusal of lgpu_rgsw_encrypt, lgpu_gen_galois_keys and
lgpu_blind_rotation_gen_evaluation_key on a host-only context, before any device work."""
import ctypes

import numpy as np
import pytest

from oracle import blindrot_evaluate as BE
from oracle import blindrot_keys as BK
from oracle import rgsw_keygen as E
from oracle import oracle as O
from oracle import rgsw as RG
from tests import helpers as H
from tests.test_oracle_blindrot_evaluate import Q_BR, Q_LWE, decrypt_coeff0, encrypt_lwe_values

U64 = np.uint64
FAKE = 1 << 20          # 16-byte aligned placeholder device address, never dereferenced


def _negacyclic(a, b, N):
    out = [0] * N
    for i, x in enumerate(a):
        if x == 0:
            continue
        for j, y in enumerate(b):
            k = i + j
            if k < N: out[k] += int(x) * int(y)
            else: out[k - N] -= int(x) * int(y)
    return out


def sk_rows(params, s):
    """(nQ + nP, N) NTT + Montgomery rows of the small secret s."""
    rows = H.small_poly_rns(s, params.qi + params.pi)
    nQ = len(params.qi)
    params.ringQ.NTT(rows[:nQ], rows[:nQ]); params.ringQ.MForm(rows[:nQ], rows[:nQ])
    if params.ringP is not None:
        params.ringP.NTT(rows[nQ:], rows[nQ:]); params.ringP.MForm(rows[nQ:], rows[nQ:])
    return rows


def gadget_samples(params, levelQ, levelP, pw2, rng):
    """(a, e) of one gadget ciphertext: a[i][j] uniform QP rows, e[i][j] rounded Gaussian."""
    n, sizes = E.gadget_layout(params, levelQ, levelP, pw2)
    mods = params.qi[: levelQ + 1] + params.pi[: levelP + 1]
    a = [[H.rand_poly(mods, params.N(), rng) for _ in range(sizes[i])] for i in range(n)]
    e = [[np.rint(rng.normal(0, 3.2, params.N())).astype(np.int64) for _ in range(sizes[i])] for i in range(n)]
    return a, e


@pytest.mark.parametrize("p_bits,levelQ,levelP,pw2,log_delta,max_err_bits", [
    ([], 1, -1, 0, 60, 52),           # no P: one Q limb per digit
    ([], 2, -1, 7, 50, 30),           # no P, base-2^7 split of every digit
    ([50], 1, 0, 7, 50, 30),          # one P limb with the base-2^7 split, levelQ below the maximum
    ([50, 50], 2, 1, 0, 50, 30),      # two P limbs
    ([50, 50], 1, 0, 0, 50, 30),      # levelP below the maximum
    ([50, 50], 2, -1, 7, 50, 30),     # P in the parameters, none in the key
])
def test_rgsw_external_product_decrypts_to_the_product(p_bits, levelQ, levelP, pw2, log_delta, max_err_bits):
    logN = 5
    q, p = O.gen_moduli(logN + 1, [45, 35, 35], p_bits)
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(levelQ * 10 + levelP + pw2)
    s = rng.integers(-1, 2, N)
    sk = sk_rows(params, s)
    m1 = np.zeros(N, dtype=np.int64); m1[rng.integers(0, N, 2)] = rng.integers(-1, 2, 2); m1[0] = 1
    pt = H.small_poly_rns(m1, q)                          # coefficient domain, not Montgomery: Encrypt takes it to NTT + MForm
    samples = [gadget_samples(params, levelQ, levelP, pw2, rng) for _ in range(2)]
    rg = E.rgsw_encrypt(params, sk, pt, [x[0] for x in samples], [x[1] for x in samples], levelQ, levelP, pw2, is_ntt=False, is_montgomery=False)
    ringQ = params.ringQ.AtLevel(levelQ)
    qs = q[: levelQ + 1]
    m0 = rng.integers(-8, 9, N)
    sn = H.small_poly_rns(s, qs); ringQ.NTT(sn, sn)
    a = H.rand_poly(qs, N, rng)
    big = [(int(x) << log_delta) + int(e) for x, e in zip(m0, np.rint(rng.normal(0, 3.2, N)))]
    me = np.stack([np.array([v % m for v in big], dtype=U64) for m in qs])
    ringQ.NTT(me, me)
    c0 = np.stack([np.array([(int(x) - int(y) * int(t)) % m for x, y, t in zip(me[l], a[l], sn[l])], dtype=U64) for l, m in enumerate(qs)])
    out = [np.zeros((levelQ + 1, N), dtype=U64) for _ in range(2)]
    RG.Evaluator(params).ExternalProduct([c0, a], rg, out)
    acc = np.stack([np.array([(int(x) + int(y) * int(t)) % m for x, y, t in zip(out[0][l], out[1][l], sn[l])], dtype=U64) for l, m in enumerate(qs)])
    back = np.empty_like(acc); ringQ.INTT(acc, back)
    Q = ringQ.ModulusAtLevel[levelQ]
    got = [v if v < Q // 2 else v - Q for v in ringQ.PolyToBigint(back)]
    want = [v << log_delta for v in _negacyclic(m0, m1, N)]
    err = max(abs(g - w) for g, w in zip(got, want))
    assert err < 1 << max_err_bits, np.log2(err + 1)


@pytest.mark.parametrize("levelP", [-1, 0])
def test_rgsw_encrypt_zero_and_plaintext_flags(levelP):
    """Every combination of the plaintext flags gives the same ciphertext for the same plaintext, and EncryptZero equals Encrypt without
    the gadget term: Value[0] and Value[1] differ from it only on component 0 resp. component 1."""
    logN, levelQ, pw2 = 4, 1, 7
    q, p = O.gen_moduli(logN + 1, [40, 35], [45])
    params = O.Parameters(logN, q, p)
    rng = np.random.default_rng(3)
    sk = sk_rows(params, rng.integers(-1, 2, params.N()))
    samples = [gadget_samples(params, levelQ, levelP, pw2, rng) for _ in range(2)]
    a, e = [x[0] for x in samples], [x[1] for x in samples]
    coeff = H.rand_poly(q, params.N(), rng)
    forms = {}
    for ntt in (False, True):
        for mont in (False, True):
            x = coeff.copy()
            if ntt: params.ringQ.NTT(x, x)
            if mont: params.ringQ.MForm(x, x)
            forms[(ntt, mont)] = x
    # a coefficient-domain plaintext flagged Montgomery is only transformed: its NTT must already carry the Montgomery factor
    params.ringQ.INTT(forms[(True, True)], forms[(False, True)])
    cts = {f: E.rgsw_encrypt(params, sk, x, a, e, levelQ, levelP, pw2, *f) for f, x in forms.items()}
    ref = cts[(True, True)]
    for f, ct in cts.items():
        for v in range(2):
            assert np.array_equal(ct[v].data, ref[v].data), f
    zero = E.rgsw_encrypt(params, sk, None, a, e, levelQ, levelP, pw2)
    for v in range(2):
        assert np.array_equal(zero[v].data[:, :, 1 - v], ref[v].data[:, :, 1 - v])
        assert not np.array_equal(zero[v].data[:, :, v], ref[v].data[:, :, v])


def test_gen_evaluation_key_new_drives_blind_rotation_to_sign():
    """blindrot_test.go's shape: N = 2^7 blind-rotation ring, N_LWE = 2^4, BaseTwoDecomposition 7, window 10; every key from the
    GenEvaluationKeyNew restatement."""
    logN, n_lwe, pw2, window = 7, 16, 7, 10
    params = O.Parameters(logN, [Q_BR], [])
    params_lwe = O.Parameters(4, [Q_LWE], [])
    rng = np.random.default_rng(11)
    s_br = rng.integers(-1, 2, params.N())
    s_lwe = rng.integers(-1, 2, n_lwe)
    brk, gks = BK.GenEvaluationKeyNew(params, sk_rows(params, s_br), s_lwe, 0, -1, pw2, window,
                                      lambda m: gadget_samples(params, 0, -1, pw2, rng))
    assert sorted(gks) == sorted(BK.galois_elements(params, window))
    scale = float(Q_BR) / 4.0
    tp = BE.InitTestPolynomial(np.sign, scale, params.ringQ, -1.0, 1.0)
    values = [-1 + 2 * i / n_lwe for i in range(n_lwe)]
    ct = encrypt_lwe_values(values, n_lwe, s_lwe, rng)
    res = BE.Evaluator(params, params_lwe, window).Evaluate(ct, {i: tp for i in range(n_lwe)}, brk, gks, is_ntt=False)
    for i, v in enumerate(values):
        if abs(v) >= 0.25:
            got = decrypt_coeff0(params, res[i], s_br) / scale
            assert round(got * 8) / 8 == np.sign(v), (i, v, got)


# ---- refusals on a host-only context ---------------------------------------------------------------------------------------------
LOGN = 8
QS = [0x7fff801]


def _ctx(P=True, ring_type=0):
    import lattigo_b200 as lb
    return lb.Context(LOGN, H.Qi60[:3], H.Pi60[:2] if P else [], device=-1, ring_type=ring_type)


def _key(levelQ=2, levelP=1, pw2=0, nd=None, npw2=1, sizes=None, addr=FAKE):
    import lattigo_b200 as lb
    nd = (levelQ + 1 if levelP == -1 else (levelQ + levelP + 1) // (levelP + 1)) if nd is None else nd
    arr = (ctypes.c_int * len(sizes))(*sizes) if sizes is not None else None
    g = lb._lib.GadgetCtStruct(ctypes.c_void_p(addr) if addr else None, levelQ, levelP, pw2, nd, npw2, arr)
    g._keep = arr
    return g


def _keys(n, stride, **kw):
    import lattigo_b200 as lb
    ks = [_key(addr=FAKE + k * stride, **kw) for k in range(n)]
    arr = (lb._lib.GadgetCtStruct * n)(*ks)
    arr._keep = ks
    return arr


KEY_BYTES = 2 * 2 * 5 * (1 << LOGN) * 8          # levelQ 2, levelP 1: 2 digits, 2 components, 5 rows
SK, E_, PTS = 1 << 40, 1 << 41, 1 << 42           # input addresses far from the keys


def _refuse(call, msg):
    import lattigo_b200 as lb
    rc = call()
    assert rc != 0
    assert msg in lb.lib().lgpu_last_error().decode(), lb.lib().lgpu_last_error().decode()


def _rgsw(ctx, v0=None, v1=None, batch=2, pts=PTS, n_pt=1, idx=(0, 0), sk=SK, e=E_, ntt=1, mont=0):
    import lattigo_b200 as lb
    v0 = _keys(batch, KEY_BYTES) if v0 is None else v0
    v1 = _keys(batch, KEY_BYTES) if v1 is None else v1
    ia = (ctypes.c_int * max(1, len(idx)))(*idx) if idx is not None else None
    return lambda: lb.lib().lgpu_rgsw_encrypt(ctx.h, ctypes.c_void_p(sk) if sk else None, ctypes.c_void_p(pts) if pts else None, n_pt, ia, ntt, mont,
                                              ctypes.c_void_p(e) if e else None, v0, v1 if v1 is not False else None, batch, None)


def test_rgsw_encrypt_refusals():
    ctx = _ctx()
    try:
        v0 = _keys(2, KEY_BYTES)
        v1 = (type(v0))(*[_key(addr=FAKE + (2 + k) * KEY_BYTES) for k in range(2)])
        ok = dict(v0=v0, v1=v1)
        _refuse(_rgsw(ctx, **ok), "host-only")                                  # a valid call reaches the device check
        _refuse(_rgsw(ctx, batch=0, **ok), "batch out of [1, 65535]")
        _refuse(_rgsw(ctx, batch=65536, **ok), "batch out of [1, 65535]")
        _refuse(_rgsw(ctx, sk=0, **ok), "null argument")
        _refuse(_rgsw(ctx, e=0, **ok), "null argument")
        _refuse(_rgsw(ctx, v0=v0, v1=False), "null argument")
        _refuse(_rgsw(ctx, idx=None, **ok), "plaintexts need")
        _refuse(_rgsw(ctx, n_pt=0, **ok), "plaintexts need")
        _refuse(_rgsw(ctx, idx=(0, 1), **ok), "pt_index out of [0, n_pt)")
        _refuse(_rgsw(ctx, pts=0, idx=None, **ok), "host-only")               # EncryptZero
        # levels and layouts
        mk = lambda addr=FAKE, **kw: (type(v0))(*[_key(addr=addr + k * KEY_BYTES if addr else 0, **kw) for k in range(2)])
        _refuse(_rgsw(ctx, v0=mk(levelQ=3), v1=v1), "level out of range")
        _refuse(_rgsw(ctx, v0=mk(levelP=2), v1=v1), "level out of range")
        _refuse(_rgsw(ctx, v0=mk(levelP=-2), v1=v1), "level out of range")
        _refuse(_rgsw(ctx, v0=mk(pw2=63), v1=v1), "BaseTwoDecomposition out of [0, 62]")
        _refuse(_rgsw(ctx, v0=mk(nd=3), v1=v1), "n_digits != BaseRNSDecompositionVectorSize")
        _refuse(_rgsw(ctx, v0=mk(levelP=0, pw2=7, nd=3), v1=v1), "pw2_sizes != BaseTwoDecompositionVectorSize")
        _refuse(_rgsw(ctx, v0=mk(levelP=0, pw2=7, nd=3, npw2=8, sizes=[8, 8, 8]), v1=v1), "pw2_sizes != BaseTwoDecompositionVectorSize")
        _refuse(_rgsw(ctx, v0=mk(levelP=0, pw2=7, nd=3, npw2=8, sizes=[9, 9, 9]), v1=v1), "n_pw2_max != max(BaseTwoDecompositionVectorSize)")
        _refuse(_rgsw(ctx, v0=mk(levelP=0, pw2=7, nd=3, npw2=9, sizes=[9, 9, 9]), v1=v1), "gadget ciphertexts of one call differ")
        _refuse(_rgsw(ctx, v0=mk(npw2=2), v1=v1), "n_pw2_max != max(BaseTwoDecompositionVectorSize)")
        # null / misaligned key data, overlaps
        _refuse(_rgsw(ctx, v0=mk(addr=0), v1=v1), "null gadget ciphertext")
        _refuse(_rgsw(ctx, v0=mk(addr=FAKE + 8), v1=v1), "16-byte aligned")
        _refuse(_rgsw(ctx, v0=v0, v1=v0), "overlap one another")
        _refuse(_rgsw(ctx, v0=v0, v1=(type(v0))(*[_key(addr=FAKE + KEY_BYTES + 64), _key(addr=FAKE + 3 * KEY_BYTES)])), "overlap one another")
        _refuse(_rgsw(ctx, sk=FAKE + 64, **ok), "overlaps an input")
        _refuse(_rgsw(ctx, e=FAKE + 64, **ok), "overlaps an input")
        _refuse(_rgsw(ctx, pts=FAKE + 64, **ok), "overlaps an input")
        ci = _ctx(ring_type=1)
        try:
            _refuse(_rgsw(ci, **ok), "ConjugateInvariant")
        finally:
            ci.close()
    finally:
        ctx.close()


def test_gen_galois_keys_refusals():
    import lattigo_b200 as lb
    ctx = _ctx()
    try:
        keys = _keys(2, KEY_BYTES)
        N2 = 2 << LOGN

        def call(gal=(5, 25), n=2, sk=SK, e=E_, ks=keys):
            g = (ctypes.c_uint64 * max(1, len(gal)))(*gal) if gal is not None else None
            return lambda: lb.lib().lgpu_gen_galois_keys(ctx.h, ctypes.c_void_p(sk) if sk else None, g, n, ctypes.c_void_p(e) if e else None, ks, None)
        _refuse(call(), "host-only")
        _refuse(call(gal=(5, N2 - 5)), "host-only")
        _refuse(call(n=0), "n_keys out of [1, 65535]")
        _refuse(call(n=65536), "n_keys out of [1, 65535]")
        _refuse(call(gal=None), "null argument")
        _refuse(call(sk=0), "null argument")
        _refuse(call(e=0), "null argument")
        _refuse(call(ks=None), "null argument")
        _refuse(call(gal=(5, 4)), "Galois elements are odd and below 2N")
        _refuse(call(gal=(5, N2 + 1)), "Galois elements are odd and below 2N")
        _refuse(call(ks=(type(keys))(*[_key(), _key(addr=FAKE + KEY_BYTES, levelQ=1)])), "differ in levels or digit layout")
        _refuse(call(ks=(type(keys))(*[_key(), _key()])), "overlap one another")
        _refuse(call(ks=(type(keys))(*[_key(), _key(addr=FAKE + KEY_BYTES, nd=1)])), "differ in levels or digit layout")
        _refuse(call(ks=(type(keys))(*[_key(nd=1), _key(addr=FAKE + KEY_BYTES, nd=1)])), "n_digits != BaseRNSDecompositionVectorSize")
        _refuse(call(sk=FAKE + KEY_BYTES), "overlaps an input")
        _refuse(call(e=FAKE), "overlaps an input")
    finally:
        ctx.close()


def test_blind_rotation_gen_evaluation_key_refusals():
    import lattigo_b200 as lb
    ctx = _ctx()
    try:
        n, w = 4, 3
        brk0, brk1 = _keys(n, KEY_BYTES), (type(_keys(n, KEY_BYTES)))(*[_key(addr=FAKE + (n + k) * KEY_BYTES) for k in range(n)])
        gks = (type(_keys(w + 1, KEY_BYTES)))(*[_key(addr=FAKE + (2 * n + k) * KEY_BYTES) for k in range(w + 1)])
        s = np.array([0, 1, -1, 1], dtype=np.int64)

        def call(n=n, w=w, sigma=3.2, bound=19.2, sk=SK, s_lwe=s, b0=brk0, b1=brk1, g=gks):
            return lambda: lb.lib().lgpu_blind_rotation_gen_evaluation_key(ctx.h, ctypes.c_void_p(sk) if sk else None,
                                                                            s_lwe.ctypes.data if s_lwe is not None else None, n, w, sigma, bound, 7,
                                                                            b0, b1, g, None)
        _refuse(call(), "host-only")
        _refuse(call(n=0), "n_lwe out of [1, 32767]")
        _refuse(call(n=32768), "n_lwe out of [1, 32767]")
        _refuse(call(w=0), "window_size out of [1, N/2)")
        _refuse(call(w=1 << (LOGN - 1)), "window_size out of [1, N/2)")
        _refuse(call(sigma=0.0), "sigma / bound out of range")
        _refuse(call(bound=0.5), "sigma / bound out of range")
        _refuse(call(sk=0), "null argument")
        _refuse(call(s_lwe=None), "null argument")
        _refuse(call(b1=None), "null argument")
        _refuse(call(g=None), "null argument")
        _refuse(call(b1=brk0), "overlap one another")
        _refuse(call(g=(type(gks))(*([_key(addr=FAKE + (2 * n + k) * KEY_BYTES) for k in range(w)] + [_key(addr=FAKE)]))), "overlap one another")
        _refuse(call(g=(type(gks))(*[_key(addr=FAKE + (2 * n + k) * KEY_BYTES, levelQ=1) for k in range(w + 1)])),
                "Galois keys and RGSW ciphertexts differ")
        _refuse(call(sk=FAKE + 64), "overlaps an input")
    finally:
        ctx.close()

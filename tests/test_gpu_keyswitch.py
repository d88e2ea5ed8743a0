"""GPU parity (bit-exact vs the oracle) of basis extension, rescaling, automorphisms, the rlwe.Evaluator
key-switch family and the CKKS MulRelin+Rescale sequence. Run with -m gpu on an H100."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
U64 = np.uint64


def _lb():
    import lattigo_b200 as lb
    return lb


def _mods(logN, lq, lp):
    return O.gen_moduli(logN + 1, lq, lp)


@pytest.fixture(scope="module")
def small():
    """logN=8 context with CKKS-like sizes (56/45-bit Q, 55-bit P) + oracle twin."""
    lb = _lb()
    logN = 8
    q, p = _mods(logN, [56, 45, 45, 45, 45, 45, 45], [55, 55, 55])
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    yield lb, ctx, params, q, p
    ctx.close()


@pytest.fixture(scope="module")
def big61():
    """61-bit primes (ring/test_params.go) stress the lazy ranges and the float64 `v` path."""
    lb = _lb()
    logN = 8
    q, p = H.Qi60[:5], H.Pi60[:2]
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    yield lb, ctx, params, q, p
    ctx.close()


@pytest.mark.parametrize("fx", ["small", "big61"])
def test_modup_exact_representatives(fx, request):
    lb, ctx, params, q, p = request.getfixturevalue(fx)
    N = params.N()
    be_o = O.BasisExtender(params.ringQ, params.ringP)
    be = lb.BasisExtender(ctx)
    rng = np.random.default_rng(1)
    for levelQ in (0, 1, len(q) - 1):
        for levelP in (0, len(p) - 1):
            batch = 2
            xq = np.stack([H.rand_poly(q[: levelQ + 1], N, rng) for _ in range(batch)])
            xp = np.stack([H.rand_poly(p[: levelP + 1], N, rng) for _ in range(batch)])
            wantP = np.zeros((batch, levelP + 1, N), dtype=U64); wantQ = np.zeros((batch, levelQ + 1, N), dtype=U64)
            for b in range(batch):
                be_o.ModUpQtoP(levelQ, levelP, xq[b], wantP[b])
                be_o.ModUpPtoQ(levelP, levelQ, xp[b], wantQ[b])
            dP = ctx.new_poly(levelP + 1, batch); dQ = ctx.new_poly(levelQ + 1, batch)
            be.ModUpQtoP(levelQ, levelP, ctx.to_device(xq), dP)
            be.ModUpPtoQ(levelP, levelQ, ctx.to_device(xp), dQ)
            assert np.array_equal(ctx.to_host(dP), wantP), (levelQ, levelP)     # exact (non-canonical) representative
            assert np.array_equal(ctx.to_host(dQ), wantQ), (levelQ, levelP)


@pytest.mark.parametrize("fx", ["small", "big61"])
def test_moddown_variants(fx, request):
    lb, ctx, params, q, p = request.getfixturevalue(fx)
    N = params.N()
    be_o = O.BasisExtender(params.ringQ, params.ringP)
    be = lb.BasisExtender(ctx)
    rng = np.random.default_rng(2)
    for levelQ in (0, 2, len(q) - 1):
        for levelP in (0, len(p) - 1):
            batch = 2
            xq = np.stack([H.rand_poly(q[: levelQ + 1], N, rng) for _ in range(batch)])
            xp = np.stack([H.rand_poly(p[: levelP + 1], N, rng) for _ in range(batch)])
            dq, dp = ctx.to_device(xq), ctx.to_device(xp)
            for name, rows, mods in (("ModDownQPtoQ", levelQ + 1, q), ("ModDownQPtoQNTT", levelQ + 1, q), ("ModDownQPtoP", levelP + 1, p)):
                want = np.zeros((batch, rows, N), dtype=U64)
                for b in range(batch):
                    getattr(be_o, name)(levelQ, levelP, xq[b].copy(), xp[b].copy(), want[b])
                out = ctx.new_poly(rows, batch)
                getattr(be, name)(levelQ, levelP, dq, dp, out)
                assert np.array_equal(ctx.to_host(out), want), (name, levelQ, levelP)
                for r in range(rows):
                    assert int(want[:, r].max()) < mods[r]


@pytest.mark.parametrize("fx", ["small", "big61"])
def test_decompose_and_split(fx, request):
    lb, ctx, params, q, p = request.getfixturevalue(fx)
    N = params.N()
    dec_o = O.Decomposer(params.ringQ, params.ringP)
    dec = lb.Decomposer(ctx)
    rng = np.random.default_rng(3)
    for levelQ in (len(q) - 1, 2, 0):
        for levelP in range(len(p)):
            nbPi = levelP + 1
            ndig = (levelQ + levelP + 1) // (levelP + 1)
            x = H.rand_poly(q[: levelQ + 1], N, rng)
            dx = ctx.to_device(x)
            for digit in range(ndig):
                wq = np.zeros((levelQ + 1, N), dtype=U64); wp = np.zeros((levelP + 1, N), dtype=U64)
                dec_o.DecomposeAndSplit(levelQ, levelP, nbPi, digit, x, wq, wp)
                gq = ctx.new_poly(levelQ + 1); gp = ctx.new_poly(levelP + 1)
                dec.DecomposeAndSplit(levelQ, levelP, nbPi, digit, dx, gq, gp)
                gq, gp = ctx.to_host(gq), ctx.to_host(gp)
                st, ed = digit * nbPi, min(digit * nbPi + nbPi, levelQ + 1)
                single = (ed - st) == 1
                for r in range(levelQ + 1):
                    if st <= r < ed and not single:
                        continue       # reference leaves unspecified values in the digit's own rows
                    assert np.array_equal(gq[r], wq[r]), (levelQ, levelP, digit, r)
                assert np.array_equal(gp, wp), (levelQ, levelP, digit)


@pytest.mark.parametrize("fx", ["small", "big61"])
def test_div_by_last_modulus_family(fx, request):
    lb, ctx, params, q, p = request.getfixturevalue(fx)
    N = params.N()
    ring = params.ringQ
    rng = np.random.default_rng(4)
    level = len(q) - 1
    batch = 2
    x = np.stack([H.rand_poly(q, N, rng) for _ in range(batch)])
    dx = ctx.to_device(x)
    for nb in (0, 1, 2, 3):
        for rnd in (True, False):
            for ntt in (True, False):
                want = np.zeros((batch, level + 1 - nb, N), dtype=U64)
                for b in range(batch):
                    tmp = np.zeros((level + 1, N), dtype=U64); buff = np.zeros((level + 1, N), dtype=U64)
                    r = ring.AtLevel(level)
                    if rnd and ntt: r.DivRoundByLastModulusManyNTT(nb, x[b].copy(), buff, tmp)
                    elif rnd: r.DivRoundByLastModulusMany(nb, x[b].copy(), buff, tmp)
                    elif ntt: r.DivFloorByLastModulusManyNTT(nb, x[b].copy(), tmp)
                    else: r.DivFloorByLastModulusMany(nb, x[b].copy(), buff, tmp)
                    want[b] = tmp[: level + 1 - nb]
                out = ctx.new_poly(level + 1 - nb, batch)
                lb.div_by_last_modulus_many(ctx, 0, level, rnd, ntt, nb, dx, out)
                assert np.array_equal(ctx.to_host(out), want), (nb, rnd, ntt)
    # single-rescale NTT variant at a lower level, in place on the first rows
    lvl = 3
    y = x[:, : lvl + 1].copy()
    want = np.zeros((batch, lvl, N), dtype=U64)
    for b in range(batch):
        tmp = np.zeros((lvl + 1, N), dtype=U64)
        ring.AtLevel(lvl).DivRoundByLastModulusNTT(y[b].copy(), tmp)
        want[b] = tmp[:lvl]
    dy = ctx.to_device(y); out = ctx.new_poly(lvl, batch)
    lb.div_by_last_modulus_many(ctx, 0, lvl, True, True, 1, dy, out)
    assert np.array_equal(ctx.to_host(out), want)


def test_automorphisms(small):
    lb, ctx, params, q, p = small
    N = params.N()
    ring = params.ringQ
    rng = np.random.default_rng(5)
    x = H.rand_poly(q, N, rng)
    dx = ctx.to_device(x)
    level = len(q) - 1
    for gal in (5, params.GaloisElement(7), params.GaloisElement(-3), 2 * N - 1):
        idx_o = ring.AutomorphismNTTIndex(gal)
        idx = lb.automorphism_ntt_index(ctx, gal)
        assert np.array_equal(ctx.to_host(idx), idx_o)
        want = np.zeros_like(x); ring.AutomorphismNTTWithIndex(x, idx_o, want)
        out = ctx.new_poly(level + 1)
        lb.automorphism_ntt_with_index(ctx, 0, level, dx, idx, out)
        assert np.array_equal(ctx.to_host(out), want)
        out2 = ctx.new_poly(level + 1)
        lb.automorphism_ntt(ctx, 0, level, dx, gal, out2)
        assert np.array_equal(ctx.to_host(out2), want)
        acc = H.rand_poly(q, N, rng); want_acc = acc.copy()
        ring.AutomorphismNTTWithIndexThenAddLazy(x, idx_o, want_acc)
        dacc = ctx.to_device(acc)
        lb.automorphism_ntt_with_index(ctx, 0, level, dx, idx, dacc, accumulate=True)
        assert np.array_equal(ctx.to_host(dacc), want_acc)
        wc = np.zeros_like(x); ring.Automorphism(x, gal, wc)
        oc = ctx.new_poly(level + 1)
        lb.automorphism(ctx, 0, level, dx, gal, oc)
        assert np.array_equal(ctx.to_host(oc), wc)
    with pytest.raises(lb.LgpuError):
        lb.automorphism_ntt(ctx, 0, level, dx, 5, dx)       # cannot be in-place (ring/automorphism.go:37)


def _gadget_case(lb, logN, q, p, pw2, levels, batch=2, seed=0):
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(seed)
    ev_o = O.Evaluator(params)
    ev = lb.Evaluator(ctx)
    evk_o = H.random_gadget_ciphertext(params, params.MaxLevelQ(), params.MaxLevelP(), rng, pw2=pw2)
    evk = lb.GadgetCiphertext(ctx, evk_o.data, evk_o.LevelQ(), evk_o.LevelP(), pw2, evk_o.pw2_sizes)
    levelP = params.MaxLevelP()
    for levelQ in levels:
        cx = np.stack([H.rand_poly(q[: levelQ + 1], N, rng) for _ in range(batch)])
        want = np.zeros((batch, 2, levelQ + 1, N), dtype=U64)
        wantlazy = [np.zeros((batch, 2, levelQ + 1, N), dtype=U64), np.zeros((batch, 2, max(levelP + 1, 1), N), dtype=U64)]
        for b in range(batch):
            ct = [want[b, 0], want[b, 1]]
            ev_o.GadgetProduct(levelQ, cx[b].copy(), evk_o, ct)
            ev_o.GadgetProductLazy(levelQ, cx[b].copy(), evk_o, [wantlazy[0][b, 0], wantlazy[0][b, 1]], [wantlazy[1][b, 0], wantlazy[1][b, 1]])
        dcx = ctx.to_device(cx)
        c0 = ctx.new_poly(levelQ + 1, batch); c1 = ctx.new_poly(levelQ + 1, batch)
        ev.GadgetProduct(levelQ, dcx, evk, c0, c1)
        assert np.array_equal(ctx.to_host(c0), want[:, 0]) and np.array_equal(ctx.to_host(c1), want[:, 1]), (pw2, levelQ)
        a0q = ctx.new_poly(levelQ + 1, batch); a1q = ctx.new_poly(levelQ + 1, batch)
        a0p = ctx.new_poly(max(levelP + 1, 1), batch); a1p = ctx.new_poly(max(levelP + 1, 1), batch)
        ev.GadgetProductLazy(levelQ, dcx, evk, a0q, a0p if levelP >= 0 else None, a1q, a1p if levelP >= 0 else None)
        assert np.array_equal(ctx.to_host(a0q), wantlazy[0][:, 0]) and np.array_equal(ctx.to_host(a1q), wantlazy[0][:, 1])
        if levelP >= 0:
            assert np.array_equal(ctx.to_host(a0p), wantlazy[1][:, 0]) and np.array_equal(ctx.to_host(a1p), wantlazy[1][:, 1])
            m0 = ctx.new_poly(levelQ + 1, batch); m1 = ctx.new_poly(levelQ + 1, batch)
            ev.ModDown(levelQ, levelP, a0q, a0p, a1q, a1p, m0, m1)
            assert np.array_equal(ctx.to_host(m0), want[:, 0]) and np.array_equal(ctx.to_host(m1), want[:, 1])
    ctx.close()
    return True


def test_gadget_product_multiple_p():
    """core/rlwe/test_params.go:17-27 shape (k = 2, no pw2) + a k = 3 chain with a ragged last digit."""
    lb = _lb()
    q, p = _mods(8, [45, 35, 35, 35, 35], [50, 50])
    _gadget_case(lb, 8, q, p, 0, (4, 3, 1, 0))
    q, p = _mods(8, [56, 45, 45, 45, 45, 45, 45], [55, 55, 55])
    _gadget_case(lb, 8, q, p, 0, (6, 4, 2), seed=1)
    _gadget_case(lb, 8, H.Qi60[:5], H.Pi60[:2], 0, (4, 2), seed=2)


def test_gadget_product_fused_pipeline_logn13():
    """logN = 13 is the smallest ring that takes the fused key-switch pipeline (keyswitch_fused.cu): FP64 rows (45-bit
    primes) and integer rows (55/56-bit) mixed, ragged last digit, single-limb last digit, k = 3 and k = 2."""
    lb = _lb()
    q, p = _mods(13, [56, 45, 45, 45, 45, 45, 45], [55, 55, 55])
    _gadget_case(lb, 13, q, p, 0, (6, 5, 4, 3, 2, 0), seed=11)
    _gadget_case(lb, 13, q, p[:2], 0, (6, 5, 1), seed=12)
    # 40-bit scale primes, 50-bit P (examples/params.go:115-120 shape)
    q, p = _mods(14, [51, 40, 40, 40, 40], [50, 50])
    _gadget_case(lb, 14, q, p, 0, (4, 3), batch=3, seed=13)


def test_gadget_product_fused_pipeline_lazy_key_words():
    """Key words are canonical residues in the reference, but MRedLazy only needs their residue class: the FP64-pipe MAC of the fused pipeline
    (K3, LGPU_K3_VARIANT=11) Barrett-reduces key words at or above 2^46 before converting them. Same product with key + m*q on the 45-bit rows."""
    lb = _lb()
    logN = 13
    q, p = _mods(logN, [56, 45, 45, 45, 45, 45, 45], [55, 55, 55])
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(21)
    ev_o = O.Evaluator(params); ev = lb.Evaluator(ctx)
    evk_o = H.random_gadget_ciphertext(params, params.MaxLevelQ(), params.MaxLevelP(), rng)
    lazy = evk_o.data.copy()                       # [digit][pw2][component][Q rows | P rows][N]
    for r, qi in enumerate(q):
        if qi < (1 << 46):
            m = rng.integers(0, 1 << 16, size=lazy[..., r, :].shape, dtype=np.uint64)
            m[..., ::3] = 0                        # a third of the words stay canonical: the guard is per group of words
            lazy[..., r, :] += m * np.uint64(qi)
    assert int(lazy.max()) >= 1 << 46
    evk = lb.GadgetCiphertext(ctx, lazy, evk_o.LevelQ(), evk_o.LevelP(), 0, evk_o.pw2_sizes)
    for levelQ in (6, 4):
        batch = 2
        cx = np.stack([H.rand_poly(q[: levelQ + 1], N, rng) for _ in range(batch)])
        want = np.zeros((batch, 2, levelQ + 1, N), dtype=U64)
        for b in range(batch):
            ev_o.GadgetProduct(levelQ, cx[b].copy(), evk_o, [want[b, 0], want[b, 1]])
        c0 = ctx.new_poly(levelQ + 1, batch); c1 = ctx.new_poly(levelQ + 1, batch)
        ev.GadgetProduct(levelQ, ctx.to_device(cx), evk, c0, c1)
        assert np.array_equal(ctx.to_host(c0), want[:, 0]) and np.array_equal(ctx.to_host(c1), want[:, 1]), levelQ
    ctx.close()


def test_gadget_product_single_p_and_bit_decomp():
    """core/rlwe/test_params.go:28-49: k = 1 with pw2 = 16; k = 0 (no P) with pw2 = 2; k = 1 without pw2."""
    lb = _lb()
    q, p = _mods(8, [45, 35, 35, 35, 35], [50, 50])
    _gadget_case(lb, 8, q, p[:1], 16, (4, 1, 0), seed=3)
    _gadget_case(lb, 8, q, [], 2, (4, 0), seed=4)
    _gadget_case(lb, 8, q, p[:1], 0, (4, 2, 0), seed=5)


def test_hoisted_automorphism_relinearize(small):
    lb, ctx, params, q, p = small
    N = params.N()
    rng = np.random.default_rng(6)
    ev_o = O.Evaluator(params); ev = lb.Evaluator(ctx)
    levelP = params.MaxLevelP()
    evk_o = H.random_gadget_ciphertext(params, params.MaxLevelQ(), levelP, rng)
    evk = lb.GadgetCiphertext(ctx, evk_o.data, evk_o.LevelQ(), evk_o.LevelP())
    batch = 2
    for levelQ in (params.MaxLevelQ(), 3):
        n = params.BaseRNSDecompositionVectorSize(levelQ, levelP)
        ct = np.stack([np.stack([H.rand_poly(q[: levelQ + 1], N, rng) for _ in range(3)]) for _ in range(batch)])   # degree 2
        dct = ctx.to_device(ct)
        # DecomposeNTT
        dec = ev.DecomposeNTT(levelQ, levelP, levelP + 1, dct[:, 1].contiguous(), True)
        dec_h = ctx.to_host(dec)
        want_h = np.zeros((batch, 2, levelQ + 1, N), dtype=U64)
        want_a = np.zeros((batch, 2, levelQ + 1, N), dtype=U64)
        want_r = np.zeros((batch, 2, levelQ + 1, N), dtype=U64)
        gal = params.GaloisElement(5)
        for b in range(batch):
            dq = [np.zeros((levelQ + 1, N), dtype=U64) for _ in range(n)]; dp = [np.zeros((levelP + 1, N), dtype=U64) for _ in range(n)]
            ev_o.DecomposeNTT(levelQ, levelP, levelP + 1, ct[b, 1].copy(), True, dq, dp)
            for i in range(n):
                assert np.array_equal(dec_h[i, b, : levelQ + 1], dq[i]) and np.array_equal(dec_h[i, b, levelQ + 1:], dp[i]), (levelQ, i)
            ev_o.GadgetProductHoisted(levelQ, dq, dp, evk_o, [want_h[b, 0], want_h[b, 1]])
            ev_o.Automorphism([ct[b, 0], ct[b, 1]], gal, evk_o, [want_a[b, 0], want_a[b, 1]])
            ev_o.Relinearize([ct[b, 0], ct[b, 1], ct[b, 2]], evk_o, [want_r[b, 0], want_r[b, 1]])
        h0 = ctx.new_poly(levelQ + 1, batch); h1 = ctx.new_poly(levelQ + 1, batch)
        ev.GadgetProductHoisted(levelQ, dec, evk, h0, h1)
        assert np.array_equal(ctx.to_host(h0), want_h[:, 0]) and np.array_equal(ctx.to_host(h1), want_h[:, 1])
        ct2 = dct[:, :2].contiguous()
        out = ctx.to_device(np.zeros((batch, 2, levelQ + 1, N), dtype=U64))
        ev.Automorphism(ct2, gal, evk, out)
        assert np.array_equal(ctx.to_host(out), want_a)
        out_h = ctx.to_device(np.zeros((batch, 2, levelQ + 1, N), dtype=U64))
        ev.Automorphism(ct2, gal, evk, out_h, decomp=dec)                  # AutomorphismHoisted
        assert np.array_equal(ctx.to_host(out_h), want_a)
        out_r = ctx.to_device(np.zeros((batch, 2, levelQ + 1, N), dtype=U64))
        ev.Relinearize(dct, evk, out_r)
        assert np.array_equal(ctx.to_host(out_r), want_r)


def test_ckks_mulrelin_rescale_small_and_host_path():
    lb = _lb()
    logN = 10
    q, p = _mods(logN, [56, 45, 45, 45, 45, 45], [55, 55])
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(7)
    rlk_o = H.random_gadget_ciphertext(params, params.MaxLevelQ(), params.MaxLevelP(), rng)
    rlk = lb.GadgetCiphertext(ctx, rlk_o.data, rlk_o.LevelQ(), rlk_o.LevelP())
    ev_o = O.CKKSEvaluator(params, rlk_o); ev = lb.CKKSEvaluator(ctx, rlk)
    batch = 5
    for level in (5, 3, 1):
        a = np.stack([np.stack([H.rand_poly(q[: level + 1], N, rng) for _ in range(2)]) for _ in range(batch)])
        b = np.stack([np.stack([H.rand_poly(q[: level + 1], N, rng) for _ in range(2)]) for _ in range(batch)])
        want_m = np.zeros((batch, 2, level + 1, N), dtype=U64); want = np.zeros((batch, 2, level, N), dtype=U64)
        for i in range(batch):
            m = ev_o.MulRelinNew([a[i, 0], a[i, 1]], [b[i, 0], b[i, 1]])
            r = ev_o.Rescale(m)
            want_m[i, 0], want_m[i, 1] = m; want[i, 0], want[i, 1] = r
        da, db = ctx.to_device(a), ctx.to_device(b)
        got_m = ev.MulRelinNew(da, db)
        assert np.array_equal(ctx.to_host(got_m), want_m), level
        assert np.array_equal(ctx.to_host(ev.Rescale(got_m)), want), level
        assert np.array_equal(ctx.to_host(ev.MulRelinRescaleNew(da, db)), want), level
        out_host = np.zeros((batch, 2, level, N), dtype=U64)
        ev.MulRelinRescaleHost(a, b, out_host, chunk=2)          # host buffers through the C ABI, copies inside
        assert np.array_equal(out_host, want), level
    ctx.close()


def test_ckks_mulrelin_rescale_full_size_pn16qp1761():
    """BASELINE config 3 at full size (N = 2^16, 34 + 4 limbs): bit-exact vs the oracle for 2 ciphertext pairs,
    and batch-consistency (element i of a batch == the same pair evaluated alone) as the size-independent check."""
    _pn16qp1761_case(batch=6, n_oracle=2)


def test_ckks_mulrelin_rescale_full_size_pn16qp1761_batch16():
    """The same at batch 16, where the ModDown INTT of the 4 P rows runs 64 limb-transforms (the persistent kernels):
    every pair against the oracle."""
    _pn16qp1761_case(batch=16, n_oracle=16)


def _pn16qp1761_case(batch, n_oracle):
    import torch
    lb = _lb()
    from lattigo_b200 import params as presets
    s = presets.PRESETS["CKKS_PN16QP1761"]
    logN, q, p = s["logN"], s["Q"], s["P"]
    ctx = lb.Context(logN, q, p)
    N = 1 << logN
    level, levelP = len(q) - 1, len(p) - 1
    nd = (level + levelP + 1) // (levelP + 1)
    g = torch.Generator(device="cuda"); g.manual_seed(11)

    def rand_rows(mods, lead):
        out = torch.empty(tuple(lead) + (len(mods), N), dtype=torch.int64, device="cuda")
        for i, m in enumerate(mods):
            out[..., i, :] = torch.randint(0, m, tuple(lead) + (N,), generator=g, device="cuda", dtype=torch.int64)
        return out

    evk_t = rand_rows(q + p, (nd, 1, 2))
    rlk = lb.GadgetCiphertext(ctx, evk_t, level, levelP)
    ev = lb.CKKSEvaluator(ctx, rlk)
    a = rand_rows(q, (batch, 2)); b = rand_rows(q, (batch, 2))
    out = ev.MulRelinRescaleNew(a, b)
    torch.cuda.synchronize()
    one = ev.MulRelinRescaleNew(a[4:5].contiguous(), b[4:5].contiguous())
    assert torch.equal(out[4:5], one)
    # oracle on the first n_oracle pairs
    params = O.Parameters(logN, q, p)
    rlk_o = O.GadgetCiphertext(ctx.to_host(evk_t), level + 1, levelP + 1)
    ev_o = O.CKKSEvaluator(params, rlk_o)
    n = n_oracle
    ah, bh, oh = ctx.to_host(a[:n]), ctx.to_host(b[:n]), ctx.to_host(out[:n])
    for i in range(n):
        r = ev_o.Rescale(ev_o.MulRelinNew([ah[i, 0], ah[i, 1]], [bh[i, 0], bh[i, 1]]))
        assert np.array_equal(oh[i, 0], r[0]) and np.array_equal(oh[i, 1], r[1]), i
    ctx.close()


def test_ringqp_dispatch(small):
    """ringqp.Ring ops = RingQ op then RingP op (ring/ringqp/operations.go:8-316)."""
    lb, ctx, params, q, p = small
    N = params.N()
    rng = np.random.default_rng(21)
    levelQ, levelP = 4, 1
    rqp = lb.RingQP(ctx).AtLevel(levelQ, levelP)
    oq, op = params.ringQ.AtLevel(levelQ), params.ringP.AtLevel(levelP)
    aq, ap = H.rand_poly(q[: levelQ + 1], N, rng), H.rand_poly(p[: levelP + 1], N, rng)
    bq, bp = H.rand_poly(q[: levelQ + 1], N, rng), H.rand_poly(p[: levelP + 1], N, rng)
    A = lb.PolyQP(ctx.to_device(aq), ctx.to_device(ap)); B = lb.PolyQP(ctx.to_device(bq), ctx.to_device(bp))
    C = rqp.NewPoly()
    for name in ("Add", "Sub", "MulCoeffsMontgomery", "MulCoeffsMontgomeryLazy"):
        wq, wp = np.zeros_like(aq), np.zeros_like(ap)
        getattr(oq, name)(aq, bq, wq); getattr(op, name)(ap, bp, wp)
        getattr(rqp, name)(A, B, C)
        assert np.array_equal(ctx.to_host(C.Q), wq) and np.array_equal(ctx.to_host(C.P), wp), name
    wq, wp = np.zeros_like(aq), np.zeros_like(ap)
    oq.NTT(aq, wq); op.NTT(ap, wp)
    rqp.NTT(A, C)
    assert np.array_equal(ctx.to_host(C.Q), wq) and np.array_equal(ctx.to_host(C.P), wp)
    rqp.INTT(C, C)
    assert np.array_equal(ctx.to_host(C.Q), aq) and np.array_equal(ctx.to_host(C.P), ap)


def test_bgv_rotate_full_size_n15qp880():
    """BASELINE config 4 shape: BGV N15QP880 RotateColumns = Evaluator.Automorphism (key-switch + NTT-domain
    permutation), batch of ciphertexts, bit-exact vs the oracle for 2 of them + batch consistency."""
    _bgv_n15qp880_rotate_case(batch=5, n_oracle=2)


def test_bgv_rotate_full_size_n15qp880_batch16():
    """The same at batch 16, every ciphertext against the oracle: the ModDown INTT of the 4 P rows runs 64
    limb-transforms of 47-bit primes at N = 2^15, the persistent integer inverse without lazy corrections
    (IntInvOps<3, 2>), which no other preset selects."""
    _bgv_n15qp880_rotate_case(batch=16, n_oracle=16)


def _bgv_n15qp880_rotate_case(batch, n_oracle):
    import torch
    lb = _lb()
    from lattigo_b200 import params as presets
    s = presets.PRESETS["BGV_N15QP880"]
    logN, q, p = s["logN"], s["Q"], s["P"]
    ctx = lb.Context(logN, q, p)
    N = 1 << logN
    level, levelP = len(q) - 1, len(p) - 1
    nd = (level + levelP + 1) // (levelP + 1)
    g = torch.Generator(device="cuda"); g.manual_seed(5)

    def rand_rows(mods, lead):
        out = torch.empty(tuple(lead) + (len(mods), N), dtype=torch.int64, device="cuda")
        for i, m in enumerate(mods):
            out[..., i, :] = torch.randint(0, m, tuple(lead) + (N,), generator=g, device="cuda", dtype=torch.int64)
        return out

    gk_t = rand_rows(q + p, (nd, 1, 2))
    gk = lb.GadgetCiphertext(ctx, gk_t, level, levelP)
    ev = lb.Evaluator(ctx)
    params = O.Parameters(logN, q, p)
    galEl = params.GaloisElement(3)
    ct = rand_rows(q, (batch, 2))
    out = torch.zeros_like(ct)
    ev.Automorphism(ct, galEl, gk, out)
    one = torch.zeros_like(ct[3:4])
    ev.Automorphism(ct[3:4].contiguous(), galEl, gk, one)
    assert torch.equal(out[3:4], one)
    gk_o = O.GadgetCiphertext(ctx.to_host(gk_t), level + 1, levelP + 1)
    ev_o = O.Evaluator(params)
    n = n_oracle
    cth, oh = ctx.to_host(ct[:n]), ctx.to_host(out[:n])
    for i in range(n):
        w = [np.zeros((level + 1, N), dtype=U64) for _ in range(2)]
        ev_o.Automorphism([cth[i, 0], cth[i, 1]], galEl, gk_o, w)
        assert np.array_equal(oh[i, 0], w[0]) and np.array_equal(oh[i, 1], w[1]), i
    ctx.close()


def test_unaligned_buffers():
    """Polynomials at an odd word offset (8- but not 16-byte aligned): ring-level calls route them to the 64-bit
    kernels and stay bit-exact; the rlwe-level calls (128-bit accesses) refuse them with an error, as the header says."""
    import torch
    lb = _lb()
    logN = 13
    q, p = _mods(logN, [56, 45, 45, 45], [55, 55])
    ctx = lb.Context(logN, q, p)
    params = O.Parameters(logN, q, p)
    N = params.N()
    rng = np.random.default_rng(71)
    level = 3

    def odd(arr):
        flat = torch.zeros(arr.size + 1, dtype=torch.int64, device="cuda")
        view = flat[1:].view(*arr.shape)
        view.copy_(ctx.to_device(arr))
        assert view.data_ptr() % 16 == 8
        return view

    x = H.rand_poly(q, N, rng)
    ring = O.Ring(N, q)
    want = np.empty_like(x); want_i = np.empty_like(x); want_m = np.empty_like(x)
    ring.NTT(x, want); ring.INTT(x, want_i); ring.MulCoeffsMontgomery(x, x, want_m)
    dx = odd(x); out = odd(np.zeros_like(x))
    ctx.ringQ.NTT(dx, out)
    assert np.array_equal(ctx.to_host(out), want)
    ctx.ringQ.INTT(dx, out)
    assert np.array_equal(ctx.to_host(out), want_i)
    ctx.ringQ.MulCoeffsMontgomery(dx, dx, out)
    assert np.array_equal(ctx.to_host(out), want_m)
    rlk_o = H.random_gadget_ciphertext(params, level, params.MaxLevelP(), rng)
    rlk = lb.GadgetCiphertext(ctx, rlk_o.data, rlk_o.LevelQ(), rlk_o.LevelP())
    cx = H.rand_poly(q, N, rng)
    c0 = ctx.ringQ.NewPoly(); c1 = ctx.ringQ.NewPoly()
    with pytest.raises(lb.LgpuError, match="16-byte aligned"):
        lb.Evaluator(ctx).GadgetProduct(level, odd(cx), rlk, c0, c1)
    with pytest.raises(lb.LgpuError, match="16-byte aligned"):
        lb.Evaluator(ctx).GadgetProduct(level, ctx.to_device(cx), rlk, odd(np.zeros_like(cx)), c1)
    bad = lb.GadgetCiphertext(ctx, odd(rlk_o.data), rlk_o.LevelQ(), rlk_o.LevelP())
    with pytest.raises(lb.LgpuError, match="16-byte aligned"):
        lb.Evaluator(ctx).GadgetProduct(level, ctx.to_device(cx), bad, c0, c1)
    a = np.stack([H.rand_poly(q, N, rng) for _ in range(2)])[None]
    with pytest.raises(lb.LgpuError, match="16-byte aligned"):
        lb.CKKSEvaluator(ctx, rlk).MulRelinRescaleNew(odd(a), ctx.to_device(a))
    ctx.close()


@pytest.mark.parametrize("env", ["LGPU_K3_VARIANT=0", "LGPU_K3_VARIANT=10", "LGPU_K3_VARIANT=12", "LGPU_K3_VARIANT=13", "LGPU_K2_SPLIT=0", "LGPU_K2_J4=0", "LGPU_FZ_VARIANT=0", "LGPU_NO_FUSED_KS=1", "LGPU_NO_FP64_NTT=1",
                                 "LGPU_SIDE_STREAM=1", "LGPU_BATCH_CHUNK=1"])
def test_fallback_kernel_variants_stay_bit_exact(env):
    """The development switches select the older / unfused kernels (read once per process, hence a subprocess); every
    one of them must reproduce the oracle on the fused-pipeline cases too."""
    import subprocess
    import sys
    k, v = env.split("=")
    e = dict(os.environ, **{k: v})
    root = os.path.dirname(HERE)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_keyswitch.py"), "-m", "gpu", "-x", "-q", "-k",
                        "fused_pipeline_logn13 or mulrelin_rescale_small"], cwd=root, env=e, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]

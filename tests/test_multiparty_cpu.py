"""Argument checks of the multiparty entry points (include/lattigo_b200.h, lgpu_mp_*), which run before any launch and so also on a
host-only context; the reference's AggregateShares errors raised by lattigo_b200.multiparty; the smudging distribution of
KeySwitchProtocol."""
import ctypes

import pytest

QI = [0x200000440001, 0x7fff80001, 0x800280001, 0x7ffd80001, 0x7ffc80001]
PJ = [0x3ffffffb80001, 0x4000000800001]
FAKE = ctypes.c_void_p(1 << 20)          # never dereferenced: every case fails its checks first


@pytest.fixture(scope="module")
def ctx():
    import lattigo_b200 as lb
    c = lb.Context(10, QI, PJ, device=-1)
    yield c
    c.close()


def _err(rc):
    import lattigo_b200 as lb
    assert rc == -1
    return lb.lib().lgpu_last_error().decode()


def _ptrs(*addrs):
    return (ctypes.c_void_p * len(addrs))(*addrs)


@pytest.mark.parametrize("lq,lp,k,n,msg", [
    (5, -1, 1, 1, "level out of range"), (-1, -1, 1, 1, "level out of range"), (4, 2, 1, 1, "level out of range"), (4, -2, 1, 1, "level out of range"),
    (4, 1, 0, 1, "n_shares out of [1, 65535]"), (4, 1, 65536, 1, "n_shares out of [1, 65535]"), (4, 1, 1, 0, "n_polys must be at least 1"),
])
def test_aggregate_rejects_bad_shapes(ctx, lq, lp, k, n, msg):
    import lattigo_b200 as lb
    ptrs = _ptrs(*([1 << 20] * max(1, min(k, 4))))
    assert msg in _err(lb.lib().lgpu_mp_aggregate(ctx.h, lq, lp, ptrs, k, FAKE, n, None))


def test_aggregate_rejects_null_and_overlap(ctx):
    import lattigo_b200 as lb
    L = lb.lib()
    assert "null argument" in _err(L.lgpu_mp_aggregate(ctx.h, 4, 1, None, 2, FAKE, 1, None))
    assert "null argument" in _err(L.lgpu_mp_aggregate(ctx.h, 4, 1, _ptrs(1 << 20, 1 << 21), 2, None, 1, None))
    assert "null share" in _err(L.lgpu_mp_aggregate(ctx.h, 4, 1, _ptrs(1 << 20, None), 2, ctypes.c_void_p(1 << 30), 1, None))
    # out may be shares[0], but not any later share, nor overlap one
    assert "overlaps" in _err(L.lgpu_mp_aggregate(ctx.h, 4, 1, _ptrs(1 << 20, 1 << 30), 2, ctypes.c_void_p(1 << 30), 1, None))
    assert "overlaps" in _err(L.lgpu_mp_aggregate(ctx.h, 4, 1, _ptrs(1 << 20, 1 << 30), 2, ctypes.c_void_p((1 << 20) + 8), 1, None))
    # valid arguments reach the device check
    assert "host-only" in _err(L.lgpu_mp_aggregate(ctx.h, 4, 1, _ptrs(1 << 20, 1 << 30), 2, ctypes.c_void_p(1 << 20), 1, None))


def test_key_switch_share_checks(ctx):
    import lattigo_b200 as lb
    L = lb.lib()
    N = ctx.N
    ok = dict(level=2, c1=ctypes.c_void_p(1 << 30), stride=6 * N, s_in=FAKE, s_out=FAKE, e=FAKE, share=ctypes.c_void_p(1 << 20), batch=3)

    def call(**kw):
        a = dict(ok, **kw)
        return _err(L.lgpu_mp_key_switch_share(ctx.h, a["level"], a["c1"], a["stride"], a["s_in"], a["s_out"], a["e"], a["share"], a["batch"], None))
    assert "level out of range" in call(level=5)
    assert "level out of range" in call(level=-1)
    assert "batch out of range" in call(batch=0)
    assert "batch out of range" in call(batch=65536)
    for k in ("c1", "s_in", "s_out", "e", "share"):
        assert "null argument" in call(**{k: None})
    assert "stride below" in call(stride=3 * N - 1)
    assert "overlaps" in call(share=ctypes.c_void_p((1 << 30) + 8 * 6 * N))
    assert "host-only" in call()


def test_public_key_switch_share_checks(ctx):
    import lattigo_b200 as lb
    L = lb.lib()
    N = ctx.N
    ok = dict(level=4, c1=ctypes.c_void_p(1 << 30), stride=10 * N, sk=FAKE, pk=FAKE, u=FAKE, e0=FAKE, e1=FAKE, ef=FAKE,
              share=ctypes.c_void_p(1 << 20), batch=2)

    def call(**kw):
        a = dict(ok, **kw)
        return _err(L.lgpu_mp_public_key_switch_share(ctx.h, a["level"], a["c1"], a["stride"], a["sk"], a["pk"], a["u"], a["e0"], a["e1"], a["ef"],
                                                      a["share"], a["batch"], None))
    assert "level out of range" in call(level=5)
    assert "batch out of range" in call(batch=0)
    for k in ("c1", "sk", "pk", "u", "e0", "e1", "ef", "share"):
        assert "null argument" in call(**{k: None})
    assert "stride below" in call(stride=5 * N - 1)
    assert "overlaps" in call(share=ctypes.c_void_p((1 << 30) - 8))
    assert "host-only" in call()


def test_aggregate_shares_raises_the_reference_errors(ctx):
    import torch
    import lattigo_b200 as lb
    from lattigo_b200 import multiparty as mp
    N = ctx.N
    S = lb.encryptor.Samplers(ctx, 1)
    cks = mp.KeySwitchProtocol(ctx, S, 8 * 3.2)
    with pytest.raises(lb.LgpuError, match="cannot AggregateShares: shares levels do not match"):
        cks.AggregateShares(torch.zeros(1, 3, N, dtype=torch.int64), torch.zeros(1, 2, N, dtype=torch.int64))
    pcks = mp.PublicKeySwitchProtocol(ctx, S, 8 * 3.2)
    with pytest.raises(lb.LgpuError, match="cannot AggregateShares: the two shares are at different levelQ"):
        pcks.AggregateShares(torch.zeros(1, 2, 3, N, dtype=torch.int64), torch.zeros(1, 2, 2, N, dtype=torch.int64))
    ckg = mp.PublicKeyGenProtocol(ctx, S)
    with pytest.raises(lb.LgpuError, match="cannot AggregateShares"):
        ckg.AggregateShares(torch.zeros(7, N, dtype=torch.int64), torch.zeros(6, N, dtype=torch.int64))
    with pytest.raises(lb.LgpuError, match="at least one share"):
        ckg.AggregateShares([])


def test_key_switch_smudging_distribution():
    """keyswitch_sk.go:45-52: sigma' = sqrt(NoiseFreshSK^2 + sigma_flood^2), bound 6 sigma'."""
    from lattigo_b200 import multiparty as mp
    p = mp.KeySwitchProtocol.__new__(mp.KeySwitchProtocol)
    mp.KeySwitchProtocol.__init__(p, None, None, 8 * 3.2)
    assert p.sigma == pytest.approx((3.2 ** 2 + 25.6 ** 2) ** 0.5) and p.bound == 6 * p.sigma
    mp.KeySwitchProtocol.__init__(p, None, None, 2.0 ** 30)
    assert p.bound < 9.0e18                                                       # inside the device Gaussian sampler's range


def test_crs_and_party_streams(ctx, monkeypatch):
    """SampleCRP of two protocol instances on CRS samplers with one seed draws the same (seed, stream id) sequence, so every party gets
    the same CRP; parties draw their own noise on their own seeds, one fresh stream id per draw."""
    import lattigo_b200 as lb
    from lattigo_b200 import multiparty as mp
    calls = []

    class FakeLib:
        def __getattr__(self, name):
            def f(h, *args):
                calls.append((name, args))
                return 0
            return f

    class T:
        is_cuda = True
        def data_ptr(self): return 1 << 20
        def is_contiguous(self): return True
        def element_size(self): return 8
        def __getitem__(self, i): return self
        def view(self, *a): return self

    monkeypatch.setattr(lb._lib, "lib", lambda: FakeLib())
    monkeypatch.setattr(lb.encryptor, "_stream", lambda: None)
    monkeypatch.setattr(lb.ring.Context, "new_poly", lambda self, limbs, batch=None: T())

    def draws(fn):
        del calls[:]
        fn()
        return [(a[-6], a[-5]) if n == "lgpu_sample_uniform" else (a[-5], a[-4]) for n, a in calls]

    crs_a, crs_b = lb.encryptor.Samplers(ctx, 42), lb.encryptor.Samplers(ctx, 42)
    pa = mp.RelinearizationKeyGenProtocol(ctx, lb.encryptor.Samplers(ctx, 1))
    pb = mp.RelinearizationKeyGenProtocol(ctx, lb.encryptor.Samplers(ctx, 2))
    ids_a = draws(lambda: pa.SampleCRP(crs_a))
    assert ids_a == draws(lambda: pb.SampleCRP(crs_b)) == [(42, 1), (42, 1)]      # Q and P rows of the CRP on one id
    assert draws(lambda: (pa._gauss((2,)), pa._gauss((2,)))) == [(1, 1), (1, 2)]
    assert draws(lambda: pb._gauss((2,))) == [(2, 1)]

"""The mpbgv protocols on the device (csrc/mp_refresh.cu, lattigo_b200/mpbgv.py) word for word against tests/mp_refresh_oracle.py on the
same samples, on the reference's test set (multiparty/mpbgv/test_parameters.go, testInsecure) with t = 0x101 (n = 128, gap 8) and
t = 0xffc001 (n = N, gap 1), K = 1, 2, 5 parties: every E2S / S2E share, aggregate, secret share and output ciphertext, at E2S levels 0
and > 0 (all four RingQ2T branches), with the ciphertext above the E2S level, batch 1 and 3; MaskedTransform with all four Decode /
Encode combinations around a permutation; the mask sampler against its restated stream; and end to end, refreshed and permuted
ciphertexts decrypting exactly under the ideal key."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests import mp_refresh_oracle as R
from tests import multiparty_oracle as M

pytestmark = pytest.mark.gpu
U64 = np.uint64
QI = [0x3fffffa8001, 0x1000090001, 0x10000c8001, 0x10000f0001, 0xffff00001]
PJ = [0x7fffffd8001]
SIGMA = 3.2


class _Env:
    def __init__(self, t, K, seed):
        import lattigo_b200 as lb
        self.lb = lb
        self.params = O.Parameters(10, QI, PJ)
        self.N = self.params.N()
        self.ctx = lb.Context(10, QI, PJ)
        self.enc = lb.BGVEncoder(self.ctx, t)
        self.t, self.n = t, self.enc.n
        self.rng = np.random.default_rng(seed)
        self.crs = lb.encryptor.Samplers(self.ctx, 0xC0FFEE + seed)
        self.party = [lb.encryptor.Samplers(self.ctx, 1000 + 17 * seed + i) for i in range(K)]
        self.s = [self.ctx.to_host(self.party[i].Ternary(P=2 / 3))[0] for i in range(K)]
        self.sk = [M.sk_rows(self.params, si) for si in self.s]
        self.d_sk = [self.ctx.to_device(x) for x in self.sk]
        self.ideal = M.sk_rows(self.params, sum(self.s))
        self.P = R.MPBGV(self.params, t)
        self.protos = [lb.mpbgv.MaskedTransformProtocol(self.enc, self.party[i], SIGMA) for i in range(K)]

    def values(self, batch):
        return [[int(v) for v in self.rng.integers(0, self.t, self.n)] for _ in range(batch)]

    def cts(self, vals, level, scale):
        out = []
        for v in vals:
            a = H.rand_poly(QI[: level + 1], self.N, self.rng)
            e = np.rint(self.rng.normal(0, SIGMA, self.N)).astype(np.int64)
            out.append(self.P.encrypt(self.ideal, v, level, scale, a, e))
        return np.stack(out)

    def host(self, x):
        return self.ctx.to_host(x)

    def close(self):
        self.enc.close()
        self.ctx.close()


@pytest.fixture
def env(request):
    e = _Env(*request.param)
    yield e
    e.close()


CASES = [(t, K, 3 * K + i) for i, t in enumerate((0x101, 0xffc001)) for K in (1, 2, 5)]
_ids = lambda c: "t%x-K%d" % c[:2]


def _perm_func(perm):
    import torch
    idx = torch.as_tensor(perm, dtype=torch.int64, device="cuda")

    def f(coeffs):
        coeffs.copy_(coeffs[:, idx])
    return f


def _run(env, level_ct, level_e2s, batch, transform_spec, scale=5):
    """GenShare of every party, AggregateShares and Transform on the device and in the oracle; every word compared."""
    ctx, P, K = env.ctx, env.P, len(env.protos)
    vals = env.values(batch)
    h_ct = env.cts(vals, level_ct, scale)
    ct = ctx.to_device(h_ct)
    crp = env.protos[0].SampleCRP(4, env.crs, batch)
    h_crp = env.host(crp)
    perm = env.rng.integers(0, env.n, env.n)
    if transform_spec is None:
        transform, o_transform = None, None
    else:
        dec, encd = transform_spec
        transform = env.lb.mpbgv.MaskedTransformFunc(dec, _perm_func(perm), encd)
        o_transform = (dec, lambda c: [c[j] for j in perm], encd)
    shares, o_e2s, o_s2e = [], [], []
    for i, p in enumerate(env.protos):
        e0 = env.party[i].Gaussian(p.e2s.cks.sigma, p.e2s.cks.bound, batch)
        e1 = env.party[i].Gaussian(p.s2e.cks.sigma, p.s2e.cks.bound, batch)
        mask = p.e2s.SampleMask(batch)
        sh = p.GenShare(env.d_sk[i], env.d_sk[i], ct, crp, transform, scale, level_e2s, e_e2s=e0, e_s2e=e1, mask=mask)
        he0, he1, hm = env.host(e0), env.host(e1), env.host(mask)
        for b in range(batch):
            we, ws = P.transform_share(level_e2s, env.sk[i], env.sk[i], h_ct[b], h_crp[b], o_transform, scale, he0[b], he1[b], hm[b])
            assert np.array_equal(env.host(sh.EncToShareShare)[b], we), "E2S share, party %d entry %d" % (i, b)
            assert np.array_equal(env.host(sh.ShareToEncShare)[b], ws), "S2E share, party %d entry %d" % (i, b)
            o_e2s.append((i, b, we))
            o_s2e.append((i, b, ws))
        shares.append(sh)
    agg = env.protos[0].AggregateShares(shares)
    lvl = min(level_ct, level_e2s)
    out = env.protos[0].Transform(ct, transform, crp, agg, scale)
    h_out = env.host(out)
    assert h_out.shape == (batch, 2, 5, env.N)
    for b in range(batch):
        ae = M.aggregate([w for (_, bb, w) in o_e2s if bb == b], QI[: lvl + 1])
        as_ = M.aggregate([w for (_, bb, w) in o_s2e if bb == b], QI)
        assert np.array_equal(env.host(agg.EncToShareShare)[b], ae)
        assert np.array_equal(env.host(agg.ShareToEncShare)[b], as_)
        want = P.transform(h_ct[b], o_transform, h_crp[b], ae, as_, scale)
        assert np.array_equal(h_out[b], want), "output ciphertext, entry %d" % b
        got = P.decrypt(env.ideal, h_out[b], scale)
        if transform_spec is None:
            assert got == vals[b]
        elif transform_spec == (True, True):
            assert got == [vals[b][j] for j in perm]
    return out


@pytest.mark.parametrize("env", CASES, indirect=True, ids=_ids)
@pytest.mark.parametrize("level_ct,level_e2s,batch", [(4, 4, 1), (4, 0, 3), (3, 1, 1), (4, 2, 3)])
def test_refresh_matches_the_oracle_and_decrypts(env, level_ct, level_e2s, batch):
    _run(env, level_ct, level_e2s, batch, None)


@pytest.mark.parametrize("env", [c for c in CASES if c[1] == 2], indirect=True, ids=_ids)
@pytest.mark.parametrize("spec", [(True, True), (True, False), (False, True), (False, False)], ids=lambda s: "dec%d-enc%d" % s)
@pytest.mark.parametrize("level_e2s", [0, 3])
def test_masked_transform_matches_the_oracle(env, spec, level_e2s):
    _run(env, 4, level_e2s, 2, spec)


@pytest.mark.parametrize("env", CASES, indirect=True, ids=_ids)
@pytest.mark.parametrize("level_e2s", [0, 2, 4])
def test_enc_to_share_and_back_match_the_oracle(env, level_e2s):
    """E2S with the secret shares left with the parties, GetShare by party 0, the shares recombining to the slots, then S2E of them."""
    ctx, P, K, batch, scale = env.ctx, env.P, len(env.protos), 2, 3
    vals = env.values(batch)
    h_ct = env.cts(vals, 4, scale)
    ct = ctx.to_device(h_ct)
    secrets, publics, e_h, m_h = [], [], [], []
    for i, p in enumerate(env.protos):
        e = env.party[i].Gaussian(p.e2s.cks.sigma, p.e2s.cks.bound, batch)
        m, pub = p.e2s.GenShare(env.d_sk[i], ct, level_e2s, e=e)
        secrets.append(m)
        publics.append(pub)
        e_h.append(env.host(e))
        m_h.append(env.host(m))
    agg = env.protos[0].e2s.AggregateShares(publics)
    own = env.protos[0].e2s.GetShare(secrets[0], agg, ct)
    h_own = env.host(own)
    for b in range(batch):
        pubs = [P.e2s_share(level_e2s, env.sk[i], h_ct[b][1], e_h[i][b], m_h[i][b]) for i in range(K)]
        for i in range(K):
            assert np.array_equal(env.host(publics[i])[b], pubs[i])
        a = M.aggregate(pubs, QI[: level_e2s + 1])
        assert np.array_equal(env.host(agg)[b], a)
        assert np.array_equal(h_own[b], P.e2s_get_share(level_e2s, h_ct[b][0], a, m_h[0][b]))
        rec = np.array(h_own[b], dtype=U64).reshape(1, -1)
        for i in range(1, K):
            P.enc.ringT.Add(rec, m_h[i][b].reshape(1, -1), rec)
        assert [int(v) for v in P.decode_ring_t(rec[0], scale)] == vals[b]
    # GetShare without a secret share: the masked decryption alone
    bare = env.host(env.protos[0].e2s.GetShare(None, agg, ct))
    assert np.array_equal(bare[0], P.e2s_get_share(level_e2s, h_ct[0][0], env.host(agg)[0]))
    # S2E of the secret shares at level 3
    crp = env.protos[0].s2e.SampleCRP(3, env.crs, batch)
    mine = [own] + secrets[1:]
    s2e = []
    for i, p in enumerate(env.protos):
        e = env.party[i].Gaussian(p.s2e.cks.sigma, p.s2e.cks.bound, batch)
        s2e.append(p.s2e.GenShare(env.d_sk[i], crp, mine[i], e=e))
        for b in range(batch):
            want = P.s2e_share(3, env.sk[i], env.host(crp)[b], env.host(e)[b], env.host(mine[i])[b])
            assert np.array_equal(env.host(s2e[i])[b], want)
    out = env.protos[0].s2e.GetEncryption(env.protos[0].s2e.AggregateShares(s2e), crp)
    for b in range(batch):
        assert P.decrypt(env.ideal, env.host(out)[b], scale) == vals[b]


@pytest.mark.parametrize("t", [0x101, 0xffc001])
def test_mask_sampler_and_ring_t_codecs_match_the_oracle(t):
    import torch
    import lattigo_b200 as lb
    ctx = lb.Context(10, QI, PJ)
    enc = lb.BGVEncoder(ctx, t)
    try:
        P = R.MPBGV(O.Parameters(10, QI, PJ), t)
        S = lb.encryptor.Samplers(ctx, 0x5EED)
        p = lb.mpbgv.EncToShareProtocol(enc, S, SIGMA)
        m = ctx.to_host(p.SampleMask(3))
        assert np.array_equal(m, R.sample_mask(0x5EED, 1, t, enc.n, 3))
        # DecodeRingT of arbitrary 64-bit words, EncodeRingT of arbitrary words
        rng = np.random.default_rng(t)
        w = rng.integers(0, (1 << 64) - 1, (3, enc.n), dtype=U64, endpoint=True)
        w[0, :4] = [0, t, 3 * t - 1, (1 << 64) - 1]
        d = torch.from_numpy(w.view(np.int64)).cuda()
        got_dec = ctx.to_host(lb.mpbgv.DecodeRingT(enc, d, 7))
        got_enc = ctx.to_host(lb.mpbgv.EncodeRingT(enc, d, 7))
        for b in range(3):
            assert np.array_equal(got_dec[b], P.decode_ring_t(w[b], 7))
            assert np.array_equal(got_enc[b], P.encode_ring_t(w[b], 7))
    finally:
        enc.close()
        ctx.close()

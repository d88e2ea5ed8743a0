"""Threshold protocols on the device (csrc/multiparty.cu, lattigo_b200/multiparty.py) bit for bit against tests/multiparty_oracle.py on
the same sampled polynomials, on the reference's test set (multiparty/test_params.go) and a ring without P, with 1, 2 and 5 parties;
lgpu_mp_aggregate's fold, chunking and alignment paths; PN16QP1761-sized shares; and end-to-end decryption of what the protocols
produce (collective public key -> Encryptor.EncryptZeroPk, collective key switching of a batch)."""
import math

import numpy as np
import pytest

from oracle import encryptor as E
from oracle import oracle as O
from tests import helpers as H
from tests import multiparty_oracle as M

pytestmark = pytest.mark.gpu
U64 = np.uint64
QI = [0x200000440001, 0x7fff80001, 0x800280001, 0x7ffd80001, 0x7ffc80001]
PJ = [0x3ffffffb80001, 0x4000000800001]
PARAMS = {"one_p": (QI, PJ[:1]), "two_p": (QI, PJ), "no_p": (QI, [])}
SIGMA = 3.2


class _Env:
    def __init__(self, name, K, seed):
        import lattigo_b200 as lb
        q, p = PARAMS[name]
        self.q, self.p = q, p
        self.params = O.Parameters(10, q, p)
        self.N = self.params.N()
        self.ctx = lb.Context(10, q, p)
        self.rng = np.random.default_rng(seed)
        self.crs = lb.encryptor.Samplers(self.ctx, 0xC0FFEE)
        self.party = [lb.encryptor.Samplers(self.ctx, 1000 + i) for i in range(K)]
        self.s = [self.ctx.to_host(self.party[i].Ternary(P=2 / 3))[0] for i in range(K)]
        self.sk = [M.sk_rows(self.params, si) for si in self.s]
        self.d_sk = [self.ctx.to_device(x) for x in self.sk]
        self.ideal = M.sk_rows(self.params, sum(self.s))
        self.oracle = M.Protocols(self.params)

    def fresh_ct(self, sk, level, batch):
        cts = []
        for _ in range(batch):
            a = H.rand_poly(self.q[: level + 1], self.N, self.rng)
            e = np.rint(self.rng.normal(0, SIGMA, self.N)).astype(np.int64)
            cts.append(np.stack([E.Encryptor(self.params).encryptZeroSkFromC1QP(level, -1, sk, a, e, True, False), a]))
        return np.stack(cts)


@pytest.fixture
def env(request):
    e = _Env(*request.param)
    yield e
    e.ctx.close()


CASES = [(n, K, 10 * K + i) for i, n in enumerate(PARAMS) for K in (1, 2, 5)]


@pytest.mark.parametrize("env", CASES, indirect=True, ids=lambda c: "%s-K%d" % c[:2])
def test_collective_public_key_matches_the_oracle_and_encrypts(env):
    import lattigo_b200 as lb
    ctx, K = env.ctx, len(env.s)
    protos = [lb.multiparty.PublicKeyGenProtocol(ctx, env.party[i]) for i in range(K)]
    crp = protos[0].SampleCRP(env.crs)
    es = [env.party[i].Gaussian(SIGMA, 6 * SIGMA) for i in range(K)]
    shares = [protos[i].GenShare(env.d_sk[i], crp, e=es[i]) for i in range(K)]
    h_crp = ctx.to_host(crp)
    want = [env.oracle.ckg_share(env.sk[i], h_crp, ctx.to_host(es[i])[0]) for i in range(K)]
    for i in range(K):
        assert np.array_equal(ctx.to_host(shares[i]), want[i])
    moduli = env.q + env.p
    agg = protos[0].AggregateShares(shares)
    assert np.array_equal(ctx.to_host(agg), M.aggregate(want, moduli))
    pk = protos[0].GenPublicKey(agg, crp)
    # the collective key feeds the existing public-key encryptor; the result decrypts under the ideal secret sum
    level, batch = 3, 2
    S = env.party[0]
    ct = lb.encryptor.Encryptor(ctx).EncryptZeroPk(level, pk, S.Ternary(P=2 / 3, batch=batch), S.Gaussian(batch=batch), S.Gaussian(batch=batch))
    h = ctx.to_host(ct)
    for b in range(batch):
        noise = M.decrypt_noise(env.params, [h[b, 0], h[b, 1]], env.ideal)
        assert M.log2_std(noise) < 16         # u e_pk + e0 + e1 s: about 2^11 at N = 2^10 and 5 parties


@pytest.mark.parametrize("env", CASES, indirect=True, ids=lambda c: "%s-K%d" % c[:2])
@pytest.mark.parametrize("sigma_flood", [8 * SIGMA, 2.0 ** 30])
def test_key_switch_matches_the_oracle_and_decrypts(env, sigma_flood):
    import lattigo_b200 as lb
    ctx, K = env.ctx, len(env.s)
    s_out = [ctx.to_host(env.party[i].Ternary(P=2 / 3))[0] for i in range(K)]
    sk_out = [M.sk_rows(env.params, x) for x in s_out]
    ideal_out = M.sk_rows(env.params, sum(s_out))
    protos = [lb.multiparty.KeySwitchProtocol(ctx, env.party[i], sigma_flood) for i in range(K)]
    for level, batch in ((4, 1), (4, 3), (2, 3)):
        ct = env.fresh_ct(env.ideal, level, batch)
        d_ct = ctx.to_device(ct)
        es = [env.party[i].Gaussian(protos[i].sigma, protos[i].bound, batch) for i in range(K)]
        shares = [protos[i].GenShare(env.d_sk[i], ctx.to_device(sk_out[i]), d_ct, e=es[i]) for i in range(K)]
        agg = protos[0].AggregateShares(shares)
        out = ctx.to_host(protos[0].KeySwitch(d_ct, agg))
        for b in range(batch):
            want = [env.oracle.cks_share(level, env.sk[i], sk_out[i], ct[b, 1], ctx.to_host(es[i])[b]) for i in range(K)]
            for i in range(K):
                assert np.array_equal(ctx.to_host(shares[i])[b], want[i]), (level, batch, b, i)
            w_agg = M.aggregate(want, env.q[: level + 1])
            assert np.array_equal(ctx.to_host(agg)[b], w_agg)
            w_out = env.oracle.cks_key_switch([ct[b, 0], ct[b, 1]], w_agg)
            assert np.array_equal(out[b, 0], w_out[0]) and np.array_equal(out[b, 1], w_out[1])
            noise = M.decrypt_noise(env.params, w_out, ideal_out)
            assert M.log2_std(noise) <= math.log2(M.noise_key_switch(K, SIGMA, sigma_flood)) + 1


@pytest.mark.parametrize("env", CASES, indirect=True, ids=lambda c: "%s-K%d" % c[:2])
@pytest.mark.parametrize("sigma_flood", [8 * SIGMA, 2.0 ** 30])
def test_public_key_switch_matches_the_oracle_and_decrypts(env, sigma_flood):
    import lattigo_b200 as lb
    ctx, K, N = env.ctx, len(env.s), env.N
    s_out = env.rng.integers(-1, 2, N)
    sk_out = M.sk_rows(env.params, s_out)
    a = H.rand_poly(env.q + env.p, N, env.rng)
    pk = np.stack([E.Encryptor(env.params).encryptZeroSkFromC1QP(len(env.q) - 1, len(env.p) - 1, sk_out, a.copy(),
                                                                 np.rint(env.rng.normal(0, SIGMA, N)).astype(np.int64), True, True), a])
    d_pk = ctx.to_device(pk)
    protos = [lb.multiparty.PublicKeySwitchProtocol(ctx, env.party[i], sigma_flood) for i in range(K)]
    for level, batch in ((4, 1), (4, 3), (2, 3)):
        ct = env.fresh_ct(env.ideal, level, batch)
        d_ct = ctx.to_device(ct)
        smp = []
        for i in range(K):
            S = env.party[i]
            smp.append((S.Ternary(P=2 / 3, batch=batch), S.Gaussian(batch=batch), S.Gaussian(batch=batch),
                        S.Gaussian(sigma_flood, 6 * sigma_flood, batch)))
        shares = [protos[i].GenShare(env.d_sk[i], d_pk, d_ct, *smp[i]) for i in range(K)]
        agg = protos[0].AggregateShares(shares)
        out = ctx.to_host(protos[0].KeySwitch(d_ct, agg))
        for b in range(batch):
            want = []
            for i in range(K):
                u, e0, e1, ef = [ctx.to_host(x)[b] for x in smp[i]]
                want.append(np.stack(env.oracle.pcks_share(level, env.sk[i], pk, ct[b, 1], u, e0, e1, ef)))
                assert np.array_equal(ctx.to_host(shares[i])[b], want[i]), (level, batch, b, i)
            w_agg = M.aggregate(want, env.q[: level + 1])
            assert np.array_equal(ctx.to_host(agg)[b], w_agg)
            w_out = env.oracle.pcks_key_switch([ct[b, 0], ct[b, 1]], w_agg)
            assert np.array_equal(out[b, 0], w_out[0]) and np.array_equal(out[b, 1], w_out[1])
            noise = M.decrypt_noise(env.params, w_out, sk_out)
            assert M.log2_std(noise) <= math.log2(M.noise_public_key_switch(N, bool(env.p), K, SIGMA, sigma_flood)) + 1


def _agg_ctx(q, p, logN=10):
    import lattigo_b200 as lb
    return lb.Context(logN, q, p)


@pytest.mark.parametrize("K", [1, 2, 5, 17, 32, 33, 64])
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("in_place", [False, True])
def test_aggregate_fold_chunks_and_alignment(K, aligned, in_place):
    import torch
    import lattigo_b200 as lb
    q, p = QI, PJ
    ctx = _agg_ctx(q, p)
    try:
        rng = np.random.default_rng(K)
        levelQ, levelP, n_polys, N = 3, 1, 3, ctx.N
        mods = q[: levelQ + 1] + p[: levelP + 1]
        rows = len(mods)
        host = [np.stack([np.stack([rng.integers(0, 2 * m, N, dtype=U64) for m in mods]) for _ in range(n_polys)]) for _ in range(K)]
        size = n_polys * rows * N
        off = 0 if aligned else 1
        pool = torch.zeros(((K + 1) * (size + 2),), dtype=torch.int64, device="cuda")
        views = [pool[k * (size + 2) + off: k * (size + 2) + off + size].view(n_polys, rows, N) for k in range(K + 1)]
        for k in range(K):
            views[k].copy_(ctx.to_device(host[k]))
        out = views[0] if in_place else views[K]
        chunks = 0 if (K == 1 and in_place) else 1 + max(0, -(-(K - 32) // 31))
        got = {}
        n = H.launch_delta(lambda: got.setdefault("r", lb.multiparty.aggregate(ctx, levelQ, levelP, views[:K], out=out)))
        assert n == chunks
        assert np.array_equal(ctx.to_host(out), M.aggregate(host, mods))
    finally:
        ctx.close()


def test_aggregate_wraps_like_go_uint64_on_61_bit_primes():
    import lattigo_b200 as lb
    q, _ = O.gen_moduli(11, [61, 61], [])
    ctx = _agg_ctx(q, [])
    try:
        K, N = 17, ctx.N
        host = [np.stack([np.full(N, 2 * m - 1, dtype=U64) for m in q])[None] for _ in range(K)]
        shares = [ctx.to_device(h) for h in host]
        got = ctx.to_host(lb.multiparty.aggregate(ctx, 1, -1, shares))
        want = M.aggregate(host, q)
        assert np.array_equal(got, want)
    finally:
        ctx.close()


def test_pn16_shares_aggregate_and_key_switch():
    """PN16QP1761: four shares of the size of a relinearization-key round-one share (beta = 9 gadget entries x 2 components of 38 rows)
    aggregated in one launch, and one KeySwitch share batch at level 33."""
    import lattigo_b200 as lb
    from lattigo_b200.params import PRESETS
    pr = PRESETS["CKKS_PN16QP1761"]
    q, p = pr["Q"], pr["P"]
    ctx = lb.Context(16, q, p)
    try:
        crs = lb.encryptor.Samplers(ctx, 7)
        lq, lp = len(q) - 1, len(p) - 1
        shares = [crs.UniformQP(lq, lp, batch=18) for _ in range(4)]
        out = {}
        assert H.launch_delta(lambda: out.setdefault("r", lb.multiparty.aggregate(ctx, lq, lp, shares))) == 1
        want = M.aggregate([ctx.to_host(s) for s in shares], q + p)
        assert np.array_equal(ctx.to_host(out["r"]), want)
        del shares, out
        params = O.Parameters(16, q, p)
        level, batch, N = 33, 2, ctx.N
        rng = np.random.default_rng(3)
        sks = [M.sk_rows(params, rng.integers(-1, 2, N)) for _ in range(2)]
        ct = np.stack([np.stack([H.rand_poly(q, N, rng), H.rand_poly(q, N, rng)]) for _ in range(batch)])
        proto = lb.multiparty.KeySwitchProtocol(ctx, lb.encryptor.Samplers(ctx, 9), 8 * SIGMA)
        e = proto.samplers.Gaussian(proto.sigma, proto.bound, batch)
        share = ctx.to_host(proto.GenShare(ctx.to_device(sks[0]), ctx.to_device(sks[1]), ctx.to_device(ct), e=e))
        orc = M.Protocols(params)
        for b in range(batch):
            assert np.array_equal(share[b], orc.cks_share(level, sks[0], sks[1], ct[b, 1], ctx.to_host(e)[b]))
    finally:
        ctx.close()


PW2 = {"one_p": 16, "two_p": 0, "no_p": 16}      # multiparty/test_params.go: BaseTwoDecomposition 16 with one P, 0 with two


def _valid(kg):
    return [(i, j) for i in range(kg.nd) for j in range(kg.sizes[i])]


@pytest.mark.parametrize("env", CASES, indirect=True, ids=lambda c: "%s-K%d" % c[:2])
def test_evaluation_and_galois_key_shares_match_the_oracle(env):
    import lattigo_b200 as lb
    ctx, K = env.ctx, len(env.s)
    name = [n for n in PARAMS if PARAMS[n] == (env.q, env.p)][0]
    pw2 = PW2[name]
    kg = M.KeyGen(env.params, pw2)
    # EVKG from s_i to t_i
    t = [ctx.to_host(env.party[i].Ternary(P=2 / 3))[0] for i in range(K)]
    tk = [M.sk_rows(env.params, x) for x in t]
    protos = [lb.multiparty.EvaluationKeyGenProtocol(ctx, env.party[i], pw2) for i in range(K)]
    crp = protos[0].SampleCRP(env.crs)
    es = [protos[i]._gauss((kg.nd, max(kg.sizes))) for i in range(K)]
    shares = [protos[i].GenShare(env.d_sk[i], ctx.to_device(tk[i]), crp, e=es[i]) for i in range(K)]
    h_crp = ctx.to_host(crp)
    want = [kg.evkg_share(env.sk[i], tk[i], h_crp, ctx.to_host(es[i])) for i in range(K)]
    for i in range(K):
        got = ctx.to_host(shares[i])
        for (a, b) in _valid(kg):
            assert np.array_equal(got[a, b], want[i][a, b]), (i, a, b)
    agg = ctx.to_host(protos[0].AggregateShares(shares))
    w_agg = M.aggregate(want, env.q + env.p)
    for (a, b) in _valid(kg):
        assert np.array_equal(agg[a, b], w_agg[a, b])
    # GKG over several Galois elements, the conjugation 2N - 1 included
    N = env.N
    gal_els = [env.params.GaloisElement(1), env.params.GaloisElement(5), 2 * N - 1]
    gprotos = [lb.multiparty.GaloisKeyGenProtocol(ctx, env.party[i], pw2) for i in range(K)]
    gcrp = gprotos[0].SampleCRP(env.crs, len(gal_els))
    ges = [gprotos[i]._gauss((len(gal_els), kg.nd, max(kg.sizes))) for i in range(K)]
    gshares = [gprotos[i].GenShare(env.d_sk[i], gal_els, gcrp, e=ges[i]) for i in range(K)]
    h_gcrp = ctx.to_host(gcrp)
    for i in range(K):
        got = ctx.to_host(gshares[i])
        for k, g in enumerate(gal_els):
            w = kg.gkg_share(env.sk[i], g, h_gcrp[k], ctx.to_host(ges[i])[k])
            for (a, b) in _valid(kg):
                assert np.array_equal(got[k, a, b], w[a, b]), (i, g, a, b)
    if name == "two_p":
        # a collective Galois key drives Evaluator.Automorphism: the result decrypts under the ideal secret with small noise
        gagg = gprotos[0].AggregateShares(gshares)
        keys = gprotos[0].GenGaloisKeys(gal_els, gagg, gcrp)
        ev = lb.Evaluator(ctx)
        ct = env.fresh_ct(env.ideal, 4, 2)
        for g in gal_els:
            out = ctx.new_poly(5, 4).view(2, 2, 5, N)
            ev.Automorphism(ctx.to_device(ct), g, keys[g], out)
            h = ctx.to_host(out)
            for b in range(2):
                assert M.log2_std(M.decrypt_noise(env.params, [h[b, 0], h[b, 1]], env.ideal)) < 20


@pytest.mark.parametrize("env", CASES, indirect=True, ids=lambda c: "%s-K%d" % c[:2])
def test_relinearization_key_rounds_match_the_oracle(env):
    import lattigo_b200 as lb
    ctx, K = env.ctx, len(env.s)
    name = [n for n in PARAMS if PARAMS[n] == (env.q, env.p)][0]
    pw2 = PW2[name]
    kg = M.KeyGen(env.params, pw2)
    protos = [lb.multiparty.RelinearizationKeyGenProtocol(ctx, env.party[i], pw2) for i in range(K)]
    crp = protos[0].SampleCRP(env.crs)
    h_crp = ctx.to_host(crp)
    lead = (kg.nd, max(kg.sizes))
    smp = [(env.party[i].Ternary(P=2 / 3)[0], protos[i]._gauss(lead), protos[i]._gauss(lead)) for i in range(K)]
    r1 = [protos[i].GenShareRoundOne(env.d_sk[i], crp, *smp[i]) for i in range(K)]
    w1 = [kg.rkg_round_one(env.sk[i], h_crp, ctx.to_host(smp[i][0]), ctx.to_host(smp[i][1]), ctx.to_host(smp[i][2])) for i in range(K)]
    for i in range(K):
        assert np.array_equal(ctx.to_host(r1[i][0]), w1[i][0])
        got = ctx.to_host(r1[i][1])
        for (a, b) in _valid(kg):
            assert np.array_equal(got[a, b], w1[i][1][a, b]), (i, a, b)
    agg1 = protos[0].AggregateShares([x[1] for x in r1])
    w_agg1 = M.aggregate([w[1] for w in w1], env.q + env.p)
    h_agg1 = ctx.to_host(agg1)
    for (a, b) in _valid(kg):
        assert np.array_equal(h_agg1[a, b], w_agg1[a, b])
    e2 = [protos[i]._gauss(lead) for i in range(K)]
    r2 = [protos[i].GenShareRoundTwo(r1[i][0], env.d_sk[i], agg1, e2=e2[i]) for i in range(K)]
    w2 = [kg.rkg_round_two(w1[i][0], env.sk[i], h_agg1, ctx.to_host(e2[i])) for i in range(K)]
    for i in range(K):
        got = ctx.to_host(r2[i])
        for (a, b) in _valid(kg):
            assert np.array_equal(got[a, b], w2[i][a, b]), (i, a, b)
            assert all(int(got[a, b, r].max()) < 2 * m for r, m in enumerate(env.q + env.p))     # round two: [0, 2q)
    agg2 = protos[0].AggregateShares(r2)
    rlk = protos[0].GenRelinearizationKey(agg1, agg2)
    w_rlk = kg.gen_relinearization_key(h_agg1, M.aggregate(w2, env.q + env.p))
    h_rlk = ctx.to_host(rlk.data)
    for (a, b) in _valid(kg):
        assert np.array_equal(h_rlk[a, b], w_rlk[a, b])
    if name == "two_p":
        # a collective relinearization key drives CKKSEvaluator.MulRelinRescaleNew: the product of two encryptions of zero decrypts
        # under the ideal secret with small noise, bit for bit with the oracle's evaluator on the same key
        ct_a, ct_b = env.fresh_ct(env.ideal, 4, 2), env.fresh_ct(env.ideal, 4, 2)
        out = ctx.to_host(lb.CKKSEvaluator(ctx, rlk).MulRelinRescaleNew(ctx.to_device(ct_a), ctx.to_device(ct_b)))
        ev_o = O.CKKSEvaluator(env.params, O.GadgetCiphertext(h_rlk, len(env.q), len(env.p)))
        for b in range(2):
            r = ev_o.Rescale(ev_o.MulRelinNew([ct_a[b, 0], ct_a[b, 1]], [ct_b[b, 0], ct_b[b, 1]]))
            assert np.array_equal(out[b, 0], r[0]) and np.array_equal(out[b, 1], r[1])
            assert M.log2_std(M.decrypt_noise(env.params, [out[b, 0], out[b, 1]], env.ideal)) < 20


def test_key_generation_shares_at_pn16():
    """PN16QP1761: GKG for 4 Galois elements in one call, the conjugation included, bit for bit with the oracle on one key."""
    import lattigo_b200 as lb
    from lattigo_b200.params import PRESETS
    pr = PRESETS["CKKS_PN16QP1761"]
    q, p = pr["Q"], pr["P"]
    ctx = lb.Context(16, q, p)
    try:
        params = O.Parameters(16, q, p)
        rng = np.random.default_rng(5)
        sk = M.sk_rows(params, rng.integers(-1, 2, ctx.N))
        S = lb.encryptor.Samplers(ctx, 3)
        g = lb.multiparty.GaloisKeyGenProtocol(ctx, S)
        els = [params.GaloisElement(k) for k in (1, 2, 3)] + [2 * ctx.N - 1]
        crp = g.SampleCRP(S, len(els))
        e = g._gauss((len(els), g.nd, g.npw2))
        share = ctx.to_host(g.GenShare(ctx.to_device(sk), els, crp, e=e))
        kg = M.KeyGen(params, 0)
        w = kg.gkg_share(sk, els[3], ctx.to_host(crp)[3], ctx.to_host(e)[3])
        assert np.array_equal(share[3], w)
    finally:
        ctx.close()

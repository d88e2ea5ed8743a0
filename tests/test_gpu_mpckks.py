"""The mpckks protocols on the device (csrc/mp_refresh.cu, lattigo_b200/mpckks.py) word for word against tests/mp_refresh_oracle.py
(MPCKKS) on the same samples, on the reference's testInsecurePrec45 and testInsecurePrec90 sets (multiparty/mpckks/test_params.go; 4 and 8
share words) at K = 1, 2, 5: every E2S / S2E share, aggregate, big-integer secret share and refreshed ciphertext; full slots and
logSlots = LogN - 3; a ciphertext above the E2S level; an input scale equal to the default and a non-integer one; batch 1 and 3; the
mask sampler against its restated stream. End to end, the shares recombine to the centred decryption and the refreshed ciphertexts
decrypt under the ideal key to the input times defaultScale / inputScaleInt within the smudging bound."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests import mp_refresh_oracle as R
from tests import multiparty_oracle as M

pytestmark = pytest.mark.gpu
U64 = np.uint64
SETS = {
    "prec45": ([0x80000000080001, 0x2000000a0001, 0x2000000e0001, 0x2000001d0001, 0x1fffffcf0001, 0x1fffffc20001, 0x200000440001],
               [0x80000000130001, 0x7fffffffe90001], 45),
    "prec90": ([0x80000000080001, 0x80000000440001, 0x2000000a0001, 0x2000000e0001, 0x1fffffc20001, 0x200000440001, 0x200000500001,
                0x200000620001, 0x1fffff980001, 0x2000006a0001, 0x1fffff7e0001, 0x200000860001],
               [0xffffffffffc0001, 0x10000000006e0001], 90),
}
SIGMA = 3.2


class _Env:
    def __init__(self, name, K, seed):
        import lattigo_b200 as lb
        self.lb = lb
        q, p, self.log_scale = SETS[name]
        self.q = q
        self.params = O.Parameters(10, q, p)
        self.N = self.params.N()
        self.ctx = lb.Context(10, q, p)
        self.rng = np.random.default_rng(seed)
        self.crs = lb.encryptor.Samplers(self.ctx, 0xC0FFEE + seed)
        self.party = [lb.encryptor.Samplers(self.ctx, 2000 + 17 * seed + i) for i in range(K)]
        self.s = [self.ctx.to_host(self.party[i].Ternary(P=2 / 3))[0] for i in range(K)]
        self.sk = [M.sk_rows(self.params, si) for si in self.s]
        self.d_sk = [self.ctx.to_device(x) for x in self.sk]
        self.ideal = M.sk_rows(self.params, sum(self.s))
        self.P = R.MPCKKS(self.params)
        self.default = Fraction(2) ** self.log_scale
        self.protos = [lb.mpckks.RefreshProtocol(self.ctx, self.party[i], SIGMA, self.default) for i in range(K)]

    def cts(self, batch, level, log_slots):
        """Ciphertexts of random plaintexts of about the default scale's size, in Y = X^gap for sparse slots."""
        gap = self.N // (2 << log_slots)
        out, ms = [], []
        for _ in range(batch):
            m = [0] * self.N
            for j in range(0, self.N, gap):
                m[j] = int(self.rng.integers(-(1 << 40), 1 << 40)) << (self.log_scale - 41)
            a = H.rand_poly(self.q[: level + 1], self.N, self.rng)
            e = np.rint(self.rng.normal(0, SIGMA, self.N)).astype(np.int64)
            out.append(self.P.encrypt_coeffs(self.ideal, m, level, a, e))
            ms.append(m)
        return np.stack(out), ms

    def close(self):
        self.ctx.close()


@pytest.fixture
def env(request):
    e = _Env(*request.param)
    yield e
    e.close()


CASES = [(n, K, 5 * K + i) for i, n in enumerate(SETS) for K in (1, 2, 5)]
_ids = lambda c: "%s-K%d" % c[:2]


@pytest.mark.parametrize("env", CASES, indirect=True, ids=_ids)
@pytest.mark.parametrize("log_slots,batch,above,scale_kind", [(9, 1, 0, "default"), (7, 3, 1, "fraction"), (9, 3, 2, "fraction"), (7, 1, 1, "default")])
def test_refresh_matches_the_oracle_and_decrypts(env, log_slots, batch, above, scale_kind):
    import lattigo_b200 as lb
    ctx, P, K = env.ctx, env.P, len(env.protos)
    min_level, log_bound, ok = lb.mpckks.GetMinimumLevelForRefresh(128, float(env.default), K, env.q)
    assert ok
    level_ct = min(min_level + above, len(env.q) - 1)
    scale = env.default if scale_kind == "default" else env.default * Fraction(5, 3)
    d, s = env.protos[0].defaultScale, lb.mpckks.input_scale_int(scale)
    dslots = 2 << log_slots
    h_ct, ms = env.cts(batch, level_ct, log_slots)
    ct = ctx.to_device(h_ct)
    max_level = len(env.q) - 1
    crp = env.protos[0].SampleCRP(max_level, env.crs, batch)
    h_crp = ctx.to_host(crp)
    shares, masks, o_e2s, o_s2e = [], [], [], []
    for i, p in enumerate(env.protos):
        e0 = env.party[i].Gaussian(p.e2s.cks.sigma, p.e2s.cks.bound, batch)
        e1 = env.party[i].Gaussian(p.s2e.cks.sigma, p.s2e.cks.bound, batch)
        sh = p.GenShare(env.d_sk[i], log_bound, ct, crp, scale, log_slots, level=min_level, e_e2s=e0, e_s2e=e1)
        shares.append(sh)
        he0, he1 = ctx.to_host(e0), ctx.to_host(e1)
        # the mask each party drew: its stream restated (the last stream id GenShare took)
        mask = R.sample_big_mask(p.e2s.samplers.seed, p.e2s.samplers._next, log_bound, dslots, batch)
        masks.append(mask)
        for b in range(batch):
            we = P.e2s_share(min_level, env.sk[i], h_ct[b][1], he0[b], mask[b])
            ws = P.s2e_share(max_level, env.sk[i], h_crp[b], he1[b], P.scale(mask[b], d, s))
            assert np.array_equal(ctx.to_host(sh.EncToShareShare)[b], we), "E2S share, party %d entry %d" % (i, b)
            assert np.array_equal(ctx.to_host(sh.ShareToEncShare)[b], ws), "S2E share, party %d entry %d" % (i, b)
        o_e2s.append([P.e2s_share(min_level, env.sk[i], h_ct[b][1], he0[b], mask[b]) for b in range(batch)])
        o_s2e.append([P.s2e_share(max_level, env.sk[i], h_crp[b], he1[b], P.scale(mask[b], d, s)) for b in range(batch)])
    agg = env.protos[0].AggregateShares(shares)
    out = env.protos[0].Finalize(ct, crp, agg, scale, log_slots)
    h_out = ctx.to_host(out)
    bound = (K + 1) * (6 * 4.6 + 2) * 8 + 64
    for b in range(batch):
        ae = M.aggregate([o_e2s[i][b] for i in range(K)], env.q[: min_level + 1])
        as_ = M.aggregate([o_s2e[i][b] for i in range(K)], env.q)
        assert np.array_equal(ctx.to_host(agg.EncToShareShare)[b], ae)
        assert np.array_equal(ctx.to_host(agg.ShareToEncShare)[b], as_)
        want = P.finalize(min_level, h_ct[b], ae, as_, h_crp[b], dslots, d, s)
        assert np.array_equal(h_out[b], want), "refreshed ciphertext, entry %d" % b
        dec = P.decrypt_coeffs(env.ideal, h_out[b])
        gap = env.N // dslots
        err = max(abs(dec[j] - R.quo(ms[b][j] * d, s)) for j in range(env.N) if j % gap == 0)
        assert err <= bound, (err, bound)


@pytest.mark.parametrize("env", CASES, indirect=True, ids=_ids)
@pytest.mark.parametrize("log_slots", [9, 7])
def test_enc_to_share_and_back_match_the_oracle(env, log_slots):
    import lattigo_b200 as lb
    ctx, P, K, batch = env.ctx, env.P, len(env.protos), 2
    min_level, log_bound, ok = lb.mpckks.GetMinimumLevelForRefresh(128, float(env.default), K, env.q)
    dslots = 2 << log_slots
    h_ct, ms = env.cts(batch, len(env.q) - 1, log_slots)
    ct = ctx.to_device(h_ct)
    secrets, publics = [], []
    for i, p in enumerate(env.protos):
        e = env.party[i].Gaussian(p.e2s.cks.sigma, p.e2s.cks.bound, batch)
        m, pub = p.e2s.GenShare(env.d_sk[i], log_bound, ct, log_slots, min_level, e=e)
        mask = lb.mpckks.to_ints(m)
        assert mask == R.sample_big_mask(p.e2s.samplers.seed, p.e2s.samplers._next, log_bound, dslots, batch)
        assert all(-(1 << (log_bound - 1)) <= v < (1 << (log_bound - 1)) for row in mask for v in row)
        for b in range(batch):
            assert np.array_equal(ctx.to_host(pub)[b], P.e2s_share(min_level, env.sk[i], h_ct[b][1], ctx.to_host(e)[b], mask[b]))
        secrets.append(m)
        publics.append(pub)
    agg = env.protos[0].e2s.AggregateShares(publics)
    own = env.protos[0].e2s.GetShare(secrets[0], agg, ct, log_slots)
    bare = env.protos[0].e2s.GetShare(None, agg, ct, log_slots)
    h_agg = ctx.to_host(agg)
    for b in range(batch):
        mine = lb.mpckks.to_ints(secrets[0])[b]
        assert lb.mpckks.to_ints(own)[b] == P.get_share(min_level, h_ct[b][0], h_agg[b], dslots, mine)
        assert lb.mpckks.to_ints(bare)[b] == P.get_share(min_level, h_ct[b][0], h_agg[b], dslots)
    # the parties' shares sum to the message up to the smudging noise
    rec = lb.mpckks.to_ints(lb.mpckks.sum_shares([own] + secrets[1:]))
    gap = env.N // dslots
    for b in range(batch):
        err = max(abs(rec[b][i] - ms[b][i * gap]) for i in range(dslots))
        assert err <= K * 6 * 4.6 + 6 * SIGMA + 1
    # S2E of the shares at the maximum level, and its decryption
    max_level = len(env.q) - 1
    crp = env.protos[0].s2e.SampleCRP(max_level, env.crs, batch)
    mine = [own] + secrets[1:]
    s2e = []
    for i, p in enumerate(env.protos):
        e = env.party[i].Gaussian(p.s2e.cks.sigma, p.s2e.cks.bound, batch)
        s2e.append(p.s2e.GenShare(env.d_sk[i], crp, log_slots, mine[i], e=e))
        for b in range(batch):
            want = P.s2e_share(max_level, env.sk[i], ctx.to_host(crp)[b], ctx.to_host(e)[b], lb.mpckks.to_ints(mine[i])[b])
            assert np.array_equal(ctx.to_host(s2e[i])[b], want)
    out = ctx.to_host(env.protos[0].s2e.GetEncryption(env.protos[0].s2e.AggregateShares(s2e), crp))
    for b in range(batch):
        dec = P.decrypt_coeffs(env.ideal, out[b])
        assert max(abs(dec[i * gap] - ms[b][i * gap]) for i in range(dslots)) <= 2 * K * 6 * 4.6 + 6 * SIGMA + 1

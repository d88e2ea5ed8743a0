"""Anchors tests/mp_refresh_oracle.py by decryption, on the reference's mpbgv test set (multiparty/mpbgv/test_parameters.go,
testInsecure) with t = 0x101 (n = 128, gap 8) and t = 0xffc001 (n = N, gap 1): the E2S shares of K parties recombine to the message,
S2E of those shares encrypts it again, a refresh gives a fresh ciphertext at the maximum level that decrypts to the input, and the masked
permutation of the reference's testRefreshAndPermutation decrypts to the permuted slots. All exactly."""
import numpy as np
import pytest

from oracle import encryptor as E
from oracle import oracle as O
from tests import helpers as H
from tests import mp_refresh_oracle as R
from tests import multiparty_oracle as M

QI = [0x3fffffa8001, 0x1000090001, 0x10000c8001, 0x10000f0001, 0xffff00001]
PJ = [0x7fffffd8001]
SIGMA = 3.2
SIGMA_SMUDGE = (SIGMA ** 2 + SIGMA ** 2) ** 0.5      # KeySwitchProtocol with noiseFlooding = Xe


class _Env:
    def __init__(self, t, K, seed):
        self.params = O.Parameters(10, QI, PJ)
        self.N = self.params.N()
        self.rng = np.random.default_rng(seed)
        self.P = R.MPBGV(self.params, t)
        self.t, self.n = t, self.P.n
        self.s = [self.rng.integers(-1, 2, self.N) for _ in range(K)]
        self.sk = [M.sk_rows(self.params, si) for si in self.s]
        self.ideal = M.sk_rows(self.params, sum(self.s))

    def e(self):
        return np.clip(np.rint(self.rng.normal(0, SIGMA_SMUDGE, self.N)), -6 * SIGMA_SMUDGE, 6 * SIGMA_SMUDGE).astype(np.int64)

    def mask(self):
        return self.rng.integers(0, self.t, self.n).astype(np.uint64)

    def crp(self, level):
        return H.rand_poly(QI[: level + 1], self.N, self.rng)

    def ct(self, values, level, scale):
        a = H.rand_poly(QI[: level + 1], self.N, self.rng)
        e = np.rint(self.rng.normal(0, SIGMA, self.N)).astype(np.int64)
        return self.P.encrypt(self.ideal, values, level, scale, a, e)

    def values(self):
        return [int(v) for v in self.rng.integers(0, self.t, self.n)]


CASES = [(t, K) for t in (0x101, 0xffc001) for K in (1, 3)]


@pytest.mark.parametrize("t,K", CASES)
@pytest.mark.parametrize("level_e2s", [0, 2])
def test_e2s_shares_recombine_and_s2e_reencrypts(t, K, level_e2s):
    env = _Env(t, K, 7 * K + level_e2s)
    P, scale = env.P, 3
    vals = env.values()
    ct = env.ct(vals, 4, scale)
    masks = [env.mask() for _ in range(K)]
    shares = [P.e2s_share(level_e2s, env.sk[i], ct[1], env.e(), masks[i]) for i in range(K)]
    agg = M.aggregate(shares, QI[: level_e2s + 1])
    # party 0 recovers its own share plus the masked decryption; the others keep their masks
    rec = np.array(P.e2s_get_share(level_e2s, ct[0], agg, masks[0]), dtype=np.uint64)
    for i in range(1, K):
        P.enc.ringT.Add(rec.reshape(1, -1), masks[i].reshape(1, -1), rec.reshape(1, -1))
    assert [int(v) for v in P.decode_ring_t(rec, scale)] == vals
    # and back: S2E of the secret shares at the maximum level
    secrets = [np.array(P.e2s_get_share(level_e2s, ct[0], agg, masks[0]), dtype=np.uint64)] + masks[1:]
    crp = env.crp(4)
    s2e = M.aggregate([P.s2e_share(4, env.sk[i], crp, env.e(), secrets[i]) for i in range(K)], QI)
    out = np.stack([s2e, crp])
    assert P.decrypt(env.ideal, out, scale) == vals


@pytest.mark.parametrize("t,K", CASES)
@pytest.mark.parametrize("level_ct,level_e2s", [(4, 4), (3, 0), (4, 1)])
def test_refresh_decrypts_to_the_input_at_the_maximum_level(t, K, level_ct, level_e2s):
    env = _Env(t, K, 100 + 7 * K + level_e2s)
    P, scale = env.P, 5
    vals = env.values()
    ct = env.ct(vals, level_ct, scale)
    crp = env.crp(4)
    parts = [P.transform_share(level_e2s, env.sk[i], env.sk[i], ct, crp, None, scale, env.e(), env.e(), env.mask()) for i in range(K)]
    agg_e2s = M.aggregate([p[0] for p in parts], QI[: min(level_ct, level_e2s) + 1])
    agg_s2e = M.aggregate([p[1] for p in parts], QI)
    out = P.transform(ct, None, crp, agg_e2s, agg_s2e, scale)
    assert out.shape == (2, 5, env.N)
    assert P.decrypt(env.ideal, out, scale) == vals


@pytest.mark.parametrize("t,K", CASES)
def test_masked_permutation_decrypts_to_the_permuted_slots(t, K):
    env = _Env(t, K, 300 + K)
    P, scale = env.P, 2
    vals = [1] * env.n                                          # newTestVectors: every slot 1
    vals[: 17] = env.values()[: 17]
    perm = env.rng.integers(0, env.n, env.n)
    transform = (True, lambda c: [c[j] for j in perm], True)
    ct = env.ct(vals, 0, scale)
    crp = env.crp(4)
    parts = [P.transform_share(0, env.sk[i], env.sk[i], ct, crp, transform, scale, env.e(), env.e(), env.mask()) for i in range(K)]
    out = P.transform(ct, transform, crp, M.aggregate([p[0] for p in parts], QI[:1]), M.aggregate([p[1] for p in parts], QI), scale)
    assert P.decrypt(env.ideal, out, scale) == [vals[j] for j in perm]


def test_gap1_ring_q2t_words_reach_the_lazy_range():
    """RingQ2T at level > 0 with gap 1 returns ModUpExact's lazy word: some words are >= t, and they are congruent to the residue."""
    env = _Env(0xffc001, 1, 5)
    P = env.P
    level = 3
    ringQ = env.params.ringQ.AtLevel(level)
    p = H.rand_poly(QI[: level + 1], env.N, env.rng)
    words = P.enc.RingQ2T(level, p, env.n)[0]
    assert int(words.max()) >= env.t
    assert int(words.max()) < 3 * env.t
    big = E.small_rows(np.zeros(env.N, dtype=np.int64), QI[: level + 1])      # a zero polynomial decodes to zero words mod t
    ringQ.Add(big, big, big)
    assert all(int(w) % env.t == 0 for w in P.enc.RingQ2T(level, big, env.n)[0])

"""The multiparty restatement (tests/multiparty_oracle.py) anchored by decryption, with the reference's test set
(multiparty/test_params.go: logN = 10, five Q primes, one P prime with BaseTwoDecomposition 16 or two P primes) plus a ring without P,
five parties, and the noise bounds of multiparty/multiparty_test.go:167, 392, 461; plus the representative ranges the device kernels
must reproduce."""
import math

import numpy as np
import pytest

from oracle import encryptor as E
from oracle import oracle as O
from tests import multiparty_oracle as M

U64 = np.uint64
QI = [0x200000440001, 0x7fff80001, 0x800280001, 0x7ffd80001, 0x7ffc80001]
PJ = [0x3ffffffb80001, 0x4000000800001]
PARAMS = {"one_p": (QI, PJ[:1]), "two_p": (QI, PJ), "no_p": (QI, [])}
SIGMA = 3.2
SIGMA_FLOOD = 8 * SIGMA        # multiparty_test.go:339


def _gauss(rng, sigma, bound, shape):
    while True:
        v = np.rint(rng.normal(0, sigma, shape))
        if np.all(np.abs(v) <= bound):
            return v.astype(np.int64)


def _rand_rows(rng, moduli, N):
    return np.stack([rng.integers(0, q, N, dtype=U64) for q in moduli])


def _setup(name, n_parties, seed):
    q, p = PARAMS[name]
    params = O.Parameters(10, q, p)
    N = params.N()
    rng = np.random.default_rng(seed)
    s = [rng.integers(-1, 2, N) for _ in range(n_parties)]
    return params, rng, s, [M.sk_rows(params, si) for si in s], M.sk_rows(params, sum(s))


@pytest.mark.parametrize("name", list(PARAMS))
def test_collective_public_key_decrypts_within_the_reference_bound(name):
    K = 5
    params, rng, s, sks, sk_ideal = _setup(name, K, 1)
    P = M.Protocols(params)
    N = params.N()
    moduli = list(params.qi) + list(params.pi)
    crp = _rand_rows(rng, moduli, N)
    shares = [P.ckg_share(sks[i], crp, _gauss(rng, SIGMA, 6 * SIGMA, N)) for i in range(K)]
    pk = P.ckg_public_key(M.aggregate(shares, moduli), crp)
    nq = len(params.qi)
    noise = M.decrypt_noise(params, [pk[0][:nq], pk[1][:nq]], sk_ideal, montgomery=True)
    assert M.log2_std(noise) <= math.log2(math.sqrt(K) * SIGMA) + 1          # multiparty_test.go:167


def _fresh_ct(params, rng, sk, level):
    N = params.N()
    a = _rand_rows(rng, params.qi[: level + 1], N)
    c0 = E.Encryptor(params).encryptZeroSkFromC1QP(level, -1, sk, a, _gauss(rng, SIGMA, 6 * SIGMA, N), True, False)
    return [c0, a]


@pytest.mark.parametrize("name", list(PARAMS))
@pytest.mark.parametrize("level", [4, 2])
def test_key_switch_decrypts_under_the_output_key(name, level):
    K = 5
    params, rng, s_in, sks_in, ideal_in = _setup(name, K, 2 + level)
    s_out = [rng.integers(-1, 2, params.N()) for _ in range(K)]
    sks_out = [M.sk_rows(params, si) for si in s_out]
    ideal_out = M.sk_rows(params, sum(s_out))
    P = M.Protocols(params)
    ct = _fresh_ct(params, rng, ideal_in, level)
    sig = math.sqrt(SIGMA ** 2 + SIGMA_FLOOD ** 2)                              # keyswitch_sk.go:45-52
    shares = [P.cks_share(level, sks_in[i], sks_out[i], ct[1], _gauss(rng, sig, 6 * sig, params.N())) for i in range(K)]
    qs = params.qi[: level + 1]
    for sh in shares:
        assert all(int(sh[r].max()) < 2 * q for r, q in enumerate(qs))        # CRed(MRedLazy + e): [0, 2q)
    agg = M.aggregate(shares, qs)
    assert all(int(agg[r].max()) < (K + 1) * q for r, q in enumerate(qs))
    out = P.cks_key_switch(ct, agg)
    noise = M.decrypt_noise(params, out, ideal_out)
    assert M.log2_std(noise) <= math.log2(M.noise_key_switch(K, SIGMA, SIGMA_FLOOD)) + 1    # multiparty_test.go:392


@pytest.mark.parametrize("name", list(PARAMS))
@pytest.mark.parametrize("level", [4, 2])
def test_public_key_switch_decrypts_under_the_output_key(name, level):
    K = 5
    params, rng, s_in, sks_in, ideal_in = _setup(name, K, 7 + level)
    N = params.N()
    s_out = rng.integers(-1, 2, N)
    sk_out = M.sk_rows(params, s_out)
    moduli = list(params.qi) + list(params.pi)
    a = _rand_rows(rng, moduli, N)
    pk = np.stack([E.Encryptor(params).encryptZeroSkFromC1QP(len(params.qi) - 1, len(params.pi) - 1, sk_out, a.copy(), _gauss(rng, SIGMA, 6 * SIGMA, N),
                                                             True, True), a])
    P = M.Protocols(params)
    ct = _fresh_ct(params, rng, ideal_in, level)
    shares = []
    for i in range(K):
        u = rng.integers(-1, 2, N)
        shares.append(np.stack(P.pcks_share(level, sks_in[i], pk, ct[1], u, _gauss(rng, SIGMA, 6 * SIGMA, N), _gauss(rng, SIGMA, 6 * SIGMA, N),
                                            _gauss(rng, SIGMA_FLOOD, 6 * SIGMA_FLOOD, N))))
    agg = M.aggregate(shares, params.qi[: level + 1])
    out = P.pcks_key_switch(ct, agg)
    noise = M.decrypt_noise(params, out, sk_out)
    bound = M.noise_public_key_switch(N, bool(params.pi), K, SIGMA, SIGMA_FLOOD)
    assert M.log2_std(noise) <= math.log2(bound) + 1                          # multiparty_test.go:461


def test_aggregate_is_the_wrapping_left_fold():
    """With every share at 2q - 1 the raw sum at step k is (k + 2) q - k: past 2^64 from k = 7 for a 61-bit q > 2^64 / 9, where Go's
    uint64 wraps and CRed's single subtract leaves the wrapped value."""
    q = O.gen_moduli(11, [61], [])[0][0]
    assert q > (1 << 64) // 9
    K = 17
    shares = [np.full((1, 8), 2 * q - 1, dtype=U64) for _ in range(K)]
    got = M.aggregate(shares, [q])
    a = 2 * q - 1
    wrapped = False
    for _ in range(1, K):
        t = a + 2 * q - 1
        wrapped |= t >= 1 << 64
        t &= (1 << 64) - 1
        a = t - q if t >= q else t
    assert wrapped
    assert int(got[0, 0]) == a


@pytest.mark.parametrize("name,pw2", [("one_p", 16), ("two_p", 0), ("no_p", 16)])
def test_evaluation_key_share_of_one_party_is_the_single_party_key(name, pw2):
    """With one party, EvaluationKeyGenProtocol.GenShare and KeyGenerator.genEvaluationKey compute the same component 0."""
    params, rng, s, sks, _ = _setup(name, 2, 3)
    kg = M.KeyGen(params, pw2)
    N = params.N()
    moduli = list(params.qi) + list(params.pi)
    crp = [[_rand_rows(rng, moduli, N) for _ in range(max(kg.sizes))] for _ in range(kg.nd)]
    e = [[_gauss(rng, SIGMA, 6 * SIGMA, N) for _ in range(max(kg.sizes))] for _ in range(kg.nd)]
    share = kg.evkg_share(sks[0], sks[1], crp, e)
    evk = E.gen_evaluation_key(params, sks[0][: len(params.qi)], sks[1], crp, e, pw2)
    for i in range(kg.nd):
        for j in range(kg.sizes[i]):
            assert np.array_equal(share[i, j], evk.data[i, j, 0])

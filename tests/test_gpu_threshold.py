"""The t-out-of-N threshold scheme on the device (lgpu_mp_shamir_share, lattigo_b200.multiparty.Thresholdizer / Combiner) word for word
against tests/threshold_oracle.py: Shamir shares on the multiparty test sets with and without P, at thresholds 1, 2, 5 and 16 (twice the
kernel's 8-point chunk), at 1, 7, 8, 9 and 17 points and at the point edges, on full-range 64-bit words, from aligned and odd-word-offset
buffers, and at PN16QP1761 size; the reference's whole flow for 5 parties; a t = 3 of 5 collective key switch and relinearization key
that decrypt under the ideal secret; and the ShamirSecretShare wire format. Run with -m gpu on an H100."""
import math

import numpy as np
import pytest

from oracle import encryptor as E
from oracle import oracle as O
from tests import helpers as H
from tests import multiparty_oracle as M
from tests import threshold_oracle as T

pytestmark = pytest.mark.gpu
U64 = np.uint64
MASK = (1 << 64) - 1
QI = [0x200000440001, 0x7fff80001, 0x800280001, 0x7ffd80001, 0x7ffc80001]
PJ = [0x3ffffffb80001, 0x4000000800001]
PARAMS = {"one_p": (QI, PJ[:1]), "two_p": (QI, PJ), "no_p": (QI, [])}
SIGMA = 3.2
CHUNK = 8                                   # kShamirPts in csrc/multiparty.cu


@pytest.fixture(scope="module")
def ctxs():
    import lattigo_b200 as lb
    cs = {name: lb.Context(10, q, p) for name, (q, p) in PARAMS.items()}
    yield cs
    for c in cs.values():
        c.close()


def _edge_points(moduli):
    return [0, MASK] + [x for q in moduli for x in (q - 1, q, q + 1)]


def _shares(ctx, moduli, t, points, rng, aligned=True):
    """lgpu_mp_shamir_share in one launch on full-range random words, polynomial and shares in one pool at an odd word offset when not
    aligned; returns (shares, expected shares) on the host."""
    import ctypes
    import torch
    import lattigo_b200 as lb
    N, rows, n = ctx.N, len(moduli), len(points)
    poly = rng.integers(0, 1 << 64, (t, rows, N), dtype=U64)
    poly[:, :, :2] = U64(MASK)
    off = 0 if aligned else 1
    pool = torch.zeros((t + n) * rows * N + 2, dtype=torch.int64, device="cuda")
    d_poly = pool[off: off + t * rows * N].view(t, rows, N)
    d_poly.copy_(ctx.to_device(poly))
    d_out = pool[off + t * rows * N: off + (t + n) * rows * N].view(n, rows, N)
    arr = (ctypes.c_uint64 * n)(*points)
    lq, lp = len(ctx.Q) - 1, len(ctx.P) - 1
    assert H.launch_delta(lambda: lb._lib.check(lb.lib().lgpu_mp_shamir_share(ctx.h, lq, lp, ctypes.c_void_p(d_poly.data_ptr()), t, arr, n,
                                                                              ctypes.c_void_p(d_out.data_ptr()), lb.ring._stream()))) == 1
    return ctx.to_host(d_out), T.shamir_shares(poly, points, moduli, N)


@pytest.mark.parametrize("name", list(PARAMS))
@pytest.mark.parametrize("t", [1, 2, 5, 2 * CHUNK])
@pytest.mark.parametrize("n", [1, CHUNK - 1, CHUNK, CHUNK + 1, 2 * CHUNK + 1])
@pytest.mark.parametrize("aligned", [True, False])
def test_shamir_shares_match_the_oracle(ctxs, name, t, n, aligned):
    q, p = PARAMS[name]
    moduli = q + p
    rng = np.random.default_rng(1000 * t + 10 * n + aligned)
    pool = _edge_points(moduli) + [int(x) for x in rng.integers(0, 1 << 63, 8)]
    points = [pool[(t + k) % len(pool)] for k in range(n)]
    got, want = _shares(ctxs[name], moduli, t, points, rng, aligned)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("name", list(PARAMS))
def test_shamir_shares_at_the_point_edges(ctxs, name):
    import lattigo_b200 as lb
    q, p = PARAMS[name]
    moduli = q + p
    rng = np.random.default_rng(5)
    points = _edge_points(moduli)
    got, want = _shares(ctxs[name], moduli, 5, points, rng)
    assert np.array_equal(got, want)
    # GenShamirSecretShare for one recipient is the same share
    ctx = ctxs[name]
    poly = ctx.to_device(rng.integers(0, 1 << 64, (3, len(moduli), ctx.N), dtype=U64))
    thr = lb.multiparty.Thresholdizer(ctx, None)
    many = ctx.to_host(thr.GenShamirSecretShares(points, poly))
    for k in (0, 1, len(points) - 1):
        assert np.array_equal(ctx.to_host(thr.GenShamirSecretShare(points[k], poly)), many[k])


def test_shamir_shares_at_pn16():
    """PN16QP1761 (38 rows of 2^16 words): t = 4 coefficients shared to 9 recipients, across two point chunks, against the oracle and
    against the ring API's EvalPolyScalar on canonical words."""
    import lattigo_b200 as lb
    from lattigo_b200.params import PRESETS
    from lattigo_b200.ringqp import Poly, RingQP
    pr = PRESETS["CKKS_PN16QP1761"]
    q, p = pr["Q"], pr["P"]
    ctx = lb.Context(16, q, p)
    try:
        rng = np.random.default_rng(16)
        points = [1, 2, 3, q[0], q[0] + 1, p[0] - 1, MASK, 12345678901234567, 9]
        got, want = _shares(ctx, q + p, 4, points, rng)
        assert np.array_equal(got, want)
        del got, want
        S = lb.encryptor.Samplers(ctx, 4)
        thr = lb.multiparty.Thresholdizer(ctx, S)
        poly = thr.GenShamirPolynomial(4, S.UniformQP(len(q) - 1, len(p) - 1)[0])
        shares = thr.GenShamirSecretShares(points, poly)
        nq = len(q)
        rqp = RingQP(ctx)
        for k in (0, 4, 8):
            out = Poly(ctx.new_poly(nq), ctx.new_poly(len(p)))
            rqp.EvalPolyScalar([Poly(poly[i, :nq].contiguous(), poly[i, nq:].contiguous()) for i in range(4)], points[k], out)
            assert np.array_equal(ctx.to_host(shares[k, :nq]), ctx.to_host(out.Q))
            assert np.array_equal(ctx.to_host(shares[k, nq:]), ctx.to_host(out.P))
    finally:
        ctx.close()


class _Parties:
    """5 parties with Shamir points 1..5 and ternary secrets drawn from their own samplers."""

    def __init__(self, ctx, name, K=5):
        import lattigo_b200 as lb
        q, p = PARAMS[name]
        self.ctx, self.q, self.p, self.moduli = ctx, q, p, q + p
        self.params = O.Parameters(10, q, p)
        self.N = self.params.N()
        self.samplers = [lb.encryptor.Samplers(ctx, 2000 + i) for i in range(K)]
        self.s = [ctx.to_host(self.samplers[i].Ternary(P=2 / 3))[0] for i in range(K)]
        self.sk = [M.sk_rows(self.params, si) for si in self.s]
        self.d_sk = [ctx.to_device(x) for x in self.sk]
        self.ideal = M.aggregate(self.sk, self.moduli)
        self.points = list(range(1, K + 1))
        self.thr = [lb.multiparty.Thresholdizer(ctx, self.samplers[i]) for i in range(K)]

    def share(self, threshold):
        """Every party's Shamir polynomial and shares, and what each party aggregates; checked against the oracle on the way."""
        ctx, K = self.ctx, len(self.s)
        polys = [self.thr[i].GenShamirPolynomial(threshold, self.d_sk[i]) for i in range(K)]
        shares = [self.thr[i].GenShamirSecretShares(self.points, polys[i]) for i in range(K)]
        h_shares = []
        for i in range(K):
            h_poly = ctx.to_host(polys[i])
            assert np.array_equal(h_poly[0], self.sk[i])
            w = T.shamir_shares(h_poly, self.points, self.moduli, self.N)
            assert np.array_equal(ctx.to_host(shares[i]), w)
            h_shares.append(w)
        tsks = [self.thr[j].AggregateShares([shares[i][j] for i in range(K)]) for j in range(K)]
        for j in range(K):
            assert np.array_equal(ctx.to_host(tsks[j]), T.aggregate([h_shares[i][j] for i in range(K)], self.moduli))
        return tsks

    def combine(self, tsks, threshold, actives):
        import lattigo_b200 as lb
        ctx = self.ctx
        out = []
        for pt in actives[:threshold]:
            add = lb.multiparty.Combiner(ctx, pt, self.points, threshold).GenAdditiveShare(actives, pt, tsks[pt - 1])
            want = T.Combiner(self.moduli, pt, self.points, threshold).gen_additive_share(actives, pt, ctx.to_host(tsks[pt - 1]), self.N)
            assert np.array_equal(ctx.to_host(add), want)
            out.append(add)
        return out


@pytest.mark.parametrize("name", list(PARAMS))
@pytest.mark.parametrize("threshold", [1, 2, 4])
def test_reference_flow_recovers_the_ideal_secret(ctxs, name, threshold):
    P = _Parties(ctxs[name], name)
    tsks = P.share(threshold)
    for actives in (P.points[:threshold], [5, 2, 4, 1, 3]):
        adds = P.combine(tsks, threshold, actives)
        rec = T.aggregate([P.ctx.to_host(a) for a in adds], P.moduli)
        assert np.array_equal(rec, P.ideal), actives


def test_three_of_five_key_switch_and_relinearization_key(ctxs):
    """t = 3 of 5: the active parties 1, 3 and 5 combine additive shares, generate a collective public key and a relinearization key,
    and key-switch a public-key encryption to the zero key; the results decrypt under the ideal secret of all 5 parties."""
    import torch
    import lattigo_b200 as lb
    name, threshold = "two_p", 3
    ctx = ctxs[name]
    P = _Parties(ctx, name)
    tsks = P.share(threshold)
    actives = [1, 3, 5]
    adds = P.combine(tsks, threshold, actives)
    assert np.array_equal(T.aggregate([ctx.to_host(a) for a in adds], P.moduli), P.ideal)
    S = [P.samplers[pt - 1] for pt in actives]
    crs = lb.encryptor.Samplers(ctx, 0xC0FFEE)
    # collective public key from the 3 additive shares
    ckg = [lb.multiparty.PublicKeyGenProtocol(ctx, S[i]) for i in range(threshold)]
    crp = ckg[0].SampleCRP(crs)
    pk = ckg[0].GenPublicKey(ckg[0].AggregateShares([ckg[i].GenShare(adds[i], crp) for i in range(threshold)]), crp)
    level, batch = 4, 2
    ct = lb.encryptor.Encryptor(ctx).EncryptZeroPk(level, pk, S[0].Ternary(P=2 / 3, batch=batch), S[0].Gaussian(batch=batch),
                                                   S[0].Gaussian(batch=batch))
    # key switch to the zero key by the 3 active parties
    sigma_flood = 8 * SIGMA
    zero = torch.zeros_like(adds[0])
    cks = [lb.multiparty.KeySwitchProtocol(ctx, S[i], sigma_flood) for i in range(threshold)]
    agg = cks[0].AggregateShares([cks[i].GenShare(adds[i], zero, ct) for i in range(threshold)])
    out = ctx.to_host(cks[0].KeySwitch(ct, agg))
    zero_sk = np.zeros((len(P.moduli), P.N), dtype=U64)
    bound = math.log2(M.noise_key_switch(threshold, M.noise_fresh_pk(P.N, True), sigma_flood)) + 1
    for b in range(batch):
        assert M.log2_std(M.decrypt_noise(P.params, [out[b, 0], out[b, 1]], zero_sk)) <= bound
    # relinearization key from the same 3 parties drives MulRelinRescaleNew; the product decrypts under the ideal key
    rkg = [lb.multiparty.RelinearizationKeyGenProtocol(ctx, S[i], 0) for i in range(threshold)]
    rcrp = rkg[0].SampleCRP(crs)
    r1 = [rkg[i].GenShareRoundOne(adds[i], rcrp) for i in range(threshold)]
    agg1 = rkg[0].AggregateShares([x[1] for x in r1])
    agg2 = rkg[0].AggregateShares([rkg[i].GenShareRoundTwo(r1[i][0], adds[i], agg1) for i in range(threshold)])
    rlk = rkg[0].GenRelinearizationKey(agg1, agg2)
    rng = np.random.default_rng(9)
    cts = []
    for _ in range(2):
        c = []
        for _ in range(2):
            a = H.rand_poly(QI, P.N, rng)
            e = np.rint(rng.normal(0, SIGMA, P.N)).astype(np.int64)
            c.append(np.stack([E.Encryptor(P.params).encryptZeroSkFromC1QP(level, -1, P.ideal, a, e, True, False), a]))
        cts.append(ctx.to_device(np.stack(c)))
    prod = ctx.to_host(lb.CKKSEvaluator(ctx, rlk).MulRelinRescaleNew(cts[0], cts[1]))
    for b in range(2):
        assert M.log2_std(M.decrypt_noise(P.params, [prod[b, 0], prod[b, 1]], P.ideal)) < 20


@pytest.mark.parametrize("name", ["one_p", "no_p"])
def test_shamir_secret_share_wire_round_trip(ctxs, name):
    import lattigo_b200 as lb
    ctx = ctxs[name]
    q, p = PARAMS[name]
    rng = np.random.default_rng(11)
    share = ctx.to_device(rng.integers(0, 1 << 64, (len(q) + len(p), ctx.N), dtype=U64))
    data = lb.wire.store_qp_poly(ctx, share)
    binary_size = lambda rows: 8 + rows * (8 + 8 * ctx.N)          # ring.Poly.BinarySize
    assert len(data) == binary_size(len(q)) + binary_size(len(p))
    back, used = lb.wire.load_qp_poly(ctx, data)
    assert used == len(data)
    assert np.array_equal(ctx.to_host(back), ctx.to_host(share))

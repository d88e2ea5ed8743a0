"""The t-out-of-N threshold scheme (multiparty/threshold.go) on the CPU: the reference's own identity (multiparty_test.go:475-560) anchors
tests/threshold_oracle.py; the oracle's MForm, EvalPolyScalar words and Lagrange scalars; lattigo_b200.multiparty.Combiner's scalars
word for word against the oracle's; the argument checks of lgpu_mp_shamir_share, which run before any launch and so also on a host-only
context; and the errors of Thresholdizer and Combiner."""
import ctypes
import re

import numpy as np
import pytest

from oracle import oracle as O
from tests import multiparty_oracle as M
from tests import threshold_oracle as T

QI = [0x200000440001, 0x7fff80001, 0x800280001, 0x7ffd80001, 0x7ffc80001]
PJ = [0x3ffffffb80001, 0x4000000800001]
MODULI = QI + PJ
MASK = (1 << 64) - 1
FAKE = ctypes.c_void_p(1 << 20)          # never dereferenced: every case fails its checks first


def _edges(q):
    return [0, 1, q - 1, q, q + 1, 2 * q - 1, MASK - 1, MASK]


def _run_scheme(threshold, actives_idx, seed):
    """5 parties with points 1..5 share their secrets, every party aggregates what it receives (from a zero share, as the reference's
    test does), and the parties of actives[:threshold] combine. Returns (sum of the additive shares, the ideal secret)."""
    params = O.Parameters(10, QI, PJ)
    N, K = params.N(), 5
    rng = np.random.default_rng(seed)
    sks = [M.sk_rows(params, rng.integers(-1, 2, N)) for _ in range(K)]
    points = list(range(1, K + 1))
    received = [[np.zeros((len(MODULI), N), dtype=np.uint64)] for _ in range(K)]
    for i in range(K):
        poly = np.stack([sks[i]] + [np.stack([rng.integers(0, q, N, dtype=np.uint64) for q in MODULI]) for _ in range(threshold - 1)])
        shares = T.shamir_shares(poly, points, MODULI, N)
        for j in range(K):
            received[j].append(shares[j])
    tsks = [T.aggregate(r, MODULI) for r in received]
    actives = [points[i] for i in actives_idx]
    rec = np.zeros((len(MODULI), N), dtype=np.uint64)
    for pt in actives[:threshold]:
        cmb = T.Combiner(MODULI, pt, points, threshold)
        rec = T.aggregate([cmb.gen_additive_share(actives, pt, tsks[pt - 1], N), rec], MODULI)
    return rec, T.aggregate(sks, MODULI)


@pytest.mark.parametrize("threshold", [1, 2, 4])
@pytest.mark.parametrize("actives_idx", [[0, 1, 2, 3], [4, 1, 3, 0], [2, 0, 4, 1, 3]], ids=["first", "non_contiguous", "longer"])
def test_reference_identity_anchors_the_oracle(threshold, actives_idx):
    rec, ideal = _run_scheme(threshold, actives_idx, 7 * threshold + len(actives_idx))
    assert np.array_equal(rec, ideal)


def test_oracle_mform_is_the_canonical_montgomery_form_at_the_point_edges():
    from lattigo_b200.params import PRESETS
    for q in MODULI + list(PRESETS["CKKS_PN16QP1761"]["Q"]) + list(PRESETS["CKKS_PN16QP1761"]["P"]):
        for a in _edges(q):
            assert T.mform(a, q) == (a << 64) % q, (q, a)


def test_oracle_words_equal_the_per_word_statement():
    """eval_poly_scalar (vector ops) against eval_poly_scalar_word (Python ints) on full-range 64-bit words, at the point edges."""
    N = 1024
    rng = np.random.default_rng(3)
    for t in (1, 2, 5):
        poly = rng.integers(0, 1 << 64, (t, len(MODULI), N), dtype=np.uint64)
        poly[:, :, :4] = np.uint64(MASK)
        for pt in _edges(QI[1]) + [int(rng.integers(0, 1 << 63)) * 2 + 1]:
            got = T.eval_poly_scalar(poly, pt, MODULI, N)
            for r, q in enumerate(MODULI):
                for j in list(range(6)) + [int(x) for x in rng.integers(0, N, 6)]:
                    assert int(got[r, j]) == T.eval_poly_scalar_word([int(c) for c in poly[:, r, j]], pt, q), (t, pt, r, j)


@pytest.fixture(scope="module")
def ctx():
    import lattigo_b200 as lb
    c = lb.Context(10, QI, PJ, device=-1)
    yield c
    c.close()


@pytest.mark.parametrize("own,others,actives,threshold", [
    (1, [1, 2, 3, 4, 5], [1, 2, 3], 3),
    (2, [1, 2, 3, 4, 5], [5, 3, 2, 1], 3),                         # own point among the first t of a longer list
    (4, [1, 2, 3, 4, 5], [1, 2, 3, 4], 3),                         # own point not among the first t
    (3, [1, 3, 3, 5], [3, 5, 5], 3),                               # duplicate actives
    (1, [1, 1 + QI[1], 1 + PJ[0], 7], [1, 1 + QI[1], 1 + PJ[0], 7], 4),     # points congruent modulo q_1 and p_0: the inverse of 0 is 0
    (MASK, [MASK, 0, 2, MASK - 1], [0, MASK, MASK - 1], 3),
])
def test_combiner_scalars_equal_the_oracle(ctx, own, others, actives, threshold):
    from lattigo_b200 import multiparty as mp
    c = mp.Combiner(ctx, own, others, threshold)
    o = T.Combiner(MODULI, own, others, threshold)
    assert c.one == o.one
    assert c.lagrangeCoeffs == o.lagrangeCoeffs
    prod = c.prod(actives, own)
    assert prod == o.prod(actives, own)
    for i, q in enumerate(MODULI):
        assert 0 <= prod[i] < 2 * q
        want = 1 << 64
        for a in actives[:threshold]:
            if a != own:
                d = (a - own) % q
                want = want * a * pow(d, -1, q) if d else 0
        assert prod[i] % q == want % q, (i, q)


def _err(rc):
    import lattigo_b200 as lb
    assert rc == -1
    return lb.lib().lgpu_last_error().decode()


def test_shamir_share_checks(ctx):
    import lattigo_b200 as lb
    L = lb.lib()
    N = ctx.N
    pts = (ctypes.c_uint64 * 3)(1, 2, 3)
    ok = dict(lq=4, lp=1, poly=ctypes.c_void_p(1 << 30), t=3, pts=pts, n=3, shares=ctypes.c_void_p(1 << 20))

    def call(**kw):
        a = dict(ok, **kw)
        return _err(L.lgpu_mp_shamir_share(ctx.h, a["lq"], a["lp"], a["poly"], a["t"], a["pts"], a["n"], a["shares"], None))
    for lq, lp in ((5, 1), (-1, 1), (4, 2), (4, -2)):
        assert "level out of range" in call(lq=lq, lp=lp)
    for t in (0, -1, 65536):
        assert "threshold out of [1, 65535]" in call(t=t)
    for n in (0, 65536):
        assert "n_points out of [1, 65535]" in call(n=n)
    for k in ("poly", "pts", "shares"):
        assert "null argument" in call(**{k: None})
    rows = 7
    assert "shares overlap the Shamir polynomial" in call(shares=ctypes.c_void_p((1 << 30) - 3 * rows * N * 8 + 8))
    assert "shares overlap the Shamir polynomial" in call(shares=ctypes.c_void_p((1 << 30) + 3 * rows * N * 8 - 8))
    assert "shares overlap the Shamir polynomial" in call(lp=-1, shares=ctypes.c_void_p((1 << 30) + 3 * 5 * N * 8 - 8))
    assert "host-only" in call(shares=ctypes.c_void_p((1 << 30) + 3 * rows * N * 8))
    assert "host-only" in call(lp=-1, shares=ctypes.c_void_p((1 << 30) + 3 * 5 * N * 8))


def test_thresholdizer_and_combiner_errors(ctx):
    import torch
    import lattigo_b200 as lb
    from lattigo_b200 import multiparty as mp
    N = ctx.N
    thr = mp.Thresholdizer(ctx, None)
    for t in (0, -3):
        with pytest.raises(lb.LgpuError) as e:
            thr.GenShamirPolynomial(t, None)
        assert str(e.value) == "threshold should be >= 1"
    with pytest.raises(lb.LgpuError) as e:
        thr.AggregateShares(torch.zeros(7, N, dtype=torch.int64), torch.zeros(6, N, dtype=torch.int64))
    assert str(e.value) == "cannot AggregateShares: shares level do not match"
    cmb = mp.Combiner(ctx, 1, [1, 2, 3, 4], 3)
    with pytest.raises(lb.LgpuError) as e:
        cmb.GenAdditiveShare([1, 2], 1, None)
    assert str(e.value) == "cannot GenAdditiveShare: Not enough active players to combine threshold shares"
    with pytest.raises(lb.LgpuError, match=re.escape("active point 9 is not among")):
        cmb.GenAdditiveShare([1, 9, 2], 1, None)
    # an unknown point after the first t actives is never read, as in the reference
    assert cmb.prod([1, 2, 3, 9], 1) == T.Combiner(MODULI, 1, [1, 2, 3, 4], 3).prod([1, 2, 3], 1)
    for bad in (-1, 1 << 64):
        with pytest.raises(lb.LgpuError, match="64-bit unsigned"):
            mp.Combiner(ctx, bad, [1, 2], 2)
        with pytest.raises(lb.LgpuError, match="64-bit unsigned"):
            thr.GenShamirSecretShares([1, bad], None)

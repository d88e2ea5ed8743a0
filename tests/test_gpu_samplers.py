"""The device samplers (csrc/encrypt.cu) bit for bit against their restatement in oracle/philox.py: uniform, ternary {P} and {H}
exactly; the Gaussian against 50-digit arithmetic on the same Philox words, where only coefficients within 2^-40 of a rounding or
rejection boundary may differ. Also the exact distributions on device output, the separation of sampler kinds and stream ids, and
lgpu_small_poly_to_rns at the edges of its range."""
import numpy as np
import pytest
from scipy.stats import binomtest

from oracle import philox as X
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64
SEED = 0x1234567890ABCDEF
P_MIN = 1e-6


def _moduli(N):
    """Q: NTT primes just above 2^60 and 2^40 (a masked word is accepted about half the time, so the second word and later
    attempts are used), just below 2^55, a 30-bit prime and a 61-bit Qi60 prime; P: Qi60[0], above every q, and one above 2^50."""
    q = [H.ntt_prime(60, N, True), H.ntt_prime(55, N, False), H.ntt_prime(40, N, True), H.ntt_prime(30, N, False), H.Qi60[1]]
    p = [H.Qi60[0], H.ntt_prime(50, N, True)]
    assert max(q) < p[0]
    return q, p


_CTX = {}


@pytest.fixture(scope="module")
def ctx_of():
    import lattigo_b200 as lb

    def get(logN):
        if logN not in _CTX:
            q, p = _moduli(1 << logN)
            _CTX[logN] = lb.Context(logN, q, p)
        return _CTX[logN]
    yield get
    for c in _CTX.values():
        c.close()
    _CTX.clear()


def _uniform_device(ctx, ring, level, sid, batch, stride):
    """lgpu_sample_uniform into a buffer of `batch` blocks of `stride` words filled with all-ones: (values, padding)."""
    import torch
    import lattigo_b200 as lb
    from lattigo_b200.ring import _dptr, _stream
    rows = level + 1
    buf = torch.full((batch * stride,), -1, dtype=torch.int64, device="cuda:%d" % ctx.device)
    lb._lib.check(lb.lib().lgpu_sample_uniform(ctx.h, ring, level, SEED, sid, _dptr(buf), batch, stride, _stream()))
    host = ctx.to_host(buf).reshape(batch, stride)
    return host[:, : rows * ctx.N].reshape(batch, rows, ctx.N), host[:, rows * ctx.N:]


def _uniform_rows(ctx, ring, level):
    from lattigo_b200.ring import RING_Q
    if ring == RING_Q:
        return ctx.Q[: level + 1], list(range(level + 1))
    return ctx.P[: level + 1], [len(ctx.Q) + j for j in range(level + 1)]


# ---- (a) uniform -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("logN", [4, 12, 17])
def test_uniform_matches_the_restatement(ctx_of, logN):
    from lattigo_b200.ring import RING_P, RING_Q
    ctx = ctx_of(logN)
    N, nQ, nP = ctx.N, len(ctx.Q), len(ctx.P)
    cases = [(RING_Q, nQ - 1, 1, 0), (RING_P, nP - 1, 1, 0), (RING_Q, 2, 5, 3), (RING_P, 0, 5, 1)]
    for k, (ring, level, batch, pad) in enumerate(cases):
        sid = 40 + k
        stride = (level + 1 + pad) * N
        got, padding = _uniform_device(ctx, ring, level, sid, batch, stride)
        mods, limbs = _uniform_rows(ctx, ring, level)
        want = X.uniform(SEED, sid, mods, limbs, batch, N)
        assert np.array_equal(got, want), (ring, level, batch, [int((got[:, r] != want[:, r]).sum()) for r in range(level + 1)])
        assert (padding == U64(0xFFFFFFFFFFFFFFFF)).all()
        if batch > 1:       # a sub-batch draws the same elements as the larger batch
            sub, _ = _uniform_device(ctx, ring, level, sid, 2, (level + 1) * N)
            assert np.array_equal(sub, want[:2])
        if logN == 17 and batch == 1:          # the exact law, on device output
            for r, q in enumerate(mods):
                p_bins, p_res = H.uniform_pvalues(got[0, r], int(q))
                assert p_bins > P_MIN and p_res > P_MIN, (hex(int(q)), p_bins, p_res)


def test_uniform_qp_rows_on_one_stream_id_are_distinct(ctx_of):
    """UniformQP draws Q and P on one id; the limb index in the counter keeps the rows apart (with the launch row instead, P row
    j would repeat Q row j's words)."""
    import lattigo_b200 as lb
    ctx = ctx_of(12)
    nQ, nP = len(ctx.Q), len(ctx.P)
    got = ctx.to_host(lb.encryptor.Samplers(ctx, SEED).UniformQP(nQ - 1, nP - 1, batch=2, stream_id=9))
    want = np.concatenate([X.uniform(SEED, 9, ctx.Q, range(nQ), 2, ctx.N), X.uniform(SEED, 9, ctx.P, range(nQ, nQ + nP), 2, ctx.N)], axis=1)
    assert np.array_equal(got, want)
    mask = (1 << 30) - 1                       # compare the low bits every row keeps
    low = got & U64(mask)
    for j in range(nP):
        assert (low[:, nQ + j] == low[:, j]).mean() < 0.01


# ---- (b) ternary -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("logN", [4, 12])
def test_ternary_p_matches_the_restatement(ctx_of, logN):
    import lattigo_b200 as lb
    ctx = ctx_of(logN)
    S = lb.encryptor.Samplers(ctx, SEED)
    for k, p in enumerate([2.0 ** -20, 1 / 3, 0.5, 2 / 3, 1.0]):
        got = S.Ternary(P=p, batch=3, stream_id=60 + k).cpu().numpy()
        assert np.array_equal(got, X.ternary_p(SEED, 60 + k, 3, ctx.N, p)), p
        if p == 1.0:
            assert (got != 0).all()
        elif logN == 12:
            nz = int((got != 0).sum())
            assert binomtest(nz, got.size, X.ternary_p_nonzero_probability(p)).pvalue > P_MIN


def test_ternary_rejects_p_out_of_range_and_recovers(ctx_of):
    import torch
    import lattigo_b200 as lb
    from lattigo_b200.ring import _dptr, _stream
    ctx = ctx_of(12)
    L = lb.lib()
    out = torch.zeros((2, ctx.N), dtype=torch.int64, device="cuda:%d" % ctx.device)
    for k, bad in enumerate([0.0, -0.25, 1.0 + 2.0 ** -52, 1.5, float("nan")]):
        assert L.lgpu_sample_ternary(ctx.h, bad, 0, SEED, 70, _dptr(out), 2, _stream()) != 0, bad
        assert "P must be in (0, 1]" in L.lgpu_last_error().decode()
        assert L.lgpu_sample_ternary(ctx.h, 0.5, 0, SEED, 71 + k, _dptr(out), 2, _stream()) == 0
        assert np.array_equal(out.cpu().numpy(), X.ternary_p(SEED, 71 + k, 2, ctx.N, 0.5)), bad


@pytest.mark.parametrize("logN", [4, 12, 16])
def test_ternary_h_matches_the_restatement(ctx_of, logN):
    import lattigo_b200 as lb
    ctx = ctx_of(logN)
    N = ctx.N
    S = lb.encryptor.Samplers(ctx, SEED)
    for k, h in enumerate([1, 32, N // 2, N - 1, N, N + 5]):
        got = S.Ternary(H=h, batch=2, stream_id=80 + k).cpu().numpy()
        assert ((got != 0).sum(axis=1) == min(h, N)).all(), h
        assert np.array_equal(got, X.ternary_h(SEED, 80 + k, 2, N, h)), h


def test_ternary_h_positions_and_signs_on_device(ctx_of):
    import lattigo_b200 as lb
    ctx = ctx_of(12)
    N, h, batch = ctx.N, 32, 1024
    t = lb.encryptor.Samplers(ctx, SEED).Ternary(H=h, batch=batch, stream_id=90).cpu().numpy()
    from scipy.stats import chi2
    counts = (t != 0).sum(axis=0)
    s2 = h / N * (1 - h / N)
    stat = (N - 1) / N * float(((counts - batch * h / N) ** 2).sum()) / (batch * s2)
    assert chi2.sf(stat, N - 1) > P_MIN, stat
    assert binomtest(int((t == 1).sum()), batch * h, 0.5).pvalue > P_MIN


# ---- (c) Gaussian ----------------------------------------------------------------------------------------------------------
def _gaussian_exact(b, i, sigma, bound):
    """The value of coefficient i of polynomial b with m at 50 digits (float64 only skips attempts at least 2^-30 above the bound)."""
    import mpmath
    for a0 in range(0, 1 << 24, 4096):
        u1, u2, neg = X.gaussian_draws(SEED, 100, U64(b), U64(i), np.arange(a0, a0 + 4096, dtype=U64))
        for k in np.nonzero(X.gaussian_m(u1, u2, sigma) <= bound * (1 + 2.0 ** -30))[0]:
            m = mpmath.sqrt(-2 * mpmath.log(mpmath.mpf(float(u1[k])))) * abs(mpmath.cospi(2 * mpmath.mpf(float(u2[k])))) * mpmath.mpf(sigma)
            if m <= bound:
                v = int(mpmath.floor(m + mpmath.mpf(0.5)))
                return -v if neg[k] else v
    raise AssertionError("no accepted attempt")


@pytest.mark.parametrize("sigma,bound,logN,batch", [(3.2, 19.2, 12, 4), (0.5, 1.0, 12, 4), (1000.0, 1.5, 12, 1), (2.0 ** 20, 6 * 2.0 ** 20, 12, 4)])
def test_gaussian_matches_high_precision(ctx_of, sigma, bound, logN, batch):
    import mpmath
    import lattigo_b200 as lb
    mpmath.mp.dps = 50
    ctx = ctx_of(logN)
    N = ctx.N
    got = lb.encryptor.Samplers(ctx, SEED).Gaussian(sigma, bound, batch=batch, stream_id=100).cpu().numpy()
    v, m, att, near = X.gaussian_float64(SEED, 100, batch, N, sigma, bound)
    # the float64 restatement agrees with 50 digits away from the boundaries; at them, the 50-digit value is the expected one
    rng = np.random.default_rng(int(sigma * 8))
    check = {(int(b), int(i)) for b, i in zip(*np.nonzero(near))}
    check |= {(int(b), int(i)) for b, i in zip(rng.integers(0, batch, 2000), rng.integers(0, N, 2000))}
    for b, i in check:
        e = _gaussian_exact(b, i, sigma, bound)
        if not near[b, i]:
            assert e == v[b, i], (b, i)
    diff = got != v
    print("sigma %g bound %g: %d coefficients within 2^-40 of a boundary, %d differ from the float64 restatement, max attempt %d"
          % (sigma, bound, int(near.sum()), int(diff.sum()), int(att.max())))
    assert not (diff & ~near).any(), [(int(b), int(i), int(got[b, i]), int(v[b, i])) for b, i in zip(*np.nonzero(diff & ~near))][:8]
    assert near.sum() <= 4
    if sigma == 3.2:       # the exact law, on device output
        edges = H.gaussian_edges(bound)
        law = X.gaussian_law(sigma, bound, edges)
        assert H.gof_pvalue(np.bincount(X.gaussian_bin_index(got.ravel(), edges), minlength=len(law)), law) > P_MIN


def test_gaussian_accepts_m_equal_to_the_bound(ctx_of):
    """m <= bound, not m < bound. For coefficients whose first attempt has |z| in (2, 3.5), sigma is chosen so that m = |z| sigma
    rounds to exactly the bound 20.25 (with correctly rounded log and cospi), and then so that it rounds to one ulp above. At the
    bound the attempt is taken (value +-20); one ulp above, it is rejected. A device function one ulp off can spoil a candidate,
    so half of them must hold."""
    import mpmath
    import lattigo_b200 as lb
    mpmath.mp.dps = 50
    ctx = ctx_of(4)
    S = lb.encryptor.Samplers(ctx, SEED)
    bound, batch = 20.25, 256
    u1, u2, neg = X.gaussian_draws(SEED, 110, np.arange(batch, dtype=U64)[:, None], np.arange(ctx.N, dtype=U64)[None, :], 0)
    exact, tried = 0, 0
    for b, i in zip(*np.nonzero(np.abs(X.gaussian_m(u1, u2, 1.0) - 2.75) < 0.75)):
        s = np.sqrt(-2.0 * float(mpmath.log(mpmath.mpf(float(u1[b, i])))))
        az = abs(s * float(mpmath.cospi(2 * mpmath.mpf(float(u2[b, i])))))
        sig = [x for x in bound / az * (1 + np.arange(-8, 9) * 2.0 ** -52) if az * x == bound]
        if not sig:
            continue
        up = sig[-1]
        while az * up <= bound:
            up = np.nextafter(up, np.inf)
        tried += 1
        at = S.Gaussian(sig[-1], bound, batch=batch, stream_id=110).cpu().numpy()[b, i]
        above = S.Gaussian(float(up), bound, batch=batch, stream_id=110).cpu().numpy()[b, i]
        want = -20 if neg[b, i] else 20
        exact += int(at == want and above != want)
        if tried == 16:
            break
    print("%d of %d candidates hit the bound exactly" % (exact, tried))
    assert tried >= 8 and 2 * exact >= tried, (exact, tried)


# ---- (e) stream separation -------------------------------------------------------------------------------------------------
def _replay_h(row0, s, h):
    """Replays the {H} placement from a uniform row drawn on the same counters: bits 32.. of a value are the first candidate's
    position and bit 0 its sign. Returns (matching non-zero coefficients, their mean and standard deviation by chance)."""
    N = len(s)
    pos = ((row0 >> U64(32)) & U64(N - 1)).astype(np.int64)
    sgn = np.where(row0 & U64(1), 1, -1)
    _, first = np.unique(pos, return_index=True)
    hits = int((s[pos[first]] == sgn[first]).sum())
    p = h / N / 2
    return hits, len(first) * p, np.sqrt(len(first) * p * (1 - p))


def test_sampler_kinds_and_calls_do_not_share_streams():
    import lattigo_b200 as lb
    from lattigo_b200.ring import RING_Q
    logN, h = 12, 1024
    N = 1 << logN
    q = [H.ntt_prime(55, N, False), H.ntt_prime(45, N, False)]
    p = [H.ntt_prime(55, N, True)]
    ctx = lb.Context(logN, q, p)
    try:
        # automatic ids, in the order a key generation draws them
        S = lb.encryptor.Samplers(ctx, SEED)
        a = ctx.to_host(S.UniformQP(1, 0))
        s = S.Ternary(H=h).cpu().numpy()[0]
        hits, mu, sd = _replay_h(a[0, 0], s, h)
        print("automatic ids: %d of %d secret coefficients replayed from the public row (chance %.0f +- %.0f)" % (hits, h, mu, sd))
        assert hits <= mu + 6 * sd
        # one explicit id for two kinds
        a = ctx.to_host(S.Uniform(RING_Q, 0, stream_id=5))
        s = S.Ternary(H=h, stream_id=5).cpu().numpy()[0]
        hits, mu, sd = _replay_h(a[0, 0], s, h)
        print("shared id: %d of %d secret coefficients replayed (chance %.0f +- %.0f)" % (hits, h, mu, sd))
        assert hits <= mu + 6 * sd
    finally:
        ctx.close()


# ---- (f) lgpu_small_poly_to_rns --------------------------------------------------------------------------------------------
def test_small_poly_to_rns_at_the_edges(ctx_of):
    import torch
    import lattigo_b200 as lb
    ctx = ctx_of(12)
    N = ctx.N
    qmin = min(ctx.Q + ctx.P)
    e = (qmin - 1) // 2
    assert max(ctx.P) > max(ctx.Q)
    rng = np.random.default_rng(4)
    small = rng.integers(-e, e + 1, (2, N), dtype=np.int64)
    small[0, :5] = [0, 1, -1, e, -e]
    small[1, -5:] = [-e, e, -1, 1, 0]
    d = torch.from_numpy(small).cuda(ctx.device)
    for lq, lp in ((len(ctx.Q) - 1, len(ctx.P) - 1), (2, 0)):
        rq, rp = lb.encryptor.small_poly_to_rns(ctx, d, lq, lp)
        rq, rp = ctx.to_host(rq), ctx.to_host(rp)
        for rows, mods in ((rq, ctx.Q[: lq + 1]), (rp, ctx.P[: lp + 1])):
            for r, m in enumerate(mods):
                want = np.array([int(x) % m for x in small.ravel()], dtype=U64).reshape(2, N)
                assert np.array_equal(rows[:, r], want), (lq, lp, hex(m))

"""CPU side of the device samplers (csrc/encrypt.cu): oracle/philox.py against the Random123 known-answer vectors, the counter
layout (no two sampler kinds or stream ids share a Philox input; lattigo_b200.encryptor.Samplers never reuses an id), and the
restated streams against the exact distributions they must follow, at sample counts too large for the device tests. The
restatement is pinned to the device's bits by tests/test_gpu_samplers.py, and every seed here is fixed, so these tests are
deterministic."""
import numpy as np
import pytest
from scipy.stats import binomtest, chi2

from oracle import philox as X
from tests import helpers as H

P_MIN = 1e-6


# Random123 known-answer vectors for philox4x32, 10 rounds: ctr0..3, key0..1 -> out0..3
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(v) for v in X.philox4x32_10(ctr, key)) == want
    # vectorised: the same block in every lane of a broadcast
    got = X.philox4x32_10(tuple(np.full(3, c, dtype=np.uint64) for c in ctr), key)
    assert all((g == w).all() for g, w in zip(got, want))


def test_counters_are_injective_across_kinds_and_stream_ids():
    seed = 0x1234567890ABCDEF
    coeffs = np.array([0, 1, 2, (1 << 16) - 1, (1 << 17) - 1, 0xFFFFFFFF], dtype=np.uint64)
    attempts = np.array([0, 1, 7, 0xFFFFFFFF], dtype=np.uint64)
    batches = np.array([0, 1, 2, 127, 128, 65534], dtype=np.uint64)
    limbs = np.array([0, 1, 5, 6, 127], dtype=np.uint64)
    polys = {X.KIND_UNIFORM: (batches[:, None] * np.uint64(X.MAX_ROWS) + limbs[None, :]).ravel()}
    for k in (X.KIND_TERNARY_P, X.KIND_TERNARY_H, X.KIND_GAUSSIAN):
        polys[k] = batches
    seen = {}
    for sid in (0, 1, 2, 3, 7, 1 << 32, (1 << 32) + 2, (1 << 64) - 1):
        for kind, poly in polys.items():
            if kind == X.KIND_TERNARY_P:
                c, a = coeffs, np.zeros(1, dtype=np.uint64)
            elif kind == X.KIND_TERNARY_H:          # counter (attempt, batch, stream, 0)
                c, a = attempts, np.zeros(1, dtype=np.uint64)
            else:
                c, a = coeffs, attempts
            P, C, A = np.meshgrid(poly, c, a, indexing="ij")
            words = X.counter(kind, seed, sid, P.ravel(), C.ravel(), A.ravel())
            assert ((words[1] >> np.uint64(X.KIND_SHIFT)) == kind).all()          # the kind field is not reached by the index
            for t in zip(*(np.broadcast_to(w, P.size).tolist() for w in words)):
                assert t not in seen, ("Philox input shared", seen[t], (kind, sid))
                seen[t] = (kind, sid)
    # one seed: distinct stream ids give distinct (key, counter word 2), also when only the high 32 bits differ
    rng = np.random.default_rng(1)
    sids = {int(s) for s in rng.integers(0, 1 << 63, 5000, dtype=np.int64)} | {s << 32 for s in range(1, 2000)} | set(range(2000))
    assert len({X.make_key(seed, s) for s in sids}) == len(sids)


class _FakeLib:
    """Records the sampler calls Samplers makes instead of launching them."""

    def __init__(self):
        self.calls = []

    def lgpu_sample_uniform(self, h, ring, level, seed, sid, out, batch, stride, stream):
        self.calls.append(("uniform", ring, level, seed, sid, batch))
        return 0

    def lgpu_sample_ternary(self, h, p, hw, seed, sid, out, batch, stream):
        self.calls.append(("ternary_h" if hw > 0 else "ternary_p", hw, None, seed, sid, batch))
        return 0

    def lgpu_sample_gaussian(self, h, sigma, bound, seed, sid, out, batch, stream):
        self.calls.append(("gaussian", None, None, seed, sid, batch))
        return 0


class _FakeCtx:
    def __init__(self, N, nQ, nP):
        self.h, self.N, self.device = None, N, 0
        self.Q, self.P = [0] * nQ, [0] * nP

    def new_poly(self, limbs, batch=None):
        import torch
        return torch.zeros((limbs, self.N) if batch is None else (batch, limbs, self.N), dtype=torch.int64)


def test_samplers_give_every_call_its_own_stream_id(monkeypatch):
    """Samplers with automatic ids, in the order a key generation uses them: every call takes one id no other call uses, and the
    Philox inputs of all the calls (restated from the recorded arguments) are pairwise disjoint."""
    import types
    from lattigo_b200 import encryptor as E
    from lattigo_b200.ring import RING_P, RING_Q
    fake = _FakeLib()
    monkeypatch.setattr(E, "_lib", types.SimpleNamespace(lib=lambda: fake, check=lambda rc: None))
    monkeypatch.setattr(E, "_dptr", lambda t: None)
    monkeypatch.setattr(E, "_stream", lambda: None)
    N, nQ, nP, seed = 16, 3, 2, 0x1234567890ABCDEF
    S = E.Samplers(_FakeCtx(N, nQ, nP), seed)
    calls = []
    for fn in (lambda: S.UniformQP(nQ - 1, nP - 1, batch=2), lambda: S.Ternary(H=4), lambda: S.Gaussian(batch=2),
               lambda: S.UniformQP(1, -1), lambda: S.Uniform(RING_Q, 2, batch=2), lambda: S.Uniform(RING_P, 1),
               lambda: S.Ternary(P=0.5, batch=2), lambda: S.UniformQP(nQ - 1, 0)):
        n0 = len(fake.calls)
        fn()
        calls.append(fake.calls[n0:])
    ids = [{c[4] for c in cs} for cs in calls]
    assert all(len(s) == 1 for s in ids), ids                      # one id per call, both rings of UniformQP included
    ids = [s.pop() for s in ids]
    assert len(set(ids)) == len(ids), ids

    def inputs(c):
        kind, a1, level, sd, sid, batch = c
        b = np.arange(batch, dtype=np.uint64)[:, None]
        i = np.arange(N, dtype=np.uint64)[None, :]
        if kind == "uniform":
            limbs = np.arange(level + 1) + (0 if a1 == RING_Q else nQ)
            out = []
            for lb in limbs:
                for a in range(3):
                    out.append(X.counter(X.KIND_UNIFORM, sd, sid, b * np.uint64(X.MAX_ROWS) + np.uint64(lb), i, a))
            return out
        if kind == "ternary_h":
            return [X.counter(X.KIND_TERNARY_H, sd, sid, b, np.arange(4 * N, dtype=np.uint64)[None, :], 0)]
        if kind == "ternary_p":
            return [X.counter(X.KIND_TERNARY_P, sd, sid, b, i, 0)]
        return [X.counter(X.KIND_GAUSSIAN, sd, sid, b, i, a) for a in range(3)]

    owner = {}
    for n, cs in enumerate(calls):
        for c in cs:
            for words in inputs(c):
                for t in zip(*(np.broadcast_to(w, np.broadcast(*words).shape).ravel().tolist() for w in words)):
                    assert owner.setdefault(t, n) == n, ("calls %d and %d share a Philox input" % (owner[t], n))


# ---- exact distributions of the restated streams -------------------------------------------------------------------------
def test_uniform_restatement_is_uniform():
    N = 1 << 12
    moduli = [H.ntt_prime(40, N, True), H.ntt_prime(55, N, False), H.Qi60[0], H.ntt_prime(30, N, False), H.ntt_prime(60, N, True)]
    v = X.uniform(7, 3, moduli, list(range(len(moduli))), 32, N)
    for r, q in enumerate(moduli):
        row = v[:, r].ravel()
        assert int(row.max()) < q
        p_bins, p_res = H.uniform_pvalues(row, q)
        assert p_bins > P_MIN and p_res > P_MIN, (hex(q), p_bins, p_res)


@pytest.mark.parametrize("p", [2.0 ** -20, 1 / 3, 0.5, 2 / 3, 1.0])
def test_ternary_p_restatement_follows_the_binomial(p):
    batch, N = 64, 1 << 14
    t = X.ternary_p(11, 5, batch, N, p)
    nz = int((t != 0).sum())
    pn = X.ternary_p_nonzero_probability(p)
    if p == 1.0:
        assert pn == 1.0 and nz == t.size
    else:
        assert binomtest(nz, t.size, pn).pvalue > P_MIN, (nz, t.size * pn)
    if nz:
        assert binomtest(int((t == 1).sum()), nz, 0.5).pvalue > P_MIN


def test_ternary_p_nonzero_probability_is_exact_at_53_bits():
    # u = k / 2^53 < p for exactly ceil(p 2^53) of the 2^53 words k
    for p in (2.0 ** -20, 1 / 3, 0.5, 2 / 3, 1.0, np.nextafter(1.0, 0.0), 2.0 ** -53, 3 * 2.0 ** -54):
        c = int(np.ceil(p * 2.0 ** 53))
        assert (c - 1) * 2.0 ** -53 < p <= c * 2.0 ** -53 or c == 0
        assert X.ternary_p_nonzero_probability(p) == c * 2.0 ** -53


@pytest.mark.parametrize("N,h,batch", [(1 << 10, 32, 2048), (1 << 10, 512, 256), (1 << 10, 1023, 256), (1 << 6, 70, 64)])
def test_ternary_h_restatement_is_uniform_over_positions(N, h, batch):
    t = X.ternary_h(13, 9, batch, N, h)
    hh = min(h, N)
    assert ((t != 0).sum(axis=1) == hh).all() and set(np.unique(t)) <= {-1, 0, 1}
    assert binomtest(int((t == 1).sum()), batch * hh, 0.5).pvalue > P_MIN
    if hh < N:
        # per polynomial the support is a uniform h-subset: Var(count_i) = batch s2, Cov = -batch s2 / (N - 1)
        counts = (t != 0).sum(axis=0)
        s2 = hh / N * (1 - hh / N)
        stat = (N - 1) / N * float(((counts - batch * hh / N) ** 2).sum()) / (batch * s2)
        assert chi2.sf(stat, N - 1) > P_MIN, stat


@pytest.mark.parametrize("sigma,bound,batch,N", [(3.2, 19.2, 64, 1 << 14), (0.5, 1.0, 64, 1 << 14), (1000.0, 1.5, 4, 1 << 12),
                                                 (2.0 ** 20, 6 * 2.0 ** 20, 64, 1 << 14)])
def test_gaussian_restatement_follows_the_truncated_discrete_law(sigma, bound, batch, N):
    v, m, att, near = X.gaussian_float64(17, 4, batch, N, sigma, bound)
    assert np.abs(v).max() <= np.floor(bound + 0.5) and (m <= bound).all()
    edges = H.gaussian_edges(bound)
    law = X.gaussian_law(sigma, bound, edges)
    counts = np.bincount(X.gaussian_bin_index(v.ravel(), edges), minlength=len(law))
    p = H.gof_pvalue(counts, law)
    assert p > P_MIN, (p, counts[:8], (law * v.size)[:8])
    assert near.sum() <= 2, int(near.sum())


def test_gaussian_float64_matches_mpmath():
    """The float64 m of the restatement against 50-digit arithmetic on the same exact (u1, u2)."""
    import mpmath
    mpmath.mp.dps = 50
    rng = np.random.default_rng(3)
    b = rng.integers(0, 8, 2000).astype(np.uint64)
    i = rng.integers(0, 1 << 16, 2000).astype(np.uint64)
    u1, u2, _ = X.gaussian_draws(5, 6, b, i, 0)
    # include the reduction's edge cases: u2 near a quarter, and u1 near 1
    u2 = np.concatenate([u2, [0.25, 0.25 - 2.0 ** -53, 0.75 + 2.0 ** -52, 0.5, 0.0, 0.125]])
    u1 = np.concatenate([u1, [1.0 - 2.0 ** -53, 2.0 ** -53, 0.5, 1.0 - 2.0 ** -40, 1e-3, 0.9]])
    m = X.gaussian_m(u1, u2, 1.0)
    for a, c, got in zip(u1, u2, m):
        want = mpmath.sqrt(-2 * mpmath.log(mpmath.mpf(a))) * abs(mpmath.cospi(2 * mpmath.mpf(c)))
        assert abs(mpmath.mpf(got) - want) <= 8 * 2.0 ** -53 * want, (a, c)

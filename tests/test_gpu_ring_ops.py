"""The ring-level kernels at every ring degree 2^4 .. 2^17, prime class and launch shape: every coefficient-wise opcode
(vecop_kernel), the automorphisms (auto_index / auto_ntt / auto_coeff / auto_coeff_ci kernels) and the coefficient-moving
kernels (shift, monomial, map_small_to_large, extend_small_norm, modup_centered).

Each result is checked bit for bit against the oracle and, where the inputs lie in the op's domain, against the exact
Python-integer reference of tests/ring_ops_cases.py (every word up to N = 2^12; above, the edge words, the first and last
64 words of each row and a stride of about 1/1000). Runs only on an H100 (-m gpu)."""
import ctypes
import functools
import itertools

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests import ring_ops_cases as C

pytestmark = pytest.mark.gpu
U64 = np.uint64
SENTINEL = 0x5A5A5A5A5A5A5A5A


def _lb():
    import lattigo_b200 as lb
    return lb


@pytest.fixture(scope="module")
def contexts():
    made = {}

    def get(logN, ci=False, Q=None, P=None):
        key = (logN, ci, tuple(Q or ()), tuple(P or ()))
        if key not in made:
            if Q is None:
                Q, P, _, _ = C.chain(logN, ci)
            made[key] = _lb().Context(logN, Q, P, ring_type=1 if ci else 0)
        return made[key]
    yield get
    for c in made.values():
        c.close()


def _sample_idx(n):
    """Word indices the exact reference sees: all of them up to 2^12, else the head (where the edge words sit), the
    first and last 64 words and a stride of about 1/1000."""
    if n <= 4096:
        return np.arange(n)
    return np.unique(np.concatenate([np.arange(256), np.arange(n - 64, n), np.arange(0, n, max(1, n // 1000))]))


@functools.lru_cache(maxsize=None)
def _combos(d1, d2, d3, q):
    w = lambda d: C.edge_words(d, q) if d != "-" else [0]
    return list(itertools.product(w(d1), w(d2), w(d3)))


def _operands(name, mods, lead, n, regime, rng, edge_k=None):
    """p1, p2, p3 of shape lead + (rows, n) and the per-row scalars. regime "any": any words and scalars (outside the
    domain included); "domain": words and scalars inside the op's domain, with its edge words at the head of each row.
    edge_k: every row takes edge scalar pair number edge_k (cycled) instead of a random draw."""
    d1, d2, d3, ds, _ = C.OPDOM[name]
    shape = tuple(lead) + (len(mods), n)
    p = [np.empty(shape, dtype=U64) for _ in range(3)]
    s0, s1 = [], []
    for i, q in enumerate(mods):
        for k, d in enumerate((d1, d2, d3)):
            p[k][..., i, :] = C.random_in("any" if regime == "any" or d == "-" else d, q, tuple(lead) + (n,), rng)
        if regime == "domain":
            combos = _combos(d1, d2, d3, q)[: max(1, n // 2)]
            for k in range(3):
                p[k][..., i, : len(combos)] = np.array([c[k] for c in combos], dtype=U64)
            sc = C.edge_scalars(ds, q)
            a, b = sc[edge_k % len(sc) if edge_k is not None else int(rng.integers(0, len(sc)))]
            if edge_k is None and ds not in ("mask", "-") and rng.integers(0, 2):
                a, b = int(rng.integers(0, q)), int(rng.integers(0, q))
        else:
            a, b = int(rng.integers(0, 1 << 64, dtype=U64)), int(rng.integers(0, 1 << 64, dtype=U64))
            if ds == "mask":
                a = int(rng.integers(0, 64))
        s0.append(a); s1.append(b)
    return p, s0, s1


def _check_exact(name, p1, p2, p3, got, s0, s1, mods):
    """got (rows, n) against the exact reference on the sampled words."""
    idx = _sample_idx(got.shape[-1])
    for i, q in enumerate(mods):
        for j in idx:
            err = C.check_exact(name, int(p1[i, j]), int(p2[i, j]), int(p3[i, j]), s0[i], s1[i], q, int(got[i, j]))
            assert err is None, (name, hex(q), i, int(j), err)


def _device(ctx, a, odd):
    """a on the device; odd: one word into its buffer (8-byte aligned only, which forces the scalar path)."""
    import torch
    if not odd:
        return ctx.to_device(a)
    flat = torch.zeros(a.size + 1, dtype=torch.int64, device="cuda")
    flat[1:].copy_(ctx.to_device(a.reshape(-1)))
    v = flat[1:].view(a.shape)
    assert v.data_ptr() % 16 == 8
    return v


def _run_ring(ctx, ring, name, lead, level, odd, regime, rng, edge_k=None):
    """One ring-level call at `level` (rows above it must stay untouched) against the oracle and the exact reference."""
    mods = ring.moduli
    N = ctx.N
    p, s0, s1 = _operands(name, mods, lead, N, regime, rng, edge_k)
    d1, d2, d3 = (_device(ctx, x, odd) for x in p)
    r = ring.AtLevel(level)
    r._vec(name, None if name == "Zero" else d1, d2, d3, s0[: level + 1], s1[: level + 1])
    got = ctx.to_host(d3)
    want = p[2].copy()
    o = O.Ring(N, mods).AtLevel(level)
    for b in np.ndindex(*lead):
        o._op(name, p[0][b], p[1][b], want[b], s0, s1)
    assert np.array_equal(got[..., : level + 1, :], want[..., : level + 1, :]), (name, regime, level, odd)
    assert np.array_equal(got[..., level + 1:, :], p[2][..., level + 1:, :]), (name, "rows above the level were written")
    if regime == "domain":
        first = (0,) * len(lead)
        _check_exact(name, p[0][first], p[1][first], p[2][first], got[first][: level + 1], s0, s1, mods[: level + 1])


@pytest.mark.parametrize("case", C.VEC_CASES, ids=lambda c: "%s-%s-%s-n%d" % (c[1], c[2], "N2^%d" % c[0], c[3]))
def test_vecop_launch_cells(case, contexts):
    """Every opcode on every prime class through the launch shape of one case (see ring_ops_cases.VEC_CASES)."""
    logN, entry, layout, n = case
    ctx = contexts(logN)
    odd = layout == "odd"
    Q, P, _, _ = C.chain(logN)
    rng = np.random.default_rng(logN * 1000 + n)
    for name in O.OPS:
        for regime in ("any", "domain"):
            if entry == "ring":
                _run_ring(ctx, ctx.ringQ, name, (3,), len(Q) - 1, odd, regime, rng)
                _run_ring(ctx, ctx.ringP, name, (), len(P) - 1, odd, regime, rng)
                if layout == "aligned":
                    _run_ring(ctx, ctx.ringQ, name, (1,), len(Q) - 3, odd, regime, rng)
                continue
            for which, mods in ((ctx.ringQ, Q), (ctx.ringP, P)):
                for limb, q in enumerate(mods):
                    p, s0, s1 = _operands(name, [q], (), n, regime, rng)
                    d = [_device(ctx, x[0], odd) for x in p]
                    which.SubRings[limb]._vec(name, None if name == "Zero" else d[0], d[1], d[2], s0[0], s1[0])
                    got = ctx.to_host(d[2])
                    want = p[2][0].copy()
                    O.get_subring(ctx.N, q).vecop(name, p[0][0], p[1][0], want, s0[0], s1[0])
                    assert np.array_equal(got, want), (name, regime, hex(q), n)
                    if regime == "domain":
                        _check_exact(name, p[0], p[1], p[2], got[None], s0, s1, [q])


@pytest.mark.parametrize("logN", [4, 6])
def test_vecop_every_edge_scalar(logN, contexts):
    """Every scalar opcode with every edge scalar pair (0, 1, q - 1 and their Montgomery forms; for Mask, shifts 0 and
    63 with the all-ones mask) on every prime class of both rings, in turn rather than by a random draw."""
    ctx = contexts(logN)
    Q, P, _, _ = C.chain(logN)
    rng = np.random.default_rng(77 + logN)
    for name in O.OPS:
        ds = C.OPDOM[name][3]
        if ds == "-":
            continue
        n_pairs = max(len(C.edge_scalars(ds, q)) for q in Q + P)
        for k in range(n_pairs):
            _run_ring(ctx, ctx.ringQ, name, (1,), len(Q) - 1, False, "domain", rng, edge_k=k)
            _run_ring(ctx, ctx.ringP, name, (), len(P) - 1, False, "domain", rng, edge_k=k)


def test_vecop_128_rows_and_batch_limits(contexts):
    """nQ + nP = 128 (P limb indices up to 127) for every opcode; batch 65535 at N = 2^4; batch 65536 refused before any
    launch; a context of 129 moduli refused when it is created."""
    lb = _lb()
    logN, N = 4, 16
    primes = C.ntt_primes(50, 2 * N, 129)
    Q, P = primes[:64], primes[64:128]
    ctx = contexts(logN, Q=Q, P=P)
    rng = np.random.default_rng(128)
    for name in O.OPS:
        for regime in ("any", "domain"):
            _run_ring(ctx, ctx.ringQ, name, (2,), 63, False, regime, rng)
            _run_ring(ctx, ctx.ringP, name, (2,), 63, False, regime, rng)
    one = contexts(logN, Q=[Q[0]], P=[P[0]])
    q = Q[0]
    batch = 65535                                              # one row per element: the flat arrays are one long oracle row
    x, y, z = (rng.integers(0, 1 << 64, (batch, 1, N), dtype=U64) for _ in range(3))
    x %= U64(q)
    d1, d2, d3 = one.to_device(x), one.to_device(y), one.to_device(z)
    n = H.launch_delta(lambda: one.ringQ.MulCoeffsMontgomeryThenAddLazy(d1, d2, d3))
    want = z.reshape(-1).copy()
    brc = np.array(O.gen_bred_constant(q), dtype=U64)
    O.lib().lo_vecop(O.OP["MulCoeffsMontgomeryThenAddLazy"], O._ptr(x.reshape(-1)), O._ptr(y.reshape(-1)), O._ptr(want), want.size, q,
                     O.gen_mred_constant(q), O._ptr(brc), 0, 0)
    assert np.array_equal(one.to_host(d3).reshape(-1), want)
    assert n == 1
    import torch
    big = torch.zeros((65536, 1, N), dtype=torch.int64, device="cuda")
    before = big.clone()
    with pytest.raises(lb.LgpuError):
        H.launch_delta(lambda: one.ringQ.Add(big, big, big))
    n0 = lb.lib().lgpu_launch_count()
    with pytest.raises(lb.LgpuError):
        one.ringQ.Neg(big, big)
    assert lb.lib().lgpu_launch_count() == n0
    assert torch.equal(big, before)
    with pytest.raises(lb.LgpuError, match="too many moduli"):
        lb.Context(logN, primes[:65], primes[65:129])


def _auto_chain(logN, ci):
    cp = C.class_primes(logN, ci)
    return [cp["b61"][0][0], cp["b45"][0][0], cp["smallest"][0][0]], [cp["b55"][1][0], cp["b33"][1][0]]


@pytest.mark.parametrize("ci", [False, True], ids=["standard", "conjugate_invariant"])
@pytest.mark.parametrize("logN", C.LOG_NS)
def test_automorphisms(logN, ci, contexts):
    lb = _lb()
    N = 1 << logN
    Q, P = _auto_chain(logN, ci)
    ctx = contexts(logN, ci, Q, P)
    nth = (4 if ci else 2) * N
    ring_o = O.Ring(N, Q, "ConjugateInvariant" if ci else "Standard")
    ringP_o = O.Ring(N, P, "ConjugateInvariant" if ci else "Standard")
    rng = np.random.default_rng(logN + 50 * ci)
    batch = 3
    x = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    x[:, :, : min(8, N // 2)] = 0                                  # negated zeros come out as q
    xp = H.rand_poly(P, N, rng)
    xp[:, ::5] = 0
    any_words = rng.integers(0, 1 << 64, (batch, len(Q), N), dtype=U64)
    near_top = (U64((1 << 64) - 1) - rng.integers(0, 1 << 40, (batch, len(Q), N), dtype=U64))
    dx, dxp, dany = ctx.to_device(x), ctx.to_device(xp), ctx.to_device(any_words)
    lg = (nth // 2).bit_length() - 1
    e = (2 * O._brev_table(lg)[:N] + 1).astype(np.int64)
    for g in C.galois_elements(N, ci):
        # coefficient domain, all rows and the whole batch: oracle, then the exact index and sign
        out = ctx.ringQ.NewPoly(batch)
        ctx.ringQ.Automorphism(dx, g, out)
        got = ctx.to_host(out)
        want = np.zeros_like(x)
        for b in range(batch):
            ring_o.Automorphism(x[b], g, want[b])
        assert np.array_equal(got, want), g
        assert np.array_equal(got, C.automorphism_exact_np(x, g, Q, ci)), g
        if N <= 4096:
            for i, q in enumerate(Q):
                assert [int(v) for v in got[0, i]] == C.automorphism_exact(x[0, i], g, q, ci), (g, i)
        # lower level: rows above it untouched
        lo = ctx.to_device(np.full((batch, len(Q), N), SENTINEL, dtype=U64))
        ctx.ringQ.AtLevel(0).Automorphism(dx, g, lo)
        gl = ctx.to_host(lo)
        assert np.array_equal(gl[:, :1], want[:, :1]) and np.all(gl[:, 1:] == U64(SENTINEL)), g
        # ringP
        op = ctx.ringP.NewPoly()
        ctx.ringP.Automorphism(dxp, g, op)
        wp = np.zeros_like(xp)
        ringP_o.Automorphism(xp, g, wp)
        assert np.array_equal(ctx.to_host(op), wp), g
        assert np.array_equal(ctx.to_host(op), C.automorphism_exact_np(xp, g, P, ci)), g
        # NTT index: oracle, and the defining property e[idx[j]] = g * e[j] mod NthRoot
        didx = ctx.ringQ.AutomorphismNTTIndex(g)
        idx = ctx.to_host(didx)
        assert np.array_equal(idx, ring_o.AutomorphismNTTIndex(g)), g
        assert np.array_equal(e[idx.astype(np.int64)], (g * e) % nth), g
        if N <= 4096:
            assert [int(v) for v in idx] == C.ntt_index_exact(N, nth, g), g
        # NTT-domain permutations on any words, batch 3, a lower level, ringP, and the lazy accumulation near 2^64
        oidx = ring_o.AutomorphismNTTIndex(g)
        want_n = np.zeros_like(any_words)
        for b in range(batch):
            ring_o.AutomorphismNTTWithIndex(any_words[b], oidx, want_n[b])
        o1 = ctx.ringQ.NewPoly(batch)
        ctx.ringQ.AutomorphismNTT(dany, g, o1)
        assert np.array_equal(ctx.to_host(o1), want_n), g
        o2 = ctx.to_device(np.full((batch, len(Q), N), SENTINEL, dtype=U64))
        ctx.ringQ.AtLevel(1).AutomorphismNTTWithIndex(dany, didx, o2)
        g2 = ctx.to_host(o2)
        assert np.array_equal(g2[:, :2], want_n[:, :2]) and np.all(g2[:, 2:] == U64(SENTINEL)), g
        acc = ctx.to_device(near_top)
        ctx.ringQ.AutomorphismNTTWithIndexThenAddLazy(dany, didx, acc)
        want_acc = near_top.copy()
        for b in range(batch):
            ring_o.AutomorphismNTTWithIndexThenAddLazy(any_words[b], oidx, want_acc[b])
        assert np.array_equal(ctx.to_host(acc), want_acc), g
        assert np.array_equal(want_acc, near_top + any_words[..., idx.astype(np.int64)]), g      # wraps mod 2^64, like the reference
        accp = ctx.to_device(near_top[0, :2].copy())
        ctx.ringP.AutomorphismNTTWithIndexThenAddLazy(dany[0, :2].contiguous(), didx, accp)
        assert np.array_equal(ctx.to_host(accp), near_top[0, :2] + any_words[0, :2][:, idx.astype(np.int64)]), g
        # identities that do not use the oracle: INTT(AutomorphismNTT(NTT(a))) = Automorphism(a), sigma_h(sigma_g) = sigma_gh
        t = ctx.ringQ.NewPoly(batch); u = ctx.ringQ.NewPoly(batch)
        ctx.ringQ.NTT(dx, t)
        ctx.ringQ.AutomorphismNTT(t, g, u)
        ctx.ringQ.INTT(u, t)
        mods = np.array(Q, dtype=U64)[None, :, None]
        assert np.array_equal(ctx.to_host(t) % mods, got % mods), g
        for h in (C.GALOIS_GEN, nth - 1) if not ci else (C.GALOIS_GEN,):
            twice = ctx.ringQ.NewPoly(batch); once = ctx.ringQ.NewPoly(batch)
            ctx.ringQ.Automorphism(out, h, twice)
            ctx.ringQ.Automorphism(dx, g * h % nth, once)
            mods = np.array(Q, dtype=U64)[None, :, None]
            assert np.array_equal(ctx.to_host(twice) % mods, ctx.to_host(once) % mods), (g, h)


MONO_K = lambda N: (0, 1, 17, N - 1, N, N + 3, 2 * N - 1, -1, -N, -N - 9, -2 * N + 1, 2 * N, 3 * N + 5)
SHIFT_K = lambda N: (0, 1, 5, N - 1, N, N + 2, -1, -3 * N - 4)


@pytest.mark.parametrize("logN", C.LOG_NS)
def test_coefficient_moves(logN, contexts):
    lb = _lb()
    N = 1 << logN
    Q, P = _auto_chain(logN, False)
    ctx = contexts(logN, False, Q, P)
    rng = np.random.default_rng(900 + logN)
    batch = 2
    x = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    x[0, :, :7] = 0
    x[1, :, N - 5:] = 0
    dx = ctx.to_device(x)
    lvl = ctx.ringQ.AtLevel(1)                                   # batch stride 3N, larger than the level's 2 rows
    ring_o = O.Ring(N, Q).AtLevel(1)
    for op, ks, exact in (("MultByMonomial", MONO_K(N), lambda a, k: C.monomial_exact_np(a, k, Q[:2])),
                          ("Shift", SHIFT_K(N), lambda a, k: C.shift_exact_np(a, k % N))):
        for k in ks:
            want = exact(x[:, :2], k)
            wo = np.zeros((batch, 2, N), dtype=U64)
            for b in range(batch):
                tmp = np.zeros((3, N), dtype=U64)
                getattr(ring_o, op)(x[b][:2], k, tmp)
                wo[b] = tmp[:2]
            assert np.array_equal(wo, want), (op, k)
            out = ctx.to_device(np.full((batch, 3, N), SENTINEL, dtype=U64))
            getattr(lvl, op)(dx, k, out)
            got = ctx.to_host(out)
            assert np.array_equal(got[:, :2], want) and np.all(got[:, 2] == U64(SENTINEL)), (op, k)
            e = dx.clone()
            getattr(lvl, op)(e, k, e)                              # in place: the copy must honour the batch stride
            ge = ctx.to_host(e)
            assert np.array_equal(ge[:, :2], want) and np.array_equal(ge[:, 2], x[:, 2]), (op, k, "in place")
    # MapSmallDimensionToLargerDimensionNTT at every ratio 1 .. N/16, several rows
    for lg_ratio in range(0, logN - 3):
        ns = N >> lg_ratio
        small = rng.integers(0, 1 << 64, (3, ns), dtype=U64)
        large = ctx.to_device(np.zeros((3, N), dtype=U64))
        lb.ring.MapSmallDimensionToLargerDimensionNTT(ctx, ctx.to_device(small), large)
        assert np.array_equal(ctx.to_host(large), np.repeat(small, 1 << lg_ratio, axis=1)), lg_ratio
    # ExtendBasisSmallNormAndCenter: the +-Q/2 boundary and Q - 1, to every P prime
    Q0 = Q[0]
    h = Q0 >> 1
    pin = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    edges = np.array([0, 1, h - 1, h, h + 1, Q0 - 1, Q0 - 2], dtype=U64)
    pin[:, 0, : min(N, len(edges))] = edges[: min(N, len(edges))]
    pin[1, 0, len(edges): N // 2] = (rng.integers(-40, 41, N // 2 - len(edges)) % Q0).astype(U64)      # small norm, both signs
    rqp = lb.RingQP(ctx)
    oq, op = ctx.ringQ.NewPoly(batch), ctx.ringP.NewPoly(batch)
    rqp.ExtendBasisSmallNormAndCenter(ctx.to_device(pin), len(P) - 1, oq, op)
    gp = ctx.to_host(op)
    c = pin[:, 0]
    neg = c > U64(h)
    for i, p in enumerate(P):
        want = np.where(neg, U64(p) - (U64(Q0) - c), c)            # literal word (wraps when |c| > p, like the reference)
        assert np.array_equal(gp[:, i], want), i
        assert [int(v) for v in gp[0, i, : len(edges)]] == [C.extend_exact(int(v), Q0, p) for v in c[0, : len(edges)]]
    wq, wp = np.zeros((3, N), dtype=U64), np.zeros((2, N), dtype=U64)
    O.ExtendBasisSmallNormAndCenter(O.Ring(N, Q), O.Ring(N, P), pin[0], len(P) - 1, wq, wp)
    assert np.array_equal(gp[0], wp)


def _modup(ctx, d_in, first_q, level_q, level_p, strict, out_q, out_p, batch, s_in, s_q, s_p):
    from lattigo_b200 import _lib
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(_lib.lib().lgpu_modup_centered(ctx.h, ptr(d_in), first_q, level_q, level_p, strict, ptr(out_q), ptr(out_p), batch, s_in, s_q, s_p, None))


@pytest.mark.parametrize("logN", [4, 10, 16])
def test_modup_centered(logN, contexts):
    """strict 0 / 1 at exactly q0/2 and q0/2 + 1, targets far below q0/2 (so the reduction is real), first_q 0 and 1,
    level_p = -1, batch strides wider than the rows written."""
    import torch
    N = 1 << logN
    Q, P = _auto_chain(logN, False)
    ctx = contexts(logN, False, Q, P)
    q0, h = Q[0], Q[0] >> 1
    rng = np.random.default_rng(logN)
    batch = 3
    x = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    edges = np.array([0, 1, h - 1, h, h + 1, h + 2, q0 - 1, q0 - Q[2], q0 - 2 * Q[2], Q[2], P[1]], dtype=U64)
    x[:, 0, : len(edges)] = edges
    d = ctx.to_device(x)
    for strict in (0, 1):
        for first_q, level_p in ((0, 1), (1, 1), (1, -1), (0, 0)):
            oq = torch.zeros((batch, 4, N), dtype=torch.int64, device="cuda")
            op = torch.zeros((batch, 3, N), dtype=torch.int64, device="cuda") if level_p >= 0 else None
            _modup(ctx, d, first_q, 2, level_p, strict, oq, op, batch, 3 * N, 4 * N, 3 * N)
            gq = ctx.to_host(oq)
            c = x[:, 0]
            neg = c > U64(h) if strict else c >= U64(h)
            mag = np.where(neg, U64(q0) - c, c)
            for i, t in enumerate(Q):
                if i < first_q:
                    assert not gq[:, i].any(), (strict, first_q, i)
                    continue
                m = mag % U64(t)
                assert np.array_equal(gq[:, i], np.where(neg, U64(t) - m, m)), (strict, first_q, i)
                assert [int(v) for v in gq[0, i, : len(edges)]] == [C.modup_centered_exact(int(v), q0, t, strict) for v in edges]
            assert not gq[:, 3].any()
            if op is not None:
                gp = ctx.to_host(op)
                for i, t in enumerate(P[: level_p + 1]):
                    m = mag % U64(t)
                    assert np.array_equal(gp[:, i], np.where(neg, U64(t) - m, m)), (strict, level_p, i)
                    assert [int(v) for v in gp[0, i, : len(edges)]] == [C.modup_centered_exact(int(v), q0, t, strict) for v in edges]
                assert not gp[:, level_p + 1:].any()


@pytest.mark.parametrize("logN", [8, 16])
def test_scalar_wrappers(logN, contexts):
    """Ring.AddScalar / SubScalar / MulScalar / MulScalarThenAdd / MulScalarThenSub with scalars >= 2^128 and negative
    scalars; the *DoubleRNSScalar family, whose halves split at N/2 (at N = 2^16 each half is a 2^15-word SubRing call)."""
    N = 1 << logN
    Q, P = _auto_chain(logN, False)
    ctx = contexts(logN, False, Q, P)
    ring_o = O.Ring(N, Q)
    rng = np.random.default_rng(logN + 7)
    x = H.rand_poly(Q, N, rng)
    z = H.rand_poly(Q, N, rng)
    idx = _sample_idx(N)
    exact = {"AddScalar": lambda a, s, w, q: (a + s) % q, "SubScalar": lambda a, s, w, q: (a - s) % q,
             "MulScalar": lambda a, s, w, q: a * s % q, "MulScalarThenAdd": lambda a, s, w, q: (w + a * s) % q,
             "MulScalarThenSub": lambda a, s, w, q: (w - a * s) % q}
    for s in ((1 << 130) + 12345, -5, -(1 << 140) - 3, (1 << 128), 0):
        for meth, f in exact.items():
            out = ctx.to_device(z)
            getattr(ctx.ringQ, meth)(ctx.to_device(x), s, out)
            got = ctx.to_host(out)
            want = z.copy()
            getattr(ring_o, meth)(x, s, want)
            assert np.array_equal(got, want), (meth, s)
            for i, q in enumerate(Q):
                for j in idx:
                    assert int(got[i, j]) == f(int(x[i, j]), s, int(z[i, j]), q), (meth, s, i, int(j))
    s0 = [int(rng.integers(0, q)) for q in Q]
    s1 = [int(rng.integers(0, q)) for q in Q]
    s0[0], s1[0] = 0, Q[0] - 1
    h = N // 2
    for meth, f in (("AddDoubleRNSScalar", lambda a, s, w, q: (a + s) % q), ("SubDoubleRNSScalar", lambda a, s, w, q: (a - s) % q),
                    ("MulDoubleRNSScalar", lambda a, s, w, q: a * s % q), ("MulDoubleRNSScalarThenAdd", lambda a, s, w, q: (w + a * s) % q)):
        out = ctx.to_device(z)
        getattr(ctx.ringQ, meth)(ctx.to_device(x), s0, s1, out)
        got = ctx.to_host(out)
        want = z.copy()
        getattr(ring_o, meth)(x, s0, s1, want)
        assert np.array_equal(got, want), meth
        for i, q in enumerate(Q):
            for j in np.unique(np.concatenate([idx, [h - 1, h]])):
                s = s0[i] if j < h else s1[i]
                assert int(got[i, j]) == f(int(x[i, j]), s, int(z[i, j]), q), (meth, i, int(j))

"""The oracle's C restatement of the ring-level kernels against the exact reference of tests/ring_ops_cases.py (no GPU):
every opcode of lo_vecop at every prime class and every edge word of its domain; MultByMonomial, Shift, Automorphism,
AutomorphismNTTIndex, MapSmallDimensionToLargerDimensionNTT and ExtendBasisSmallNormAndCenter at small degrees on both
ring types. This pins the oracle independently of the kernels it checks. Also: the GPU case list of
tests/test_gpu_ring_ops.py reaches every launch-shape cell, and no case in it is spare."""
import itertools

import numpy as np
import pytest

from oracle import oracle as O
from tests import ring_ops_cases as C

U64 = np.uint64


def _class_moduli():
    """Every prime of every class, at the degrees where its class changes (2^4, 2^10, 2^12, 2^17), both ring types."""
    out = {}
    for lg, ci in ((4, False), (10, False), (12, False), (17, False), (17, True)):
        for c, (qs, ps) in C.class_primes(lg, ci).items():
            for q in qs + ps:
                out[q] = c
    return sorted(out.items())


MODULI = _class_moduli()


@pytest.mark.parametrize("name", O.OPS)
def test_lo_vecop_matches_exact_reference_on_edge_words(name):
    d1, d2, d3, ds, _ = C.OPDOM[name]
    for q, cls in MODULI:
        brc = np.array(O.gen_bred_constant(q), dtype=U64)
        qinv = O.gen_mred_constant(q)
        w1 = C.edge_words(d1, q) if d1 != "-" else [0]
        w2 = C.edge_words(d2, q) if d2 != "-" else [0]
        w3 = C.edge_words(d3, q) if d3 != "-" else [0]
        combos = list(itertools.product(w1, w2, w3))
        x = np.array([c[0] for c in combos], dtype=U64)
        y = np.array([c[1] for c in combos], dtype=U64)
        for s0, s1 in C.edge_scalars(ds, q):
            z = np.array([c[2] for c in combos], dtype=U64)
            rc = O.lib().lo_vecop(O.OP[name], O._ptr(x) if d1 != "-" else None, O._ptr(y) if d2 != "-" else None, O._ptr(z), len(combos),
                                  q, qinv, O._ptr(brc), s0, s1)
            assert rc == 0
            bad = []
            for (a, b, c), got in zip(combos, z):
                err = C.check_exact(name, a, b, c, s0, s1, q, int(got))
                if err:
                    bad.append((a, b, c, err))
            assert not bad, (name, cls, hex(q), s0, s1, bad[:4])


@pytest.mark.parametrize("name", O.OPS)
def test_lo_vecop_matches_exact_reference_on_random_words(name):
    """Random words inside the domain, 256 per class prime (the edge test above sees only the corners)."""
    d1, d2, d3, ds, _ = C.OPDOM[name]
    rng = np.random.default_rng(O.OP[name])
    for q, cls in MODULI:
        brc = np.array(O.gen_bred_constant(q), dtype=U64)
        x = C.random_in(d1 if d1 != "-" else "q", q, 256, rng)
        y = C.random_in(d2 if d2 != "-" else "q", q, 256, rng)
        z0 = C.random_in(d3 if d3 != "-" else "q", q, 256, rng)
        if ds == "mask":
            s0, s1 = int(rng.integers(0, 64)), int(rng.integers(0, 1 << 64, dtype=U64))
        else:
            s0, s1 = int(rng.integers(0, q)), int(rng.integers(0, q))
        z = z0.copy()
        O.lib().lo_vecop(O.OP[name], O._ptr(x), O._ptr(y), O._ptr(z), 256, q, O.gen_mred_constant(q), O._ptr(brc), s0, s1)
        for i in range(256):
            err = C.check_exact(name, int(x[i]), int(y[i]), int(z0[i]), s0, s1, q, int(z[i]))
            assert err is None, (name, cls, hex(q), i, err)


def test_edge_words_and_scalars():
    q = 0x3001
    assert C.edge_words("q", q) == [0, 1, q - 1]
    assert C.edge_words("2q", q) == [0, 1, q - 1, q, 2 * q - 1]
    assert C.edge_words("any", q)[-2:] == [1 << 63, (1 << 64) - 1]
    assert (63, (1 << 64) - 1) in C.edge_scalars("mask", q)
    assert (1, (1 << 64) % q) in C.edge_scalars("q", q)


@pytest.mark.parametrize("logN", [4, 5, 6, 7, 8])
def test_oracle_monomial_and_shift_match_exact(logN):
    N = 1 << logN
    Q = C.chain(logN)[0][:3]
    ring = O.Ring(N, Q)
    rng = np.random.default_rng(logN)
    x = np.stack([rng.integers(0, q, N, dtype=U64) for q in Q])
    x[:, :3] = 0
    for k in (0, 1, 17, N - 1, N, N + 3, 2 * N - 1, -1, -N, -N - 9, -2 * N + 1, 2 * N, 3 * N + 5):
        got = np.zeros_like(x)
        ring.MultByMonomial(x, k, got)
        for i, q in enumerate(Q):
            assert [int(v) for v in got[i]] == C.monomial_exact(x[i], k, q), (k, i)
        assert np.array_equal(C.monomial_exact_np(x, k, Q), got), k
        got = np.zeros_like(x)
        ring.Shift(x, k, got)
        for i in range(len(Q)):
            assert [int(v) for v in got[i]] == [int(x[i][(j + k) % N]) for j in range(N)], (k, i)
        assert np.array_equal(C.shift_exact_np(x, k % N), got)


@pytest.mark.parametrize("logN", range(4, 13))
@pytest.mark.parametrize("ci", [False, True], ids=["standard", "conjugate_invariant"])
def test_oracle_automorphisms_match_exact(logN, ci):
    """Ring.Automorphism and AutomorphismNTTIndex at N = 2^4 .. 2^12 on both ring types, every Galois element of the GPU
    suite, against the index and sign written out from X -> X^g."""
    N = 1 << logN
    Q = [C.class_primes(logN, ci)["b61"][0][0], C.class_primes(logN, ci)["smallest"][0][0]]
    ring = O.Ring(N, Q, "ConjugateInvariant" if ci else "Standard")
    nth = ring.NthRoot()
    rng = np.random.default_rng(logN + 100 * ci)
    x = np.stack([rng.integers(0, q, N, dtype=U64) for q in Q])
    x[:, 0] = 0
    x[:, N - 1] = 0
    for g in C.galois_elements(N, ci):
        got = np.zeros_like(x)
        ring.Automorphism(x, g, got)
        want = C.automorphism_exact_np(x, g, Q, ci)
        assert np.array_equal(got, want), g
        if logN <= 8:
            for i, q in enumerate(Q):
                assert [int(v) for v in got[i]] == C.automorphism_exact(x[i], g, q, ci), (g, i)
        idx = ring.AutomorphismNTTIndex(g)
        assert [int(v) for v in idx] == C.ntt_index_exact(N, nth, g), g


@pytest.mark.parametrize("logN", [4, 6, 8])
def test_ntt_slot_order_is_the_evaluation_order(logN):
    """The slot exponents ntt_index_exact relies on: NTT(X)[j] = psi^(2 brev(j) + 1), with psi the 2N-th root the oracle's
    tables are built from, and NTT(a)[j] = a(psi^e_j) for a random a (both ring types)."""
    N = 1 << logN
    for ci in (False, True):
        q = C.class_primes(logN, ci)["b45"][0][0]
        sr = O.SubRing(N, q, ring_type="ConjugateInvariant" if ci else "Standard")
        psi = pow(sr.PrimitiveRoot, (q - 1) // sr.NthRoot, q)
        e = C.ntt_slot_exponents(N, sr.NthRoot)
        rng = np.random.default_rng(logN)
        a = rng.integers(0, q, N, dtype=U64)
        out = np.empty(N, dtype=U64)
        sr.NTT(a, out)
        if not ci:
            want = [sum(int(a[i]) * pow(psi, i * ej, q) for i in range(N)) % q for ej in e]
        else:   # a_0 + sum_{i>0} a_i (X^i + X^-i) at X = psi^e (the element is invariant under X -> X^-1)
            want = [(int(a[0]) + sum(int(a[i]) * (pow(psi, i * ej, q) + pow(psi, (sr.NthRoot - i) * ej % sr.NthRoot, q)) for i in range(1, N))) % q
                    for ej in e]
        assert [int(v) for v in out] == want, ci


def test_oracle_map_and_extend_match_exact():
    rng = np.random.default_rng(3)
    for logN in (4, 7, 10):
        N = 1 << logN
        for ratio in [1 << k for k in range(0, logN - 3)]:
            small = rng.integers(0, 1 << 64, (3, N // ratio), dtype=U64)
            large = np.zeros((3, N), dtype=U64)
            O.MapSmallDimensionToLargerDimensionNTT(small, large)
            assert all(int(large[r, c]) == int(small[r, c // ratio]) for r in range(3) for c in range(N))
    Q, P, _, _ = C.chain(6)
    N = 64
    ringQ, ringP = O.Ring(N, Q), O.Ring(N, P)
    Q0 = Q[0]
    edges = [0, 1, Q0 // 2 - 1, Q0 // 2, Q0 // 2 + 1, Q0 - 1]
    x = np.stack([rng.integers(0, q, N, dtype=U64) for q in Q])
    x[0, : len(edges)] = edges
    oq, op = np.zeros_like(x), np.zeros((len(P), N), dtype=U64)
    O.ExtendBasisSmallNormAndCenter(ringQ, ringP, x, len(P) - 1, oq, op)
    for i, p in enumerate(P):
        assert [int(v) for v in op[i]] == [C.extend_exact(int(c), Q0, p) for c in x[0]], i


def test_exact_maps_are_ring_automorphisms():
    """Self-checks of the reference: sigma_h(sigma_g(a)) = sigma_gh(a) mod q; sigma_g(a*b) = sigma_g(a) sigma_g(b) for
    negacyclic products; X^k X^l = X^(k+l)."""
    N, q = 16, 97
    rng = np.random.default_rng(0)

    def mul(a, b):
        out = [0] * N
        for i in range(N):
            for j in range(N):
                k = i + j
                if k < N:
                    out[k] += a[i] * b[j]
                else:
                    out[k - N] -= a[i] * b[j]
        return [v % q for v in out]

    a = [int(v) for v in rng.integers(0, q, N)]
    b = [int(v) for v in rng.integers(0, q, N)]
    for g in (3, 5, 25, 31):
        for h in (5, 7, 31):
            lhs = [v % q for v in C.automorphism_exact(C.automorphism_exact(a, g, q), h, q)]
            assert lhs == [v % q for v in C.automorphism_exact(a, g * h % (2 * N), q)]
        assert [v % q for v in C.automorphism_exact(mul(a, b), g, q)] == \
            mul([v % q for v in C.automorphism_exact(a, g, q)], [v % q for v in C.automorphism_exact(b, g, q)])
    for k in (1, 5, N + 3):
        xk = [0] * N
        xk[k % N] = 1 if k < N else q - 1
        assert [v % q for v in C.monomial_exact(a, k, q)] == mul(a, xk)
    # conjugate-invariant: the image is again invariant, and composition holds
    for g in (5, 25, 125 % 64):
        for h in (5, 13):
            lhs = [v % q for v in C.automorphism_exact(C.automorphism_exact(a, g, q, True), h, q, True)]
            assert lhs == [v % q for v in C.automorphism_exact(a, g * h % (4 * N), q, True)]


def test_centred_lifts():
    q0 = 0x1fffffffffe00001
    h = q0 >> 1
    assert C.modup_centered_exact(h, q0, 97, 0) == 97 - (q0 - h) % 97
    assert C.modup_centered_exact(h, q0, 97, 1) == h % 97
    assert C.modup_centered_exact(h + 1, q0, 97, 1) == 97 - (q0 - h - 1) % 97
    assert C.modup_centered_exact(q0 - 97, q0, 97, 0) == 97           # -97 mod 97 is written as 97
    assert C.extend_exact(q0 - 1, q0, 257) == 256 and C.extend_exact(h, q0, 257) == h


def test_launch_shape_restatement():
    assert C.launch_shape(1 << 10, True) == (2, 2, 1, "one")
    assert C.launch_shape(1 << 15, True) == (2, 64, 1, "one")
    assert C.launch_shape(1 << 16, True) == (2, 32, 4, "several")
    assert C.launch_shape(1 << 15, False) == (1, 32, 4, "several")
    assert C.launch_shape(2 * (256 * 65 + 17), True)[1:] == (17, 4, "ragged")
    assert C.launch_shape(256 * 65 + 1, False)[1:] == (17, 4, "ragged")
    assert C.launch_shape(1001, C.vec2(1001, True)) == (1, 4, 1, "one")
    assert not C.vec2(1001, True) and not C.vec2(1000, False) and C.vec2(1000, True)


def test_cases_reach_every_cell():
    missing = C.required_cells() - C.reached_cells(C.VEC_CASES)
    assert not missing, sorted(missing, key=str)[:20]


def test_removing_a_case_leaves_a_cell():
    req = C.required_cells()
    for case in C.VEC_CASES:
        rest = [c for c in C.VEC_CASES if c != case]
        assert req - C.reached_cells(rest), case


def test_required_cells_do_not_depend_on_the_cases(monkeypatch):
    """The required set is the same whatever the case list holds, so deleting a case (the one ragged 128-bit case
    included) makes test_cases_reach_every_cell fail."""
    req = C.required_cells()
    assert any(c[:3] == (2, "ragged", "subring") for c in req)
    for case in C.VEC_CASES:
        rest = [c for c in C.VEC_CASES if c != case]
        monkeypatch.setattr(C, "VEC_CASES", rest)
        assert C.required_cells() == req, case
        assert req - C.reached_cells(rest), case
    monkeypatch.undo()
    ragged2 = [c for c in C.VEC_CASES if c[1] == "subring" and C.launch_shape(c[3], C.vec2(c[3], c[2] == "aligned"))[::3] == (2, "ragged")]
    assert len(ragged2) == 1
    assert {c for c in req if c[:3] == (2, "ragged", "subring")} - C.reached_cells([c for c in C.VEC_CASES if c not in ragged2])

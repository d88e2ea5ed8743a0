"""GPU parity (bit-exact) of the ring-level C ABI against the oracle: NTT / INTT (canonical and exact-lazy),
every coefficient-wise opcode, batches, in-place. Runs only on an H100 (-m gpu)."""
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64
HERE = os.path.dirname(os.path.abspath(__file__))


def _lb():
    import lattigo_b200 as lb
    return lb


def test_golden_vectors_through_gpu():
    """The reference's own KAT (ring/ntt_test.go:10-119) through the CUDA kernels."""
    lb = _lb()
    vecs = json.load(open(os.path.join(HERE, "golden", "ntt_vectors.json")))["vectors"]
    for v in vecs:
        logN = v["N"].bit_length() - 1
        ctx = lb.Context(logN, v["Qis"])
        poly = np.array(v["poly"], dtype=U64)
        want = np.array(v["polyNTT"], dtype=U64)
        d = ctx.to_device(poly)
        out = ctx.ringQ.NewPoly()
        ctx.ringQ.NTT(d, out)
        assert np.array_equal(ctx.to_host(out), want), v["N"]
        back = ctx.ringQ.NewPoly()
        ctx.ringQ.INTT(out, back)
        assert np.array_equal(ctx.to_host(back), poly), v["N"]
        ctx.close()


@pytest.mark.parametrize("primes", ["q61", "q45_56"])
@pytest.mark.parametrize("logN", [4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17])
def test_ntt_matches_oracle_all_sizes(logN, primes):
    """Covers every chunk-size instantiation and every strided radix (C1 is logN=12), with 61-bit primes (lazy
    corrections every other stage, corrected inverse) and with CKKS-sized 45/55/56-bit primes (no forward
    correction at all, correction-free inverse for the 45-bit ones)."""
    lb = _lb()
    N = 1 << logN
    if primes == "q61":
        Q = H.Qi60[:3]
    else:
        q, p = O.gen_moduli(logN + 1, [56, 45, 45], [55])
        Q = [q[1], q[0], p[0]]
    ctx = lb.Context(logN, Q)
    ring = O.Ring(N, Q)
    rng = np.random.default_rng(100 + logN)
    batch = 2
    x = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    want = np.empty_like(x); want_lazy = np.empty_like(x); want_inv = np.empty_like(x)
    for b in range(batch):
        ring.NTT(x[b], want[b]); ring.NTTLazy(x[b], want_lazy[b]); ring.INTT(x[b], want_inv[b])
    d = ctx.to_device(x)
    out = ctx.ringQ.NewPoly(batch)
    ctx.ringQ.NTT(d, out)
    assert np.array_equal(ctx.to_host(out), want)
    ctx.ringQ.NTTLazy(d, out)
    assert np.array_equal(ctx.to_host(out), want_lazy)          # exact lazy representative in [0, 6q)
    ctx.ringQ.INTT(d, out)
    assert np.array_equal(ctx.to_host(out), want_inv)
    ctx.ringQ.INTTLazy(d, out)
    assert np.array_equal(ctx.to_host(out), want_inv)           # INTTLazy is fully reduced for N >= 16
    # in place + round trip
    e = d.clone()
    ctx.ringQ.NTT(e, e)
    assert np.array_equal(ctx.to_host(e), want)
    ctx.ringQ.INTT(e, e)
    assert np.array_equal(ctx.to_host(e), x)
    # level < max and single rows
    lvl = ctx.ringQ.AtLevel(0)
    o1 = ctx.new_poly(1)
    lvl.NTT(d[0], o1)
    assert np.array_equal(ctx.to_host(o1)[0], want[0][0])
    sr = ctx.ringQ.SubRings[2]
    row = ctx.to_device(x[1][2].copy())
    sr.NTTLazy(row, row)
    assert np.array_equal(ctx.to_host(row), want_lazy[1][2])
    ctx.close()


def test_ntt_ring_p_and_error_paths():
    lb = _lb()
    Q, P = H.Qi60[:2], H.Pi60[:2]
    ctx = lb.Context(10, Q, P)
    ring = O.Ring(1024, P)
    rng = np.random.default_rng(5)
    x = H.rand_poly(P, 1024, rng)
    want = np.empty_like(x); ring.NTT(x, want)
    out = ctx.ringP.NewPoly()
    ctx.ringP.NTT(ctx.to_device(x), out)
    assert np.array_equal(ctx.to_host(out), want)
    with pytest.raises(lb.LgpuError):
        ctx.ringQ.AtLevel(5)
    with pytest.raises(lb.LgpuError):
        lb.Context(10, [Q[0], Q[0]])                      # moduli not distinct (ring/ring.go:270)
    with pytest.raises(lb.LgpuError):
        lb.Context(10, [0x1fffffffffe00001 + 2])          # not prime / not NTT friendly
    ctx.close()


SCALARS = {
    "AddLazyThenMulScalarMontgomery": 1, "AddScalarLazyThenMulScalarMontgomery": 2, "AddScalar": 1, "AddScalarLazy": 1,
    "AddScalarLazyThenNegTwoModulusLazy": 1, "SubScalar": 1, "MulScalarMontgomery": 1, "MulScalarMontgomeryLazy": 1,
    "MulScalarMontgomeryThenAdd": 1, "MulScalarMontgomeryThenAddScalar": 2, "SubThenMulScalarMontgomeryTwoModulus": 1, "Mask": 2,
}


@pytest.mark.parametrize("name", O.OPS)
def test_vecop_matches_oracle(name):
    """Every kernel of ring/vec_ops.go: ring-level (all limbs, batch 2) and SubRing-level (one row, ragged n)."""
    lb = _lb()
    logN, N = 10, 1024
    Q = H.Qi60[:3]
    ctx = lb.Context(logN, Q)
    ring = O.Ring(N, Q)
    rng = np.random.default_rng(abs(hash(name)) % 2**31)
    batch = 2
    mk = lambda: np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    p1, p2, p3 = mk(), mk(), mk()
    if name in ("Reduce", "ReduceLazy", "MForm", "MFormLazy"):      # accept any a < 2^64
        p1 = rng.integers(0, 2**64, p1.shape, dtype=U64)
    ns = SCALARS.get(name, 0)
    if name == "Mask":
        s0 = [7] * len(Q); s1 = [0xFFFF] * len(Q)
    else:
        s0 = [int(rng.integers(0, q)) for q in Q] if ns >= 1 else None
        s1 = [int(rng.integers(0, q)) for q in Q] if ns >= 2 else None
    want = p3.copy()
    for b in range(batch):
        ring._op(name, p1[b], p2[b], want[b], s0, s1)
    d1, d2, d3 = ctx.to_device(p1), ctx.to_device(p2), ctx.to_device(p3)
    ctx.ringQ._vec(name, d1, d2, d3, s0, s1)
    assert np.array_equal(ctx.to_host(d3), want), name
    # SubRing-level, ragged length (not a multiple of the vector width) on limb 1
    n = 1001
    r1 = ctx.to_device(p1[0][1][:n].copy()); r2 = ctx.to_device(p2[0][1][:n].copy()); r3 = ctx.to_device(p3[0][1][:n].copy())
    w = p3[0][1][:n].copy()
    ring.SubRings[1].vecop(name, np.ascontiguousarray(p1[0][1][:n]), np.ascontiguousarray(p2[0][1][:n]), w,
                           s0[1] if s0 else 0, s1[1] if s1 else 0)
    ctx.ringQ.SubRings[1]._vec(name, r1, r2, r3, s0[1] if s0 else 0, s1[1] if s1 else 0)
    assert np.array_equal(ctx.to_host(r3), w), name
    ctx.close()


def test_ring_scalar_wrappers():
    """Ring.AddScalar / SubScalar / MulScalar / MulScalarThenAdd with big-int scalars (ring/operations.go:151-247)."""
    lb = _lb()
    Q = H.Qi60[:3]
    N = 256
    ctx = lb.Context(8, Q)
    ring = O.Ring(N, Q)
    rng = np.random.default_rng(3)
    x = H.rand_poly(Q, N, rng)
    big = (1 << 150) + 12345
    for meth in ("AddScalar", "SubScalar", "MulScalar", "MulScalarThenAdd"):
        want = x.copy(); getattr(ring, meth)(x, big, want)
        d = ctx.to_device(x); o = ctx.to_device(x)
        getattr(ctx.ringQ, meth)(d, big, o)
        assert np.array_equal(ctx.to_host(o), want), meth
    ctx.close()


def test_full_size_properties_c2():
    """BASELINE config 2 shape (N=2^16, 44 limbs): size-independent properties instead of a full oracle pass --
    INTT(NTT(x)) == x, linearity NTT(a+b) == NTT(a)+NTT(b), and NTT(a)*NTT(b) == NTT(negacyclic a*b) on a sparse b;
    plus an oracle spot check on 3 of the 44 limbs."""
    lb = _lb()
    logN, N = 16, 1 << 16
    Q = H.Qi60[:32] + H.Pi60[:12]
    ctx = lb.Context(logN, Q)
    rq = ctx.ringQ
    rng = np.random.default_rng(2)
    a = H.rand_poly(Q, N, rng); b = H.rand_poly(Q, N, rng)
    da, db = ctx.to_device(a), ctx.to_device(b)
    na, nb = rq.NewPoly(), rq.NewPoly()
    rq.NTT(da, na); rq.NTT(db, nb)
    back = rq.NewPoly(); rq.INTT(na, back)
    assert np.array_equal(ctx.to_host(back), a)
    s = rq.NewPoly(); rq.Add(da, db, s)
    ns = rq.NewPoly(); rq.NTT(s, ns)
    ns2 = rq.NewPoly(); rq.Add(na, nb, ns2)
    assert np.array_equal(ctx.to_host(ns), ctx.to_host(ns2))
    for i in (0, 17, 43):
        sr = O.get_subring(N, Q[i])
        want = np.empty(N, dtype=U64); sr.NTT(a[i], want)
        assert np.array_equal(ctx.to_host(na[i]), want)
    # multiply by X^k (monomial): NTT(a) * NTT(X^k) == NTT(a * X^k)
    k = 12345
    mono = np.zeros((len(Q), N), dtype=U64); mono[:, k] = 1
    dm = ctx.to_device(mono); nm = rq.NewPoly(); rq.NTT(dm, nm)
    rq.MForm(nm, nm)
    prod = rq.NewPoly(); rq.MulCoeffsMontgomery(na, nm, prod)
    rq.INTT(prod, prod)
    got = ctx.to_host(prod)
    want = np.empty_like(a)
    for i, q in enumerate(Q):
        want[i, k:] = a[i, : N - k]
        want[i, :k] = (U64(q) - a[i, N - k:]) % U64(q)
    assert np.array_equal(got, want)
    ctx.close()


@pytest.mark.parametrize("logN,family", [(13, "ckks"), (16, "ckks"), (16, "q61"), (14, "mixed"), (10, "ckks")])
def test_ntt_then_mul_coeffs_montgomery_fused(logN, family):
    """lgpu_ntt_then_mul_coeffs_montgomery == Ring.NTT followed by Ring.MulCoeffsMontgomery (ring/ntt.go:127-131 +
    ring/operations.go:88-92): the fused last-pass epilogue (2^13..2^16, FP64-pipe and integer rows) and the two-launch
    fallback (2^10), against the oracle on sampled rows and against the unfused device path on all rows; lazily
    accumulated inputs above 2^52 included."""
    lb = _lb()
    N = 1 << logN
    if family == "ckks":
        Q, _ = O.gen_moduli(logN + 1, [56] + [45] * 7, [])
    elif family == "q61":
        Q = H.Qi60[:6]
    else:
        Q = O.gen_moduli(logN + 1, [56, 45, 45], [])[0] + H.Qi60[:2]
    ctx = lb.Context(logN, Q)
    rq = ctx.ringQ
    rng = np.random.default_rng(logN)
    batch = 13                                                 # rows x batch >= 64: the persistent (fused-epilogue) kernels; fewer take two launches
    a = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    for i, q in enumerate(Q):
        if q < (1 << 58):
            a[0, i, ::7] += U64(1) << U64(62)                       # lazy inputs (NTTStandard accepts any uint64 that does not wrap)
    b = np.stack([H.rand_poly([(1 << 64) - 1] * len(Q), N, rng) for _ in range(batch)])     # any uint64 multiplicand
    da, db = ctx.to_device(a), ctx.to_device(b)
    fused = rq.NewPoly(batch)
    rq.NTTThenMulCoeffsMontgomery(da, db, fused)
    ref = rq.NewPoly(batch)
    rq.NTT(da, ref); rq.MulCoeffsMontgomery(ref, db, ref)
    assert np.array_equal(ctx.to_host(fused), ctx.to_host(ref))
    ring = O.Ring(N, Q)
    want = np.empty_like(a)
    for i in range(batch):                                      # every element, the lazily accumulated element 0 included
        ring.NTT(a[i], want[i]); ring.MulCoeffsMontgomery(want[i], b[i], want[i])
    got = ctx.to_host(fused)
    assert [i for i in range(batch) if not np.array_equal(got[i], want[i])] == []
    small = rq.NewPoly(2)                                       # below the persistent kernels' threshold: transform + coefficient-wise kernel
    rq.NTTThenMulCoeffsMontgomery(da[:2].contiguous(), db[:2].contiguous(), small)
    assert np.array_equal(ctx.to_host(small), ctx.to_host(ref)[:2])
    # in place (in == out) and the aliasing error
    inpl = da.clone()
    rq.NTTThenMulCoeffsMontgomery(inpl, db, inpl)
    assert np.array_equal(ctx.to_host(inpl), ctx.to_host(ref))
    with pytest.raises(lb.LgpuError, match="multiplicand"):
        rq.NTTThenMulCoeffsMontgomery(da, fused, fused)
    ctx.close()

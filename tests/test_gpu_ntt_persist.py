"""GPU parity (bit-exact vs the oracle) of the persistent single-pass NTT / INTT kernels (lattigo_b200/csrc/ntt_persist.cu).

Canonical transforms of at least 64 limb-transforms (rows x batch) at 2^13 <= N <= 2^16 run these kernels; smaller
launches run the two-pass kernels. Every case asserts the path it takes through the launch counter (1 launch per
persistent transform, 2 per two-pass transform at N > 2^12) and compares every limb-transform with the oracle.

Each launch selects one tile code by the class of its rows (upload_limb_tables, tables.cu), instantiated for
RL = logN - 12 in {1, 2, 3, 4}:

| family       | rows                                                       | forward                | inverse          |
|--------------|------------------------------------------------------------|------------------------|------------------|
| `fp`         | `fp_ok`: 45-bit CKKS primes + the last prime inside the edge | `FpFwdOps2<RL>`       | `FpInvOps<RL>`   |
| `int_lazy`   | first primes past the `fp_ok` edge, last below `inv_lazy`'s  | `IntFwdOps2<RL,false>` | `IntInvOps<RL,2>` |
| `int_nocorr` | first prime past the `inv_lazy` edge, last < 2^(64-logN), last <= 2^57, last <= 2^58 | `IntFwdOps2<RL,false>` | `IntInvOps<RL,1>` |
| `int_corr`   | first prime above 2^58 + the 61-bit `Qi60`                 | `IntFwdOps2<RL,true>`  | `IntInvOps<RL,1>` |

test_persist_shape_classes[logN-family] reaches every cell of that table. The names of the tests that run persistent
shapes contain `persist_shape`; test_development_switches_stay_bit_exact re-runs them under the kernels' development
switches. Run with -m gpu on an H100."""
import functools
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64
HERE = os.path.dirname(os.path.abspath(__file__))
LOGNS = (13, 14, 15, 16)
OPS = {"fp": ("FpFwdOps2", "FpInvOps"), "int_lazy": ("IntFwdOps2<false>", "IntInvOps<2>"),
       "int_nocorr": ("IntFwdOps2<false>", "IntInvOps<1>"), "int_corr": ("IntFwdOps2<true>", "IntInvOps<1>")}


def _lb():
    import lattigo_b200 as lb
    return lb


# ---- the three row classifiers of upload_limb_tables (tables.cu), restated --------------------------------------------
def fp_ok(q, logN):
    return q * (10 + logN) < 1 << 51


def inv_lazy(q, logN):
    return q << (logN + 1) < 1 << 64


def fwd_mask(q, logN):
    K = 1
    while 2 * K * q <= 1 << 63:
        K *= 2
    b, mask = min(2 * K, 8), 0
    for st in range(logN):
        if b + 2 > 2 * K:
            mask |= 1 << st
            b = K
        b += 2
    return mask


# ---- edge primes: q = 1 mod 2N on either side of a class bound ----------------------------------------------------------
@functools.lru_cache(maxsize=None)
def primes_below(bound, m, k):
    """The k largest primes q = 1 mod m with q < bound, largest last."""
    out, q = [], ((bound - 2) // m) * m + 1
    while len(out) < k:
        if O.is_prime(q):
            out.append(q)
        q -= m
    return out[::-1]


@functools.lru_cache(maxsize=None)
def primes_from(bound, m, k):
    """The k smallest primes q = 1 mod m with q >= bound, smallest first."""
    out, q = [], ((bound - 2 + m) // m) * m + 1
    while len(out) < k:
        if O.is_prime(q):
            out.append(q)
        q += m
    return out


def fp_bound(logN):
    return -(-(1 << 51) // (10 + logN))          # fp_ok <=> q < fp_bound


# fwd_mask == 0 <=> q <= 2^58 for 2^13 <= N <= 2^16: up to 2^58 the headroom 2K*q <= 2^63 keeps K = 32, which absorbs the
# 2q per stage growth of all 16 stages from the assumed input bound 8q; above it K = 16 runs out at stage 12
FWD_BOUND = 1 << 58


@functools.lru_cache(maxsize=None)
def family(name, logN):
    """Four rows of one class (the table of the module docstring); each row's class is checked against the restated
    classifiers, and every edge prime sits next to its bound."""
    m = 2 << logN
    if name == "fp":
        Q = O.gen_moduli(logN + 1, [45, 45, 45], [])[0] + primes_below(fp_bound(logN), m, 1)
        assert all(fp_ok(q, logN) for q in Q)
        assert not fp_ok(primes_from(fp_bound(logN), m, 1)[0], logN)
    elif name == "int_lazy":
        Q = primes_from(fp_bound(logN), m, 2) + primes_below(1 << (63 - logN), m, 2)
        assert all(not fp_ok(q, logN) and inv_lazy(q, logN) and fwd_mask(q, logN) == 0 for q in Q)
        assert fp_ok(primes_below(fp_bound(logN), m, 1)[0], logN)
        assert not inv_lazy(primes_from(1 << (63 - logN), m, 1)[0], logN)
    elif name == "int_nocorr":
        # the first prime past the inv_lazy edge, and the last one below 2^(64 - logN): a lazy inverse would wrap there
        Q = (primes_from(1 << (63 - logN), m, 1) + primes_below(1 << (64 - logN), m, 1) + primes_below((1 << 57) + 1, m, 1)
             + primes_below(FWD_BOUND + 1, m, 1))
        assert all(not fp_ok(q, logN) and not inv_lazy(q, logN) and fwd_mask(q, logN) == 0 for q in Q)
        assert inv_lazy(primes_below(1 << (63 - logN), m, 1)[0], logN)
    elif name == "int_corr":
        Q = primes_from(FWD_BOUND + 1, m, 1) + H.Qi60[:3]
        assert all(not fp_ok(q, logN) and not inv_lazy(q, logN) and fwd_mask(q, logN) != 0 for q in Q)
        assert fwd_mask(primes_below(FWD_BOUND + 1, m, 1)[0], logN) == 0
    else:
        raise ValueError(name)
    assert len(set(Q)) == len(Q) == 4
    return list(Q)


def test_edge_primes_match_the_documented_values():
    """The logN = 16 edge primes (fp_ok: 0x4ec4ec1c0001 | 0x4ec4ec580001, inv_lazy: 0x7ffffff00001 | 0x800000020001), and the
    forward no-correction edge at 2^58 (not 2^57) at every size the persistent kernels serve."""
    m = 2 << 16
    assert primes_below(fp_bound(16), m, 1) == [0x4ec4ec1c0001] and primes_from(fp_bound(16), m, 1) == [0x4ec4ec580001]
    assert primes_below(1 << 47, m, 1) == [0x7ffffff00001] and primes_from(1 << 47, m, 1) == [0x800000020001]
    assert primes_below((1 << 57) + 1, m, 1) == [0x1fffffffffc0001]
    for logN in LOGNS:
        m = 2 << logN
        assert all(fwd_mask(q, logN) == 0 for q in primes_below(FWD_BOUND + 1, m, 1) + [(1 << 57) + 1])
        assert fwd_mask(primes_from(FWD_BOUND + 1, m, 1)[0], logN) != 0


# ---- expected kernel launches (ntt.cu: persistent, transform) ----------------------------------------------------------------
_FORCED = os.environ.get("LGPU_NTT_PERSIST")


def persistent(limb_transforms):
    """Whether a transform group of this many limb-transforms runs the persistent kernels. LGPU_NTT_PERSIST=0 disables
    them, =1 selects them for every canonical transform."""
    if _FORCED is not None and int(_FORCED) == 0:
        return False
    return (_FORCED is not None and int(_FORCED) == 1) or limb_transforms >= 64


def launches(*groups):
    return sum(1 if persistent(n) else 2 for n in groups if n)


def fwd_launches(n_fp, n_int, batch, aligned=True):
    """Forward: the FP64-pipe rows go persistent on the size of the WHOLE launch, the integer rows on their own size.
    A two-pass FP64 forward needs 16-byte aligned rows; otherwise every row takes the integer kernels."""
    total = (n_fp + n_int) * batch
    if n_fp and (persistent(total) or aligned):
        return launches(total) + launches(n_int * batch)
    return launches(total)


def inv_launches(n_fp, n_int, batch):
    """Inverse: each row kind goes persistent on its own size."""
    return launches(n_fp * batch, n_int * batch)


def fused_launches(n_fp, n_int, batch):
    """NTTThenMulCoeffsMontgomery: persistent FP64 rows fuse the product; integer rows take their transform and then the
    coefficient-wise kernel."""
    if persistent((n_fp + n_int) * batch):
        return (1 if n_fp else 0) + (launches(n_int * batch) + 1 if n_int else 0)
    return fwd_launches(n_fp, n_int, batch) + 1


# ---- inputs and the oracle -----------------------------------------------------------------------------------------------
def inputs(Q, N, batch, rng):
    """Different data in every (batch element, row): element 0 = all q - 1 (largest lazy growth), element 1 = a single
    nonzero coefficient in the last position, element 2 = zero, element 3 = zero then q - 1 in the upper half (the largest
    U - V difference at the last inverse stage), the others uniform."""
    x = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    qv = np.array(Q, dtype=U64)[:, None]
    x[0] = qv - U64(1)
    x[1] = 0
    x[1, :, -1] = [int(rng.integers(1, q)) for q in Q]
    x[2] = 0
    x[3, :, : N // 2] = 0
    x[3, :, N // 2:] = qv - U64(1)
    return x


def lazy_inputs(x, Q, logN, rng):
    """Lazily accumulated words that Ring.NTT accepts (NTTStandard reduces at the end): up to 2^63 on FP64-pipe rows,
    + 2^62 on the other rows with q < 2^58; canonical on the rest."""
    y = x.copy()
    for i, q in enumerate(Q):
        if fp_ok(q, logN):
            y[:, i] = rng.integers(0, 1 << 63, y[:, i].shape, dtype=U64)
            y[0, i] = U64((1 << 63) - 1)
        elif q < 1 << 58:
            y[:, i] += U64(1 << 62)
    return y


def oracle(method, Q, x):
    ring = O.Ring(x.shape[-1], Q)
    out = np.empty_like(x)
    for b in range(x.shape[0]):
        getattr(ring, method)(x[b], out[b])
    return out


def assert_same(got, want, what):
    """Every limb-transform equal; a failure names the mismatching (batch element, row) pairs."""
    if not np.array_equal(got, want):
        bad = sorted({(int(b), int(r)) for b, r, _ in zip(*np.nonzero(got != want))})
        raise AssertionError("%s: %d of %d limb-transforms differ from the oracle, (batch, row) = %s"
                             % (what, len(bad), got.shape[0] * got.shape[1], bad[:16]))


def run_both(ctx, ring, Q, logN, x, n_fp, n_int, what, rng, odd=None):
    """NTT, INTT, INTTLazy (== INTT for N >= 16) and NTT on lazy words of a batched x, out of place and in place, each
    compared with the oracle on every limb-transform and checked for its launch count."""
    batch = x.shape[0]
    dev = odd if odd is not None else ctx.to_device
    aligned = odd is None
    want_f, want_i = oracle("NTT", Q, x), oracle("INTT", Q, x)
    d, o = dev(x), dev(np.zeros_like(x))
    assert H.launch_delta(lambda: ring.NTT(d, o)) == fwd_launches(n_fp, n_int, batch, aligned), what
    assert_same(ctx.to_host(o), want_f, what + " NTT")
    assert H.launch_delta(lambda: ring.INTT(d, o)) == inv_launches(n_fp, n_int, batch), what
    assert_same(ctx.to_host(o), want_i, what + " INTT")
    assert H.launch_delta(lambda: ring.INTTLazy(d, o)) == inv_launches(n_fp, n_int, batch), what
    assert_same(ctx.to_host(o), want_i, what + " INTTLazy")
    e = dev(x)
    ring.NTT(e, e)
    assert_same(ctx.to_host(e), want_f, what + " NTT in place")
    ring.INTT(e, e)
    assert_same(ctx.to_host(e), x, what + " INTT in place")
    y = lazy_inputs(x, Q, logN, rng)
    dy = dev(y)
    assert H.launch_delta(lambda: ring.NTT(dy, o)) == fwd_launches(n_fp, n_int, batch, aligned), what
    assert_same(ctx.to_host(o), oracle("NTT", Q, y), what + " NTT on lazy words")


# ---- every default instantiation ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", list(OPS))
@pytest.mark.parametrize("logN", LOGNS)
def test_persist_shape_classes(logN, fam):
    """4 rows x 16 polynomials = 64 limb-transforms of one class: one persistent launch per transform, running the
    forward / inverse tile code of OPS[fam] at RL = logN - 12."""
    lb = _lb()
    Q = family(fam, logN)
    ctx = lb.Context(logN, Q)
    rng = np.random.default_rng(1000 * logN + list(OPS).index(fam))
    x = inputs(Q, 1 << logN, 16, rng)
    n_fp = len(Q) if fam == "fp" else 0
    run_both(ctx, ctx.ringQ, Q, logN, x, n_fp, len(Q) - n_fp, "%s logN=%d" % (fam, logN), rng)
    ctx.close()


@pytest.mark.parametrize("logN", LOGNS)
def test_threshold_63_two_pass(logN):
    """Below the 64 limb-transform threshold: 3 rows x 21 = 63 and single rows take the two-pass kernels, on FP64-pipe
    rows and on integer rows (64 = 4 x 16 is test_persist_shape_classes). 8 rows x 8 = 64 with half of them FP64-pipe
    rows: the forward FP64 rows go persistent on the whole launch, the 32 integer limb-transforms stay two-pass. Under
    LGPU_NTT_PERSIST=1 every one of these is persistent, a single row included (grid clamped to its tiles, distance
    larger than the number of limb-transforms)."""
    lb = _lb()
    N = 1 << logN
    rng = np.random.default_rng(63 + logN)
    for fams in (("fp",), ("int_lazy",), ("int_corr",), ("fp", "int_nocorr")):
        Q = [q for f in fams for q in family(f, logN)]
        ctx = lb.Context(logN, Q)
        n_fp = 4 if "fp" in fams else 0
        if len(Q) == 4:
            q3 = Q[:3]
            x = inputs(q3, N, 21, rng)
            assert launches(63) == (1 if _FORCED == "1" else 2)
            run_both(ctx, ctx.ringQ.AtLevel(2), q3, logN, x, min(n_fp, 3), 3 - min(n_fp, 3), "%s 3x21" % fams[0], rng)
            sr = ctx.ringQ.SubRings[3]
            row = H.rand_poly(Q[3:], N, rng)[0]
            d, o = ctx.to_device(row), ctx.to_device(np.zeros_like(row))
            assert H.launch_delta(lambda: sr.NTT(d, o)) == launches(1)
            assert_same(ctx.to_host(o)[None, None], oracle("NTT", Q[3:], row[None, None]), "%s single row NTT" % fams[0])
            assert H.launch_delta(lambda: sr.INTT(d, o)) == launches(1)
            assert_same(ctx.to_host(o)[None, None], oracle("INTT", Q[3:], row[None, None]), "%s single row INTT" % fams[0])
        else:
            x = inputs(Q, 1 << logN, 8, rng)
            run_both(ctx, ctx.ringQ, Q, logN, x, n_fp, 4, "fp+int_nocorr 8x8", rng)
        ctx.close()


@pytest.mark.parametrize("logN", LOGNS)
def test_persist_shape_many_tiles(logN):
    """8 rows x 40 = 320 limb-transforms in one call (160 FP64-pipe, 160 integer with lazy corrections): the ticket queue
    cycles many times past the resident grid, and a (row, batch element) mix-up in the tile mapping shows."""
    lb = _lb()
    Q = family("fp", logN) + family("int_corr", logN)
    ctx = lb.Context(logN, Q)
    rng = np.random.default_rng(320 + logN)
    x = inputs(Q, 1 << logN, 40, rng)
    run_both(ctx, ctx.ringQ, Q, logN, x, 4, 4, "8x40 logN=%d" % logN, rng)
    ctx.close()


# ---- layouts ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("logN", LOGNS)
def test_persist_shape_layouts(logN):
    """AtLevel on batched full-level buffers (batch stride > rows * N, the rows above the level keep a sentinel), ringP
    (global limb index offset by nQ), an odd word offset, and one call mixing FP64-pipe rows with integer rows where
    the forward transform goes persistent on the whole launch and the inverse stays two-pass on the FP64 rows alone."""
    import torch
    lb = _lb()
    N = 1 << logN
    Q = family("fp", logN) + family("int_lazy", logN)
    P = family("int_corr", logN)
    ctx = lb.Context(logN, Q + [family("int_nocorr", logN)[2]], P)        # 9 Q rows, 4 P rows
    rng = np.random.default_rng(7 * logN)
    sentinel = U64(0xDEADBEEFDEADBEEF)

    # AtLevel(7) on (batch, 9, N) buffers: 4 FP64 rows + 4 integer rows x 16 = 128 limb-transforms
    lvl = ctx.ringQ.AtLevel(7)
    x = inputs(Q, N, 16, rng)
    full = np.full((16, 9, N), sentinel, dtype=U64)
    full[:, :8] = x
    d, o = ctx.to_device(full), ctx.to_device(full)
    assert H.launch_delta(lambda: lvl.NTT(d, o)) == fwd_launches(4, 4, 16)
    got = ctx.to_host(o)
    assert_same(got[:, :8], oracle("NTT", Q, x), "AtLevel NTT")
    assert (got[:, 8] == sentinel).all()
    assert H.launch_delta(lambda: lvl.INTT(d, o)) == inv_launches(4, 4, 16)
    got = ctx.to_host(o)
    assert_same(got[:, :8], oracle("INTT", Q, x), "AtLevel INTT")
    assert (got[:, 8] == sentinel).all()
    lvl.NTT(d, d)
    lvl.INTT(d, d)
    assert np.array_equal(ctx.to_host(d), full)

    # ringP: 4 rows x 16
    xp = inputs(P, N, 16, rng)
    run_both(ctx, ctx.ringP, P, logN, xp, 0, 4, "ringP", rng)

    # odd word offset (8- but not 16-byte aligned), 4 FP64 rows x 16 and the 8 mixed rows x 8
    def odd(arr):
        flat = torch.zeros(arr.size + 1, dtype=torch.int64, device="cuda")
        view = flat[1:].view(*arr.shape)
        view.copy_(ctx.to_device(arr))
        assert view.data_ptr() % 16 == 8
        return view

    xf = inputs(Q[:4], N, 16, rng)
    run_both(ctx, ctx.ringQ.AtLevel(3), Q[:4], logN, xf, 4, 0, "odd offset fp", rng, odd=odd)
    xm = inputs(Q, N, 8, rng)
    run_both(ctx, lvl, Q, logN, xm, 4, 4, "odd offset mixed", rng, odd=odd)

    # 2 FP64 + 2 integer rows x 20: forward FP64 rows persistent (80 limb-transforms), inverse FP64 rows two-pass (40)
    Qm = Q[2:6]
    xm = inputs(Qm, N, 20, rng)
    mixed = lb.Context(logN, Qm)
    if _FORCED is None:
        assert fwd_launches(2, 2, 20) == 3 and inv_launches(2, 2, 20) == 4
    run_both(mixed, mixed.ringQ, Qm, logN, xm, 2, 2, "mixed 2+2 x20", rng)
    mixed.close()
    ctx.close()


# ---- fused epilogue ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("logN", LOGNS)
def test_persist_shape_ntt_then_mul_coeffs_montgomery(logN):
    """NTTThenMulCoeffsMontgomery on the persistent path (4 FP64-pipe rows with the fused product, 4 integer rows with
    transform + coefficient-wise kernel) x 10 polynomials, every batch element against the oracle, the lazily
    accumulated one (element 3) included."""
    lb = _lb()
    N = 1 << logN
    Q = family("fp", logN) + family("int_nocorr", logN)
    ctx = lb.Context(logN, Q)
    rq = ctx.ringQ
    rng = np.random.default_rng(5 * logN)
    batch = 10
    a = inputs(Q, N, batch, rng)
    a[3] = lazy_inputs(a[3:4], Q, logN, rng)[0]
    b = np.stack([H.rand_poly([(1 << 64) - 1] * len(Q), N, rng) for _ in range(batch)])      # any uint64 multiplicand
    ring = O.Ring(N, Q)
    want = np.empty_like(a)
    for i in range(batch):
        ring.NTT(a[i], want[i])
        ring.MulCoeffsMontgomery(want[i], b[i], want[i])
    da, db, out = ctx.to_device(a), ctx.to_device(b), rq.NewPoly(batch)
    assert H.launch_delta(lambda: rq.NTTThenMulCoeffsMontgomery(da, db, out)) == fused_launches(4, 4, batch)
    assert_same(ctx.to_host(out), want, "NTTThenMulCoeffsMontgomery logN=%d" % logN)
    rq.NTTThenMulCoeffsMontgomery(da, db, da)
    assert_same(ctx.to_host(da), want, "NTTThenMulCoeffsMontgomery in place logN=%d" % logN)
    ctx.close()


# ---- development switches ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("env", ["LGPU_NTT_PERSIST=0", "LGPU_NTT_PERSIST=1", "LGPU_NTT_PERSIST_V=1", "LGPU_NTT_PERSIST_V=2",
                                 "LGPU_NTT_PERSIST_V=4", "LGPU_NTT_PERSIST_V=5", "LGPU_NTT_PERSIST_IV=2", "LGPU_NTT_PH1INT=1",
                                 "LGPU_NTT_PERSIST_D=1", "LGPU_NTT_PERSIST_D=100000"])
def test_development_switches_stay_bit_exact(env):
    """The persistent kernels' development switches (read once per process, hence a subprocess) re-run every
    persist_shape case: PERSIST=0 (two-pass only; the launch counts follow), PERSIST=1 (persistent also below 64
    limb-transforms), V=1 / 2 (first-generation tile code, serial ticket / claim-ahead loop), V=4 (TMA prefetch), V=5
    (register copy-out), IV=2 (IntFwdOps, 256 x 16 padded), PH1INT=1 (FpFwdOps with an integer first pass), D=1 and D far
    above the number of limb-transforms (the distance between a limb-transform's pass-1 and pass-2 tiles).
    LGPU_NTT_PERSIST_V=6 is left out: its static schedule spins on tiles owned by other CTAs and is deadlock-free only
    when every CTA of the grid is resident at once, which a GPU shared with other work does not guarantee."""
    import subprocess
    import sys
    k, v = env.split("=")
    e = dict(os.environ, **{k: v})
    root = os.path.dirname(HERE)
    sel = "persist_shape or threshold" if k == "LGPU_NTT_PERSIST" else "persist_shape"
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(HERE, "test_gpu_ntt_persist.py"), "-m", "gpu", "-x", "-q",
                        "-k", sel], cwd=root, env=e, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]

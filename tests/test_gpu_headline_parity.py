"""GPU parity at the sizes the benchmark actually runs (VERDICT r1, "parity gaps under the headline"):
 * the benchmarked configuration itself (CKKS_L44: N = 2^16, 44 Q + 4 P limbs, beta = 11) against the oracle, device path
   and host-buffer entry point;
 * BASELINE config 2 (N = 2^16, 44 limbs) with ALL limbs against the oracle for both prime families (61-bit integer
   kernels, 45-bit FP64-pipe kernels): forward, inverse, lazy;
 * the fused key-switch pipeline at N = 2^16 with k = 2 and k = 3 P-limbs and ragged / single-limb last digits;
 * Ring.NTT on words above 2^52 (lazily accumulated inputs; ADVICE r1).
Run with -m gpu on an H100."""
import numpy as np
import pytest

from oracle import oracle as O
from tests import helpers as H
from tests.test_gpu_keyswitch import _gadget_case, _mods

pytestmark = pytest.mark.gpu
U64 = np.uint64


def _lb():
    import lattigo_b200 as lb
    return lb


def _torch_rand_rows(N, mods, lead, g):
    import torch
    out = torch.empty(tuple(lead) + (len(mods), N), dtype=torch.int64, device="cuda")
    for i, m in enumerate(mods):
        out[..., i, :] = torch.randint(0, m, tuple(lead) + (N,), generator=g, device="cuda", dtype=torch.int64)
    return out


def test_ckks_l44_headline_config_vs_oracle():
    """bench.py's workload (preset CKKS_L44, level 43, beta = 11 digits of 4 limbs, lazy u64 accumulation over 11 terms
    in K3) bit-exact against the oracle for every pair of a batch of 5 (device-resident entry point), for 2 pairs through
    the host-buffer entry point, and batch consistency against a single-pair call. At batch 5 the fused ModDown INTT
    (4 P rows x 5 polynomials per component) and the rescale INTT (the last row) both take the two-pass kernels.
    Reference op sequence: schemes/ckks/evaluator.go:719-872 + :477-515 over core/rlwe/evaluator_gadget_product.go:129-201."""
    _ckks_l44_case(5)


@pytest.mark.parametrize("batch", [63, 64])
def test_ckks_l44_headline_persistent_batches_vs_oracle(batch):
    """The headline case of test_ckks_l44_headline_config_vs_oracle at the batches where its inverse transforms run the
    persistent kernels: at 63 the ModDown INTT (252 limb-transforms) goes persistent and the rescale INTT (63) stays
    two-pass, at 64 (the benchmark's shape and sub-batch) both are persistent. Every pair against the oracle; the
    single-pair call of the batch-consistency check runs the two-pass kernels, so it compares the two paths on the
    device."""
    _ckks_l44_case(batch)


def _ckks_l44_case(batch):
    import torch
    lb = _lb()
    from lattigo_b200 import params as presets
    s = presets.PRESETS["CKKS_L44"]
    logN, q, p = s["logN"], s["Q"], s["P"]
    assert len(q) == 44 and len(p) == 4
    ctx = lb.Context(logN, q, p)
    N = 1 << logN
    level, levelP = len(q) - 1, len(p) - 1
    nd = (level + levelP + 1) // (levelP + 1)
    assert nd == 11
    g = torch.Generator(device="cuda"); g.manual_seed(44)
    evk_t = _torch_rand_rows(N, q + p, (nd, 1, 2), g)
    rlk = lb.GadgetCiphertext(ctx, evk_t, level, levelP)
    ev = lb.CKKSEvaluator(ctx, rlk)
    a = _torch_rand_rows(N, q, (batch, 2), g); b = _torch_rand_rows(N, q, (batch, 2), g)
    out = ev.MulRelinRescaleNew(a, b)
    torch.cuda.synchronize()
    one = ev.MulRelinRescaleNew(a[3:4].contiguous(), b[3:4].contiguous())
    assert torch.equal(out[3:4], one)
    params = O.Parameters(logN, q, p)
    ev_o = O.CKKSEvaluator(params, O.GadgetCiphertext(ctx.to_host(evk_t), level + 1, levelP + 1))
    ah, bh, oh = ctx.to_host(a), ctx.to_host(b), ctx.to_host(out)
    bad = []
    for i in range(batch):
        r = ev_o.Rescale(ev_o.MulRelinNew([ah[i, 0], ah[i, 1]], [bh[i, 0], bh[i, 1]]))
        if not (np.array_equal(oh[i, 0], r[0]) and np.array_equal(oh[i, 1], r[1])):
            bad.append(i)
    assert bad == [], "pairs that differ from the oracle: %s" % bad
    # host-buffer entry point at the same size (lgpu_ckks_mulrelin_rescale_batch_host, chunked 2-stream pipeline), against
    # the device results just checked
    out_host = np.zeros((2, 2, level, N), dtype=U64)
    ev.MulRelinRescaleHost(np.ascontiguousarray(ah[:2]), np.ascontiguousarray(bh[:2]), out_host, chunk=1)
    assert np.array_equal(out_host, oh[:2])
    ctx.close()


@pytest.mark.parametrize("family", ["q61", "ckks45"])
def test_c2_all_44_limbs_vs_oracle(family):
    """BASELINE config 2: Ring.NTT / INTT / NTTLazy / INTTLazy on N = 2^16 x 44 limbs, every limb compared with the
    oracle (ring/ntt.go:127-152). q61 = the reference's Qi60/Pi60 test primes (integer kernels, lazy corrections);
    ckks45 = the 44 Q primes of the headline literal (43 FP64-pipe rows + the 56-bit q0 on the integer kernels)."""
    lb = _lb()
    logN, N = 16, 1 << 16
    if family == "q61":
        Q = H.Qi60[:32] + H.Pi60[:12]
    else:
        from lattigo_b200 import params as presets
        Q = presets.PRESETS["CKKS_L44"]["Q"]
    assert len(Q) == 44
    ctx = lb.Context(logN, Q)
    rq = ctx.ringQ
    ring = O.Ring(N, Q)
    rng = np.random.default_rng(1616)
    batch = 2
    x = np.stack([H.rand_poly(Q, N, rng) for _ in range(batch)])
    want = np.empty_like(x); want_lazy = np.empty_like(x); want_inv = np.empty_like(x); want_inv_lazy = np.empty_like(x)
    for b in range(batch):
        ring.NTT(x[b], want[b]); ring.NTTLazy(x[b], want_lazy[b])
        ring.INTT(x[b], want_inv[b]); ring.INTTLazy(x[b], want_inv_lazy[b])
    d = ctx.to_device(x)
    o = rq.NewPoly(batch)
    rq.NTT(d, o); assert np.array_equal(ctx.to_host(o), want)
    rq.NTTLazy(d, o); assert np.array_equal(ctx.to_host(o), want_lazy)
    rq.INTT(d, o); assert np.array_equal(ctx.to_host(o), want_inv)
    rq.INTTLazy(d, o); assert np.array_equal(ctx.to_host(o), want_inv_lazy)
    # in place, forward then inverse
    e = ctx.to_device(x)
    rq.NTT(e, e); assert np.array_equal(ctx.to_host(e), want)
    rq.INTT(e, e); assert np.array_equal(ctx.to_host(e), x)
    ctx.close()


def test_fused_keyswitch_logn16_k2_k3_ragged():
    """Fused K1/K2/K3 pipeline at N = 2^16 with k = 3 (beta = 3: digits 3+3+1 -> single-limb last digit at level 6,
    ragged 3+2 at level 4, 3+3 at level 5) and k = 2 (beta = 4 with a ragged last digit at level 6), FP64 rows and
    integer rows mixed; reference loop core/rlwe/evaluator_gadget_product.go:129-201."""
    lb = _lb()
    q, p = _mods(16, [56, 45, 45, 45, 45, 45, 45], [55, 55, 55])
    _gadget_case(lb, 16, q, p, 0, (6, 5, 4), batch=2, seed=61)
    _gadget_case(lb, 16, q, p[:2], 0, (6, 3), batch=2, seed=62)


def test_ntt_accepts_words_above_2_52():
    """Ring.NTT ends in a full reduction in the reference (NTTStandard = nttCoreLazy + reducevec, ring/ntt.go:174-177), so
    it accepts lazily accumulated words; the FP64-pipe kernels must not assume inputs below 2^52."""
    lb = _lb()
    # (logN, batch, kernel launches): at N = 2^16 one polynomial takes the two-pass kernels (2 launches for the 2 FP64-pipe
    # rows, 2 for the 56-bit row), 64 polynomials the persistent ones (1 + 1)
    for logN, batch, launches in ((12, 1, None), (16, 1, 4), (16, 64, 2)):
        N = 1 << logN
        q, p = O.gen_moduli(logN + 1, [56, 45, 45], [55])
        Q = [q[1], q[2], q[0]]
        ctx = lb.Context(logN, Q)
        ring = O.Ring(N, Q)
        rng = np.random.default_rng(52 + logN + batch)
        # values up to 2^63: the reference's lazy arithmetic does not wrap for 45/56-bit primes there
        x = rng.integers(0, 1 << 63, (batch, len(Q), N), dtype=U64)
        x[:, :, ::7] = rng.integers(0, 1 << 40, (batch, len(Q), (N + 6) // 7), dtype=U64)
        want = np.empty_like(x)
        for b in range(batch):
            ring.NTT(x[b], want[b])
        d = ctx.to_device(x); o = ctx.ringQ.NewPoly(batch)
        n = H.launch_delta(lambda: ctx.ringQ.NTT(d, o))
        assert launches is None or n == launches, (logN, batch, n)
        assert np.array_equal(ctx.to_host(o), want), (logN, batch)
        ctx.close()


def test_fused_keyswitch_wide_primes_and_k5_k6():
    """The fused pipeline on what the reference's bootstrapping literals need (VERDICT r1 item 5;
    circuits/ckks/bootstrapping/default_parameters.go:118-134): 61-bit special primes (integer rows that need the lazy
    correction schedule at every stage), k = 5 and k = 6, chains that mix 40-bit FP64-pipe rows with 56/60-bit integer rows,
    full / ragged / single-limb last digits. N = 2^13 (smallest fused size) against the oracle."""
    lb = _lb()
    q = O.gen_moduli(14, [60, 40, 40, 40, 39, 60, 60, 56, 56, 40, 40], [])[0]
    p6 = O.gen_moduli(14, [], [61] * 6)[1]
    _gadget_case(lb, 13, q, p6, 0, (10, 7, 6, 5), batch=2, seed=71)        # k = 6: digits 6+5, 6+2, 6+1 (single-limb last digit), 6
    _gadget_case(lb, 13, q, p6[:5], 0, (10, 9, 4), batch=2, seed=72)      # k = 5: 5+5+1, 5+5, 5
    _gadget_case(lb, 13, H.Qi60[:7], H.Pi60[:3], 0, (6, 5, 3), batch=2, seed=73)   # all rows 61-bit


def test_boot_chain_keyswitch_and_mulrelin_logn16():
    """N16QP1767H32768H32's chain at full size (30 Q limbs: 60 + 13x40 + 3x39 + 9x60 + 4x56 bits, 6 x 61-bit P limbs, beta = 5):
    gadget product at the top level and at an EvalMod level, plus MulRelin + Rescale, against the oracle."""
    import torch
    lb = _lb()
    from lattigo_b200 import params as presets
    s = presets.PRESETS["BOOT_N16QP1767"]
    logN, q, p = s["logN"], s["Q"], s["P"]
    _gadget_case(lb, logN, q, p, 0, (29, 23, 20), batch=1, seed=81)
    ctx = lb.Context(logN, q, p)
    N = 1 << logN
    level, levelP = 25, len(p) - 1                           # a rescale from a 60-bit last modulus over 40-bit rows
    params = O.Parameters(logN, q, p)
    nd = params.BaseRNSDecompositionVectorSize(len(q) - 1, levelP)
    g = torch.Generator(device="cuda"); g.manual_seed(82)
    evk_t = _torch_rand_rows(N, q + p, (nd, 1, 2), g)
    ev = lb.CKKSEvaluator(ctx, lb.GadgetCiphertext(ctx, evk_t, len(q) - 1, levelP))
    a = _torch_rand_rows(N, q[: level + 1], (2, 2), g); b = _torch_rand_rows(N, q[: level + 1], (2, 2), g)
    out = ev.MulRelinRescaleNew(a, b)
    ev_o = O.CKKSEvaluator(params, O.GadgetCiphertext(ctx.to_host(evk_t), len(q), levelP + 1))
    ah, bh, oh = ctx.to_host(a), ctx.to_host(b), ctx.to_host(out)
    r = ev_o.Rescale(ev_o.MulRelinNew([ah[0, 0], ah[0, 1]], [bh[0, 0], bh[0, 1]]))
    assert np.array_equal(oh[0, 0], r[0]) and np.array_equal(oh[0, 1], r[1])
    ctx.close()

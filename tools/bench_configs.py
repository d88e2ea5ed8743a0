"""SURVEY.md section 8(d) configurations C1-C4 measured on one GPU (CUDA events on the launching stream, warm-up, an
L2 flush before every timed iteration). bench.py stays the contract bench (headline L=44 mul+relin line); this script
produces the per-config table that DESIGN.md quotes and writes it as JSON (default: bench_out/configs.json).

  C1  N=2^12, 1 limb (q = Qi60[0]): NTT then INTT, latency
  C2  N=2^16, 44 limbs (Qi60[0:32] + Pi60[0:12], 61-bit -> integer-pipe kernels) and the same shape with the
      CKKS_L44 45/56-bit primes (FP64-pipe kernels): (i) NTT GB/s, algorithmic bytes 2*S(44);
      (ii) NTT + MulCoeffsMontgomery, algorithmic bytes 5*S(44) as two calls, 3*S(44) through the fused
      lgpu_ntt_then_mul_coeffs_montgomery
  C3  CKKS PN16QP1761, batch 64 pairs at level 33: MulRelin + Rescale, ct/s
  C4  BGV N15QP880, batch 128 at level 19: one Galois rotation (Evaluator.Automorphism), ct/s
  C4mul  the same ciphertexts: BGV MulRelin + Rescale and BFV MulRelinScaleInvariant (lgpu_bgv_mulrelin_batch), ct/s;
         algorithmic bytes 4*S(20) in + 2*S(19) (BGV) or 2*S(20) (BFV) out per pair + the relinearization key once per batch
  C4sum  the same ciphertexts: bgv.Evaluator.InnerSum(batchSize = 1, n = N) -- the n * batchSize == Slots() rule,
         PartialTracesSum(1, N/2) (14 key switches) + RotateRows + Add -- through lgpu_evaluator_partial_traces_sum, ct/s
  C3sum  PN16QP1761 batch 64 at level 33: RotateAndAdd(batchSize = 1, n = 7) = PartialTracesSum(1, 7) (4 key switches, two of them
         lazy QP terms; InnerSum rejects n * batchSize = 7), ct/s
  C3sum / C4sum also time the same schedule composed from the existing entry points (lgpu_decompose_ntt,
  lgpu_evaluator_automorphism_hoisted_lazy, lgpu_evaluator_automorphism with the hoisted decomposition, vecops, ModDown) in the
  same run, and report the kernel launches of one call. Algorithmic bytes: every input and output ciphertext once plus every
  Galois key once.
  C4expand  BGV N15QP880 at level 3, one ciphertext: RingPackingEvaluator.Expand(logGap = 7), 256 outputs (262 key switches)
  C4pack    the 256 outputs of C4expand: Repack = Pack(cts, LogN, true) back into one ciphertext (262 key switches)
  C4expand / C4pack also time the same schedule issued one ciphertext at a time from the existing entry points
  (lgpu_evaluator_automorphism + vecops, what a shim looping like the reference does) and check that both give the same output.
  C3aek_down / C3aek_up  CKKS PN16QP1761, batch 64 at level 33, NTT domain: Evaluator.ApplyEvaluationKey 2^16 -> 2^15 and
         2^15 -> 2^16 through lgpu_evaluator_apply_evaluation_key, against the same work composed from the existing entry points
         (GadgetProduct + Add + INTT at 2^16 + a strided copy + NTT at 2^15 going down; MapSmallDimensionToLargerDimensionNTT +
         GadgetProduct + Add going up), with both outputs compared.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200 import params as presets  # noqa: E402


def timeit(fn, iters, warmup, flush):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.add_(1)
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(ts)), float(np.min(ts))


def power_limit_w():
    """Enforced power limit of GPU 0 (read-only nvidia-smi query), or None where it cannot be read."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def rand_rows(moduli, N, batch, rng, dev):
    out = torch.empty((batch, len(moduli), N), dtype=torch.int64, device=dev)
    for i, q in enumerate(moduli):
        out[:, i] = torch.from_numpy(rng.integers(0, q, size=(batch, N), dtype=np.uint64).view(np.int64)).to(dev)
    return out


def rand_evk(ctx, levelQ, levelP, rng, dev):
    nq, npp = levelQ + 1, levelP + 1
    nd = (levelQ + levelP + 1) // (levelP + 1)
    mods = ctx.Q[:nq] + ctx.P[:npp]
    data = torch.empty((nd, 1, 2, nq + npp, ctx.N), dtype=torch.int64, device=dev)
    for i, q in enumerate(mods):
        data[:, :, :, i] = torch.from_numpy(rng.integers(0, q, size=(nd, 1, 2, ctx.N), dtype=np.uint64).view(np.int64)).to(dev)
    return data


def _pts_schedule(ctx, offset, n):
    """PartialTracesSum's key switches (core/rlwe/inner_sum.go:217-283): per iteration below the top bit of n, the lazy term's
    rotation (or None) and the doubling rotation."""
    out = []
    i, j = 0, n
    while j > 1:
        out.append(((n - (n & ((2 << i) - 1))) * offset if j & 1 else None, (1 << i) * offset))
        i, j = i + 1, j >> 1
    return out


def composed_pts(ctx, rl, keys, ct, offset, n, out):
    """PartialTracesSum(ct, offset, n), NTT domain, built from the existing entry points: what a caller without the fused call
    does. Lazy terms use the one-pass QP-stacked AutomorphismHoistedLazy, doublings Evaluator.Automorphism with the hoisted
    decomposition, then vecop adds and one ModDown."""
    import ctypes
    L = lb.lib()
    b, _, nq, N = ct.shape
    level, levelP = nq - 1, len(ctx.P) - 1
    np_ = levelP + 1
    vp = ctypes.c_void_p
    gal = lambda k: pow(5, k & (2 * N - 1), 2 * N)
    st = lb.ring._stream()
    ADD = lb.OP["Add"]
    x = ct.clone()
    tmp = torch.empty_like(x)
    acc = torch.empty((2, b, nq + np_, N), dtype=torch.int64, device=ct.device)
    cqp = torch.empty_like(acc)
    dec = torch.empty((rl.BaseRNSDecompositionVectorSize(level, levelP), b, nq + np_, N), dtype=torch.int64, device=ct.device)
    W = 8 * N
    first = True
    for lazy, dbl in _pts_schedule(ctx, offset, n):
        lb._lib.check(L.lgpu_decompose_ntt(ctx.h, level, levelP, levelP + 1, vp(x.data_ptr() + nq * W), 1, vp(dec.data_ptr()), b, 2 * nq * N, st))
        if lazy is not None:
            base = (acc if first else cqp).data_ptr()
            lb._lib.check(L.lgpu_evaluator_automorphism_hoisted_lazy(
                ctx.h, level, vp(x.data_ptr()), vp(dec.data_ptr()), level, gal(lazy), keys[gal(lazy)].ref(), vp(base), vp(base + nq * W),
                vp(base + b * (nq + np_) * W), vp(base + (b * (nq + np_) + nq) * W), b, 2 * nq * N, (nq + np_) * N, (nq + np_) * N, st))
            if not first:          # ringQP.Add(accQP, cQP, accQP) on both components
                for ring, lvl, off in ((lb.ring.RING_Q, level, 0), (lb.ring.RING_P, levelP, nq * W)):
                    pa, pc = vp(acc.data_ptr() + off), vp(cqp.data_ptr() + off)
                    lb._lib.check(L.lgpu_vecop(ctx.h, ring, lvl, ADD, pa, pc, pa, None, None, 2 * b, (nq + np_) * N, st))
            first = False
        rl.Automorphism(x, gal(dbl), keys[gal(dbl)], tmp, decomp=dec)
        ringQ = ctx.ringQ.AtLevel(level)
        ringQ.Add(x.view(-1, nq, N), tmp.view(-1, nq, N), x.view(-1, nq, N))
    if n & (n - 1):
        a = acc.data_ptr()
        lb._lib.check(L.lgpu_evaluator_moddown(ctx.h, level, levelP, vp(a), vp(a + nq * W), vp(a + b * (nq + np_) * W), vp(a + (b * (nq + np_) + nq) * W),
                                               vp(tmp.data_ptr()), vp(tmp.data_ptr() + nq * W), b, (nq + np_) * N, (nq + np_) * N, 2 * nq * N, st))
        ctx.ringQ.AtLevel(level).Add(tmp.view(-1, nq, N), x.view(-1, nq, N), out.view(-1, nq, N))
    else:
        out.copy_(x)


def bench_innersum(name, iters, rng, dev, flush):
    if name == "C4sum":
        P, logN, batch, n = presets.PRESETS["BGV_N15QP880"], 15, 128, 1 << 15
        desc = "BGV N15QP880, batch 128 at level 19: InnerSum(1, N) = PartialTracesSum(1, N/2) + RotateRows + Add"
    else:
        P, logN, batch, n = presets.PRESETS["CKKS_PN16QP1761"], 16, 64, 7
        desc = "CKKS PN16QP1761, batch 64 at level 33: RotateAndAdd(1, 7) = PartialTracesSum(1, 7) (2 doublings + 2 lazy QP terms)"
    ctx = lb.Context(logN, P["Q"], P["P"])
    N = ctx.N
    level, levelP = len(P["Q"]) - 1, len(P["P"]) - 1
    gal = lambda k: pow(5, k & (2 * N - 1), 2 * N)
    pts_n = n // 2 if name == "C4sum" else n
    els = set()
    for lazy, dbl in _pts_schedule(ctx, 1, pts_n):
        els.add(gal(dbl))
        if lazy is not None:
            els.add(gal(lazy))
    if name == "C4sum":
        els.add(2 * N - 1)
    keys = {g: lb.GadgetCiphertext(ctx, rand_evk(ctx, level, levelP, rng, dev), level, levelP) for g in sorted(els)}
    ev = lb.innersum.Evaluator(ctx, keys)
    rl = lb.Evaluator(ctx)
    ct = rand_rows(ctx.Q, N, batch * 2, rng, dev).view(batch, 2, level + 1, N)
    out_f, out_c = torch.empty_like(ct), torch.empty_like(ct)
    tmp = torch.empty_like(ct)

    def fused():
        if name == "C4sum":
            ev.InnerSum(ct, 1, n, out_f, N, bgv=True)
        else:                                     # InnerSum itself rejects n * batchSize = 7 (not a power of two)
            ev.RotateAndAdd(ct, 1, n, out_f)

    def composed():
        composed_pts(ctx, rl, keys, ct, 1, pts_n, out_c)
        if name == "C4sum":                       # RotateRows + Add
            rl.Automorphism(out_c, 2 * N - 1, keys[2 * N - 1], tmp)
            ctx.ringQ.Add(out_c.view(-1, level + 1, N), tmp.view(-1, level + 1, N), out_c.view(-1, level + 1, N))
    res = {}
    fused(); composed(); torch.cuda.synchronize()
    same = bool(torch.equal(out_f, out_c))
    Sl = lambda l: l * N * 8
    alg = batch * 4 * Sl(level + 1) + len(keys) * rand_evk_digits(level, levelP) * 2 * Sl(level + 1 + levelP + 1)
    for tag, fn in (("fused", fused), ("composed", composed)):
        launches = lb.lib().lgpu_launch_count()
        fn(); torch.cuda.synchronize()
        launches = lb.lib().lgpu_launch_count() - launches
        med, mn = timeit(fn, iters, 3, flush)
        res["%s_%s" % (name, tag)] = {"workload": desc + (" (one call)" if tag == "fused" else " (composed from existing entry points)"),
                                      "ms_per_batch": med * 1e3, "ct_per_s": batch / med, "alg_bytes_per_batch": alg, "alg_GBs": alg / med / 1e9,
                                      "launches_per_call": int(launches), "key_switches": len(_pts_schedule(ctx, 1, pts_n)) +
                                      sum(1 for lz, _ in _pts_schedule(ctx, 1, pts_n) if lz is not None) + (1 if name == "C4sum" else 0),
                                      "outputs_equal_fused_vs_composed": same}
    res["%s_fused" % name]["speedup_vs_composed"] = res["%s_composed" % name]["ms_per_batch"] / res["%s_fused" % name]["ms_per_batch"]
    del keys, ev
    ctx.close()
    return res


def _xpow2_ntt(ctx, level, div):
    """GenXPow2NTT (core/rlwe/ring_packing.go:773-810) on the device: X^(+-2^i) in the NTT domain, Montgomery form."""
    N, nq = ctx.N, level + 1
    ringQ = ctx.ringQ.AtLevel(level)
    x = torch.zeros((nq, N), dtype=torch.int64, device="cuda:0")
    for i, q in enumerate(ctx.Q[:nq]):
        x[i, N - 1 if div else 1] = int(((1 << 64) % q))
    ringQ.NTT(x, x)
    xs = [x]
    for _ in range(1, ctx.logN):
        y = torch.empty_like(x)
        ringQ.MulCoeffsMontgomery(xs[-1], xs[-1], y)
        xs.append(y)
    if div:
        ringQ.Neg(xs[0], xs[0])
    return [t.expand(2, nq, N).contiguous() for t in xs]


def _scale(ctx, level, x, s):
    """x *= 2^-s mod Q_level (MulScalarBigint) on a (2, level+1, N) ciphertext."""
    inv = [((pow(1 << s, -1, q)) << 64) % q for q in ctx.Q[: level + 1]]
    ctx.ringQ.AtLevel(level).MulRNSScalarMontgomery(x, inv, x)


def composed_expand(ctx, rl, keys, ct, logGap, xinv, out):
    """Expand(ct, logGap) of one NTT-domain ciphertext, one Evaluator.Automorphism per ciphertext plus vecops (ring_packing.go:457-571).
    out: (1, N >> logGap, 2, level+1, N); slot k holds cts[k << logGap]."""
    level, N, gap = ct.shape[-2] - 1, ctx.N, 1 << logGap
    ringQ = ctx.ringQ.AtLevel(level)
    cts = {0: out[0, 0]}
    cts[0].copy_(ct[0])
    _scale(ctx, level, cts[0], ctx.logN)
    tmp = torch.empty_like(cts[0])
    for i in range(ctx.logN):
        n = 1 << i
        g = N // n + 1
        for j in range(0, n, gap):
            c0 = cts[j]
            rl.Automorphism(c0, g, keys[g], tmp)
            if n >= gap:
                c1 = out[0, (j + n) // gap]
                ringQ.Sub(c0, tmp, c1)
                ringQ.Add(c0, tmp, c0)
                ringQ.MulCoeffsMontgomery(c1, xinv[i], c1)
                cts[j + n] = c1
            else:
                ringQ.Add(c0, tmp, c0)


def composed_pack(ctx, rl, keys, cts_in, xpow, out):
    """Repack(cts) = Pack(cts, LogN, true) of NTT-domain ciphertexts, one Evaluator.Automorphism per ciphertext plus vecops
    (ring_packing.go:600-770); cts_in is left as it was."""
    keys_sorted = sorted(cts_in)
    level, logN = cts_in[keys_sorted[0]].shape[-2] - 1, ctx.logN
    ringQ = ctx.ringQ.AtLevel(level)
    cts = {k: v.clone() for k, v in cts_in.items()}
    for v in cts.values():
        _scale(ctx, level, v, logN)
    tmpa = torch.empty_like(out)
    for i in range(logN):
        t = 1 << (logN - 1 - i)
        g = 2 * ctx.N - 1 if i == 0 else pow(5, 1 << (i - 1), 2 * ctx.N)
        for jx in range(t):
            a, b = cts.get(jx), cts.get(jx + t)
            if b is not None:
                ringQ.MulCoeffsMontgomery(b, xpow[logN - i - 1], b)
                if a is not None:
                    ringQ.Sub(a, b, tmpa)
                    ringQ.Add(a, b, a)
                else:
                    cts[jx] = b
                cts[jx + t] = None
            if a is not None:
                rl.Automorphism(tmpa if b is not None else a, g, keys[g], tmpa)
                ringQ.Add(a, tmpa, a)
            elif b is not None:
                rl.Automorphism(b, g, keys[g], tmpa)
                ringQ.Sub(b, tmpa, b)
    out.copy_(cts[0])


def bench_ringpacking(iters, rng, dev, flush):
    P, logN, level, logGap = presets.PRESETS["BGV_N15QP880"], 15, 3, 7
    ctx = lb.Context(logN, P["Q"], P["P"])
    N, levelP = ctx.N, len(P["P"]) - 1
    els = sorted(set(lb.ringpacking.GaloisElementsForExpand(ctx, logN)) | set(lb.ringpacking.GaloisElementsForPack(ctx, logN)))
    keys = {g: lb.GadgetCiphertext(ctx, rand_evk(ctx, level, levelP, rng, dev), level, levelP) for g in els}
    ev = lb.ringpacking.RingPackingEvaluator(ctx, keys, keys)
    rl = lb.Evaluator(ctx)
    S = N >> logGap
    ct = rand_rows(ctx.Q[: level + 1], N, 2, rng, dev).view(1, 2, level + 1, N)
    xinv, xpow = _xpow2_ntt(ctx, level, True), _xpow2_ntt(ctx, level, False)
    out_c = torch.empty((1, S, 2, level + 1, N), dtype=torch.int64, device=dev)
    got = {}
    packed_c = torch.empty((2, level + 1, N), dtype=torch.int64, device=dev)

    def expand_f():
        got["e"] = ev.Expand(ct, logGap)

    def expand_c():
        composed_expand(ctx, rl, keys, ct, logGap, xinv, out_c)
    expand_f(); expand_c(); torch.cuda.synchronize()
    cts = {k: v[0] for k, v in got["e"].items()}                     # (2, level+1, N) views of the device output

    def pack_f():
        got["p"] = ev.Repack(cts)

    def pack_c():
        composed_pack(ctx, rl, keys, cts, xpow, packed_c)
    pack_f(); pack_c(); torch.cuda.synchronize()
    same = {"C4expand": all(torch.equal(got["e"][k << logGap][0], out_c[0, k]) for k in range(S)), "C4pack": bool(torch.equal(got["p"], packed_c))}
    Sl = lambda l: l * N * 8
    key_bytes = rand_evk_digits(level, levelP) * 2 * Sl(level + 1 + levelP + 1)
    res = {}
    for name, f, c, desc in (("C4expand", expand_f, expand_c, "BGV N15QP880 at level 3, one ciphertext: Expand(logGap = 7) -> 256 ciphertexts"),
                             ("C4pack", pack_f, pack_c, "BGV N15QP880 at level 3: Repack of the 256 Expand outputs into one ciphertext")):
        for tag, fn in (("batched", f), ("per_ciphertext", c)):
            launches = lb.lib().lgpu_launch_count()
            fn(); torch.cuda.synchronize()
            launches = lb.lib().lgpu_launch_count() - launches
            med, mn = timeit(fn, iters, 2, flush)
            res["%s_%s" % (name, tag)] = {"workload": desc + (" (one call, one gadget product per tree step)" if tag == "batched" else
                                                              " (one Evaluator.Automorphism per ciphertext + vecops)"),
                                          "ms_per_call": med * 1e3, "ms_min": mn * 1e3, "launches_per_call": int(launches), "key_switches": 262,
                                          "galois_key_bytes": key_bytes, "outputs_equal_batched_vs_per_ciphertext": same[name]}
        res["%s_batched" % name]["speedup_vs_per_ciphertext"] = res["%s_per_ciphertext" % name]["ms_per_call"] / res["%s_batched" % name]["ms_per_call"]
    del keys, ev
    ctx.close()
    return res


def bench_apply_evk(iters, rng, dev, flush):
    P = presets.PRESETS["CKKS_PN16QP1761"]
    big, small = lb.Context(16, P["Q"], P["P"]), lb.Context(15, P["Q"], P["P"])
    level, levelP, B = len(P["Q"]) - 1, len(P["P"]) - 1, 64
    N, n, nq = big.N, small.N, level + 1
    key = lb.GadgetCiphertext(big, rand_evk(big, level, levelP, rng, dev), level, levelP)
    rl = lb.Evaluator(big)
    ringL, ringS = big.ringQ.AtLevel(level), small.ringQ.AtLevel(level)
    L = lb.lib()
    res = {}
    for name, n_in, n_out in (("C3aek_down", N, n), ("C3aek_up", n, N)):
        # the composed arm keeps the two components apart, as a shim on rlwe.Ciphertext polynomials does
        c0, c1 = rand_rows(big.Q, n_in, B, rng, dev), rand_rows(big.Q, n_in, B, rng, dev)
        ct = torch.stack([c0, c1], dim=1).contiguous()
        out_f = torch.empty((B, 2, nq, n_out), dtype=torch.int64, device=dev)
        o0, o1 = (torch.empty((B, nq, n_out), dtype=torch.int64, device=dev) for _ in range(2))
        ks0, ks1 = (torch.empty((B, nq, N), dtype=torch.int64, device=dev) for _ in range(2))
        g = torch.empty((2, B, nq, N), dtype=torch.int64, device=dev)   # GadgetProduct's two outputs in one block: the fused ModDown applies

        def fused():
            rl.ApplyEvaluationKey(ct, key, out_f)
        if n_out < n_in:
            def composed():
                rl.GadgetProduct(level, c1, key, g[0], g[1])
                ringL.Add(c0, g[0], g[0])
                ringL.INTT(g[0], g[0]); ringL.INTT(g[1], g[1])
                ringS.NTT(g[0][..., ::2].contiguous(), o0); ringS.NTT(g[1][..., ::2].contiguous(), o1)
        else:
            def composed():
                for src, dst in ((c0, ks0), (c1, ks1)):
                    lb._lib.check(L.lgpu_map_small_dimension_to_larger_dimension_ntt(big.h, ctypes.c_void_p(src.data_ptr()), n, ctypes.c_void_p(dst.data_ptr()), N,
                                                                                      B * nq, None))
                rl.GadgetProduct(level, ks1, key, g[0], g[1])
                ringL.Add(ks0, g[0], o0)                                  # component 1 is g[1]
        fused(); composed(); torch.cuda.synchronize()
        same = bool(torch.equal(out_f[:, 0], o0) and torch.equal(out_f[:, 1], o1 if n_out < n_in else g[1]))
        row = {"workload": "CKKS PN16QP1761, batch %d at level %d, NTT domain: ApplyEvaluationKey 2^%d -> 2^%d" % (B, level, n_in.bit_length() - 1,
                                                                                                                 n_out.bit_length() - 1),
               "outputs_equal_fused_vs_composed": same}
        for tag, fn in (("fused", fused), ("composed", composed)):
            launches = L.lgpu_launch_count()
            fn(); torch.cuda.synchronize()
            launches = L.lgpu_launch_count() - launches
            med, mn = timeit(fn, iters, 2, flush)
            row[tag] = {"ms_per_batch": med * 1e3, "ms_min": mn * 1e3, "ct_per_s": B / med, "launches_per_call": int(launches)}
        row["speedup_vs_composed"] = row["composed"]["ms_per_batch"] / row["fused"]["ms_per_batch"]
        res[name] = row
        del c0, c1, ct, out_f, o0, o1, ks0, ks1, g
    del key
    big.close(); small.close()
    return res


def rand_evk_digits(levelQ, levelP):
    return (levelQ + levelP + 1) // (levelP + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="bench_out/configs.json")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    rng = np.random.default_rng(20260922)
    flush = torch.zeros(256 << 20, dtype=torch.uint8, device=dev)   # 256 MiB > the 126 MB L2
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "timing": "cuda events, median of %d, L2 flushed before every iteration" % args.iters}
    want = set(args.only.split(",")) if args.only else None

    def on(name):
        return want is None or name in want

    if on("C1"):
        ctx = lb.Context(12, presets.QI60[:1])
        x = rand_rows(ctx.Q, ctx.N, 1, rng, dev)[0]
        y = ctx.ringQ.NewPoly()

        def f():
            ctx.ringQ.NTT(x, y); ctx.ringQ.INTT(y, y)
        med, mn = timeit(f, args.iters * 5, 5, flush)
        res["C1"] = {"workload": "N=4096 l=1 q=Qi60[0]: NTT then INTT", "us_median": med * 1e6, "us_min": mn * 1e6}
        ctx.close()

    if on("C2"):
        N, nl = 1 << 16, 44
        S = nl * N * 8
        for tag, Q in (("q61", presets.QI60[:32] + presets.PI60[:12]), ("ckks45", presets.PRESETS["CKKS_L44"]["Q"][:nl])):
            ctx = lb.Context(16, Q)
            for batch in (1, 16):
                x = rand_rows(Q, N, batch, rng, dev); y = torch.empty_like(x); z = torch.empty_like(x); w = rand_rows(Q, N, batch, rng, dev)

                def ntt():
                    ctx.ringQ.NTT(x, y)

                def ntt_mul():
                    ctx.ringQ.NTT(x, y); ctx.ringQ.MulCoeffsMontgomery(y, w, z)
                def ntt_mul_fused():
                    ctx.ringQ.NTTThenMulCoeffsMontgomery(x, w, z)
                m1, _ = timeit(ntt, args.iters, 3, flush)
                m2, _ = timeit(ntt_mul, args.iters, 3, flush)
                m3, _ = timeit(ntt_mul_fused, args.iters, 3, flush)
                res["C2_%s_batch%d" % (tag, batch)] = {
                    "workload": "N=65536 l=44 (%s primes), %d polynomial(s) per call" % (tag, batch),
                    "ntt_us": m1 * 1e6, "ntt_alg_GBs": 2 * S * batch / m1 / 1e9,
                    "ntt_mul_us": m2 * 1e6, "ntt_mul_alg_GBs_unfused": 5 * S * batch / m2 / 1e9,
                    "ntt_mul_fused_us": m3 * 1e6, "ntt_mul_fused_alg_GBs": 3 * S * batch / m3 / 1e9, "ntt_mul_fused_speedup": m2 / m3,
                    "us_per_limb_ntt": m1 * 1e6 / (nl * batch)}
            ctx.close()

    if on("C3"):
        P = presets.PRESETS["CKKS_PN16QP1761"]
        ctx = lb.Context(16, P["Q"], P["P"])
        level, levelP, batch = len(P["Q"]) - 1, len(P["P"]) - 1, 64
        evk = lb.GadgetCiphertext(ctx, rand_evk(ctx, level, levelP, rng, dev), level, levelP)
        ev = lb.CKKSEvaluator(ctx, evk)
        a = rand_rows(ctx.Q, ctx.N, batch * 2, rng, dev).view(batch, 2, level + 1, ctx.N)
        b = rand_rows(ctx.Q, ctx.N, batch * 2, rng, dev).view(batch, 2, level + 1, ctx.N)
        med, mn = timeit(lambda: ev.MulRelinRescaleNew(a, b), args.iters, 3, flush)
        Sl = lambda l: l * ctx.N * 8
        alg = batch * (4 * Sl(level + 1) + 2 * Sl(level)) + evk.struct.n_digits * 2 * Sl(level + 1 + levelP + 1)
        res["C3"] = {"workload": "CKKS PN16QP1761, batch 64 pairs at level 33: MulRelin + Rescale", "ms_per_batch": med * 1e3,
                     "ct_per_s": batch / med, "alg_bytes_per_batch": alg, "alg_GBs": alg / med / 1e9}
        ctx.close()

    if on("C4"):
        P = presets.PRESETS["BGV_N15QP880"]
        ctx = lb.Context(15, P["Q"], P["P"])
        level, levelP, batch = len(P["Q"]) - 1, len(P["P"]) - 1, 128
        gk = lb.GadgetCiphertext(ctx, rand_evk(ctx, level, levelP, rng, dev), level, levelP)
        ev = lb.Evaluator(ctx)
        ct = rand_rows(ctx.Q, ctx.N, batch * 2, rng, dev).view(batch, 2, level + 1, ctx.N)
        out = torch.empty_like(ct)
        gal = pow(5, 1, 2 * ctx.N)
        med, mn = timeit(lambda: ev.Automorphism(ct, gal, gk, out), args.iters, 3, flush)
        Sl = lambda l: l * ctx.N * 8
        alg = batch * 4 * Sl(level + 1) + gk.struct.n_digits * 2 * Sl(level + 1 + levelP + 1) + ctx.N * 8
        res["C4"] = {"workload": "BGV N15QP880, batch 128 at level 19: Evaluator.Automorphism (rotate by 1)", "ms_per_batch": med * 1e3,
                     "ct_per_s": batch / med, "alg_bytes_per_batch": alg, "alg_GBs": alg / med / 1e9}
        ctx.close()

    if on("C4mul"):
        P = presets.PRESETS["BGV_N15QP880"]
        ctx = lb.Context(15, P["Q"], P["P"])
        level, levelP, batch = len(P["Q"]) - 1, len(P["P"]) - 1, 128
        rlk = lb.GadgetCiphertext(ctx, rand_evk(ctx, level, levelP, rng, dev), level, levelP)
        a = rand_rows(ctx.Q, ctx.N, batch * 2, rng, dev).view(batch, 2, level + 1, ctx.N)
        b = rand_rows(ctx.Q, ctx.N, batch * 2, rng, dev).view(batch, 2, level + 1, ctx.N)
        Sl = lambda l: l * ctx.N * 8
        key = rlk.struct.n_digits * 2 * Sl(level + 1 + levelP + 1)
        for name, si, out_limbs in (("C4mul_bgv", False, level), ("C4mul_bfv", True, level + 1)):
            ev = lb.BGVEvaluator(ctx, P["T"], P["QMul"], rlk, scale_invariant=si)
            fn = (lambda: ev.MulRelinNew(a, b)) if si else (lambda: ev.MulRelinRescaleNew(a, b))
            med, mn = timeit(fn, args.iters, 3, flush)
            alg = batch * (4 * Sl(level + 1) + 2 * Sl(out_limbs)) + key
            res[name] = {"workload": "BGV N15QP880 (t = 65537, 12 QMul primes), batch 128 pairs at level 19: "
                         + ("MulRelinScaleInvariant (BFV)" if si else "MulRelin + Rescale (BGV)"),
                         "ms_per_batch": med * 1e3, "ct_per_s": batch / med, "alg_bytes_per_batch": alg, "alg_GBs": alg / med / 1e9}
            ev.close()
        ctx.close()

    for name in ("C4sum", "C3sum"):
        if on(name):
            res.update(bench_innersum(name, args.iters, rng, dev, flush))

    if on("C4expand") or on("C4pack"):
        res.update(bench_ringpacking(args.iters, rng, dev, flush))

    if on("C3aek"):
        res.update(bench_apply_evk(args.iters, rng, dev, flush))

    if on("BOOT"):
        P = presets.PRESETS["BOOT_N16QP1767"]
        ctx = lb.Context(16, P["Q"], P["P"])
        level, levelP, batch = len(P["Q"]) - 1, len(P["P"]) - 1, 32
        evk = lb.GadgetCiphertext(ctx, rand_evk(ctx, level, levelP, rng, dev), level, levelP)
        ev = lb.CKKSEvaluator(ctx, evk)
        for lv in (level, 25):
            a = rand_rows(ctx.Q[: lv + 1], ctx.N, batch * 2, rng, dev).view(batch, 2, lv + 1, ctx.N)
            b = rand_rows(ctx.Q[: lv + 1], ctx.N, batch * 2, rng, dev).view(batch, 2, lv + 1, ctx.N)
            med, mn = timeit(lambda: ev.MulRelinRescaleNew(a, b), args.iters, 3, flush)
            nd_lv = (lv + levelP + 1) // (levelP + 1)
            res["BOOT_level%d" % lv] = {"workload": "N16QP1767H32768H32 chain (30 Q limbs 60/40/39/60/56 bits, 6 x 61-bit P), batch 32 pairs at level %d: MulRelin + Rescale" % lv,
                                        "ms_per_batch": med * 1e3, "ct_per_s": batch / med, "digits": nd_lv,
                                        "us_per_ct_per_row_digit": med * 1e6 / batch / ((lv + 1 + levelP + 1) * nd_lv)}
        ctx.close()
        # the same cost figure for the 45-bit chain (C3) is C3.ms_per_batch / 64 / ((34 + 4) * 9)
        if "C3" in res:
            res["C3"]["us_per_ct_per_row_digit"] = res["C3"]["ms_per_batch"] * 1e3 / 64 / (38 * 9)

    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

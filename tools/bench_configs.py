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
"""
import argparse
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

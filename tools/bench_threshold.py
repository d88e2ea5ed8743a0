"""Thresholdizer.GenShamirSecretShares (lattigo_b200.multiparty, lgpu_mp_shamir_share) on one GPU at CKKS_PN16QP1761 (N = 2^16,
34 Q limbs, 4 P limbs; one share S = 38 rows x N words = 19.9 MB): one party's shares of a degree t - 1 Shamir polynomial for n
recipients, n in {8, 16, 32} and t in {2, 4, 8, 16}, next to the same shares from n calls of the ring API's RingQP.EvalPolyScalar (the
reference's chain of MulScalar and Add per ring), outputs asserted equal.
  alg_bytes    (t + n) S: read every coefficient once, write every share once;
  model_bytes  (ceil(n / 8) t + n) S: what the kernel moves, re-reading the coefficients once per chunk of 8 points.
Each is timed with CUDA events around one call, after a warm-up, as the median (and minimum) of --iters runs, with a 256 MB buffer
rewritten before every run so that no operand starts in L2. Bandwidth shares are against the H100 SXM data-sheet 3.35 TB/s. The card's
name and power limit are read in the same run. Writes JSON (default: bench_out/threshold.json); bench.py stays the contract benchmark."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402
from lattigo_b200.ringqp import Poly, RingQP  # noqa: E402
from tools.bench_encoder import gpu_info, timed  # noqa: E402

PEAK_BPS = 3.35e12
CHUNK = 8                  # kShamirPts in csrc/multiparty.cu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=os.path.join("bench_out", "threshold.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_threshold.py needs a CUDA device"
    assert args.iters >= 5
    name, limit = gpu_info()
    pr = PRESETS["CKKS_PN16QP1761"]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    nq, npp = len(pr["Q"]), len(pr["P"])
    flush = torch.zeros(32 << 20, dtype=torch.float64, device="cuda")
    S = lb.encryptor.Samplers(ctx, 1)
    thr = lb.multiparty.Thresholdizer(ctx, S)
    rqp = RingQP(ctx)
    sk = S.UniformQP(nq - 1, npp - 1)[0]
    share_bytes = sk.numel() * 8
    rep = {"gpu": name, "power_limit_w": limit, "params": "CKKS_PN16QP1761", "iters": args.iters, "share_bytes": share_bytes, "workloads": {}}
    for t in (2, 4, 8, 16):
        poly = thr.GenShamirPolynomial(t, sk)
        coeffs = [Poly(poly[i, :nq].contiguous(), poly[i, nq:].contiguous()) for i in range(t)]
        for n in (8, 16, 32):
            points = list(range(1, n + 1))
            med, mn = timed(lambda: thr.GenShamirSecretShares(points, poly), args.iters, flush)
            outs = [Poly(ctx.new_poly(nq), ctx.new_poly(npp)) for _ in range(n)]

            def unfused():
                for k in range(n):
                    rqp.EvalPolyScalar(coeffs, points[k], outs[k])
            umed, umn = timed(unfused, args.iters, flush)
            fused = thr.GenShamirSecretShares(points, poly)
            for k in range(n):
                assert torch.equal(fused[k, :nq], outs[k].Q) and torch.equal(fused[k, nq:], outs[k].P), "fused and unfused shares differ"
            del fused, outs
            alg = (t + n) * share_bytes
            model = (-(-n // CHUNK) * t + n) * share_bytes
            rep["workloads"]["t%d_n%d" % (t, n)] = {
                "t": t, "n": n, "ms": med, "ms_min": mn, "alg_bytes": alg, "model_bytes": model, "alg_GBps": alg / med / 1e6,
                "share_of_3.35TBps": alg / (med * 1e-3) / PEAK_BPS, "model_share_of_3.35TBps": model / (med * 1e-3) / PEAK_BPS,
                "unfused_ms": umed, "unfused_ms_min": umn, "unfused_model_bytes": n * (2 + 5 * (t - 1)) * share_bytes, "speedup": umed / med}
        del poly, coeffs
        torch.cuda.empty_cache()
    ctx.close()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit,
                      **{k: [round(w["ms"], 3), round(w["unfused_ms"], 3)] for k, w in rep["workloads"].items()}}))


if __name__ == "__main__":
    main()

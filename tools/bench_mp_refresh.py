"""Collective BGV refresh and masked transform (lattigo_b200.mpbgv) on one GPU at BGV_N15QP880 (N = 2^15, 20 Q limbs), t = 0x10001,
128 ciphertexts at level 19, K = 4 parties:
  refresh_genshare     RefreshProtocol.GenShare of one party (E2S at level 19, S2E at level 19), mask and smudging noise given;
  refresh_aggregate    AggregateShares of the K parties' RefreshShares (one fold per component);
  refresh_finalize     RefreshProtocol.Finalize: Add(aggE2S, c0), INTT, RingQ2T, RingT2Q, NTT, Add(aggS2E), c1 = crp;
  transform_genshare / transform   MaskedTransformProtocol.GenShare / Transform with Decode + a slot permutation + Encode.
On CKKS_PN16QP1761 (64 ciphertexts at level 33, K = 4, scale 2^45, full slots): mpckks RefreshProtocol.GenShare of one party from the
minimum refresh level (GetMinimumLevelForRefresh) back to level 33, and Finalize.
Finalize's algorithmic minimum traffic: read the aggregated S2E share, the CRP, the input c0 and the aggregated E2S share, write c0 and
c1 once; its share of the H100 SXM data-sheet 3.35 TB/s is reported against that minimum. Each workload is timed with CUDA events around
one call after a warm-up, median (and minimum) of --iters runs, with a 256 MB buffer rewritten before every run so that no operand starts
in L2. The card's name and power limit are read in the same run. Writes JSON (default: bench_out/mp_refresh.json)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402
from tools.bench_encoder import gpu_info, timed  # noqa: E402

PEAK_BPS = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--parties", type=int, default=4)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=os.path.join("bench_out", "mp_refresh.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mp_refresh.py needs a CUDA device"
    assert args.iters >= 5
    name, limit = gpu_info()
    pr = PRESETS["BGV_N15QP880"]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    enc = lb.BGVEncoder(ctx, pr["T"])
    N, L, B, K = ctx.N, len(pr["Q"]) - 1, args.batch, args.parties
    flush = torch.zeros(32 << 20, dtype=torch.float64, device="cuda")
    crs = lb.encryptor.Samplers(ctx, 1)
    party = [lb.encryptor.Samplers(ctx, 100 + i) for i in range(K)]
    sks = [party[i].UniformQP(L, len(pr["P"]) - 1)[0] for i in range(K)]
    ct = crs.Uniform(lb.ring.RING_Q, L, batch=2 * B).view(B, 2, L + 1, N)
    protos = [lb.mpbgv.RefreshProtocol(enc, party[i], 3.2) for i in range(K)]
    crp = protos[0].SampleCRP(L, crs, B)
    p0 = protos[0]
    e0 = party[0].Gaussian(p0.e2s.cks.sigma, p0.e2s.cks.bound, B)
    e1 = party[0].Gaussian(p0.s2e.cks.sigma, p0.s2e.cks.bound, B)
    mask = p0.e2s.SampleMask(B)
    rep = {"gpu": name, "power_limit_w": limit, "params": "BGV_N15QP880", "t": pr["T"], "batch": B, "parties": K, "level": L,
           "iters": args.iters, "workloads": {}}
    W = rep["workloads"]

    med, mn = timed(lambda: p0.GenShare(sks[0], ct, crp, 1, e_e2s=e0, e_s2e=e1, mask=mask), args.iters, flush)
    W["refresh_genshare"] = {"ms": med, "ms_min": mn}
    shares = [p.GenShare(sks[i], ct, crp, 1) for i, p in enumerate(protos)]
    med, mn = timed(lambda: p0.AggregateShares(shares), args.iters, flush)
    W["refresh_aggregate"] = {"ms": med, "ms_min": mn}
    agg = p0.AggregateShares(shares)
    del shares
    med, mn = timed(lambda: p0.Finalize(ct, crp, agg, 1), args.iters, flush)
    poly = B * (L + 1) * N * 8
    alg = 4 * poly + 2 * poly
    W["refresh_finalize"] = {"ms": med, "ms_min": mn, "alg_bytes": alg, "alg_GBps": alg / med / 1e6, "share_of_3.35TBps": alg / (med * 1e-3) / PEAK_BPS}
    del agg
    torch.cuda.empty_cache()

    perm = torch.randperm(enc.n, device="cuda")

    def permute(c):
        c.copy_(c[:, perm])
    tf = lb.mpbgv.MaskedTransformFunc(True, permute, True)
    mt = [lb.mpbgv.MaskedTransformProtocol(enc, party[i], 3.2) for i in range(K)]
    med, mn = timed(lambda: mt[0].GenShare(sks[0], sks[0], ct, crp, tf, 1, e_e2s=e0, e_s2e=e1, mask=mask), args.iters, flush)
    W["transform_genshare"] = {"ms": med, "ms_min": mn}
    agg = mt[0].AggregateShares([m.GenShare(sks[i], sks[i], ct, crp, tf, 1) for i, m in enumerate(mt)])
    med, mn = timed(lambda: mt[0].Transform(ct, tf, crp, agg, 1), args.iters, flush)
    W["transform"] = {"ms": med, "ms_min": mn}
    enc.close()
    ctx.close()
    del ct, crp, sks, agg, mask, e0, e1
    torch.cuda.empty_cache()

    # CKKS_PN16QP1761: 64 ciphertexts at level 33, E2S at the minimum refresh level, S2E back to level 33
    cp = PRESETS["CKKS_PN16QP1761"]
    ctx = lb.Context(cp["logN"], cp["Q"], cp["P"])
    N, L, B = ctx.N, 33, 64
    log_scale, log_slots = 45, cp["logN"] - 1
    crs = lb.encryptor.Samplers(ctx, 1)
    party = [lb.encryptor.Samplers(ctx, 200 + i) for i in range(K)]
    sks = [party[i].UniformQP(len(cp["Q"]) - 1, len(cp["P"]) - 1)[0] for i in range(K)]
    ct = crs.Uniform(lb.ring.RING_Q, L, batch=2 * B).view(B, 2, L + 1, N)
    protos = [lb.mpckks.RefreshProtocol(ctx, party[i], 3.2, 2 ** log_scale) for i in range(K)]
    lmin, log_bound, ok = lb.mpckks.GetMinimumLevelForRefresh(128, 2.0 ** log_scale, K, cp["Q"])
    assert ok
    crp = protos[0].SampleCRP(L, crs, B)
    p0 = protos[0]
    e0 = party[0].Gaussian(p0.e2s.cks.sigma, p0.e2s.cks.bound, B)
    e1 = party[0].Gaussian(p0.s2e.cks.sigma, p0.s2e.cks.bound, B)
    words = lb.mpckks.share_words(ctx, lmin)
    mask = p0.e2s.SampleMask(log_slots, log_bound, words, B)
    scale = 2 ** log_scale
    rep["ckks"] = {"params": "CKKS_PN16QP1761", "batch": B, "parties": K, "level": L, "e2s_level": lmin, "log_bound": log_bound, "share_words": words}
    med, mn = timed(lambda: p0.GenShare(sks[0], log_bound, ct, crp, scale, log_slots, level=lmin, e_e2s=e0, e_s2e=e1, mask=mask), args.iters, flush)
    W["ckks_refresh_genshare"] = {"ms": med, "ms_min": mn}
    agg = p0.AggregateShares([p.GenShare(sks[i], log_bound, ct, crp, scale, log_slots, level=lmin) for i, p in enumerate(protos)])
    med, mn = timed(lambda: p0.Finalize(ct, crp, agg, scale, log_slots), args.iters, flush)
    pin, pout = B * (lmin + 1) * N * 8, B * (L + 1) * N * 8
    alg = 2 * pin + 2 * pout + 2 * pout                 # read c0 and the E2S share at lmin, the S2E share and the CRP; write c0, c1
    W["ckks_refresh_finalize"] = {"ms": med, "ms_min": mn, "alg_bytes": alg, "alg_GBps": alg / med / 1e6,
                                   "share_of_3.35TBps": alg / (med * 1e-3) / PEAK_BPS}
    ctx.close()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit, **{k: round(w["ms"], 3) for k, w in W.items()}}))


if __name__ == "__main__":
    main()

"""Threshold-protocol shares (lattigo_b200.multiparty) on one GPU at CKKS_PN16QP1761 (N = 2^16, 34 Q limbs, 4 P limbs):
  aggregate_K  lgpu_mp_aggregate of K in {2, 4, 8, 16} shares the size of a relinearization-key round-one share (beta = 9 gadget
               entries x 2 components x 38 rows x N words, S = 359 MB), next to the same fold as K - 1 binary Ring.Add calls on the same
               inputs (outputs asserted equal). Algorithmic bytes: (K + 1) S for the one-pass fold (read K shares, write one);
  cks_share    KeySwitchProtocol.GenShare of 64 ciphertexts at level 33;
  pcks_share   PublicKeySwitchProtocol.GenShare of 64 ciphertexts at level 33;
  rkg_round_one / rkg_round_two   RelinearizationKeyGenProtocol shares of one party;
  gkg_16       GaloisKeyGenProtocol.GenShare for 16 Galois elements in one call, on BOOT_N16QP1767.
Each is timed with CUDA events around one call, after a warm-up, as the median (and minimum) of --iters runs, with a 256 MB buffer
rewritten before every run so that no operand starts in L2. Bandwidth shares are against the H100 SXM data-sheet 3.35 TB/s. The card's
name and power limit are read in the same run. Writes JSON (default: bench_out/multiparty.json); bench.py stays the contract benchmark."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402
from tools.bench_encoder import gpu_info, timed  # noqa: E402

PEAK_BPS = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=os.path.join("bench_out", "multiparty.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_multiparty.py needs a CUDA device"
    assert args.iters >= 5
    name, limit = gpu_info()
    pr = PRESETS["CKKS_PN16QP1761"]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    N, L, LP = ctx.N, len(pr["Q"]) - 1, len(pr["P"]) - 1
    flush = torch.zeros(32 << 20, dtype=torch.float64, device="cuda")
    crs = lb.encryptor.Samplers(ctx, 1)
    rep = {"gpu": name, "power_limit_w": limit, "params": "CKKS_PN16QP1761", "iters": args.iters, "workloads": {}}

    entries = 2 * 9                                   # (digit, component) blocks of an RKG round-one share with BaseTwoDecomposition 0
    shares = [crs.UniformQP(L, LP, batch=entries) for _ in range(16)]
    S = shares[0].numel() * 8
    ringQP_add = [(lb.ring.Ring(ctx, lb.ring.RING_Q, L), slice(0, L + 1)), (lb.ring.Ring(ctx, lb.ring.RING_P, LP), slice(L + 1, L + 2 + LP))]
    qs = torch.empty_like(shares[0][:, : L + 1]); ps = torch.empty_like(shares[0][:, L + 1:])
    out = torch.empty_like(shares[0])

    def binary_fold(K):
        # the reference's composition: agg = s0; agg = Add(agg, s_k), one Ring.Add per ring and share
        qs.copy_(shares[0][:, : L + 1]); ps.copy_(shares[0][:, L + 1:])
        for k in range(1, K):
            ringQP_add[0][0].Add(qs, shares[k][:, : L + 1].contiguous(), qs)
            ringQP_add[1][0].Add(ps, shares[k][:, L + 1:].contiguous(), ps)
        return torch.cat([qs, ps], dim=1)

    for K in (2, 4, 8, 16):
        med, mn = timed(lambda: lb.multiparty.aggregate(ctx, L, LP, shares[:K], out=out), args.iters, flush)
        assert torch.equal(out, binary_fold(K)), "the one-pass fold differs from K - 1 binary Adds"
        # the binary composition's Adds alone (its slicing copies are not charged to it)
        sq = [s[:, : L + 1].contiguous() for s in shares[:K]]; sp = [s[:, L + 1:].contiguous() for s in shares[:K]]

        def adds():
            for k in range(1, K):
                ringQP_add[0][0].Add(qs, sq[k], qs)
                ringQP_add[1][0].Add(ps, sp[k], ps)
        bmed, bmn = timed(adds, args.iters, flush)
        del sq, sp
        alg = (K + 1) * S
        rep["workloads"]["aggregate_%d" % K] = {"share_bytes": S, "ms": med, "ms_min": mn, "alg_bytes": alg, "alg_GBps": alg / med / 1e6,
                                                "share_of_3.35TBps": alg / (med * 1e-3) / PEAK_BPS,
                                                "binary_adds_ms": bmed, "binary_adds_alg_bytes": 3 * (K - 1) * S}
    del shares, out, qs, ps
    torch.cuda.empty_cache()

    B = args.batch
    party = lb.encryptor.Samplers(ctx, 2)
    s_in = party.UniformQP(L, LP)[0]; s_out = party.UniformQP(L, LP)[0]
    ct = party.Uniform(lb.ring.RING_Q, L, batch=2 * B).view(B, 2, L + 1, N)
    pk = party.UniformQP(L, LP, batch=2)
    cks = lb.multiparty.KeySwitchProtocol(ctx, party, 8 * 3.2)
    pcks = lb.multiparty.PublicKeySwitchProtocol(ctx, party, 8 * 3.2)
    e = party.Gaussian(cks.sigma, cks.bound, B)
    u, e0, e1, ef = party.Ternary(P=2 / 3, batch=B), party.Gaussian(batch=B), party.Gaussian(batch=B), party.Gaussian(8 * 3.2, 6 * 8 * 3.2, B)
    runs = {"cks_share": lambda: cks.GenShare(s_in, s_out, ct, e=e),
            "pcks_share": lambda: pcks.GenShare(s_in, pk, ct, u, e0, e1, ef)}
    for k, fn in runs.items():
        med, mn = timed(fn, args.iters, flush)
        rep["workloads"][k] = {"batch": B, "level": L, "ms": med, "ms_min": mn}
    rkg = lb.multiparty.RelinearizationKeyGenProtocol(ctx, party)
    crp = rkg.SampleCRP(crs)
    eph, r1 = rkg.GenShareRoundOne(s_in, crp)
    med, mn = timed(lambda: rkg.GenShareRoundOne(s_in, crp), args.iters, flush)
    rep["workloads"]["rkg_round_one"] = {"share_bytes": r1.numel() * 8, "ms": med, "ms_min": mn}
    med, mn = timed(lambda: rkg.GenShareRoundTwo(eph, s_in, r1), args.iters, flush)
    rep["workloads"]["rkg_round_two"] = {"share_bytes": r1.numel() * 4, "ms": med, "ms_min": mn}
    del crp, eph, r1
    ctx.close()
    torch.cuda.empty_cache()
    bp = PRESETS["BOOT_N16QP1767"]
    ctx = lb.Context(bp["logN"], bp["Q"], bp["P"])
    S = lb.encryptor.Samplers(ctx, 3)
    gkg = lb.multiparty.GaloisKeyGenProtocol(ctx, S)
    els = [int(lb.lib().lgpu_galois_element(ctx.h, k)) for k in range(1, 16)] + [2 * ctx.N - 1]
    sk = S.UniformQP(len(bp["Q"]) - 1, len(bp["P"]) - 1)[0]
    gcrp = gkg.SampleCRP(S, len(els))
    med, mn = timed(lambda: gkg.GenShare(sk, els, gcrp), args.iters, flush)
    rep["workloads"]["gkg_16"] = {"params": "BOOT_N16QP1767", "n_keys": len(els), "share_bytes": gcrp.numel() * 8, "ms": med, "ms_min": mn}
    ctx.close()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit, **{k: round(w["ms"], 3) for k, w in rep["workloads"].items()}}))


if __name__ == "__main__":
    main()

"""Batched key generation on one GPU:
  brk_ref      rgsw.GenEvaluationKeyNew (lgpu_blind_rotation_gen_evaluation_key) at blindrot_test.go's shape: N = 2^10 over 0x7fff801,
               N_LWE = 2^9, BaseTwoDecomposition 7, window 10 (512 RGSW ciphertexts, 11 Galois keys);
  brk_ss       the same at examples/singleparty/ckks_scheme_switching's shape: N = 2^12, Q = [0x800004001, 0x40002001],
               P = [0x4000026001], N_LWE = 2^11, BaseTwoDecomposition 12 (2048 RGSW ciphertexts, 11 Galois keys);
  gal16        KeyGenerator.GenGaloisKeysNew for 16 Galois elements on BOOT_N16QP1767 in one lgpu_gen_galois_keys call, next to the
               per-key loop a caller had before it (AutomorphismNTT of sk, then lgpu_gen_evaluation_key, 16 times) on the same samples;
               the two arms' keys are compared word for word.
Each is timed with CUDA events around one call, after a warm-up, as the median (and minimum) of --iters runs, with a 256 MB buffer
rewritten before every run. Reported: key bytes written per second (the keys' words over the call time) and the kernel launches of one
call (lgpu_launch_count). The card's name and power limit are read in the same run. Writes JSON (default: bench_out/keygen.json)."""
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


def launches(fn):
    n0 = lb.lib().lgpu_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(lb.lib().lgpu_launch_count() - n0)


def ternary_sk(ctx, S):
    """(nQ + nP, N) NTT + Montgomery secret key from a device ternary sample, and its first row's centred values."""
    s = S.Ternary(P=2.0 / 3.0)
    levelQ, levelP = len(ctx.Q) - 1, len(ctx.P) - 1
    out = lb.encryptor.small_poly_to_rns(ctx, s, levelQ, levelP)
    q, p = (out[0], out[1]) if levelP >= 0 else (out, None)
    ctx.ringQ.NTT(q, q); ctx.ringQ.MForm(q, q)
    if p is not None:
        ctx.ringP.NTT(p, p); ctx.ringP.MForm(p, p)
    return (torch.cat([q[0], p[0]]) if p is not None else q[0]).contiguous()


def brk_workload(name, logN, Q, P, logN_lwe, Q_lwe, P_lwe, pw2, iters, flush):
    ctx, ctx_lwe = lb.Context(logN, Q, P), lb.Context(logN_lwe, Q_lwe, P_lwe)
    sk = ternary_sk(ctx, lb.encryptor.Samplers(ctx, 1))
    sk_lwe = ternary_sk(ctx_lwe, lb.encryptor.Samplers(ctx_lwe, 2))
    keep = {}

    def run():
        keep.clear()
        keep["k"] = lb.rgsw.GenEvaluationKeyNew(ctx, sk, ctx_lwe, sk_lwe, pw2=pw2, window_size=10, seed=5)
    med, mn = timed(run, iters, flush)
    brk, gks = keep["k"]
    key_bytes = sum(c.Value[v].data.numel() * 8 for c in brk for v in range(2)) + sum(g.data.numel() * 8 for g in gks.values())
    n = launches(run)
    keep.clear()
    ctx.close(); ctx_lwe.close()
    torch.cuda.empty_cache()
    return {"logN": logN, "logN_lwe": logN_lwe, "n_rgsw": 1 << logN_lwe, "n_galois_keys": 11, "BaseTwoDecomposition": pw2,
            "key_bytes": key_bytes, "ms": med, "ms_min": mn, "key_GBps": key_bytes / (med * 1e-3) / 1e9, "launches_per_call": n}


def gal_workload(iters, flush):
    bp = PRESETS["BOOT_N16QP1767"]
    ctx = lb.Context(bp["logN"], bp["Q"], bp["P"])
    S = lb.encryptor.Samplers(ctx, 3)
    sk = ternary_sk(ctx, S)
    L, LP = len(bp["Q"]) - 1, len(bp["P"]) - 1
    nQ, N = L + 1, ctx.N
    els = [int(lb.lib().lgpu_galois_element(ctx.h, k)) for k in range(1, 16)] + [2 * N - 1]
    kg = lb.encryptor.KeyGenerator(ctx)
    nd, sizes = lb.encryptor.gadget_layout(ctx, L, LP, 0)
    rows = L + 1 + LP + 1
    a = S.UniformQP(L, LP, batch=len(els) * nd).view(len(els), nd, 1, rows, N)
    e = S.Gaussian(batch=len(els) * nd).view(len(els), nd, 1, N)
    out = {}

    def batched():
        out["b"] = kg.GenGaloisKeysNew(els, sk, L, LP, 0, a=a, e=e)

    sk_out = torch.empty_like(sk)

    def per_key():
        keys = []
        for k, g in enumerate(els):
            inv = pow(g, -1, 2 * N)
            ctx.ringQ.AutomorphismNTT(sk[:nQ], inv, sk_out[:nQ])
            ctx.ringP.AutomorphismNTT(sk[nQ:], inv, sk_out[nQ:])
            keys.append(kg.GenEvaluationKey(sk[:nQ], sk_out, a[k], e[k]))
        out["l"] = keys

    med_b, mn_b = timed(batched, iters, flush)
    med_l, mn_l = timed(per_key, iters, flush)
    n_b, n_l = launches(batched), launches(per_key)
    same = all(torch.equal(x.data, y.data) for x, y in zip(out["b"], out["l"]))
    key_bytes = sum(k.data.numel() * 8 for k in out["b"])
    out.clear()
    ctx.close()
    return {"params": "BOOT_N16QP1767", "n_keys": len(els), "key_bytes": key_bytes,
            "batched": {"ms": med_b, "ms_min": mn_b, "key_GBps": key_bytes / (med_b * 1e-3) / 1e9, "launches_per_call": n_b},
            "per_key_loop": {"ms": med_l, "ms_min": mn_l, "key_GBps": key_bytes / (med_l * 1e-3) / 1e9, "launches_per_call": n_l},
            "outputs_equal": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=os.path.join("bench_out", "keygen.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_keygen.py needs a CUDA device"
    assert args.iters >= 5
    name, limit = gpu_info()
    flush = torch.zeros(32 << 20, dtype=torch.float64, device="cuda")
    rep = {"gpu": name, "power_limit_w": limit, "iters": args.iters, "workloads": {}}
    rep["workloads"]["brk_ref"] = brk_workload("brk_ref", 10, [0x7fff801], [], 9, [0x3001], [], 7, args.iters, flush)
    rep["workloads"]["brk_ss"] = brk_workload("brk_ss", 12, [0x800004001, 0x40002001], [0x4000026001], 11, [0x800004001], [0x42001], 12,
                                              args.iters, flush)
    rep["workloads"]["gal16"] = gal_workload(args.iters, flush)
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    w = rep["workloads"]
    print(json.dumps({"gpu": name, "power_limit_w": limit, "brk_ref_ms": round(w["brk_ref"]["ms"], 3), "brk_ss_ms": round(w["brk_ss"]["ms"], 3),
                      "gal16_batched_ms": round(w["gal16"]["batched"]["ms"], 3), "gal16_loop_ms": round(w["gal16"]["per_key_loop"]["ms"], 3),
                      "gal16_outputs_equal": w["gal16"]["outputs_equal"]}))


if __name__ == "__main__":
    main()

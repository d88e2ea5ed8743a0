"""CKKS encoding and decoding (ckks.Encoder Embed / DecodePublic) on one GPU: CKKS_PN16QP1761 (N = 2^16, 34 Q limbs, 4 P limbs), a batch
of 64 vectors of 2^15 complex slots, scale 2^45, NTT domain. Four workloads, each one lgpu_ckks_encode / lgpu_ckks_decode call:
  encode_q     Embed into a ring.Poly at level 33 (34 rows);
  encode_qp    Embed into the ringqp.Poly of a linear-transformation diagonal: level 33 + 4 P rows, NTT + Montgomery;
  decode_l0    DecodePublic of a level-0 plaintext;
  decode_l33   DecodePublic of a level-33 plaintext (the multiword CRT path).
Each is timed with CUDA events around one call, after a warm-up, as the median (and minimum) of --iters runs, with a 256 MB buffer
rewritten before every run so that no operand starts in L2. Algorithmic bytes are computed from the shapes: the values read or
written once (16 B per slot) plus the plaintext words written or read once (8 B per row and coefficient). The card's name and power
limit are read in the same run. Writes JSON (default: bench_out/encoder.json); bench.py stays the contract benchmark."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(limit)


def timed(fn, iters, flush):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        flush.add_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(min(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=os.path.join("bench_out", "encoder.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_encoder.py needs a CUDA device"
    assert args.iters >= 5
    name, limit = gpu_info()
    pr = PRESETS["CKKS_PN16QP1761"]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    enc = lb.Encoder(ctx)
    N, L, LP, B = ctx.N, len(pr["Q"]) - 1, len(pr["P"]) - 1, args.batch
    slots = N // 2
    flush = torch.zeros(32 << 20, dtype=torch.float64, device="cuda")
    rng = np.random.default_rng(1)
    v = torch.tensor(rng.uniform(-1, 1, (B, slots)) + 1j * rng.uniform(-1, 1, (B, slots)), dtype=torch.complex128, device="cuda")
    pt33 = enc.Encode(v, L, 2.0 ** 45)
    pt0 = enc.Encode(v, 0, 2.0 ** 45)
    torch.cuda.synchronize()
    rows = {"encode_q": L + 1, "encode_qp": L + 1 + LP + 1, "decode_l0": 1, "decode_l33": L + 1}
    runs = {
        "encode_q": lambda: enc.Encode(v, L, 2.0 ** 45),
        "encode_qp": lambda: enc.Encode(v, L, 2.0 ** 45, montgomery=True, level_p=LP),
        "decode_l0": lambda: enc.Decode(pt0, 2.0 ** 45, 15),
        "decode_l33": lambda: enc.Decode(pt33, 2.0 ** 45, 15),
    }
    rep = {"gpu": name, "power_limit_w": limit, "params": "CKKS_PN16QP1761", "batch": B, "slots": slots, "iters": args.iters,
           "workloads": {}}
    for k, fn in runs.items():
        med, mn = timed(fn, args.iters, flush)
        alg = B * (16 * slots + 8 * rows[k] * N)
        rep["workloads"][k] = {"rows": rows[k], "ms_per_batch": med, "ms_min": mn, "alg_bytes": alg, "alg_GBps": alg / med / 1e6}
    ctx.close()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit, **{k: round(w["ms_per_batch"], 3) for k, w in rep["workloads"].items()}}))


if __name__ == "__main__":
    main()

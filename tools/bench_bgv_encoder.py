"""BGV encoding and decoding (bgv.Encoder Encode / Embed / Decode) on one GPU. BGV_N15QP880 (N = 2^15, 20 Q limbs, 4 P limbs), t = 0x10001
(2^15 slots, gap 1), a batch of 128 vectors of uint64 slot values, NTT domain. Five workloads, each one lgpu_bgv_encode / lgpu_bgv_decode
call:
  encode_l19   Encode into a ring.Poly at level 19 (20 rows);
  embed_qp     Embed into a ringqp.Poly at level 19 + 4 P rows, NTT + Montgomery;
  decode_l0    Decode of a level-0 plaintext;
  decode_l19   Decode of a level-19 plaintext (the fused ModUpExact pass);
  decode_gap2  N = 2^16 (45-bit primes, level 15), t = 0x10001: 2^15 slots at gap 2, decoded through the 16-word CRT.
Each is timed with CUDA events around one call, after a warm-up, as the median (and minimum) of --iters runs, with a 256 MB buffer
rewritten before every run so that no operand starts in L2. Algorithmic bytes are computed from the shapes: the values read or written
once (8 B per slot) plus the plaintext words written or read once (8 B per row and coefficient). The card's name and power limit are read
in the same run. Writes JSON (default: bench_out/bgv_encoder.json); bench.py stays the contract benchmark."""
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


def gen_ntt_primes(bits, m, count):
    """`count` primes q = 1 mod m just below 2^bits (downwards), for the N = 2^16 case."""
    out, x = [], ((1 << bits) - 1) // m * m + 1
    while len(out) < count:
        if pow(2, x - 1, x) == 1 and all(pow(a, x - 1, x) == 1 for a in (3, 5, 7, 11, 13)):
            out.append(x)
        x -= m
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--out", default=os.path.join("bench_out", "bgv_encoder.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_bgv_encoder.py needs a CUDA device"
    assert args.iters >= 5
    name, limit = gpu_info()
    pr = PRESETS["BGV_N15QP880"]
    t = pr["T"]
    ctx = lb.Context(pr["logN"], pr["Q"], pr["P"])
    enc = lb.BGVEncoder(ctx, t)
    N, L, LP, B = ctx.N, len(pr["Q"]) - 1, len(pr["P"]) - 1, args.batch
    slots = enc.MaxSlots()
    flush = torch.zeros(32 << 20, dtype=torch.float64, device="cuda")
    rng = np.random.default_rng(1)
    v = torch.from_numpy(rng.integers(0, t, (B, slots), dtype=np.uint64).view(np.int64)).cuda().view(torch.uint64)
    pt19 = enc.Encode(v, L)
    pt0 = enc.Encode(v, 0)
    # N = 2^16, gap 2
    ctx16 = lb.Context(16, gen_ntt_primes(45, 1 << 17, 16), [])
    enc16 = lb.BGVEncoder(ctx16, t)
    v16 = torch.from_numpy(rng.integers(0, t, (B, enc16.MaxSlots()), dtype=np.uint64).view(np.int64)).cuda().view(torch.uint64)
    pt16 = enc16.Encode(v16, 15)
    torch.cuda.synchronize()
    shapes = {"encode_l19": (L + 1, N, slots), "embed_qp": (L + 1 + LP + 1, N, slots), "decode_l0": (1, N, slots),
              "decode_l19": (L + 1, N, slots), "decode_gap2": (16, ctx16.N, enc16.MaxSlots())}
    runs = {
        "encode_l19": lambda: enc.Encode(v, L),
        "embed_qp": lambda: enc.Embed(v, L, montgomery=True, level_p=LP),
        "decode_l0": lambda: enc.Decode(pt0),
        "decode_l19": lambda: enc.Decode(pt19),
        "decode_gap2": lambda: enc16.Decode(pt16),
    }
    assert torch.equal(enc.Decode(pt19), v.view(torch.int64)) and torch.equal(enc16.Decode(pt16), v16.view(torch.int64))
    rep = {"gpu": name, "power_limit_w": limit, "params": "BGV_N15QP880", "t": t, "batch": B, "iters": args.iters, "workloads": {}}
    for k, fn in runs.items():
        med, mn = timed(fn, args.iters, flush)
        rows, n, s = shapes[k]
        alg = B * (8 * s + 8 * rows * n)
        rep["workloads"][k] = {"rows": rows, "N": n, "slots": s, "ms_per_batch": med, "ms_min": mn, "alg_bytes": alg, "alg_GBps": alg / med / 1e6}
    enc.close(); enc16.close(); ctx.close(); ctx16.close()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit, **{k: round(w["ms_per_batch"], 3) for k, w in rep["workloads"].items()}}))


if __name__ == "__main__":
    main()

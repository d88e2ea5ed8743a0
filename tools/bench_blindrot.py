"""Blind rotation (blindrot.Evaluator.Evaluate) on one GPU at the reference's test shape (core/rgsw/blindrot/blindrot_test.go): N = 2^10,
Q = 0x7fff801, BaseTwoDecomposition 7, N_LWE = 2^9, q_LWE = 0x3001, window 10, every one of the 512 slots of one LWE-ring ciphertext.

Two arms, timed with CUDA events after a warm-up, keys and inputs uniform and seeded:
  fused     one lgpu_blind_rotation_evaluate call for all 512 slots;
  per-slot  the loop a caller runs today: one lgpu_blind_rotate_core call per slot, on a seeded subset of the slots (the whole loop
            would take minutes), with the mask and the initial accumulator prepared on the host beforehand (not timed).
Both arms' outputs are compared on the subset. Reported: time per blind rotation, kernel launches per call (lgpu_launch_count), and
the card's name and power limit, read in the same run. bench.py stays the contract benchmark; this script writes JSON
(default: bench_out/blindrot.json)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from oracle import blindrot_evaluate as BE  # noqa: E402
from oracle import oracle as O  # noqa: E402

LOGN, LOGN_LWE, Q, Q_LWE, PW2, WINDOW = 10, 9, 0x7fff801, 0x3001, 7, 10


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(limit)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return float(np.median(ts)), float(np.min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--loop-slots", type=int, default=8, help="slots of the per-slot arm (seeded subset)")
    ap.add_argument("--out", default="bench_out/blindrot.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    name, limit = gpu_info()
    rng = np.random.default_rng(2022)
    N, n_lwe = 1 << LOGN, 1 << LOGN_LWE
    ctx = lb.Context(LOGN, [Q], [])
    ctx_lwe = lb.Context(LOGN_LWE, [Q_LWE], [])
    nj = (27 + PW2 - 1) // PW2
    sizes = [nj]
    key = lambda: lb.GadgetCiphertext(ctx, rng.integers(0, Q, (1, nj, 2, 1, N), dtype=np.uint64), 0, -1, PW2, sizes)
    brk = [lb.rgsw.Ciphertext(key(), key()) for _ in range(n_lwe)]
    params = O.Parameters(LOGN, [Q], [])
    gals = [params.GaloisElement(k) for k in range(1, WINDOW + 1)] + [2 * N - 5]
    ev = lb.rgsw.BlindRotationEvaluator(ctx, brk, {g: key() for g in gals}, WINDOW)
    ct = rng.integers(0, Q_LWE, (1, 2, 1, n_lwe), dtype=np.uint64)
    tp = rng.integers(0, Q, (1, N), dtype=np.uint64)
    d_ct, d_tp = ctx_lwe.to_device(ct), ctx.to_device(tp)
    slots = {s: d_tp for s in range(n_lwe)}

    res = {}
    run = lambda: res.update(ev.Evaluate(d_ct, slots, ctx_lwe, is_ntt=False))
    fused_med, fused_min = timed(run, args.iters, args.warmup)
    n0 = lb.lib().lgpu_launch_count(); run(); torch.cuda.synchronize()
    fused_launches = lb.lib().lgpu_launch_count() - n0

    # per-slot arm: the host prepares each slot's mask and initial accumulator (evaluator.go:65-111) as the shim would
    subset = sorted(int(x) for x in rng.choice(n_lwe, args.loop_slots, replace=False))
    twoN, mask = 2 * N, 2 * N - 1
    a2n = BE.mod_switch_to_2n(ct[0, 1, 0], Q_LWE, twoN, True)
    a0 = [a2n[0]] + [-a2n[n_lwe - j] & mask for j in range(1, n_lwe)]
    b2n = BE.mod_switch_to_2n(ct[0, 0, 0], Q_LWE, twoN, False)
    ring = params.ringQ
    masks, accs = [], []
    for s in subset:
        masks.append(np.array(BE.mul_by_small_monomial_mod2n(mask, list(a0), s), dtype=np.uint64))
        xb = ring.NewPoly()
        i = b2n[s] - twoN if b2n[s] >= N else b2n[s]
        if i < 0: xb[0, N + i] = Q - 1
        else: xb[0, i] = 1
        ring.NTT(xb, xb); ring.MForm(xb, xb)
        t = ring.NewPoly(); ring.MulCoeffsMontgomery(tp, xb, t)
        a = ring.NewPoly(); ring.AutomorphismNTT(t, 2 * N - 5, a)
        accs.append(np.stack([a, np.zeros_like(a)]))
    d_init = [ctx.to_device(a) for a in accs]
    d_accs = [torch.empty_like(a) for a in d_init]

    def loop():
        for m, a, h in zip(masks, d_init, d_accs):
            h.copy_(a)
            ev.BlindRotateCore(m, h)
    loop_med, loop_min = timed(loop, max(1, args.iters // 2), 1)
    n0 = lb.lib().lgpu_launch_count(); loop(); torch.cuda.synchronize()
    loop_launches = (lb.lib().lgpu_launch_count() - n0) / len(subset)
    same = all(torch.equal(res[s][0], h) for s, h in zip(subset, d_accs))

    out = {
        "workload": "blindrot.Evaluator.Evaluate, N=2^10 Q=0x7fff801 BaseTwoDecomposition=7 N_LWE=2^9 q_LWE=0x3001 window=10, 512 slots",
        "gpu": name, "power_limit_w": limit,
        "fused": {"slots": n_lwe, "call_s_median": fused_med, "call_s_min": fused_min,
                  "per_blind_rotation_us": fused_med / n_lwe * 1e6, "launches_per_call": fused_launches},
        "per_slot_loop": {"slots_timed": subset, "loop_s_median": loop_med, "loop_s_min": loop_min,
                          "per_blind_rotation_us": loop_med / len(subset) * 1e6, "launches_per_blind_rotation": loop_launches,
                          "note": "seeded subset of the 512 slots; host-side mask and accumulator preparation not timed"},
        "speedup_per_blind_rotation": (loop_med / len(subset)) / (fused_med / n_lwe),
        "outputs_identical_on_subset": bool(same),
    }
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out))
    ctx.close(); ctx_lwe.close()
    if not same:
        sys.exit("fused and per-slot outputs differ")


if __name__ == "__main__":
    main()

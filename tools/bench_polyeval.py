"""CKKS polynomial evaluation (polynomial.Evaluator.Evaluate) on one GPU: CKKS_PN16QP1761 (N = 2^16, 34 Q limbs), a batch of 64
ciphertexts at the top level, scale 2^45, Chebyshev polynomials of degree 30 (even) and 63 (odd); relinearization key and inputs
uniform and seeded.

Two arms run the SAME planned program (same ops, same order, same weights), timed in the same run with CUDA events after a warm-up,
with a 256 MB buffer rewritten before every run so that no operand starts in L2:
  fused     one lgpu_ckks_polynomial_evaluate call;
  composed  the reference's op sequence from the existing entry points: lgpu_ckks_mulrelin_rescale_batch with nb_rescales = 0 for
            MULRELIN; the tensor as MForm / MulCoeffsMontgomery[ThenAdd] vecops, the scale ratios as MulScalarMontgomery and the Add
            as Add for TENSOR; lgpu_evaluator_relinearize for RELIN; lgpu_div_by_last_modulus_many for RESCALE; and for every baby
            step a zero accumulator, one MulScalarMontgomeryThenAdd pass per term (the MulThenAdd of each power) and one AddScalar for
            the constant (the DoubleRNSScalar ops, one call over all limbs and the whole batch when the two NTT halves share their
            scalars, as they do for real coefficients). Operands at a higher level than an op are first copied down to its rows,
            since one vecop call applies one batch stride to all of its operands. Where the arm's working set (every live
            ciphertext held by torch, plus the key-switch scratch) does not fit for the whole batch, it runs in halved sub-batches,
            as a caller of these entry points would; the sub-batch is recorded.
The two outputs are asserted byte-identical. Reported: median and minimum of each arm, ciphertexts per second, the speed-up, the
program's op counts, kernel launches per call (lgpu_launch_count), and the card's name and power limit, read in the same run.
bench.py stays the contract benchmark; this script writes JSON (default: bench_out/polyeval.json)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")   # the composed arm allocates many differently sized tensors
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200 import polyeval as PE  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(limit)


def composed(ctx, ckks, rlk, prog, ct, lpr, extra=None):
    """The program's op sequence through the existing entry points (see the module docstring). ct: (batch, 2, L+1, N)."""
    from lattigo_b200.ring import SubRing
    N, batch = ctx.N, ct.shape[0]
    Q = ctx.Q
    last = {}
    for i, o in enumerate(prog.ops):
        for key in ("src0", "src1", "addend"):
            if o.get(key, -1) >= 0:
                last[o[key]] = i
        for t in o.get("terms", []):
            last[t] = i
    slots = {0: ("il", ct)}
    cache = {}

    def rows(sl):
        kind, v = slots[sl]
        return v.shape[2] if kind == "il" else v[0].shape[1]

    def comp(sl, c, lv):
        kind, v = slots[sl]
        if rows(sl) == lv + 1 and kind == "pc":
            return v[c]
        key = (sl, c, lv)
        if key not in cache:
            cache[key] = (v[:, c, : lv + 1] if kind == "il" else v[c][:, : lv + 1]).contiguous()
        return cache[key]

    def interleaved(sl, deg, lv):
        kind, v = slots[sl]
        if kind == "il" and rows(sl) == lv + 1:
            return v
        return torch.stack([comp(sl, c, lv) for c in range(deg + 1)], 1)

    def ring(lv): return ctx.ringQ.AtLevel(lv)

    def mont(vals, lv): return [(int(v) << 64) % Q[r] for r, v in enumerate(vals[: lv + 1])]

    def scalar_op(name, p1, p3, s_lo, s_hi, lv, montgomery):
        """A DoubleRNSScalar op: one ring call when both halves share their scalars, per-limb half rows otherwise."""
        if list(s_lo) == list(s_hi):
            ring(lv)._vec(name, p1, None, p3, mont(s_lo, lv) if montgomery else list(s_lo[: lv + 1]))
            return
        h = N >> 1
        for r in range(lv + 1):
            sr = SubRing(ctx, 0, r)
            for b in range(batch):
                for half, s in ((slice(0, h), s_lo[r]), (slice(h, N), s_hi[r])):
                    v = (int(s) << 64) % Q[r] if montgomery else int(s)
                    sr._vec(name, p1[b, r, half] if p1 is not None else None, None, p3[b, r, half], v)

    deg = {0: 1}
    for i, o in enumerate(prog.ops):
        k, lv = o["kind"], o["level"]
        if k == PE.MULRELIN:
            a, b = interleaved(o["src0"], 1, lv), interleaved(o["src1"], 1, lv)
            slots[o["dst"]] = ("il", ckks.MulRelinNew(a, b)); deg[o["dst"]] = 1
        elif k == PE.TENSOR:
            R = ring(lv)
            b0, b1, x0, x1 = comp(o["src0"], 0, lv), comp(o["src0"], 1, lv), comp(o["src1"], 0, lv), comp(o["src1"], 1, lv)
            c00, c01 = torch.empty_like(b0), torch.empty_like(b0)
            R.MForm(b0, c00); R.MForm(b1, c01)
            d = [torch.empty_like(b0) for _ in range(3)]
            R.MulCoeffsMontgomery(c00, x0, d[0]); R.MulCoeffsMontgomery(c01, x1, d[2])
            R.MulCoeffsMontgomery(c00, x1, d[1]); R.MulCoeffsMontgomeryThenAdd(c01, x0, d[1])
            rb, ra = o["weights"][: lv + 1], o["weights"][lv + 1:]
            if any(v != 1 for v in rb):                  # Mul(b, ratio): the larger-scale side is b (x) X^k
                for c in range(3):
                    scalar_op("MulScalarMontgomery", d[c], d[c], rb, rb, lv, True)
            for c in range(deg[o["addend"]] + 1):        # Add(b, a) after Mul(a, ratio) into a buffer
                ac = comp(o["addend"], c, lv)
                if any(v != 1 for v in ra):
                    t = torch.empty_like(ac)
                    scalar_op("MulScalarMontgomery", ac, t, ra, ra, lv, True)
                    ac = t
                R.Add(d[c], ac, d[c])
            slots[o["dst"]] = ("pc", d); deg[o["dst"]] = 2
        elif k == PE.RELIN:
            src = interleaved(o["src0"], 2, lv)
            out = torch.empty((batch, 2, lv + 1, N), dtype=torch.int64, device=ct.device)
            ckks.Relinearize(src, rlk, out)
            slots[o["dst"]] = ("il", out); deg[o["dst"]] = 1
        elif k == PE.RESCALE:
            src = o["src0"]
            kind, v = slots[src]
            if kind == "il":                             # every polynomial of the batch in one call
                y = torch.empty((batch, deg[src] + 1, lv + 1, N), dtype=torch.int64, device=ct.device)
                lb.div_by_last_modulus_many(ctx, lb.ring.RING_Q, rows(src) - 1, True, True, lpr, v.reshape(-1, rows(src), N),
                                            y.view(-1, lv + 1, N))
                slots[o["dst"]] = ("il", y); deg[o["dst"]] = deg[src]
                continue_after = True
            else:
                continue_after = False
            d = []
            for c in range(0 if continue_after else deg[src] + 1):
                x = comp(src, c, rows(src) - 1)
                y = torch.empty((batch, lv + 1, N), dtype=torch.int64, device=ct.device)
                lb.div_by_last_modulus_many(ctx, lb.ring.RING_Q, rows(src) - 1, True, True, lpr, x, y)
                d.append(y)
            if not continue_after:
                slots[o["dst"]] = ("pc", d); deg[o["dst"]] = deg[src]
        elif k == PE.LINCOMB:
            L, terms, nt = lv, o["terms"], len(o["terms"])
            W = np.array(o["weights"], dtype=object).reshape(len(o["outs"]), nt + 1, L + 1, 2)
            order = sorted(range(len(o["outs"])), key=lambda j: -o["out_levels"][j])
            for n_done, i_out in enumerate(order):
                olv = o["out_levels"][i_out]
                acc = [torch.zeros((batch, olv + 1, N), dtype=torch.int64, device=ct.device) for _ in range(2)]
                cst = W[i_out, nt, : olv + 1]
                scalar_op("AddScalar", acc[0], acc[0], cst[:, 0], cst[:, 1], olv, False)
                for kk, sl in enumerate(terms):
                    w = W[i_out, kk, : olv + 1]
                    if not w.any():
                        continue
                    for c in range(2):                   # MulThenAdd(X^k, coefficient, res)
                        scalar_op("MulScalarMontgomeryThenAdd", comp(sl, c, olv), acc[c], w[:, 0], w[:, 1], olv, True)
                slots[o["outs"][i_out]] = ("pc", acc); deg[o["outs"][i_out]] = 1
                if n_done + 1 == len(order) or o["out_levels"][order[n_done + 1]] != olv:
                    for key in [key for key in cache if key[2] == olv and key[0] in terms]:      # copies made for this level
                        del cache[key]
        else:                                            # an op of another program kind: extra(op, comp, slots, deg)
            extra(o, comp, slots, deg)
        for sl in [s_ for s_, j in last.items() if j == i and s_ != 0 and s_ != prog.out_slot]:
            slots.pop(sl, None)
            for key in [key for key in cache if key[0] == sl]:
                del cache[key]
    return interleaved(prog.out_slot, 1, prog.out_level).contiguous()


def trim_pool():
    """Returns the blocks cached in the device's default stream-ordered pool (the library's scratch allocator, which keeps freed
    blocks: tables.cu) to the driver, so that the arm that runs next (torch's caching allocator) can use that memory."""
    torch.cuda.synchronize()
    cu = ctypes.CDLL("libcuda.so.1")
    dev, pool = ctypes.c_int(), ctypes.c_void_p()
    assert cu.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    assert cu.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0
    assert cu.cuMemPoolTrimTo(pool, ctypes.c_size_t(0)) == 0


def timed(fn, iters, flush):
    ts = []
    for _ in range(iters):
        flush.fill_(1)
        a = torch.cuda.Event(enable_timing=True); b = torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1, help=">= 1")
    ap.add_argument("--out", default="bench_out/polyeval.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    name, limit = gpu_info()
    pr = PRESETS["CKKS_PN16QP1761"]
    Q, P, logN = pr["Q"], pr["P"], pr["logN"]
    N, L, LP = 1 << logN, len(Q) - 1, len(P) - 1
    ctx = lb.Context(logN, Q, P)
    nd = (L + 1 + LP) // (LP + 1)
    gen = torch.Generator(device="cuda").manual_seed(1761)
    q_t = torch.tensor(Q + P, dtype=torch.float64, device="cuda")[:, None]

    def uniform(shape_lead, mods):
        m = q_t[: len(mods)]                            # Q limbs, then P limbs
        u = torch.rand(tuple(shape_lead) + (len(mods), N), generator=gen, device="cuda", dtype=torch.float64)
        return (u * m).to(torch.int64)                  # < q (float64 keeps 53 bits: uniform enough for timing)

    rlk = lb.GadgetCiphertext(ctx, uniform((nd, 1, 2), Q + P).contiguous(), L, LP)
    ct = uniform((args.batch, 2), Q).contiguous()
    ev = PE.PolynomialEvaluator(ctx, rlk, 1, 53)
    ckks = lb.CKKSEvaluator(ctx, rlk, 1)
    flush = torch.empty(64 << 20, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(63)
    results = []
    for deg, odd, even in ((30, False, True), (63, True, False)):
        coeffs = [0.0 if (k & 1 and not odd) or (k & 1 == 0 and not even) else float(rng.uniform(-1, 1)) / (k + 1) for k in range(deg + 1)]
        scale = Fraction(2) ** 45
        prog = ev.plan(L, scale, coeffs, PE.CHEBYSHEV, scale, odd, even)
        out = torch.empty((args.batch, 2, prog.out_level + 1, N), dtype=torch.int64, device="cuda")
        run = lambda: ev.run(prog, ct, out, args.batch)
        box = {}
        chunk = [args.batch]                             # the composed arm's sub-batch: halved while its working set does not fit

        def run_c():
            c = chunk[0]
            parts = [composed(ctx, ckks, rlk, prog, ct[k: k + c], 1) for k in range(0, args.batch, c)]
            box["out"] = parts[0] if len(parts) == 1 else torch.cat(parts)
        # fused arm: warm-up and timed runs, then its cached scratch goes back to the driver
        torch.cuda.empty_cache()
        for _ in range(args.warmup):
            run()
        ts = timed(run, args.iters, flush)
        n0 = lb.lib().lgpu_launch_count(); run(); torch.cuda.synchronize()
        launches = lb.lib().lgpu_launch_count() - n0
        trim_pool()
        # composed arm
        while True:
            try:
                run_c()
                break
            except (torch.OutOfMemoryError, lb.LgpuError) as e:
                if chunk[0] == 1 or "out of memory" not in str(e):
                    raise
                box.clear(); torch.cuda.empty_cache(); trim_pool()
                chunk[0] //= 2
        for _ in range(args.warmup - 1):
            run_c()
        torch.cuda.synchronize()
        assert torch.equal(out, box["out"]), "the fused and the composed arms differ (degree %d)" % deg
        box.clear()
        tc = timed(run_c, args.iters, flush)
        n0 = lb.lib().lgpu_launch_count(); run_c(); torch.cuda.synchronize()
        launches_c = lb.lib().lgpu_launch_count() - n0
        assert torch.equal(out, box["out"]), "the fused and the composed arms differ (degree %d)" % deg
        box.clear()
        trim_pool()
        kinds = prog.kinds()
        med, med_c = float(np.median(ts)), float(np.median(tc))
        results.append({"degree": deg, "basis": "chebyshev", "parity": "odd" if not even else "even", "batch": args.batch,
                        "fused": {"median_s": med, "min_s": float(np.min(ts)), "runs_s": ts, "ct_per_s": args.batch / med,
                                  "launches_per_call": int(launches)},
                        "composed": {"median_s": med_c, "min_s": float(np.min(tc)), "runs_s": tc, "ct_per_s": args.batch / med_c,
                                     "launches_per_call": int(launches_c), "sub_batch": chunk[0]},
                        "speedup_median": med_c / med, "outputs_identical": True,
                        "ops": {k: kinds.count(v) for k, v in (("MULRELIN", PE.MULRELIN), ("TENSOR", PE.TENSOR), ("RELIN", PE.RELIN),
                                                               ("RESCALE", PE.RESCALE), ("LINCOMB", PE.LINCOMB))},
                        "output_level": prog.out_level})
        print("degree %d: fused %.1f ms (%d launches), composed %.1f ms (%d launches, sub-batches of %d), %.2fx, outputs identical"
              % (deg, med * 1e3, launches, med_c * 1e3, launches_c, chunk[0], med_c / med))
    rep = {"gpu": name, "power_limit_w": limit, "params": "CKKS_PN16QP1761", "input_level": L, "iters": args.iters,
           "warmup": args.warmup, "l2_flush_bytes": flush.numel() * 4, "results": results}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit,
                      "results": [(r["degree"], r["fused"]["median_s"], r["composed"]["median_s"]) for r in results]}))
    ctx.close()


if __name__ == "__main__":
    main()

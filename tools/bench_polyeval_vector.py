"""Polynomial-vector evaluation (Evaluate with a PolynomialVector and a Mapping) on one GPU: CKKS_PN16QP1761 (N = 2^16), batch 64 and
batch 1 at the top level, scale 2^45, two Chebyshev polynomials of degree 30 and of degree 63 mapped to the even and the odd slots; and
BGV / BFV on BGV_N15QP880 (t = 0x10001, level 19, batch 16), two degree-15 monomial polynomials. Relinearization key and inputs
uniform, seeded.

Two arms run the SAME planned program on the SAME encoded plaintexts, timed with CUDA events after a warm-up, with a 256 MB buffer
rewritten before every run so that no operand starts in L2:
  fused     one lgpu_*_polynomial_vector_evaluate call (RunVector);
  composed  the reference's op sequence through the existing entry points: every op but the baby steps as tools/bench_polyeval.py
            (CKKS) and tools/bench_bgv_polyeval.py (BGV) compose them, and for each baby step, in the reference's order, Add(res,
            vector) as one Add vecop per ciphertext, MulThenAdd(X^k, vector, res) as MForm(pt) (CKKS) or MulRNSScalarMontgomery(pt,
            tMontgomery) (BGV) once and one MulCoeffsMontgomeryThenAdd per component and ciphertext, and every multiplication of res
            (the equal-scale q_level product; BGV r1) as MulScalarMontgomery. Where its working set does not fit for the whole batch it
            runs in halved sub-batches, as a caller of these entry points would; the sub-batch is recorded.
The two outputs are asserted byte-identical. BFV has no composed arm: no existing entry point gives the unrelinearized
scale-invariant tensor that its giant steps need.
Encoding is shared by both arms and timed on its own: the host plan (plan_vector, wall clock) and the device encode of its slot vectors
(encode_plaintexts: the vectors built on the host, copied, and one lgpu_*_encode call per (level, scale); wall clock around a
synchronised call), median and minimum of --steps runs each after a warm-up.
Reported besides: ciphertexts per second, kernel launches per call (lgpu_launch_count), the program's op counts, and the PTLINCOMB op's
bytes against its minimum (each power once per batch entry, each plaintext once, each output once) as the kernel moves them; plus the
card's name and power limit, read in the same run. Writes JSON (default: bench_out/polyeval_vector.json)."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time
from fractions import Fraction

import numpy as np

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")   # the composed arm allocates many differently sized tensors
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200 import polyeval as PE  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402
import bench_bgv_polyeval as BB  # noqa: E402
import bench_polyeval as BC  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return name, float(limit)


FLUSH = None


def timed(fn, steps, warmup):
    global FLUSH
    if FLUSH is None:
        FLUSH = torch.empty(32 << 20, dtype=torch.int64, device="cuda")
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        FLUSH.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), runs_ms=ts)


def wall(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median_ms=float(np.median(ts)), min_ms=float(np.min(ts)), runs_ms=ts)


def launches(fn):
    torch.cuda.synchronize()
    c0 = lb._lib.lib().lgpu_launch_count()
    fn()
    torch.cuda.synchronize()
    return int(lb._lib.lib().lgpu_launch_count() - c0)


def op_bytes(prog, N, batch):
    """The PTLINCOMB op's bytes: the minimum (powers once per batch entry, plaintexts once, outputs once) and what the kernel moves
    (plaintexts once per tile: the whole batch up to 8 ciphertexts, else tiles of 8)."""
    o = [o for o in prog.ops if o["kind"] == PE.PTLINCOMB][0]
    K1 = len(o["terms"]) + 1
    R = o["level"] + 1
    pts = sum(o["out_levels"][i] + 1 for i in range(len(o["outs"])) for k in range(K1) if o["index"][i * K1 + k] >= 0)
    outs = sum(lv + 1 for lv in o["out_levels"])
    tiles = -(-batch // 8)
    minimum = 8 * N * (2 * batch * R * len(o["terms"]) + pts + 2 * batch * outs)
    moved = 8 * N * (2 * batch * R * len(o["terms"]) + pts * tiles + 2 * batch * outs)
    return dict(min_bytes=minimum, kernel_bytes=moved, ratio=moved / minimum)


def ptlincomb_composed(ctx, pt, tmont=None):
    """The composed arms' handler of the PTLINCOMB op: each baby step's Add / MulThenAdd / res multiplications in the reference's order
    (op["sequence"]) through the ring vecops, one call per ciphertext as the reference's evaluator runs them. pt: the encoded block."""
    Q, N = ctx.Q, ctx.N

    def extra(o, comp, slots, deg):
        terms, nt = o["terms"], len(o["terms"])
        K = nt + 1
        batch = slots[0][1].shape[0]

        def x(sl, c, b, lv):
            kind, v = slots[sl]
            return v[b, c, : lv + 1] if kind == "il" else v[c][b, : lv + 1]
        for i_out, olv in enumerate(o["out_levels"]):
            R = ctx.ringQ.AtLevel(olv)
            acc = [torch.zeros((batch, olv + 1, N), dtype=torch.int64, device=pt.device) for _ in range(2)]
            for kind, arg in o["sequence"][i_out]:
                if kind == "mul":                        # Mul(res, scalar): every component of res
                    for c in range(2):
                        R._vec("MulScalarMontgomery", acc[c], None, acc[c], [(int(v) << 64) % Q[r] for r, v in enumerate(arg[: olv + 1])])
                    continue
                p = pt[o["index"][i_out * K + arg], : olv + 1]
                if arg == nt:                            # Add(res, vector): the encoded vector on component 0
                    for b in range(batch):
                        R.Add(acc[0][b], p, acc[0][b])
                    continue
                c00 = torch.empty_like(p)                # MulThenAdd(X^k, vector, res): mulRelinThenAdd's degree-0 branch
                if tmont is None:
                    R.MForm(p, c00)
                else:
                    R._vec("MulScalarMontgomery", p, None, c00, tmont[: olv + 1])
                for b in range(batch):
                    for c in range(2):
                        R.MulCoeffsMontgomeryThenAdd(x(terms[arg], c, b, olv), c00, acc[c][b])
            slots[o["outs"][i_out]] = ("pc", acc)
            deg[o["outs"][i_out]] = 1
    return extra


def compare(fused_out, run_c, batch, steps, warmup):
    """Runs the composed arm (halving its sub-batch while it does not fit), asserts its output equals the fused one, and times it."""
    box, chunk = {}, [batch]

    def go():
        box["out"] = run_c(chunk[0])
    while True:
        try:
            go()
            break
        except (torch.OutOfMemoryError, lb.LgpuError) as e:
            if chunk[0] == 1 or "out of memory" not in str(e):
                raise
            box.clear(); torch.cuda.empty_cache(); BC.trim_pool()
            chunk[0] //= 2
    torch.cuda.synchronize()
    assert torch.equal(fused_out, box["out"]), "the fused and the composed arms differ"
    box.clear()
    t = timed(go, steps, max(0, warmup - 1))
    n = launches(go)
    assert torch.equal(fused_out, box["out"]), "the fused and the composed arms differ"
    box.clear()
    BC.trim_pool()
    return dict(t, launches_per_call=n, sub_batch=chunk[0], outputs_identical=True)


def release():
    """Hands every cached block back to the driver between workloads: torch's caching allocator (the composed arm) and the library's
    stream-ordered pool (the fused arm's scratch)."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    BC.trim_pool()


def uniform_like(gen, q_t, shape_lead, nmods, N):
    u = torch.rand(tuple(shape_lead) + (nmods, N), generator=gen, device="cuda", dtype=torch.float64)
    return (u * q_t[:nmods]).to(torch.int64)


def ckks_workload(degree, batch, steps, warmup, rng):
    pr = PRESETS["CKKS_PN16QP1761"]
    Q, P, logN = pr["Q"], pr["P"], pr["logN"]
    N, L, LP = 1 << logN, len(Q) - 1, len(P) - 1
    release()
    ctx = lb.Context(logN, Q, P)
    gen = torch.Generator(device="cuda").manual_seed(1761 + degree + batch)
    q_t = torch.tensor(Q + P, dtype=torch.float64, device="cuda")[:, None]
    nd = (L + 1 + LP) // (LP + 1)
    rlk = lb.GadgetCiphertext(ctx, uniform_like(gen, q_t, (nd, 1, 2), L + 1 + LP + 1, N).contiguous(), L, LP)
    ct = uniform_like(gen, q_t, (batch, 2), L + 1, N).contiguous()
    ev = PE.PolynomialEvaluator(ctx, rlk, 1, 53)
    ckks = lb.CKKSEvaluator(ctx, rlk, 1)
    polys = [PE.Polynomial([float(rng.uniform(-1, 1)) / (k + 1) for k in range(degree + 1)], PE.CHEBYSHEV) for _ in range(2)]
    pv = PE.NewPolynomialVector(polys, {0: list(range(0, N // 2, 2)), 1: list(range(1, N // 2, 2))})
    scale = Fraction(2) ** 45
    prep = ev.PrepareVector(L, scale, pv, scale)
    plan_t = wall(lambda: ev.plan_vector(L, scale, pv, scale), steps, 1)
    enc_t = wall(lambda: ev.encode_plaintexts(prep.prog), steps, 1)      # re-encodes the same program into a new block
    out = ev.RunVector(prep, ct)
    fused = timed(lambda: ev.RunVector(prep, ct), steps, warmup)
    fused["launches_per_call"] = launches(lambda: ev.RunVector(prep, ct))
    BC.trim_pool()
    extra = ptlincomb_composed(ctx, prep.pt)
    comp = compare(out, lambda c: torch.cat([BC.composed(ctx, ckks, rlk, prep.prog, ct[k: k + c], 1, extra) for k in range(0, batch, c)]),
                   batch, steps, warmup)
    kinds = prep.prog.kinds()
    res = dict(workload="CKKS_PN16QP1761 Chebyshev degree %d x2, even / odd slots" % degree, batch=batch, plan_host=plan_t,
               encode_device=enc_t, fused=dict(fused, ct_per_s=batch / (fused["median_ms"] / 1e3)),
               composed=dict(comp, ct_per_s=batch / (comp["median_ms"] / 1e3)), speedup_median=comp["median_ms"] / fused["median_ms"],
               n_plaintexts=len(prep.prog.plaintexts), output_level=prep.out_level,
               ops={n: kinds.count(k) for n, k in (("MULRELIN", PE.MULRELIN), ("TENSOR", PE.TENSOR), ("RELIN", PE.RELIN),
                                                    ("RESCALE", PE.RESCALE), ("LINCOMB", PE.LINCOMB), ("PTLINCOMB", PE.PTLINCOMB))},
               ptlincomb_bytes=op_bytes(prep.prog, N, batch))
    del prep, out, ct, rlk, ckks, ev, extra
    ctx.close()
    release()
    return res


def bgv_workload(si, batch, steps, warmup, rng):
    pr = PRESETS["BGV_N15QP880"]
    Q, P, logN, QMul = pr["Q"], pr["P"], pr["logN"], pr["QMul"]
    N, Lm, LP, L, t = 1 << logN, len(Q) - 1, len(P) - 1, 19, 0x10001
    ctx = lb.Context(logN, Q, P)
    gen = torch.Generator(device="cuda").manual_seed(880 + si)
    q_t = torch.tensor(Q + P, dtype=torch.float64, device="cuda")[:, None]
    nd = (Lm + 1 + LP) // (LP + 1)
    rlk = lb.GadgetCiphertext(ctx, uniform_like(gen, q_t, (nd, 1, 2), Lm + 1 + LP + 1, N).contiguous(), Lm, LP)
    ct = uniform_like(gen, q_t, (batch, 2), L + 1, N).contiguous()
    enc = lb.BGVEncoder(ctx, t)
    bgv = lb.BGVEvaluator(ctx, t, QMul, rlk, scale_invariant=si)
    pev = lb.BGVPolynomialEvaluator(bgv)
    ckks = lb.CKKSEvaluator(ctx, rlk, 1)
    polys = [PE.Polynomial([int(x) for x in rng.integers(0, t, 16)]) for _ in range(2)]
    ms = enc.MaxSlots()
    pv = PE.NewPolynomialVector(polys, {0: list(range(0, ms, 2)), 1: list(range(1, ms, 2))})
    prep = pev.PrepareVector(L, 1, pv, 1, enc)
    plan_t = wall(lambda: pev.plan_vector(L, 1, pv, 1), steps, 1)
    enc_t = wall(lambda: pev.encode_plaintexts(prep.prog, enc), steps, 1)
    out = pev.RunVector(prep, ct)
    fused = timed(lambda: pev.RunVector(prep, ct), steps, warmup)
    fused["launches_per_call"] = launches(lambda: pev.RunVector(prep, ct))
    BC.trim_pool()
    res = dict(workload="BGV_N15QP880 level 19, degree 15 x2, even / odd slots, " + ("BFV" if si else "BGV"), batch=batch, plan_host=plan_t,
               encode_device=enc_t, fused=dict(fused, ct_per_s=batch / (fused["median_ms"] / 1e3)), n_plaintexts=len(prep.prog.plaintexts),
               output_level=prep.out_level, ptlincomb_bytes=op_bytes(prep.prog, N, batch))
    if si:
        res["composed"] = None                           # no unrelinearized scale-invariant tensor among the existing entry points
    else:
        tmont = [(t << 128) % q for q in Q]
        extra = ptlincomb_composed(ctx, prep.pt, tmont)
        comp = compare(out, lambda c: torch.cat([BB.composed(ctx, bgv, ckks, rlk, prep.prog, ct[k: k + c], t, extra)
                                                 for k in range(0, batch, c)]), batch, steps, warmup)
        res["composed"] = dict(comp, ct_per_s=batch / (comp["median_ms"] / 1e3))
        res["speedup_median"] = comp["median_ms"] / fused["median_ms"]
    bgv.close()
    enc.close()
    del prep, out, ct, rlk, ckks, pev
    ctx.close()
    release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default="bench_out/polyeval_vector.json")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    rng = np.random.default_rng(1)
    name, limit = gpu_info()
    rows = []
    short = lambda r: {k: (v["median_ms"] if isinstance(v, dict) and "median_ms" in v else v)
                       for k, v in r.items() if k not in ("ops", "ptlincomb_bytes")}
    for degree in (30, 63):
        for batch in (64, 1):
            rows.append(ckks_workload(degree, batch, a.steps, a.warmup, rng))
            print(json.dumps(short(rows[-1])), flush=True)
    for si in (False, True):
        rows.append(bgv_workload(si, 16, a.steps, a.warmup, rng))
        print(json.dumps(short(rows[-1])), flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(dict(gpu=name, power_limit_w=limit, steps=a.steps, warmup=a.warmup, l2_flush_bytes=32 << 23, results=rows), f, indent=1)
    print(json.dumps(dict(gpu=name, power_limit_w=limit)))


if __name__ == "__main__":
    main()

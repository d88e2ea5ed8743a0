"""BGV / BFV polynomial evaluation (bgv polynomial.Evaluator.Evaluate) on one GPU: BGV_N15QP880 (N = 2^15, 20 Q limbs), t = 0x10001,
a batch of 64 ciphertexts at level 19, monomial polynomials of degree 15 and 63 with uint64 coefficients; relinearization key and
inputs uniform and seeded. Both tensorings: BGV (tensorStandard) and BFV (tensorScaleInvariant).

For BGV two arms run the SAME planned program, timed in the same run with CUDA events after a warm-up, with a 256 MB buffer rewritten
before every run so that no operand starts in L2:
  fused     one lgpu_bgv_polynomial_evaluate call;
  composed  the reference's op sequence from the existing entry points: lgpu_bgv_mulrelin_batch for MULRELIN; for TENSOR the tensor as
            per-limb MulScalarMontgomery by tMontgomery and MulCoeffsMontgomery[ThenAdd] vecops, then the ratios (always 1 here) and Add;
            lgpu_evaluator_relinearize for RELIN; lgpu_div_by_last_modulus_many for RESCALE; and for every baby step a zero accumulator,
            one MulScalarMontgomeryThenAdd pass per term and one AddScalar for the constant.
The two outputs are asserted byte-identical. The existing entry points have no unrelinearized scale-invariant tensor, so BFV is
reported for the fused arm alone. Reported: median and minimum, ciphertexts per second, the op counts, kernel launches per call
(lgpu_launch_count), and the card's name and power limit, read in the same run. Writes JSON (default: bench_out/bgv_polyeval.json)."""
import argparse
import json
import os
import sys

import numpy as np

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import lattigo_b200 as lb  # noqa: E402
from lattigo_b200 import polyeval as PE  # noqa: E402
from lattigo_b200.params import PRESETS  # noqa: E402
from bench_polyeval import gpu_info, timed, trim_pool  # noqa: E402


def composed(ctx, bgv, ckks, rlk, prog, ct, t, extra=None):
    """The BGV program's op sequence through the existing entry points (see the module docstring). ct: (batch, 2, L+1, N)."""
    N, batch, Q = ctx.N, ct.shape[0], ctx.Q
    tmont = [(t << 128) % q for q in Q]             # tMontgomery = MForm(t 2^64 mod q)
    last = {}
    for i, o in enumerate(prog.ops):
        for key in ("src0", "src1", "addend"):
            if o.get(key, -1) >= 0:
                last[o[key]] = i
        for s_ in o.get("terms", []):
            last[s_] = i
    slots, deg, cache = {0: ("il", ct)}, {0: 1}, {}

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

    def interleaved(sl, d, lv):
        kind, v = slots[sl]
        if kind == "il" and rows(sl) == lv + 1:
            return v
        return torch.stack([comp(sl, c, lv) for c in range(d + 1)], 1)

    def ring(lv): return ctx.ringQ.AtLevel(lv)

    for i, o in enumerate(prog.ops):
        k, lv = o["kind"], o["level"]
        if k == PE.MULRELIN:
            a = interleaved(o["src0"], 1, lv)
            b = a if o["src1"] == o["src0"] else interleaved(o["src1"], 1, lv)
            slots[o["dst"]] = ("il", bgv.MulRelinNew(a, b)); deg[o["dst"]] = 1
        elif k == PE.TENSOR:
            R = ring(lv)
            b0, b1, x0, x1 = comp(o["src0"], 0, lv), comp(o["src0"], 1, lv), comp(o["src1"], 0, lv), comp(o["src1"], 1, lv)
            c00, c01 = torch.empty_like(b0), torch.empty_like(b0)
            R._vec("MulScalarMontgomery", b0, None, c00, tmont[: lv + 1]); R._vec("MulScalarMontgomery", b1, None, c01, tmont[: lv + 1])
            d = [torch.empty_like(b0) for _ in range(3)]
            R.MulCoeffsMontgomery(c00, x0, d[0]); R.MulCoeffsMontgomery(c01, x1, d[2])
            R.MulCoeffsMontgomery(c00, x1, d[1]); R.MulCoeffsMontgomeryThenAdd(c01, x0, d[1])
            rb, ra = o["weights"][: lv + 1], o["weights"][lv + 1:]
            assert set(rb) == {1} and set(ra) == {1}       # EvaluateMonomial's InDelta check leaves equal scales
            for c in range(deg[o["addend"]] + 1):
                R.Add(d[c], comp(o["addend"], c, lv), d[c])
            slots[o["dst"]] = ("pc", d); deg[o["dst"]] = 2
        elif k == PE.RELIN:
            out = torch.empty((batch, 2, lv + 1, N), dtype=torch.int64, device=ct.device)
            ckks.Relinearize(interleaved(o["src0"], 2, lv), rlk, out)
            slots[o["dst"]] = ("il", out); deg[o["dst"]] = 1
        elif k == PE.RESCALE:
            src = o["src0"]
            x = interleaved(src, deg[src], rows(src) - 1).contiguous()
            y = torch.empty((batch, deg[src] + 1, lv + 1, N), dtype=torch.int64, device=ct.device)
            lb.div_by_last_modulus_many(ctx, lb.ring.RING_Q, rows(src) - 1, True, True, 1, x.reshape(-1, rows(src), N), y.view(-1, lv + 1, N))
            slots[o["dst"]] = ("il", y); deg[o["dst"]] = deg[src]
        elif k == PE.LINCOMB:
            L, terms, nt = lv, o["terms"], len(o["terms"])
            W = np.array(o["weights"], dtype=object).reshape(len(o["outs"]), nt + 1, L + 1, 2)
            for i_out, olv in enumerate(o["out_levels"]):
                acc = [torch.zeros((batch, olv + 1, N), dtype=torch.int64, device=ct.device) for _ in range(2)]
                ring(olv)._vec("AddScalar", acc[0], None, acc[0], [int(x) for x in W[i_out, nt, : olv + 1, 0]])
                for kk, sl in enumerate(terms):
                    w = W[i_out, kk, : olv + 1, 0]
                    if not w.any():
                        continue
                    for c in range(2):                     # MulThenAdd(X^k, coefficient, res)
                        ring(olv)._vec("MulScalarMontgomeryThenAdd", comp(sl, c, olv), None, acc[c],
                                       [(int(v) << 64) % Q[r] for r, v in enumerate(w)])
                slots[o["outs"][i_out]] = ("pc", acc); deg[o["outs"][i_out]] = 1
        else:                                            # an op of another program kind: extra(op, comp, slots, deg)
            extra(o, comp, slots, deg)
        for sl in [s_ for s_, j in last.items() if j == i and s_ != 0 and s_ != prog.out_slot]:
            slots.pop(sl, None)
            for key in [key for key in cache if key[0] == sl]:
                del cache[key]
    return interleaved(prog.out_slot, 1, prog.out_level).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1, help=">= 1")
    ap.add_argument("--out", default="bench_out/bgv_polyeval.json")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
    name, limit = gpu_info()
    pr = PRESETS["BGV_N15QP880"]
    Q, P, logN, T, QMul = pr["Q"], pr["P"], pr["logN"], pr["T"], pr["QMul"]
    N, L, LP = 1 << logN, len(Q) - 1, len(P) - 1
    ctx = lb.Context(logN, Q, P)
    nd = (L + 1 + LP) // (LP + 1)
    gen = torch.Generator(device="cuda").manual_seed(880)
    q_t = torch.tensor(Q + P, dtype=torch.float64, device="cuda")[:, None]

    def uniform(shape_lead, mods):
        u = torch.rand(tuple(shape_lead) + (len(mods), N), generator=gen, device="cuda", dtype=torch.float64)
        return (u * q_t[: len(mods)]).to(torch.int64)

    rlk = lb.GadgetCiphertext(ctx, uniform((nd, 1, 2), Q + P).contiguous(), L, LP)
    ct = uniform((args.batch, 2), Q).contiguous()
    ckks = lb.CKKSEvaluator(ctx, rlk, 1)
    flush = torch.empty(64 << 20, dtype=torch.int32, device="cuda")
    rng = np.random.default_rng(63)
    results = []
    for si in (False, True):
        bgv = lb.BGVEvaluator(ctx, T, QMul, rlk, scale_invariant=si)
        pe = lb.BGVPolynomialEvaluator(bgv)
        for deg in (15, 63):
            coeffs = [int(x) for x in rng.integers(0, T, deg + 1)]
            prog = pe.plan(L, 1, coeffs, 1)
            out = torch.empty((args.batch, 2, prog.out_level + 1, N), dtype=torch.int64, device="cuda")
            run = lambda: pe.run(prog, ct, out, args.batch)
            torch.cuda.empty_cache()
            for _ in range(args.warmup):
                run()
            ts = timed(run, args.iters, flush)
            n0 = lb.lib().lgpu_launch_count(); run(); torch.cuda.synchronize()
            launches = lb.lib().lgpu_launch_count() - n0
            trim_pool()
            kinds = prog.kinds()
            med = float(np.median(ts))
            r = {"scheme": "BFV" if si else "BGV", "degree": deg, "basis": "monomial", "batch": args.batch,
                 "fused": {"median_s": med, "min_s": float(np.min(ts)), "runs_s": ts, "ct_per_s": args.batch / med,
                           "launches_per_call": int(launches)},
                 "ops": {k: kinds.count(v) for k, v in (("MULRELIN", PE.MULRELIN), ("TENSOR", PE.TENSOR), ("RELIN", PE.RELIN),
                                                        ("RESCALE", PE.RESCALE), ("LINCOMB", PE.LINCOMB))},
                 "output_level": prog.out_level}
            line = "%s degree %d: fused %.1f ms (%d launches)" % (r["scheme"], deg, med * 1e3, launches)
            if not si:
                box = {}

                def run_c():
                    box["out"] = composed(ctx, bgv, ckks, rlk, prog, ct, T)
                for _ in range(args.warmup):
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
                med_c = float(np.median(tc))
                r["composed"] = {"median_s": med_c, "min_s": float(np.min(tc)), "runs_s": tc, "ct_per_s": args.batch / med_c,
                                 "launches_per_call": int(launches_c)}
                r["speedup_median"] = med_c / med
                r["outputs_identical"] = True
                line += ", composed %.1f ms (%d launches), %.2fx, outputs identical" % (med_c * 1e3, launches_c, med_c / med)
            else:
                r["composed"] = None                        # no unrelinearized scale-invariant tensor among the existing entry points
            results.append(r)
            print(line, flush=True)
        bgv.close()
    rep = {"gpu": name, "power_limit_w": limit, "params": "BGV_N15QP880", "t": T, "input_level": L, "iters": args.iters,
           "warmup": args.warmup, "l2_flush_bytes": flush.numel() * 4, "results": results}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rep, f, indent=1)
    print(json.dumps({"gpu": name, "power_limit_w": limit,
                      "results": [(r["scheme"], r["degree"], r["fused"]["median_s"], (r["composed"] or {}).get("median_s"))
                                  for r in results]}))
    ctx.close()


if __name__ == "__main__":
    main()

"""Shared setup of the polynomial-vector tests: the cases (two or more polynomials, each mapped to its own slots), an exact CPU
interpreter of the planner's vector programs (PTLINCOMB with the plaintexts encoded by the oracle encoders, every other op on the
oracle's evaluators), and the literal oracle's result for a case."""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from lattigo_b200 import polyeval as PE
from lattigo_b200 import bgv_polyeval as BPE
from oracle import oracle as O
from oracle import polyeval as OP
from tests import bgv_polyeval_oracle as BP
from tests import polyvec_oracle as V

U64 = np.uint64
M, C = OP.MONOMIAL, OP.CHEBYSHEV


def _coeffs(rng, deg, odd=True, even=True, cplx=False):
    c = [float(rng.uniform(-1, 1)) / (k + 1) for k in range(deg + 1)]
    if cplx:
        c = [complex(x, float(rng.uniform(-0.5, 0.5)) / (k + 1)) for k, x in enumerate(c)]
    for k in range(deg + 1):
        if (k & 1 and not odd) or (k & 1 == 0 and not even):
            c[k] = 0.0
    return c


def even_odd(n_slots):
    return {0: list(range(0, n_slots, 2)), 1: list(range(1, n_slots, 2))}


def ckks_cases():
    """name -> (basis, [(coeffs, odd, even)], mapping kind, levels_per_rescale, target scale as a multiple of the input scale).
    mapping kind: "eo" (polynomial 0 on the even slots, 1 on the odd ones), "half" (the first quarter and the third quarter of the
    slots; the rest unmapped), "three" (three polynomials on slots mod 3, slot 0 mapped twice)."""
    rng = np.random.default_rng(11)
    out = {}
    out["mono3"] = (M, [(_coeffs(rng, 3), True, True), (_coeffs(rng, 3), True, True)], "eo", 1, 1)
    out["mono7_half"] = (M, [(_coeffs(rng, 7), True, True), (_coeffs(rng, 7), True, True)], "half", 1, 1)
    out["cheb12"] = (C, [(_coeffs(rng, 12), True, True), (_coeffs(rng, 12), True, True)], "eo", 1, 1)
    out["cheb30"] = (C, [(_coeffs(rng, 30), True, True), (_coeffs(rng, 30), True, True)], "eo", 1, 1)
    out["cheb15_odd"] = (C, [(_coeffs(rng, 15, even=False), True, False), (_coeffs(rng, 15, even=False), True, False)], "eo", 1, 1)
    out["cheb14_even"] = (C, [(_coeffs(rng, 14, odd=False), False, True), (_coeffs(rng, 14, odd=False), False, True)], "eo", 1, 1)
    # mixed flags: the power basis takes odd OR even, the baby steps odd AND even (none), so every key is read; the odd polynomial's
    # quotients have nil even coefficients, which encode as 0
    out["cheb15_mixed"] = (C, [(_coeffs(rng, 15, even=False), True, False), (_coeffs(rng, 15), True, True)], "eo", 1, 1)
    out["mono5_complex"] = (M, [(_coeffs(rng, 5, cplx=True), True, True), (_coeffs(rng, 5, cplx=True), True, True)], "eo", 1, 1)
    out["mono7_three"] = (M, [(_coeffs(rng, 7), True, True) for _ in range(3)], "three", 1, 1)
    out["mono7_lpr2"] = (M, [(_coeffs(rng, 7), True, True), (_coeffs(rng, 7), True, True)], "eo", 2, 1)
    out["mono3_target"] = (M, [(_coeffs(rng, 3), True, True), (_coeffs(rng, 3), True, True)], "eo", 1, Fraction(1, 2))
    return out


def mapping(kind, n_slots, n_polys):
    if kind == "eo":
        return even_odd(n_slots)
    if kind == "half":
        q = n_slots // 4
        return {0: list(range(q)), 1: list(range(2 * q, 3 * q))}
    out = {i: list(range(i, n_slots, 3)) for i in range(n_polys)}
    out[n_polys - 1] = [0] + out[n_polys - 1]
    return out


def pvec(basis, polys, mp):
    return PE.NewPolynomialVector([PE.Polynomial(c, basis, o, e) for c, o, e in polys], mp)


def oracle_polys(basis, polys):
    return [OP.new_polynomial(basis, c, o, e) for c, o, e in polys]


def bgv_oracle_polys(polys):
    return [BP.new_polynomial(c, o, e) for c, o, e in polys]


# ---- the interpreter -------------------------------------------------------------------------------------------------------------
def ckks_encode_plaintexts(params, prog):
    """The program's plaintexts with the oracle encoder (what lgpu_ckks_encode computes): [level + 1][N] rows each."""
    from oracle import encoder as E
    logN = params.N().bit_length() - 1
    return [E.embed_double(params.ringQ, None, prog.values(j), logN - 1, float(p["scale"]), True, False, p["level"])[0]
            for j, p in enumerate(prog.plaintexts)]


def bgv_encode_plaintexts(enc, prog):
    return [np.array(enc.Encode([int(v) for v in prog.values(j, np.uint64)], False, int(p["scale"]), True, False, p["level"]), dtype=U64)
            for j, p in enumerate(prog.plaintexts)]


def ptlincomb(o, slots, pts, Q, N):
    """outs[i] = sum_k s PT X_k + s PT (component 0), in exact integers."""
    L, terms, nt = o["level"], o["terms"], len(o["terms"])
    K = nt + 1
    for i, (d, lv) in enumerate(zip(o["outs"], o["out_levels"])):
        out = []
        for c in range(2):
            rows = []
            for r in range(lv + 1):
                acc = np.zeros(N, dtype=object)
                for k in range(K):
                    j = o["index"][i * K + k]
                    if j < 0 or (k == nt and c == 1):
                        continue
                    s = o["scalars"][(i * K + k) * (L + 1) + r]
                    v = pts[j][r].astype(object) * s
                    if k < nt:
                        v = v * slots[terms[k]][c][r].astype(object)
                    acc += v
                rows.append(np.array(acc % Q[r], dtype=U64))
            out.append(np.stack(rows))
        slots[d] = out


def interpret(prog, ct_value, pts, Q, N, ops):
    """ops: mulrelin(a, b), relin(x), rescale(x), tensor(b, x, level) -> the degree-2 product before the TENSOR weights."""
    slots = {0: [np.array(v) for v in ct_value]}
    for o in prog.ops:
        k = o["kind"]
        if k == PE.MULRELIN:
            a = slots[o["src0"]]
            slots[o["dst"]] = ops["mulrelin"](a, a if o["src1"] == o["src0"] else slots[o["src1"]])
        elif k == PE.RELIN:
            slots[o["dst"]] = ops["relin"](slots[o["src0"]])
        elif k == PE.RESCALE:
            slots[o["dst"]] = ops["rescale"](slots[o["src0"]])
        elif k == PE.TENSOR:
            lv = o["level"]
            t = ops["tensor"]([v[: lv + 1] for v in slots[o["src0"]]], [v[: lv + 1] for v in slots[o["src1"]]])
            a = slots[o["addend"]]
            rb, ra = o["weights"][: lv + 1], o["weights"][lv + 1:]
            out = []
            for c in range(3):
                rows = []
                for r in range(lv + 1):
                    v = t[c][r].astype(object) * rb[r]
                    if c < len(a):
                        v = v + a[c][r].astype(object) * ra[r]
                    rows.append(np.array(v % Q[r], dtype=U64))
                out.append(np.stack(rows))
            slots[o["dst"]] = out
        elif k == PE.PTLINCOMB:
            ptlincomb(o, slots, pts, Q, N)
        else:
            L, terms, nt = o["level"], o["terms"], len(o["terms"])
            W = np.array(o["weights"], dtype=object).reshape(len(o["outs"]), nt + 1, L + 1, 2)
            for i, (d, lv) in enumerate(zip(o["outs"], o["out_levels"])):
                out = []
                for c in range(2):
                    rows = []
                    for r in range(lv + 1):
                        acc = np.zeros(N, dtype=object)
                        for kk, s in enumerate(terms):
                            if r >= len(slots[s][c]):
                                continue
                            x = slots[s][c][r].astype(object)
                            acc[: N // 2] += x[: N // 2] * W[i, kk, r, 0]
                            acc[N // 2:] += x[N // 2:] * W[i, kk, r, 1]
                        if c == 0:
                            acc[: N // 2] += W[i, nt, r, 0]
                            acc[N // 2:] += W[i, nt, r, 1]
                        rows.append(np.array(acc % Q[r], dtype=U64))
                    out.append(np.stack(rows))
                slots[d] = out
    return slots[prog.out_slot]


def ckks_ops(toy):
    ev = O.CKKSEvaluator(toy.params, toy.rlk, toy.lpr)
    pe = OP.PolyEvaluator(toy.params, toy.rlk, toy.lpr, toy.prec)
    return dict(mulrelin=ev.MulRelinNew, relin=lambda x: pe.relinearize(OP.Ct(x, 1)).Value, rescale=ev.Rescale,
                tensor=lambda b, x: pe.mul_tensor(OP.Ct(b, 1), OP.Ct(x, 1)).Value)


def bgv_ops(toy, invariant):
    ev = toy.evaluator(invariant).ev

    def relin(x):
        out = [np.empty_like(x[0]) for _ in range(2)]
        ev.Relinearize(x, toy.rlk, out)
        return out

    def rescale(x):
        ev.ScaleInvariant, si = False, ev.ScaleInvariant
        try:
            return ev.Rescale(x)
        finally:
            ev.ScaleInvariant = si
    return dict(mulrelin=ev.MulRelinNew, relin=relin, rescale=rescale, tensor=ev.MulNew)


def ckks_plan(toy, case, level=None, log_slots=None):
    basis, polys, kind, lpr, tmul = case
    L = toy.params.MaxLevelQ() if level is None else level
    mp = mapping(kind, toy.N // 2, len(polys))
    return PE.plan_vector(toy.q, L, toy.scale, pvec(basis, polys, mp), toy.scale * tmul, lpr, toy.prec, toy.logN, log_slots), mp


def ckks_oracle(toy, case, ct, mp):
    basis, polys, kind, lpr, tmul = case
    pe = V.CKKSPolyVectorEvaluator(toy.params, toy.rlk, lpr, toy.prec)
    return pe.EvaluateVector(OP.Ct(ct, toy.scale), oracle_polys(basis, polys), mp, toy.scale * tmul)


def bgv_cases(t, seed=5):
    """name -> ([(coeffs, odd, even)], mapping kind)."""
    from tests import bgv_polyeval_cases as BC
    rng = np.random.default_rng(seed)
    return {
        "d7": ([(BC._coeffs(rng, 7, t), True, True), (BC._coeffs(rng, 7, t), True, True)], "eo"),
        "d15": ([(BC._coeffs(rng, 15, t), True, True), (BC._coeffs(rng, 15, t), True, True)], "eo"),
        "d31_three": ([(BC._coeffs(rng, 31, t), True, True) for _ in range(3)], "three"),
        "odd15": ([(BC._coeffs(rng, 15, t, odd=True, even=False), True, False)] * 2, "eo"),
        "even14": ([(BC._coeffs(rng, 14, t, odd=False, even=True), False, True), (BC._coeffs(rng, 14, t, odd=False, even=True), False, True)], "half"),
    }


def bgv_plan(toy, polys, kind, invariant, level, scale=1, target=1):
    mp = mapping(kind, toy.enc.MaxSlots(), len(polys))
    pv = PE.NewPolynomialVector([PE.Polynomial(c, PE.MONOMIAL, o, e) for c, o, e in polys], mp)
    return BPE.plan_vector(toy.q, toy.t, level, scale, pv, target, invariant, toy.enc.MaxSlots()), mp


def bgv_oracle(toy, polys, mp, invariant, ct, scale=1, target=1):
    pe = V.BGVPolyVectorEvaluator(toy.params, toy.rlk, toy.t, toy.qmul, invariant)
    return pe.EvaluateVector(BP.P.Ct(ct, scale), bgv_oracle_polys(polys), mp, target), pe

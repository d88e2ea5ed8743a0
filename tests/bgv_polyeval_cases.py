"""Shared fixtures of the BGV / BFV polynomial evaluation tests: a toy scheme with real keys (slot encoding by oracle/bgv_encoder.py),
the polynomial cases, and an exact CPU interpreter of the planner's folded programs."""
from __future__ import annotations

import numpy as np

from lattigo_b200 import polyeval as PE
from oracle import bgv_encoder as OE
from oracle import oracle as O
from tests import bgv_oracle as B
from tests import bgv_polyeval_oracle as BP
from tests import helpers as H

U64 = np.uint64

# bgv.testInsecure (circuits/bgv/polynomial/polynomial_evaluator_test.go)
INSECURE_Q = [0x3fffffa8001, 0x1000090001, 0x10000c8001, 0x10000f0001, 0xffff00001]
INSECURE_P = [0x7fffffd8001]
INSECURE_T = [0x101, 0xffc001]


def _coeffs(rng, deg, t, odd=True, even=True, sparse=False):
    c = [int(x) for x in rng.integers(0, t, deg + 1)]
    for k in range(deg + 1):
        if sparse and k not in (0, 1, deg) and k % 5:
            c[k] = 0
        if (odd and not even and k % 2 == 0) or (even and not odd and k % 2 == 1):
            c[k] = 0
    c[deg] = c[deg] or 1
    return c


def cases(t, seed=3):
    """name -> (coeffs, odd, even): x^2, dense degrees, odd-only, even-only and sparse polynomials."""
    rng = np.random.default_rng(seed)
    out = {"x2": ([0, 0, 1], True, True)}
    for d in (3, 7, 8, 15, 16, 31, 63):
        out["d%d" % d] = (_coeffs(rng, d, t), True, True)
    out["odd15"] = (_coeffs(rng, 15, t, odd=True, even=False), True, False)
    out["even14"] = (_coeffs(rng, 14, t, odd=False, even=True), False, True)
    out["sparse31"] = (_coeffs(rng, 31, t, sparse=True), True, True)
    return out


def eval_poly_mod(coeffs, x, t):
    """ring.EvalPolyModP with the parity flags applied the way the evaluator reads the coefficients."""
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % t
    return acc


def parity(coeffs, odd, even):
    """The coefficients Evaluate reads: with exactly one flag set, the other parity is skipped."""
    if odd == even:
        return list(coeffs)
    return [c if (k % 2 == 1 and odd) or (k % 2 == 0 and even) else 0 for k, c in enumerate(coeffs)]


class Toy:
    """Keys, slot encoding, encryption and decryption for a (Q, P, t) chain."""

    def __init__(self, logN, q, p, t, seed=1):
        self.logN, self.q, self.p, self.t = logN, [int(x) for x in q], [int(x) for x in p], int(t)
        self.params = O.Parameters(logN, self.q, self.p)
        self.N = self.params.N()
        self.qmul = B.qmul_moduli(logN, self.q)
        self.rng = np.random.default_rng(seed)
        self.s = self.rng.integers(-1, 2, self.N)
        s2 = self._sq(self.s)
        self.rlk = H.gen_switching_key(self.params, s2, self.s, self.rng)
        self.enc = OE.BGVEncoder(self.params.ringQ, self.t)

    @staticmethod
    def _sq(s):
        N = len(s)
        full = np.convolve(s.astype(np.int64), s.astype(np.int64))
        out = full[:N].copy()
        out[: N - 1] -= full[N:]
        return [int(x) for x in out]

    def evaluator(self, invariant):
        return BP.PolyEvaluator(self.params, self.rlk, self.t, self.qmul, invariant)

    def _ntt(self, rows, level):
        out = np.empty_like(rows)
        self.params.ringQ.AtLevel(level).NTT(rows, out)
        return out

    def encrypt(self, values, level):
        """Encode (scale 1, NTT) then (-a s + e + pt, a)."""
        mods = self.q[: level + 1]
        pt = np.array(self.enc.Encode(values, False, 1, True, False, level), dtype=U64)
        ring = self.params.ringQ.AtLevel(level)
        a = H.rand_poly(mods, self.N, self.rng)
        e = self._ntt(H.small_poly_rns(np.rint(self.rng.normal(0, 3.2, self.N)).astype(np.int64), mods), level)
        s = self._ntt(H.small_poly_rns(self.s, mods), level)
        c0 = np.empty_like(a)
        ring.MulCoeffsBarrett(a, s, c0)
        ring.Neg(c0, c0)
        ring.Add(c0, e, c0)
        ring.Add(c0, pt, c0)
        return [c0, a]

    def decrypt(self, ct, scale):
        level = ct[0].shape[0] - 1
        ring = self.params.ringQ.AtLevel(level)
        s = self._ntt(H.small_poly_rns(self.s, self.q[: level + 1]), level)
        x = np.empty_like(ct[0])
        ring.MulCoeffsBarrett(ct[1], s, x)
        ring.Add(x, ct[0], x)
        if len(ct) == 3:
            y = np.empty_like(x)
            ring.MulCoeffsBarrett(ct[2], s, y)
            ring.MulCoeffsBarrett(y, s, y)
            ring.Add(x, y, x)
        return self.enc.Decode(x, level, scale, True)

    def random_values(self):
        return [int(v) for v in self.rng.integers(0, self.t, self.enc.MaxSlots())]


def interpret(toy, invariant, prog, ct_value):
    """Runs a planned program with the oracle's tensor / relinearization / rescale; LINCOMB and TENSOR weights in exact integers."""
    Q, N = toy.q, toy.N
    pe = toy.evaluator(invariant)
    ev = pe.ev
    slots = {0: [np.array(v) for v in ct_value]}
    for o in prog.ops:
        k = o["kind"]
        if k == PE.MULRELIN:
            a = slots[o["src0"]]
            b = a if o["src1"] == o["src0"] else slots[o["src1"]]
            slots[o["dst"]] = ev.MulRelinNew(a, b)
        elif k == PE.RELIN:
            out = [np.empty_like(slots[o["src0"]][0]) for _ in range(2)]
            ev.Relinearize(slots[o["src0"]], toy.rlk, out)
            slots[o["dst"]] = out
        elif k == PE.RESCALE:
            ev.ScaleInvariant, si = False, ev.ScaleInvariant
            slots[o["dst"]] = ev.Rescale(slots[o["src0"]])
            ev.ScaleInvariant = si
        elif k == PE.TENSOR:
            lv = o["level"]
            b, x = [v[: lv + 1] for v in slots[o["src0"]]], [v[: lv + 1] for v in slots[o["src1"]]]
            t = ev.MulNew(b, x)
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
                                assert W[i, kk, r, 0] == 0 and W[i, kk, r, 1] == 0
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


def oracle_eval(toy, invariant, ct_value, scale, coeffs, target, odd=True, even=True):
    pe = toy.evaluator(invariant)
    r = pe.Evaluate(BP.P.Ct(ct_value, scale), BP.new_polynomial(coeffs, odd, even), target)
    return r, pe

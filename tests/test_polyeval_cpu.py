"""The polynomial-evaluation planner (lattigo_b200/polyeval.py) on the CPU:
- its folded program, interpreted op by op with the oracle's rounding ops (MulRelinNew, Relinearize, Rescale, the tensor) and Python
  integers for LINCOMB / TENSOR weights, equals oracle/polyeval.py's literal op-by-op evaluation bit for bit, with the same level and scale;
- the op and launch counts of each case, with every baby step in one LINCOMB;
- lgpu_ckks_polynomial_evaluate rejects malformed programs on a host-only context."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest

from lattigo_b200 import polyeval as PE
from oracle import oracle as O
from oracle import polyeval as OP
from tests import polyeval_cases as PC

U64 = np.uint64


@pytest.fixture(scope="module")
def toys():
    return {1: PC.Toy(lpr=1), 2: PC.Toy(lpr=2, nlevels=4, logscale=80)}


def interpret(toy, prog, ct_value):
    """Runs a planned program with the oracle's rounding ops; LINCOMB / TENSOR weights in exact integers."""
    Q, N = toy.q, toy.N
    ev = O.CKKSEvaluator(toy.params, toy.rlk, toy.lpr)
    pe = OP.PolyEvaluator(toy.params, toy.rlk, toy.lpr, toy.prec)
    slots = {0: [np.array(v) for v in ct_value]}
    for o in prog.ops:
        k = o["kind"]
        if k == PE.MULRELIN:
            a, b = slots[o["src0"]], slots[o["src1"]]
            slots[o["dst"]] = ev.MulRelinNew(a, b)
        elif k == PE.RELIN:
            slots[o["dst"]] = pe.relinearize(OP.Ct(slots[o["src0"]], 1)).Value
        elif k == PE.RESCALE:
            slots[o["dst"]] = ev.Rescale(slots[o["src0"]])
        elif k == PE.TENSOR:
            lv = o["level"]
            b, x = OP.Ct([v[: lv + 1] for v in slots[o["src0"]]], 1), OP.Ct([v[: lv + 1] for v in slots[o["src1"]]], 1)
            t = pe.mul_tensor(b, x).Value
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


def _plan(toy, case):
    basis, coeffs, odd, even, lpr, tmul = case
    L = toy.params.MaxLevelQ()
    roots1 = [int(sr.RootsForward[1]) for sr in toy.params.ringQ.SubRings]      # what PolynomialEvaluator reads from the context
    return PE.plan(toy.q, L, toy.scale, coeffs, basis, toy.scale * tmul, lpr, toy.prec, odd, even, roots1)


@pytest.mark.parametrize("name", sorted(PC.cases()))
def test_folded_program_equals_the_literal_oracle(name, toys):
    case = PC.cases()[name]
    basis, coeffs, odd, even, lpr, tmul = case
    toy = toys[lpr]
    x = np.random.default_rng(5).uniform(-1, 1, toy.N // 2)
    ct = toy.encrypt(x)
    prog = _plan(toy, case)
    got = interpret(toy, prog, ct)
    want = OP.PolyEvaluator(toy.params, toy.rlk, lpr, toy.prec).Evaluate(OP.Ct(ct, toy.scale), OP.new_polynomial(basis, coeffs, odd, even),
                                                                         toy.scale * tmul)
    assert prog.out_level == want.Level() and prog.out_scale == want.Scale
    assert len(got) == 2 and all(np.array_equal(g, w) for g, w in zip(got, want.Value))
    if any(complex(c).imag for c in coeffs):
        # the halves really differ: some LINCOMB weight of the lower NTT half is not the upper half's
        w = [o["weights"] for o in prog.ops if o["kind"] == PE.LINCOMB][-1]
        assert any(w[k] != w[k + 1] for k in range(0, len(w), 2))


# op counts: (MULRELIN, TENSOR, RELIN, RESCALE, LINCOMB)
EXPECTED_OPS = {
    "mono1": (0, 0, 0, 1, 1),
    "mono2": (1, 1, 1, 3, 1),
    "mono3": (1, 1, 1, 3, 1),
    "mono5_giant2": (3, 1, 1, 5, 1),
    "mono7": (3, 2, 2, 6, 1),
    "mono15": (4, 4, 3, 9, 1),
    "const_only": (0, 0, 0, 1, 1),
    "cheb12_general": (4, 3, 2, 8, 5),
    "cheb30_even": (6, 4, 3, 11, 7),
    "cheb63_odd": (8, 9, 6, 18, 9),
}


@pytest.mark.parametrize("name", sorted(EXPECTED_OPS))
def test_program_op_counts_and_one_lincomb_for_all_baby_steps(name, toys):
    case = PC.cases()[name]
    prog = _plan(toys[case[4]], case)
    kinds = prog.kinds()
    got = tuple(kinds.count(k) for k in (PE.MULRELIN, PE.TENSOR, PE.RELIN, PE.RESCALE, PE.LINCOMB))
    assert got == EXPECTED_OPS[name], got
    # the power basis' Chebyshev combines are one-output LINCOMBs; the baby steps are ONE LINCOMB with every baby step as an output
    lin = [o for o in prog.ops if o["kind"] == PE.LINCOMB]
    assert sum(1 for o in lin if len(o["outs"]) > 1 or o is lin[-1]) == 1
    assert len(lin[-1]["terms"]) <= PE.MAX_TERMS
    # the baby-step LINCOMB comes after the last power and before the first giant step
    i = prog.ops.index(lin[-1])
    assert all(o["kind"] != PE.TENSOR for o in prog.ops[:i])
    assert all(o["kind"] != PE.MULRELIN for o in prog.ops[i:])


def test_degree_255_fits_the_term_bound():
    toyQ = O.gen_moduli(11, [60] + [40] * 10, [55])[0]
    prog = PE.plan(toyQ, 10, 2 ** 40, [0.01] * 256, PE.CHEBYSHEV, 2 ** 40)
    lin = [o for o in prog.ops if o["kind"] == PE.LINCOMB][-1]
    assert len(lin["terms"]) == 15 and len(lin["outs"]) == 20          # the reference re-splits the leading baby steps
    with pytest.raises(ValueError):
        PE.plan(toyQ, 10, 2 ** 40, [0.01] * 257, PE.CHEBYSHEV, 2 ** 40)


# ---- C-ABI checks on a host-only context --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host():
    import lattigo_b200 as lb
    q, p = O.gen_moduli(11, [55] + [40] * 8, [55, 55])
    ctx = lb.Context(10, q, p, device=-1)
    yield ctx, q
    ctx.close()


def _call(ctx, level, prog_struct, rlk=None, batch=1):
    import lattigo_b200 as lb
    buf = (ctypes.c_uint64 * 2)()
    addr = (ctypes.addressof(buf) + 15) & ~15
    g = None
    if rlk is not False:
        data = (ctypes.c_uint64 * 4)()
        g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), level, 1, 0, 8, 1, None)
    return lb._lib.lib().lgpu_ckks_polynomial_evaluate(ctx.h, level, ctypes.c_void_p(addr), batch, ctypes.byref(prog_struct),
                                                       ctypes.byref(g) if g is not None else None, ctypes.c_void_p(addr), None)


def _err(ctx, level, prog, lpr=1, rlk=None):
    import lattigo_b200 as lb
    rc = _call(ctx, level, prog.to_c(lpr), rlk)
    return None if rc == 0 else lb._lib.lib().lgpu_last_error().decode()


def test_well_formed_program_reaches_the_device_check(host):
    ctx, q = host
    prog = PE.plan(q, 8, 2 ** 40, [0.1, 0.2, 0.3, 0.4], PE.MONOMIAL, 2 ** 40)
    assert "host-only" in _err(ctx, 8, prog)


def _mutated(q, fn):
    prog = PE.plan(q, 8, 2 ** 40, [0.1, 0.2, 0.3, 0.4], PE.CHEBYSHEV, 2 ** 40)
    fn(prog)
    return prog


def test_malformed_programs_are_rejected_before_any_launch(host):
    ctx, q = host
    lin = lambda p: [o for o in p.ops if o["kind"] == PE.LINCOMB][-1]
    bad = {
        "slot count": lambda p: setattr(p, "n_slots", 1),
        "reads a slot before": lambda p: p.ops[0].update(src0=p.n_slots - 1),
        "writes a slot twice": lambda p: [o for o in p.ops if o["kind"] == PE.RESCALE][-1].update(dst=p.ops[0]["dst"]),
        "minimum level": lambda p: p.ops[0].update(level=p.ops[0]["level"] - 1),
        "RESCALE level": lambda p: [o.update(level=o["level"] + 1) for o in p.ops if o["kind"] == PE.RESCALE][:1],
        "below its modulus": lambda p: lin(p)["weights"].__setitem__(0, q[0]),
        "term count": lambda p: lin(p).update(terms=list(range(PE.MAX_TERMS + 1))),
        "output slot": lambda p: setattr(p, "out_slot", 0),
        "output level": lambda p: lin(p).update(out_levels=[9] * len(lin(p)["outs"])),
    }
    for msg, fn in bad.items():
        e = _err(ctx, 8, _mutated(q, fn))
        assert e is not None and msg in e, (msg, e)
    # levels_per_rescale inconsistent with the RESCALE levels
    e = _err(ctx, 8, _mutated(q, lambda p: None), lpr=2)
    assert "Rescale" in e
    # input level above the context
    assert "level out of range" in _err(ctx, 9, _mutated(q, lambda p: None))
    # a relinearization key below the level of a MULRELIN
    prog = _mutated(q, lambda p: None)
    cp = prog.to_c(1)
    import lattigo_b200 as lb
    data = (ctypes.c_uint64 * 4)()
    g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), 3, 1, 0, 8, 1, None)
    buf = (ctypes.c_uint64 * 4)()
    addr = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    assert lb._lib.lib().lgpu_ckks_polynomial_evaluate(ctx.h, 8, addr, 1, ctypes.byref(cp), ctypes.byref(g), addr, None) != 0
    assert "levelQ out of range for this evaluation key" in lb._lib.lib().lgpu_last_error().decode()
    # no key at all
    assert "relinearization key" in _err(ctx, 8, _mutated(q, lambda p: None), rlk=False)


def test_planner_rejects_what_the_reference_rejects():
    q = O.gen_moduli(11, [55] + [40] * 8, [55])[0]
    with pytest.raises(ValueError):
        PE.plan(q, 8, 2 ** 40, [0.5], PE.MONOMIAL, 2 ** 40)                 # degree 0
    with pytest.raises(ValueError):
        PE.plan(q, 2, 2 ** 40, [0.5] * 16, PE.MONOMIAL, 2 ** 40)           # 2 levels < Depth(15) = 4
    with pytest.raises(ValueError):
        PE.plan(q, 8, 2 ** 40, [0.5, 0.5j], PE.MONOMIAL, 2 ** 40)          # complex coefficient without RootsForward[1]
    assert PE.plan(q, 8, Fraction(2 ** 40), [0.5, 0.25], PE.MONOMIAL, 2 ** 40).out_level == 7

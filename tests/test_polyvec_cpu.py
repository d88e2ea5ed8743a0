"""Polynomial-vector evaluation (Evaluate with a PolynomialVector and a Mapping) on the CPU:
- the planner's vector program, run by an exact interpreter (PTLINCOMB on the oracle-encoded plaintexts), equals the literal oracle
  (tests/polyvec_oracle.py) word for word, with the same output level and scale, for CKKS and BGV / BFV;
- the oracle is pinned by decryption with real keys (the reference's Polynomial/PolyVector/Exp test);
- a nil Mapping plans exactly the scalar program;
- the planner and lgpu_*_polynomial_vector_evaluate refuse what they must, before any launch, on a host-only context."""
import ctypes
import math

import numpy as np
import pytest

from lattigo_b200 import bgv_polyeval as BPE
from lattigo_b200 import polyeval as PE
from oracle import oracle as O
from tests import bgv_polyeval_cases as BC
from tests import polyeval_cases as PC
from tests import polyvec_cases as VC


@pytest.fixture(scope="module")
def toys():
    return {1: PC.Toy(lpr=1), 2: PC.Toy(lpr=2, nlevels=4, logscale=50)}


@pytest.fixture(scope="module")
def bgv_toy():
    q, p = O.gen_moduli(11, [55] + [45] * 9, [60, 60])
    return BC.Toy(10, q, p, 0xffc001, seed=9)


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _ckks_check(toy, case, ct):
    prog, mp = VC.ckks_plan(toy, case)
    pts = VC.ckks_encode_plaintexts(toy.params, prog)
    got = VC.interpret(prog, ct, pts, toy.q, toy.N, VC.ckks_ops(toy))
    want = VC.ckks_oracle(toy, case, ct, mp)
    assert (prog.out_level, prog.out_scale) == (want.Level(), want.Scale)
    assert _same(got, want.Value)
    return prog


@pytest.mark.parametrize("name", sorted(VC.ckks_cases()))
def test_ckks_vector_program_equals_the_literal_oracle(name, toys):
    case = VC.ckks_cases()[name]
    toy = toys[case[3]]
    ct = toy.encrypt(np.random.default_rng(5).uniform(-1, 1, toy.N // 2))
    prog = _ckks_check(toy, case, ct)
    kinds = prog.kinds()
    assert kinds.count(PE.PTLINCOMB) == 1                     # every baby step in one op
    assert case[0] == VC.C or PE.LINCOMB not in kinds         # only the Chebyshev power basis keeps LINCOMBs
    o = [o for o in prog.ops if o["kind"] == PE.PTLINCOMB][0]
    assert len(o["terms"]) <= PE.MAX_TERMS
    assert all(o["kind"] != PE.TENSOR for o in prog.ops[: prog.ops.index(o)])


def test_ckks_lpr2_keeps_the_encoding_precision_at_53_bits(toys):
    """lpr = 2 on 25-bit primes: a 50-bit scale, so EncodingPrecision = 53 and the float64 encoder path applies."""
    toy = toys[2]
    assert toy.prec == 53
    case = VC.ckks_cases()["mono7_lpr2"]
    ct = toy.encrypt(np.random.default_rng(6).uniform(-1, 1, toy.N // 2))
    _ckks_check(toy, case, ct)


def test_ckks_equal_scale_branch_is_reached(toys):
    """MulThenAdd(X^k, vector, res) with X^k.Scale == res.Scale multiplies res by q_level first, even for integer coefficients: a
    degree-1 polynomial whose target scale makes the baby step's scale the input's."""
    toy = toys[1]
    L = toy.params.MaxLevelQ()
    target = OP_scale = toy.scale / toy.q[L]                 # the baby step's scale target * q_L is the input's
    case = (VC.M, [([0.5, 2.0], True, True), ([1.0, -3.0], True, True)], "eo", 1, 1)
    mp = VC.mapping("eo", toy.N // 2, 2)
    prog = PE.plan_vector(toy.q, L, toy.scale, VC.pvec(case[0], case[1], mp), target, 1, toy.prec, toy.logN)
    o = [o for o in prog.ops if o["kind"] == PE.PTLINCOMB][0]
    K = len(o["terms"]) + 1
    # the constant (added before the q_level product) carries s = q_level mod q_r; the term carries 1
    assert o["scalars"][(K - 1) * (o["level"] + 1)] == toy.q[L] % toy.q[0]
    ct = toy.encrypt(np.random.default_rng(7).uniform(-1, 1, toy.N // 2))
    pts = VC.ckks_encode_plaintexts(toy.params, prog)
    got = VC.interpret(prog, ct, pts, toy.q, toy.N, VC.ckks_ops(toy))
    from oracle import polyeval as OP
    from tests import polyvec_oracle as V
    want = V.CKKSPolyVectorEvaluator(toy.params, toy.rlk, 1, toy.prec).EvaluateVector(OP.Ct(ct, toy.scale), VC.oracle_polys(case[0], case[1]),
                                                                                     mp, OP_scale)
    assert _same(got, want.Value) and prog.out_scale == want.Scale


def test_ckks_poly_vector_exp_decrypts(toys):
    """The reference's Polynomial/PolyVector/Exp test: Taylor exp of degree 7 on the even slots, nothing on the odd ones."""
    toy = toys[1]
    x = np.random.default_rng(8).uniform(-1, 1, toy.N // 2)
    ct = toy.encrypt(x)
    coeffs = [1 / math.factorial(k) for k in range(8)]
    mp = {0: list(range(0, toy.N // 2, 2))}
    from oracle import polyeval as OP
    from tests import polyvec_oracle as V
    out = V.CKKSPolyVectorEvaluator(toy.params, toy.rlk, 1, toy.prec).EvaluateVector(OP.Ct(ct, toy.scale), [OP.new_polynomial(VC.M, coeffs)],
                                                                                    mp, toy.scale)
    got = toy.decrypt(out.Value, out.Scale)
    want = np.where(np.arange(toy.N // 2) % 2 == 0, np.polynomial.polynomial.polyval(x, coeffs), 0)
    assert np.max(np.abs(got - want)) < 2 ** -20


@pytest.mark.parametrize("invariant", [False, True])
def test_bgv_vector_program_equals_the_literal_oracle(bgv_toy, invariant):
    toy = bgv_toy
    L = len(toy.q) - 1
    ct = toy.encrypt(toy.random_values(), L)
    for name, (polys, kind) in VC.bgv_cases(toy.t).items():
        for scale, target in ((1, 1), (12345, 777)):
            prog, mp = VC.bgv_plan(toy, polys, kind, invariant, L, scale, target)
            pts = VC.bgv_encode_plaintexts(toy.enc, prog)
            got = VC.interpret(prog, ct, pts, toy.q, toy.N, VC.bgv_ops(toy, invariant))
            want, pe = VC.bgv_oracle(toy, polys, mp, invariant, ct, scale, target)
            assert (prog.out_level, prog.out_scale) == (want.Level(), int(want.Scale)), name
            assert _same(got, want.Value), name
            # MulThenAdd(X^k, vector, res) encodes at X^k.Scale^-1 res.Scale, so op0.Scale * pt.Scale = res.Scale and
            # matchScalesBinary is never reached (r0 = 1): see test_bgv_match_scales_unreachable
            assert pe.counts["vector_matchScalesBinary"] == 0
            K = len([o for o in prog.ops if o["kind"] == PE.PTLINCOMB][0]["terms"])
            assert K <= PE.MAX_TERMS


def test_bgv_match_scales_unreachable():
    """r0 != 1 is not reachable: for any scales a = X^k.Scale, c = res.Scale in [1, t) (t prime), pt.Scale = a^-1 c (or 1 when a = c)
    gives a pt.Scale = c mod t, the target scale mulRelinThenAdd compares with res.Scale."""
    t = 0xffc001
    rng = np.random.default_rng(1)
    for a, c in [(1, 1), (t - 1, 2)] + [tuple(int(v) for v in rng.integers(1, t, 2)) for _ in range(200)]:
        pt = 1 if a == c else pow(a, t - 2, t) * c % t
        assert a * pt % t == c


@pytest.mark.parametrize("invariant", [False, True])
def test_bgv_poly_vector_decrypts_exactly(bgv_toy, invariant):
    toy = bgv_toy
    L = len(toy.q) - 1
    vals = toy.random_values()
    ct = toy.encrypt(vals, L)
    polys, kind = VC.bgv_cases(toy.t)["d7"]
    prog, mp = VC.bgv_plan(toy, polys, kind, invariant, L)
    want, _ = VC.bgv_oracle(toy, polys, mp, invariant, ct)
    got = toy.decrypt(want.Value, int(want.Scale))
    for i, js in mp.items():
        for j in js:
            assert got[j] == BC.eval_poly_mod(polys[i][0], vals[j], toy.t)


def test_nil_mapping_plans_the_scalar_program(toys, bgv_toy):
    toy = toys[1]
    L = toy.params.MaxLevelQ()
    for name, (basis, coeffs, odd, even, lpr, tmul) in PC.cases().items():
        if lpr != 1:
            continue
        roots1 = [int(sr.RootsForward[1]) for sr in toy.params.ringQ.SubRings]
        a = PE.plan(toy.q, L, toy.scale, coeffs, basis, toy.scale * tmul, 1, toy.prec, odd, even, roots1)
        b = PE.plan_vector(toy.q, L, toy.scale, PE.NewPolynomialVector([PE.Polynomial(coeffs, basis, odd, even)], None), toy.scale * tmul,
                           1, toy.prec, toy.logN, roots1=roots1)
        assert a.ops == b.ops and (a.n_slots, a.out_slot, a.out_level, a.out_scale) == (b.n_slots, b.out_slot, b.out_level, b.out_scale)
        assert not b.plaintexts
    bt = bgv_toy
    coeffs, odd, even = BC.cases(bt.t)["d15"]
    a = BPE.plan(bt.q, bt.t, 9, 1, coeffs, 1, False, odd, even)
    b = BPE.plan_vector(bt.q, bt.t, 9, 1, PE.NewPolynomialVector([PE.Polynomial(coeffs)], None), 1, False, bt.enc.MaxSlots())
    assert a.ops == b.ops and a.out_slot == b.out_slot


def test_planner_refusals(toys):
    toy = toys[1]
    L = toy.params.MaxLevelQ()
    P = PE.Polynomial
    with pytest.raises(ValueError, match="polynomial degree must all be the same"):
        PE.NewPolynomialVector([P([1, 2, 3]), P([1, 2])], {0: [0]})
    with pytest.raises(ValueError, match="polynomial basis must be the same for all polynomials in a polynomial vector"):
        PE.NewPolynomialVector([P([1, 2], PE.CHEBYSHEV), P([1, 2], PE.MONOMIAL)], {0: [0]})
    pv = PE.NewPolynomialVector([P([0.1, 0.2, 0.3]), P([0.3, 0.2, 0.1])], VC.even_odd(toy.N // 2))
    with pytest.raises(ValueError, match="cannot Embed: ensure that #values"):
        PE.plan_vector(toy.q, L, toy.scale, pv, toy.scale, 1, toy.prec, toy.logN, log_slots=toy.logN - 2)
    with pytest.raises(ValueError, match="EncodingPrecision"):
        PE.plan_vector(toy.q, L, toy.scale, pv, toy.scale, 1, 60, toy.logN)
    with pytest.raises(ValueError, match="out of range"):
        PE.plan_vector(toy.q, L, toy.scale, PE.NewPolynomialVector([P([0.1, 0.2])], {0: [toy.N // 2]}), toy.scale, 1, toy.prec, toy.logN)
    # complex coefficients need no RootsForward[1]: the slot vectors are encoded
    pvc = PE.NewPolynomialVector([P([0.1j, 0.2]), P([0.3, 0.2j])], VC.even_odd(toy.N // 2))
    assert PE.plan_vector(toy.q, L, toy.scale, pvc, toy.scale, 1, toy.prec, toy.logN).plaintexts


# ---- C-ABI checks on a host-only context --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host():
    import lattigo_b200 as lb
    q, p = O.gen_moduli(11, [55] + [40] * 8, [55, 55])
    ctx = lb.Context(10, q, p, device=-1)
    yield ctx, q
    ctx.close()


class _Buf:
    def __init__(self, words):
        self.raw = (ctypes.c_uint64 * (words + 2))()
        self.addr = (ctypes.addressof(self.raw) + 15) & ~15


def _vec_prog(q):
    pv = PE.NewPolynomialVector([PE.Polynomial([0.1, 0.2, 0.3, 0.4]), PE.Polynomial([0.4, 0.3, 0.2, 0.1])], VC.even_odd(512))
    return PE.plan_vector(q, 8, 2 ** 40, pv, 2 ** 40, 1, 53, 10)


def _vcall(ctx, prog, pts=None, level=8, mutate_w=None, ct=None, lpr=1):
    import lattigo_b200 as lb
    N = 1024
    rows = max(p["level"] for p in prog.plaintexts) + 1
    block = pts or _Buf(len(prog.plaintexts) * rows * N)
    levels = [p["level"] for p in prog.plaintexts]
    cp = prog.to_c(lpr)
    vw = prog.pt_weights_to_c(block.addr, rows * N, levels)
    if mutate_w:
        mutate_w(vw)
    ctb = ct or _Buf(2 * 2 * (level + 1) * N)
    out = _Buf(2 * 2 * (level + 1) * N)
    data = (ctypes.c_uint64 * 4)()
    g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), level, 1, 0, 8, 1, None)
    rc = lb._lib.lib().lgpu_ckks_polynomial_vector_evaluate(ctx.h, level, ctypes.c_void_p(ctb.addr), 1, ctypes.byref(cp), ctypes.byref(vw),
                                                            ctypes.byref(g), ctypes.c_void_p(out.addr), None)
    return None if rc == 0 else lb._lib.lib().lgpu_last_error().decode()


def test_well_formed_vector_program_reaches_the_device_check(host):
    ctx, q = host
    assert "host-only" in _vcall(ctx, _vec_prog(q))


def test_malformed_vector_programs_are_rejected_before_any_launch(host):
    ctx, q = host
    ptl = lambda p: [o for o in p.ops if o["kind"] == PE.PTLINCOMB][0]
    bad = {
        "plaintext index out of range": lambda p: ptl(p)["index"].__setitem__(0, len(p.plaintexts)),
        "PTLINCOMB scalar not below its modulus": lambda p: ptl(p)["scalars"].__setitem__(0, q[0]),
        "PTLINCOMB term count": lambda p: ptl(p).update(terms=list(range(PE.MAX_TERMS + 1))),
        "PTLINCOMB output level": lambda p: ptl(p).update(out_levels=[9] * len(ptl(p)["outs"])),
        "exactly one PTLINCOMB": lambda p: p.ops.__setitem__(0, dict(p.ops[0], kind=PE.PTLINCOMB, outs=[1], out_levels=[p.ops[0]["level"]],
                                                                     terms=[], index=[0], scalars=[1] * (p.ops[0]["level"] + 1))),
    }
    for msg, fn in bad.items():
        prog = _vec_prog(q)
        fn(prog)
        e = _vcall(ctx, prog)
        assert e is not None and msg in e, (msg, e)
    prog = _vec_prog(q)
    prog.plaintexts[0]["level"] = 0                           # below the output that uses it
    assert "plaintext below its level" in _vcall(ctx, prog)
    prog = _vec_prog(q)
    prog.plaintexts[0]["level"] = 9
    assert "plaintext level out of range" in _vcall(ctx, prog)
    assert "plaintext count" in _vcall(ctx, _vec_prog(q), mutate_w=lambda w: setattr(w, "n_pt", 0))
    assert "null plaintext table" in _vcall(ctx, _vec_prog(q), mutate_w=lambda w: setattr(w, "index", None))
    assert "stride" in _vcall(ctx, _vec_prog(q), mutate_w=lambda w: setattr(w, "pt_stride", 1024))
    # the plaintext block overlapping the input
    prog = _vec_prog(q)
    ct = _Buf(2 * 2 * 9 * 1024 + len(prog.plaintexts) * 9 * 1024)
    assert "overlaps" in _vcall(ctx, prog, pts=ct, ct=ct)


def test_the_new_kind_is_unknown_to_the_scalar_entry_point(host):
    import lattigo_b200 as lb
    ctx, q = host
    prog = _vec_prog(q)
    cp = prog.to_c(1)
    buf = _Buf(2 * 2 * 9 * 1024)
    data = (ctypes.c_uint64 * 4)()
    g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), 8, 1, 0, 8, 1, None)
    assert lb._lib.lib().lgpu_ckks_polynomial_evaluate(ctx.h, 8, ctypes.c_void_p(buf.addr), 1, ctypes.byref(cp), ctypes.byref(g),
                                                       ctypes.c_void_p(buf.addr), None) != 0
    assert "unknown polynomial program op" in lb._lib.lib().lgpu_last_error().decode()
    # and a vector entry point without a table
    assert lb._lib.lib().lgpu_ckks_polynomial_vector_evaluate(ctx.h, 8, ctypes.c_void_p(buf.addr), 1, ctypes.byref(cp), None, ctypes.byref(g),
                                                              ctypes.c_void_p(buf.addr), None) != 0
    assert "null plaintext table" in lb._lib.lib().lgpu_last_error().decode()


def test_bgv_vector_entry_point_checks(host):
    import lattigo_b200 as lb
    ctx, q = host
    t = 0xffc001
    h = ctypes.c_void_p()
    qmul = O.gen_moduli(11, [61] * 12, [])[0]
    qm = (ctypes.c_uint64 * len(qmul))(*qmul)
    lb._lib.check(lb._lib.lib().lgpu_bgv_create(ctx.h, t, qm, len(qmul), ctypes.byref(h)))
    try:
        pv = PE.NewPolynomialVector([PE.Polynomial([1, 2, 3, 4]), PE.Polynomial([4, 3, 2, 1])], VC.even_odd(512))
        prog = BPE.plan_vector(q, t, 8, 1, pv, 1, False, 1024)
        N = 1024
        rows = max(p["level"] for p in prog.plaintexts) + 1
        block = _Buf(len(prog.plaintexts) * rows * N)
        vw = prog.pt_weights_to_c(block.addr, rows * N, [p["level"] for p in prog.plaintexts])
        cp = prog.to_c(1)
        buf = _Buf(2 * 2 * 9 * N)
        data = (ctypes.c_uint64 * 4)()
        g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), 8, 1, 0, 8, 1, None)
        call = lambda si, p: lb._lib.lib().lgpu_bgv_polynomial_vector_evaluate(h, 8, ctypes.c_void_p(buf.addr), 1, ctypes.byref(p), ctypes.byref(vw),
                                                                             ctypes.byref(g), si, ctypes.c_void_p(buf.addr + 8 * 2 * 9 * N), None)
        assert call(0, cp) != 0 and "host-only" in lb._lib.lib().lgpu_last_error().decode()
        assert call(1, cp) != 0 and "RESCALE in a scale_invariant program" in lb._lib.lib().lgpu_last_error().decode()
        assert call(2, cp) != 0 and "scale_invariant must be 0 or 1" in lb._lib.lib().lgpu_last_error().decode()
        assert lb._lib.lib().lgpu_bgv_polynomial_evaluate(h, 8, ctypes.c_void_p(buf.addr), 1, ctypes.byref(cp), ctypes.byref(g), 0,
                                                          ctypes.c_void_p(buf.addr), None) != 0
        assert "unknown polynomial program op" in lb._lib.lib().lgpu_last_error().decode()
    finally:
        lb._lib.lib().lgpu_bgv_destroy(h)


def _replayed_scalars(o, Q, term_factor):
    """The per-limb scalars that the op's recorded reference order (sequence) implies: each plaintext product is multiplied by every
    later multiplication of res; a term's product also by term_factor (BGV: t, from MRed(pt, tMontgomery))."""
    nt, L = len(o["terms"]), o["level"]
    K = nt + 1
    out = [0] * (len(o["outs"]) * K * (L + 1))
    for i, (seq, lv) in enumerate(zip(o["sequence"], o["out_levels"])):
        prod = [1] * (lv + 1)
        for kind, arg in reversed(seq):
            if kind == "mul":
                prod = [p * m % q for p, m, q in zip(prod, arg, Q)]
                continue
            for r in range(lv + 1):
                out[(i * K + arg) * (L + 1) + r] = prod[r] * (term_factor if arg < nt else 1) % Q[r]
    return out


def test_recorded_reference_order_replays_to_the_folded_scalars(toys, bgv_toy):
    """The op's `sequence` (the reference's Add / MulThenAdd / Mul order that the composed benchmark arm replays through the existing
    entry points) implies exactly the scalars the kernel applies, and every weight with a plaintext appears in it once."""
    toy = toys[1]
    for name, case in VC.ckks_cases().items():
        if case[3] != 1:
            continue
        prog, _ = VC.ckks_plan(toy, case)
        o = [o for o in prog.ops if o["kind"] == PE.PTLINCOMB][0]
        assert _replayed_scalars(o, toy.q, 1) == o["scalars"], name
        K = len(o["terms"]) + 1
        for i, seq in enumerate(o["sequence"]):
            used = sorted(a for kind, a in seq if kind == "pt")
            assert used == [k for k in range(K) if o["index"][i * K + k] >= 0], name
    bt = bgv_toy
    for name, (polys, kind) in VC.bgv_cases(bt.t).items():
        prog, _ = VC.bgv_plan(bt, polys, kind, False, len(bt.q) - 1, 12345, 777)
        o = [o for o in prog.ops if o["kind"] == PE.PTLINCOMB][0]
        assert _replayed_scalars(o, bt.q, bt.t) == o["scalars"], name


def test_nil_mapping_over_several_values_takes_every_values_flags(toys):
    """A nil Mapping reads Value[0]'s coefficients, but under the OR of every Value's flags for the powers and the AND for the baby
    steps: with Value[0] general and Value[1] odd, the baby steps read only the odd coefficients of Value[0], so the program is not the
    scalar program of Value[0]; with equal flags it is."""
    toy = toys[1]
    L = toy.params.MaxLevelQ()
    rng = np.random.default_rng(3)
    c0 = [float(rng.uniform(-1, 1)) for _ in range(8)]
    c1 = [0.0 if k % 2 == 0 else float(rng.uniform(-1, 1)) for k in range(8)]
    a = PE.plan(toy.q, L, toy.scale, c0, PE.MONOMIAL, toy.scale, 1, toy.prec)
    pv = PE.NewPolynomialVector([PE.Polynomial(c0), PE.Polynomial(c1, PE.MONOMIAL, True, False)], None)
    b = PE.plan_vector(toy.q, L, toy.scale, pv, toy.scale, 1, toy.prec, toy.logN)
    assert not b.plaintexts and PE.PTLINCOMB not in b.kinds()
    assert b.ops != a.ops
    lin, lin_a = [o for o in b.ops if o["kind"] == PE.LINCOMB][-1], [o for o in a.ops if o["kind"] == PE.LINCOMB][-1]
    assert len(lin["terms"]) < len(lin_a["terms"])          # only the odd powers are read
    same = PE.NewPolynomialVector([PE.Polynomial(c0), PE.Polynomial(c0)], None)
    assert PE.plan_vector(toy.q, L, toy.scale, same, toy.scale, 1, toy.prec, toy.logN).ops == a.ops


def test_plan_vector_needs_the_ring_degree(toys):
    toy = toys[1]
    pv = PE.NewPolynomialVector([PE.Polynomial([0.1, 0.2]), PE.Polynomial([0.2, 0.1])], VC.even_odd(toy.N // 2))
    with pytest.raises(ValueError, match="log_n must be the ring's LogN"):
        PE.plan_vector(toy.q, toy.params.MaxLevelQ(), toy.scale, pv, toy.scale)
    with pytest.raises(ValueError, match="max_slots must be"):
        BPE.plan_vector(toy.q, 0xffc001, 3, 1, PE.NewPolynomialVector([PE.Polynomial([1, 2]), PE.Polynomial([2, 1])], {0: [0]}), 1)

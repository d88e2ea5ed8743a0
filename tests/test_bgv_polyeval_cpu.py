"""The BGV / BFV polynomial-evaluation planner (lattigo_b200/bgv_polyeval.py) against the literal oracle, on the CPU: an exact
interpreter of the folded program equals the oracle word for word, with the same output level and scale; op counts; coefficient and
scale edges; and every argument check of lgpu_bgv_polynomial_evaluate on a host-only handle, before any launch."""
import ctypes

import numpy as np
import pytest

from lattigo_b200 import bgv_polyeval as BPE
from lattigo_b200 import polyeval as PE
from oracle import oracle as O
from tests import bgv_polyeval_cases as C


@pytest.fixture(scope="module")
def toy():
    q, p = O.gen_moduli(11, [55] + [45] * 9, [60, 60])
    return C.Toy(10, q, p, 0xffc001, seed=9)


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def _check(toy, invariant, ct, level, coeffs, scale=1, target=1, odd=True, even=True):
    r, _ = C.oracle_eval(toy, invariant, [v[: level + 1] for v in ct], scale, coeffs, target, odd, even)
    prog = BPE.plan(toy.q, toy.t, level, scale, coeffs, target, invariant, odd, even)
    got = C.interpret(toy, invariant, prog, [v[: level + 1] for v in ct])
    assert _same(got, r.Value)
    assert (prog.out_level, prog.out_scale) == (r.Level(), int(r.Scale))
    return prog


@pytest.mark.parametrize("invariant", [False, True])
def test_folded_program_equals_the_literal_oracle(toy, invariant):
    L = len(toy.q) - 1
    ct = toy.encrypt(toy.random_values(), L)
    for name, (coeffs, odd, even) in C.cases(toy.t).items():
        _check(toy, invariant, ct, L, coeffs, odd=odd, even=even)
        # the lowest level the reference accepts
        low = min(lv for lv in range(L + 1) if _plans(toy, lv, coeffs, invariant, odd, even))
        _check(toy, invariant, ct, low, coeffs, odd=odd, even=even)


def _plans(toy, level, coeffs, invariant, odd, even):
    try:
        BPE.plan(toy.q, toy.t, level, 1, coeffs, 1, invariant, odd, even)
        return True
    except ValueError:
        return False


@pytest.mark.parametrize("invariant", [False, True])
def test_coefficient_edges(toy, invariant):
    t = toy.t
    L = len(toy.q) - 1
    ct = toy.encrypt(toy.random_values(), L)
    edges = [0, t - 1, t, t // 2, t // 2 + 1, (1 << 64) - 1, 1, 2]
    _check(toy, invariant, ct, L, edges)
    _check(toy, invariant, ct, L, edges[::-1])


@pytest.mark.parametrize("invariant", [False, True])
def test_input_scale_differs_from_target(toy, invariant):
    """Scales other than 1 reach the MulThenAdd ratio and the tInvModQ constant; EvaluateMonomial's InDelta check then only lets equal
    scales reach the Add, so no TENSOR carries matchScalesBinary weights (r_b = r_a = 1 throughout)."""
    L = len(toy.q) - 1
    ct = toy.encrypt(toy.random_values(), L)
    coeffs = C.cases(toy.t)["d15"][0]
    for scale, target in ((1, 3), (5, 1), (12345, 777), (toy.t - 1, 2)):
        prog = _check(toy, invariant, ct, L, coeffs, scale, target)
        assert prog.out_scale == target
        for o in prog.ops:
            if o["kind"] == PE.TENSOR:
                assert set(o["weights"]) == {1}


def test_op_counts(toy):
    L = len(toy.q) - 1
    for name, (coeffs, odd, even) in C.cases(toy.t).items():
        for invariant in (False, True):
            prog = BPE.plan(toy.q, toy.t, L, 1, coeffs, 1, invariant, odd, even)
            kinds = prog.kinds()
            assert kinds.count(PE.LINCOMB) == 1, name                 # every baby step in one LINCOMB
            if invariant:
                assert PE.RESCALE not in kinds, name


def test_degree_255_fits_the_term_bound():
    q = O.gen_moduli(11, [55] + [45] * 12, [60])[0]
    for invariant in (False, True):
        prog = BPE.plan(q, 0x10001, len(q) - 1, 1, list(range(1, 257)), 1, invariant)
        lin = [o for o in prog.ops if o["kind"] == PE.LINCOMB]
        assert len(lin) == 1 and len(lin[0]["terms"]) <= PE.MAX_TERMS


def test_planner_rejects_what_the_reference_rejects(toy):
    q, t = toy.q, toy.t
    for invariant in (False, True):
        with pytest.raises(ValueError, match="degree"):
            BPE.plan(q, t, 5, 1, [3], 1, invariant)
        with pytest.raises(ValueError, match="cannot evaluate poly"):
            BPE.plan(q, t, 2, 1, [1] * 16, 1, invariant)              # 2 levels < Depth(15) = 4, BFV too
        with pytest.raises(ValueError, match="Chebyshev"):
            BPE.plan(q, t, 5, 1, [1, 2, 3], 1, invariant, basis=PE.CHEBYSHEV)
        with pytest.raises(ValueError, match="degree-0 baby step"):
            BPE.plan(q, t, 9, 1, [1, 0, 2, 0, 3, 0, 4, 0, 5, 0, 6, 0, 7, 0, 8, 0, 9], 1, invariant, odd=False, even=True)
        with pytest.raises(ValueError, match="uint64"):
            BPE.plan(q, t, 5, 1, [1, 1 << 64], 1, invariant)
        with pytest.raises(ValueError, match=r"\[1, t\)"):
            BPE.plan(q, t, 5, t, [1, 2], 1, invariant)
    with pytest.raises(ValueError, match="cannot rescale"):
        BPE.plan(q, t, 1, 1, [0, 0, 1], 1, False)                     # passes the Depth check, no level for the last Rescale
    assert BPE.plan(q, t, 1, 1, [0, 0, 1], 1, True).out_level == 1


# ---- C ABI on a host-only handle -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host(toy):
    import lattigo_b200 as lb
    ctx = lb.Context(toy.logN, toy.q, toy.p, device=-1)
    a = np.array(toy.qmul, dtype=np.uint64)
    h = ctypes.c_void_p()
    lb._lib.check(lb.lib().lgpu_bgv_create(ctx.h, toy.t, a.ctypes.data, len(toy.qmul), ctypes.byref(h)))
    yield ctx, h
    lb.lib().lgpu_bgv_destroy(h)
    ctx.close()


def _err(h, level, cp, si, rlk=True, batch=1, null_ev=False):
    import lattigo_b200 as lb
    buf = (ctypes.c_uint64 * 4)()
    addr = ctypes.c_void_p((ctypes.addressof(buf) + 15) & ~15)
    data = (ctypes.c_uint64 * 4)()
    g = lb._lib.GadgetCtStruct(ctypes.c_void_p((ctypes.addressof(data) + 15) & ~15), rlk if rlk not in (True, False) else 9, 1, 0, 5, 1, None)
    rc = lb._lib.lib().lgpu_bgv_polynomial_evaluate(None if null_ev else h, level, addr, batch, ctypes.byref(cp) if cp is not None else None,
                                                    ctypes.byref(g) if rlk is not False else None, si, addr, None)
    return None if rc == 0 else lb._lib.lib().lgpu_last_error().decode()


def _prog(toy, si, fn=None):
    prog = BPE.plan(toy.q, toy.t, 9, 1, C.cases(toy.t)["d15"][0], 1, si)
    if fn:
        fn(prog)
    return prog


def test_well_formed_programs_reach_the_device_check(toy, host):
    _, h = host
    for si in (0, 1):
        assert "host-only" in _err(h, 9, _prog(toy, si).to_c(1), si)


def test_malformed_programs_are_rejected_before_any_launch(toy, host):
    _, h = host
    lin = lambda p: [o for o in p.ops if o["kind"] == PE.LINCOMB][-1]
    bad = {
        "slot count": lambda p: setattr(p, "n_slots", 1),
        "reads a slot before": lambda p: p.ops[0].update(src0=p.n_slots - 1),
        "minimum level": lambda p: p.ops[0].update(level=p.ops[0]["level"] - 1),
        "below its modulus": lambda p: lin(p)["weights"].__setitem__(0, toy.q[0]),
        "term count": lambda p: lin(p).update(terms=list(range(PE.MAX_TERMS + 1))),
        "output slot": lambda p: setattr(p, "out_slot", 0),
    }
    for si in (0, 1):
        for msg, fn in bad.items():
            e = _err(h, 9, _prog(toy, si, fn).to_c(1), si)
            assert e is not None and msg in e, (si, msg, e)
    # RESCALE in a scale-invariant program (a BGV program run as BFV)
    assert "does not rescale" in _err(h, 9, _prog(toy, 0).to_c(1), 1)
    # levels_per_rescale != 1 (a program without RESCALE, so that the generic RESCALE level check does not fire first)
    for si in (0, 1):
        assert "levels_per_rescale must be 1" in _err(h, 9, _prog(toy, 1).to_c(2), si)
    # scale-invariant tensor operands below the op's level
    def lower(p):
        lo = lin(p)
        lo["out_levels"] = [8] + lo["out_levels"][1:]
    e = _err(h, 9, _prog(toy, 1, lower).to_c(1), 1)
    assert e is not None and ("level" in e), e


def test_argument_checks(toy, host):
    _, h = host
    cp = _prog(toy, 0).to_c(1)
    assert "null BGV evaluator" in _err(h, 9, cp, 0, null_ev=True)
    assert "scale_invariant must be 0 or 1" in _err(h, 9, cp, 2)
    assert "level out of range" in _err(h, 10, cp, 0)
    assert "batch out of range" in _err(h, 9, cp, 0, batch=0)
    assert "empty polynomial program" in _err(h, 9, None, 0)
    assert "relinearization key" in _err(h, 9, cp, 0, rlk=False)
    assert "levelQ out of range for this evaluation key" in _err(h, 9, cp, 0, rlk=3)

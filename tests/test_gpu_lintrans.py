"""GPU parity of the device linear-transformation driver (lgpu_lintrans_evaluate_many, lattigo_b200/csrc/lintrans.cu)
against oracle/lintrans.py = circuits/common/lintrans/lintrans_evaluator.go:28-470, bit for bit: naive (single hoisting)
and BSGS (double hoisting) evaluators, several matrices sharing one decomposition and one set of pre-rotations, matrices
below the ciphertext level, in-place output, batch of ciphertexts, missing-key error. Operands are uniform residues (the
arithmetic does not care whether keys / diagonals are meaningful: parity is over Z_q identities)."""
import numpy as np
import pytest

from oracle import lintrans as LT
from oracle import oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64


EDGE_POS = (0, 1, 2, 3, 5)       # coefficients set to 0, q - 1, q - 1, q - 1, 0 on every row by `edges=True`


def _rand(moduli, N, rng, edges):
    """Uniform residues; with `edges`, 0 and q - 1 at EDGE_POS of every row (the largest lazy sums of the MACs)."""
    x = H.rand_poly(moduli, N, rng)
    if edges:
        top = np.array([int(m) - 1 for m in moduli], dtype=U64)
        x[:, EDGE_POS[0]] = 0; x[:, EDGE_POS[4]] = 0
        for c in EDGE_POS[1:4]:
            x[:, c] = top
    return x


def _setup(logN, lq, lp, mats, seed, batch=2, primes=None, ring_type=0, log_slots=None, levelP=None, edges=False, ct_level=None):
    """mats: list of (rotations, N1, levelQ). Returns everything both sides need.
    ring_type: 0 standard, 1 conjugate invariant (primes = 1 mod 4N, NthRoot 4N). log_slots: the matrices' LogSlots
    (default logN - 1 on the standard ring, logN on the conjugate-invariant one). levelP: the matrices' LevelP, at which the
    Galois keys are made too (default the context's last P prime). primes: explicit (Q, P) lists. edges: 0 and q - 1 words at
    EDGE_POS of the ciphertext, the diagonals and the keys. ct_level: level of the input ciphertexts (default the top)."""
    import lattigo_b200 as lb
    if primes is None:
        q, p = O.gen_moduli(logN + 1 + ring_type, lq, lp)
    else:
        q, p = primes
    params = O.Parameters(logN, q, p, "ConjugateInvariant" if ring_type else "Standard")
    N = params.N()
    rng = np.random.default_rng(seed)
    ctx = lb.Context(logN, q, p, ring_type=ring_type)
    level = len(q) - 1
    levelP = len(p) - 1 if levelP is None else levelP
    ct_level = level if ct_level is None else ct_level
    if log_slots is None:
        log_slots = logN if ring_type else logN - 1
    slots = 1 << log_slots
    need = set()
    for rots, N1, _ in mats:
        if N1:
            _, rotN1, rotN2 = LT.bsgs_index(rots, slots, N1)
            need |= {r for r in rotN1 if r} | {r for r in rotN2 if r}
        else:
            need |= {r & (slots - 1) for r in rots if r & (slots - 1)}
    keys_o, keys_d = {}, {}
    for r in sorted(need):
        g = params.GaloisElement(r)
        gk = H.random_gadget_ciphertext(params, level, levelP, rng)
        if edges:
            for d in range(gk.data.shape[0]):
                for c in range(2):
                    gk.data[d, 0, c] = _rand(q + p[: levelP + 1], N, rng, True)
        keys_o[g] = gk
        keys_d[g] = lb.GadgetCiphertext(ctx, gk.data, level, levelP)
    lts_o, lts_d = [], []
    for rots, N1, lvl in mats:
        vo, vd = {}, {}
        for r in rots:
            dq = _rand(q[: lvl + 1], N, rng, edges); dp = _rand(p[: levelP + 1], N, rng, edges)
            vo[r] = (dq, dp)
            vd[r] = ctx.to_device(np.concatenate([dq, dp]))
        lts_o.append(LT.LinearTransformation(vo, lvl, levelP, log_slots, N1))
        lts_d.append(lb.lintrans.LinearTransformation(vd, lvl, levelP, log_slots, N1))
    qc = q[: ct_level + 1]
    ct = np.stack([np.stack([_rand(qc, N, rng, edges), _rand(qc, N, rng, edges)]) for _ in range(batch)])
    return lb, ctx, params, keys_o, keys_d, lts_o, lts_d, ct


def _oracle_many(params, keys_o, lts_o, ct, out_levels):
    ev = LT.Evaluator(params, keys_o)
    N = params.N()
    res = []
    for b in range(ct.shape[0]):
        outs = [[np.zeros((lv + 1, N), dtype=U64) for _ in range(2)] for lv in out_levels]
        ev.EvaluateMany([ct[b, 0], ct[b, 1]], lts_o, outs)
        res.append(outs)
    return res


def _check(ctx, got, want, levels):
    for i, lv in enumerate(levels):
        g = ctx.to_host(got[i])
        for b in range(g.shape[0]):
            for k in range(2):
                assert np.array_equal(g[b, k, : lv + 1], want[b][i][k][: lv + 1]), (i, b, k)


@pytest.mark.parametrize("primes", ["ckks", "q61"])
def test_lintrans_naive_and_bsgs_small(primes):
    logN = 8
    pr = (H.Qi60[:5], H.Pi60[:2]) if primes == "q61" else None
    mats = [([0, 1, 2, 5, 6, 9], 0, 4), ([0, 1, 2, 3, 4, 5, 8, 9, 12, 17, 33, 127], 4, 4), ([3, 4, 7, 64], 2, 4)]
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(logN, [55, 45, 45, 45, 45], [55, 55], mats, 11, batch=3, primes=pr)
    try:
        N = params.N()
        ev = lb.lintrans.Evaluator(ctx, kd)
        assert ev.GaloisElement(5) == params.GaloisElement(5) and ev.GaloisElement(-3) == params.GaloisElement(-3)
        d_ct = ctx.to_device(ct)
        import torch
        outs = [torch.zeros((3, 2, 5, N), dtype=torch.int64, device=d_ct.device) for _ in mats]
        levels = ev.EvaluateMany(d_ct, ld, outs)
        assert levels == [4, 4, 4]
        want = _oracle_many(params, ko, lo, ct, [4, 4, 4])
        _check(ctx, outs, want, levels)
        # each matrix on its own gives the same result (the shared pre-rotation cache does not leak between matrices)
        for i in range(len(mats)):
            o1 = torch.zeros((3, 2, 5, N), dtype=torch.int64, device=d_ct.device)
            ev.Evaluate(d_ct, ld[i], o1)
            assert torch.equal(o1, outs[i])
    finally:
        ctx.close()


def test_lintrans_lower_matrix_level_and_inplace():
    """One matrix at the ciphertext level and one two levels below (the decomposition is taken at the highest, the
    reference reads its first rows: lintrans_evaluator.go:40-58), receiver with a higher level than the result, and
    in-place evaluation as EvaluateSequential uses it (:117-139)."""
    logN = 8
    mats = [([1, 2, 3, 6, 7], 2, 4), ([0, 1, 4, 5], 4, 2), ([0, 3, 9], 0, 2)]
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(logN, [55, 45, 45, 45, 45], [55, 55], mats, 5, batch=2)
    try:
        import torch
        N = params.N()
        ev = lb.lintrans.Evaluator(ctx, kd)
        d_ct = ctx.to_device(ct)
        outs = [torch.zeros((2, 2, 5, N), dtype=torch.int64, device=d_ct.device) for _ in mats]
        levels = ev.EvaluateMany(d_ct, ld, outs)
        assert levels == [4, 2, 2]
        want = _oracle_many(params, ko, lo, ct, [4, 4, 4])
        _check(ctx, outs, want, levels)
        for o in outs[1:]:
            assert int(o[:, :, 3:].abs().max()) == 0            # rows above the result level are left untouched
        inpl = d_ct.clone()
        ev.Evaluate(inpl, ld[0], inpl)
        assert torch.equal(inpl, outs[0])
    finally:
        ctx.close()


def test_lintrans_missing_key_and_bad_arguments():
    logN = 8
    mats = [([1, 2], 0, 2)]
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(logN, [55, 45, 45], [55, 55], mats, 3, batch=1)
    try:
        import torch
        del kd[params.GaloisElement(2)]
        ev = lb.lintrans.Evaluator(ctx, kd)
        d_ct = ctx.to_device(ct)
        out = torch.zeros_like(d_ct)
        with pytest.raises(lb.LgpuError, match="GaloisKey"):
            ev.Evaluate(d_ct, ld[0], out)
    finally:
        ctx.close()


@pytest.mark.parametrize("logN,nq,np_", [(13, 6, 2), (16, 12, 3)])
def test_lintrans_bsgs_large(logN, nq, np_):
    """N = 2^13 and N = 2^16 (fused key-switch pipeline inside the giant steps), BSGS with 3 giant x 4 baby steps."""
    mats = [([0, 1, 2, 3, 4, 5, 6, 8, 9, 11], 4, nq - 1)]
    lb, ctx, params, ko, kd, lo, ld, ct = _setup(logN, [56] + [45] * (nq - 1), [55] * np_, mats, 21, batch=2)
    try:
        import torch
        N = params.N()
        ev = lb.lintrans.Evaluator(ctx, kd)
        d_ct = ctx.to_device(ct)
        out = torch.zeros_like(d_ct)
        levels = ev.EvaluateMany(d_ct, ld, [out])
        want = _oracle_many(params, ko, lo, ct[:1], [nq - 1])
        _check(ctx, [out[:1]], want, levels)
        # second ciphertext of the batch: same matrix, independent result -- check it through linearity-free identity:
        # evaluating it alone gives the same words
        o2 = torch.zeros_like(d_ct[1:])
        ev.Evaluate(d_ct[1:].contiguous(), ld[0], o2)
        assert torch.equal(o2, out[1:])
    finally:
        ctx.close()

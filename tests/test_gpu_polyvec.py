"""lgpu_ckks_polynomial_vector_evaluate and lgpu_bgv_polynomial_vector_evaluate (Evaluate with a PolynomialVector and a Mapping) against
the literal op-by-op oracle (tests/polyvec_oracle.py), bit for bit, with the output level and scale. The slot vectors are encoded on the
device (lgpu_ckks_encode / lgpu_bgv_encode). Cases:
- every CKKS vector case at N = 2^12, batch 1 and 3; CKKS_N15QP881 batch 4 with two Chebyshev degree-30 polynomials; BOOT_N16QP1767 at
  its EvalMod levels; BGV and BFV at N = 2^12 and BGV_N15QP880 level 19, batch 16;
- a batch larger than batch_chunk();
- PTLINCOMB at the maximum term and output counts on 61-bit primes, with words near q - 1 that differ per plaintext, coefficient, batch
  entry and component, a scalar per (output, term, limb) and missing weights; every output read back against Python integers, at batch
  sizes that reach every tile size;
- one run end to end: encryption on the host, evaluation on the device, decryption and decoding."""
from fractions import Fraction

import numpy as np
import pytest

from lattigo_b200 import polyeval as PE
from lattigo_b200.params import PRESETS
from oracle import oracle as O
from oracle import polyeval as OP
from tests import bgv_oracle as B
from tests import helpers as H
from tests import polyeval_cases as PC
from tests import polyvec_cases as VC
from tests import polyvec_oracle as V

pytestmark = pytest.mark.gpu
U64 = np.uint64


def _ckks_run(logN, q, p, level, batch, cases, scale, lpr=1, prec=53, seed=0, idx=None):
    import lattigo_b200 as lb
    rng = np.random.default_rng(seed)
    params = O.Parameters(logN, q, p)
    rlk = H.random_gadget_ciphertext(params, len(q) - 1, len(p) - 1, rng)
    ctx = lb.Context(logN, q, p, device=0)
    grlk = lb.GadgetCiphertext(ctx, rlk.data, len(q) - 1, len(p) - 1)
    N = 1 << logN
    cts = np.stack([np.stack([H.rand_poly(q[: level + 1], N, rng) for _ in range(2)]) for _ in range(batch)])
    dev = ctx.to_device(cts)
    ev = PE.PolynomialEvaluator(ctx, grlk, lpr, prec)
    oev = V.CKKSPolyVectorEvaluator(params, rlk, lpr, prec)
    for basis, polys, kind, tmul in cases:
        mp = VC.mapping(kind, N // 2, len(polys))
        target = scale * tmul
        out, lv, sc = ev.EvaluateVector(dev, scale, VC.pvec(basis, polys, mp), target)
        got = ctx.to_host(out)
        for b in (range(batch) if idx is None else idx):
            want = oev.EvaluateVector(OP.Ct([cts[b, 0], cts[b, 1]], scale), VC.oracle_polys(basis, polys), mp, target)
            assert lv == want.Level() and sc == want.Scale
            assert np.array_equal(got[b, 0], want.Value[0]) and np.array_equal(got[b, 1], want.Value[1]), "batch entry %d differs" % b
    ctx.close()


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("lpr", [1, 2])
def test_every_ckks_vector_case_at_n4096(batch, lpr):
    logscale = 25 * lpr                                        # lpr = 2: pairs of 25-bit primes, a 50-bit scale (precision 53)
    q, p = O.gen_moduli(13, [55] + [logscale // lpr] * (8 * lpr), [55, 55])
    cases = [(b, ps, k, t) for (b, ps, k, l, t) in VC.ckks_cases().values() if l == lpr]
    _ckks_run(12, q, p, len(q) - 1, batch, cases, Fraction(2) ** logscale, lpr, 53)


def _two_cheb30(seed, even_only=False):
    rng = np.random.default_rng(seed)
    polys = []
    for _ in range(2):
        c = [0.0 if (even_only and k & 1) else float(rng.uniform(-1, 1)) / (k + 1) for k in range(31)]
        polys.append((c, not even_only, True))
    return polys


def test_n15qp881_batch4_two_chebyshev30():
    pr = PRESETS["CKKS_N15QP881"]
    _ckks_run(pr["logN"], pr["Q"], pr["P"], len(pr["Q"]) - 1, 4, [(PE.CHEBYSHEV, _two_cheb30(21), "eo", 1)], Fraction(2) ** 40, idx=[0, 3])


def test_boot_n16qp1767_evalmod_levels():
    pr = PRESETS["BOOT_N16QP1767"]
    _ckks_run(pr["logN"], pr["Q"], pr["P"], 25, 2, [(PE.CHEBYSHEV, _two_cheb30(22, even_only=True), "eo", 1)], Fraction(2) ** 60, idx=[1])


def test_batch_larger_than_batch_chunk():
    """LGPU_BATCH_CHUNK is read once per process; the default 64 is crossed by a batch of 66."""
    q, p = O.gen_moduli(11, [55] + [40] * 6, [55, 55])
    case = VC.ckks_cases()["mono7_half"]
    _ckks_run(10, q, p, len(q) - 1, 66, [(case[0], case[1], case[2], case[4])], Fraction(2) ** 40, idx=[0, 63, 64, 65])


class _BGV:
    def __init__(self, logN, q, p, t, seed):
        import lattigo_b200 as lb
        self.N, self.q, self.p, self.t = 1 << logN, list(q), list(p), int(t)
        self.params = O.Parameters(logN, self.q, self.p)
        self.qmul = B.qmul_moduli(logN, self.q)
        self.rng = np.random.default_rng(seed)
        self.rlk_o = H.random_gadget_ciphertext(self.params, len(q) - 1, len(p) - 1, self.rng)
        self.ctx = lb.Context(logN, self.q, self.p)
        self.rlk = lb.GadgetCiphertext(self.ctx, self.rlk_o.data, len(q) - 1, len(p) - 1)
        self.enc = lb.BGVEncoder(self.ctx, self.t)
        self.pev = {si: lb.BGVPolynomialEvaluator(lb.BGVEvaluator(self.ctx, self.t, self.qmul, self.rlk, scale_invariant=si))
                    for si in (False, True)}

    def check(self, si, level, batch, polys, kind, scale=1, target=1, idx=None):
        cts = np.stack([np.stack([H.rand_poly(self.q[: level + 1], self.N, self.rng) for _ in range(2)]) for _ in range(batch)])
        mp = VC.mapping(kind, self.enc.MaxSlots(), len(polys))
        pv = PE.NewPolynomialVector([PE.Polynomial(c, PE.MONOMIAL, o, e) for c, o, e in polys], mp)
        out, lv, sc = self.pev[si].EvaluateVector(self.ctx.to_device(cts), scale, pv, target, self.enc)
        out = self.ctx.to_host(out)
        pe = V.BGVPolyVectorEvaluator(self.params, self.rlk_o, self.t, self.qmul, si)
        for k in (range(batch) if idx is None else idx):
            r = pe.EvaluateVector(OP.Ct([cts[k, 0], cts[k, 1]], scale), VC.bgv_oracle_polys(polys), mp, target)
            assert (lv, sc) == (r.Level(), int(r.Scale))
            assert np.array_equal(out[k], np.stack(r.Value)), k

    def close(self):
        self.enc.close()
        self.ctx.close()


@pytest.mark.parametrize("si", [False, True])
def test_bgv_vector_cases_at_n4096(si):
    q, p = O.gen_moduli(13, [55] + [45] * 9, [60, 60])
    d = _BGV(12, q, p, 0xffc001, 3)
    try:
        for name, (polys, kind) in VC.bgv_cases(d.t).items():
            for batch in (1, 3):
                d.check(si, len(q) - 1, batch, polys, kind, 12345, 777, idx=[0, batch - 1])
    finally:
        d.close()


@pytest.mark.parametrize("si", [False, True])
def test_bgv_n15qp880_level19_batch16(si):
    pr = PRESETS["BGV_N15QP880"]
    d = _BGV(pr["logN"], pr["Q"], pr["P"], 0x10001, 4)
    try:
        polys, kind = VC.bgv_cases(d.t)["d15"]
        d.check(si, 19, 16, polys, kind, idx=[0, 15])
    finally:
        d.close()


@pytest.mark.parametrize("batch", [1, 2, 3, 5, 9])
def test_ptlincomb_at_the_maximum_counts_near_q_minus_1(batch):
    """16 terms and 64 outputs at three levels, on 61-bit primes: words within 30 of q - 1 that differ per coefficient, per batch entry,
    per component and per plaintext; a distinct scalar per (output, term, limb); some weights missing. Every output is read back (each
    made the program's output in turn) and compared with Python integers. Batches 1, 2, 3, 5 and 9 reach every tile size, a tile
    rounded up past the batch, and a batch of two tiles."""
    import lattigo_b200 as lb
    import torch
    logN, q = 12, H.Qi60[:3]
    N = 1 << logN
    ctx = lb.Context(logN, q, H.Pi60[:1], device=0)
    L, K, n_out = 2, PE.MAX_TERMS, PE.MAX_OUTPUTS
    K1 = K + 1
    j = np.arange(N)
    x = np.stack([np.stack([np.stack([(qi - 1 - (j + 3 * b + 5 * c) % 13).astype(U64) for qi in q]) for c in range(2)]) for b in range(batch)])
    n_pt = n_out * K1
    pts = np.stack([np.stack([(qi - 1 - (7 * j + t) % 29).astype(U64) for qi in q]) for t in range(n_pt)])
    index = [-1 if (i + k) % 5 == 0 else i * K1 + k for i in range(n_out) for k in range(K1)]
    scalars = [qi - 1 - (17 * i + k + 1000 * r) % 4099 for i in range(n_out) for k in range(K1) for r, qi in enumerate(q)]
    out_levels = [L] + [L - (i % 3) for i in range(1, n_out)]
    pt = torch.from_numpy(pts.view(np.int64)).cuda()
    xd = ctx.to_device(x)
    ev = PE.PolynomialEvaluator(ctx, None)
    xo = x.astype(object)
    for i in range(n_out):
        prog = PE.Program()
        prog.n_slots = 1 + n_out
        prog.ops = [dict(kind=PE.PTLINCOMB, level=L, outs=list(range(1, n_out + 1)), out_levels=out_levels, terms=[0] * K, index=index,
                         scalars=scalars)]
        prog.out_slot, prog.out_level = 1 + i, out_levels[i]
        got = ctx.to_host(ev.RunVector(PE.PreparedVector(prog, pt, [L] * n_pt), xd))
        assert got.shape == (batch, 2, out_levels[i] + 1, N)
        for r in range(out_levels[i] + 1):
            qi = q[r]
            s = lambda k: scalars[(i * K1 + k) * (L + 1) + r]
            A = sum(s(k) * pts[index[i * K1 + k], r].astype(object) for k in range(K) if index[i * K1 + k] >= 0) % qi
            C = s(K) * pts[index[i * K1 + K], r].astype(object) % qi if index[i * K1 + K] >= 0 else 0
            for b in range(batch):
                assert np.array_equal(got[b, 0, r], ((A * xo[b, 0, r] + C) % qi).astype(U64)), (i, r, b)
                assert np.array_equal(got[b, 1, r], (A * xo[b, 1, r] % qi).astype(U64)), (i, r, b)
    ctx.close()


def test_end_to_end_encrypt_evaluate_decrypt():
    """Encrypt on the host, evaluate on the device (slot vectors encoded there), decrypt and decode on the host."""
    import lattigo_b200 as lb
    toy = PC.Toy(logN=12, nlevels=6, seed=4)
    x = np.random.default_rng(9).uniform(-1, 1, toy.N // 2)
    ct = toy.encrypt(x)
    ctx = lb.Context(toy.logN, toy.q, toy.p, device=0)
    rlk = lb.GadgetCiphertext(ctx, toy.rlk.data, len(toy.q) - 1, len(toy.p) - 1)
    ev = PE.PolynomialEvaluator(ctx, rlk, 1, toy.prec)
    c0 = [1 / (k + 1) for k in range(8)]
    c1 = [(-1) ** k / (k + 2) for k in range(8)]
    mp = VC.even_odd(toy.N // 2)
    pv = PE.NewPolynomialVector([PE.Polynomial(c0), PE.Polynomial(c1)], mp)
    out, lv, sc = ev.EvaluateVector(ctx.to_device(np.stack(ct)), toy.scale, pv, toy.scale)
    got = toy.decrypt(list(ctx.to_host(out)), sc)
    want = np.where(np.arange(toy.N // 2) % 2 == 0, np.polynomial.polynomial.polyval(x, c0), np.polynomial.polynomial.polyval(x, c1))
    assert np.max(np.abs(got - want)) < 2 ** -20
    ctx.close()

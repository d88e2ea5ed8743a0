"""lgpu_bgv_mulrelin_batch against the CPU restatement of schemes/bgv (tests/bgv_oracle.py), bit for bit: BGV MulRelin (+ Rescale) and
BFV MulRelinScaleInvariant on uniform ciphertexts with a uniform relinearization key.

- logN = 8: two-pass transforms and the unfused key-switch; every level where levelQMul changes, level 0 (BFV) / 1 (BGV + Rescale),
  squaring, ct_out == ct_a, batch 1 and 3, and batch consistency.
- BGV_N15QP880 at full size: batch 1, 2, 4 and 16. The BFV steps group polynomials into launches as follows (B = batch):
  per operand one INTT of its 2B Q polynomials, one ModUpQtoP and one NTT of its 2B QMul polynomials; then one INTT of the 3B
  Q products, one of the 3B QMul products, the quantize kernel and one NTT of the 3B Q products. Every transform splits its rows
  into FP64-pipe rows (primes with (10 + logN) q < 2^51) and integer rows; each part runs one persistent launch from 64
  limb-transforms on (the forward transform decides on all its rows) and two launches below. The difference between the BFV and
  the BGV launch counts at the same shape is asserted from these rules, so every batch states which side of the threshold the
  Q and QMul transforms are on.
- logN = 16 with 12 Q and 4 P limbs: fused key-switch and 61-bit persistent QMul rows at 2^16.
"""
import ctypes

import numpy as np
import pytest

from lattigo_b200 import params as presets
from oracle import oracle as O
from tests import bgv_oracle as B
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64
T = 0x10001


class Setup:
    def __init__(self, logN, q, p, seed):
        import lattigo_b200 as lb
        self.logN, self.N = logN, 1 << logN
        self.q, self.p = list(q), list(p)
        self.qmul = B.qmul_moduli(logN, q)
        self.params = O.Parameters(logN, q, p)
        self.rng = np.random.default_rng(seed)
        self.rlk_o = H.random_gadget_ciphertext(self.params, len(q) - 1, len(p) - 1, self.rng)
        self.ctx = lb.Context(logN, q, p)
        self.rlk = lb.GadgetCiphertext(self.ctx, self.rlk_o.data, len(q) - 1, len(p) - 1)
        self.ev = {si: lb.BGVEvaluator(self.ctx, T, self.qmul, self.rlk, scale_invariant=si) for si in (False, True)}
        self.oev = {si: B.BGVEvaluator(self.params, T, self.qmul, self.rlk_o, scale_invariant=si) for si in (False, True)}

    def cts(self, level, batch):
        return np.stack([np.stack([H.rand_poly(self.q[: level + 1], self.N, self.rng) for _ in range(2)]) for _ in range(batch)])

    def oracle(self, si, a, b, nb_rescales, square=False):
        ev = self.oev[si]
        x = [a[0].copy(), a[1].copy()]
        y = x if square else [b[0].copy(), b[1].copy()]
        out = ev.MulRelinNew(x, y)
        for _ in range(nb_rescales):
            out = ev.Rescale(out)
        return np.stack(out)

    def gpu(self, si, A, Bt, nb_rescales):
        ev = self.ev[si]
        return ev.MulRelinRescaleNew(A, Bt) if nb_rescales else ev.MulRelinNew(A, Bt)


@pytest.fixture(scope="module")
def small():
    q, p = O.gen_moduli(9, [55, 40, 40, 40, 50, 50, 58, 58], [60, 60])
    return Setup(8, q, p, 11)


def _levels(s, si, nb):
    lq = B.level_qmul(s.logN, s.q)
    lv = {l for l in range(1, len(lq)) if lq[l] != lq[l - 1]} | {len(lq) - 1}
    lv.add(1 if nb else 0)
    return sorted(lv)


@pytest.mark.parametrize("si,nb", [(False, 0), (False, 1), (True, 0)])
def test_small_every_level_vs_oracle(small, si, nb):
    s = small
    assert B.level_qmul(s.logN, s.q) == [1, 1, 2, 3, 3, 4, 5, 6]
    for level in _levels(s, si, nb):
        a, b = s.cts(level, 3), s.cts(level, 3)
        out = s.ctx.to_host(s.gpu(si, s.ctx.to_device(a), s.ctx.to_device(b), nb))
        assert out.shape == (3, 2, level + 1 - nb, s.N)
        for k in range(3):
            assert np.array_equal(out[k], s.oracle(si, a[k], b[k], nb)), (level, k)


@pytest.mark.parametrize("si,nb", [(False, 0), (False, 1), (True, 0)])
def test_small_squaring_in_place_and_batch_consistency(small, si, nb):
    s = small
    level = 5
    a = s.cts(level, 3)
    A = s.ctx.to_device(a)
    sq = s.ctx.to_host(s.gpu(si, A, A, nb))
    for k in range(3):
        ref = s.oracle(si, a[k], None, nb, square=True)
        assert np.array_equal(sq[k], ref), k
        # batch 1 call on element k alone
        one = s.ctx.to_host(s.gpu(si, A[k], A[k], nb))
        assert np.array_equal(one, ref), k
    if nb == 0:
        # ct_out == ct_a
        b = s.cts(level, 3)
        ref = [s.oracle(si, a[k], b[k], 0) for k in range(3)]
        X, Y = s.ctx.to_device(a), s.ctx.to_device(b)
        s.ev[si].MulRelin(X, Y, X)
        got = s.ctx.to_host(X)
        for k in range(3):
            assert np.array_equal(got[k], ref[k]), k


def _fp_ok(q, logN):
    return logN >= 10 and q * (10 + logN) < (1 << 51)


def _transform_launches(primes, polys, logN, forward):
    """Launches of one canonical transform of `polys` polynomials over `primes` (ntt.cu: launch_ntt / launch_intt)."""
    persist_ok = 13 <= logN <= 16
    two = 2 if logN > 12 else 1
    fp = [q for q in primes if _fp_ok(q, logN)]
    rest = [q for q in primes if not _fp_ok(q, logN)]
    n = 0
    if fp:
        rows = len(primes) if forward else len(fp)
        n += 1 if persist_ok and rows * polys >= 64 else two
    if rest:
        n += 1 if persist_ok and len(rest) * polys >= 64 else two
    return n


def _bfv_extra_launches(s, level, batch, square):
    """BFV launches minus BGV (no rescale) launches at the same level and batch (one sub-batch)."""
    lq = B.level_qmul(s.logN, s.q)[level]
    Q, M = s.q[: level + 1], s.qmul[: lq + 1]
    ops = 1 if square else 2
    per_operand = _transform_launches(Q, 2 * batch, s.logN, False) + 1 + _transform_launches(M, 2 * batch, s.logN, True)
    return (ops * per_operand + _transform_launches(Q, 3 * batch, s.logN, False) + _transform_launches(M, 3 * batch, s.logN, False)
            + 1 + _transform_launches(Q, 3 * batch, s.logN, True))


@pytest.fixture(scope="module")
def n15():
    sp = presets.PRESETS["BGV_N15QP880"]
    s = Setup(sp["logN"], sp["Q"], sp["P"], 5)
    assert s.qmul == sp["QMul"]
    return s


def _full_size(s, batches, level, cmp_all_upto, seed_cts):
    a, b = seed_cts
    refs = {}
    for si, nb in ((False, 1), (True, 0)):
        for batch in batches:
            A, Bt = s.ctx.to_device(a[:batch]), s.ctx.to_device(b[:batch])
            out = s.ctx.to_host(s.gpu(si, A, Bt, nb))
            idx = range(batch) if batch <= cmp_all_upto else (0, batch - 1)
            for k in idx:
                if (si, k) not in refs:
                    refs[(si, k)] = s.oracle(si, a[k], b[k], nb)
                assert np.array_equal(out[k], refs[(si, k)]), (si, batch, k)


def test_n15qp880_full_size_vs_oracle(n15):
    s = n15
    level = len(s.q) - 1
    cts = (s.cts(level, 16), s.cts(level, 16))
    _full_size(s, (1, 2, 4, 16), level, 4, cts)


@pytest.mark.parametrize("batch", [1, 2, 4, 16])
def test_n15qp880_launch_grouping(n15, batch):
    s = n15
    level = len(s.q) - 1
    A = s.ctx.to_device(s.cts(level, batch))
    Bt = s.ctx.to_device(s.cts(level, batch))
    for square in (False, True):
        Y = A if square else Bt
        s.gpu(False, A, Y, 0)   # warm-up (lazy allocations)
        bgv = H.launch_delta(lambda: s.gpu(False, A, Y, 0))
        bfv = H.launch_delta(lambda: s.gpu(True, A, Y, 0))
        assert bfv - bgv == _bfv_extra_launches(s, level, batch, square), (batch, square)


def test_pn16_bfv_12q_4p_vs_oracle():
    sp = presets.PRESETS["CKKS_PN16QP1761"]
    s = Setup(16, sp["Q"][:12], sp["P"], 9)
    level = 11
    a, b = s.cts(level, 8), s.cts(level, 8)
    for batch, idx in ((3, (0, 1, 2)), (8, (0, 7))):
        out = s.ctx.to_host(s.gpu(True, s.ctx.to_device(a[:batch]), s.ctx.to_device(b[:batch]), 0))
        for k in idx:
            assert np.array_equal(out[k], s.oracle(True, a[k], b[k], 0)), (batch, k)


def test_errors(small):
    import lattigo_b200 as lb
    import torch
    s = small
    L = lb.lib()
    level = 3
    A = s.ctx.to_device(s.cts(level, 2))
    out = torch.empty_like(A)
    h = s.ev[True].h
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + 8 * off)

    def call(ev_h, lvl, a, b, si, nb, o, batch=2):
        return L.lgpu_bgv_mulrelin_batch(ev_h, lvl, a, b, s.rlk.ref(), si, nb, o, batch, st)

    assert call(h, level, p(A), p(A), 1, 0, p(out)) == 0
    assert call(h, level, p(A), p(A), 1, 1, p(out)) != 0 and b"nb_rescales" in L.lgpu_last_error()
    assert call(h, len(s.q), p(A), p(A), 0, 0, p(out)) != 0 and b"level" in L.lgpu_last_error()
    assert call(h, -1, p(A), p(A), 0, 0, p(out)) != 0
    assert call(h, level, p(A, 1), p(A), 0, 0, p(out)) != 0 and b"aligned" in L.lgpu_last_error()
    assert call(h, level, p(A), p(A), 0, 0, p(out, 1)) != 0 and b"aligned" in L.lgpu_last_error()
    assert call(h, level, p(A), p(A), 0, 0, p(out), batch=0) != 0
    assert call(h, level, p(A), p(A), 0, 1, p(A)) != 0 and b"overlaps" in L.lgpu_last_error()   # in place with a rescale
    assert call(h, level, p(A), p(out), 0, 0, p(out)) != 0 and b"overlaps" in L.lgpu_last_error()
    assert call(h, level, p(A), p(A), 0, 0, p(A, 2 * 4 * s.N)) != 0 and b"overlaps" in L.lgpu_last_error()
    torch.cuda.synchronize()

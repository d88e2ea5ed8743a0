"""Algebraic anchoring of oracle/innersum.py (core/rlwe/inner_sum.go). The reference has no bit-level vectors for these methods,
so the restatement is pinned by decryption with real Galois keys (rlwe.GaloisKey convention: the key of g switches from
pi_g(s) back to s): PartialTracesSum(offset, n) must decrypt to sum_{i<n} pi_{GaloisElement(i * offset)}(m), and Trace(log_n) to
m with every coefficient off the multiples of gap zeroed, up to key-switch noise. The Galois elements the restatement asks for
are exactly the schedule's and are covered by the reference's GaloisElementsFor* sets."""
import numpy as np
import pytest

from oracle import innersum as OI
from oracle import oracle as O
from tests import helpers as H

U64 = np.uint64
NOISE_LOG2 = 14      # |decryption error| < 2^14 against messages of 2^20 (observed: at most ~2^9)


class _Setup:
    def __init__(self, logN, seed):
        self.params = O.Parameters(logN, H.RLWE_TEST_Q, H.RLWE_TEST_P)
        p = self.params
        N = p.N()
        self.rng = np.random.default_rng(seed)
        self.s = self.rng.integers(-1, 2, N)
        self.q = p.qi
        self.levelQ = p.MaxLevelQ()
        self.sn = np.empty((self.levelQ + 1, N), dtype=U64)
        p.ringQ.NTT(H.small_poly_rns(self.s, self.q), self.sn)
        self._keys = {}

    def key(self, g):
        if g not in self._keys:
            p = self.params
            N = p.N()
            ring1 = O.Ring(N, [self.q[0]])
            sp = H.small_poly_rns(self.s, [self.q[0]])
            row = np.empty_like(sp)
            ring1.Automorphism(sp, pow(g, -1, 2 * N), row)
            s_out = [int(v) if int(v) < self.q[0] // 2 else int(v) - self.q[0] for v in row[0]]
            self._keys[g] = H.gen_switching_key(p, self.s, s_out, self.rng)
        return self._keys[g]

    def keys_for(self, els):
        return {g: self.key(g) for g in set(els)}

    def encrypt(self, m, is_ntt=True):
        p = self.params
        N = p.N()
        a = H.rand_poly(self.q, N, self.rng)
        me = H.small_poly_rns(np.asarray(m) + np.rint(self.rng.normal(0, 3.2, N)).astype(np.int64), self.q)
        p.ringQ.NTT(me, me)
        c0 = np.stack([np.array([(int(x) - int(y) * int(t)) % int(mod) for x, y, t in zip(me[l], a[l], self.sn[l])], dtype=U64)
                       for l, mod in enumerate(self.q)])
        ct = [c0, a]
        if not is_ntt:
            for k in range(2):
                p.ringQ.INTT(ct[k], ct[k])
        return ct

    def decrypt(self, ct, level, is_ntt=True):
        p = self.params
        ringQ = p.ringQ.AtLevel(level)
        c = [ct[0][: level + 1].copy(), ct[1][: level + 1].copy()]
        if not is_ntt:
            for k in range(2):
                ringQ.NTT(c[k], c[k])
        acc = np.stack([np.array([(int(x) + int(y) * int(t)) % int(mod) for x, y, t in zip(c[0][l], c[1][l], self.sn[l])], dtype=U64)
                        for l, mod in enumerate(self.q[: level + 1])])
        back = np.empty_like(acc)
        ringQ.INTT(acc, back)
        Q = ringQ.ModulusAtLevel[level]
        return [v if v < Q // 2 else v - Q for v in ringQ.PolyToBigint(back)]


def _auto(params, poly, g):
    N = params.N()
    out = [0] * N
    for i in range(N):
        e = (i * g) % (2 * N)
        if e < N:
            out[e] += int(poly[i])
        else:
            out[e - N] -= int(poly[i])
    return out


def _schedule(params, offset, n):
    out = []
    i, j = 0, n
    while j > 1:
        if j & 1:
            out.append(params.GaloisElement((n - (n & ((2 << i) - 1))) * offset))
        out.append(params.GaloisElement((1 << i) * offset))
        i, j = i + 1, j >> 1
    return out


def _err_log2(got, want):
    return float(np.log2(float(max(abs(a - b) for a, b in zip(got, want)) + 1)))


@pytest.mark.parametrize("offset", [1, 3, -1, -4])
def test_partial_traces_sum_decrypts_to_the_sum_of_rotations(offset):
    S = _Setup(6, 100 + offset)
    p = S.params
    N = p.N()
    m = S.rng.integers(-(1 << 20), 1 << 20, N)
    for n in (1, 2, 3, 4, 5, 7, 8):
        for is_ntt in (True, False) if n in (2, 5) else (True,):     # n = 1 in the coefficient domain: see the next test
            ct = S.encrypt(m, is_ntt)
            ev = OI.Evaluator(p, S.keys_for(_schedule(p, offset, n)))
            out = [np.zeros((S.levelQ + 1, N), dtype=U64) for _ in range(2)]
            ev.PartialTracesSum(ct, offset, n, out, is_ntt)
            assert ev.asked == _schedule(p, offset, n)
            assert set(ev.asked) <= set(OI.GaloisElementsForInnerSum(p, offset, n))
            want = [0] * N
            for i in range(n):
                for k, v in enumerate(_auto(p, m, p.GaloisElement(i * offset))):
                    want[k] += v
            got = S.decrypt(out, S.levelQ, is_ntt)
            assert _err_log2(got, want) < NOISE_LOG2, (offset, n, is_ntt, _err_log2(got, want))
            for l, mod in enumerate(p.qi):
                assert int(out[0][l].max()) < mod and int(out[1][l].max()) < mod


def test_partial_traces_sum_n1_coefficient_domain_applies_the_trailing_intt():
    """inner_sum.go:179-183 then :286-289: with n = 1 and a coefficient-domain input, opOut is a copy of the input and the trailing
    INTT is applied to it anyway."""
    S = _Setup(6, 5)
    p = S.params
    ct = S.encrypt(S.rng.integers(-100, 100, p.N()), is_ntt=False)
    out = [np.zeros_like(ct[0]) for _ in range(2)]
    OI.Evaluator(p, {}).PartialTracesSum(ct, 1, 1, out, is_ntt=False)
    for k in range(2):
        want = np.empty_like(ct[k])
        p.ringQ.INTT(ct[k], want)
        assert np.array_equal(out[k], want)


def test_replicate_is_partial_traces_sum_with_negative_offset():
    S = _Setup(6, 9)
    p = S.params
    N = p.N()
    m = S.rng.integers(-(1 << 20), 1 << 20, N)
    ct = S.encrypt(m)
    ev = OI.Evaluator(p, S.keys_for(_schedule(p, -2, 3)))
    a = [np.zeros((S.levelQ + 1, N), dtype=U64) for _ in range(2)]
    b = [np.zeros((S.levelQ + 1, N), dtype=U64) for _ in range(2)]
    ev.Replicate(ct, 2, 3, a)
    ev.PartialTracesSum(ct, -2, 3, b)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert set(ev.asked) <= set(OI.GaloisElementsForReplicate(p, 2, 3))


@pytest.mark.parametrize("logN,log_ns", [(6, (0, 1, 4, 5)), (7, (0, 3)), (8, (0,))])
def test_trace_keeps_the_multiples_of_gap(logN, log_ns):
    S = _Setup(logN, 40 + logN)
    p = S.params
    N = p.N()
    m = S.rng.integers(-(1 << 20), 1 << 20, N)
    for log_n in log_ns:
        for is_ntt in (True, False):
            gap = (1 << (logN - log_n - 1)) * (2 if log_n == 0 else 1)
            ct = S.encrypt(m, is_ntt)
            ev = OI.Evaluator(p, S.keys_for(OI.GaloisElementsForTrace(p, log_n)))
            lvl_out = S.levelQ - 1
            out = [np.zeros((lvl_out + 1, N), dtype=U64) for _ in range(2)]
            level = ev.Trace(ct, log_n, out, is_ntt)
            assert level == lvl_out
            assert ev.asked == (OI.GaloisElementsForTrace(p, log_n) if gap > 1 else [])
            want = [int(v) if k % gap == 0 else 0 for k, v in enumerate(m)]
            got = S.decrypt(out, level, is_ntt)
            assert _err_log2(got, want) < NOISE_LOG2, (logN, log_n, is_ntt, _err_log2(got, want))

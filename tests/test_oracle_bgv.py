"""Anchors the BGV / BFV multiplication restatement (tests/bgv_oracle.py) by decryption with real keys: plaintexts are
encoded like bgv.Encoder.RingT2Q(scaleUp) (schemes/bgv/encoder.go:378-407), encrypted under a ternary secret, multiplied,
decrypted and decoded like RingQ2T(scaleDown) (:412-467). The result must be the negacyclic product m0 * m1 mod t times the
output scale the reference assigns: 1 for MulRelin, q_level^-1 after Rescale, (-Q_level mod t)^-1 for MulRelinScaleInvariant
(MulScaleInvariant, evaluator.go:983-989). Also pins the BGV_N15QP880 preset's T / QMul literals."""
import numpy as np
import pytest

from lattigo_b200 import params as presets
from oracle import oracle as O
from tests import bgv_oracle as B
from tests import helpers as H

U64 = np.uint64
LOGN = 11
T = 0x10001


def negacyclic(a, b, t):
    N = len(a)
    full = np.convolve(np.asarray(a, dtype=np.int64), np.asarray(b, dtype=np.int64))
    out = full[:N].copy()
    out[: N - 1] -= full[N:]
    return [int(x) % t for x in out]


class Scheme:
    """Keys, encryption and decryption at logN = 11 over a 4-limb chain whose levelQMul drops at every level."""

    def __init__(self):
        self.q, self.p = O.gen_moduli(LOGN + 1, [55, 45, 45, 45], [60])
        self.params = O.Parameters(LOGN, self.q, self.p)
        self.N = self.params.N()
        self.qmul = B.qmul_moduli(LOGN, self.q)
        rng = np.random.default_rng(7)
        self.rng = rng
        self.s = rng.integers(-1, 2, self.N)
        s2 = negacyclic(self.s, self.s, 1 << 62)
        s2 = [x - (1 << 62) if x >= 1 << 61 else x for x in s2]
        self.rlk = H.gen_switching_key(self.params, s2, self.s, rng)

    def ntt(self, rows, level):
        out = np.empty_like(rows)
        self.params.ringQ.AtLevel(level).NTT(rows, out)
        return out

    def encrypt(self, m, level):
        """Encoder.RingT2Q(level, scaleUp = true) + NTT, then (-a s + e + pt, a)."""
        mods = self.q[: level + 1]
        Ql = 1
        for q in mods:
            Ql *= q
        tinv = pow(T, -1, Ql)
        pt = np.stack([np.array([int(x) * (tinv % q) % q for x in m], dtype=U64) for q in mods])
        ring = self.params.ringQ.AtLevel(level)
        pt = self.ntt(pt, level)
        a = H.rand_poly(mods, self.N, self.rng)
        e = self.ntt(H.small_poly_rns(np.rint(self.rng.normal(0, 3.2, self.N)).astype(np.int64), mods), level)
        s = self.ntt(H.small_poly_rns(self.s, mods), level)
        c0 = np.empty_like(a)
        ring.MulCoeffsBarrett(a, s, c0)
        ring.Neg(c0, c0)
        ring.Add(c0, e, c0)
        ring.Add(c0, pt, c0)
        return [c0, a]

    def decrypt(self, ct):
        """c0 + c1 s, INTT, Encoder.RingQ2T(level, scaleDown = true): [t x]_Q centred, mod t."""
        level = ct[0].shape[0] - 1
        mods = self.q[: level + 1]
        ring = self.params.ringQ.AtLevel(level)
        s = self.ntt(H.small_poly_rns(self.s, mods), level)
        x = np.empty_like(ct[0])
        ring.MulCoeffsBarrett(ct[1], s, x)
        ring.Add(x, ct[0], x)
        ring.INTT(x, x)
        Ql = ring.ModulusAtLevel[level]
        out = []
        for v in ring.PolyToBigint(x):
            y = T * v % Ql
            if y >= Ql // 2:
                y -= Ql
            out.append(y % T)
        return out


@pytest.fixture(scope="module")
def sch():
    return Scheme()


def _msgs(sch, k):
    return [sch.rng.integers(0, T, sch.N) for _ in range(k)]


def test_qmul_and_level_qmul(sch):
    assert len(set(sch.qmul) & set(sch.q)) == 0
    assert B.level_qmul(LOGN, sch.q) == [1, 1, 2, 3]
    assert len(sch.qmul) == 4


@pytest.mark.parametrize("level", [3, 1])
def test_bgv_mulrelin_decrypts(sch, level):
    ev = B.BGVEvaluator(sch.params, T, sch.qmul, sch.rlk)
    m0, m1 = _msgs(sch, 2)
    out = ev.MulRelinNew(sch.encrypt(m0, level), sch.encrypt(m1, level))
    assert out[0].shape[0] == level + 1
    assert sch.decrypt(out) == negacyclic(m0, m1, T)


@pytest.mark.parametrize("level", [3, 1])
def test_bgv_mulrelin_rescale_decrypts(sch, level):
    ev = B.BGVEvaluator(sch.params, T, sch.qmul, sch.rlk)
    m0, m1 = _msgs(sch, 2)
    out = ev.Rescale(ev.MulRelinNew(sch.encrypt(m0, level), sch.encrypt(m1, level)))
    assert out[0].shape[0] == level
    scale = pow(sch.q[level], -1, T)
    assert sch.decrypt(out) == [x * scale % T for x in negacyclic(m0, m1, T)]


@pytest.mark.parametrize("level", [3, 2, 1])
def test_bfv_mulrelin_scale_invariant_decrypts(sch, level):
    ev = B.BGVEvaluator(sch.params, T, sch.qmul, sch.rlk, scale_invariant=True)
    assert ev.levelQMul[level] == [1, 1, 2, 3][level]
    m0, m1 = _msgs(sch, 2)
    out = ev.MulRelinNew(sch.encrypt(m0, level), sch.encrypt(m1, level))
    Ql = sch.params.ringQ.ModulusAtLevel[level]
    scale = pow((-Ql) % T, -1, T)
    assert sch.decrypt(out) == [x * scale % T for x in negacyclic(m0, m1, T)]
    # Rescale is a no-op for the scale-invariant evaluator
    r = ev.Rescale(out)
    assert all(np.array_equal(a, b) for a, b in zip(r, out))


@pytest.mark.parametrize("scale_invariant", [False, True])
def test_squaring_matches_two_operand_product(sch, scale_invariant):
    level = 2
    ev = B.BGVEvaluator(sch.params, T, sch.qmul, sch.rlk, scale_invariant=scale_invariant)
    (m0,) = _msgs(sch, 1)
    ct = sch.encrypt(m0, level)
    sq = ev.MulRelinNew(ct, ct)
    two = ev.MulRelinNew(ct, [ct[0].copy(), ct[1].copy()])
    assert all(np.array_equal(a, b) for a, b in zip(sq, two))
    Ql = sch.params.ringQ.ModulusAtLevel[level]
    scale = pow((-Ql) % T, -1, T) if scale_invariant else 1
    assert sch.decrypt(sq) == [x * scale % T for x in negacyclic(m0, m0, T)]


def test_bgv_preset_qmul_regenerates():
    s = presets.PRESETS["BGV_N15QP880"]
    assert s["T"] == T
    assert B.qmul_moduli(s["logN"], s["Q"]) == s["QMul"]
    assert B.level_qmul(s["logN"], s["Q"]) == [1, 1, 2, 2, 3, 3, 4, 4, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 11, 11]
    assert not set(s["QMul"]) & set(s["Q"])
    assert len(set(s["QMul"]) & set(presets.QI60)) == 6

"""lgpu_bgv_mulrelin_batch and one BFV polynomial against the CPU restatement of schemes/bgv (tests/bgv_oracle.py), bit for bit, at the
shapes where the BFV quantize and the operand ModUp change kernels (tests/test_bgv_shapes_cpu.py: predict, CASES) and with inputs at
the edges of quantize stage 1's float v.

- Every case of CASES: BFV, and BGV with one Rescale (none at level 0), batch 2, t = 65537. Chain A (64 x 30-bit FP64-pipe rows at
  2^10) at both sides of every bfv_quantize_kernel<NM> / modup_kernel<NSMAX> / > 48 KB shared-memory change, chain B (31 x 61-bit
  integer rows) at its top, chain A at 2^14 (persistent transforms on FP64 rows with NM = 32), and chain R at nq = 64.
- t in {2, Q[0] - 1} at the top of A and B (on A, Q[0] - 1 exceeds every other q_i).
- Edge inputs at the edge cases: a = (NTT(alpha), uniform), b = (NTT(beta), uniform) with beta = (edge words) alpha^-1 mod Q at random
  coefficients, so the Q-side product d0 = alpha beta carries the edge words into quantize stage 1; alpha = 3 keeps them out of the
  operand ModUp, alpha = 1 puts them there too. Plus all-zero and all-(q - 1) ciphertexts.
- BGV with 2 and `level` rescales, squaring in place (X, X, X), and a batch of batch_chunk() + 3 on a 2^8 chain.
- A BFV degree-3 polynomial on A at level 63 (MULRELIN and TENSOR at NM = 32).
- Chain R (66 moduli): BFV at levels 64 and 65 is refused before any launch; BGV at level 65 still matches the oracle.
Run with -m gpu on an H100."""
import ctypes
import functools
import os

import numpy as np
import pytest

from oracle import oracle as O
from tests import bgv_oracle as B
from tests import helpers as H
from tests import test_bgv_shapes_cpu as S
from tests.test_gpu_keyswitch_fused import digit_edges

pytestmark = pytest.mark.gpu
U64 = np.uint64
T = 0x10001


class Setup:
    """One chain: the device context with a uniform relinearization key, and per (scale_invariant, t) the device and oracle
    evaluators."""

    def __init__(self, logN, q, p, seed):
        import lattigo_b200 as lb
        self.logN, self.N = logN, 1 << logN
        self.q, self.p = [int(x) for x in q], [int(x) for x in p]
        self.qmul = B.qmul_moduli(logN, self.q)
        self.params = O.Parameters(logN, self.q, self.p)
        self.rng = np.random.default_rng(seed)
        self.rlk_o = H.random_gadget_ciphertext(self.params, len(q) - 1, len(p) - 1, self.rng)
        self.ctx = lb.Context(logN, self.q, self.p)
        self.rlk = lb.GadgetCiphertext(self.ctx, self.rlk_o.data, len(q) - 1, len(p) - 1)
        self._ev = {}

    def ev(self, si, t=T):
        import lattigo_b200 as lb
        if (si, t) not in self._ev:
            self._ev[(si, t)] = (lb.BGVEvaluator(self.ctx, t, self.qmul, self.rlk, scale_invariant=si),
                                 B.BGVEvaluator(self.params, t, self.qmul, self.rlk_o, scale_invariant=si))
        return self._ev[(si, t)]

    def cts(self, level, batch):
        return np.stack([np.stack([H.rand_poly(self.q[: level + 1], self.N, self.rng) for _ in range(2)]) for _ in range(batch)])

    def oracle(self, si, a, b, nb, t=T):
        """MulRelinNew (b is None: the squaring) followed by nb Rescales."""
        ev = self.ev(si, t)[1]
        x = [a[0].copy(), a[1].copy()]
        out = ev.MulRelinNew(x, x if b is None else [b[0].copy(), b[1].copy()])
        for _ in range(nb):
            out = ev.Rescale(out)
        return np.stack(out)

    def call(self, si, level, A, Bt, nb, out, batch, t=T):
        """lgpu_bgv_mulrelin_batch: (return code, last error)."""
        import torch
        import lattigo_b200 as lb
        L = lb.lib()
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda x: ctypes.c_void_p(x.data_ptr())
        rc = L.lgpu_bgv_mulrelin_batch(self.ev(si, t)[0].h, level, p(A), p(Bt), self.rlk.ref(), int(si), nb, p(out), batch, st)
        return rc, (L.lgpu_last_error().decode() if rc else None)

    def mul(self, si, A, Bt, nb=0, t=T, out=None):
        import torch
        batch, _, nq, N = A.shape
        if out is None:
            out = torch.empty((batch, 2, nq - nb, N), dtype=torch.int64, device=A.device)
        rc, err = self.call(si, nq - 1, A, Bt, nb, out, batch, t)
        assert rc == 0, err
        return out


@functools.lru_cache(maxsize=None)
def setup(name, logN):
    if name == "2^8":
        q, p = O.gen_moduli(9, [55, 40, 40, 40, 50, 50, 58, 58], [60, 60])
    else:
        q, p = S.chain(name, logN)
    return Setup(logN, q, p, seed=logN * 100 + len(q))


def _check(got, want, what):
    if not np.array_equal(got, want):
        bad = sorted({tuple(int(i) for i in ix[:-1]) for ix in zip(*np.nonzero(got != want))})
        raise AssertionError("%s: %d rows differ from the oracle, e.g. %s" % (what, len(bad), bad[:8]))


def _products(s, level, a, b, t=T, what=""):
    """BFV, and BGV with one Rescale (none at level 0), on the whole batch; every entry against the oracle."""
    A, Bt = s.ctx.to_device(a), s.ctx.to_device(b)
    for si, nb in ((True, 0), (False, 1 if level > 0 else 0)):
        out = s.ctx.to_host(s.mul(si, A, Bt, nb, t))
        for k in range(len(a)):
            _check(out[k], s.oracle(si, a[k], b[k], nb, t), "%s si=%d nb=%d t=%d entry %d" % (what, si, nb, t, k))


def _case_id(c):
    return "%s-2^%d-level%d" % c[:3]


@pytest.mark.parametrize("case", S.CASES, ids=_case_id)
def test_products_at_every_case(case):
    name, logN, level, _ = case
    s = setup(name, logN)
    _products(s, level, s.cts(level, 2), s.cts(level, 2), what=_case_id(case))


@pytest.mark.parametrize("name", ["A", "B"])
def test_plaintext_moduli(name):
    """t = 2 and t = Q[0] - 1 (tMontgomery, MForm(t mod q_i) with t > q_i on A) at the top level."""
    s = setup(name, S.LOGN)
    level = len(s.q) - 1
    a, b = s.cts(level, 2), s.cts(level, 2)
    for t in (2, s.q[0] - 1):
        _products(s, level, a, b, t, what=name)


def _ntt(s, level, coef):
    out = np.empty_like(coef)
    s.params.ringQ.AtLevel(level).NTT(coef, out)
    return out


def _edge_pair(s, level, alpha, words):
    """(a, b): a = (NTT(alpha), uniform), b = (NTT(beta), uniform), beta uniform except for words * alpha^-1 mod q_i at random
    coefficients, so that INTT(a_0 b_0) holds the words there."""
    Q = s.q[: level + 1]
    const = np.zeros((level + 1, s.N), dtype=U64)
    const[:, 0] = [alpha % q for q in Q]
    beta = H.rand_poly(Q, s.N, s.rng)
    pos = s.rng.choice(s.N, size=len(words), replace=False)
    for w, x in zip(words, pos):
        beta[:, x] = [int(wi) * pow(alpha, -1, q) % q for wi, q in zip(w, Q)]
    a = np.stack([_ntt(s, level, const), H.rand_poly(Q, s.N, s.rng)])
    b = np.stack([_ntt(s, level, beta), H.rand_poly(Q, s.N, s.rng)])
    return a, b


@pytest.mark.parametrize("case", S.edge_cases(), ids=lambda c: "%s-2^%d-level%d" % c)
def test_edge_inputs(case):
    name, logN, level = case
    s = setup(name, logN)
    words, _ = digit_edges(tuple(s.q[: level + 1]))
    pairs = [_edge_pair(s, level, 3, words), _edge_pair(s, level, 1, words)]
    mods = np.array(s.q[: level + 1], dtype=U64)[None, :, None]
    zero = np.zeros((2, level + 1, s.N), dtype=U64)
    top = np.broadcast_to(mods - U64(1), zero.shape).copy()
    pairs += [(zero, zero), (top, top)]
    a = np.stack([x for x, _ in pairs])
    b = np.stack([y for _, y in pairs])
    _products(s, level, a, b, what="%s-level%d edges" % (name, level))


@pytest.mark.parametrize("nb", [2, 6])
def test_bgv_several_rescales(nb):
    s = setup("A", S.LOGN)
    level = 6
    a, b = s.cts(level, 2), s.cts(level, 2)
    out = s.ctx.to_host(s.mul(False, s.ctx.to_device(a), s.ctx.to_device(b), nb))
    assert out.shape == (2, 2, level + 1 - nb, s.N)
    for k in range(2):
        _check(out[k], s.oracle(False, a[k], b[k], nb), "nb=%d entry %d" % (nb, k))


@pytest.mark.parametrize("si", [False, True])
def test_squaring_in_place(si):
    s = setup("A", S.LOGN)
    level = 32
    a = s.cts(level, 2)
    X = s.ctx.to_device(a)
    s.mul(si, X, X, 0, out=X)
    got = s.ctx.to_host(X)
    for k in range(2):
        _check(got[k], s.oracle(si, a[k], None, 0), "si=%d entry %d" % (si, k))


def test_batch_larger_than_batch_chunk():
    """batch_chunk() + 3 ciphertexts on the 2^8 chain of tests/test_gpu_bgv.py: BFV and BGV + Rescale, squaring and not."""
    s = setup("2^8", 8)
    level = len(s.q) - 1
    batch = int(os.environ.get("LGPU_BATCH_CHUNK", "64")) + 3          # batch_chunk() + 3
    a, b = s.cts(level, batch), s.cts(level, batch)
    A, Bt = s.ctx.to_device(a), s.ctx.to_device(b)
    for si, nb in ((True, 0), (False, 1)):
        for square in (False, True):
            out = s.ctx.to_host(s.mul(si, A, A if square else Bt, nb))
            for k in range(batch):
                _check(out[k], s.oracle(si, a[k], None if square else b[k], nb), "si=%d square=%d entry %d" % (si, square, k))


def test_bfv_polynomial_at_nm32():
    """lgpu_bgv_polynomial_evaluate, BFV degree 3 on A at level 63: its MULRELIN and TENSOR (poly_tensor_add_kernel) run the
    NM = 32 quantize."""
    import lattigo_b200 as lb
    from tests import bgv_polyeval_cases as C
    from tests import bgv_polyeval_oracle as BP
    s = setup("A", S.LOGN)
    level = 63
    coeffs = C.cases(T)["d3"][0]
    cts = s.cts(level, 2)
    pe = lb.BGVPolynomialEvaluator(s.ev(True)[0])
    out, lv, sc = pe.Evaluate(s.ctx.to_device(cts), 1, coeffs, 1)
    out = s.ctx.to_host(out)
    for k in range(2):
        r = BP.PolyEvaluator(s.params, s.rlk_o, T, s.qmul, True).Evaluate(BP.P.Ct([cts[k][0], cts[k][1]], 1), BP.new_polynomial(coeffs, True, True), 1)
        assert (lv, sc) == (r.Level(), int(r.Scale)) == (level, 1)
        _check(out[k], np.stack(r.Value), "entry %d" % k)


def test_bfv_refused_above_64_moduli():
    """Chain R: BFV at levels 64 and 65 fails its argument check with no launch; BGV at level 65 is unaffected."""
    import torch
    s = setup("R", S.LOGN)
    for level in (S.KMAX_SRC, S.KMAX_SRC + 1):
        A = torch.zeros((2, 2, level + 1, s.N), dtype=torch.int64, device="cuda")
        out = torch.empty_like(A)
        res = []
        n = H.launch_delta(lambda: res.append(s.call(True, level, A, A, 0, out, 2)))
        rc, err = res[0]
        assert rc != 0 and S.REFUSAL in err, (level, err)
        assert n == 0, (level, n)
    torch.cuda.synchronize()
    level = len(s.q) - 1
    a, b = s.cts(level, 2), s.cts(level, 2)
    out = s.ctx.to_host(s.mul(False, s.ctx.to_device(a), s.ctx.to_device(b), 0))
    for k in range(2):
        _check(out[k], s.oracle(False, a[k], b[k], 0), "BGV level %d entry %d" % (level, k))

"""GPU parity of lgpu_blind_rotation_evaluate (rgsw.BlindRotationEvaluator.Evaluate) with oracle/blindrot_evaluate.py
(blindrot.Evaluator.Evaluate, core/rgsw/blindrot/evaluator.go:49-132), bit for bit: uniform keys, test polynomials and LWE ciphertexts
(parity is over Z_q identities), on every variant of the fused kernel (csrc/blindrot.cu), on the per-slot fallback, and on every error."""
import numpy as np
import pytest

from oracle import blindrot_evaluate as BE
from oracle import oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu
U64 = np.uint64
Q_BR, Q_LWE = 0x7fff801, 0x3001        # core/rgsw/blindrot/blindrot_test.go


def _is_prime(n):
    if n < 2 or n % 2 == 0:
        return n == 2
    d = 3
    while d * d <= n:
        if n % d == 0:
            return False
        d += 2
    return True


def _prime_below(bound, two_n):
    p = (bound - 1) // two_n * two_n + 1
    while not _is_prime(p):
        p -= two_n
    return p


class Case:
    def __init__(self, logN, q, p, pw2, log_lwe, window, seed, q_lwe=Q_LWE, levelQ=None):
        import lattigo_b200 as lb
        self.params = O.Parameters(logN, q, p)
        self.params_lwe = O.Parameters(log_lwe, [q_lwe], [])
        self.N, self.n_lwe, self.window, self.q, self.q_lwe = 1 << logN, 1 << log_lwe, window, q, q_lwe
        self.level = len(q) - 1 if levelQ is None else levelQ
        levelP = len(p) - 1
        rng = self.rng = np.random.default_rng(seed)
        self.brk = [[H.random_gadget_ciphertext(self.params, self.level, levelP, rng, pw2=pw2) for _ in range(2)] for _ in range(self.n_lwe)]
        gals = [self.params.GaloisElement(k) for k in range(1, window + 1)] + [2 * self.N - 5]
        self.gks = {g: H.random_gadget_ciphertext(self.params, self.level, levelP, rng, pw2=pw2) for g in gals}
        self.ctx = lb.Context(logN, q, p)
        self.ctx_lwe = lb.Context(log_lwe, [q_lwe], [])
        mk = lambda g: lb.GadgetCiphertext(self.ctx, g.data, self.level, levelP, pw2, g.pw2_sizes)
        self.ev = lb.rgsw.BlindRotationEvaluator(self.ctx, [lb.rgsw.Ciphertext(mk(b[0]), mk(b[1])) for b in self.brk],
                                                 {g: mk(k) for g, k in self.gks.items()}, window)
        self.oracle = BE.Evaluator(self.params, self.params_lwe, window)

    def close(self):
        self.ctx.close(); self.ctx_lwe.close()

    def lwe(self, batch):
        ct = self.rng.integers(0, self.q_lwe, (batch, 2, 1, self.n_lwe), dtype=U64)
        ct[0, 1, 0, :2] = [0, self.q_lwe - 1]                 # edge words of the mask and of b
        ct[0, 0, 0, -2:] = [self.q_lwe - 1, 0]
        return ct

    def test_polys(self, slots, shared=False):
        one = H.rand_poly(self.q[: self.level + 1], self.N, self.rng)
        return {s: one if shared else H.rand_poly(self.q[: self.level + 1], self.N, self.rng) for s in slots}

    def want(self, ct, tps, is_ntt, ntt_out):
        return self.oracle.Evaluate([ct[0], ct[1]], tps, self.brk, self.gks, is_ntt=is_ntt, ntt_flag=ntt_out)

    def run(self, ct, tps, is_ntt=True, ntt_out=True):
        d = {s: self.ctx.to_device(t) for s, t in tps.items()}
        res = self.ev.Evaluate(self.ctx_lwe.to_device(ct), d, self.ctx_lwe, is_ntt=is_ntt, ntt_out=ntt_out)
        return {s: self.ctx.to_host(v) for s, v in res.items()}

    def check(self, batch=1, slots=None, is_ntt=True, ntt_out=True, shared=False, check_slots=None):
        slots = list(range(self.n_lwe)) if slots is None else slots
        ct = self.lwe(batch)
        if is_ntt:
            ring = self.params_lwe.ringQ
            for b in range(batch):
                for c in range(2):
                    ring.NTT(ct[b, c], ct[b, c])
        tps = self.test_polys(slots, shared)
        got = self.run(ct, tps, is_ntt, ntt_out)
        for b in range(batch):
            sel = {s: tps[s] for s in (slots if check_slots is None else check_slots)}
            want = self.want(ct[b], sel, is_ntt, ntt_out)
            for s, w in want.items():
                g = got[s][b]
                assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1]), (b, s)
        return ct, tps, got


def test_reference_shape_all_slots():
    """N = 2^10, Q = 0x7fff801, BaseTwoDecomposition 7, N_LWE = 2^9, q_LWE = 0x3001, window 10 (blindrot_test.go), all 512 slots in one
    call: slots 0, 1, 256 and 511 against the oracle, every slot against a one-slot call, and the same launch count at 1 and 512 slots."""
    c = Case(10, [Q_BR], [], 7, 9, 10, seed=1)
    try:
        ct, tps, got = c.check(slots=None, check_slots=[0, 1, 256, 511], shared=True)
        d_ct = c.ctx_lwe.to_device(ct)
        d_tp = c.ctx.to_device(tps[0])
        for s in range(c.n_lwe):
            one = c.ev.Evaluate(d_ct, {s: d_tp}, c.ctx_lwe)[s]
            assert np.array_equal(c.ctx.to_host(one), got[s]), s
        n1 = H.launch_delta(lambda: c.ev.Evaluate(d_ct, {7: d_tp}, c.ctx_lwe))
        n512 = H.launch_delta(lambda: c.ev.Evaluate(d_ct, {s: d_tp for s in range(c.n_lwe)}, c.ctx_lwe))
        assert n1 == n512 == 3, (n1, n512)                    # INTT of the LWE ciphertexts, modulus switch, fused kernel
        n0 = H.launch_delta(lambda: c.ev.Evaluate(c.ctx_lwe.to_device(ct[0]), {7: d_tp}, c.ctx_lwe, is_ntt=False))
        assert n0 == 2
    finally:
        c.close()


def test_small_q_domains_batches_and_per_slot_polynomials():
    """q < 2^29 with BaseTwoDecomposition 7: coefficient- and NTT-domain inputs, ntt_out 0 and 1, batches 1 and 3, a different test
    polynomial per slot, a subset of slots."""
    c = Case(8, [Q_BR], [], 7, 5, 10, seed=2)
    try:
        for is_ntt, ntt_out, batch in ((True, True, 1), (False, True, 3), (True, False, 3), (False, False, 1)):
            c.check(batch=batch, slots=[0, 3, 17, 31], is_ntt=is_ntt, ntt_out=ntt_out)
    finally:
        c.close()


@pytest.mark.parametrize("pw2", [1, 2])
def test_small_q_near_2_29_wrapping_accumulator(pw2):
    """q just below 2^29 with BaseTwoDecomposition 1 / 2: 2 * ceil(29 / w) products, each below 6q * q, are summed in the reference's
    64-bit word (externalProduct32Bit), which wraps; the fused kernel keeps that word."""
    logN = 8
    q = _prime_below(1 << 29, 1 << (logN + 1))
    c = Case(logN, [q], [], pw2, 4, 10, seed=3 + pw2)
    try:
        # the oracle's accumulator on these operands, in Python integers: some coefficient's sum exceeds 2^64
        ring = c.params.ringQ.AtLevel(0)
        s0 = ring.SubRings[0]
        acc = [H.rand_poly([q], c.N, c.rng), H.rand_poly([q], c.N, c.rng)]
        total = [0] * c.N
        for i, el in enumerate(c.brk[0]):
            inv = np.empty_like(acc[i]); ring.INTT(acc[i], inv)
            for j in range(el.BaseTwoDecompositionVectorSize()[0]):
                cw = np.array([(int(x) >> (j * pw2)) & ((1 << pw2) - 1) for x in inv[0]], dtype=U64)
                cwn = np.empty_like(cw); s0.NTTLazy(cw, cwn)
                for k in range(c.N):
                    total[k] += int(el.Q(0, j, 0)[0][k]) * int(cwn[k])
        assert max(total) >= 1 << 64, max(total).bit_length()
        c.check(slots=[0, 5, 15], is_ntt=False)
    finally:
        c.close()


def test_montgomery_path_50_bit_q():
    q, _ = O.gen_moduli(9, [50], [])
    c = Case(8, q, [], 10, 5, 10, seed=6)
    try:
        c.check(batch=2, slots=[1, 30])
    finally:
        c.close()


def test_largest_fused_ring_degree():
    """N = 2^12 (the largest N whose six working polynomials fit one CTA's shared memory) with a window of 64."""
    q, _ = O.gen_moduli(13, [27], [])
    c = Case(12, q, [], 7, 4, 64, seed=7)
    try:
        c.check(slots=[0, 9])
        d = c.ctx_lwe.to_device(c.lwe(1))
        assert H.launch_delta(lambda: c.ev.Evaluate(d, {9: c.ctx.to_device(c.test_polys([9])[9])}, c.ctx_lwe, is_ntt=False)) == 2
    finally:
        c.close()


def test_fallback_first_degree_above_the_bound():
    q, _ = O.gen_moduli(14, [27], [])
    c = Case(13, q, [], 7, 4, 64, seed=8)
    try:
        c.check(slots=[2], ntt_out=False)
        d = c.ctx_lwe.to_device(c.lwe(1))
        assert H.launch_delta(lambda: c.ev.Evaluate(d, {2: c.ctx.to_device(c.test_polys([2])[2])}, c.ctx_lwe, is_ntt=False)) > 100
    finally:
        c.close()


def test_fallback_two_q_limbs_and_p_keys():
    q, _ = O.gen_moduli(9, [45, 40], [])
    c = Case(8, q, [], 10, 4, 10, seed=9)
    try:
        c.check(batch=2, slots=[0, 7])
    finally:
        c.close()
    q, p = O.gen_moduli(9, [45], [50])
    c = Case(8, q, p, 0, 4, 10, seed=10)
    try:
        c.check(slots=[3, 15], is_ntt=False, ntt_out=False)
    finally:
        c.close()


def test_errors():
    import ctypes
    import lattigo_b200 as lb
    c = Case(8, [Q_BR], [], 7, 5, 4, seed=11)
    try:
        ct = c.lwe(1)
        d = c.ctx_lwe.to_device(ct)
        tp = c.ctx.to_device(c.test_polys([0])[0])
        ev = c.ev
        with pytest.raises(lb.LgpuError, match="duplicate slot"):
            polys = (ctypes.c_void_p * 2)(tp.data_ptr(), tp.data_ptr())
            out = c.ctx.to_device(np.zeros((1, 2, 2, 1, c.N), dtype=U64))
            lb._lib.check(lb.lib().lgpu_blind_rotation_evaluate(c.ctx.h, c.ctx_lwe.h, d.data_ptr(), 0, 1, (ctypes.c_int * 2)(3, 3), 2, polys,
                                                                ev._b0, ev._b1, len(ev.brk), ctypes.byref(ev._gks), ev.window, 1,
                                                                out.data_ptr(), 1, None))
        with pytest.raises(lb.LgpuError, match="out of range"):
            ev.Evaluate(d, {c.n_lwe: tp}, c.ctx_lwe)
        with pytest.raises(lb.LgpuError, match="above level 0"):
            ev.Evaluate(c.ctx_lwe.to_device(np.zeros((1, 2, 2, c.n_lwe), dtype=U64)), {0: tp}, c.ctx_lwe)
        missing = lb.rgsw.BlindRotationEvaluator(c.ctx, ev.brk, {g: k for g, k in ev.keys.items() if g != c.params.GaloisElement(3)}, 4)
        n0 = lb.lib().lgpu_launch_count()
        with pytest.raises(lb.LgpuError, match=r"GaloisKey\[%d\] is missing" % c.params.GaloisElement(3)):
            missing.Evaluate(d, {0: tp}, c.ctx_lwe)
        assert lb.lib().lgpu_launch_count() == n0
        few = lb.rgsw.BlindRotationEvaluator(c.ctx, ev.brk[:-1], ev.keys, 4)
        with pytest.raises(lb.LgpuError, match="fewer blind-rotation keys"):
            few.Evaluate(d, {0: tp}, c.ctx_lwe)
        big = lb.Context(9, [Q_LWE], [])
        try:
            with pytest.raises(lb.LgpuError, match="LWE ring degree is larger"):
                ev.Evaluate(big.to_device(np.zeros((1, 2, 1, 2 * c.N), dtype=U64)), {0: tp}, big)
        finally:
            big.close()
        # a correct call afterwards still matches the oracle
        want = c.want(ct[0], {0: c.ctx.to_host(tp)}, True, True)
        got = c.ctx.to_host(ev.Evaluate(d, {0: tp}, c.ctx_lwe)[0])
        assert np.array_equal(got[0][0], want[0][0]) and np.array_equal(got[0][1], want[0][1])
    finally:
        c.close()

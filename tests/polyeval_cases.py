"""Shared setup of the polynomial-evaluation tests: toy CKKS parameters with a real secret key and relinearization key, slots
encoded with the reference encoder's special FFT (oracle/specialfft.py), and the polynomial cases the oracle, the planner and the
device are checked on."""
from fractions import Fraction

import numpy as np

from oracle import oracle as O
from oracle import polyeval as OP
from oracle import specialfft as SF
from tests import helpers as H

U64 = np.uint64
M, C = OP.MONOMIAL, OP.CHEBYSHEV


def _coeffs(rng, deg, odd=True, even=True):
    c = [float(rng.uniform(-1, 1)) / (k + 1) for k in range(deg + 1)]
    for k in range(deg + 1):
        if (k & 1 and not odd) or (k & 1 == 0 and not even):
            c[k] = 0.0
    return c


def cases():
    """name -> (basis, coefficients, odd, even, levels_per_rescale, target scale as a multiple of the input scale)."""
    rng = np.random.default_rng(7)
    out = {}
    for d in (1, 2, 3, 7, 15):
        out["mono%d" % d] = (M, _coeffs(rng, d), True, True, 1, 1)
    out["mono5_giant2"] = (M, _coeffs(rng, 5), True, True, 1, 1)            # babySteps [3, 1]: the giantsteps[i] == 2 carry
    out["cheb30_even"] = (C, _coeffs(rng, 30, odd=False), False, True, 1, 1)
    out["cheb63_odd"] = (C, _coeffs(rng, 63, even=False), True, False, 1, 1)
    out["const_only"] = (M, [0.3125, 0.0], False, True, 1, 1)               # even, degree 1: the baby step is Add(res, c0) only
    out["mono7_lpr2"] = (M, _coeffs(rng, 7), True, True, 2, 1)
    out["mono3_target"] = (M, _coeffs(rng, 3), True, True, 1, Fraction(1, 2))
    out["cheb12_general"] = (C, _coeffs(rng, 12), True, True, 1, 1)
    # complex coefficients: the two NTT halves get different scalars (evaluateWithScalar's MRed(imag, RootsForward[1]))
    out["mono3_complex"] = (M, [0.25 + 0.125j, 0.5 - 0.25j, 0.1j, 0.3 + 0.05j], True, True, 1, 1)
    out["cheb7_complex"] = (C, [complex(c, 0.5 * c) for c in _coeffs(rng, 7)], True, True, 1, 1)
    return out


def expected(basis, coeffs, x):
    if basis == M:
        return np.polynomial.polynomial.polyval(x, coeffs)
    return np.polynomial.chebyshev.chebval(x, coeffs)


def negacyclic(a, b):
    N = len(a)
    full = np.convolve(np.asarray(a, dtype=np.int64), np.asarray(b, dtype=np.int64))
    out = full[:N].copy()
    out[: N - 1] -= full[N:]
    return out


class Toy:
    """Parameters, keys and an encryption of random real slots in [-1, 1]. lpr = 2 uses pairs of 40-bit primes per rescale."""

    def __init__(self, logN=10, lpr=1, nlevels=8, seed=1, logscale=40):
        self.logN, self.lpr = logN, lpr
        q, p = O.gen_moduli(logN + 1, [55] + [logscale // lpr] * (nlevels * lpr), [55, 55])
        self.q, self.p = q, p
        self.params = O.Parameters(logN, q, p)
        N = self.N = 1 << logN
        rng = self.rng = np.random.default_rng(seed)
        self.s = rng.integers(-1, 2, N)
        s2 = negacyclic(self.s, self.s)
        self.rlk = H.gen_switching_key(self.params, s2, self.s, rng)
        self.scale = Fraction(2) ** logscale
        self.prec = max(53, logscale)
        L = self.params.MaxLevelQ()
        self.sn = np.empty((L + 1, N), dtype=U64)
        self.params.ringQ.NTT(H.small_poly_rns(self.s, q), self.sn)

    def encrypt(self, values):
        """(c0, c1) = (-a s + m + e, a) in the NTT domain at the top level; m encodes `values` (N/2 real slots) at self.scale."""
        N, q, rng = self.N, self.q, self.rng
        n, m = N // 2, 2 * N
        v = [complex(x) for x in values]
        SF.special_ifft(v, n, m, SF.rot_group(m), SF.roots(m))
        coeffs = np.zeros(N, dtype=object)
        for i in range(n):
            coeffs[i] = int(round(v[i].real * float(self.scale)))
            coeffs[n + i] = int(round(v[i].imag * float(self.scale)))
        e = np.rint(rng.normal(0, 3.2, N)).astype(np.int64)
        ringQ = self.params.ringQ
        me = np.stack([np.array([(int(c) + int(ei)) % qi for c, ei in zip(coeffs, e)], dtype=U64) for qi in q])
        ringQ.NTT(me, me)
        a = H.rand_poly(q, N, rng)
        c0 = np.stack([np.array([(int(x) - int(y) * int(t)) % int(mod) for x, y, t in zip(me[l], a[l], self.sn[l])], dtype=U64)
                       for l, mod in enumerate(q)])
        return [c0, a]

    def decrypt(self, ct, scale):
        level = ct[0].shape[0] - 1
        ringQ = self.params.ringQ.AtLevel(level)
        q = self.q[: level + 1]
        acc = np.stack([np.array([(int(a) + int(b) * int(t)) % int(mod) for a, b, t in zip(ct[0][l], ct[1][l], self.sn[l])], dtype=U64)
                        for l, mod in enumerate(q)])
        back = np.empty_like(acc)
        ringQ.INTT(acc, back)
        Q = ringQ.ModulusAtLevel[level]
        c = [x if x < Q // 2 else x - Q for x in ringQ.PolyToBigint(back)]
        N, n = self.N, self.N // 2
        v = [complex(float(Fraction(c[i]) / scale), float(Fraction(c[n + i]) / scale)) for i in range(n)]
        SF.special_fft(v, n, 2 * N, SF.rot_group(2 * N), SF.roots(2 * N))
        return np.array(v)

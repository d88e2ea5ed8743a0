"""oracle/oracle.py -- TEST INFRASTRUCTURE ONLY (CPU oracle, "port" of the reference).

A CPU restatement of tuneinsight/lattigo v6.2.0's RNS polynomial-ring hot path:
the per-coefficient arithmetic lives in ``lattigo_oracle.c`` (plain C, built by
``oracle/Makefile``); this module restates the Go *control flow* around it
(``ring.Ring``, ``ring.BasisExtender``, ``ring.Decomposer``, ``rlwe.Evaluator``'s
GadgetProduct family, ``ckks.Evaluator.mulRelin`` / ``Rescale``) and regenerates
every constant table with Python big integers, independently of the product's
own (modular-arithmetic) table generation in ``lattigo_b200/csrc``.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline``
/ ``--impl reference`` legs may import this module. The product package
``lattigo_b200`` never does.

Parity pinning: ``tests/test_oracle_golden.py`` checks this oracle against the
reference's own golden NTT vectors (ring/ntt_test.go:10-89, committed as
tests/golden/ntt_vectors.json) and against big-integer ground truth for
ModUp/ModDown/DivRound/DivFloor (mirroring ring/ring_test.go:245-334,710-887).
GadgetProduct / Automorphism / mulRelin have no bit-level vectors in the
reference (only noise bounds); for those the oracle is anchored by the pinned
building blocks plus the algebraic decrypt-style check in tests/.

All ``file:line`` citations are relative to the upstream tree.
"""
from __future__ import annotations

import ctypes
import math
import os
import subprocess
from typing import List, Optional, Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liblattigo_oracle.so")
U64 = np.uint64
MASK64 = (1 << 64) - 1


def build(force: bool = False) -> str:
    """Compile oracle/lattigo_oracle.c with oracle/Makefile (gcc)."""
    src = os.path.join(_HERE, "lattigo_oracle.c")
    if force or not os.path.exists(_SO) or (
        os.path.exists(src) and os.path.getmtime(src) > os.path.getmtime(_SO)
    ):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_SO)
        c = ctypes
        p = c.c_void_p
        u = c.c_uint64
        i = c.c_int
        z = c.c_size_t
        L.lo_ntt.argtypes = [p, p, i, u, u, p, p]
        L.lo_ntt_lazy.argtypes = [p, p, i, u, u, p]
        L.lo_intt.argtypes = [p, p, i, u, u, u, p]
        L.lo_intt_lazy.argtypes = [p, p, i, u, u, u, p]
        L.lo_ntt_ci.argtypes = [p, p, i, u, u, p, p]
        L.lo_ntt_ci_lazy.argtypes = [p, p, i, u, u, p]
        L.lo_intt_ci.argtypes = [p, p, i, u, u, u, p]
        L.lo_intt_ci_lazy.argtypes = [p, p, i, u, u, u, p]
        L.lo_vecop.argtypes = [i, p, p, p, i, u, u, p, u, u]
        L.lo_vecop.restype = i
        L.lo_modup_exact.argtypes = [p, z, i, p, z, i, i, p, p, p, p, p, p, z, p, z]
        L.lo_decompose_reconstruct.argtypes = [p, z, i, p, i, i, p, p, p, p, p, p, p, p]
        L.lo_decompose_single.argtypes = [p, u, p, i, i, p, p]
        L.lo_automorphism_ntt_index.argtypes = [i, u, u, p]
        L.lo_automorphism_ntt_row.argtypes = [p, p, p, i, i]
        L.lo_automorphism_row.argtypes = [p, p, i, u, u]
        L.lo_automorphism_row_ci.argtypes = [p, p, i, u, u]
        for name in ("lo_mred", "lo_mred_lazy"):
            f = getattr(L, name); f.argtypes = [u, u, u, u]; f.restype = u
        for name in ("lo_mform", "lo_mform_lazy", "lo_bred_add", "lo_bred_add_lazy"):
            f = getattr(L, name); f.argtypes = [u, u, p]; f.restype = u
        for name in ("lo_bred", "lo_bred_lazy"):
            f = getattr(L, name); f.argtypes = [u, u, u, p]; f.restype = u
        L.lo_imform.argtypes = [u, u, u]; L.lo_imform.restype = u
        L.lo_cred.argtypes = [u, u]; L.lo_cred.restype = u
        _lib = L
    return _lib


def _ptr(a: Optional[np.ndarray]):
    if a is None:
        return None
    assert a.dtype == np.uint64 and a.flags["C_CONTIGUOUS"], (a.dtype, a.flags)
    return a.ctypes.data


# Opcode numbering shared with include/lattigo_b200.h (LGPU_OP_*) and
# oracle/lattigo_oracle.c. Names are the reference's vec_ops.go kernels.
OPS = [
    "Add", "AddLazy", "Sub", "SubLazy", "Neg", "Reduce", "ReduceLazy",
    "MulCoeffsLazy", "MulCoeffsLazyThenAddLazy",
    "MulCoeffsBarrett", "MulCoeffsBarrettLazy", "MulCoeffsBarrettThenAdd", "MulCoeffsBarrettThenAddLazy",
    "MulCoeffsMontgomery", "MulCoeffsMontgomeryLazy", "MulCoeffsMontgomeryThenAdd",
    "MulCoeffsMontgomeryThenAddLazy", "MulCoeffsMontgomeryLazyThenAddLazy",
    "MulCoeffsMontgomeryThenSub", "MulCoeffsMontgomeryThenSubLazy", "MulCoeffsMontgomeryLazyThenSubLazy",
    "MulCoeffsMontgomeryLazyThenNeg",
    "AddLazyThenMulScalarMontgomery", "AddScalarLazyThenMulScalarMontgomery",
    "AddScalar", "AddScalarLazy", "AddScalarLazyThenNegTwoModulusLazy", "SubScalar",
    "MulScalarMontgomery", "MulScalarMontgomeryLazy", "MulScalarMontgomeryThenAdd",
    "MulScalarMontgomeryThenAddScalar", "SubThenMulScalarMontgomeryTwoModulus",
    "MForm", "MFormLazy", "IMForm", "Zero", "Mask",
]
OP = {n: k for k, n in enumerate(OPS)}


# --------------------------------------------------------------------------
# number theory helpers (setup only; Python big ints)
# --------------------------------------------------------------------------
def bit_reverse64(x: int, bits: int) -> int:
    """utils/utils.go:34"""
    return int(format(x, "064b")[::-1], 2) >> (64 - bits) if bits else 0


def is_prime(n: int) -> bool:
    """ring/primes.go:11 (Baillie-PSW in Go; deterministic Miller-Rabin here, exact below 2^64)."""
    if n < 2:
        return False
    small = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)
    for p in small:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d //= 2; s += 1
    for a in small:
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def _pollard_rho(n: int) -> int:
    if n % 2 == 0:
        return 2
    c = 1
    while True:
        f = lambda v: (v * v + c) % n
        x = y = 2; d = 1
        while d == 1:
            x = f(x); y = f(f(y)); d = math.gcd(abs(x - y), n)
        if d != n:
            return d
        c += 1


def unique_factors(n: int) -> List[int]:
    """Unique prime factors of n (utils/factorization.GetFactors, used by ring/subring.go:171)."""
    out = set()
    stack = [n]
    while stack:
        m = stack.pop()
        if m == 1:
            continue
        if is_prime(m):
            out.add(m); continue
        for p in (2, 3, 5, 7, 11, 13):
            if m % p == 0:
                out.add(p)
                while m % p == 0:
                    m //= p
                stack.append(m)
                break
        else:
            d = _pollard_rho(m)
            stack += [d, m // d]
    return sorted(out)


def primitive_root(q: int) -> int:
    """ring/subring.go:161-194: g starts at 2 and is incremented BEFORE testing,
    so the smallest candidate ever tested is 3."""
    factors = unique_factors(q - 1)
    g = 2
    while True:
        g += 1
        if all(pow(g, (q - 1) // f, q) != 1 for f in factors):
            return g


def gen_bred_constant(q: int):
    """ring/modular_reduction.go:99-107 -> [hi, lo] of floor(2^128/q)"""
    r = (1 << 128) // q
    return [r >> 64, r & MASK64]


def gen_mred_constant(q: int) -> int:
    """ring/modular_reduction.go:68-75 -> q^-1 mod 2^64"""
    return pow(q, -1, 1 << 64)


def mform(a: int, q: int) -> int:
    return (a << 64) % q


# --------------------------------------------------------------------------
# ring.SubRing / ring.Ring
# --------------------------------------------------------------------------
class SubRing:
    """ring/subring.go:15-35 (+ NTTTable ring/ntt.go:38-44)."""

    def __init__(self, N: int, q: int, nthroot: Optional[int] = None, ring_type: str = "Standard"):
        self.N = N
        self.Modulus = q
        self.Type = ring_type
        self.NthRoot = nthroot if nthroot is not None else (2 * N if ring_type == "Standard" else 4 * N)
        assert is_prime(q) and q % self.NthRoot == 1, "modulus must be an NTT-friendly prime"
        self.BRedConstant = gen_bred_constant(q)
        self.brc = np.array(self.BRedConstant, dtype=U64)
        self.MRedConstant = gen_mred_constant(q)
        self.Mask = (1 << (q - 1).bit_length()) - 1
        # generateNTTConstants, ring/subring.go:99-159
        self.PrimitiveRoot = primitive_root(q)
        nr = self.NthRoot
        log = (nr >> 1).bit_length() - 1
        self.NInv = mform(pow(nr >> 1, q - 2, q), q)
        psi = pow(self.PrimitiveRoot, (q - 1) // nr, q)
        psi_inv = pow(psi, q - 2, q)
        half = nr >> 1
        idx = _brev_table(log)
        fw = np.empty(half, dtype=object); bw = np.empty(half, dtype=object)
        cf, cb = mform(1, q), mform(1, q)
        for j in range(half):
            fw[j] = cf; bw[j] = cb
            cf = cf * psi % q; cb = cb * psi_inv % q
        self.RootsForward = np.empty(half, dtype=U64); self.RootsBackward = np.empty(half, dtype=U64)
        self.RootsForward[idx] = fw.astype(U64)
        self.RootsBackward[idx] = bw.astype(U64)

    # --- SubRing methods, ring/subring_ops.go:6-273 (all via lo_vecop) ---
    def vecop(self, name, p1, p2, p3, s0=0, s1=0):
        rc = lib().lo_vecop(OP[name], _ptr(p1), _ptr(p2), _ptr(p3), p3.shape[-1], self.Modulus,
                            self.MRedConstant, _ptr(self.brc), int(s0) & MASK64, int(s1) & MASK64)
        assert rc == 0

    def NTT(self, p1, p2):
        f = lib().lo_ntt if self.Type == "Standard" else lib().lo_ntt_ci
        f(_ptr(p1), _ptr(p2), self.N, self.Modulus, self.MRedConstant, _ptr(self.brc), _ptr(self.RootsForward))

    def NTTLazy(self, p1, p2):
        f = lib().lo_ntt_lazy if self.Type == "Standard" else lib().lo_ntt_ci_lazy
        f(_ptr(p1), _ptr(p2), self.N, self.Modulus, self.MRedConstant, _ptr(self.RootsForward))

    def INTT(self, p1, p2):
        f = lib().lo_intt if self.Type == "Standard" else lib().lo_intt_ci
        f(_ptr(p1), _ptr(p2), self.N, self.NInv, self.Modulus, self.MRedConstant, _ptr(self.RootsBackward))

    def INTTLazy(self, p1, p2):
        f = lib().lo_intt_lazy if self.Type == "Standard" else lib().lo_intt_ci_lazy
        f(_ptr(p1), _ptr(p2), self.N, self.NInv, self.Modulus, self.MRedConstant, _ptr(self.RootsBackward))


_BREV_CACHE = {}


def _brev_table(log: int) -> np.ndarray:
    if log not in _BREV_CACHE:
        n = 1 << log
        idx = np.arange(n, dtype=np.int64)
        r = np.zeros(n, dtype=np.int64)
        for b in range(log):
            r |= ((idx >> b) & 1) << (log - 1 - b)
        _BREV_CACHE[log] = r
    return _BREV_CACHE[log]


_SUBRING_CACHE = {}


def get_subring(N, q, ring_type="Standard") -> SubRing:
    key = (N, q, ring_type)
    if key not in _SUBRING_CACHE:
        _SUBRING_CACHE[key] = SubRing(N, q, ring_type=ring_type)
    return _SUBRING_CACHE[key]


class Ring:
    """ring/ring.go:71-82. Polynomials are numpy uint64 arrays of shape (limbs, N)."""

    def __init__(self, N: int, moduli: Sequence[int], ring_type: str = "Standard", _share=None, level=None):
        if _share is not None:
            self.__dict__.update(_share.__dict__)
            self.level = level
            return
        self.SubRings = [get_subring(N, int(q), ring_type) for q in moduli]
        self.Type = ring_type
        self.ModulusAtLevel = []
        acc = 1
        for q in moduli:
            acc *= int(q); self.ModulusAtLevel.append(acc)
        # rewRescaleConstants, ring/ring.go:329-346
        self.RescaleConstants = []
        for j in range(1, len(moduli)):
            qj = int(moduli[j])
            self.RescaleConstants.append([mform(int(qi) - pow(qj, int(qi) - 2, int(qi)), int(qi)) for qi in moduli[:j]])
        self.level = len(moduli) - 1

    def N(self): return self.SubRings[0].N
    def NthRoot(self): return self.SubRings[0].NthRoot
    def Level(self): return self.level
    def MaxLevel(self): return len(self.SubRings) - 1
    def ModuliChain(self): return [s.Modulus for s in self.SubRings]
    def ModuliChainLength(self): return len(self.SubRings)
    def AtLevel(self, level): return Ring(0, [], _share=self, level=level)
    def NewPoly(self): return np.zeros((self.level + 1, self.N()), dtype=U64)

    # --- coefficient-wise ops, ring/operations.go:11-392 ---
    def _op(self, name, p1, p2, p3, s0=None, s1=None):
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            a = p1[i] if p1 is not None else None
            b = p2[i] if p2 is not None else None
            x0 = s0[i] if isinstance(s0, (list, tuple, np.ndarray)) else (s0 or 0)
            x1 = s1[i] if isinstance(s1, (list, tuple, np.ndarray)) else (s1 or 0)
            s.vecop(name, a, b, p3[i], x0, x1)

    def __getattr__(self, name):
        # Generic dispatch for the 2/3-operand vec ops: ring.X(p1, p2, p3) / ring.X(p1, p2)
        if name in OP:
            three = {"Add", "AddLazy", "Sub", "SubLazy"} | {n for n in OPS if n.startswith("MulCoeffs")}
            if name in three:
                return lambda p1, p2, p3: self._op(name, p1, p2, p3)
            if name in ("Neg", "Reduce", "ReduceLazy", "MForm", "MFormLazy", "IMForm"):
                return lambda p1, p2: self._op(name, p1, None, p2)
        raise AttributeError(name)

    def AddScalar(self, p1, scalar, p2):      # ring/operations.go:151
        self._op("AddScalar", p1, None, p2, [scalar % s.Modulus for s in self.SubRings[: self.level + 1]])

    def SubScalar(self, p1, scalar, p2):      # ring/operations.go:186
        self._op("SubScalar", p1, None, p2, [scalar % s.Modulus for s in self.SubRings[: self.level + 1]])

    def AddScalarBigint(self, p1, scalar: int, p2):   # ring/operations.go:158-163
        self._op("AddScalar", p1, None, p2, [scalar % s.Modulus for s in self.SubRings[: self.level + 1]])

    def SubScalarBigint(self, p1, scalar: int, p2):   # ring/operations.go:193-198
        self._op("SubScalar", p1, None, p2, [scalar % s.Modulus for s in self.SubRings[: self.level + 1]])

    def MulScalar(self, p1, scalar, p2):      # ring/operations.go:201-205
        self._op("MulScalarMontgomery", p1, None, p2, [mform(scalar % s.Modulus, s.Modulus) for s in self.SubRings[: self.level + 1]])

    def MulScalarThenAdd(self, p1, scalar, p2):   # ring/operations.go:208-213
        self._op("MulScalarMontgomeryThenAdd", p1, None, p2, [mform(scalar % s.Modulus, s.Modulus) for s in self.SubRings[: self.level + 1]])

    def _mods(self): return [s.Modulus for s in self.SubRings[: self.level + 1]]

    def AddDoubleRNSScalar(self, p1, scalar0, scalar1, p2):      # ring/operations.go:167-173
        h = self.N() >> 1
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            s.vecop("AddScalar", p1[i][:h], None, p2[i][:h], scalar0[i])
            s.vecop("AddScalar", p1[i][h:], None, p2[i][h:], scalar1[i])

    def SubDoubleRNSScalar(self, p1, scalar0, scalar1, p2):      # ring/operations.go:177-183
        h = self.N() >> 1
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            s.vecop("SubScalar", p1[i][:h], None, p2[i][:h], scalar0[i])
            s.vecop("SubScalar", p1[i][h:], None, p2[i][h:], scalar1[i])

    def MulRNSScalarMontgomery(self, p1, scalar, p2):           # ring/operations.go:216-220
        self._op("MulScalarMontgomery", p1, None, p2, list(scalar))

    def MulScalarThenSub(self, p1, scalar, p2):                 # ring/operations.go:223-228
        self._op("MulScalarMontgomeryThenAdd", p1, None, p2,
                 [mform(s.Modulus - scalar % s.Modulus, s.Modulus) for s in self.SubRings[: self.level + 1]])

    MulScalarBigint = MulScalar                                 # ring/operations.go:231-237
    MulScalarBigintThenAdd = MulScalarThenAdd                   # ring/operations.go:240-246

    def MulDoubleRNSScalar(self, p1, scalar0, scalar1, p2):     # ring/operations.go:250-256
        h = self.N() >> 1
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            s.vecop("MulScalarMontgomery", p1[i][:h], None, p2[i][:h], mform(scalar0[i], s.Modulus))
            s.vecop("MulScalarMontgomery", p1[i][h:], None, p2[i][h:], mform(scalar1[i], s.Modulus))

    def MulDoubleRNSScalarThenAdd(self, p1, scalar0, scalar1, p2):   # ring/operations.go:260-266
        h = self.N() >> 1
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            s.vecop("MulScalarMontgomeryThenAdd", p1[i][:h], None, p2[i][:h], mform(scalar0[i], s.Modulus))
            s.vecop("MulScalarMontgomeryThenAdd", p1[i][h:], None, p2[i][h:], mform(scalar1[i], s.Modulus))

    def EvalPolyScalar(self, p1, scalar, p2):                   # ring/operations.go:269-275
        p2[: self.level + 1] = p1[-1][: self.level + 1]
        for i in range(len(p1) - 1, 0, -1):
            self.MulScalar(p2, scalar, p2)
            self.Add(p2, p1[i - 1], p2)

    def Shift(self, p1, k, p2):                                 # ring/operations.go:278-282 (all rows of p1)
        n = self.N()
        k %= n
        for i in range(p1.shape[0]):
            p2[i] = np.concatenate([p1[i][k:], p1[i][:k]])

    def MultByMonomial(self, p1, k, p2):                        # ring/operations.go:306-363
        N = self.N()
        shift = (k + (N << 1)) % (N << 1)
        if shift == 0:
            p2[: self.level + 1] = p1[: self.level + 1]
            return
        tmpx = np.zeros_like(p1)
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            tmpx[i] = p1[i] if shift < N else (np.uint64(s.Modulus) - p1[i])
        shift %= N
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            out = np.empty(N, dtype=U64)
            out[:shift] = np.uint64(s.Modulus) - tmpx[i][N - shift:]
            out[shift:] = tmpx[i][: N - shift]
            p2[i] = out

    def MulByVectorMontgomery(self, p1, vector, p2):            # ring/operations.go:366-370
        for i, s in enumerate(self.SubRings[: self.level + 1]): s.vecop("MulCoeffsMontgomery", p1[i], vector, p2[i])

    def MulByVectorMontgomeryThenAddLazy(self, p1, vector, p2):  # ring/operations.go:373-377
        for i, s in enumerate(self.SubRings[: self.level + 1]): s.vecop("MulCoeffsMontgomeryThenAddLazy", p1[i], vector, p2[i])

    def NTT(self, p1, p2):        # ring/ntt.go:127
        for i, s in enumerate(self.SubRings[: self.level + 1]): s.NTT(p1[i], p2[i])

    def NTTLazy(self, p1, p2):    # ring/ntt.go:134
        for i, s in enumerate(self.SubRings[: self.level + 1]): s.NTTLazy(p1[i], p2[i])

    def INTT(self, p1, p2):       # ring/ntt.go:141
        for i, s in enumerate(self.SubRings[: self.level + 1]): s.INTT(p1[i], p2[i])

    def INTTLazy(self, p1, p2):   # ring/ntt.go:148
        for i, s in enumerate(self.SubRings[: self.level + 1]): s.INTTLazy(p1[i], p2[i])

    # --- ring/automorphism.go ---
    def AutomorphismNTTIndex(self, galEl: int) -> np.ndarray:
        idx = np.empty(self.N(), dtype=U64)
        lib().lo_automorphism_ntt_index(self.N(), self.NthRoot(), galEl, _ptr(idx))
        return idx

    def AutomorphismNTTWithIndex(self, polIn, index, polOut):       # :50-77
        for i in range(self.level + 1):
            lib().lo_automorphism_ntt_row(_ptr(polIn[i]), _ptr(index), _ptr(polOut[i]), self.N(), 0)

    def AutomorphismNTTWithIndexThenAddLazy(self, polIn, index, polOut):   # :82-109
        for i in range(self.level + 1):
            lib().lo_automorphism_ntt_row(_ptr(polIn[i]), _ptr(index), _ptr(polOut[i]), self.N(), 1)

    def AutomorphismNTT(self, polIn, gen, polOut):                  # :38-45
        self.AutomorphismNTTWithIndex(polIn, self.AutomorphismNTTIndex(gen), polOut)

    def Automorphism(self, polIn, gen, polOut):                     # :113-176
        f = lib().lo_automorphism_row if self.Type == "Standard" else lib().lo_automorphism_row_ci
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            f(_ptr(polIn[i]), _ptr(polOut[i]), self.N(), gen, s.Modulus)

    # --- ring/scaling.go ---
    def DivFloorByLastModulusNTT(self, p0, p1):     # :6-22
        level = self.level
        N = self.N()
        buff0 = np.empty(N, dtype=U64); buff1 = np.empty(N, dtype=U64)
        self.SubRings[level].INTTLazy(p0[level], buff0)
        for i, s in enumerate(self.SubRings[:level]):
            s.NTTLazy(buff0, buff1)
            s.vecop("SubThenMulScalarMontgomeryTwoModulus", buff1, p0[i], p1[i], self.RescaleConstants[level - 1][i])

    def DivFloorByLastModulus(self, p0, p1):        # :26-33
        level = self.level
        for i, s in enumerate(self.SubRings[:level]):
            s.vecop("SubThenMulScalarMontgomeryTwoModulus", p0[level], p0[i], p1[i], self.RescaleConstants[level - 1][i])

    def DivFloorByLastModulusManyNTT(self, nb, p0, p1):   # :37-61
        if nb == 0:
            if p0 is not p1: p1[: self.level + 1] = p0[: self.level + 1]
            return
        r = self.AtLevel(self.level)
        buff = np.empty((self.level + 1, self.N()), dtype=U64)
        r.INTT(p0, buff)
        for _ in range(nb):
            r.DivFloorByLastModulus(buff, buff)
            r = r.AtLevel(r.level - 1)
        r.NTT(buff, p1)

    def DivFloorByLastModulusMany(self, nb, p0, buff, p1):   # :65-97
        if nb == 0:
            if p0 is not p1: p1[: self.level + 1] = p0[: self.level + 1]
            return
        r = self.AtLevel(self.level)
        cur = p0
        for i in range(nb):
            dst = p1 if i == nb - 1 else buff
            r.DivFloorByLastModulus(cur, dst)
            cur = dst
            r = r.AtLevel(r.level - 1)

    def DivRoundByLastModulusNTT(self, p0, p1):     # :101-122
        level = self.level
        N = self.N()
        buff0 = np.empty(N, dtype=U64); buff1 = np.empty(N, dtype=U64)
        sl = self.SubRings[level]
        sl.INTTLazy(p0[level], buff0)
        pHalf = (sl.Modulus - 1) >> 1
        sl.vecop("AddScalar", buff0, None, buff0, pHalf)
        for i, s in enumerate(self.SubRings[:level]):
            s.vecop("AddScalarLazy", buff0, None, buff1, s.Modulus - pHalf % s.Modulus)
            s.NTTLazy(buff1, buff1)
            s.vecop("SubThenMulScalarMontgomeryTwoModulus", buff1, p0[i], p1[i], self.RescaleConstants[level - 1][i])

    def DivRoundByLastModulus(self, p0, p1):        # :126-144
        level = self.level
        N = self.N()
        buff0 = np.empty(N, dtype=U64); buff1 = np.empty(N, dtype=U64)
        sl = self.SubRings[level]
        pHalf = (sl.Modulus - 1) >> 1
        sl.vecop("AddScalar", p0[level], None, buff0, pHalf)
        for i, s in enumerate(self.SubRings[:level]):
            s.vecop("AddScalarLazyThenNegTwoModulusLazy", p0[i], None, buff1, s.Modulus - pHalf % s.Modulus)
            s.vecop("AddLazyThenMulScalarMontgomery", buff0, buff1, p1[i], self.RescaleConstants[level - 1][i])

    def DivRoundByLastModulusManyNTT(self, nb, p0, buff, p1):   # :148-176
        if nb == 0:
            if p0 is not p1: p1[: self.level + 1] = p0[: self.level + 1]
        elif nb > 1:
            r = self.AtLevel(self.level)
            b = np.empty((self.level + 1, self.N()), dtype=U64)
            r.INTT(p0, b)
            for _ in range(nb):
                r.DivRoundByLastModulus(b, b)
                r = r.AtLevel(r.level - 1)
            r.NTT(b, p1)
        else:
            self.DivRoundByLastModulusNTT(p0, p1)

    def DivRoundByLastModulusMany(self, nb, p0, buff, p1):      # :180-212
        if nb == 0:
            if p0 is not p1: p1[: self.level + 1] = p0[: self.level + 1]
            return
        r = self.AtLevel(self.level)
        cur = p0
        for i in range(nb):
            dst = p1 if i == nb - 1 else buff
            r.DivRoundByLastModulus(cur, dst)
            cur = dst
            r = r.AtLevel(r.level - 1)

    # big-int helpers for the property tests (ring/ring.go PolyToBigint / SetCoefficientsBigint)
    def PolyToBigint(self, p) -> List[int]:
        Q = self.ModulusAtLevel[self.level]
        out = [0] * self.N()
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            qi = s.Modulus
            Qi = Q // qi
            c = Qi * pow(Qi % qi, -1, qi)
            row = [int(v) % qi for v in p[i]]
            for j in range(self.N()):
                out[j] += row[j] * c
        return [v % Q for v in out]

    def SetCoefficientsBigint(self, coeffs: Sequence[int], p):
        for i, s in enumerate(self.SubRings[: self.level + 1]):
            p[i] = np.array([c % s.Modulus for c in coeffs], dtype=U64)


# --------------------------------------------------------------------------
# ring/basis_extension.go
# --------------------------------------------------------------------------
def MapSmallDimensionToLargerDimensionNTT(polSmall, polLarge):      # ring/operations.go:380-392
    gap = polLarge.shape[1] // polSmall.shape[1]
    for j in range(min(polSmall.shape[0], polLarge.shape[0])):
        polLarge[j] = np.repeat(polSmall[j], gap)


def ExtendBasisSmallNormAndCenter(ringQ: "Ring", ringP: "Ring", polyInQ, levelP, polyOutQ, polyOutP):
    """ringqp.Ring.ExtendBasisSmallNormAndCenter, ring/ringqp/operations.go:325-351."""
    Q = ringQ.SubRings[0].Modulus
    QHalf = Q >> 1
    if polyOutQ is not polyInQ:
        polyOutQ[...] = polyInQ
    c = polyInQ[0].copy()
    negm = c > np.uint64(QHalf)
    mag = np.where(negm, np.uint64(Q) - c, c)
    for i, pi in enumerate(ringP.ModuliChain()[: levelP + 1]):
        polyOutP[i] = np.where(negm, np.uint64(pi) - mag, mag)


class ModUpConstants:
    """GenModUpConstants, ring/basis_extension.go:101-172 (big-int restatement)."""

    def __init__(self, Q: Sequence[int], P: Sequence[int]):
        Q = [int(x) for x in Q]; P = [int(x) for x in P]
        prod = 1
        for q in Q: prod *= q
        self.qoverqiinvqi = np.array([mform(pow((prod // qi) % qi, -1, qi), qi) for qi in Q], dtype=U64)
        self.qoverqimodp = np.array([[mform((prod // qi) % pj, pj) for qi in Q] for pj in P], dtype=U64).reshape(len(P), len(Q))
        vt = []
        for pj in P:
            v = pj - prod % pj
            row = [0]
            for _ in range(len(Q)):
                nxt = row[-1] + v
                row.append(nxt - pj if nxt >= pj else nxt)   # CRed
            vt.append(row)
        self.vtimesqmodp = np.array(vt, dtype=U64).reshape(len(P), len(Q) + 1)


def mod_up_exact(p1, p2, ringQ: Ring, ringP: Ring, muc: ModUpConstants):
    """ModUpExact, ring/basis_extension.go:282-308. p1: (levelQ+1, N), p2: (levelP+1, N)."""
    nQ, nP, n = p1.shape[0], p2.shape[0], p1.shape[1]
    assert p1.strides[1] == 8 and p2.strides[1] == 8
    assert nQ <= 64, "lo_modup_exact holds at most 64 source limbs"
    Q = np.array(ringQ.ModuliChain()[:nQ], dtype=U64); mq = np.array([s.MRedConstant for s in ringQ.SubRings[:nQ]], dtype=U64)
    P = np.array(ringP.ModuliChain()[:nP], dtype=U64); mp = np.array([s.MRedConstant for s in ringP.SubRings[:nP]], dtype=U64)
    lib().lo_modup_exact(p1.ctypes.data, p1.strides[0] // 8, nQ, p2.ctypes.data, p2.strides[0] // 8, nP, n,
                         _ptr(Q), _ptr(mq), _ptr(P), _ptr(mp), _ptr(muc.qoverqiinvqi),
                         _ptr(muc.qoverqimodp), muc.qoverqimodp.shape[1], _ptr(muc.vtimesqmodp), muc.vtimesqmodp.shape[1])


class BasisExtender:
    """ring/basis_extension.go:14-87."""

    def __init__(self, ringQ: Ring, ringP: Ring):
        self.ringQ, self.ringP = ringQ, ringP
        Q, P = ringQ.ModuliChain(), ringP.ModuliChain()
        self.constantsQtoP = [ModUpConstants(Q[: i + 1], P) for i in range(len(Q))]
        self.constantsPtoQ = [ModUpConstants(P[: i + 1], Q) for i in range(len(P))]
        self.modDownConstantsPtoQ = self._gen_moddown(ringQ, ringP)
        self.modDownConstantsQtoP = self._gen_moddown(ringP, ringQ)

    @staticmethod
    def _gen_moddown(ringQ: Ring, ringP: Ring):
        """genmodDownConstants, ring/basis_extension.go:25-49: [j][i] = MForm((p_0..p_j)^-1 mod q_i)."""
        out = []
        acc = 1
        for pj in ringP.ModuliChain():
            acc *= pj
            out.append([mform(pow(acc % qi, -1, qi), qi) for qi in ringQ.ModuliChain()])
        return out

    def ModUpQtoP(self, levelQ, levelP, polQ, polP):      # :177-190
        ringQ, ringP = self.ringQ.AtLevel(levelQ), self.ringP.AtLevel(levelP)
        buffQ = np.empty((levelQ + 1, ringQ.N()), dtype=U64)
        QHalf = ringQ.ModulusAtLevel[levelQ] >> 1
        ringQ.AddScalarBigint(polQ, QHalf, buffQ)
        mod_up_exact(buffQ[: levelQ + 1], polP[: levelP + 1], self.ringQ, self.ringP, self.constantsQtoP[levelQ])
        ringP.SubScalarBigint(polP, QHalf, polP)

    def ModUpPtoQ(self, levelP, levelQ, polP, polQ):      # :195-209
        ringQ, ringP = self.ringQ.AtLevel(levelQ), self.ringP.AtLevel(levelP)
        buffP = np.empty((levelP + 1, ringP.N()), dtype=U64)
        PHalf = ringP.ModulusAtLevel[levelP] >> 1
        ringP.AddScalarBigint(polP, PHalf, buffP)
        mod_up_exact(buffP[: levelP + 1], polQ[: levelQ + 1], self.ringP, self.ringQ, self.constantsPtoQ[levelP])
        ringQ.SubScalarBigint(polQ, PHalf, polQ)

    def ModDownQPtoQ(self, levelQ, levelP, p1Q, p1P, p2Q):      # :215-228
        ringQ = self.ringQ.AtLevel(levelQ)
        mdc = self.modDownConstantsPtoQ[levelP]
        buffQ = np.empty((levelQ + 1, ringQ.N()), dtype=U64)
        self.ModUpPtoQ(levelP, levelQ, p1P, buffQ)
        for i, s in enumerate(ringQ.SubRings[: levelQ + 1]):
            s.vecop("SubThenMulScalarMontgomeryTwoModulus", buffQ[i], p1Q[i], p2Q[i], s.Modulus - mdc[i])

    def ModDownQPtoQNTT(self, levelQ, levelP, p1Q, p1P, p2Q):   # :235-256
        ringQ, ringP = self.ringQ.AtLevel(levelQ), self.ringP.AtLevel(levelP)
        mdc = self.modDownConstantsPtoQ[levelP]
        buffP = np.empty((levelP + 1, ringQ.N()), dtype=U64)
        buffQ = np.empty((levelQ + 1, ringQ.N()), dtype=U64)
        ringP.INTTLazy(p1P, buffP)
        self.ModUpPtoQ(levelP, levelQ, buffP, buffQ)
        ringQ.NTTLazy(buffQ, buffQ)
        for i, s in enumerate(ringQ.SubRings[: levelQ + 1]):
            s.vecop("SubThenMulScalarMontgomeryTwoModulus", buffQ[i], p1Q[i], p2Q[i], s.Modulus - mdc[i])

    def ModDownQPtoP(self, levelQ, levelP, p1Q, p1P, p2P):      # :262-278
        ringP = self.ringP.AtLevel(levelP)
        mdc = self.modDownConstantsQtoP[levelQ]
        buffP = np.empty((levelP + 1, ringP.N()), dtype=U64)
        self.ModUpQtoP(levelQ, levelP, p1Q, buffP)
        for i, s in enumerate(ringP.SubRings[: levelP + 1]):
            s.vecop("SubThenMulScalarMontgomeryTwoModulus", buffP[i], p1P[i], p2P[i], s.Modulus - mdc[i])


class Decomposer:
    """ring/basis_extension.go:313-377 (NewDecomposer) and :381-502 (DecomposeAndSplit)."""

    def __init__(self, ringQ: Ring, ringP: Optional[Ring]):
        self.ringQ, self.ringP = ringQ, ringP
        self.ModUpConstants = []
        self._cache = {}

    def _muc(self, nbPi, digit, decompLvl) -> ModUpConstants:
        """Lazily builds ModUpConstants[nbPi-2][digit][decompLvl] (:333-373): source = Q[digit*nbPi : +decompLvl+2],
        target = all of Q (full chain) followed by P[:nbPi]."""
        key = (nbPi, digit, decompLvl)
        if key not in self._cache:
            Q = self.ringQ.ModuliChain(); P = self.ringP.ModuliChain()[:nbPi]
            Qi = Q[digit * nbPi: digit * nbPi + decompLvl + 2]
            self._cache[key] = ModUpConstants(Qi, Q + P)
        return self._cache[key]

    def DecomposeAndSplit(self, levelQ, levelP, nbPi, digit, p0Q, p1Q, p1P):
        ringQ = self.ringQ.AtLevel(levelQ)
        ringP = self.ringP.AtLevel(levelP) if self.ringP is not None else None
        N = ringQ.N()
        lvlQStart = digit * nbPi
        if levelQ > nbPi * (digit + 1) - 1:
            decompLvl = nbPi - 2
        else:
            decompLvl = (levelQ % nbPi) - 1
        Qc = ringQ.ModuliChain()
        if decompLvl < 0:
            # :402-436 single-limb digit: centre and reduce into every Q and P limb
            rows, T, brc = [], [], []
            for i in range(levelQ + 1):
                rows.append(p1Q[i]); T.append(Qc[i]); brc += ringQ.SubRings[i].BRedConstant
            if ringP is not None:
                for i in range(levelP + 1):
                    rows.append(p1P[i]); T.append(ringP.SubRings[i].Modulus); brc += ringP.SubRings[i].BRedConstant
            ptrs = (ctypes.c_void_p * len(rows))(*[r.ctypes.data for r in rows])
            Ta = np.array(T, dtype=U64); ba = np.array(brc, dtype=U64)
            lib().lo_decompose_single(_ptr(p0Q[lvlQStart]), Qc[lvlQStart], ptrs, len(rows), N, _ptr(Ta), _ptr(ba))
            return
        p0idxst = digit * nbPi
        p0idxed = min(p0idxst + nbPi, levelQ + 1)
        muc = self._muc(nbPi, digit, decompLvl)
        nQfull = self.ringQ.ModuliChainLength()
        QBig = 1
        for i in range(p0idxst, p0idxed): QBig *= Qc[i]
        QHalf = QBig >> 1
        nD = p0idxed - p0idxst
        assert nD == decompLvl + 2
        assert nD <= 64, "lo_decompose_reconstruct holds at most 64 source limbs"
        Qd = np.array(Qc[p0idxst:p0idxed], dtype=U64)
        mq = np.array([ringQ.SubRings[i].MRedConstant for i in range(p0idxst, p0idxed)], dtype=U64)
        qh = np.array([QHalf % Qc[i] for i in range(p0idxst, p0idxed)], dtype=U64)
        rows, T, mT, crow, vrow = [], [], [], [], []
        for j in list(range(0, p0idxst)) + list(range(p0idxed, levelQ + 1)):
            rows.append(p1Q[j]); T.append(Qc[j]); mT.append(ringQ.SubRings[j].MRedConstant)
            crow.append(muc.qoverqimodp[j]); vrow.append(muc.vtimesqmodp[j])
        for j in range(levelP + 1):
            u = nQfull + j
            rows.append(p1P[j]); T.append(ringP.SubRings[j].Modulus); mT.append(ringP.SubRings[j].MRedConstant)
            crow.append(muc.qoverqimodp[u]); vrow.append(muc.vtimesqmodp[u])
        nT = len(rows)
        src = np.ascontiguousarray(p0Q[p0idxst:p0idxed])
        P3 = ctypes.c_void_p * nT
        Ta, mTa = np.array(T, dtype=U64), np.array(mT, dtype=U64)      # keep alive across the call
        crow = [np.ascontiguousarray(c) for c in crow]; vrow = [np.ascontiguousarray(v) for v in vrow]
        lib().lo_decompose_reconstruct(src.ctypes.data, N, nD, P3(*[r.ctypes.data for r in rows]), nT, N,
                                       _ptr(Qd), _ptr(mq), _ptr(qh), _ptr(muc.qoverqiinvqi),
                                       _ptr(Ta), _ptr(mTa),
                                       P3(*[c.ctypes.data for c in crow]),
                                       P3(*[v.ctypes.data for v in vrow]))
        # :499-500 -- SubScalarBigint over ALL limbs of p1Q / p1P (the digit's own rows included; the
        # caller overwrites those afterwards in DecomposeSingleNTT).
        ringQ.SubScalarBigint(p1Q, QHalf, p1Q)
        ringP.SubScalarBigint(p1P, QHalf, p1P)


# --------------------------------------------------------------------------
# core/rlwe: parameters-lite, GadgetCiphertext layout, Evaluator (key-switch family)
# --------------------------------------------------------------------------
class GadgetCiphertext:
    """core/rlwe/gadgetciphertext.go:19-45. ``Value[digit][pw2][component]`` is a ringqp.Poly, always NTT +
    Montgomery. Stored here as one array of shape (digits, pw2, 2, nQ + nP, N): Q limbs first, then P limbs."""

    def __init__(self, data: np.ndarray, nQ: int, nP: int, base_two_decomposition: int = 0, pw2_sizes=None):
        self.data = data
        self.nQ, self.nP = nQ, nP
        self.BaseTwoDecomposition = base_two_decomposition
        # ragged second dimension of Value[digit][pw2] (only != 1 when BaseTwoDecomposition != 0)
        self.pw2_sizes = list(pw2_sizes) if pw2_sizes is not None else [data.shape[1]] * data.shape[0]

    def BaseTwoDecompositionVectorSize(self):   # core/rlwe/gadgetciphertext.go:67-73
        return self.pw2_sizes

    def LevelQ(self): return self.nQ - 1
    def LevelP(self): return self.nP - 1
    def Q(self, d, j, c): return self.data[d, j, c, : self.nQ]
    def P(self, d, j, c): return self.data[d, j, c, self.nQ:]


class Parameters:
    """The slice of core/rlwe/params.go the hot path needs."""

    def __init__(self, logN: int, Q: Sequence[int], P: Sequence[int], ring_type="Standard"):
        self.logN = logN
        self.qi = [int(x) for x in Q]; self.pi = [int(x) for x in P]
        self.ringQ = Ring(1 << logN, self.qi, ring_type)
        self.ringP = Ring(1 << logN, self.pi, ring_type) if len(P) else None

    def N(self): return 1 << self.logN
    def MaxLevelQ(self): return len(self.qi) - 1
    def MaxLevelP(self): return len(self.pi) - 1

    def BaseRNSDecompositionVectorSize(self, levelQ, levelP):   # core/rlwe/params.go:543-550
        if levelP == -1:
            return levelQ + 1
        return (levelQ + levelP + 1) // (levelP + 1)

    def BaseTwoDecompositionVectorSize(self, levelQ, levelP, pw2):   # core/rlwe/params.go:520-540
        logqi = [int(round(math.log2(float(q)))) for q in self.qi]    # LogQi, :474-481
        if pw2 == 0 or levelP > 0:
            return [1] * len(logqi)
        return [(l + pw2 - 1) // pw2 for l in logqi]

    def QiOverflowMargin(self, level):      # core/rlwe/params.go:554-559
        return int(math.pow(2.0, 64) / float(max(self.qi[: level + 1])))

    def PiOverflowMargin(self, level):      # core/rlwe/params.go:563-568
        return int(math.pow(2.0, 64) / float(max(self.pi[: level + 1])))

    def GaloisElement(self, k: int) -> int:   # core/rlwe/params.go:580-584 (GaloisGen = 5)
        nr = self.ringQ.NthRoot()
        return pow(5, k & (nr - 1), nr)

    def GaloisElementOrderTwoOrthogonalSubgroup(self) -> int:   # :592-597
        return self.ringQ.NthRoot() - 1


class Evaluator:
    """core/rlwe/evaluator.go:12-21, key-switch family only. Ciphertexts are lists [c0, c1] of (limbs, N) arrays."""

    def __init__(self, params: Parameters):
        self.params = params
        self.BasisExtender = BasisExtender(params.ringQ, params.ringP) if params.ringP is not None else None
        self.Decomposer = Decomposer(params.ringQ, params.ringP)

    # core/rlwe/evaluator_gadget_product.go:487-510
    def DecomposeSingleNTT(self, levelQ, levelP, nbPi, digit, c2NTT, c2InvNTT, c2QiQ, c2QiP):
        ringQ = self.params.ringQ.AtLevel(levelQ)
        self.Decomposer.DecomposeAndSplit(levelQ, levelP, nbPi, digit, c2InvNTT, c2QiQ, c2QiP)
        p0idxst = digit * nbPi
        p0idxed = p0idxst + nbPi
        for x in range(levelQ + 1):
            if p0idxst <= x < p0idxed:
                c2QiQ[x] = c2NTT[x]
            else:
                ringQ.SubRings[x].NTT(c2QiQ[x], c2QiQ[x])
        if self.params.ringP is not None:
            self.params.ringP.AtLevel(levelP).NTT(c2QiP, c2QiP)

    # core/rlwe/evaluator_gadget_product.go:459-483
    def DecomposeNTT(self, levelQ, levelP, nbPi, c2, c2IsNTT, decompQ: list, decompP: list):
        ringQ = self.params.ringQ.AtLevel(levelQ)
        buff = np.empty((levelQ + 1, ringQ.N()), dtype=U64)
        if c2IsNTT:
            polyNTT, polyInvNTT = c2, buff
            ringQ.INTT(polyNTT, polyInvNTT)
        else:
            polyNTT, polyInvNTT = buff, c2
            ringQ.NTT(polyInvNTT, polyNTT)
        for i in range(self.params.BaseRNSDecompositionVectorSize(levelQ, levelP)):
            self.DecomposeSingleNTT(levelQ, levelP, nbPi, i, polyNTT, polyInvNTT, decompQ[i], decompP[i])

    def _mac(self, first, ringQ, ringP, evk: GadgetCiphertext, d, j, cQ, cP, accQ, accP, levelQ, levelP):
        name = "MulCoeffsMontgomeryLazy" if first else "MulCoeffsMontgomeryLazyThenAddLazy"
        for comp in range(2):
            ringQ._op(name, evk.Q(d, j, comp), cQ, accQ[comp])
            if ringP is not None:
                ringP._op(name, evk.P(d, j, comp), cP, accP[comp])

    # core/rlwe/evaluator_gadget_product.go:129-201
    def gadgetProductMultiplePLazy(self, levelQ, cx, evk: GadgetCiphertext, accQ, accP, isNTT=True):
        levelP = evk.LevelP()
        ringQ = self.params.ringQ.AtLevel(levelQ); ringP = self.params.ringP.AtLevel(levelP)
        N = ringQ.N()
        c2Q = np.empty((levelQ + 1, N), dtype=U64); c2P = np.empty((levelP + 1, N), dtype=U64)
        buffQ = np.empty((levelQ + 1, N), dtype=U64)
        if isNTT:
            cxNTT, cxInv = cx, buffQ
            ringQ.INTT(cxNTT, cxInv)
        else:
            cxNTT, cxInv = buffQ, cx
            ringQ.NTT(cxInv, cxNTT)
        n = self.params.BaseRNSDecompositionVectorSize(levelQ, levelP)
        QiOverF = self.params.QiOverflowMargin(levelQ) >> 1
        PiOverF = self.params.PiOverflowMargin(levelP) >> 1
        reduce = 0
        for i in range(n):
            self.DecomposeSingleNTT(levelQ, levelP, levelP + 1, i, cxNTT, cxInv, c2Q, c2P)
            self._mac(i == 0, ringQ, ringP, evk, i, 0, c2Q, c2P, accQ, accP, levelQ, levelP)
            if reduce % QiOverF == QiOverF - 1:
                ringQ.Reduce(accQ[0], accQ[0]); ringQ.Reduce(accQ[1], accQ[1])
            if reduce % PiOverF == PiOverF - 1:
                ringP.Reduce(accP[0], accP[0]); ringP.Reduce(accP[1], accP[1])
            reduce += 1
        if reduce % QiOverF != 0:
            ringQ.Reduce(accQ[0], accQ[0]); ringQ.Reduce(accQ[1], accQ[1])
        if reduce % PiOverF != 0:
            ringP.Reduce(accP[0], accP[0]); ringP.Reduce(accP[1], accP[1])

    # core/rlwe/evaluator_gadget_product.go:203-338
    def gadgetProductSinglePAndBitDecompLazy(self, levelQ, cx, evk: GadgetCiphertext, accQ, accP, isNTT=True):
        levelP = evk.LevelP()
        ringQ = self.params.ringQ.AtLevel(levelQ)
        ringP = self.params.ringP.AtLevel(levelP) if levelP >= 0 else None
        N = ringQ.N()
        if isNTT:
            cxInv = np.empty((levelQ + 1, N), dtype=U64)
            ringQ.INTT(cx, cxInv)
        else:
            cxInv = cx
        pw2 = evk.BaseTwoDecomposition
        nRNS = levelQ + 1
        nPw2 = evk.BaseTwoDecompositionVectorSize()
        mask = (1 << pw2) - 1
        c2Q = np.empty((levelQ + 1, N), dtype=U64)
        c2P = np.empty((max(levelP + 1, 1), N), dtype=U64)
        cw = np.empty(N, dtype=U64); cwNTT = np.empty(N, dtype=U64)
        QiOverF = self.params.QiOverflowMargin(levelQ) >> 1
        PiOverF = (self.params.PiOverflowMargin(levelP) >> 1) if ringP is not None else 1
        reduce = 0
        for i in range(nRNS):
            if mask == 0:
                self.Decomposer.DecomposeAndSplit(levelQ, levelP, levelP + 1, i, cxInv, c2Q, c2P)
            for j in range(nPw2[i]):
                if mask != 0:
                    ringQ.SubRings[0].vecop("Mask", cxInv[i], None, cw, j * pw2, mask)
                first = (i == 0 and j == 0)
                name = "MulCoeffsMontgomeryLazy" if first else "MulCoeffsMontgomeryLazyThenAddLazy"
                for u, s in enumerate(ringQ.SubRings[: levelQ + 1]):
                    s.NTTLazy(c2Q[u] if mask == 0 else cw, cwNTT)
                    s.vecop(name, evk.Q(i, j, 0)[u], cwNTT, accQ[0][u])
                    s.vecop(name, evk.Q(i, j, 1)[u], cwNTT, accQ[1][u])
                if ringP is not None:
                    for u, s in enumerate(ringP.SubRings[: levelP + 1]):
                        s.NTTLazy(c2P[u] if mask == 0 else cw, cwNTT)
                        s.vecop(name, evk.P(i, j, 0)[u], cwNTT, accP[0][u])
                        s.vecop(name, evk.P(i, j, 1)[u], cwNTT, accP[1][u])
                if reduce % QiOverF == QiOverF - 1:
                    ringQ.Reduce(accQ[0], accQ[0]); ringQ.Reduce(accQ[1], accQ[1])
                if ringP is not None and reduce % PiOverF == PiOverF - 1:
                    ringP.Reduce(accP[0], accP[0]); ringP.Reduce(accP[1], accP[1])
                reduce += 1
        if reduce % QiOverF != 0:
            ringQ.Reduce(accQ[0], accQ[0]); ringQ.Reduce(accQ[1], accQ[1])
        if ringP is not None and reduce % PiOverF != 0:
            ringP.Reduce(accP[0], accP[0]); ringP.Reduce(accP[1], accP[1])

    # core/rlwe/evaluator_gadget_product.go:108-127
    def GadgetProductLazy(self, levelQ, cx, evk: GadgetCiphertext, accQ, accP, isNTT=True):
        if evk.LevelP() > 0:
            self.gadgetProductMultiplePLazy(levelQ, cx, evk, accQ, accP, isNTT)
        else:
            self.gadgetProductSinglePAndBitDecompLazy(levelQ, cx, evk, accQ, accP, isNTT)
        if not isNTT:
            ringQ = self.params.ringQ.AtLevel(levelQ)
            for c in range(2):
                ringQ.INTT(accQ[c], accQ[c])
                if evk.LevelP() >= 0:
                    self.params.ringP.AtLevel(evk.LevelP()).INTT(accP[c], accP[c])

    # core/rlwe/evaluator_gadget_product.go:39-97
    def ModDown(self, levelQ, levelP, accQ, accP, ct, ctQP_isNTT=True, ct_isNTT=True):
        ringQ = self.params.ringQ.AtLevel(levelQ)
        if levelP != -1:
            be = self.BasisExtender
            ringP = self.params.ringP.AtLevel(levelP)
            if ctQP_isNTT and ct_isNTT:
                for c in range(2): be.ModDownQPtoQNTT(levelQ, levelP, accQ[c], accP[c], ct[c])
            elif ctQP_isNTT and not ct_isNTT:
                for c in range(2):
                    ringQ.INTTLazy(accQ[c], accQ[c]); ringP.INTTLazy(accP[c], accP[c])
                for c in range(2): be.ModDownQPtoQ(levelQ, levelP, accQ[c], accP[c], ct[c])
            elif (not ctQP_isNTT) and ct_isNTT:
                for c in range(2): be.ModDownQPtoQ(levelQ, levelP, accQ[c], accP[c], ct[c])
                for c in range(2): ringQ.NTT(ct[c], ct[c])
            else:
                for c in range(2): be.ModDownQPtoQ(levelQ, levelP, accQ[c], accP[c], ct[c])
        else:
            for c in range(2):
                if ctQP_isNTT == ct_isNTT:
                    ct[c][: levelQ + 1] = accQ[c][: levelQ + 1]
                elif ctQP_isNTT:
                    ringQ.INTT(accQ[c], ct[c])
                else:
                    ringQ.NTT(accQ[c], ct[c])

    # core/rlwe/evaluator_gadget_product.go:16-36
    def GadgetProduct(self, levelQ, cx, evk: GadgetCiphertext, ct, isNTT=True):
        levelQ = min(levelQ, evk.LevelQ())
        levelP = evk.LevelP()
        N = self.params.N()
        accP = [np.empty((max(levelP + 1, 1), N), dtype=U64) for _ in range(2)]
        # ctTmp.Value[c].Q aliases ct.Value[c] in the reference (:27)
        self.GadgetProductLazy(levelQ, cx, evk, ct, accP, isNTT)
        self.ModDown(levelQ, levelP, ct, accP, ct, isNTT, isNTT)

    # core/rlwe/evaluator_gadget_product.go:401-453 + :348-399
    def GadgetProductHoistedLazy(self, levelQ, decompQ, decompP, evk: GadgetCiphertext, accQ, accP):
        levelP = evk.LevelP()
        ringQ = self.params.ringQ.AtLevel(levelQ); ringP = self.params.ringP.AtLevel(levelP)
        n = self.params.BaseRNSDecompositionVectorSize(levelQ, levelP)
        QiOverF = self.params.QiOverflowMargin(levelQ) >> 1
        PiOverF = self.params.PiOverflowMargin(levelP) >> 1
        reduce = 0
        for i in range(n):
            self._mac(i == 0, ringQ, ringP, evk, i, 0, decompQ[i], decompP[i], accQ, accP, levelQ, levelP)
            if reduce % QiOverF == QiOverF - 1:
                ringQ.Reduce(accQ[0], accQ[0]); ringQ.Reduce(accQ[1], accQ[1])
            if reduce % PiOverF == PiOverF - 1:
                ringP.Reduce(accP[0], accP[0]); ringP.Reduce(accP[1], accP[1])
            reduce += 1
        if reduce % QiOverF != 0:
            ringQ.Reduce(accQ[0], accQ[0]); ringQ.Reduce(accQ[1], accQ[1])
        if reduce % PiOverF != 0:
            ringP.Reduce(accP[0], accP[0]); ringP.Reduce(accP[1], accP[1])

    def GadgetProductHoisted(self, levelQ, decompQ, decompP, evk: GadgetCiphertext, ct):
        levelP = evk.LevelP()
        accP = [np.empty((levelP + 1, self.params.N()), dtype=U64) for _ in range(2)]
        self.GadgetProductHoistedLazy(levelQ, decompQ, decompP, evk, ct, accP)
        self.ModDown(levelQ, levelP, ct, accP, ct)

    # core/rlwe/evaluator_automorphism.go:13-57 (NTT-domain ciphertexts)
    def Automorphism(self, ctIn, galEl, evk: GadgetCiphertext, opOut, level=None):
        level = min(ctIn[0].shape[0], opOut[0].shape[0]) - 1 if level is None else level
        ringQ = self.params.ringQ.AtLevel(level)
        N = ringQ.N()
        tmp = [np.empty((level + 1, N), dtype=U64) for _ in range(2)]
        self.GadgetProduct(level, ctIn[1], evk, tmp)
        ringQ.Add(tmp[0], ctIn[0], tmp[0])
        index = ringQ.AutomorphismNTTIndex(galEl)
        ringQ.AutomorphismNTTWithIndex(tmp[0], index, opOut[0])
        ringQ.AutomorphismNTTWithIndex(tmp[1], index, opOut[1])

    # core/rlwe/evaluator_automorphism.go:63-102
    def AutomorphismHoisted(self, level, ctIn, decompQ, decompP, galEl, evk: GadgetCiphertext, ctOut):
        ringQ = self.params.ringQ.AtLevel(level)
        N = ringQ.N()
        tmp = [np.empty((level + 1, N), dtype=U64) for _ in range(2)]
        self.GadgetProductHoisted(level, decompQ, decompP, evk, tmp)
        ringQ.Add(tmp[0], ctIn[0], tmp[0])
        index = ringQ.AutomorphismNTTIndex(galEl)
        ringQ.AutomorphismNTTWithIndex(tmp[0], index, ctOut[0])
        ringQ.AutomorphismNTTWithIndex(tmp[1], index, ctOut[1])

    # core/rlwe/evaluator_automorphism.go:107-165 (ctQP.IsNTT branch): result modulo QP, scaled by P.
    # ctQP = ([Q0, Q1], [P0, P1]) pre-allocated (levelQ+1 / levelP+1 rows).
    def AutomorphismHoistedLazy(self, levelQ, ctIn, decompQ, decompP, galEl, evk: GadgetCiphertext, ctQP_Q, ctQP_P):
        levelP = evk.LevelP()
        ringQ = self.params.ringQ.AtLevel(levelQ); ringP = self.params.ringP.AtLevel(levelP)
        N = ringQ.N()
        tQ = [np.empty((levelQ + 1, N), dtype=U64) for _ in range(2)]
        tP = [np.empty((levelP + 1, N), dtype=U64) for _ in range(2)]
        self.GadgetProductHoistedLazy(levelQ, decompQ, decompP, evk, tQ, tP)
        index = ringQ.AutomorphismNTTIndex(galEl)
        ringQ.AutomorphismNTTWithIndex(tQ[1], index, ctQP_Q[1]); ringP.AutomorphismNTTWithIndex(tP[1], index, ctQP_P[1])
        if levelP > -1:
            ringQ.MulScalarBigint(ctIn[0], ringP.ModulusAtLevel[levelP], tQ[1])
        ringQ.Add(tQ[0], tQ[1], tQ[0])
        ringQ.AutomorphismNTTWithIndex(tQ[0], index, ctQP_Q[0]); ringP.AutomorphismNTTWithIndex(tP[0], index, ctQP_P[0])

    # core/rlwe/evaluator_evaluationkey.go:121-148
    def Relinearize(self, ctIn, rlk: GadgetCiphertext, opOut):
        level = min(ctIn[0].shape[0], opOut[0].shape[0]) - 1
        ringQ = self.params.ringQ.AtLevel(level)
        N = ringQ.N()
        tmp = [np.empty((level + 1, N), dtype=U64) for _ in range(2)]
        self.GadgetProduct(level, ctIn[2], rlk, tmp)
        ringQ.Add(ctIn[0], tmp[0], opOut[0])
        ringQ.Add(ctIn[1], tmp[1], opOut[1])


# --------------------------------------------------------------------------
# schemes/ckks: the measured op sequences
# --------------------------------------------------------------------------
class CKKSEvaluator(Evaluator):
    def __init__(self, params: Parameters, rlk: Optional[GadgetCiphertext] = None, levels_per_rescale: int = 1):
        super().__init__(params)
        self.rlk = rlk
        self.nbRescales = levels_per_rescale

    def MulRelinNew(self, op0, op1):
        """schemes/ckks/evaluator.go:719-872, ciphertext x ciphertext (degree 1 x 1), relin=True."""
        level = min(op0[0].shape[0], op1[0].shape[0]) - 1
        ringQ = self.params.ringQ.AtLevel(level)
        N = ringQ.N()
        mk = lambda: np.empty((level + 1, N), dtype=U64)
        c00, c01, c0, c1, c2 = mk(), mk(), mk(), mk(), mk()
        ringQ.MForm(op0[0], c00)
        ringQ.MForm(op0[1], c01)
        ringQ.MulCoeffsMontgomery(c00, op1[0], c0)
        ringQ.MulCoeffsMontgomery(c01, op1[1], c2)
        ringQ.MulCoeffsMontgomery(c00, op1[1], c1)
        ringQ.MulCoeffsMontgomeryThenAdd(c01, op1[0], c1)
        tmp = [mk(), mk()]
        self.GadgetProduct(level, c2, self.rlk, tmp)
        out = [mk(), mk()]
        ringQ.Add(c0, tmp[0], out[0])
        ringQ.Add(c1, tmp[1], out[1])
        return out

    def Rescale(self, op0):
        """schemes/ckks/evaluator.go:477-515"""
        level = op0[0].shape[0] - 1
        nb = self.nbRescales
        assert level > nb - 1
        ringQ = self.params.ringQ.AtLevel(level)
        out = [np.empty((level + 1 - nb, ringQ.N()), dtype=U64) for _ in op0]
        for i in range(len(op0)):
            ringQ.DivRoundByLastModulusManyNTT(nb, op0[i], None, out[i])
        return out


# --------------------------------------------------------------------------
# prime generation: ring/primes.go:24-229 + core/rlwe/params.go:811-862
# --------------------------------------------------------------------------
class NTTFriendlyPrimesGenerator:
    def __init__(self, bit_size: int, nthroot: int):
        self.Size = float(bit_size)
        self.NthRoot = nthroot
        self.NextPrime = (1 << bit_size) + 1
        self.PrevPrime = (1 << bit_size) + 1
        self.CheckNextPrime = not (self.NextPrime > 0xFFFFFFFFFFFFFFFF - nthroot)
        self.CheckPrevPrime = not (self.PrevPrime < nthroot)
        self.PrevPrime -= nthroot

    def NextDownstreamPrime(self):      # ring/primes.go:126-156
        p = self.PrevPrime
        while True:
            if not self.CheckPrevPrime:
                raise RuntimeError("downstream primes exhausted")
            if self.Size - math.log2(float(p)) >= 0.5 or p < self.NthRoot:
                self.CheckPrevPrime = False
                raise RuntimeError("downstream primes exhausted")
            if is_prime(p):
                self.PrevPrime = p - self.NthRoot
                return p
            p -= self.NthRoot

    def NextAlternatingPrime(self):     # ring/primes.go:159-229
        nxt, prv = self.NextPrime, self.PrevPrime
        cn, cp = self.CheckNextPrime, self.CheckPrevPrime
        while True:
            if not (cn or cp):
                raise RuntimeError("alternating primes exhausted")
            if cn:
                if math.log2(float(nxt)) - self.Size >= 0.5 or nxt > 0xFFFFFFFFFFFFFFFF - self.NthRoot:
                    cn = False
                else:
                    if is_prime(nxt):
                        self.NextPrime, self.PrevPrime = nxt + self.NthRoot, prv
                        self.CheckNextPrime, self.CheckPrevPrime = cn, cp
                        return nxt
                    nxt += self.NthRoot
            if cp:
                if self.Size - math.log2(float(prv)) >= 0.5 or prv < self.NthRoot:
                    cp = False
                else:
                    if is_prime(prv):
                        self.NextPrime, self.PrevPrime = nxt, prv - self.NthRoot
                        self.CheckNextPrime, self.CheckPrevPrime = cn, cp
                        return prv
                    prv -= self.NthRoot


def gen_moduli(log_nthroot: int, logQ: Sequence[int], logP: Sequence[int]):
    """GenModuli, core/rlwe/params.go:811-862."""
    count = {}
    for b in list(logQ) + list(logP):
        count[b] = count.get(b, 0) + 1
    primes = {}
    for b, n in count.items():
        g = NTTFriendlyPrimesGenerator(b, 1 << log_nthroot)
        primes[b] = [g.NextDownstreamPrime() if b == 61 else g.NextAlternatingPrime() for _ in range(n)]
    q = [primes[b].pop(0) for b in logQ]
    p = [primes[b].pop(0) for b in logP]
    return q, p

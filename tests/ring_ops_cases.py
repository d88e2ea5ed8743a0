"""Cases and an exact reference for the ring-level kernels: the coefficient-wise opcodes (csrc/vecops.cu), the
automorphisms (csrc/composite.cu) and the coefficient-moving kernels (csrc/ringmisc.cu).

The reference here is the plain mathematical definition in Python integers, written without the oracle's C
restatement, so that a mistake shared by the oracle and a kernel still shows. Where the upstream code returns a
literal word (a negated 0 is q, a lazy sum is the raw sum) the reference gives that word; where only the residue is
defined (the lazy Montgomery and Barrett products) it gives the residue and the range the word must lie in.

It also restates the host launch choice of launch_vecop / launch_one, and lists the GPU cases that reach every
launch-shape cell (tests/test_ring_ops_model_cpu.py checks that the list reaches them all and that none is spare)."""
import functools

import numpy as np

from oracle import oracle as O
from tests import helpers as H

U64 = np.uint64
M64 = (1 << 64) - 1
R64 = 1 << 64
LOG_NS = list(range(4, 18))

# ---------------------------------------------------------------------------------------------------------------
# Prime classes
# ---------------------------------------------------------------------------------------------------------------
REAL_SMALL = {0x3001: 11, 0x10001: 15, 0x7fff801: 10}       # LWE ring, BGV plaintext ring, blind-rotation ring: largest logN
CLASSES = ["real", "smallest", "b33", "b45", "b50", "b55", "b61"]


def ntt_primes(bits, m, count, skip=()):
    """`count` primes that are 1 mod m, going down from 2^bits (NTT-friendly for NthRoot m)."""
    out, k = [], ((1 << bits) - 1) // m
    while len(out) < count:
        p = k * m + 1
        if p not in skip and p < (1 << bits) and O.is_prime(p):
            out.append(p)
        k -= 1
    return out


def smallest_primes(m, count, skip=()):
    out, k = [], 1
    while len(out) < count:
        p = k * m + 1
        if p not in skip and O.is_prime(p):
            out.append(p)
        k += 1
    return out


def class_primes(logN, ci=False):
    """{class: ([primes for ringQ], [primes for ringP])} at ring degree 2^logN; NthRoot is 2N, or 4N on the
    conjugate-invariant ring. The real small primes that fit are dealt to ringP first and then to ringQ, so that
    each ring gets one where two fit (only one of each exists)."""
    m = (4 if ci else 2) << logN
    real = [p for p, lg in sorted(REAL_SMALL.items(), key=lambda t: t[1]) if (p - 1) % m == 0 and logN <= lg]
    out = {}
    if real:
        out["real"] = (real[1:] if len(real) > 1 else real, real[:1] if len(real) > 1 else [])
    small = smallest_primes(m, 2, skip=real)
    out["smallest"] = ([small[0]], [small[1]])
    for name, (bq, bp) in {"b33": (33, 36), "b45": (45, 45), "b50": (50, 50), "b55": (55, 56)}.items():
        if bq == bp:
            a, b = ntt_primes(bq, m, 2)
        else:
            a, b = ntt_primes(bq, m, 1)[0], ntt_primes(bp, m, 1)[0]
        out[name] = ([a], [b])
    out["b61"] = ([[q for q in H.Qi60 if (q - 1) % m == 0][0]], [[p for p in H.Pi60 if (p - 1) % m == 0][0]])
    return out


def chain(logN, ci=False):
    """(Q, P, class of every Q row, class of every P row): every prime class on both rings where its primes fit."""
    Q, P, cq, cpl = [], [], [], []
    for c, (qs, ps) in class_primes(logN, ci).items():
        Q += qs; cq += [c] * len(qs)
        P += ps; cpl += [c] * len(ps)
    return Q, P, cq, cpl


# ---------------------------------------------------------------------------------------------------------------
# Opcode domain table
# ---------------------------------------------------------------------------------------------------------------
# Input bounds: "q" = canonical [0, q), "2q" = [0, 2q), "4q" = [0, 4q), "any" = any uint64, "-" = not read.
# Output: ("word", f) - the reference returns exactly the word f(...);
#         ("res", f, lo, hi) - only the residue f(...) mod q is defined, and the word lies in [lo(q, z), hi(q, z)].
# Montgomery products are x*y/2^64 mod q; MRed needs x*y < q*2^64, which a canonical factor guarantees; BRed takes any
# 64-bit factors; CRed takes [0, 2q). These follow the doc comments of ring/modular_reduction.go and the callers of
# ring/vec_ops.go (lazy sums come from NTT outputs and MulCoeffs*Lazy, hence [0, 2q) / [0, 4q)).


@functools.lru_cache(maxsize=None)
def _ri(q):
    return pow(R64, -1, q)


def _mont(x, y, q):
    return x * y * _ri(q) % q


LAZY2 = lambda q, z: (0, 2 * q - 1)

# name: (p1, p2, p3, scalar domain, output)
OPDOM = {
    "Add": ("q", "q", "-", "-", ("word", lambda x, y, z, s0, s1, q: (x + y) % q)),
    "AddLazy": ("2q", "2q", "-", "-", ("word", lambda x, y, z, s0, s1, q: x + y)),
    "Sub": ("q", "q", "-", "-", ("word", lambda x, y, z, s0, s1, q: (x - y) % q)),
    "SubLazy": ("q", "q", "-", "-", ("word", lambda x, y, z, s0, s1, q: x + q - y)),
    "Neg": ("q", "-", "-", "-", ("word", lambda x, y, z, s0, s1, q: q - x)),
    "Reduce": ("any", "-", "-", "-", ("word", lambda x, y, z, s0, s1, q: x % q)),
    "ReduceLazy": ("any", "-", "-", "-", ("res", lambda x, y, z, s0, s1, q: x % q, LAZY2)),
    "MulCoeffsLazy": ("any", "any", "-", "-", ("word", lambda x, y, z, s0, s1, q: x * y & M64)),
    "MulCoeffsLazyThenAddLazy": ("any", "any", "any", "-", ("word", lambda x, y, z, s0, s1, q: (z + x * y) & M64)),
    "MulCoeffsBarrett": ("any", "any", "-", "-", ("word", lambda x, y, z, s0, s1, q: x * y % q)),
    "MulCoeffsBarrettLazy": ("any", "any", "-", "-", ("res", lambda x, y, z, s0, s1, q: x * y % q, LAZY2)),
    "MulCoeffsBarrettThenAdd": ("any", "any", "q", "-", ("word", lambda x, y, z, s0, s1, q: (z + x * y) % q)),
    "MulCoeffsBarrettThenAddLazy": ("any", "any", "4q", "-", ("word", lambda x, y, z, s0, s1, q: z + x * y % q)),
    "MulCoeffsMontgomery": ("q", "any", "-", "-", ("word", lambda x, y, z, s0, s1, q: _mont(x, y, q))),
    "MulCoeffsMontgomeryLazy": ("q", "any", "-", "-", ("res", lambda x, y, z, s0, s1, q: _mont(x, y, q), LAZY2)),
    "MulCoeffsMontgomeryThenAdd": ("q", "any", "q", "-", ("word", lambda x, y, z, s0, s1, q: (z + _mont(x, y, q)) % q)),
    "MulCoeffsMontgomeryThenAddLazy": ("q", "any", "4q", "-", ("word", lambda x, y, z, s0, s1, q: z + _mont(x, y, q))),
    "MulCoeffsMontgomeryLazyThenAddLazy": ("q", "any", "4q", "-",
                                           ("res", lambda x, y, z, s0, s1, q: (z + _mont(x, y, q)) % q, lambda q, z: (z, z + 2 * q - 1))),
    "MulCoeffsMontgomeryThenSub": ("q", "any", "q", "-", ("word", lambda x, y, z, s0, s1, q: (z - _mont(x, y, q)) % q)),
    "MulCoeffsMontgomeryThenSubLazy": ("q", "any", "4q", "-", ("word", lambda x, y, z, s0, s1, q: z + q - _mont(x, y, q))),
    "MulCoeffsMontgomeryLazyThenSubLazy": ("q", "any", "4q", "-",
                                           ("res", lambda x, y, z, s0, s1, q: (z - _mont(x, y, q)) % q, lambda q, z: (z + 1, z + 2 * q))),
    "MulCoeffsMontgomeryLazyThenNeg": ("q", "any", "-", "-", ("res", lambda x, y, z, s0, s1, q: -_mont(x, y, q) % q, lambda q, z: (1, 2 * q))),
    "AddLazyThenMulScalarMontgomery": ("2q", "2q", "-", "q", ("word", lambda x, y, z, s0, s1, q: _mont(x + y, s0, q))),
    "AddScalarLazyThenMulScalarMontgomery": ("2q", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: _mont(x + s0, s1, q))),
    "AddScalar": ("q", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: (x + s0) % q)),
    "AddScalarLazy": ("2q", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: x + s0)),
    "AddScalarLazyThenNegTwoModulusLazy": ("2q", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: s0 + 2 * q - x)),
    "SubScalar": ("q", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: (x - s0) % q)),
    "MulScalarMontgomery": ("any", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: _mont(x, s0, q))),
    "MulScalarMontgomeryLazy": ("any", "-", "-", "q", ("res", lambda x, y, z, s0, s1, q: _mont(x, s0, q), LAZY2)),
    "MulScalarMontgomeryThenAdd": ("any", "-", "q", "q", ("word", lambda x, y, z, s0, s1, q: (z + _mont(x, s0, q)) % q)),
    "MulScalarMontgomeryThenAddScalar": ("any", "-", "-", "q", ("word", lambda x, y, z, s0, s1, q: (_mont(x, s1, q) + s0) % q)),
    "SubThenMulScalarMontgomeryTwoModulus": ("2q", "2q", "-", "q", ("word", lambda x, y, z, s0, s1, q: _mont(x - y, s0, q))),
    "MForm": ("any", "-", "-", "-", ("word", lambda x, y, z, s0, s1, q: (x << 64) % q)),
    "MFormLazy": ("any", "-", "-", "-", ("res", lambda x, y, z, s0, s1, q: (x << 64) % q, LAZY2)),
    "IMForm": ("any", "-", "-", "-", ("word", lambda x, y, z, s0, s1, q: x * _ri(q) % q)),
    "Zero": ("-", "-", "-", "-", ("word", lambda x, y, z, s0, s1, q: 0)),
    "Mask": ("any", "-", "-", "mask", ("word", lambda x, y, z, s0, s1, q: (x >> s0) & s1)),
}
assert list(OPDOM) == O.OPS


def bound(dom, q):
    """Exclusive upper bound of an input domain."""
    return {"q": q, "2q": 2 * q, "4q": 4 * q, "any": R64}[dom]


def edge_words(dom, q):
    """0, 1, q-1, q, 2q-1, 2q, 4q-1, 2^63, 2^64-1, kept to the domain."""
    b = bound(dom, q)
    return sorted({w for w in (0, 1, q - 1, q, 2 * q - 1, 2 * q, 4 * q - 1, 1 << 63, M64) if w < b})


def edge_scalars(dom, q):
    """(s0, s1) pairs: 0, 1, q-1 and their Montgomery forms; for Mask, shifts 0 and 63 with the all-ones mask (the RGSW
    path's raw-limb digit) and a 16-bit mask."""
    if dom == "mask":
        return [(0, M64), (63, M64), (0, 0xFFFF), (7, 0xFFFF)]
    if dom == "-":
        return [(0, 0)]
    s = sorted({0, 1, q - 1, (1 << 64) % q, ((q - 1) << 64) % q})
    return [(a, b) for a in s for b in s]


def exact(name, x, y, z, s0, s1, q):
    """(kind, value, lo, hi): the reference's word ("word") or residue ("res") of one opcode at one coefficient."""
    out = OPDOM[name][4]
    v = out[1](x, y, z, s0, s1, q)
    if out[0] == "word":
        return "word", v, v, v
    lo, hi = out[2](q, z)
    return "res", v % q, lo, hi


def check_exact(name, x, y, z, s0, s1, q, got):
    """None if the word `got` is what the reference defines, else a description of the mismatch."""
    kind, v, lo, hi = exact(name, x, y, z, s0, s1, q)
    if kind == "word":
        return None if got == v else "word %d != %d" % (got, v)
    if not (lo <= got <= hi):
        return "word %d outside [%d, %d]" % (got, lo, hi)
    return None if got % q == v else "residue %d != %d" % (got % q, v)


def random_in(dom, q, shape, rng):
    if dom == "any":
        return rng.integers(0, 1 << 64, shape, dtype=U64, endpoint=False)
    return rng.integers(0, bound(dom, q), shape, dtype=U64)


# ---------------------------------------------------------------------------------------------------------------
# Exact reference of the coefficient-moving maps (plain index arithmetic, literal negation words)
# ---------------------------------------------------------------------------------------------------------------
def monomial_exact(row, k, q):
    """row * X^k in Z_q[X]/(X^N + 1), with the reference's literal words: a coefficient carried across X^N once comes out
    as q - v (so 0 becomes q); one carried twice is v again."""
    N = len(row)
    out = [None] * N
    for j in range(N):
        e = (j + k) % (2 * N)
        v = int(row[j])
        if e < N:
            out[e] = v
        else:
            out[e - N] = q - v
    return out


def monomial_exact_np(rows, k, qs):
    N = rows.shape[-1]
    j = np.arange(N)
    e = (j + (k % (2 * N))) % (2 * N)
    out = np.empty_like(rows)
    for i, q in enumerate(qs):
        pos = e < N
        out[..., i, e[pos]] = rows[..., i, j[pos]]
        out[..., i, e[~pos] - N] = U64(q) - rows[..., i, j[~pos]]
    return out


def shift_exact_np(rows, k):
    N = rows.shape[-1]
    src = (np.arange(N) + k) % N
    return rows[..., src]


def automorphism_exact(row, g, q, ci=False):
    """X -> X^g on one row. Standard ring Z_q[X]/(X^N+1): X^i goes to +-X^(ig mod N), negative when ig mod 2N >= N.
    Conjugate-invariant ring: the row a_0..a_{N-1} stands for the element of Z_q[X]/(X^2N+1) with c_i = a_i and
    c_{2N-i} = -a_i; its image is read back on 0..N-1."""
    N = len(row)
    out = [None] * N
    if not ci:
        for i in range(N):
            e = i * g % (2 * N)
            v = int(row[i])
            if e < N:
                out[e] = v
            else:
                out[e - N] = q - v
        return out
    M = 2 * N
    for i in range(M):
        if i == N:
            continue                                   # c_N = 0 (it would be its own negation)
        if i < N:
            v, neg = int(row[i]), False
        else:
            v, neg = int(row[M - i]), True
        e = i * g % (2 * M)
        if e >= M:
            e -= M
            neg = not neg
        if e < N:
            out[e] = q - v if neg else v
    return out


def automorphism_exact_np(rows, g, qs, ci=False):
    """Vectorised form of automorphism_exact (same index and sign, numpy index arithmetic)."""
    N = rows.shape[-1]
    out = np.empty_like(rows)
    if not ci:
        i = np.arange(N, dtype=np.int64)
        e = (i * (g % (2 * N))) % (2 * N)
        neg = e >= N
        dst = np.where(neg, e - N, e)
        for r, q in enumerate(qs):
            v = rows[..., r, :]
            out[..., r, dst] = np.where(neg, U64(q) - v, v)
        return out
    M = 2 * N
    i = np.array([x for x in range(M) if x != N], dtype=np.int64)
    src = np.where(i < N, i, M - i)
    neg = i >= N
    e = (i * (g % (2 * M))) % (2 * M)
    neg = neg ^ (e >= M)
    e = np.where(e >= M, e - M, e)
    keep = e < N
    for r, q in enumerate(qs):
        v = rows[..., r, :][..., src[keep]]
        out[..., r, e[keep]] = np.where(neg[keep], U64(q) - v, v)
    return out


def ntt_slot_exponents(N, nthroot):
    """Exponent of the evaluation point psi^e at each NTT slot (ring/ntt.go's bit-reversed order): e_j = 2*brev(j) + 1
    over log2(NthRoot/2) bits."""
    lg = (nthroot // 2).bit_length() - 1
    return [2 * O.bit_reverse64(j, lg) + 1 for j in range(N)]


def ntt_index_exact(N, nthroot, g):
    """AutomorphismNTTIndex from its meaning: slot j of the image holds a(psi^(g*e_j)), which is slot k of a with
    e_k = g*e_j mod NthRoot."""
    e = ntt_slot_exponents(N, nthroot)
    where = {x: k for k, x in enumerate(e)}
    return [where[g * x % nthroot] for x in e]


def extend_exact(c, Q, p):
    """ExtendBasisSmallNormAndCenter on one coefficient: the centred lift of c mod Q (negative above Q/2) written mod p as
    the literal word p - |c| for a negative value."""
    half = Q >> 1
    if c > half:
        return (p - (Q - c)) & M64
    return c


def modup_centered_exact(c, q0, t, strict):
    """modup_centered on one coefficient: c is negative at or above q0/2 (strict: above), its magnitude is reduced mod the
    target t, and a negative value is written as t - (|c| mod t) (a negative multiple of t is t, not 0)."""
    neg = c > (q0 >> 1) if strict else c >= (q0 >> 1)
    mag = q0 - c if neg else c
    m = mag % t
    return t - m if neg else m


GALOIS_GEN = 5


def galois_elements(N, ci=False):
    """1, 5, 5^2, 5^(N/4-1), 5^(N/2-1), and on the standard ring 2N-1 and its products with those powers."""
    nth = (4 if ci else 2) * N
    ks = [0, 1, 2, max(N // 4 - 1, 1), max(N // 2 - 1, 1)]
    pw = sorted({pow(GALOIS_GEN, k, nth) for k in ks})
    if ci:
        return pw
    return sorted(set(pw) | {nth - 1} | {(nth - 1) * g % nth for g in pw})


# ---------------------------------------------------------------------------------------------------------------
# Launch-shape restatement (launch_vecop / launch_one in csrc/vecops.cu)
# ---------------------------------------------------------------------------------------------------------------
THREADS = 256


def vec2(n, aligned, strides_even=True):
    """launch_vecop takes the 128-bit path when n is even and every operand is 16-byte aligned with even strides."""
    return n % 2 == 0 and aligned and strides_even


def launch_shape(n, is_vec2):
    """(VEC, blocks, grid-stride passes, pass class) of launch_one."""
    vec = 2 if is_vec2 else 1
    nv = n // vec
    blocks0 = (nv + THREADS - 1) // THREADS
    blocks = (blocks0 + 3) // 4 if blocks0 > 64 else blocks0
    blocks = max(blocks, 1)
    passes = max(1, -(-nv // (blocks * THREADS)))
    if blocks0 <= 64:
        cls = "one"
    elif blocks0 % 4:
        cls = "ragged"
    else:
        cls = "several"
    return vec, blocks, passes, cls


# GPU vecop cases: (logN, entry, layout, n).
#   entry "ring": Ring ops on ringQ (every row, batch 3, and AtLevel below the maximum) and ringP (batch 1); n = N.
#   entry "subring": one row of ringQ and one of ringP through the SubRing entry, length n.
#   layout "aligned": 16-byte aligned tensors; "odd": every operand starts one word into its buffer (scalar path).
VEC_CASES = [(lg, "ring", "aligned", 1 << lg) for lg in LOG_NS] + [
    (10, "ring", "odd", 1 << 10),
    (15, "ring", "odd", 1 << 15),
    (10, "subring", "aligned", 1000),
    (10, "subring", "aligned", 1001),
    (17, "subring", "aligned", 65536),
    (16, "subring", "aligned", 2 * (THREADS * 65 + 17)),     # VEC 2, 66 blocks -> 17 (ragged), several passes
    (15, "subring", "aligned", THREADS * 68 - 1),             # VEC 1, 68 blocks -> 17, several passes
    (15, "subring", "odd", THREADS * 65 + 1),                 # VEC 1, 66 blocks -> 17 (ragged)
]


def case_cells(case):
    """The cells one GPU case reaches: (vec, pass class, source, prime class, op), and ("degree", logN) for an aligned
    whole-ring case."""
    logN, entry, layout, n = case
    vec, _, _, cls = launch_shape(n, vec2(n, layout == "aligned"))
    Q, P, cq, cp = chain(logN)
    cells = set()
    if entry == "ring":
        if layout == "aligned":
            cells.add(("degree", logN))
        srcs = [("ringQ", cq), ("ringP", cp)]
    else:
        srcs = [("subring", cq + cp)]
    for src, classes in srcs:
        for c in classes:
            for op in O.OPS:
                cells.add((vec, cls, src, c, op))
    return cells


def ragged_candidate_lengths():
    """Row lengths at the edge of launch_one's block rounding, fixed here without reference to the case list: for VEC 2
    (even lengths) and VEC 1 (odd lengths), the shortest and the longest length whose block count before the grid-stride
    division is each of 65 .. 68 (65, 66 and 67 are ragged; 68 is a whole number of four-block groups)."""
    out = set()
    for b in range(65, 69):
        out |= {2 * (THREADS * (b - 1) + 1), 2 * THREADS * b}          # VEC 2: n / 2 words in b blocks
        out |= {THREADS * (b - 1) + 1, THREADS * b - 1}                # VEC 1: odd n in b blocks
    return sorted(out)


def required_cells():
    """Every launch-shape cell the two entries can reach: {VEC 1, 2} x {one pass, several passes, ragged} x {ringQ, ringP,
    subring} x prime class x opcode, over every ring degree 2^4 .. 2^17 and both layouts; for the SubRing entry the row
    lengths are N, N - 1 and ragged_candidate_lengths() up to N. A whole-ring row has N = 2^logN words, so a ragged
    block count is reachable only through the SubRing entry, and a real small prime only at the degrees it admits.
    Every ring degree is a cell of its own. Nothing here is taken from VEC_CASES, so deleting a case cannot shrink
    what is required."""
    universe = []
    for lg in LOG_NS:
        N = 1 << lg
        for layout in ("aligned", "odd"):
            universe.append((lg, "ring", layout, N))
            for n in {N, N - 1} | {n for n in ragged_candidate_lengths() if n <= N}:
                universe.append((lg, "subring", layout, n))
    return reached_cells(universe)


def reached_cells(cases):
    out = set()
    for c in cases:
        out |= case_cells(c)
    return out

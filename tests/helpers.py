"""Shared test helpers: seeded inputs, synthetic/real evaluation keys (built with the ORACLE's ring ops;
test infrastructure only)."""
import numpy as np

from oracle import oracle as O
from oracle import philox as PH

U64 = np.uint64

# ring/test_params.go:17-32 (61-bit NTT-friendly primes valid up to N = 2^17)
Qi60 = [0x1fffffffffe00001, 0x1fffffffffc80001, 0x1fffffffffb40001, 0x1fffffffff500001,
        0x1fffffffff380001, 0x1fffffffff000001, 0x1ffffffffef00001, 0x1ffffffffee80001,
        0x1ffffffffeb40001, 0x1ffffffffe780001, 0x1ffffffffe600001, 0x1ffffffffe4c0001,
        0x1ffffffffdf40001, 0x1ffffffffdac0001, 0x1ffffffffda40001, 0x1ffffffffc680001,
        0x1ffffffffc000001, 0x1ffffffffb880001, 0x1ffffffffb7c0001, 0x1ffffffffb300001,
        0x1ffffffffb1c0001, 0x1ffffffffadc0001, 0x1ffffffffa400001, 0x1ffffffffa140001,
        0x1ffffffff9d80001, 0x1ffffffff9140001, 0x1ffffffff8ac0001, 0x1ffffffff8a80001,
        0x1ffffffff81c0001, 0x1ffffffff7800001, 0x1ffffffff7680001, 0x1ffffffff7080001]
Pi60 = [0x1ffffffff6c80001, 0x1ffffffff6140001, 0x1ffffffff5f40001, 0x1ffffffff5700001,
        0x1ffffffff4bc0001, 0x1ffffffff4380001, 0x1ffffffff3240001, 0x1ffffffff2dc0001,
        0x1ffffffff1a40001, 0x1ffffffff11c0001, 0x1ffffffff0fc0001, 0x1ffffffff0d80001]

# core/rlwe/test_params.go:11-13
RLWE_TEST_Q = [0x200000440001, 0x7fff80001, 0x800280001, 0x7ffd80001, 0x7ffc80001]
RLWE_TEST_P = [0x3ffffffb80001, 0x4000000800001]


def rand_poly(moduli, N, rng):
    """Uniform residues in [0, q_i) per limb (SURVEY 8(d) synthetic inputs)."""
    return np.stack([rng.integers(0, int(q), N, dtype=U64) for q in moduli])


def launch_delta(fn):
    """Kernel launches that one call of fn() makes, from the library's launch counter (lgpu_launch_count). An NTT / INTT at
    N > 2^12 counts 1 for a persistent single-pass launch and 2 for the two-pass kernels, so a test can assert which path
    a call took."""
    import lattigo_b200 as lb
    n0 = lb.lib().lgpu_launch_count()
    fn()
    return lb.lib().lgpu_launch_count() - n0


def ntt_prime(bits, N, above):
    """The NTT-friendly prime (1 mod 2N) closest to 2^bits from above or below."""
    step = 2 * N
    k = (1 << bits) // step + (1 if above else 0)
    while not O.is_prime(k * step + 1):
        k += 1 if above else -1
    return k * step + 1


def gof_pvalue(counts, probs, statistic="log-likelihood", min_expected=5.0):
    """p-value of a G-test (or another scipy power-divergence statistic, e.g. "pearson") of observed counts against exact bin
    probabilities; 0 if a bin of probability 0 has a draw. Bins are taken in order and merged until each expects at least
    min_expected draws (a short last group joins the one before it)."""
    from scipy.stats import power_divergence
    counts = np.asarray(counts, dtype=np.float64)
    probs = np.asarray(probs, dtype=np.float64)
    if (counts[probs == 0] > 0).any():
        return 0.0
    o, e, acc_o, acc_e = [], [], 0.0, 0.0
    for ci, ei in zip(counts, probs * counts.sum()):
        acc_o += ci; acc_e += ei
        if acc_e >= min_expected:
            o.append(acc_o); e.append(acc_e); acc_o = acc_e = 0.0
    if o:
        o[-1] += acc_o; e[-1] += acc_e
    if len(o) < 2:
        return 1.0
    return float(power_divergence(np.array(o), np.array(e) * (sum(o) / sum(e)), lambda_=statistic).pvalue)


def uniform_pvalues(v, q):
    """Chi-square p-values of uniform values in [0, q) over 256 equal bins and over the residue mod 3 (exact bin edges)."""
    v = np.asarray(v, dtype=np.uint64)
    edge = np.array([-(-k * q // 256) for k in range(257)], dtype=np.uint64)
    bins = np.searchsorted(edge, v, side="right") - 1
    p_bins = gof_pvalue(np.bincount(bins, minlength=256), PH.uniform_bin_probabilities(q, 256), "pearson")
    p_res = gof_pvalue(np.bincount((v % np.uint64(3)).astype(np.int64), minlength=3), PH.uniform_residue_probabilities(q, 3), "pearson")
    return p_bins, p_res


def gaussian_edges(bound):
    """Bin edges of |v| for oracle.philox.gaussian_law: one bin per value up to 64, else 80 bins of equal width."""
    K = int(np.floor(bound + 0.5))
    if K <= 64:
        return list(range(K + 2))
    return [0, 1] + [int(x) for x in np.unique(np.round(np.linspace(2, K + 1, 80)))]


def small_poly_rns(coeffs, moduli):
    """Signed small integer coefficients -> RNS rows."""
    return np.stack([np.array([int(c) % int(q) for c in coeffs], dtype=U64) for q in moduli])


def random_gadget_ciphertext(params: O.Parameters, levelQ, levelP, rng, pw2=0):
    """A GadgetCiphertext of the right shape with uniform entries (throughput / parity vs oracle)."""
    n = params.BaseRNSDecompositionVectorSize(levelQ, levelP)
    sizes = params.BaseTwoDecompositionVectorSize(levelQ, levelP, pw2)[:n]
    mods = params.qi[: levelQ + 1] + params.pi[: levelP + 1]
    N = params.N()
    data = np.zeros((n, max(sizes), 2, len(mods), N), dtype=U64)
    for i in range(n):
        for j in range(sizes[i]):
            for c in range(2):
                data[i, j, c] = rand_poly(mods, N, rng)
    return O.GadgetCiphertext(data, levelQ + 1, levelP + 1, pw2, sizes)


def gen_switching_key(params: O.Parameters, s_in, s_out, rng, pw2=0, sigma=3.2):
    """Real evaluation key encrypting s_in under s_out (core/rlwe/keygenerator.go:286-328 +
    core/rlwe/gadgetciphertext.go:172-241): evk[i][j] = (-a*s_out + e + P*w^j*s_in*[limb in digit i], a),
    NTT domain, Montgomery form, over Q (max level) and P."""
    levelQ, levelP = params.MaxLevelQ(), params.MaxLevelP()
    N = params.N()
    ringQ = params.ringQ
    ringP = params.ringP
    Qm, Pm = params.qi, params.pi
    mods = Qm + Pm
    n = params.BaseRNSDecompositionVectorSize(levelQ, levelP)
    sizes = params.BaseTwoDecompositionVectorSize(levelQ, levelP, pw2)[:n]

    def ntt_qp(rows):
        out = np.empty_like(rows)
        ringQ.NTT(rows[: levelQ + 1], out[: levelQ + 1])
        if ringP is not None:
            ringP.NTT(rows[levelQ + 1:], out[levelQ + 1:])
        return out

    def mulmod(a, b):   # plain coefficient-wise product mod each limb (python ints; setup only, small N)
        return np.stack([np.array([int(x) * int(y) % int(q) for x, y in zip(a[i], b[i])], dtype=U64) for i, q in enumerate(mods)])

    def addmod(a, b):
        return np.stack([np.array([(int(x) + int(y)) % int(q) for x, y in zip(a[i], b[i])], dtype=U64) for i, q in enumerate(mods)])

    s_out_ntt = ntt_qp(small_poly_rns(s_out, mods))
    s_in_ntt = ntt_qp(small_poly_rns(s_in, mods))
    Pprod = 1
    for p in Pm:
        Pprod *= p
    data = np.zeros((n, max(sizes), 2, len(mods), N), dtype=U64)
    kP = max(levelP + 1, 1)
    for i in range(n):
        for j in range(sizes[i]):
            a = rand_poly(mods, N, rng)
            e = ntt_qp(small_poly_rns(np.rint(rng.normal(0, sigma, N)).astype(np.int64), mods))
            neg_as = np.stack([np.array([(int(q) - int(x) * int(y) % int(q)) % int(q) for x, y in zip(a[l], s_out_ntt[l])], dtype=U64) for l, q in enumerate(mods)])
            c0 = addmod(neg_as, e)
            for k in range(kP):
                idx = i * kP + k
                if idx >= levelQ + 1:
                    break
                q = Qm[idx]
                f = Pprod * (1 << (pw2 * j)) % q
                c0[idx] = np.array([(int(x) + f * int(y)) % q for x, y in zip(c0[idx], s_in_ntt[idx])], dtype=U64)
            R = 1 << 64
            data[i, j, 0] = np.stack([np.array([int(x) * R % int(q) for x in c0[l]], dtype=U64) for l, q in enumerate(mods)])
            data[i, j, 1] = np.stack([np.array([int(x) * R % int(q) for x in a[l]], dtype=U64) for l, q in enumerate(mods)])
    return O.GadgetCiphertext(data, levelQ + 1, levelP + 1, pw2, sizes)


def keyswitch_noise_log2(params: O.Parameters, levelQ, cx_ntt, ct, s_in, s_out):
    """log2 of the max centred |d0 + d1*s_out - cx*s_in| (coefficient domain, mod Q_level)."""
    ringQ = params.ringQ.AtLevel(levelQ)
    mods = params.qi[: levelQ + 1]
    so = small_poly_rns(s_out, mods); si = small_poly_rns(s_in, mods)
    son = np.empty_like(so); sin = np.empty_like(si)
    ringQ.NTT(so, son); ringQ.NTT(si, sin)
    acc = np.empty_like(so)
    for l, q in enumerate(mods):
        q = int(q)
        acc[l] = np.array([(int(a) + int(b) * int(s) - int(c) * int(t)) % q
                           for a, b, s, c, t in zip(ct[0][l], ct[1][l], son[l], cx_ntt[l], sin[l])], dtype=U64)
    back = np.empty_like(acc)
    ringQ.INTT(acc, back)
    Q = ringQ.ModulusAtLevel[levelQ]
    vals = ringQ.PolyToBigint(back)
    m = max(min(v, Q - v) for v in vals)
    return float(np.log2(float(m))) if m else 0.0


# ---- the reference's wire format, written the way its WriteTo methods do (little-endian uint64 words) --------------------
def marshal_poly(rows) -> bytes:
    """ring.Poly.MarshalBinary (ring/poly.go:132-142 -> structs.Matrix[uint64].WriteTo, utils/structs/matrix.go:80-108)."""
    rows = np.asarray(rows, dtype=U64)
    out = [np.array([rows.shape[0]], dtype="<u8").tobytes()]
    for r in rows:
        out.append(np.array([r.shape[0]], dtype="<u8").tobytes())
        out.append(np.ascontiguousarray(r).astype("<u8").tobytes())
    return b"".join(out)


def marshal_gadget_ct(gct: "O.GadgetCiphertext") -> bytes:
    """rlwe.GadgetCiphertext.MarshalBinary (core/rlwe/gadgetciphertext.go:101-121): BaseTwoDecomposition, then
    structs.Matrix[VectorQP]: len(Value), per digit len(Value[i]), per entry len(VectorQP) = 2, per ringqp.Poly Q then P."""
    d = gct.data
    nq = gct.nQ
    n_digits = d.shape[0]
    sizes = list(gct.pw2_sizes)
    out = [np.array([gct.BaseTwoDecomposition, n_digits], dtype="<u8").tobytes()]
    for i in range(n_digits):
        out.append(np.array([sizes[i]], dtype="<u8").tobytes())
        for j in range(sizes[i]):
            out.append(np.array([2], dtype="<u8").tobytes())
            for k in range(2):
                out.append(marshal_poly(d[i, j, k, :nq]))
                out.append(marshal_poly(d[i, j, k, nq:]))
    return b"".join(out)


def marshal_galois_key(gal_el: int, nth_root: int, gct) -> bytes:
    """rlwe.GaloisKey.MarshalBinary (core/rlwe/keys.go:628-657)."""
    return np.array([gal_el, nth_root], dtype="<u8").tobytes() + marshal_gadget_ct(gct)


def gen_rgsw(params: "O.Parameters", m1, s, rng, pw2=0):
    """Real RGSW encryption of the small polynomial m1 under s (core/rgsw/encryptor.go:34-88 + elements.go:11-13):
    Value[0] = gadget encryption of m1 (message on component 0), Value[1] = gadget encryption of zero with
    P * w^j * m1 added to component 1 on the digit's own limbs (i.e. of m1 * s)."""
    v0 = gen_switching_key(params, m1, s, rng, pw2=pw2)
    v1 = gen_switching_key(params, [0] * params.N(), s, rng, pw2=pw2)
    levelQ, levelP = params.MaxLevelQ(), params.MaxLevelP()
    Qm, Pm = params.qi, params.pi
    mods = Qm + Pm
    m_ntt = np.empty((len(mods), params.N()), dtype=U64)
    rows = small_poly_rns(m1, mods)
    params.ringQ.NTT(rows[: levelQ + 1], m_ntt[: levelQ + 1])
    if params.ringP is not None:
        params.ringP.NTT(rows[levelQ + 1:], m_ntt[levelQ + 1:])
    Pprod = 1
    for p in Pm:
        Pprod *= p
    kP = max(levelP + 1, 1)
    R = 1 << 64
    for i in range(v1.data.shape[0]):
        for j in range(v1.pw2_sizes[i]):
            for k in range(kP):
                idx = i * kP + k
                if idx >= levelQ + 1:
                    break
                q = Qm[idx]
                f = Pprod * (1 << (pw2 * j)) % q * R % q          # Montgomery form, like the key rows
                v1.data[i, j, 1, idx] = np.array([(int(x) + f * int(y)) % q for x, y in zip(v1.data[i, j, 1, idx], m_ntt[idx])], dtype=U64)
    return [v0, v1]

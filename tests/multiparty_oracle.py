"""CPU restatement of the threshold protocols of multiparty/ that csrc/multiparty.cu serves, on oracle.oracle.Parameters with the
samplers' outputs as explicit arguments (as in oracle/encryptor.py):

    PublicKeyGenProtocol.GenShare / GenPublicKey          multiparty/keygen_cpk.go:70-99
    KeySwitchProtocol.GenShare (ct.IsNTT) / KeySwitch     multiparty/keyswitch_sk.go:85-147
    PublicKeySwitchProtocol.GenShare (ct.IsNTT) / KeySwitch   multiparty/keyswitch_pk.go:69-134
    EvaluationKeyGenProtocol.GenShare / GenEvaluationKey  multiparty/keygen_evk.go:86-231
    GaloisKeyGenProtocol.GenShare                         multiparty/keygen_gal.go:48-70
    RelinearizationKeyGenProtocol rounds one and two, GenRelinearizationKey   multiparty/keygen_relin.go:91-276
    AggregateShares (all of them)                         e.g. keyswitch_sk.go:123-130: ring Add = CRed(a + b), left fold
    NoiseFreshSK / NoiseFreshPK                           core/rlwe/params.go:335-384
    NoiseKeySwitch / NoisePublicKeySwitch                 multiparty/utils.go

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import math

import numpy as np

from oracle import encryptor as E
from oracle import oracle as O

U64 = np.uint64


def cred_add(a, b, q):
    """SubRing.Add on uint64 arrays: CRed(a + b) on the wrapping 64-bit sum, as Go computes it."""
    with np.errstate(over="ignore"):
        s = a.astype(U64) + b.astype(U64)
    return np.where(s >= U64(q), s - U64(q), s).astype(U64)


def aggregate(shares, moduli):
    """agg = shares[0]; agg = Add(agg, s) for s in shares[1:]. shares: arrays (..., rows, N); moduli: one per row."""
    agg = np.array(shares[0], dtype=U64, copy=True)
    for s in shares[1:]:
        for r, q in enumerate(moduli):
            agg[..., r, :] = cred_add(agg[..., r, :], s[..., r, :], q)
    return agg


class Protocols:
    def __init__(self, params: O.Parameters):
        self.params = params
        self.enc = E.Encryptor(params)

    # keygen_cpk.go:70-83: e -> NTT -> MForm -> MulCoeffsMontgomeryThenSub(sk, crp)
    def ckg_share(self, sk, crp, e):
        p = self.params
        return self.enc.encryptZeroSkFromC1QP(p.MaxLevelQ(), p.MaxLevelP(), sk, np.array(crp, dtype=U64, copy=True), e, True, True)

    def ckg_public_key(self, share, crp):
        return np.stack([share, crp])

    # keyswitch_sk.go:85-118, ct.IsNTT branch
    def cks_share(self, level, sk_in, sk_out, c1, e):
        ringQ = self.params.ringQ.AtLevel(level)
        delta = ringQ.NewPoly()
        ringQ.Sub(sk_in[: level + 1], sk_out[: level + 1], delta)
        share = ringQ.NewPoly()
        ringQ.MulCoeffsMontgomeryLazy(c1, delta, share)
        buf = E.small_rows(e, self.params.qi[: level + 1])
        ringQ.NTT(buf, buf)
        ringQ.Add(share, buf, share)
        return share

    def cks_key_switch(self, ct, combined):
        level = ct[0].shape[0] - 1
        out0 = ct[0].copy()
        self.params.ringQ.AtLevel(level).Add(ct[0], combined, out0)
        return [out0, ct[1].copy()]

    # keyswitch_pk.go:69-105, ct.IsNTT branch (ct.IsMontgomery = false)
    def pcks_share(self, level, sk, pk, c1, u, e0, e1, e_flood):
        p = self.params
        if p.ringP is not None:
            s0, s1 = self.enc.encryptZeroPk(level, pk, u, e0, e1, True, False)
        else:
            s0, s1 = self.enc.encryptZeroPkNoP(level, pk, u, e0, e1, True)
        ringQ = p.ringQ.AtLevel(level)
        ringQ.MulCoeffsMontgomeryThenAdd(c1, sk[: level + 1], s0)
        buf = E.small_rows(e_flood, p.qi[: level + 1])
        ringQ.NTT(buf, buf)
        ringQ.Add(s0, buf, s0)
        return [s0, s1]

    def pcks_key_switch(self, ct, combined):
        level = ct[0].shape[0] - 1
        out0 = ct[0].copy()
        self.params.ringQ.AtLevel(level).Add(ct[0], combined[0], out0)
        return [out0, combined[1].copy()]


class KeyGen:
    """The key-generation shares at the maximum levels. crp[i][j], shares[i][j]: (nQ + nP, N) rows; e[i][j]: signed small polynomials.
    Entries with j >= BaseTwoDecompositionVectorSize[i] stay zero, as in the reference's freshly allocated shares."""

    def __init__(self, params: O.Parameters, pw2: int):
        self.params, self.pw2 = params, pw2
        self.levelQ, self.levelP = params.MaxLevelQ(), params.MaxLevelP()
        self.nd = params.BaseRNSDecompositionVectorSize(self.levelQ, self.levelP)
        self.sizes = params.BaseTwoDecompositionVectorSize(self.levelQ, self.levelP, pw2)[: self.nd]
        self.nq, self.np = self.levelQ + 1, self.levelP + 1
        self.ringQ = params.ringQ
        self.ringP = params.ringP

    def _qp(self, op, *args):
        """Apply a ring method on the Q rows and the P rows of QP-stacked arrays."""
        nq = self.nq
        getattr(self.ringQ, op)(*[a[:nq] for a in args])
        if self.np:
            getattr(self.ringP, op)(*[a[nq:] for a in args])

    def _small(self, e):
        return E.small_rows(e, list(self.params.qi) + list(self.params.pi))

    def _gadget_factor(self, sk_in):
        buff = self.ringQ.NewPoly()
        if self.np:
            self.ringQ.MulScalarBigint(sk_in[: self.nq], self.ringP.ModulusAtLevel[self.levelP], buff)
        else:
            buff[...] = sk_in[: self.nq]
        return buff

    def _add_digit(self, m, buff, i):
        for k in range(max(self.np, 1)):
            index = i * max(self.np, 1) + k
            if index >= self.nq:
                break
            self.ringQ.SubRings[index].vecop("Add", m[index], buff[index], m[index])

    def _zeros(self, ncomp=None):
        shape = (self.nd, max(self.sizes)) + ((ncomp,) if ncomp else ()) + (self.nq + self.np, self.params.N())
        return np.zeros(shape, dtype=U64)

    # keygen_evk.go:86-183
    def evkg_share(self, sk_in, sk_out, crp, e):
        buff = self._gadget_factor(sk_in)
        out = self._zeros()
        for j in range(max(self.sizes)):
            for i in range(self.nd):
                if j < self.sizes[i]:
                    m = self._small(e[i][j])
                    self._qp("NTTLazy", m, m)
                    self._qp("MForm", m, m)
                    self._add_digit(m, buff, i)
                    self._qp("MulCoeffsMontgomeryThenSub", np.array(crp[i][j]), self._kp(sk_out), m)
                    out[i, j] = m
            self.ringQ.MulScalar(buff, 1 << self.pw2, buff)
        return out

    def _kp(self, sk):
        """A secret key's rows at the maximum levels, QP-stacked."""
        return np.array(sk[: self.nq + self.np])

    # keygen_gal.go:48-70
    def gkg_share(self, sk, gal_el, crp, e):
        nthroot = 2 * self.params.N()
        inv = pow(int(gal_el), nthroot - 1, nthroot)
        sk_out = np.zeros_like(self._kp(sk))
        self.ringQ.AutomorphismNTT(sk[: self.nq], inv, sk_out[: self.nq])
        if self.np:
            self.ringP.AutomorphismNTT(sk[self.nq: self.nq + self.np], inv, sk_out[self.nq:])
        return self.evkg_share(sk, sk_out, crp, e)

    def gen_evaluation_key(self, share, crp):
        return np.stack([share, np.asarray(crp)], axis=2)

    # keygen_relin.go:91-184
    def rkg_round_one(self, sk, crp, u, e0, e1):
        buff = self._gadget_factor(sk)
        self.ringQ.IMForm(buff, buff)
        eph = self._small(u)
        self._qp("NTT", eph, eph)
        self._qp("MForm", eph, eph)
        out = self._zeros(2)
        for j in range(max(self.sizes)):
            for i in range(self.nd):
                if j < self.sizes[i]:
                    m0 = self._small(e0[i][j])
                    self._qp("NTT", m0, m0)
                    self._add_digit(m0, buff, i)
                    self._qp("MulCoeffsMontgomeryThenSub", eph, np.array(crp[i][j]), m0)
                    m1 = self._small(e1[i][j])
                    self._qp("NTT", m1, m1)
                    self._qp("MulCoeffsMontgomeryThenAdd", self._kp(sk), np.array(crp[i][j]), m1)
                    out[i, j, 0], out[i, j, 1] = m0, m1
            self.ringQ.MulScalar(buff, 1 << self.pw2, buff)
        return eph, out

    # :193-234
    def rkg_round_two(self, eph, sk, round1, e2):
        delta = np.zeros_like(eph)
        self._qp("Sub", eph, self._kp(sk), delta)
        out = self._zeros()
        for i in range(self.nd):
            for j in range(self.sizes[i]):
                m = np.zeros_like(eph)
                self._qp("MulCoeffsMontgomeryLazy", np.array(round1[i, j, 0]), self._kp(sk), m)
                b = self._small(e2[i][j])
                self._qp("NTT", b, b)
                self._qp("Add", m, b, m)
                self._qp("MulCoeffsMontgomeryThenAdd", delta, np.array(round1[i, j, 1]), m)
                out[i, j] = m
        return out

    # :261-276
    def gen_relinearization_key(self, round1, round2):
        out = self._zeros(2)
        for i in range(self.nd):
            for j in range(self.sizes[i]):
                self._qp("MForm", np.array(round2[i, j]), out[i, j, 0])
                self._qp("MForm", np.array(round1[i, j, 1]), out[i, j, 1])
        return out


# core/rlwe/params.go:335-384 with Xs = Ternary{P} or Ternary{H} and Xe = DiscreteGaussian(sigma)
def xs_hamming_weight(N, xs_p=2 / 3, xs_h=0):
    return xs_h if xs_h else int(math.ceil(N * xs_p))


def noise_fresh_sk(sigma=3.2):
    return sigma


def noise_fresh_pk(N, has_p, sigma=3.2, xs_p=2 / 3, xs_h=0):
    std = float(xs_hamming_weight(N, xs_p, xs_h) + 1)
    std *= 1 / 12.0 if has_p else sigma * sigma
    return math.sqrt(std)


# multiparty/utils.go
def _smudged(n_parties, noisect, noisefresh, noiseflood):
    std = noisefresh * noisefresh + noiseflood * noiseflood
    return math.sqrt(std * n_parties + noisect * noisect)


def noise_key_switch(n_parties, noisect, noiseflood, sigma=3.2):
    return _smudged(n_parties, noisect, noise_fresh_sk(sigma), noiseflood)


def noise_public_key_switch(N, has_p, n_parties, noisect, noiseflood, sigma=3.2):
    return _smudged(n_parties, noisect, noise_fresh_pk(N, has_p, sigma), noiseflood)


def sk_rows(params: O.Parameters, s):
    """A signed ternary secret as rlwe.SecretKey rows over QP, NTT + Montgomery."""
    q, p = list(params.qi), list(params.pi)
    sk = E.small_rows(s, q + p)
    params.ringQ.NTT(sk[: len(q)], sk[: len(q)]); params.ringQ.MForm(sk[: len(q)], sk[: len(q)])
    if p:
        params.ringP.NTT(sk[len(q):], sk[len(q):]); params.ringP.MForm(sk[len(q):], sk[len(q):])
    return sk


def decrypt_noise(params: O.Parameters, ct, sk, montgomery=False):
    """Centred coefficients of INTT(c0 + c1 s) on ct's Q rows (IMForm first for a Montgomery-form ct, such as a public key); asserts
    that every row holds the same small integer."""
    level = ct[0].shape[0] - 1
    ringQ = params.ringQ.AtLevel(level)
    m = np.array(ct[0], dtype=U64, copy=True)
    ringQ.Reduce(m, m)
    ringQ.MulCoeffsMontgomeryThenAdd(ct[1], sk[: level + 1], m)
    if montgomery:
        ringQ.IMForm(m, m)
    ringQ.INTT(m, m)
    rows = []
    for i, q in enumerate(params.qi[: level + 1]):
        v = m[i].astype(object)
        rows.append(np.array([int(x) - q if int(x) > q // 2 else int(x) for x in v], dtype=object))
    for r in rows[1:]:
        assert np.array_equal(r, rows[0]), "decryption is not small: rows disagree"
    return rows[0].astype(np.float64)


def log2_std(v):
    return math.log2(float(np.std(v))) if np.std(v) > 0 else -math.inf

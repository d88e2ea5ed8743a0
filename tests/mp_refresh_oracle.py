"""CPU restatement of the mpbgv protocols that csrc/mp_refresh.cu serves, on oracle.oracle.Parameters and oracle/bgv_encoder.py, with the
samplers' outputs as explicit arguments:

    EncToShareProtocol.GenShare / GetShare               multiparty/mpbgv/sharing.go:62-91
    ShareToEncProtocol.GenShare / GetEncryption          multiparty/mpbgv/sharing.go:126-154
    MaskedTransformProtocol.GenShare / Transform         multiparty/mpbgv/transform.go:67-181 (Decode / Func / Encode on the mask)
    RefreshProtocol                                       multiparty/mpbgv/refresh.go (no transform, skIn = skOut)
    the mask sampler's stream                             lgpu_mpbgv_sample_mask (csrc/encrypt.cu, sample_mask_kernel)

Every step uses the reference's ring operations (oracle.oracle's restatement of them), so the words are the reference's: Sub / Add
with CRed, RingQ2T's lazy ModUpExact word, RingT2Q of that word as it is.

TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import numpy as np

from oracle import bgv_encoder as BE
from oracle import oracle as O
from oracle import philox as PH
from tests import multiparty_oracle as M

U64 = np.uint64
MASK_DOMAIN = 1 << 29      # kMaskDomain: bit 29 of the Philox counter's polynomial word, set by the mask draws only


def sample_mask(seed: int, stream_id: int, t: int, n: int, batch: int) -> np.ndarray:
    """lgpu_mpbgv_sample_mask: (batch, n) words uniform in [0, t). Polynomial word = entry | MASK_DOMAIN | KIND_UNIFORM << 30; per
    attempt the masked words (x:y) then (z:w), the first below t taken -- the uniform sampler's rule on another polynomial word."""
    mask = U64((1 << (t - 1).bit_length()) - 1)
    out = np.zeros((batch, n), dtype=U64)
    for b in range(batch):
        i = np.arange(n, dtype=U64)
        val = np.zeros(n, dtype=U64)
        pending = np.arange(n)
        a = 0
        while pending.size:
            x, y, z, w = PH.draw(PH.KIND_UNIFORM, seed, stream_id, b | MASK_DOMAIN, i[pending], a)
            v1 = ((x << U64(32)) | y) & mask
            v2 = ((z << U64(32)) | w) & mask
            ok1, ok2 = v1 < U64(t), v2 < U64(t)
            val[pending] = np.where(ok1, v1, v2)
            pending = pending[~(ok1 | ok2)]
            a += 1
        out[b] = val
    return out


class MPBGV:
    def __init__(self, params: O.Parameters, t: int):
        self.params = params
        self.enc = BE.BGVEncoder(params.ringQ, t, params.ringP)
        self.t, self.n = t, self.enc.n
        self.cks = M.Protocols(params)

    def _zero(self, level):
        return np.zeros((level + 1, self.params.N()), dtype=U64)

    def _lift_ntt(self, level, mask):
        """NTT(RingT2Q(level, true, mask))."""
        ringQ = self.params.ringQ.AtLevel(level)
        buf = self.enc.RingT2Q(level, True, np.asarray(mask, dtype=U64).reshape(1, -1), ringQ)
        ringQ.NTT(buf, buf)
        return buf

    # sharing.go:62-71
    def e2s_share(self, level, sk, c1, e, mask):
        share = self.cks.cks_share(level, sk, self._zero(level), np.asarray(c1)[: level + 1], e)
        self.params.ringQ.AtLevel(level).Sub(share, self._lift_ntt(level, mask), share)
        return share

    # sharing.go:78-91
    def e2s_get_share(self, level, ct0, agg, secret=None):
        ringQ = self.params.ringQ.AtLevel(level)
        buf = np.empty((level + 1, self.params.N()), dtype=U64)
        ringQ.Add(np.asarray(agg)[: level + 1], np.asarray(ct0)[: level + 1], buf)
        ringQ.INTT(buf, buf)
        pT = self.enc.RingQ2T(level, buf, self.n)
        if secret is not None:
            self.enc.ringT.Add(np.asarray(secret, dtype=U64).reshape(1, -1), pT, pT)
        return pT[0]

    # sharing.go:126-143
    def s2e_share(self, level, sk, crp, e, mask):
        share = self.cks.cks_share(level, self._zero(level), sk, np.asarray(crp), e)
        self.params.ringQ.AtLevel(level).Add(share, self._lift_ntt(level, mask), share)
        return share

    # transform.go:173-180
    def recrypt(self, level, mask, agg, crp):
        c0 = self._lift_ntt(level, mask)
        self.params.ringQ.AtLevel(level).Add(c0, np.asarray(agg), c0)
        return np.stack([c0, np.asarray(crp)])

    def decode_ring_t(self, pT, scale):
        return np.array(self.enc.DecodeRingT(np.asarray(pT, dtype=U64).reshape(1, -1), scale, False), dtype=U64)

    def encode_ring_t(self, values, scale):
        return self.enc.EncodeRingT([int(v) for v in values], False, scale)[0]

    def apply(self, transform, mask, scale):
        """MaskedTransformFunc on one mask: (decode, func on a list of ints, encode)."""
        if transform is None:
            return mask
        decode, func, encode = transform
        coeffs = self.decode_ring_t(mask, scale) if decode else np.array(mask, dtype=U64)
        coeffs = np.array(func([int(c) for c in coeffs]), dtype=U64)
        return self.encode_ring_t(coeffs, scale) if encode else coeffs

    # transform.go:67-109 for one ciphertext
    def transform_share(self, level_e2s, sk_in, sk_out, ct, crp, transform, scale, e0, e1, mask):
        level = min(ct[1].shape[0] - 1, level_e2s)
        e2s = self.e2s_share(level, sk_in, ct[1], e0, mask)
        m = self.apply(transform, mask, scale)
        s2e = self.s2e_share(crp.shape[0] - 1, sk_out, crp, e1, m)
        return e2s, s2e

    # transform.go:129-181 for one ciphertext
    def transform(self, ct, transform, crp, agg_e2s, agg_s2e, scale_out):
        level = min(ct[0].shape[0] - 1, agg_e2s.shape[0] - 1)
        mask = self.e2s_get_share(level, ct[0], agg_e2s)
        mask = self.apply(transform, mask, scale_out)
        return self.recrypt(crp.shape[0] - 1, mask, agg_s2e, crp)

    # ---- encryption / decryption under a secret key (for the end-to-end checks) ----
    def encrypt(self, sk, values, level, scale, a, e):
        """Encode (batched, NTT) + encryptZeroSk: (c0 + pt, a)."""
        pt = self.enc.Encode(list(values), False, scale, True, False, level)
        c0 = self.cks.enc.encryptZeroSkFromC1QP(level, -1, sk, np.asarray(a), e, True, False)
        self.params.ringQ.AtLevel(level).Add(c0, pt, c0)
        return np.stack([c0, np.asarray(a)])

    def decrypt(self, sk, ct, scale):
        level = ct[0].shape[0] - 1
        ringQ = self.params.ringQ.AtLevel(level)
        m = np.array(ct[0], dtype=U64, copy=True)
        ringQ.Reduce(m, m)
        ringQ.MulCoeffsMontgomeryThenAdd(np.asarray(ct[1]), sk[: level + 1], m)
        return self.enc.Decode(m, level, scale, True)


# ---- mpckks -----------------------------------------------------------------------------------------------------------------------
BIG_MASK_DOMAIN = 1 << 28      # kBigMaskDomain: the mpckks masks' polynomial word also carries this bit


def sample_big_mask(seed: int, stream_id: int, log_bound: int, dslots: int, batch: int):
    """lgpu_mpckks_sample_mask as Python ints: attempt a of value i gives the 64-bit words 2a = (x:y) and 2a + 1 = (z:w); the low
    log_bound bits are RandInt(2^log_bound), and values >= 2^(log_bound - 1) have 2^log_bound subtracted."""
    nwords = (log_bound + 63) // 64
    out = []
    for b in range(batch):
        i = np.arange(dslots, dtype=U64)
        words = []
        for a in range((nwords + 1) // 2):
            x, y, z, w = PH.draw(PH.KIND_UNIFORM, seed, stream_id, b | MASK_DOMAIN | BIG_MASK_DOMAIN, i, a)
            words += [(x << U64(32)) | y, (z << U64(32)) | w]
        vals = []
        for j in range(dslots):
            v = sum(int(words[k][j]) << (64 * k) for k in range(nwords)) & ((1 << log_bound) - 1)
            vals.append(v - (1 << log_bound) if v >> (log_bound - 1) else v)
        out.append(vals)
    return out


def quo(a: int, b: int) -> int:
    """big.Int.Quo: truncation toward zero."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


class MPCKKS:
    def __init__(self, params: O.Parameters):
        self.params = params
        self.cks = M.Protocols(params)
        self.N = params.N()

    def _zero(self, level):
        return np.zeros((level + 1, self.N), dtype=U64)

    def set_coefficients_bigint(self, level, values):
        """SetCoefficientsBigint + NTTSparseAndMontgomery (IsNTT, not Montgomery): the NTT of the values spread at gap N / dslots."""
        gap = self.N // len(values)
        qs = self.params.qi[: level + 1]
        p = np.zeros((level + 1, self.N), dtype=U64)
        for r, q in enumerate(qs):
            p[r, ::gap] = np.array([v % q for v in values], dtype=U64)
        self.params.ringQ.AtLevel(level).NTT(p, p)
        return p

    def e2s_share(self, level, sk, c1, e, mask):
        share = self.cks.cks_share(level, sk, self._zero(level), np.asarray(c1)[: level + 1], e)
        self.params.ringQ.AtLevel(level).Sub(share, self.set_coefficients_bigint(level, mask), share)
        return share

    def s2e_share(self, level, sk, crp, e, secret):
        share = self.cks.cks_share(level, self._zero(level), sk, np.asarray(crp), e)
        self.params.ringQ.AtLevel(level).Add(share, self.set_coefficients_bigint(level, secret), share)
        return share

    def get_share(self, level, ct0, agg, dslots, secret=None):
        ringQ = self.params.ringQ.AtLevel(level)
        buf = np.empty((level + 1, self.N), dtype=U64)
        ringQ.Add(np.asarray(agg)[: level + 1], np.asarray(ct0)[: level + 1], buf)
        ringQ.INTT(buf, buf)
        vals = BE._poly_to_bigint_centered(ringQ, buf, self.N // dslots)
        return [v + s for v, s in zip(vals, secret)] if secret is not None else vals

    @staticmethod
    def scale(values, d, s):
        return [quo(v * d, s) for v in values]

    def finalize(self, level_in, ct, agg_e2s, agg_s2e, crp, dslots, d, s):
        mask = self.scale(self.get_share(level_in, ct[0], agg_e2s, dslots), d, s)
        level = crp.shape[0] - 1
        c0 = self.set_coefficients_bigint(level, mask)
        self.params.ringQ.AtLevel(level).Add(c0, np.asarray(agg_s2e), c0)
        return np.stack([c0, np.asarray(crp)])

    def decrypt_coeffs(self, sk, ct):
        """Centred coefficients of INTT(c0 + c1 s) as Python ints (CRT over the ciphertext's level)."""
        level = ct[0].shape[0] - 1
        ringQ = self.params.ringQ.AtLevel(level)
        m = np.array(ct[0], dtype=U64, copy=True)
        ringQ.Reduce(m, m)
        ringQ.MulCoeffsMontgomeryThenAdd(np.asarray(ct[1]), sk[: level + 1], m)
        ringQ.INTT(m, m)
        return BE._poly_to_bigint_centered(ringQ, m, 1)

    def encrypt_coeffs(self, sk, coeffs, level, a, e):
        """A ciphertext (c0, a) of the integer polynomial `coeffs` (NTT domain): encryptZeroSk + NTT(coeffs)."""
        c0 = self.cks.enc.encryptZeroSkFromC1QP(level, -1, sk, np.asarray(a), e, True, False)
        p = np.zeros((level + 1, self.N), dtype=U64)
        for r, q in enumerate(self.params.qi[: level + 1]):
            p[r] = np.array([c % q for c in coeffs], dtype=U64)
        ringQ = self.params.ringQ.AtLevel(level)
        ringQ.NTT(p, p)
        ringQ.Add(c0, p, c0)
        return np.stack([c0, np.asarray(a)])

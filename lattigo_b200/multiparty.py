"""Host-side mirror of the threshold protocols of multiparty/ on the device (include/lattigo_b200.h, csrc/multiparty.cu):
collective public-key generation (PublicKeyGenProtocol, multiparty/keygen_cpk.go), collective relinearization-, evaluation- and
Galois-key generation (RelinearizationKeyGenProtocol, EvaluationKeyGenProtocol, GaloisKeyGenProtocol: keygen_relin.go, keygen_evk.go,
keygen_gal.go; at the maximum levels), collective key switching to a secret key (KeySwitchProtocol, keyswitch_sk.go) and to a public key
(PublicKeySwitchProtocol, keyswitch_pk.go), NTT-domain ciphertexts on the Standard ring; and the t-out-of-N access structure
(Thresholdizer, Combiner: threshold.go), with which any t of N parties turn their Shamir shares into additive shares of the secret and
then run the protocols above as t-out-of-t.

Randomness: every protocol instance draws its private samples from one encryptor.Samplers (the party's own seed), and SampleCRP
draws the common reference polynomial from a Samplers keyed by a seed all parties share, the CRS. These are the device samplers'
Philox streams, not the reference's blake2b XOF: parties that must agree on the CRP must all run this library. Each GenShare also
takes its samples as keyword arguments, so that a caller can hand the same arrays to another implementation.

Shares keep the reference's representatives: a KeySwitch share lies in [0, 2q), and AggregateShares is the reference's left fold of
Add = CRed(a + b), so K such shares aggregate to a value in [0, (K + 1) q) (see lgpu_mp_aggregate)."""
from __future__ import annotations

import ctypes
import math

from . import _lib
from .encryptor import Samplers
from .ring import Context, _dptr, _stream
from .rlwe import GadgetCiphertext


def _torch():
    import torch
    return torch


def aggregate(ctx: Context, levelQ: int, levelP: int, shares, out=None, mismatch="cannot AggregateShares: shares levels do not match"):
    """The left fold shares[0] + shares[1] + ... of one protocol's shares in one pass (lgpu_mp_aggregate): every share is a device
    tensor of the same shape whose last two dimensions are (levelQ+1 + levelP+1, N). out may be shares[0]."""
    torch = _torch()
    shares = list(shares)
    if not shares:
        raise _lib.LgpuError("AggregateShares needs at least one share")
    rows = levelQ + 1 + levelP + 1
    shape = shares[0].shape
    for s in shares:
        if s.shape != shape or not s.is_contiguous():
            raise _lib.LgpuError(mismatch)
    if shape[-2] != rows or shape[-1] != ctx.N:
        raise _lib.LgpuError(mismatch)
    for s in shares:
        if s.dtype != torch.int64 or not s.is_cuda:
            raise _lib.LgpuError("shares are 64-bit device tensors")
    if out is None:
        out = torch.empty_like(shares[0])
    elif out.shape != shape or out.dtype != torch.int64 or not out.is_cuda or not out.is_contiguous():
        raise _lib.LgpuError("out must be a contiguous 64-bit device tensor of the shares' shape")
    ptrs = (ctypes.c_void_p * len(shares))(*[s.data_ptr() for s in shares])
    n_polys = shares[0].numel() // (rows * ctx.N)
    _lib.check(_lib.lib().lgpu_mp_aggregate(ctx.h, levelQ, levelP, ptrs, len(shares), _dptr(out), n_polys, _stream()))
    return out


def _shares_arg(share1, share2, rest):
    """AggregateShares(share1, share2) as in the reference, or AggregateShares([s0, s1, ...]) for the whole fold in one call."""
    if share2 is None and isinstance(share1, (list, tuple)):
        return list(share1)
    return [share1, share2] + list(rest)


def _ct_level(ct):
    if ct.dim() != 4 or ct.shape[1] != 2 or not ct.is_contiguous():
        raise _lib.LgpuError("ciphertexts are contiguous (batch, 2, level+1, N) device tensors")
    return ct.shape[2] - 1


def _c1(ct):
    """ct.Value[1] of every ciphertext of a (batch, 2, level+1, N) block; its batch stride is 2 (level+1) N words."""
    return ctypes.c_void_p(ct.data_ptr() + ct[0, 0].numel() * 8)


class PublicKeyGenProtocol:
    """multiparty.PublicKeyGenProtocol (multiparty/keygen_cpk.go). Shares and the CRP are (nQ + nP, N) ringqp.Poly rows."""

    def __init__(self, ctx: Context, samplers: Samplers, sigma: float = 3.2, bound: float = 19.2):
        self.ctx, self.samplers, self.sigma, self.bound = ctx, samplers, sigma, bound
        self.levelQ, self.levelP = len(ctx.Q) - 1, len(ctx.P) - 1

    def SampleCRP(self, crs: Samplers):
        return crs.UniformQP(self.levelQ, self.levelP)[0]

    def GenShare(self, sk, crp, e=None):
        """sk: (nQ + nP, N) NTT + Montgomery; returns e - crp * sk over QP (NTT + Montgomery), keygen_cpk.go:70-83."""
        if e is None:
            e = self.samplers.Gaussian(self.sigma, self.bound)
        share = _torch().empty_like(crp)
        _lib.check(_lib.lib().lgpu_encrypt_zero_sk(self.ctx.h, self.levelQ, self.levelP, _dptr(sk), _dptr(crp), _dptr(e.reshape(1, -1)),
                                                   _dptr(share), 1, 1, 1, _stream()))
        return share

    def AggregateShares(self, share1, share2=None, *rest):
        return aggregate(self.ctx, self.levelQ, self.levelP, _shares_arg(share1, share2, rest))

    def GenPublicKey(self, roundShare, crp):
        """rlwe.PublicKey.Value = (aggregated share, crp) as a (2, nQ + nP, N) tensor, the layout Encryptor.EncryptZeroPk takes."""
        return _torch().stack([roundShare, crp])


class KeySwitchProtocol:
    """multiparty.KeySwitchProtocol (multiparty/keyswitch_sk.go): re-encrypts ciphertexts from the collective key s_in to s_out.
    The smudging noise is DiscreteGaussian(sigma', 6 sigma') with sigma' = sqrt(NoiseFreshSK^2 + sigma_flood^2) (:45-52)."""

    def __init__(self, ctx: Context, samplers: Samplers, sigma_flood: float, noise_fresh_sk: float = 3.2):
        self.ctx, self.samplers = ctx, samplers
        self.sigma = math.sqrt(noise_fresh_sk * noise_fresh_sk + sigma_flood * sigma_flood)
        self.bound = 6 * self.sigma

    def GenShare(self, skInput, skOutput, ct, e=None):
        """ct: (batch, 2, level+1, N) NTT-domain ciphertexts; returns the (batch, level+1, N) shares, keyswitch_sk.go:85-118."""
        level = _ct_level(ct)
        batch = ct.shape[0]
        if e is None:
            e = self.samplers.Gaussian(self.sigma, self.bound, batch)
        share = self.ctx.new_poly(level + 1, batch)
        _lib.check(_lib.lib().lgpu_mp_key_switch_share(self.ctx.h, level, _c1(ct), 2 * (level + 1) * self.ctx.N, _dptr(skInput), _dptr(skOutput),
                                                       _dptr(e), _dptr(share), batch, _stream()))
        return share

    def AggregateShares(self, share1, share2=None, *rest):
        shares = _shares_arg(share1, share2, rest)
        return aggregate(self.ctx, shares[0].shape[-2] - 1, -1, shares)

    def KeySwitch(self, ctIn, combined):
        """(ctIn[0] + combined, ctIn[1]), keyswitch_sk.go:133-147."""
        level = _ct_level(ctIn)
        if combined.shape[-2] != level + 1:
            raise _lib.LgpuError("cannot KeySwitch: share and ciphertext levels do not match")
        out = ctIn.clone()
        c0 = ctIn[:, 0].contiguous()
        self.ctx.ringQ.AtLevel(level).Add(c0, combined, c0)
        out[:, 0] = c0
        return out


class PublicKeySwitchProtocol:
    """multiparty.PublicKeySwitchProtocol (multiparty/keyswitch_pk.go): re-encrypts ciphertexts from the collective key s to a public
    key. The zero encryption draws u from the ternary secret distribution and e0, e1 from the error distribution; the smudging noise
    is DiscreteGaussian(sigma_flood, bound_flood) as given, which the reference's tests take as (8 * 3.2, 6 * 8 * 3.2)."""

    def __init__(self, ctx: Context, samplers: Samplers, sigma_flood: float, bound_flood: float = None, xs_p: float = 2 / 3, xs_h: int = 0,
                 sigma: float = 3.2, bound: float = 19.2):
        self.ctx, self.samplers = ctx, samplers
        self.sigma_flood = sigma_flood
        self.bound_flood = 6 * sigma_flood if bound_flood is None else bound_flood
        self.xs_p, self.xs_h, self.sigma, self.bound = xs_p, xs_h, sigma, bound

    def GenShare(self, sk, pk, ct, u=None, e0=None, e1=None, e_flood=None):
        """sk: (nQ + nP, N); pk: (2, nQ + nP, N); ct: (batch, 2, level+1, N) NTT domain. Returns (batch, 2, level+1, N) shares."""
        level = _ct_level(ct)
        batch = ct.shape[0]
        S = self.samplers
        if u is None:
            u = S.Ternary(self.xs_p, self.xs_h, batch)
        if e0 is None:
            e0 = S.Gaussian(self.sigma, self.bound, batch)
        if e1 is None:
            e1 = S.Gaussian(self.sigma, self.bound, batch)
        if e_flood is None:
            e_flood = S.Gaussian(self.sigma_flood, self.bound_flood, batch)
        share = _torch().empty_like(ct)
        _lib.check(_lib.lib().lgpu_mp_public_key_switch_share(self.ctx.h, level, _c1(ct), 2 * (level + 1) * self.ctx.N, _dptr(sk), _dptr(pk),
                                                              _dptr(u), _dptr(e0), _dptr(e1), _dptr(e_flood), _dptr(share), batch, _stream()))
        return share

    def AggregateShares(self, share1, share2=None, *rest):
        shares = _shares_arg(share1, share2, rest)
        return aggregate(self.ctx, shares[0].shape[-2] - 1, -1, shares, mismatch="cannot AggregateShares: the two shares are at different levelQ")

    def KeySwitch(self, ctIn, combined):
        """(ctIn[0] + combined[0], combined[1]), keyswitch_pk.go:122-134."""
        level = _ct_level(ctIn)
        if combined.shape != ctIn.shape:
            raise _lib.LgpuError("cannot KeySwitch: share and ciphertext levels do not match")
        c0 = ctIn[:, 0].contiguous()
        self.ctx.ringQ.AtLevel(level).Add(c0, combined[:, 0].contiguous(), c0)
        return _torch().stack([c0, combined[:, 1]], dim=1)


def _gadget_layout(ctx: Context, pw2: int):
    """(levelQ, levelP, BaseRNSDecompositionVectorSize, BaseTwoDecompositionVectorSize) at the maximum levels
    (core/rlwe/params.go:520-550)."""
    levelQ, levelP = len(ctx.Q) - 1, len(ctx.P) - 1
    nd = (levelQ + levelP + 1) // (levelP + 1) if levelP >= 0 else levelQ + 1
    if pw2 == 0 or levelP > 0:
        sizes = [1] * nd
    else:
        sizes = [(int(round(math.log2(float(q)))) + pw2 - 1) // pw2 for q in ctx.Q][:nd]
    return levelQ, levelP, nd, sizes


class _KeyGenBase:
    def __init__(self, ctx: Context, samplers: Samplers, pw2: int = 0, sigma: float = 3.2, bound: float = 19.2):
        self.ctx, self.samplers, self.pw2, self.sigma, self.bound = ctx, samplers, pw2, sigma, bound
        self.levelQ, self.levelP, self.nd, self.sizes = _gadget_layout(ctx, pw2)
        self.npw2 = max(self.sizes)
        self.rows = self.levelQ + 1 + self.levelP + 1

    def _sample_crp(self, crs: Samplers, n_keys=None):
        lead = (self.nd, self.npw2) if n_keys is None else (n_keys, self.nd, self.npw2)
        n = 1
        for x in lead:
            n *= x
        return crs.UniformQP(self.levelQ, self.levelP, batch=n).view(*lead, self.rows, self.ctx.N)

    def _gauss(self, lead):
        n = 1
        for x in lead:
            n *= x
        return self.samplers.Gaussian(self.sigma, self.bound, n).view(*lead, self.ctx.N)

    def _struct(self, data, ncomp):
        """lgpu_gadget_ct describing a share's layout; data: [.., n_digits, n_pw2_max, (ncomp,) rows, N]."""
        sizes = (ctypes.c_int * self.nd)(*self.sizes)
        st = _lib.GadgetCtStruct(ctypes.c_void_p(data.data_ptr()), self.levelQ, self.levelP, self.pw2, self.nd, self.npw2, sizes)
        return st, sizes

    def AggregateShares(self, share1, share2=None, *rest):
        return aggregate(self.ctx, self.levelQ, self.levelP, _shares_arg(share1, share2, rest))

    def _gadget(self, data):
        return GadgetCiphertext(self.ctx, data, self.levelQ, self.levelP, self.pw2, self.sizes)


class EvaluationKeyGenProtocol(_KeyGenBase):
    """multiparty.EvaluationKeyGenProtocol (multiparty/keygen_evk.go) at the maximum levels. Shares and CRPs are
    (n_digits, n_pw2_max, nQ + nP, N) tensors; entries with j >= BaseTwoDecompositionVectorSize[i] are unspecified."""

    def SampleCRP(self, crs: Samplers):
        return self._sample_crp(crs)

    def GenShare(self, skIn, skOut, crp, e=None):
        """skIn, skOut: (nQ + nP, N) NTT + Montgomery; returns -crp skOut + e + P 2^(w j) skIn (NTT + Montgomery), :86-183."""
        return self._gen(skIn, skOut, None, crp, e)

    def _gen(self, skIn, skOut, gal_els, crp, e):
        n_keys = 1 if gal_els is None else len(gal_els)
        lead = (self.nd, self.npw2) if gal_els is None else (n_keys, self.nd, self.npw2)
        if tuple(crp.shape) != lead + (self.rows, self.ctx.N):
            raise _lib.LgpuError("crp does not have the share's gadget layout")
        if e is None:
            e = self._gauss(lead)
        share = _torch().empty_like(crp)
        st, _sizes = self._struct(share, 1)
        els = None if gal_els is None else (ctypes.c_uint64 * n_keys)(*[int(g) for g in gal_els])
        _lib.check(_lib.lib().lgpu_mp_evaluation_key_gen_share(self.ctx.h, _dptr(skIn), _dptr(skOut), els, n_keys, _dptr(crp), _dptr(e.contiguous()),
                                                               ctypes.byref(st), _stream()))
        return share

    def GenEvaluationKey(self, share, crp) -> GadgetCiphertext:
        """The aggregated share and the CRP as the two components of an rlwe.EvaluationKey (keygen_evk.go:212-231)."""
        return self._gadget(_torch().stack([share, crp], dim=2).contiguous())


class GaloisKeyGenProtocol(EvaluationKeyGenProtocol):
    """multiparty.GaloisKeyGenProtocol (multiparty/keygen_gal.go), batched over a list of Galois elements: shares and CRPs carry a
    leading key index, (n_keys, n_digits, n_pw2_max, nQ + nP, N)."""

    def SampleCRP(self, crs: Samplers, n_keys: int = 1):
        return self._sample_crp(crs, n_keys)

    def GenShare(self, sk, galEls, crp, e=None):
        """One share per Galois element: EvaluationKeyGen with skOut = AutomorphismNTT(sk, galEl^-1 mod 2N), :48-70."""
        return self._gen(sk, None, list(galEls), crp, e)

    def GenGaloisKeys(self, galEls, share, crp):
        """{galEl: GadgetCiphertext}, the Galois keys the evaluators take."""
        return {int(g): self.GenEvaluationKey(share[k], crp[k]) for k, g in enumerate(galEls)}


class RelinearizationKeyGenProtocol(_KeyGenBase):
    """multiparty.RelinearizationKeyGenProtocol (multiparty/keygen_relin.go), two rounds, at the maximum levels. Round-one shares are
    (n_digits, n_pw2_max, 2, nQ + nP, N), round-two shares (n_digits, n_pw2_max, nQ + nP, N), both in plain (not Montgomery) form."""

    def __init__(self, ctx: Context, samplers: Samplers, pw2: int = 0, sigma: float = 3.2, bound: float = 19.2, xs_p: float = 2 / 3, xs_h: int = 0):
        super().__init__(ctx, samplers, pw2, sigma, bound)
        self.xs_p, self.xs_h = xs_p, xs_h

    def SampleCRP(self, crs: Samplers):
        return self._sample_crp(crs)

    def AllocateShare(self):
        """(ephSk, r1, r2) buffers, as the reference's AllocateShare."""
        torch = _torch()
        N, dev = self.ctx.N, "cuda"
        return (torch.zeros((self.rows, N), dtype=torch.int64, device=dev),
                torch.zeros((self.nd, self.npw2, 2, self.rows, N), dtype=torch.int64, device=dev),
                torch.zeros((self.nd, self.npw2, self.rows, N), dtype=torch.int64, device=dev))

    def GenShareRoundOne(self, sk, crp, u=None, e0=None, e1=None):
        """Returns (ephSk, round-one share), :91-184. u: (N,) ternary; e0, e1: (n_digits, n_pw2_max, N)."""
        if tuple(crp.shape) != (self.nd, self.npw2, self.rows, self.ctx.N):
            raise _lib.LgpuError("crp does not have the share's gadget layout")
        if u is None:
            u = self.samplers.Ternary(self.xs_p, self.xs_h)
        if e0 is None:
            e0 = self._gauss((self.nd, self.npw2))
        if e1 is None:
            e1 = self._gauss((self.nd, self.npw2))
        eph, share, _ = self.AllocateShare()
        st, _sizes = self._struct(share, 2)
        _lib.check(_lib.lib().lgpu_mp_rkg_share_round_one(self.ctx.h, _dptr(sk), _dptr(u.contiguous()), _dptr(crp), _dptr(e0.contiguous()),
                                                          _dptr(e1.contiguous()), _dptr(eph), ctypes.byref(st), _stream()))
        return eph, share

    def GenShareRoundTwo(self, ephSk, sk, round1, e2=None):
        """round1: the aggregated round-one share. Returns the round-two share, :193-234."""
        if tuple(round1.shape) != (self.nd, self.npw2, 2, self.rows, self.ctx.N) or not round1.is_contiguous():
            raise _lib.LgpuError("round1 does not have the share's gadget layout")
        if e2 is None:
            e2 = self._gauss((self.nd, self.npw2))
        share = _torch().empty((self.nd, self.npw2, self.rows, self.ctx.N), dtype=_torch().int64, device=round1.device)
        st1, _s1 = self._struct(round1, 2)
        st2, _s2 = self._struct(share, 1)
        _lib.check(_lib.lib().lgpu_mp_rkg_share_round_two(self.ctx.h, _dptr(ephSk), _dptr(sk), ctypes.byref(st1), _dptr(e2.contiguous()),
                                                          ctypes.byref(st2), _stream()))
        return share

    def GenRelinearizationKey(self, round1, round2) -> GadgetCiphertext:
        """MForm of the aggregated round-two share and of round-one component 1 (:261-276): the degree-1 GadgetCiphertext the evaluators
        take as rlk."""
        torch = _torch()
        data = torch.stack([round2, round1[:, :, 1]], dim=2).contiguous()
        flat = data.view(-1, self.rows, self.ctx.N)
        from .ring import Ring, RING_Q, RING_P
        q = flat[:, : self.levelQ + 1].contiguous()
        Ring(self.ctx, RING_Q, self.levelQ).MForm(q, q)
        flat[:, : self.levelQ + 1] = q
        if self.levelP >= 0:
            p = flat[:, self.levelQ + 1:].contiguous()
            Ring(self.ctx, RING_P, self.levelP).MForm(p, p)
            flat[:, self.levelQ + 1:] = p
        return self._gadget(data)


_MASK64 = (1 << 64) - 1


def _mform(a: int, q: int) -> int:
    """ring.MForm (ring/modular_reduction.go:11-35): a 2^64 mod q in the Barrett form, for any 64-bit a."""
    r = (1 << 128) // q
    mhi = (a * (r & _MASK64)) >> 64
    x = (-(a * (r >> 64) + mhi) * q) & _MASK64
    return x - q if x >= q else x


def _mred_lazy(x: int, y: int, q: int) -> int:
    """ring.MRedLazy (:88-95): x y 2^-64 in [0, 2q), with the reference's 64-bit wrap."""
    lo = (x * y) & _MASK64
    return (((x * y) >> 64) - ((((lo * pow(q, -1, 1 << 64)) & _MASK64) * q) >> 64) + q) & _MASK64


def _mred(x: int, y: int, q: int) -> int:
    r = _mred_lazy(x, y, q)
    return r - q if r >= q else r


def _modexp_montgomery(x: int, e: int, q: int) -> int:
    """ring.ModexpMontgomery (ring/utils.go:58-69)."""
    result = _mform(1, q)
    while e > 0:
        if e & 1:
            result = _mred(result, x, q)
        x = _mred(x, x, q)
        e >>= 1
    return result


def _point(x) -> int:
    x = int(x)
    if not 0 <= x <= _MASK64:
        raise _lib.LgpuError("a ShamirPublicPoint is a 64-bit unsigned integer")
    return x


class Thresholdizer:
    """multiparty.Thresholdizer (multiparty/threshold.go:14-113): t-out-of-N Shamir sharing of a ringqp.Poly secret, at the maximum
    levels. A ShamirPolynomial is a (t, nQ + nP, N) tensor whose block 0 is the secret; a ShamirSecretShare is a (nQ + nP, N) tensor.
    ShamirPublicPoints are Python ints in [0, 2^64)."""

    def __init__(self, ctx: Context, samplers: Samplers):
        self.ctx, self.samplers = ctx, samplers
        self.levelQ, self.levelP = len(ctx.Q) - 1, len(ctx.P) - 1
        self.rows = len(ctx.Q) + len(ctx.P)

    def GenShamirPolynomial(self, threshold: int, sk, coeffs=None):
        """A degree threshold - 1 polynomial with constant term sk (NTT + Montgomery, (nQ + nP, N)) and the other coefficients uniform
        from one UniformQP draw of the party's samplers (coeffs, a (threshold - 1, nQ + nP, N) tensor, replaces the draw), :81-93."""
        if threshold < 1:
            raise _lib.LgpuError("threshold should be >= 1")
        torch = _torch()
        shape = (self.rows, self.ctx.N)
        if tuple(sk.shape) != shape:
            raise _lib.LgpuError("sk is a (nQ + nP, N) tensor")
        poly = torch.empty((threshold,) + shape, dtype=torch.int64, device=sk.device)
        poly[0].copy_(sk)
        if threshold > 1:
            if coeffs is None:
                coeffs = self.samplers.UniformQP(self.levelQ, self.levelP, batch=threshold - 1)
            if tuple(coeffs.shape) != (threshold - 1,) + shape:
                raise _lib.LgpuError("coeffs is a (threshold - 1, nQ + nP, N) tensor")
            poly[1:].copy_(coeffs)
        return poly

    def AllocateThresholdSecretShare(self):
        return self.ctx.new_poly(self.rows)

    def GenShamirSecretShare(self, recipient, secretPoly):
        """The share for one recipient, :102-104."""
        return self.GenShamirSecretShares([recipient], secretPoly)[0]

    def GenShamirSecretShares(self, recipients, secretPoly):
        """The shares for every recipient in one pass (lgpu_mp_shamir_share): a (len(recipients), nQ + nP, N) tensor."""
        pts = [_point(r) for r in recipients]
        if not pts:
            raise _lib.LgpuError("GenShamirSecretShares needs at least one recipient")
        if secretPoly.dim() != 3 or tuple(secretPoly.shape[1:]) != (self.rows, self.ctx.N):
            raise _lib.LgpuError("secretPoly is a (threshold, nQ + nP, N) tensor")
        shares = _torch().empty((len(pts), self.rows, self.ctx.N), dtype=_torch().int64, device=secretPoly.device)
        arr = (ctypes.c_uint64 * len(pts))(*pts)
        _lib.check(_lib.lib().lgpu_mp_shamir_share(self.ctx.h, self.levelQ, self.levelP, _dptr(secretPoly), secretPoly.shape[0], arr, len(pts),
                                                   _dptr(shares), _stream()))
        return shares

    def AggregateShares(self, share1, share2=None, *rest):
        """:106-113, or the whole list of received shares in one call."""
        return aggregate(self.ctx, self.levelQ, self.levelP, _shares_arg(share1, share2, rest), mismatch="cannot AggregateShares: shares level do not match")


class Combiner:
    """multiparty.Combiner (multiparty/threshold.go:115-179): turns a party's aggregated Shamir share into a t-out-of-t additive share
    of the secret. The Lagrange scalars are host work on Python ints, word for word the reference's RNS scalars: `one` = MForm(1),
    lagrangeCoeffs[that] = MulRNSScalar(Inverse(SubRNSScalar(that, this)), that), MulRNSScalar being MRedLazy, so scalars lie in [0, 2q)."""

    def __init__(self, ctx: Context, own, others, threshold: int):
        self.ctx, self.threshold = ctx, threshold
        self.moduli = list(ctx.Q) + list(ctx.P)
        self.one = [_mform(1, q) for q in self.moduli]
        own = _point(own)
        self.lagrangeCoeffs = {}
        for spk in others:
            spk = _point(spk)
            if spk != own:
                self.lagrangeCoeffs[spk] = self._lagrange_coeff(own, spk)

    def _lagrange_coeff(self, this: int, that: int):
        out = []
        for q in self.moduli:
            a, b = that % q, this % q                               # NewRNSScalarFromUInt64
            d = a + q - b if b > a else a - b                       # SubRNSScalar(that, this)
            out.append(_mred_lazy(_modexp_montgomery(d, q - 2, q), a, q))   # Inverse, then MulRNSScalar(., that)
        return out

    def prod(self, activesPoints, ownPoint):
        """The RNS scalar GenAdditiveShare multiplies the share by: 2^64 prod over the first threshold actives other than ownPoint of
        that / (that - ownPoint), in [0, 2q)."""
        if len(activesPoints) < self.threshold:
            raise _lib.LgpuError("cannot GenAdditiveShare: Not enough active players to combine threshold shares")
        own = _point(ownPoint)
        prod = list(self.one)
        for active in activesPoints[: self.threshold]:
            active = _point(active)
            if active != own:
                c = self.lagrangeCoeffs.get(active)
                if c is None:
                    raise _lib.LgpuError("cannot GenAdditiveShare: active point %d is not among the points the Combiner was created with" % active)
                prod = [_mred_lazy(x, y, q) for x, y, q in zip(prod, c, self.moduli)]
        return prod

    def GenAdditiveShare(self, activesPoints, ownPoint, ownShare):
        """MulRNSScalarMontgomery(ownShare, prod) (:148-167) through the existing vector kernel: a (nQ + nP, N) tensor, the party's
        additive share of the secret, to use as its secret key in the N-out-of-N protocols."""
        from .ringqp import Poly, RingQP
        prod = self.prod(activesPoints, ownPoint)
        nq = len(self.ctx.Q)
        if tuple(ownShare.shape) != (len(self.moduli), self.ctx.N):
            raise _lib.LgpuError("ownShare is a (nQ + nP, N) tensor")
        out = _torch().empty_like(ownShare)
        P = (lambda t: t[nq:]) if self.ctx.P else (lambda t: None)
        RingQP(self.ctx).MulRNSScalarMontgomery(Poly(ownShare[:nq], P(ownShare)), prod, Poly(out[:nq], P(out)))
        return out

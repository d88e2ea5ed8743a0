"""Host-side mirror of multiparty/mpbgv on the device (include/lattigo_b200.h, csrc/mp_refresh.cu): encryption to additive shares
(EncToShareProtocol, mpbgv/sharing.go), shares to encryption (ShareToEncProtocol), the masked transform (MaskedTransformProtocol,
mpbgv/transform.go) and the collective refresh built on it (RefreshProtocol, mpbgv/refresh.go), for batches of NTT-domain BGV / BFV
ciphertexts on the Standard ring with paramsIn == paramsOut.

Layouts: ciphertexts are (batch, 2, level+1, N) device tensors, KeySwitch shares, CRPs and their aggregates (batch, level+1, N), an
AdditiveShare (batch, n) words mod t with n = RingT().N() = BGVEncoder.MaxSlots(). Secret keys are (nQ + nP, N) rows, NTT + Montgomery.

Randomness as in lattigo_b200.multiparty: a protocol draws its smudging noise and masks from the party's encryptor.Samplers and the CRP
from a Samplers keyed by the CRS. The masks use a domain of the Philox counter no other sampler uses. Every GenShare also takes its
samples (e, mask) as keyword arguments.

Scales follow the reference: GenShare decodes and encodes the mask of a MaskedTransformFunc with the input ciphertext's scale and stores
it as the share's MetaData; Transform checks the input scale against that MetaData and decodes / encodes with the output ciphertext's
scale, so both are arguments. Results keep the reference's words (see include/lattigo_b200.h)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Optional

from . import _lib
from .bgv_encoder import BGVEncoder
from .encryptor import Samplers
from .multiparty import KeySwitchProtocol, _c1, _ct_level, _shares_arg, aggregate
from .ring import RING_Q, _dptr, _stream


def _torch():
    import torch
    return torch


@dataclass(frozen=True)
class MetaData:
    """The part of rlwe.MetaData these protocols see: Scale (Scale.Uint64()); ciphertexts here are always NTT and batched."""
    Scale: int = 1
    IsNTT: bool = True


@dataclass
class RefreshShare:
    """multiparty.RefreshShare (multiparty/refresh.go): the E2S and S2E KeySwitch shares and the input ciphertext's MetaData."""
    EncToShareShare: object
    ShareToEncShare: object
    MetaData: MetaData


@dataclass
class MaskedTransformFunc:
    """mpbgv.MaskedTransformFunc: Func(coeffs) rewrites a (batch, n) int64 device tensor of uint64 words in place, after DecodeRingT
    when Decode, before EncodeRingT when Encode."""
    Decode: bool
    Func: Callable
    Encode: bool


def NewAdditiveShare(enc: BGVEncoder, batch: int = 1):
    return _torch().zeros((batch, enc.n), dtype=_torch().int64, device="cuda:%d" % enc.ctx.device)


def _words(enc: BGVEncoder, x, what):
    torch = _torch()
    if x.dim() != 2 or x.shape[1] != enc.n or x.dtype != torch.int64 or not x.is_cuda or not x.is_contiguous():
        raise _lib.LgpuError("%s: a contiguous (batch, %d) int64 device tensor" % (what, enc.n))
    return x


def _level_of(p):
    if p.dim() != 3 or not p.is_contiguous():
        raise _lib.LgpuError("shares and CRPs are contiguous (batch, level+1, N) device tensors")
    return p.shape[1] - 1


def DecodeRingT(enc: BGVEncoder, pT, scale: int):
    """encoder.DecodeRingT of every entry of a (batch, n) ring-T block into n uint64 values (as int64 words)."""
    _words(enc, pT, "pT")
    out = _torch().empty_like(pT)
    _lib.check(_lib.lib().lgpu_mpbgv_decode_ring_t(enc.h, _dptr(pT), int(scale) & (2 ** 64 - 1), _dptr(out), pT.shape[0], _stream()))
    return out


def EncodeRingT(enc: BGVEncoder, values, scale: int):
    """encoder.EncodeRingT of n uint64 values (int64 words) per entry into a (batch, n) ring-T block."""
    _words(enc, values, "values")
    out = _torch().empty_like(values)
    _lib.check(_lib.lib().lgpu_mpbgv_encode_ring_t(enc.h, _dptr(values), int(scale) & (2 ** 64 - 1), _dptr(out), values.shape[0], _stream()))
    return out


class EncToShareProtocol:
    """mpbgv.EncToShareProtocol: a KeySwitchProtocol to the zero key plus a ring-T mask per party. The smudging noise is the
    KeySwitchProtocol's DiscreteGaussian(sqrt(NoiseFreshSK^2 + sigma_flood^2), 6 sigma')."""

    def __init__(self, enc: BGVEncoder, samplers: Samplers, sigma_flood: float, noise_fresh_sk: float = 3.2):
        self.enc, self.ctx, self.samplers = enc, enc.ctx, samplers
        self.cks = KeySwitchProtocol(enc.ctx, samplers, sigma_flood, noise_fresh_sk)

    def AllocateShare(self, level: int, batch: int = 1):
        return self.ctx.new_poly(level + 1, batch)

    def SampleMask(self, batch: int = 1):
        """ring.UniformSampler over RingT: (batch, n) words uniform in [0, t) on the party's Samplers."""
        out = NewAdditiveShare(self.enc, batch)
        S = self.samplers
        _lib.check(_lib.lib().lgpu_mpbgv_sample_mask(self.enc.h, S.seed, S._sid(None), _dptr(out), batch, _stream()))
        return out

    def GenShare(self, sk, ct, level: Optional[int] = None, e=None, mask=None):
        """sharing.go:62-71 at min(ct level, level) (level: the public share's level, default the ciphertext's). Returns
        (secretShareOut, publicShareOut): the party's mask and Sub(KeySwitch(sk, 0) share, NTT(RingT2Q(mask)))."""
        ct_level = _ct_level(ct)
        level = ct_level if level is None else min(ct_level, level)
        batch = ct.shape[0]
        if e is None:
            e = self.samplers.Gaussian(self.cks.sigma, self.cks.bound, batch)
        if mask is None:
            mask = self.SampleMask(batch)
        _words(self.enc, mask, "mask")
        share = self.ctx.new_poly(level + 1, batch)
        _lib.check(_lib.lib().lgpu_mpbgv_e2s_share(self.enc.h, level, _c1(ct), 2 * (ct_level + 1) * self.ctx.N, _dptr(sk), _dptr(e), _dptr(mask),
                                                   _dptr(share), batch, _stream()))
        return mask, share

    def AggregateShares(self, share1, share2=None, *rest):
        shares = _shares_arg(share1, share2, rest)
        return aggregate(self.ctx, _level_of(shares[0]), -1, shares)

    def GetShare(self, secretShare, aggregatePublicShare, ct):
        """sharing.go:78-91: RingQ2T(INTT(aggregate + ct[0])) at min(ct level, share level), plus secretShare (ring-T Add) unless it
        is None. Returns the (batch, n) secret share."""
        ct_level = _ct_level(ct)
        level = min(ct_level, _level_of(aggregatePublicShare))
        agg = aggregatePublicShare[:, : level + 1].contiguous()
        batch = ct.shape[0]
        if agg.shape[0] != batch:
            raise _lib.LgpuError("cannot GetShare: the share and the ciphertexts differ in batch")
        if secretShare is not None:
            _words(self.enc, secretShare, "secretShare")
        out = NewAdditiveShare(self.enc, batch)
        _lib.check(_lib.lib().lgpu_mpbgv_e2s_get_share(self.enc.h, level, _dptr(ct), 2 * (ct_level + 1) * self.ctx.N, _dptr(agg),
                                                       _dptr(secretShare) if secretShare is not None else None, _dptr(out), batch, _stream()))
        return out


class ShareToEncProtocol:
    """mpbgv.ShareToEncProtocol: a KeySwitchProtocol from the zero key on the CRP plus the party's secret share."""

    def __init__(self, enc: BGVEncoder, samplers: Samplers, sigma_flood: float, noise_fresh_sk: float = 3.2):
        self.enc, self.ctx, self.samplers = enc, enc.ctx, samplers
        self.cks = KeySwitchProtocol(enc.ctx, samplers, sigma_flood, noise_fresh_sk)

    def AllocateShare(self, level: int, batch: int = 1):
        return self.ctx.new_poly(level + 1, batch)

    def SampleCRP(self, level: int, crs: Samplers, batch: int = 1):
        return crs.Uniform(RING_Q, level, batch)

    def GenShare(self, sk, crp, secretShare, level: Optional[int] = None, e=None):
        """sharing.go:126-143: Add(KeySwitch(0, sk) share on the crp, NTT(RingT2Q(secretShare))) at the crp's level."""
        crp_level = _level_of(crp)
        if level is not None and level != crp_level:
            raise _lib.LgpuError("cannot GenShare: crp and c0ShareOut level must be equal")
        batch = crp.shape[0]
        _words(self.enc, secretShare, "secretShare")
        if secretShare.shape[0] != batch:
            raise _lib.LgpuError("cannot GenShare: the crp and the secret share differ in batch")
        if e is None:
            e = self.samplers.Gaussian(self.cks.sigma, self.cks.bound, batch)
        share = self.ctx.new_poly(crp_level + 1, batch)
        _lib.check(_lib.lib().lgpu_mpbgv_s2e_share(self.enc.h, crp_level, _dptr(crp), _dptr(sk), _dptr(e), _dptr(secretShare), _dptr(share),
                                                   batch, _stream()))
        return share

    def AggregateShares(self, share1, share2=None, *rest):
        shares = _shares_arg(share1, share2, rest)
        return aggregate(self.ctx, _level_of(shares[0]), -1, shares)

    def GetEncryption(self, c0Agg, crp):
        """sharing.go:147-154: the ciphertexts (c0Agg, crp)."""
        if c0Agg.shape != crp.shape:
            raise _lib.LgpuError("cannot GetEncryption: the aggregated share and the crp differ in shape")
        return _torch().stack([c0Agg, crp], dim=1)


class MaskedTransformProtocol:
    """mpbgv.MaskedTransformProtocol with paramsIn == paramsOut: E2S of the input to a mask, an optional MaskedTransformFunc on the mask,
    S2E back to a fresh ciphertext at the CRP's level."""

    def __init__(self, enc: BGVEncoder, samplers: Samplers, sigma_flood: float, noise_fresh_sk: float = 3.2):
        self.enc, self.ctx = enc, enc.ctx
        self.e2s = EncToShareProtocol(enc, samplers, sigma_flood, noise_fresh_sk)
        self.s2e = ShareToEncProtocol(enc, samplers, sigma_flood, noise_fresh_sk)

    def SampleCRP(self, level: int, crs: Samplers, batch: int = 1):
        return self.s2e.SampleCRP(level, crs, batch)

    def _apply(self, transform: Optional[MaskedTransformFunc], mask, scale: int):
        if transform is None:
            return mask
        coeffs = DecodeRingT(self.enc, mask, scale) if transform.Decode else mask.clone()
        transform.Func(coeffs)
        coeffs = coeffs.contiguous()
        return EncodeRingT(self.enc, coeffs, scale) if transform.Encode else coeffs

    def GenShare(self, skIn, skOut, ct, crp, transform: Optional[MaskedTransformFunc] = None, scale: int = 1, level: Optional[int] = None,
                 e_e2s=None, e_s2e=None, mask=None) -> RefreshShare:
        """transform.go:67-109. level: the E2S share's level (default the ciphertext's); scale: ct.Scale, with which the mask is decoded
        and encoded and which the share records as its MetaData."""
        ct_level = _ct_level(ct)
        if level is not None and ct_level < level:
            raise _lib.LgpuError("cannot GenShare: ct[1] level must be at least equal to EncToShareShare level")
        _level_of(crp)
        secret, e2s = self.e2s.GenShare(skIn, ct, level, e=e_e2s, mask=mask)
        m = self._apply(transform, secret, scale)
        s2e = self.s2e.GenShare(skOut, crp, m, e=e_s2e)
        return RefreshShare(e2s, s2e, MetaData(int(scale)))

    def AggregateShares(self, share1, share2=None, *rest) -> RefreshShare:
        """transform.go:112-126, as one fold per component (lgpu_mp_aggregate)."""
        shares = _shares_arg(share1, share2, rest)
        e2s = [s.EncToShareShare for s in shares]
        s2e = [s.ShareToEncShare for s in shares]
        if any(x.shape != e2s[0].shape for x in e2s):
            raise _lib.LgpuError("cannot AggregateShares: all e2s shares must be at the same level")
        if any(x.shape != s2e[0].shape for x in s2e):
            raise _lib.LgpuError("cannot AggregateShares: all s2e shares must be at the same level")
        return RefreshShare(self.e2s.AggregateShares(e2s), self.s2e.AggregateShares(s2e), shares[0].MetaData)

    def Transform(self, ct, transform: Optional[MaskedTransformFunc], crp, share: RefreshShare, scale: int = 1, scale_out: Optional[int] = None):
        """transform.go:129-181: the fresh ciphertexts at the crp's level. scale: ct.Scale (checked against share.MetaData); scale_out:
        ciphertextOut.Scale, used by the transform's Decode / Encode (default scale)."""
        if MetaData(int(scale)) != share.MetaData:
            raise _lib.LgpuError("cannot Transform: input ct.MetaData != share.MetaData")
        if _ct_level(ct) < _level_of(share.EncToShareShare):
            raise _lib.LgpuError("cannot Transform: input ciphertext level must be at least equal to e2s level")
        max_level = _level_of(crp)
        if max_level != _level_of(share.ShareToEncShare):
            raise _lib.LgpuError("cannot Transform: crs level and s2e level must be the same")
        batch = ct.shape[0]
        if crp.shape[0] != batch or share.ShareToEncShare.shape[0] != batch:
            raise _lib.LgpuError("cannot Transform: the ciphertexts, the crp and the share differ in batch")
        mask = self.e2s.GetShare(None, share.EncToShareShare, ct)
        mask = self._apply(transform, mask, scale if scale_out is None else scale_out)
        out = _torch().empty((batch, 2, max_level + 1, self.ctx.N), dtype=_torch().int64, device=ct.device)
        _lib.check(_lib.lib().lgpu_mpbgv_recrypt(self.enc.h, max_level, _dptr(mask), _dptr(share.ShareToEncShare), _dptr(crp), _dptr(out), batch,
                                                 _stream()))
        return out


class RefreshProtocol(MaskedTransformProtocol):
    """mpbgv.RefreshProtocol: MaskedTransformProtocol without a transform, skIn = skOut."""

    def GenShare(self, sk, ct, crp, scale: int = 1, level: Optional[int] = None, e_e2s=None, e_s2e=None, mask=None) -> RefreshShare:
        return super().GenShare(sk, sk, ct, crp, None, scale, level, e_e2s, e_s2e, mask)

    def Finalize(self, ctIn, crp, share: RefreshShare, scale: int = 1):
        return self.Transform(ctIn, None, crp, share, scale)

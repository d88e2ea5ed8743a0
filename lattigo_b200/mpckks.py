"""Host-side mirror of multiparty/mpckks on the device (include/lattigo_b200.h, csrc/mp_refresh.cu): encryption to additive big-integer
shares (EncToShareProtocol, mpckks/sharing.go), shares to encryption (ShareToEncProtocol) and the collective refresh (RefreshProtocol,
mpckks/refresh.go: MaskedLinearTransformationProtocol without a transform), plus GetMinimumLevelForRefresh (mpckks/utils.go), for batches
of NTT-domain CKKS ciphertexts on the Standard ring with paramsIn == paramsOut.

An AdditiveShareBigint is a (batch, dslots, W) int64 device tensor, dslots = 2 slots, W little-endian two's-complement words per value;
W (4 or 8) is fixed by Q at the E2S level (share_words). to_ints / from_ints convert to and from Python ints and sum_shares adds the
parties' shares exactly (the reference's reconstruction rec += share). Samples come from the party's encryptor.Samplers (masks on their
own Philox domain) and the CRP from the CRS's; every GenShare also takes its samples as keyword arguments.

Scales: RefreshProtocol multiplies each mask by defaultScale (big.Float at the encoder's precision, truncated to an integer) and divides
by inputScaleInt (big.Float.Int of ct.Scale, plus 1 when that truncated: the ceiling of a positive non-integer scale), truncating toward
zero as big.Int.Quo does. Both must be integers below 2^128; larger ones are refused. The output scale is defaultScale."""
from __future__ import annotations

import ctypes
import math
from dataclasses import dataclass
from fractions import Fraction
from typing import Optional

from . import _lib
from .encryptor import Samplers
from .multiparty import KeySwitchProtocol, _c1, _ct_level, _shares_arg, aggregate
from .ring import RING_Q, Context, _dptr, _stream


def _torch():
    import torch
    return torch


def GetMinimumLevelForRefresh(lam: int, scale: float, nParties: int, moduli):
    """mpckks/utils.go: (minLevel, logBound, ok)."""
    logBound = lam + int(math.ceil(math.log2(float(scale))))
    maxBound = math.ceil(float(logBound) + math.log2(float(nParties)))
    minLevel, logQ, i = -1, 0.0, 0
    while logQ < maxBound:
        if i >= len(moduli):
            return 0, 0, False
        logQ += math.log2(float(moduli[i]))
        minLevel += 1
        i += 1
    if len(moduli) < minLevel:
        return 0, 0, False
    return minLevel, logBound, True


def share_words(ctx: Context, level: int) -> int:
    """Words per share value at an E2S level: the smallest of 4 and 8 with 64 W >= sum of bits(q_i) + 16 (sums of up to 2^15 shares stay
    exact); refused past 8."""
    bits = sum(int(q).bit_length() for q in ctx.Q[: level + 1]) + 16
    if bits <= 256:
        return 4
    if bits <= 512:
        return 8
    raise _lib.LgpuError("the E2S level's Q needs more than 8 words per share value")


def to_ints(words):
    """(batch, dslots, W) words -> lists of Python ints."""
    import numpy as np
    a = words.detach().cpu().numpy().view(np.uint64)
    W = a.shape[-1]
    out = []
    for row in a.reshape(-1, a.shape[-2], W):
        vals = []
        for v in row:
            x = sum(int(w) << (64 * k) for k, w in enumerate(v))
            vals.append(x - (1 << (64 * W)) if x >> (64 * W - 1) else x)
        out.append(vals)
    return out


def from_ints(values, W: int, device="cuda"):
    """Lists of Python ints -> (batch, dslots, W) two's-complement words."""
    import numpy as np
    M = (1 << 64) - 1
    arr = np.array([[[((v % (1 << (64 * W))) >> (64 * k)) & M for k in range(W)] for v in row] for row in values], dtype=np.uint64)
    return _torch().from_numpy(arr.view(np.int64)).to(device)


def sum_shares(shares):
    """The exact sum of the parties' AdditiveShareBigint tensors."""
    W = shares[0].shape[-1]
    tot = None
    for s in shares:
        v = to_ints(s)
        tot = v if tot is None else [[a + b for a, b in zip(x, y)] for x, y in zip(tot, v)]
    return from_ints(tot, W, shares[0].device)


def default_scale_int(scale, prec: int = 53) -> int:
    """new(big.Float).SetPrec(prec).Set(scale).Int(nil): the scale rounded to prec bits (to nearest even), truncated."""
    f = Fraction(scale)
    if f <= 0:
        raise _lib.LgpuError("scales are positive")
    e = f.numerator.bit_length() - f.denominator.bit_length()
    if Fraction(2) ** e > f:
        e -= 1                                          # f in [2^e, 2^(e+1))
    unit = Fraction(2) ** (e - prec + 1)
    r = round(f / unit) * unit                          # Fraction rounding is half to even
    return r.numerator // r.denominator


def input_scale_int(scale) -> int:
    """big.Float.Int of a positive scale (truncation), plus 1 when it truncated: the ceiling."""
    f = Fraction(scale)
    n = f.numerator // f.denominator
    return n + 1 if n < f else n


def _scales(d: int, s: int):
    if not (0 < d < 1 << 128 and 0 < s < 1 << 128):
        raise _lib.LgpuError("defaultScale and inputScaleInt must be positive integers below 2^128")
    M = (1 << 64) - 1
    return (ctypes.c_uint64 * 4)(d & M, d >> 64, s & M, s >> 64)


def _level_of(p):
    if p.dim() != 3 or not p.is_contiguous():
        raise _lib.LgpuError("shares and CRPs are contiguous (batch, level+1, N) device tensors")
    return p.shape[1] - 1


def _big(x, dslots, what):
    torch = _torch()
    if x.dim() != 3 or x.shape[1] != dslots or x.shape[2] not in (4, 8) or x.dtype != torch.int64 or not x.is_cuda or not x.is_contiguous():
        raise _lib.LgpuError("%s: a contiguous (batch, %d, W) int64 device tensor, W = 4 or 8" % (what, dslots))
    return x


@dataclass(frozen=True)
class MetaData:
    """The part of rlwe.MetaData these protocols see: Scale and LogSlots; ciphertexts are NTT, batched, not Montgomery."""
    Scale: Fraction
    LogSlots: int


@dataclass
class RefreshShare:
    EncToShareShare: object
    ShareToEncShare: object
    MetaData: MetaData


class EncToShareProtocol:
    """mpckks.EncToShareProtocol. The smudging noise is the KeySwitchProtocol's DiscreteGaussian(sqrt(NoiseFreshSK^2 + sigma^2), 6 sigma')."""

    def __init__(self, ctx: Context, samplers: Samplers, sigma_flood: float, noise_fresh_sk: float = 3.2):
        self.ctx, self.samplers = ctx, samplers
        self.cks = KeySwitchProtocol(ctx, samplers, sigma_flood, noise_fresh_sk)

    def AllocateShare(self, level: int, batch: int = 1):
        return self.ctx.new_poly(level + 1, batch)

    def SampleMask(self, logSlots: int, logBound: int, W: int, batch: int = 1):
        dslots = 2 << logSlots
        out = _torch().empty((batch, dslots, W), dtype=_torch().int64, device="cuda:%d" % self.ctx.device)
        S = self.samplers
        _lib.check(_lib.lib().lgpu_mpckks_sample_mask(self.ctx.h, logSlots, logBound, W, S.seed, S._sid(None), _dptr(out), batch, _stream()))
        return out

    def GenShare(self, sk, logBound: int, ct, logSlots: int, level: Optional[int] = None, e=None, mask=None):
        """sharing.go GenShare at min(ct level, level). Returns (secretShareOut, publicShareOut)."""
        ct_level = _ct_level(ct)
        level = ct_level if level is None else min(ct_level, level)
        batch = ct.shape[0]
        W = share_words(self.ctx, level)
        if e is None:
            e = self.samplers.Gaussian(self.cks.sigma, self.cks.bound, batch)
        if mask is None:
            mask = self.SampleMask(logSlots, logBound, W, batch)
        _big(mask, 2 << logSlots, "mask")
        share = self.ctx.new_poly(level + 1, batch)
        _lib.check(_lib.lib().lgpu_mpckks_e2s_share(self.ctx.h, level, logSlots, logBound, _c1(ct), 2 * (ct_level + 1) * self.ctx.N, _dptr(sk),
                                                    _dptr(e), _dptr(mask), mask.shape[2], _dptr(share), batch, _stream()))
        return mask, share

    def AggregateShares(self, share1, share2=None, *rest):
        shares = _shares_arg(share1, share2, rest)
        return aggregate(self.ctx, _level_of(shares[0]), -1, shares)

    def GetShare(self, secretShare, aggregatePublicShare, ct, logSlots: int):
        """sharing.go GetShare: PolyToBigintCentered(INTT(aggregate + ct[0])) (+ secretShare), at min(ct level, share level)."""
        ct_level = _ct_level(ct)
        level = min(ct_level, _level_of(aggregatePublicShare))
        agg = aggregatePublicShare[:, : level + 1].contiguous()
        batch, dslots = ct.shape[0], 2 << logSlots
        W = share_words(self.ctx, level)
        if secretShare is not None:
            _big(secretShare, dslots, "secretShare")
            W = secretShare.shape[2]
        out = _torch().empty((batch, dslots, W), dtype=_torch().int64, device=ct.device)
        _lib.check(_lib.lib().lgpu_mpckks_e2s_get_share(self.ctx.h, level, logSlots, _dptr(ct), 2 * (ct_level + 1) * self.ctx.N, _dptr(agg),
                                                        _dptr(secretShare) if secretShare is not None else None, W, _dptr(out), batch, _stream()))
        return out


class ShareToEncProtocol:
    """mpckks.ShareToEncProtocol."""

    def __init__(self, ctx: Context, samplers: Samplers, sigma_flood: float, noise_fresh_sk: float = 3.2):
        self.ctx, self.samplers = ctx, samplers
        self.cks = KeySwitchProtocol(ctx, samplers, sigma_flood, noise_fresh_sk)

    def AllocateShare(self, level: int, batch: int = 1):
        return self.ctx.new_poly(level + 1, batch)

    def SampleCRP(self, level: int, crs: Samplers, batch: int = 1):
        return crs.Uniform(RING_Q, level, batch)

    def GenShare(self, sk, crp, logSlots: int, secretShare, level: Optional[int] = None, e=None, _scale=None):
        """sharing.go GenShare: Add(KeySwitch(0, sk) share on the crp, NTT(SetCoefficientsBigint(secretShare)))."""
        crp_level = _level_of(crp)
        if level is not None and level != crp_level:
            raise _lib.LgpuError("cannot GenShare: crs and c0ShareOut level must be equal")
        batch = crp.shape[0]
        _big(secretShare, 2 << logSlots, "secretShare")
        if e is None:
            e = self.samplers.Gaussian(self.cks.sigma, self.cks.bound, batch)
        share = self.ctx.new_poly(crp_level + 1, batch)
        _lib.check(_lib.lib().lgpu_mpckks_s2e_share(self.ctx.h, crp_level, logSlots, _dptr(crp), _dptr(sk), _dptr(e), _dptr(secretShare),
                                                    secretShare.shape[2], _scale, _dptr(share), batch, _stream()))
        return share

    def AggregateShares(self, share1, share2=None, *rest):
        shares = _shares_arg(share1, share2, rest)
        return aggregate(self.ctx, _level_of(shares[0]), -1, shares)

    def GetEncryption(self, c0Agg, crp):
        if _level_of(c0Agg) != _level_of(crp):
            raise _lib.LgpuError("cannot GetEncryption: c0Agg level must be equal to crs level")
        return _torch().stack([c0Agg, crp], dim=1)


class RefreshProtocol:
    """mpckks.RefreshProtocol (MaskedLinearTransformationProtocol with transform == nil, paramsIn == paramsOut)."""

    def __init__(self, ctx: Context, samplers: Samplers, sigma_flood: float, default_scale, prec: int = 53, noise_fresh_sk: float = 3.2):
        self.ctx = ctx
        self.e2s = EncToShareProtocol(ctx, samplers, sigma_flood, noise_fresh_sk)
        self.s2e = ShareToEncProtocol(ctx, samplers, sigma_flood, noise_fresh_sk)
        self.default_scale = Fraction(default_scale)
        self.defaultScale = default_scale_int(default_scale, prec)

    def SampleCRP(self, level: int, crs: Samplers, batch: int = 1):
        return self.s2e.SampleCRP(level, crs, batch)

    def GenShare(self, sk, logBound: int, ct, crp, scale, logSlots: int, level: Optional[int] = None, e_e2s=None, e_s2e=None,
                 mask=None) -> RefreshShare:
        """transform.go GenShare: E2S at min(ct level, level), the mask times defaultScale / inputScaleInt, S2E at the crp's level."""
        ct_level = _ct_level(ct)
        if level is not None and ct_level < level:
            raise _lib.LgpuError("cannot GenShare: ct[1] level must be at least equal to EncToShareShare level")
        sc = _scales(self.defaultScale, input_scale_int(scale))
        _level_of(crp)
        secret, e2s = self.e2s.GenShare(sk, logBound, ct, logSlots, level, e=e_e2s, mask=mask)
        s2e = self.s2e.GenShare(sk, crp, logSlots, secret, e=e_s2e, _scale=sc)
        return RefreshShare(e2s, s2e, MetaData(Fraction(scale), logSlots))

    def AggregateShares(self, share1, share2=None, *rest) -> RefreshShare:
        shares = _shares_arg(share1, share2, rest)
        e2s = [s.EncToShareShare for s in shares]
        s2e = [s.ShareToEncShare for s in shares]
        if any(x.shape != e2s[0].shape for x in e2s):
            raise _lib.LgpuError("cannot AggregateShares: all e2s shares must be at the same level")
        if any(x.shape != s2e[0].shape for x in s2e):
            raise _lib.LgpuError("cannot AggregateShares: all s2e shares must be at the same level")
        return RefreshShare(self.e2s.AggregateShares(e2s), self.s2e.AggregateShares(s2e), shares[0].MetaData)

    def Finalize(self, ct, crp, share: RefreshShare, scale, logSlots: int):
        """transform.go Transform with transform == nil: the fresh ciphertexts at the crp's level; their scale is default_scale."""
        ct_level = _ct_level(ct)
        lvl_e2s = _level_of(share.EncToShareShare)
        if ct_level < lvl_e2s:
            raise _lib.LgpuError("cannot Transform: input ciphertext level must be at least equal to e2s level")
        if MetaData(Fraction(scale), logSlots) != share.MetaData:
            raise _lib.LgpuError("cannot Transform: input ciphertext MetaData is not equal to share.MetaData")
        max_level = _level_of(crp)
        if max_level != _level_of(share.ShareToEncShare):
            raise _lib.LgpuError("cannot Transform: crs level and s2e level must be the same")
        sc = _scales(self.defaultScale, input_scale_int(scale))
        batch = ct.shape[0]
        level = min(ct_level, lvl_e2s)
        agg = share.EncToShareShare[:, : level + 1].contiguous()
        out = _torch().empty((batch, 2, max_level + 1, self.ctx.N), dtype=_torch().int64, device=ct.device)
        _lib.check(_lib.lib().lgpu_mpckks_refresh_finalize(self.ctx.h, level, logSlots, _dptr(ct), 2 * (ct_level + 1) * self.ctx.N, _dptr(agg),
                                                           max_level, _dptr(share.ShareToEncShare), _dptr(crp), share_words(self.ctx, level),
                                                           sc, _dptr(out), batch, _stream()))
        return out

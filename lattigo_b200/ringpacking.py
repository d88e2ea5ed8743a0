"""Host-side mirror of core/rlwe/ring_packing.go (RingPackingEvaluator.Expand, Pack, Extract, Repack) and of the key lists of
core/rlwe/ring_packing_keys.go, bound to the C ABI, on a single ring degree (the reference's MinLogN == MaxLogN == ctx.logN).
Ciphertexts are degree-1 contiguous int64 CUDA tensors of shape (2, level+1, N) or (batch, 2, level+1, N); is_ntt plays the role of
the reference's MetaData.IsNTT. One set of Galois keys serves the whole batch. Results are always in the NTT domain."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Tuple

from . import _lib
from .ring import Context, _dptr, _stream
from .rlwe import GadgetCiphertext, _bs


def _nthroot(ctx: Context) -> int:
    return (4 if ctx.ring_type == 1 else 2) * ctx.N


def GaloisElementsForExpand(ctx: Context, logN: int) -> List[int]:
    """ring_packing_keys.go:143-153."""
    return [_nthroot(ctx) // (2 << i) + 1 for i in range(logN)]


def GaloisElementsForPack(ctx: Context, logGap: int) -> List[int]:
    """ring_packing_keys.go:156-180; its panics are ValueErrors."""
    if logGap > ctx.logN or logGap < 0:
        raise ValueError("cannot GaloisElementsForPack: logGap > logN || logGap < 0")
    m = _nthroot(ctx)
    gal = [pow(5, (1 << i) & (m - 1), m) for i in range(logGap)]
    if ctx.ring_type != 0:
        raise ValueError("cannot GaloisElementsForPack: invalid ring type")
    if logGap == ctx.logN:
        gal.append(m - 1)                           # GaloisElementOrderTwoOrthogonalSubgroup
    return gal


def getMinimumGap(keys: List[int]) -> Tuple[int, int]:
    """ring_packing.go:812-845: (gap, logGap), logGap the 2-adic valuation of the smallest consecutive difference (the scan stops at
    a difference of 1). A single key gives gap = 2^63 - 1, logGap = 0."""
    gap, logGap = 0x7FFFFFFFFFFFFFFF, 0
    for i in range(1, len(keys)):
        a, b = keys[i - 1], keys[i]
        if a > b:
            raise ValueError("invalid index list: element must be sorted from smallest to largest")
        if a == b:
            raise ValueError("invalid index list: contains duplicated elements")
        gap = min(gap, b - a)
        if gap == 1:
            break
    while gap & 1 == 0:
        logGap += 1
        gap >>= 1
    return gap, logGap


class RingPackingEvaluator:
    """rlwe.RingPackingEvaluator with MinLogN == MaxLogN == ctx.logN. extract_keys / repack_keys: {galEl: GadgetCiphertext}
    (RingPackingEvaluationKey.ExtractKeys / RepackKeys at that degree; see GaloisElementsForExpand / GaloisElementsForPack)."""

    def __init__(self, ctx: Context, extract_keys: Dict[int, GadgetCiphertext], repack_keys: Dict[int, GadgetCiphertext]):
        self.ctx = ctx
        self._extract = _lib.GaloisKeys(extract_keys)
        self._repack = _lib.GaloisKeys(repack_keys)

    def Expand(self, ct, logGap: int, is_ntt: bool = True) -> Dict[int, object]:
        """:457-571. Returns {j: ciphertext} for the N / 2^logGap multiples j of 2^logGap, each encrypting coefficient j of ct at
        X^0, in the NTT domain whatever is_ntt (the reference's quirk). The values are views of one (batch, S, 2, level+1, N) block."""
        import torch
        b, _ = _bs(ct, 3)
        level = ct.shape[-2] - 1
        if not 0 <= logGap <= self.ctx.logN:
            raise ValueError("Expand: logGap out of range [0, LogN]")
        S = self.ctx.N >> logGap
        out = torch.empty((b, S, 2, level + 1, self.ctx.N), dtype=torch.int64, device=ct.device)
        _lib.check(_lib.lib().lgpu_ring_packing_expand(self.ctx.h, level, _dptr(ct), 1 if is_ntt else 0, logGap, ctypes.byref(self._extract.gks),
                                                       _dptr(out), b, _stream()))
        batched = ct.dim() == 4
        return {k << logGap: (out[:, k] if batched else out[0, k]) for k in range(S)}

    def Pack(self, cts: Dict[int, object], inputLogGap: int, zeroGarbageSlots: bool, is_ntt: bool = True):
        """:600-770. cts: {index: ciphertext}, all of one shape; the inputs are not modified. Returns the packed ciphertext (NTT)."""
        import torch
        if len(cts) == 0:
            raise _lib.LgpuError("len(cts) = 0")
        keys = sorted(cts)
        first = cts[keys[0]]
        batched = first.dim() == 4
        stacked = torch.stack([cts[k] for k in keys], dim=1 if batched else 0).contiguous()
        if not batched:
            stacked = stacked.unsqueeze(0)
        b, level = stacked.shape[0], stacked.shape[-2] - 1
        out = torch.empty((b, 2, level + 1, self.ctx.N), dtype=torch.int64, device=first.device)
        idx = (ctypes.c_int * len(keys))(*keys)
        _lib.check(_lib.lib().lgpu_ring_packing_pack(self.ctx.h, level, _dptr(stacked), 1 if is_ntt else 0, idx, len(keys), inputLogGap,
                                                     1 if zeroGarbageSlots else 0, ctypes.byref(self._repack.gks), _dptr(out), b, _stream()))
        return out if batched else out[0]

    def Extract(self, ct, idx, is_ntt: bool = True) -> Dict[int, object]:
        """:56-171 with logNFactor = 0: Expand(ct, logGap of getMinimumGap(sorted idx)) restricted to idx."""
        keys = sorted(idx)
        try:
            _, logGap = getMinimumGap(keys)
        except ValueError as e:
            raise ValueError("getMinimumGap: %s" % e) from None
        cts = self.Expand(ct, logGap, is_ntt)
        out = {}
        for j in keys:
            if j not in cts:
                raise ValueError("invalid ciphertexts map: index i+j*(NFactor*gap)=%d is nil" % (j * (1 << logGap)))
            out[j] = cts[j]
        return out

    def Repack(self, cts: Dict[int, object], is_ntt: bool = True):
        """:273-374 with logNFactor = 0: Pack(cts, LogN, True)."""
        return self.Pack(cts, self.ctx.logN, True, is_ntt)

"""bgv.Encoder (schemes/bgv/encoder.go; BFV uses the same encoder) bound to the C ABI (lgpu_bgv_encoder_create / lgpu_bgv_encode /
lgpu_bgv_decode, csrc/bgv_encoder.cu): batched Encode / Embed of integer slot values into plaintext rows and Decode back, bit for bit the
reference's words. Plaintexts are int64 CUDA tensors (batch, rows, N) (bit pattern of uint64); values are int64 / uint64 arrays or tensors
(batch, n) or (n,); decoded values come back as int64 CUDA tensors (the uint64 bit pattern unless signed)."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .ring import Context, _stream

ENC_NTT, ENC_MONTGOMERY, ENC_COEFFS, ENC_SIGNED, ENC_SCALE_UP = 1, 2, 4, 8, 16


def plaintext_slots(N: int, t: int) -> int:
    """RingT().N() of bgv.NewParameters (params.go:119-129): min(N, order / 2), order the largest power of two with t = 1 mod order."""
    order = 1 << t.bit_length()
    while order and t & (order - 1) != 1:
        order >>= 1
    return min(N, order >> 1)


def _vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class BGVEncoder:
    """bgv.Encoder for one context (ring.Standard) and plaintext modulus t: ring T and permuteMatrix live on the device once."""

    def __init__(self, ctx: Context, t: int):
        self.ctx = ctx
        self.t = int(t)
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().lgpu_bgv_encoder_create(ctx.h, self.t, ctypes.byref(h)))
        self.h = h
        self.n = plaintext_slots(ctx.N, self.t)

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().lgpu_bgv_encoder_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def MaxSlots(self) -> int:
        return self.n

    def PlaintextModulus(self) -> int:
        return self.t

    def _input(self, values):
        """(batch, n) int64 device tensor of the words, and the SIGNED flag (int64 input) -- uint64 arrays keep their bit pattern."""
        import torch
        if isinstance(values, torch.Tensor):
            signed = values.dtype != torch.uint64
            t = values.to(torch.int64) if signed else values.view(torch.int64)
        else:
            a = np.asarray(values)
            signed = a.dtype != np.uint64
            a = np.ascontiguousarray(a.astype(np.int64) if signed else a.view(np.int64))
            t = torch.from_numpy(a)
        single = t.dim() == 1
        t = t.to(device="cuda:%d" % self.ctx.device)
        return (t.reshape(1, -1) if single else t).contiguous(), signed, single

    def _encode(self, values, flags, level, scale, level_p):
        v, signed, single = self._input(values)
        batch, n = v.shape
        N = self.ctx.N
        rows = level + 1 + level_p + 1
        out = self.ctx.new_poly(rows, batch)
        out_p = ctypes.c_void_p(out.data_ptr() + 8 * (level + 1) * N) if level_p >= 0 else None
        flags |= ENC_SIGNED if signed else 0
        _lib.check(_lib.lib().lgpu_bgv_encode(self.h, _vp(v), n, flags, int(scale) & (2 ** 64 - 1), level, _vp(out), level_p, out_p, batch,
                                              n, rows * N, rows * N, _stream()))
        return out[0] if single else out

    def Encode(self, values, level: int, scale: int = 1, ntt: bool = True, montgomery: bool = False, batched: bool = True):
        """Encode (encoder.go:140-199) into (batch, level+1, N): with batched, EncodeRingT + RingT2Q(scaleUp) of n <= MaxSlots values;
        otherwise n <= N values as coefficients (IsMontgomery ignored, as in the reference)."""
        flags = ENC_SCALE_UP | (ENC_NTT if ntt else 0) | (ENC_MONTGOMERY if montgomery else 0) | (0 if batched else ENC_COEFFS)
        return self._encode(values, flags, level, scale, -1)

    def Embed(self, values, level: int, scale: int = 1, ntt: bool = True, montgomery: bool = False, level_p: int = -1):
        """Embed (encoder.go:335-337): EncodeRingT + RingT2Q without the t^-1 scaling, into (batch, level+1 [+ level_p+1], N): the Q rows,
        then the P rows of the ringqp.Poly when level_p >= 0."""
        flags = (ENC_NTT if ntt else 0) | (ENC_MONTGOMERY if montgomery else 0)
        return self._encode(values, flags, level, scale, level_p)

    def Decode(self, pt, scale: int = 1, ntt: bool = True, batched: bool = True, signed: bool = False, out=None):
        """Decode (encoder.go:471-521) of (batch, level+1, N) plaintexts into (batch, MaxSlots) values, or (batch, N) with batched False.
        Signed coefficient decoding writes only the first MaxSlots words of each entry (the reference's loop bound); the rest of `out`
        (zeros when it is allocated here) is left as it was."""
        import torch
        single = pt.dim() == 2
        p = pt.reshape(1, *pt.shape) if single else pt
        assert p.is_cuda and p.is_contiguous() and p.dtype == torch.int64
        batch, rows, N = p.shape
        n = self.n if batched else N
        if out is None:
            out = torch.zeros((batch, n), dtype=torch.int64, device=p.device)
        assert out.is_contiguous() and out.dtype == torch.int64 and tuple(out.shape) == (batch, n)
        flags = (ENC_NTT if ntt else 0) | (0 if batched else ENC_COEFFS) | (ENC_SIGNED if signed else 0)
        _lib.check(_lib.lib().lgpu_bgv_decode(self.h, _vp(p), rows - 1, flags, int(scale) & (2 ** 64 - 1), _vp(out), batch, rows * N, n,
                                              _stream()))
        return out[0] if single else out

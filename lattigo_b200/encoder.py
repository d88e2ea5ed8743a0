"""ckks.Encoder (schemes/ckks/encoder.go) on the prec <= 53 path, bound to the C ABI (lgpu_ckks_encode / lgpu_ckks_decode, csrc/encoder.cu):
batched Embed / Encode into plaintext rows and DecodePublic back to slot values, bit for bit the reference's on the same rotGroup / roots
tables. Plaintexts are int64 CUDA tensors (batch, rows, N) (bit pattern of uint64); values are complex128 / float64 tensors or arrays."""
from __future__ import annotations

import ctypes
import math

import numpy as np

from . import _lib
from .ring import Context, _stream

ENC_NTT, ENC_MONTGOMERY, ENC_COEFFS = 1, 2, 4


def rot_group(m: int):
    """Encoder.rotGroup (encoder.go:83-112): 5^i mod m for i < m/4."""
    out, f = [], 1
    for _ in range(m >> 2):
        out.append(f)
        f = f * 5 & (m - 1)
    return out


def roots_complex128(m: int):
    """GetRootsComplex128(m) (schemes/ckks/utils.go:53-77): cosines of the first quarter, the rest by its symmetries. The Go shim passes
    the Go encoder's own table instead, so results never depend on how this host's cosine rounds."""
    roots = [0j] * (m + 1)
    quarm = m >> 2
    angle = 2 * 3.141592653589793 / float(m)
    for i in range(quarm):
        roots[i] = complex(math.cos(angle * float(i)), 0)
    for i in range(quarm):
        roots[quarm - i] += complex(0, roots[i].real)
    for i in range(1, quarm + 1):
        roots[i + quarm] = complex(-roots[quarm - i].real, roots[quarm - i].imag)
        roots[i + 2 * quarm] = -roots[i]
        roots[i + 3 * quarm] = complex(roots[quarm - i].real, -roots[quarm - i].imag)
    roots[m] = roots[0]
    return roots


def _vp(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class Encoder:
    """ckks.Encoder for one context (ring.Standard): rotGroup and the complex128 roots of unity live on the device once."""

    def __init__(self, ctx: Context):
        import torch
        self.ctx = ctx
        self.m = 2 * ctx.N
        dev = "cuda:%d" % ctx.device
        self.rot_group = torch.tensor(rot_group(self.m), dtype=torch.int64, device=dev)
        self.roots = torch.tensor(np.array(roots_complex128(self.m), dtype=np.complex128), device=dev)

    def _input(self, values, dtype):
        import torch
        t = values if isinstance(values, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(values, dtype=dtype)))
        single = t.dim() == 1
        t = t.to(device="cuda:%d" % self.ctx.device, dtype=torch.complex128 if dtype == np.complex128 else torch.float64)
        return (t.reshape(1, -1) if single else t).contiguous(), single

    def _encode(self, values, dtype, flags, level, scale, level_p, log_slots):
        v, single = self._input(values, dtype)
        batch, n = v.shape
        N = self.ctx.N
        rows = level + 1 + level_p + 1
        out = self.ctx.new_poly(rows, batch)
        out_p = ctypes.c_void_p(out.data_ptr() + 8 * (level + 1) * N) if level_p >= 0 else None
        _lib.check(_lib.lib().lgpu_ckks_encode(self.ctx.h, _vp(v), n, log_slots, float(scale), flags, _vp(self.rot_group), _vp(self.roots),
                                               level, _vp(out), level_p, out_p, batch, n, rows * N, rows * N, _stream()))
        return out[0] if single else out

    def Encode(self, values, level: int, scale: float, ntt: bool = True, montgomery: bool = False, level_p: int = -1, log_slots=None):
        """Embed (IsBatched) of (batch, n) or (n,) complex values, n <= 2^log_slots (default N/2 slots), zero-padded. Returns
        (batch, level+1 [+ level_p+1], N): the Q rows, then the P rows of the ringqp.Poly when level_p >= 0."""
        ls = self.ctx.logN - 1 if log_slots is None else log_slots
        flags = (ENC_NTT if ntt else 0) | (ENC_MONTGOMERY if montgomery else 0)
        return self._encode(values, np.complex128, flags, level, scale, level_p, ls)

    def EncodeCoeffs(self, values, level: int, scale: float, ntt: bool = True):
        """Encode with IsBatched = false: n <= N float64 values as coefficients (Float64ToFixedPointCRT), then the NTT when ntt."""
        return self._encode(values, np.float64, ENC_COEFFS | (ENC_NTT if ntt else 0), level, scale, -1, 0)

    def _decode(self, pt, scale, log_slots, flags, logprec, coeffs):
        import torch
        single = pt.dim() == 2
        p = pt.reshape(1, *pt.shape) if single else pt
        assert p.is_cuda and p.is_contiguous() and p.dtype == torch.int64
        batch, rows, N = p.shape
        n = N if coeffs else 1 << log_slots
        out = torch.empty((batch, n), dtype=torch.float64 if coeffs else torch.complex128, device=p.device)
        _lib.check(_lib.lib().lgpu_ckks_decode(self.ctx.h, _vp(p), rows - 1, log_slots, float(scale), flags, float(logprec), _vp(self.rot_group),
                                               _vp(self.roots), _vp(out), batch, rows * N, n, _stream()))
        return out[0] if single else out

    def Decode(self, pt, scale: float, log_slots: int, ntt: bool = True, logprec: float = 0):
        """DecodePublic of (batch, level+1, N) plaintexts into complex128 (batch, 2^log_slots); logprec != 0 rounds to 2^-logprec."""
        return self._decode(pt, scale, log_slots, ENC_NTT if ntt else 0, logprec, False)

    def DecodeCoeffs(self, pt, scale: float, ntt: bool = True):
        """Decode of an IsBatched = false plaintext: float64 (batch, N) coefficients divided by the scale."""
        return self._decode(pt, scale, self.ctx.logN - 1, ENC_COEFFS | (ENC_NTT if ntt else 0), 0, True)

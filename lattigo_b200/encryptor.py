"""Host-side mirror of the encryptor / key-generator inner loops and the samplers (include/lattigo_b200.h, csrc/encrypt.cu,
csrc/keygen.cu): rlwe.Encryptor.EncryptZero (core/rlwe/encryptor.go:170-430), rlwe.KeyGenerator.GenEvaluationKey
(core/rlwe/keygenerator.go:261-330) and GenGaloisKeysNew (:123-209), ring.{Uniform,Ternary,Gaussian}Sampler."""
from __future__ import annotations

import ctypes
import math

from . import _lib
from .ring import Context, RING_Q, RING_P, _dptr, _stream
from .rlwe import GadgetCiphertext


class Samplers:
    """Device samplers: the reference's distributions on counter-based streams keyed by (seed, stream id). Every call takes
    one stream id, stream_id if given and otherwise the next of 1, 2, 3, ...; UniformQP draws both rings on that id."""

    def __init__(self, ctx: Context, seed: int):
        self.ctx, self.seed = ctx, seed & 0xFFFFFFFFFFFFFFFF
        self._next = 0

    def _sid(self, stream_id):
        if stream_id is None:
            self._next += 1
            return self._next
        return stream_id

    def Uniform(self, ring: int, level: int, batch: int = 1, stream_id=None):
        out = self.ctx.new_poly(level + 1, batch)
        _lib.check(_lib.lib().lgpu_sample_uniform(self.ctx.h, ring, level, self.seed, self._sid(stream_id), _dptr(out), batch, (level + 1) * self.ctx.N, _stream()))
        return out

    def UniformQP(self, levelQ: int, levelP: int, batch: int = 1, stream_id=None):
        """A uniform ringqp.Poly block (batch, levelQ+1 + levelP+1, N)."""
        sid = self._sid(stream_id)
        rows = levelQ + 1 + levelP + 1
        out = self.ctx.new_poly(rows, batch)
        L = _lib.lib()
        _lib.check(L.lgpu_sample_uniform(self.ctx.h, RING_Q, levelQ, self.seed, sid, ctypes.c_void_p(out.data_ptr()), batch, rows * self.ctx.N, _stream()))
        if levelP >= 0:      # the P limbs' counters differ from the Q limbs' (include/lattigo_b200.h), so the id is shared
            _lib.check(L.lgpu_sample_uniform(self.ctx.h, RING_P, levelP, self.seed, sid,
                                             ctypes.c_void_p(out.data_ptr() + 8 * (levelQ + 1) * self.ctx.N), batch, rows * self.ctx.N, _stream()))
        return out

    def _small(self, batch):
        return self.ctx.new_poly(batch)

    def Ternary(self, P: float = 0.0, H: int = 0, batch: int = 1, stream_id=None):
        out = self._small(batch)
        _lib.check(_lib.lib().lgpu_sample_ternary(self.ctx.h, float(P), int(H), self.seed, self._sid(stream_id), _dptr(out), batch, _stream()))
        return out

    def Gaussian(self, sigma: float = 3.2, bound: float = 19.2, batch: int = 1, stream_id=None):
        out = self._small(batch)
        _lib.check(_lib.lib().lgpu_sample_gaussian(self.ctx.h, float(sigma), float(bound), self.seed, self._sid(stream_id), _dptr(out), batch, _stream()))
        return out


def gadget_layout(ctx: Context, levelQ: int, levelP: int, pw2: int):
    """(BaseRNSDecompositionVectorSize, BaseTwoDecompositionVectorSize) of a key at these levels and base (core/rlwe/params.go:520-550)."""
    nd = levelQ + 1 if levelP == -1 else (levelQ + levelP + 1) // (levelP + 1)
    if pw2 == 0 or levelP > 0:
        return nd, [1] * nd
    return nd, [(int(round(math.log2(float(q)))) + pw2 - 1) // pw2 for q in ctx.Q[:nd]]


def new_gadget_block(ctx: Context, n: int, levelQ: int, levelP: int, pw2: int):
    """Room for n keys in one tensor (n, digits, pw2, 2, levelQ+1 + levelP+1, N) and the layout: (data, sizes). Every word of it is
    written by the key generators that use it, so it is not zeroed."""
    import torch
    nd, sizes = gadget_layout(ctx, levelQ, levelP, pw2)
    data = torch.empty((n, nd, max(sizes), 2, levelQ + 1 + levelP + 1, ctx.N), dtype=torch.int64, device="cuda:%d" % ctx.device)
    return data, sizes


def draw_gadget_samples(samplers: "Samplers", data, levelQ: int, levelP: int, sigma: float, bound: float):
    """Uniform component 1 of every entry of the keys in `data` (new_gadget_block) and their errors (entries, N), each on one stream id."""
    ctx = samplers.ctx
    rows, N = levelQ + 1 + levelP + 1, ctx.N
    entries = data.shape[0] * data.shape[1] * data.shape[2]
    sid = samplers._sid(None)
    base = data.data_ptr() + 8 * rows * N                       # component 1 of entry 0
    L = _lib.lib()
    _lib.check(L.lgpu_sample_uniform(ctx.h, RING_Q, levelQ, samplers.seed, sid, ctypes.c_void_p(base), entries, 2 * rows * N, _stream()))
    if levelP >= 0:
        _lib.check(L.lgpu_sample_uniform(ctx.h, RING_P, levelP, samplers.seed, sid, ctypes.c_void_p(base + 8 * (levelQ + 1) * N), entries,
                                         2 * rows * N, _stream()))
    return samplers.Gaussian(sigma, bound, batch=entries).view(tuple(data.shape[:3]) + (N,))


def small_poly_to_rns(ctx: Context, small, levelQ: int, levelP: int = -1):
    """(batch, N) signed coefficients -> (batch, levelQ+1, N) [and (batch, levelP+1, N)] residues."""
    batch = small.shape[0]
    outq = ctx.new_poly(levelQ + 1, batch)
    outp = ctx.new_poly(levelP + 1, batch) if levelP >= 0 else None
    _lib.check(_lib.lib().lgpu_small_poly_to_rns(ctx.h, levelQ, levelP, _dptr(small), _dptr(outq), _dptr(outp), batch, (levelQ + 1) * ctx.N,
                                                 (levelP + 1) * ctx.N, _stream()))
    return (outq, outp) if levelP >= 0 else outq


class Encryptor:
    """rlwe.Encryptor's zero-encryption paths with the sampled polynomials as arguments."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def EncryptZeroPk(self, levelQ: int, pk, u, e0, e1, is_ntt=True, is_montgomery=False):
        """pk: (2, nQ + nP, N) device tensor; u, e0, e1: (batch, N) int64 -> (batch, 2, levelQ+1, N)."""
        import torch
        batch = u.shape[0]
        out = torch.empty((batch, 2, levelQ + 1, self.ctx.N), dtype=torch.int64, device=u.device)
        _lib.check(_lib.lib().lgpu_encrypt_zero_pk(self.ctx.h, levelQ, _dptr(pk), _dptr(u), _dptr(e0), _dptr(e1), _dptr(out), int(is_ntt), int(is_montgomery),
                                                   batch, _stream()))
        return out

    def EncryptZeroSk(self, levelQ: int, levelP: int, sk, c1, e, is_ntt=True, is_montgomery=False):
        """sk: (nQ + nP, N); c1: (batch, levelQ+1 + levelP+1, N) uniform (NTT domain); e: (batch, N) -> c0, same shape as c1."""
        import torch
        c0 = torch.empty_like(c1)
        _lib.check(_lib.lib().lgpu_encrypt_zero_sk(self.ctx.h, levelQ, levelP, _dptr(sk), _dptr(c1), _dptr(e), _dptr(c0), int(is_ntt), int(is_montgomery),
                                                   c1.shape[0], _stream()))
        return c0


class KeyGenerator:
    """rlwe.KeyGenerator.GenEvaluationKey at the maximum levels (core/rlwe/keygenerator.go:261-330) and GenGaloisKeysNew at any levels
    (:123-209)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def GenEvaluationKey(self, skIn, skOut, a, e, pw2: int = 0, pw2_sizes=None) -> GadgetCiphertext:
        """a: (digits, pw2, nQ + nP, N) uniform; e: (digits, pw2, N) int64. Returns the device-resident key."""
        import torch
        ctx = self.ctx
        nd, npw2 = a.shape[0], a.shape[1]
        rows = len(ctx.Q) + len(ctx.P)
        data = torch.zeros((nd, npw2, 2, rows, ctx.N), dtype=torch.int64, device=a.device)
        data[:, :, 1] = a
        evk = GadgetCiphertext(ctx, data, len(ctx.Q) - 1, len(ctx.P) - 1, pw2, pw2_sizes)
        _lib.check(_lib.lib().lgpu_gen_evaluation_key(ctx.h, _dptr(skIn), _dptr(skOut), evk.ref(), _dptr(e.contiguous()), _stream()))
        return evk

    def GenGaloisKeysNew(self, galEls, sk, levelQ: int = None, levelP: int = None, pw2: int = 0, samplers: Samplers = None, sigma: float = 3.2,
                         bound: float = 19.2, a=None, e=None):
        """One Galois key per element of galEls (odd, below 2N) for sk ((nQ + nP, N), NTT + Montgomery), in one device call. The
        samples come from `samplers`, or are given: a (n, digits, pw2, levelQ+1 + levelP+1, N) uniform, e (n, digits, pw2, N).
        Returns the keys as a list of GadgetCiphertext in the order of galEls."""
        import numpy as np
        ctx = self.ctx
        levelQ = len(ctx.Q) - 1 if levelQ is None else levelQ
        levelP = len(ctx.P) - 1 if levelP is None else levelP
        n = len(galEls)
        data, sizes = new_gadget_block(ctx, n, levelQ, levelP, pw2)
        if a is None:
            e = draw_gadget_samples(samplers, data, levelQ, levelP, sigma, bound)
        else:
            data[:, :, :, 1] = a
        keys = [GadgetCiphertext(ctx, data[k], levelQ, levelP, pw2, sizes) for k in range(n)]
        arr = (_lib.GadgetCtStruct * n)(*[k.struct for k in keys])
        g = np.ascontiguousarray(np.asarray(galEls, dtype=np.uint64))
        _lib.check(_lib.lib().lgpu_gen_galois_keys(ctx.h, _dptr(sk), g.ctypes.data, n, _dptr(e.contiguous()), arr, _stream()))
        return keys

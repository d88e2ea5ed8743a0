"""Host-side mirror of core/rgsw (rgsw.Ciphertext, rgsw.Evaluator.ExternalProduct) bound to the C ABI."""
from __future__ import annotations

from . import _lib
from .ring import Context, _dptr, _stream
from .rlwe import GadgetCiphertext


class Ciphertext:
    """rgsw.Ciphertext (core/rgsw/elements.go:11-13): Value = [2]rlwe.GadgetCiphertext, device resident."""

    def __init__(self, v0: GadgetCiphertext, v1: GadgetCiphertext):
        self.Value = [v0, v1]

    def LevelQ(self): return self.Value[0].LevelQ()
    def LevelP(self): return self.Value[0].LevelP()


class Evaluator:
    """rgsw.Evaluator (core/rgsw/evaluator.go:12-24)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def ExternalProduct(self, op0, op1: Ciphertext, opOut):
        """op0 / opOut: (batch, 2, level+1, N) or (2, level+1, N) NTT-domain RLWE ciphertexts; rows 0..op1.LevelQ() of opOut are written."""
        batch = op0.shape[0] if op0.dim() == 4 else 1
        _lib.check(_lib.lib().lgpu_rgsw_external_product(self.ctx.h, _dptr(op0), op0.shape[-2] - 1, op1.Value[0].ref(), op1.Value[1].ref(),
                                                         _dptr(opOut), opOut.shape[-2] - 1, batch, _stream()))


class BlindRotationEvaluator:
    """blindrot.Evaluator.BlindRotateCore (core/rgsw/blindrot/evaluator.go:144-229) on the device: the accumulator-loop of Algorithm 3
    (eprint 2022/198), driven by the host-side LWE mask `a` (values modulo 2N), in place on `acc` ((2, level+1, N), NTT domain)."""

    def __init__(self, ctx: Context, blind_rotation_keys, automorphism_keys, window_size: int = 10):
        self.ctx = ctx
        self.brk = list(blind_rotation_keys)                      # rgsw.Ciphertext per LWE coefficient: RGSW(X^{s_j})
        n = len(self.brk)
        self._b0 = (_lib.GadgetCtStruct * n)(*[k.Value[0].struct for k in self.brk])
        self._b1 = (_lib.GadgetCtStruct * n)(*[k.Value[1].struct for k in self.brk])
        keys = _lib.GaloisKeys(automorphism_keys)                 # {galEl: GadgetCiphertext}
        self.keys, self._gks = keys.keys, keys.gks
        self.window = window_size

    def BlindRotateCore(self, a, acc):
        import ctypes
        import numpy as np
        a = np.ascontiguousarray(np.asarray(a, dtype=np.uint64))
        assert len(a) == len(self.brk)
        _lib.check(_lib.lib().lgpu_blind_rotate_core(self.ctx.h, a.ctypes.data, len(a), _dptr(acc), acc.shape[-2] - 1, self._b0, self._b1,
                                                     ctypes.byref(self._gks), self.window, _stream()))

    def Evaluate(self, ct_lwe, test_polys, ctx_lwe: Context = None, is_ntt: bool = True, ntt_out: bool = True):
        """blindrot.Evaluator.Evaluate (core/rgsw/blindrot/evaluator.go:49-132) in one device call: ct_lwe is a level-0 LWE-ring ciphertext
        (2, 1, N_LWE) or a batch (batch, 2, 1, N_LWE) in ctx_lwe (default: this evaluator's ring), in the NTT domain when is_ntt;
        test_polys maps slot -> NTT-domain test polynomial (level+1, N). Returns {slot: (2, level+1, N) or (batch, 2, level+1, N)},
        in the NTT domain unless ntt_out is False (the reference's !NTTFlag branch)."""
        import ctypes
        import torch
        ctx_lwe = self.ctx if ctx_lwe is None else ctx_lwe
        single = ct_lwe.dim() == 3
        ct = ct_lwe.unsqueeze(0) if single else ct_lwe
        ct = ct.contiguous()
        slots = sorted(test_polys)
        polys = [test_polys[s].contiguous() for s in slots]
        level = self.brk[0].LevelQ()
        N = self.ctx.N
        out = torch.empty((ct.shape[0], len(slots), 2, level + 1, N), dtype=ct.dtype, device=ct.device)
        c_slots = (ctypes.c_int * len(slots))(*slots)
        c_polys = (ctypes.c_void_p * len(slots))(*[_dptr(p) for p in polys])
        _lib.check(_lib.lib().lgpu_blind_rotation_evaluate(self.ctx.h, ctx_lwe.h, _dptr(ct), ct.shape[-2] - 1, int(is_ntt), c_slots, len(slots),
                                                           c_polys, self._b0, self._b1, len(self.brk), ctypes.byref(self._gks), self.window,
                                                           int(ntt_out), _dptr(out), ct.shape[0], _stream()))
        return {s: (out[0, k] if single else out[:, k]) for k, s in enumerate(slots)}

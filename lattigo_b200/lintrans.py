"""Host-side mirror of circuits/common/lintrans (lintrans.LinearTransformation, lintrans.Evaluator) bound to the C ABI:
same names and argument meaning as the reference, ciphertexts are (batch, 2, level+1, N) int64 CUDA tensors in the NTT
domain, one plaintext matrix applied to every ciphertext of the batch."""
from __future__ import annotations

import ctypes
from typing import Dict, Sequence

from . import _lib
from .ring import Context, _dptr, _stream
from .rlwe import GadgetCiphertext


class LinearTransformation:
    """lintrans.LinearTransformation (circuits/common/lintrans/lintrans.go:150-160). Vec[k]: device tensor
    (LevelQ+1 + LevelP+1, N) holding the Q rows then the P rows of the k-th diagonal in NTT + Montgomery form;
    N1 = 0 selects the naive evaluator."""

    def __init__(self, vec: Dict[int, "object"], levelQ: int, levelP: int, log_slots: int, N1: int = 0):
        self.Vec, self.LevelQ, self.LevelP, self.LogSlots, self.N1 = vec, levelQ, levelP, log_slots, N1
        self._keys = list(vec.keys())
        for t in vec.values():
            assert t.is_cuda and t.is_contiguous() and t.shape[-2] == levelQ + 1 + levelP + 1
        self._idx = (ctypes.c_int * len(self._keys))(*self._keys)
        self._ptrs = (ctypes.c_void_p * len(self._keys))(*[vec[k].data_ptr() for k in self._keys])

    def struct(self):
        return _lib.LinTransStruct(self.LevelQ, self.LevelP, self.LogSlots, self.N1, len(self._keys), self._idx, self._ptrs)


class Evaluator:
    """lintrans.Evaluator (lintrans_evaluator.go:12-24) over a set of Galois keys {galEl: GadgetCiphertext}
    (rlwe.MemEvaluationKeySet.GaloisKeys)."""

    def __init__(self, ctx: Context, galois_keys: Dict[int, GadgetCiphertext]):
        self.ctx = ctx
        keys = _lib.GaloisKeys(galois_keys)
        self.keys, self._gks = keys.keys, keys.gks

    def GaloisElement(self, k: int) -> int:
        return int(_lib.lib().lgpu_galois_element(self.ctx.h, k))

    def EvaluateMany(self, ctIn, linearTransformations: Sequence[LinearTransformation], opOut: Sequence["object"]):
        """opOut[i]: (batch, 2, level_i+1, N) tensors; returns the result levels (the reference Resizes opOut[i])."""
        n = len(linearTransformations)
        assert len(opOut) >= n, "output *rlwe.Ciphertext slice is too small"
        batch = ctIn.shape[0] if ctIn.dim() == 4 else 1
        level_in = ctIn.shape[-2] - 1
        mats = (_lib.LinTransStruct * n)(*[m.struct() for m in linearTransformations])
        outs = (ctypes.c_void_p * n)(*[o.data_ptr() for o in opOut[:n]])
        lv = (ctypes.c_int * n)(*[o.shape[-2] - 1 for o in opOut[:n]])
        _lib.check(_lib.lib().lgpu_lintrans_evaluate_many(self.ctx.h, level_in, _dptr(ctIn), mats, n, ctypes.byref(self._gks), outs, lv, batch, _stream()))
        return [int(x) for x in lv]

    def Evaluate(self, ctIn, linearTransformation: LinearTransformation, opOut):
        return self.EvaluateMany(ctIn, [linearTransformation], [opOut])[0]

    def EvaluateNew(self, ctIn, linearTransformation: LinearTransformation):
        import torch
        level = min(ctIn.shape[-2] - 1, linearTransformation.LevelQ)
        out = torch.empty(tuple(ctIn.shape[:-2]) + (level + 1, self.ctx.N), dtype=torch.int64, device=ctIn.device)
        self.Evaluate(ctIn, linearTransformation, out)
        return out

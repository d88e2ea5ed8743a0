"""bgv.Evaluator's ciphertext x ciphertext multiplication (schemes/bgv/evaluator.go) bound to the C ABI: MulRelin with
standard tensoring (BGV) or, with scale_invariant=True, MulRelinScaleInvariant (BFV), and Rescale. Ciphertexts are
degree-1, NTT-domain, contiguous int64 CUDA tensors of shape (2, level+1, N) or (batch, 2, level+1, N).
Scales are the caller's: the reference multiplies them (BGV), divides by q_level on Rescale, and divides the product by
(-Q_level mod t) for BFV (MulScaleInvariant, :983-989)."""
from __future__ import annotations

import ctypes
from typing import Sequence

import numpy as np

from . import _lib
from .ring import Context, RING_Q, _dptr, _stream
from .rlwe import GadgetCiphertext, _bs, div_by_last_modulus_many


class BGVEvaluator:
    """bgv.Evaluator (evaluator.go:18-29) for the multiplication path. qmul: Parameters.RingQMul() moduli
    (params.go:98-109, e.g. params.PRESETS["BGV_N15QP880"]["QMul"])."""

    def __init__(self, ctx: Context, t: int, qmul: Sequence[int], rlk: GadgetCiphertext, scale_invariant: bool = False):
        self.ctx = ctx
        self.t = int(t)
        self.QMul = [int(x) for x in qmul]
        self.rlk = rlk
        self.ScaleInvariant = bool(scale_invariant)
        qa = np.array(self.QMul, dtype=np.uint64)
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().lgpu_bgv_create(ctx.h, self.t, qa.ctypes.data, len(self.QMul), ctypes.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            _lib.lib().lgpu_bgv_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _mul(self, op0, op1, nb_rescales, out=None):
        import torch
        b, _ = _bs(op0, 3)
        level = op0.shape[-2] - 1
        if op1.shape != op0.shape:
            raise ValueError("operands must have the same shape (batch, 2, level+1, N)")
        if out is None:
            shape = tuple(op0.shape[:-2]) + (level + 1 - nb_rescales, self.ctx.N)
            out = torch.empty(shape, dtype=torch.int64, device=op0.device)
        _lib.check(_lib.lib().lgpu_bgv_mulrelin_batch(self.h, level, _dptr(op0), _dptr(op1), self.rlk.ref(), 1 if self.ScaleInvariant else 0,
                                                      nb_rescales, _dptr(out), b, _stream()))
        return out

    def MulRelinNew(self, op0, op1):
        """MulRelinNew (evaluator.go:576-590); op1 may be op0 (squaring)."""
        return self._mul(op0, op1, 0)

    def MulRelin(self, op0, op1, opOut):
        """MulRelin (evaluator.go:529-556) into opOut; opOut may be op0."""
        self._mul(op0, op1, 0, opOut)

    def MulRelinRescaleNew(self, op0, op1):
        """MulRelinNew followed by Rescale, fused (BGV only: the scale-invariant evaluator does not rescale)."""
        return self._mul(op0, op1, 1)

    def Rescale(self, op0):
        """Rescale (evaluator.go:1363-1393): DivRoundByLastModulusNTT of every polynomial; a copy for the scale-invariant evaluator."""
        import torch
        if self.ScaleInvariant:
            return op0.clone()
        level = op0.shape[-2] - 1
        out = torch.empty(tuple(op0.shape[:-2]) + (level, self.ctx.N), dtype=torch.int64, device=op0.device)
        div_by_last_modulus_many(self.ctx, RING_Q, level, True, True, 1, op0.reshape(-1, level + 1, self.ctx.N),
                                 out.view(-1, level, self.ctx.N))
        return out

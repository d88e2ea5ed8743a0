"""Host-side mirror of the slot-aggregation methods of core/rlwe/inner_sum.go (Evaluator.PartialTracesSum, Trace, Replicate) and
of the scheme methods built on them (ckks / bgv InnerSum, RotateAndAdd, ckks Average), bound to the C ABI. Same names and argument
meaning as the reference. Ciphertexts are degree-1 contiguous int64 CUDA tensors of shape (2, level+1, N) or
(batch, 2, level+1, N); is_ntt plays the role of the reference's MetaData.IsNTT. One set of Galois keys serves the whole batch."""
from __future__ import annotations

import ctypes
from typing import Dict, List

from . import _lib
from .ring import Context, _dptr, _stream
from .rlwe import GadgetCiphertext, _bs


def _galois_element(ctx: Context, k: int) -> int:
    """rlwe.Parameters.GaloisElement (core/rlwe/params.go:580-583): GaloisGen^k mod NthRoot, Standard ring (NthRoot = 2N)."""
    m = 2 * ctx.N
    return pow(5, k & (m - 1), m)


def GaloisElementsForTrace(ctx: Context, logN: int) -> List[int]:
    """inner_sum.go:120-141: the keys Trace(., logN, .) uses."""
    if ctx.ring_type != 0:
        raise ValueError("cannot GaloisElementsForTrace: Galois element GaloisGen^-1 is undefined in ConjugateInvariant Ring")
    gal = [_galois_element(ctx, 1 << i) for i in range(logN, ctx.logN - 1)]
    if logN == 0:
        gal.append(2 * ctx.N - 1)                   # GaloisElementOrderTwoOrthogonalSubgroup
    return gal


def GaloisElementsForInnerSum(ctx: Context, batch: int, n: int) -> List[int]:
    """inner_sum.go:442-466 (sorted; the reference returns them in map order). A superset of what PartialTracesSum(batch, n) uses:
    it also lists GaloisElement(0) = 1 when n is not a power of two and GaloisElement(n * batch) when it is."""
    rot = set()
    i = 1
    while i < n:
        rot.add(i * batch)
        rot.add((n - (n & ((i << 1) - 1))) * batch)
        i <<= 1
    return sorted({_galois_element(ctx, k) for k in rot})


def GaloisElementsForReplicate(ctx: Context, batch: int, n: int) -> List[int]:
    """inner_sum.go:481-483."""
    return GaloisElementsForInnerSum(ctx, -batch, n)


class Evaluator:
    """rlwe.Evaluator restricted to inner_sum.go, plus the scheme-level wrappers, over a set of Galois keys
    {galEl: GadgetCiphertext} (rlwe.MemEvaluationKeySet.GaloisKeys)."""

    def __init__(self, ctx: Context, galois_keys: Dict[int, GadgetCiphertext]):
        self.ctx = ctx
        keys = _lib.GaloisKeys(galois_keys)
        self.keys, self._gks = keys.keys, keys.gks

    def GaloisElement(self, k: int) -> int:
        return int(_lib.lib().lgpu_galois_element(self.ctx.h, k))

    def _new_like(self, ct, level=None):
        import torch
        level = ct.shape[-2] - 1 if level is None else level
        return torch.empty(tuple(ct.shape[:-2]) + (level + 1, self.ctx.N), dtype=torch.int64, device=ct.device)

    # --- core/rlwe/inner_sum.go ------------------------------------------------------------------------------
    def PartialTracesSum(self, ctIn, offset: int, n: int, opOut, is_ntt: bool = True):
        """:147-292: opOut = sum_{i<n} phi(i * offset)(ctIn). opOut has ctIn's shape and may be ctIn."""
        b, _ = _bs(ctIn, 3)
        if opOut.shape != ctIn.shape:
            raise ValueError("opOut must have the shape of ctIn (batch, 2, level+1, N)")
        level = ctIn.shape[-2] - 1
        _lib.check(_lib.lib().lgpu_evaluator_partial_traces_sum(self.ctx.h, level, _dptr(ctIn), 1 if is_ntt else 0, offset, n, ctypes.byref(self._gks),
                                                                _dptr(opOut), b, _stream()))

    def Trace(self, ctIn, logN: int, opOut, is_ntt: bool = True) -> int:
        """:36-116. Returns the level of the result, min(ctIn level, opOut level); rows 0..level of each component of opOut are written."""
        b, _ = _bs(ctIn, 3)
        if _bs(opOut, 3)[0] != b:
            raise ValueError("ctIn and opOut hold different numbers of ciphertexts")
        level_in, level_out = ctIn.shape[-2] - 1, opOut.shape[-2] - 1
        _lib.check(_lib.lib().lgpu_evaluator_trace(self.ctx.h, level_in, _dptr(ctIn), 1 if is_ntt else 0, logN, ctypes.byref(self._gks), _dptr(opOut),
                                                   level_out, b, _stream()))
        return min(level_in, level_out)

    def TraceNew(self, ctIn, logN: int, is_ntt: bool = True):
        out = self._new_like(ctIn)
        self.Trace(ctIn, logN, out, is_ntt)
        return out

    def Replicate(self, ctIn, batchSize: int, n: int, opOut, is_ntt: bool = True):
        """:475-477."""
        self.PartialTracesSum(ctIn, -batchSize, n, opOut, is_ntt)

    def RotateAndAdd(self, ctIn, batchSize: int, n: int, opOut, is_ntt: bool = True):
        """ckks / bgv Evaluator.RotateAndAdd: PartialTracesSum(ctIn, batchSize, n)."""
        self.PartialTracesSum(ctIn, batchSize, n, opOut, is_ntt)

    # --- schemes ---------------------------------------------------------------------------------------------
    def InnerSum(self, ctIn, batchSize: int, n: int, opOut, slots: int, bgv: bool = False, is_ntt: bool = True):
        """ckks.Evaluator.InnerSum (schemes/ckks/evaluator.go:1285-1302) or, with bgv = True, bgv.Evaluator.InnerSum
        (schemes/bgv/evaluator.go:1475-1517), whose n * batchSize == slots case is PartialTracesSum(n / 2) + RotateRows + Add.
        slots = ctIn.Slots()."""
        l = n * batchSize
        if n <= 0 or batchSize <= 0:
            raise ValueError("innersum: invalid parameter (n <= 0 or batchSize <= 0)")
        if l > slots:
            raise ValueError("innersum: invalid parameters (n*batchSize=%d > #slots=%d)" % (l, slots))
        if l & (l - 1) != 0:
            raise ValueError("innersum: invalid parameters (n*batchSize=%d does not divide #slots=%d)" % (l, slots))
        if bgv and l == slots:
            if n == 1:
                if opOut.data_ptr() != ctIn.data_ptr():
                    opOut.copy_(ctIn)
                return
            g = 2 * self.ctx.N - 1                  # RotateRows: GaloisElementOrderTwoOrthogonalSubgroup, checked before any work
            if g not in self.keys:
                raise _lib.LgpuError("GaloisKey[%d] is missing" % g)
            if not is_ntt:
                raise ValueError("bgv.Evaluator.InnerSum: RotateRows expects NTT-domain ciphertexts")
            self.PartialTracesSum(ctIn, batchSize, n // 2, opOut, is_ntt)
            self._rotate_rows_add(opOut, g)
            return
        self.PartialTracesSum(ctIn, batchSize, n, opOut, is_ntt)

    def _rotate_rows_add(self, ct, g):
        """ct += bgv.Evaluator.RotateRows(ct) (Automorphism by g = NthRoot - 1), in place, from the existing entry points."""
        from .rlwe import Evaluator as RlweEvaluator
        tmp = self._new_like(ct)
        RlweEvaluator(self.ctx).Automorphism(ct, g, self.keys[g], tmp)
        level = ct.shape[-2] - 1
        ringQ = self.ctx.ringQ.AtLevel(level)
        flat, ftmp = ct.view(-1, level + 1, self.ctx.N), tmp.view(-1, level + 1, self.ctx.N)
        ringQ.Add(flat, ftmp, flat)

    def Average(self, ctIn, logBatchSize: int, opOut, log_slots: int, is_ntt: bool = True):
        """ckks.Evaluator.Average (schemes/ckks/linear_transformation.go:27-52): opOut = InnerSum(n^-1 * ctIn, 2^logBatchSize, n),
        n = 2^(log_slots - logBatchSize); log_slots = ctIn.LogDimensions.Cols. opOut has ctIn's shape and may be ctIn."""
        if logBatchSize > log_slots:
            raise ValueError("cannot Average: batchSize must be smaller or equal to the number of slots")
        if opOut.shape != ctIn.shape:
            raise ValueError("opOut must have the shape of ctIn (batch, 2, level+1, N)")
        level = ctIn.shape[-2] - 1
        n = 1 << (log_slots - logBatchSize)
        ringQ = self.ctx.ringQ.AtLevel(level)
        # pre-multiplication by n^-1: MulScalarMontgomery by MForm(n^(q_i - 2) mod q_i) on every limb
        inv = [((pow(n, q - 2, q)) << 64) % q for q in self.ctx.Q[: level + 1]]
        ringQ.MulRNSScalarMontgomery(ctIn.reshape(-1, level + 1, self.ctx.N), inv, opOut.view(-1, level + 1, self.ctx.N))
        self.InnerSum(opOut, 1 << logBatchSize, n, opOut, 1 << log_slots, False, is_ntt)

"""Host-side mirror of ring.BasisExtender / ring.Decomposer / rlwe.Evaluator (key-switch family) and the two
CKKS op sequences that define the measured workloads, bound to the C ABI. Same method names and argument
meaning as the reference; polynomials / ciphertexts are contiguous int64 CUDA tensors:
  poly        (limbs, N)            or (batch, limbs, N)
  ciphertext  (degree+1, limbs, N)  or (batch, degree+1, limbs, N)
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence

import numpy as np

from . import _lib
from .ring import Context, RING_Q, RING_P, _dptr, _stream


def _bs(t, nd_single):
    """(batch, stride in words) of a tensor whose un-batched rank is nd_single."""
    if t.dim() == nd_single + 1:
        stride = 1
        for s in t.shape[1:]:
            stride *= s
        return t.shape[0], stride
    assert t.dim() == nd_single
    return 1, 0


class GadgetCiphertext:
    """rlwe.GadgetCiphertext (core/rlwe/gadgetciphertext.go:19-45) resident on the device:
    data[digit][pw2][component][Q limbs then P limbs][N], NTT + Montgomery form."""

    def __init__(self, ctx: Context, data, levelQ: int, levelP: int, base_two_decomposition: int = 0,
                 pw2_sizes: Optional[Sequence[int]] = None):
        self.ctx = ctx
        self.data = data if hasattr(data, "is_cuda") else ctx.to_device(np.ascontiguousarray(data))
        assert self.data.dim() == 5 and self.data.shape[2] == 2 and self.data.shape[3] == levelQ + 1 + levelP + 1
        self.levelQ, self.levelP = levelQ, levelP
        self.BaseTwoDecomposition = base_two_decomposition
        self._sizes = (ctypes.c_int * self.data.shape[0])(*([int(x) for x in pw2_sizes] if pw2_sizes is not None
                                                            else [self.data.shape[1]] * self.data.shape[0]))
        self.struct = _lib.GadgetCtStruct(ctypes.c_void_p(self.data.data_ptr()), levelQ, levelP, base_two_decomposition,
                                          self.data.shape[0], self.data.shape[1], self._sizes)

    def LevelQ(self): return self.levelQ
    def LevelP(self): return self.levelP
    def ref(self): return ctypes.byref(self.struct)


class BasisExtender:
    """ring.BasisExtender (ring/basis_extension.go:14-87)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def ModUpQtoP(self, levelQ, levelP, polQ, polP):
        b, sq = _bs(polQ, 2); _, sp = _bs(polP, 2)
        _lib.check(_lib.lib().lgpu_modup_qtop(self.ctx.h, levelQ, levelP, _dptr(polQ), _dptr(polP), b, sq, sp, _stream()))

    def ModUpPtoQ(self, levelP, levelQ, polP, polQ):
        b, sp = _bs(polP, 2); _, sq = _bs(polQ, 2)
        _lib.check(_lib.lib().lgpu_modup_ptoq(self.ctx.h, levelP, levelQ, _dptr(polP), _dptr(polQ), b, sp, sq, _stream()))

    def _md(self, fn, levelQ, levelP, p1Q, p1P, p2):
        b, sq = _bs(p1Q, 2); _, sp = _bs(p1P, 2)
        _lib.check(fn(self.ctx.h, levelQ, levelP, _dptr(p1Q), _dptr(p1P), _dptr(p2), b, sq, sp, _stream()))

    def ModDownQPtoQ(self, levelQ, levelP, p1Q, p1P, p2Q): self._md(_lib.lib().lgpu_moddown_qp_to_q, levelQ, levelP, p1Q, p1P, p2Q)
    def ModDownQPtoQNTT(self, levelQ, levelP, p1Q, p1P, p2Q): self._md(_lib.lib().lgpu_moddown_qp_to_q_ntt, levelQ, levelP, p1Q, p1P, p2Q)
    def ModDownQPtoP(self, levelQ, levelP, p1Q, p1P, p2P): self._md(_lib.lib().lgpu_moddown_qp_to_p, levelQ, levelP, p1Q, p1P, p2P)


class Decomposer:
    """ring.Decomposer (ring/basis_extension.go:313-502)."""

    def __init__(self, ctx: Context):
        self.ctx = ctx

    def DecomposeAndSplit(self, levelQ, levelP, nbPi, BaseRNSDecompositionVectorSize, p0Q, p1Q, p1P):
        b, sq = _bs(p0Q, 2)
        sp = _bs(p1P, 2)[1] if p1P is not None else 0
        _lib.check(_lib.lib().lgpu_decompose_and_split(self.ctx.h, levelQ, levelP, nbPi, BaseRNSDecompositionVectorSize,
                                                       _dptr(p0Q), _dptr(p1Q), _dptr(p1P), b, sq, sp, _stream()))


def div_by_last_modulus_many(ctx: Context, ring: int, level: int, round_: bool, ntt: bool, nb: int, p0, p1):
    """Ring.Div{Round,Floor}ByLastModulus[Many][NTT] (ring/scaling.go:6-212)."""
    b, si = _bs(p0, 2); _, so = _bs(p1, 2)
    flags = (1 if round_ else 0) | (2 if ntt else 0)
    _lib.check(_lib.lib().lgpu_div_by_last_modulus_many(ctx.h, ring, level, flags, nb, _dptr(p0), _dptr(p1), b, si, so, _stream()))


def automorphism_ntt_index(ctx: Context, galEl: int):
    idx = ctx.new_poly(1)[0]
    _lib.check(_lib.lib().lgpu_automorphism_ntt_index(ctx.h, galEl, _dptr(idx), _stream()))
    return idx


def automorphism_ntt_with_index(ctx: Context, ring: int, level: int, polIn, index, polOut, accumulate=False):
    b, s = _bs(polIn, 2)
    _lib.check(_lib.lib().lgpu_automorphism_ntt_with_index(ctx.h, ring, level, _dptr(polIn), _dptr(index), _dptr(polOut),
                                                           1 if accumulate else 0, b, s, _stream()))


def automorphism_ntt(ctx: Context, ring: int, level: int, polIn, galEl: int, polOut):
    b, s = _bs(polIn, 2)
    _lib.check(_lib.lib().lgpu_automorphism_ntt(ctx.h, ring, level, _dptr(polIn), galEl, _dptr(polOut), b, s, _stream()))


def automorphism(ctx: Context, ring: int, level: int, polIn, galEl: int, polOut):
    b, s = _bs(polIn, 2)
    _lib.check(_lib.lib().lgpu_automorphism(ctx.h, ring, level, _dptr(polIn), galEl, _dptr(polOut), b, s, _stream()))


class Evaluator:
    """rlwe.Evaluator (core/rlwe/evaluator.go:12-21), key-switch family."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.BasisExtender = BasisExtender(ctx)
        self.Decomposer = Decomposer(ctx)

    def BaseRNSDecompositionVectorSize(self, levelQ, levelP):   # core/rlwe/params.go:543-550
        return levelQ + 1 if levelP == -1 else (levelQ + levelP + 1) // (levelP + 1)

    def GadgetProduct(self, levelQ, cx, gadgetCt: GadgetCiphertext, ct0, ct1):
        b, scx = _bs(cx, 2); _, sct = _bs(ct0, 2)
        _lib.check(_lib.lib().lgpu_gadget_product(self.ctx.h, levelQ, _dptr(cx), gadgetCt.ref(), _dptr(ct0), _dptr(ct1), b, scx, sct, _stream()))

    def GadgetProductLazy(self, levelQ, cx, gadgetCt: GadgetCiphertext, acc0Q, acc0P, acc1Q, acc1P):
        b, scx = _bs(cx, 2); _, sq = _bs(acc0Q, 2)
        sp = _bs(acc0P, 2)[1] if acc0P is not None else 0
        _lib.check(_lib.lib().lgpu_gadget_product_lazy(self.ctx.h, levelQ, _dptr(cx), gadgetCt.ref(), _dptr(acc0Q), _dptr(acc0P),
                                                       _dptr(acc1Q), _dptr(acc1P), b, scx, sq, sp, _stream()))

    def ModDown(self, levelQ, levelP, acc0Q, acc0P, acc1Q, acc1P, ct0, ct1):
        b, sq = _bs(acc0Q, 2); _, sct = _bs(ct0, 2)
        sp = _bs(acc0P, 2)[1] if acc0P is not None else 0
        _lib.check(_lib.lib().lgpu_evaluator_moddown(self.ctx.h, levelQ, levelP, _dptr(acc0Q), _dptr(acc0P), _dptr(acc1Q), _dptr(acc1P),
                                                     _dptr(ct0), _dptr(ct1), b, sq, sp, sct, _stream()))

    def DecomposeSingleNTT(self, levelQ, levelP, nbPi, digit, c2NTT, c2InvNTT, c2QiQ, c2QiP):
        b, si = _bs(c2NTT, 2); _, sq = _bs(c2QiQ, 2); _, sp = _bs(c2QiP, 2)
        _lib.check(_lib.lib().lgpu_decompose_single_ntt(self.ctx.h, levelQ, levelP, nbPi, digit, _dptr(c2NTT), _dptr(c2InvNTT),
                                                        _dptr(c2QiQ), _dptr(c2QiP), b, si, sq, sp, _stream()))

    def DecomposeNTT(self, levelQ, levelP, nbPi, c2, c2IsNTT: bool):
        """Returns the device array [digit][batch][levelQ+1 + levelP+1][N]."""
        b, si = _bs(c2, 2)
        n = self.BaseRNSDecompositionVectorSize(levelQ, levelP)
        import torch
        out = torch.empty((n, b, levelQ + 1 + levelP + 1, self.ctx.N), dtype=torch.int64, device=c2.device)
        _lib.check(_lib.lib().lgpu_decompose_ntt(self.ctx.h, levelQ, levelP, nbPi, _dptr(c2), 1 if c2IsNTT else 0, _dptr(out), b, si, _stream()))
        return out

    def GadgetProductHoisted(self, levelQ, decomp, gadgetCt: GadgetCiphertext, ct0, ct1):
        b = decomp.shape[1]
        sct = _bs(ct0, 2)[1]
        _lib.check(_lib.lib().lgpu_gadget_product_hoisted(self.ctx.h, levelQ, _dptr(decomp), gadgetCt.ref(), _dptr(ct0), _dptr(ct1), b, sct, _stream()))

    def GadgetProductHoistedLazy(self, levelQ, decomp, gadgetCt: GadgetCiphertext, acc0Q, acc0P, acc1Q, acc1P):
        b = decomp.shape[1]
        sq = _bs(acc0Q, 2)[1]; sp = _bs(acc0P, 2)[1]
        _lib.check(_lib.lib().lgpu_gadget_product_hoisted_lazy(self.ctx.h, levelQ, _dptr(decomp), gadgetCt.ref(), _dptr(acc0Q), _dptr(acc0P),
                                                               _dptr(acc1Q), _dptr(acc1P), b, sq, sp, _stream()))

    def Automorphism(self, ctIn, galEl: int, gk: GadgetCiphertext, ctOut, decomp=None):
        """Evaluator.Automorphism / AutomorphismHoisted on (batch, 2, limbs, N) NTT-domain ciphertexts."""
        b, _ = _bs(ctIn, 3)
        level = ctIn.shape[-2] - 1
        _lib.check(_lib.lib().lgpu_evaluator_automorphism(self.ctx.h, level, _dptr(ctIn), galEl, gk.ref(), _dptr(decomp), _dptr(ctOut), b, _stream()))

    def AutomorphismHoistedLazy(self, levelQ, ctIn, decomp, galEl: int, gk: GadgetCiphertext, ctQP_Q, ctQP_P):
        """Evaluator.AutomorphismHoistedLazy (core/rlwe/evaluator_automorphism.go:107-165), ctQP.IsNTT branch: the result
        stays modulo QP, scaled by P. ctIn: (2, levelQ+1, N); decomp: DecomposeNTT output; ctQP_Q / ctQP_P: pairs of
        (levelQ+1, N) / (levelP+1, N) output polynomials. Same op sequence as the reference, each op one C-ABI call."""
        ctx = self.ctx
        levelP = gk.LevelP()
        ringQ = ctx.ringQ.AtLevel(levelQ); ringP = ctx.ringP.AtLevel(levelP)
        tQ = [ringQ.NewPoly(), ringQ.NewPoly()]
        tP = [ringP.NewPoly(), ringP.NewPoly()]
        self.GadgetProductHoistedLazy(levelQ, decomp, gk, tQ[0], tP[0], tQ[1], tP[1])
        index = ringQ.AutomorphismNTTIndex(galEl)
        ringQ.AutomorphismNTTWithIndex(tQ[1], index, ctQP_Q[1]); ringP.AutomorphismNTTWithIndex(tP[1], index, ctQP_P[1])
        if levelP > -1:
            Pprod = 1
            for pj in ctx.P[: levelP + 1]: Pprod *= pj
            ringQ.MulScalarBigint(ctIn[0], Pprod, tQ[1])
        ringQ.Add(tQ[0], tQ[1], tQ[0])
        ringQ.AutomorphismNTTWithIndex(tQ[0], index, ctQP_Q[0]); ringP.AutomorphismNTTWithIndex(tP[0], index, ctQP_P[0])

    def Relinearize(self, ctIn, rlk: GadgetCiphertext, ctOut):
        b, _ = _bs(ctIn, 3)
        level = ctIn.shape[-2] - 1
        _lib.check(_lib.lib().lgpu_evaluator_relinearize(self.ctx.h, level, _dptr(ctIn), rlk.ref(), _dptr(ctOut), b, _stream()))

    def ApplyEvaluationKey(self, ctIn, evk: GadgetCiphertext, ctOut, is_ntt: bool = True):
        """Evaluator.ApplyEvaluationKey (core/rlwe/evaluator_evaluationkey.go:36-107) on (2, level+1, n) or (batch, 2, level+1, n)
        ciphertexts. The ring degrees are the tensors' last dimensions; this evaluator's context is the larger one. Rows
        0..min(levels) of ctOut are written; ctOut may be ctIn at the same degree."""
        b, _ = _bs(ctIn, 3)
        bo, _ = _bs(ctOut, 3)
        if b != bo:
            raise ValueError("ApplyEvaluationKey: ctIn and ctOut batch sizes differ")
        log_n = []
        for t in (ctIn, ctOut):
            n = t.shape[-1]
            if n <= 0 or n & (n - 1):
                raise ValueError("ApplyEvaluationKey: ring degree %d is not a power of two" % n)
            log_n.append(n.bit_length() - 1)
        _lib.check(_lib.lib().lgpu_evaluator_apply_evaluation_key(self.ctx.h, _dptr(ctIn), log_n[0], ctIn.shape[-2] - 1, 1 if is_ntt else 0, evk.ref(),
                                                                  _dptr(ctOut), log_n[1], ctOut.shape[-2] - 1, b, _stream()))


class CKKSEvaluator(Evaluator):
    """ckks.Evaluator: MulRelinNew (schemes/ckks/evaluator.go:719-872) and Rescale (:477-515) for degree-1
    NTT-domain ciphertexts stored as (batch, 2, level+1, N)."""

    def __init__(self, ctx: Context, rlk: GadgetCiphertext, levels_per_rescale: int = 1):
        super().__init__(ctx)
        self.rlk = rlk
        self.nbRescales = levels_per_rescale

    def MulRelinRescaleNew(self, op0, op1, rescale: bool = True):
        import torch
        b, _ = _bs(op0, 3)
        level = op0.shape[-2] - 1
        nb = self.nbRescales if rescale else 0
        shape = (op0.shape[0], 2, level + 1 - nb, self.ctx.N) if op0.dim() == 4 else (2, level + 1 - nb, self.ctx.N)
        out = torch.empty(shape, dtype=torch.int64, device=op0.device)
        _lib.check(_lib.lib().lgpu_ckks_mulrelin_rescale_batch(self.ctx.h, level, _dptr(op0), _dptr(op1), self.rlk.ref(), nb, _dptr(out), b, _stream()))
        return out

    def MulRelinNew(self, op0, op1):
        return self.MulRelinRescaleNew(op0, op1, rescale=False)

    def Rescale(self, op0):
        import torch
        b, _ = _bs(op0, 3)
        level = op0.shape[-2] - 1
        nb = self.nbRescales
        lead = op0.shape[:-2]
        out = torch.empty(tuple(lead) + (level + 1 - nb, self.ctx.N), dtype=torch.int64, device=op0.device)
        # every polynomial of every ciphertext is an independent (level+1, N) block
        flat_in = op0.reshape(-1, level + 1, self.ctx.N)
        flat_out = out.view(-1, level + 1 - nb, self.ctx.N)
        div_by_last_modulus_many(self.ctx, RING_Q, level, True, True, nb, flat_in, flat_out)
        return out

    def MulRelinRescaleHost(self, a_host: np.ndarray, b_host: np.ndarray, out_host: np.ndarray, chunk: int = 0):
        """Host-buffer entry point (copies inside): a/b (batch, 2, level+1, N) uint64 numpy (ideally pinned)."""
        batch = a_host.shape[0]
        level = a_host.shape[-2] - 1
        _lib.check(_lib.lib().lgpu_ckks_mulrelin_rescale_batch_host(self.ctx.h, level, a_host.ctypes.data, b_host.ctypes.data, self.rlk.ref(),
                                                                    self.nbRescales, out_host.ctypes.data, batch, chunk))

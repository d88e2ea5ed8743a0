"""Host-side mirror of core/rgsw (rgsw.Ciphertext, rgsw.Encryptor, rgsw.Evaluator.ExternalProduct, blindrot.GenEvaluationKeyNew and
blindrot.Evaluator) bound to the C ABI."""
from __future__ import annotations

from . import _lib
from .encryptor import Samplers, draw_gadget_samples, new_gadget_block
from .ring import Context, _dptr, _stream
from .rlwe import GadgetCiphertext


class Ciphertext:
    """rgsw.Ciphertext (core/rgsw/elements.go:11-13): Value = [2]rlwe.GadgetCiphertext, device resident."""

    def __init__(self, v0: GadgetCiphertext, v1: GadgetCiphertext):
        self.Value = [v0, v1]

    def LevelQ(self): return self.Value[0].LevelQ()
    def LevelP(self): return self.Value[0].LevelP()


def _ciphertexts(ctx, data, levelQ, levelP, pw2, sizes):
    """rgsw.Ciphertext views of a (batch, 2, digits, pw2, 2, rows, N) block and the two lgpu_gadget_ct arrays over it."""
    batch = data.shape[0]
    cts = [Ciphertext(*[GadgetCiphertext(ctx, data[b, v], levelQ, levelP, pw2, sizes) for v in range(2)]) for b in range(batch)]
    v0 = (_lib.GadgetCtStruct * batch)(*[c.Value[0].struct for c in cts])
    v1 = (_lib.GadgetCtStruct * batch)(*[c.Value[1].struct for c in cts])
    return cts, v0, v1


class Encryptor:
    """rgsw.Encryptor (core/rgsw/encryptor.go:12-121): secret-key RGSW encryption of a batch in one device call. sk: (nQ + nP, N), NTT +
    Montgomery. The samples come from `samplers` (Gaussian errors of the given sigma and bound) unless a call gives them."""

    def __init__(self, ctx: Context, sk, samplers: Samplers = None, sigma: float = 3.2, bound: float = 19.2):
        self.ctx, self.sk, self.samplers, self.sigma, self.bound = ctx, sk, samplers, sigma, bound

    def Encrypt(self, pts, levelQ: int, levelP: int, pw2: int = 0, pt_index=None, is_ntt: bool = True, is_montgomery: bool = False, a=None,
                e=None):
        """pts: (n_pt, levelQ+1, N) distinct plaintexts (IsNTT / IsMontgomery as flagged), or None for EncryptZero; ciphertext b encrypts
        pts[pt_index[b]] (default: one ciphertext per plaintext). a: (batch, 2, digits, pw2, levelQ+1 + levelP+1, N) uniform, e:
        (batch, 2, digits, pw2, N), [b][v] for Value[v]. Returns a list of rgsw.Ciphertext."""
        if pts is not None and pt_index is None:
            pt_index = list(range(pts.shape[0]))
        batch = len(pt_index) if pts is not None else (a.shape[0] if a is not None else None)
        if batch is None:
            raise ValueError("EncryptZero needs the samples a and e, or Encrypt's batch")
        return self._run(pts, pt_index, batch, levelQ, levelP, pw2, is_ntt, is_montgomery, a, e)

    def EncryptZero(self, batch: int, levelQ: int, levelP: int, pw2: int = 0, a=None, e=None):
        """`batch` RGSW encryptions of zero (encryptor.go:74-121)."""
        return self._run(None, None, batch, levelQ, levelP, pw2, True, True, a, e)

    def _run(self, pts, pt_index, batch, levelQ, levelP, pw2, is_ntt, is_montgomery, a, e):
        import ctypes
        ctx = self.ctx
        if a is None and self.samplers is None:
            raise ValueError("rgsw.Encryptor needs samplers, or the samples a and e")
        data, sizes = new_gadget_block(ctx, 2 * batch, levelQ, levelP, pw2)
        if a is None:
            e = draw_gadget_samples(self.samplers, data, levelQ, levelP, self.sigma, self.bound)
        else:
            data[:, :, :, 1] = a.reshape((2 * batch,) + tuple(a.shape[2:]))
        data = data.view((batch, 2) + tuple(data.shape[1:]))
        cts, v0, v1 = _ciphertexts(ctx, data, levelQ, levelP, pw2, sizes)
        idx = (ctypes.c_int * batch)(*[int(x) for x in pt_index]) if pts is not None else None
        _lib.check(_lib.lib().lgpu_rgsw_encrypt(ctx.h, _dptr(self.sk), _dptr(pts.contiguous()) if pts is not None else None,
                                                pts.shape[0] if pts is not None else 0, idx, int(is_ntt), int(is_montgomery),
                                                _dptr(e.contiguous()), v0, v1, batch, _stream()))
        return cts


def GenEvaluationKeyNew(ctx_br: Context, sk_br, ctx_lwe: Context, sk_lwe, levelQ: int = None, levelP: int = None, pw2: int = 0,
                        window_size: int = 10, sigma: float = 3.2, bound: float = 19.2, seed: int = 0):
    """blindrot.GenEvaluationKeyNew (core/rgsw/blindrot/keys.go:52-108) in one device call: RGSW(X^{s_i}) under sk_br ((nQ + nP, N), NTT +
    Montgomery) for every coefficient of the LWE key sk_lwe (rows of ctx_lwe, NTT + Montgomery; level 0 is read), and the Galois keys
    of GaloisElement(1..window_size) and NthRoot - GaloisGen. The samples are drawn on the device from `seed` (the stream layout of
    lgpu_blind_rotation_gen_evaluation_key). Returns (brk, {galEl: GadgetCiphertext}), as rgsw.BlindRotationEvaluator takes them."""
    import numpy as np
    levelQ = len(ctx_br.Q) - 1 if levelQ is None else levelQ
    levelP = len(ctx_br.P) - 1 if levelP is None else levelP
    # the LWE key's centred coefficients: INTT, IMForm, PolyToBigintCentered at level 0 (keys.go:57-65)
    s = ctx_lwe.new_poly(1)
    ctx_lwe.ringQ.AtLevel(0).INTT(sk_lwe[:1].contiguous(), s)
    ctx_lwe.ringQ.AtLevel(0).IMForm(s, s)
    q0 = ctx_lwe.Q[0]
    v = ctx_lwe.to_host(s)[0].astype(object)
    s_lwe = np.array([int(x) - q0 if int(x) >= (q0 + 1) // 2 else int(x) for x in v], dtype=np.int64)
    n_lwe = len(s_lwe)
    data, sizes = new_gadget_block(ctx_br, 2 * n_lwe + window_size + 1, levelQ, levelP, pw2)
    rg = data[: 2 * n_lwe].view((n_lwe, 2) + tuple(data.shape[1:]))
    brk, v0, v1 = _ciphertexts(ctx_br, rg, levelQ, levelP, pw2, sizes)
    gals = [int(_lib.lib().lgpu_galois_element(ctx_br.h, k)) for k in range(1, window_size + 1)] + [2 * ctx_br.N - 5]
    gks = [GadgetCiphertext(ctx_br, data[2 * n_lwe + t], levelQ, levelP, pw2, sizes) for t in range(window_size + 1)]
    arr = (_lib.GadgetCtStruct * len(gks))(*[k.struct for k in gks])
    _lib.check(_lib.lib().lgpu_blind_rotation_gen_evaluation_key(ctx_br.h, _dptr(sk_br), s_lwe.ctypes.data, n_lwe, window_size, float(sigma),
                                                                  float(bound), seed & 0xFFFFFFFFFFFFFFFF, v0, v1, arr, _stream()))
    return brk, dict(zip(gals, gks))


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

"""Wire-format entry points (include/lattigo_b200.h, csrc/wire.cu): the reference's WriteTo / ReadFrom byte streams
(ring.Poly, rlwe.GadgetCiphertext / EvaluationKey / RelinearizationKey, rlwe.GaloisKey) loaded straight into device memory."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .ring import Context, _stream
from .rlwe import GadgetCiphertext


def gadget_ct_info(ctx: Context, data: bytes) -> _lib.EvkInfoStruct:
    """Sizes a serialised rlwe.GadgetCiphertext without touching the device (works on host-only contexts)."""
    info = _lib.EvkInfoStruct()
    buf = (ctypes.c_char * len(data)).from_buffer_copy(data)
    _lib.check(_lib.lib().lgpu_gadget_ct_load(ctx.h, buf, len(data), None, 0, ctypes.byref(info), None))
    return info


def _finish(ctx, data_t, info):
    sizes = [info.pw2_sizes[i] for i in range(info.n_digits)]
    return GadgetCiphertext(ctx, data_t, info.level_q, info.level_p, info.base_two_decomposition, sizes)


def load_gadget_ct(ctx: Context, data: bytes) -> GadgetCiphertext:
    """rlwe.GadgetCiphertext.UnmarshalBinary (core/rlwe/gadgetciphertext.go:161-167) -> device-resident key."""
    import torch
    info = gadget_ct_info(ctx, data)
    rows = info.level_q + 1 + info.level_p + 1
    t = torch.zeros((info.n_digits, info.n_pw2_max, 2, rows, ctx.N), dtype=torch.int64, device="cuda:%d" % ctx.device)
    buf = (ctypes.c_char * len(data)).from_buffer_copy(data)
    _lib.check(_lib.lib().lgpu_gadget_ct_load(ctx.h, buf, len(data), ctypes.c_void_p(t.data_ptr()), t.numel() * 8, ctypes.byref(info), _stream()))
    torch.cuda.current_stream().synchronize()          # the byte buffer may go away after this call
    return _finish(ctx, t, info)


def load_galois_key(ctx: Context, data: bytes):
    """rlwe.GaloisKey.UnmarshalBinary (core/rlwe/keys.go:670-700) -> (GaloisElement, device-resident key)."""
    import torch
    info = _lib.EvkInfoStruct()
    g, nr = ctypes.c_uint64(), ctypes.c_uint64()
    buf = (ctypes.c_char * len(data)).from_buffer_copy(data)
    _lib.check(_lib.lib().lgpu_galois_key_load(ctx.h, buf, len(data), ctypes.byref(g), ctypes.byref(nr), None, 0, ctypes.byref(info), None))
    rows = info.level_q + 1 + info.level_p + 1
    t = torch.zeros((info.n_digits, info.n_pw2_max, 2, rows, ctx.N), dtype=torch.int64, device="cuda:%d" % ctx.device)
    _lib.check(_lib.lib().lgpu_galois_key_load(ctx.h, buf, len(data), ctypes.byref(g), ctypes.byref(nr), ctypes.c_void_p(t.data_ptr()), t.numel() * 8,
                                               ctypes.byref(info), _stream()))
    torch.cuda.current_stream().synchronize()
    return int(g.value), _finish(ctx, t, info)


def load_poly(ctx: Context, data: bytes, rows_cap: int):
    """ring.Poly.UnmarshalBinary -> ((rows, N) device tensor, bytes consumed)."""
    import torch
    t = torch.zeros((rows_cap, ctx.N), dtype=torch.int64, device="cuda:%d" % ctx.device)
    n, used = ctypes.c_int(), ctypes.c_size_t()
    buf = (ctypes.c_char * len(data)).from_buffer_copy(data)
    _lib.check(_lib.lib().lgpu_poly_load(ctx.h, buf, len(data), ctypes.c_void_p(t.data_ptr()), rows_cap, ctypes.byref(n), ctypes.byref(used), _stream()))
    torch.cuda.current_stream().synchronize()
    return t[: n.value], int(used.value)


def store_poly(ctx: Context, poly) -> bytes:
    """ring.Poly.MarshalBinary of a (rows, N) device tensor."""
    rows = poly.shape[0]
    cap = 8 + rows * (8 + 8 * ctx.N)
    out = np.empty(cap, dtype=np.uint8)
    w = ctypes.c_size_t()
    _lib.check(_lib.lib().lgpu_poly_store(ctx.h, ctypes.c_void_p(poly.data_ptr()), rows, out.ctypes.data, cap, ctypes.byref(w), _stream()))
    return out[: w.value].tobytes()


def store_qp_poly(ctx: Context, poly, levelQ: int = None) -> bytes:
    """ringqp.Poly.MarshalBinary (ring/ringqp/poly.go:90-160) of a (levelQ+1 + levelP+1, N) device tensor, Q rows first: the Q
    ring.Poly bytes, then the P ring.Poly bytes. Without P rows the P part is the empty ring.Poly, a zero row count."""
    nq = len(ctx.Q) if levelQ is None else levelQ + 1
    q = store_poly(ctx, poly[:nq])
    return q + (store_poly(ctx, poly[nq:]) if poly.shape[0] > nq else bytes(8))


def load_qp_poly(ctx: Context, data: bytes):
    """ringqp.Poly.UnmarshalBinary -> ((Q rows then P rows, N) device tensor, bytes consumed)."""
    import torch
    q, used = load_poly(ctx, data, len(ctx.Q))
    if ctx.P:
        p, used_p = load_poly(ctx, data[used:], len(ctx.P))
        return torch.cat([q, p]), used + used_p
    if len(data) < used + 8:
        raise _lib.LgpuError("wire: truncated ring.Poly header")
    if int.from_bytes(data[used: used + 8], "little") != 0:
        raise _lib.LgpuError("wire: destination polynomial has fewer rows than the encoded one")
    return q, used + 8

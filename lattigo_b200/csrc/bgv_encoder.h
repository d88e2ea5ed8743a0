// bgv_encoder.h -- the ring-T steps of bgv.Encoder (bgv_encoder.cu) that the multiparty BGV protocols (mp_refresh.cu) run on their own.
// Ring-T polynomials are n words per entry (n = RingT().N()), entries `batch stride` words apart; Q rows are coefficient domain.
#pragma once
#include "capi_common.h"

namespace lgpu {

struct BgvEncInfo {
    lgpu_ctx* ctx;
    const Ctx* T;     // ring T: degree n over {t}
    u64 t;
    int n;
};
BgvEncInfo bgv_encoder_info(const lgpu_bgv_encoder* e);
// the argument check of RingQ2T at `level` (the CRT accumulator of the big-integer branch); -1 with the error set
int bgv_q2t_check(const lgpu_bgv_encoder* e, int level, int log_gap);
// RingQ2T(level, scaleDown = true), encoder.go:412-467: the reference's words, [0, 3t) on the ModUpExact branch, canonical otherwise
int bgv_ring_q2t(const lgpu_bgv_encoder* e, int level, const u64* src, size_t src_bs, u64* out, size_t out_bs, int batch, cudaStream_t st);
// RingT2Q(level, scaleUp = true), encoder.go:378-407: every ring-T word lifted as the integer it is, times t^-1 mod q_i, spread by gap
int bgv_ring_t2q(const lgpu_bgv_encoder* e, int level, const u64* pT, size_t pT_bs, u64* out, size_t out_bs, int batch, cudaStream_t st);
// EncodeRingT of n []uint64 values per entry (encoder.go:203-262); pT is dense (stride n)
int bgv_encode_ring_t(const lgpu_bgv_encoder* e, const u64* values, size_t vs, u64 scale, u64* pT, int batch, cudaStream_t st);
// DecodeRingT into n []uint64 values per entry (encoder.go:341-374)
int bgv_decode_ring_t(const lgpu_bgv_encoder* e, const u64* pT, size_t pT_bs, u64 scale, u64* values, size_t vs, int batch, cudaStream_t st);

}  // namespace lgpu

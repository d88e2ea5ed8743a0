// encoder.cu -- the CKKS encoder around the special FFT, batched on the device (prec <= 53, ring.Standard):
//   Encoder.Embed / Encode (IsBatched)        schemes/ckks/encoder.go:208-337   IFFT, Complex128ToFixedPointCRT, NTTSparseAndMontgomery
//   Encoder.Encode (!IsBatched)               schemes/ckks/encoder.go:156-189   Float64ToFixedPointCRT, NTT
//   Encoder.Decode / DecodePublic             schemes/ckks/encoder.go:497-762   INTT, polyTo{Complex,Float}{NoCRT,CRT}, FFT, logprec rounding
// The transform itself is lgpu_ckks_special_fft (specialfft.cu), called here through its public entry point.
//
// Floating point is evaluated with explicit round-to-nearest intrinsics in the reference's order (the library also builds with
// --fmad=false), so the quantized words and the decoded doubles equal the Go code's bit for bit (tests/test_gpu_encoder.py, tolerance 0).
//
// Kernels:
//   enc_load_kernel      values -> zero-padded complex scratch (the caller's input is never written)
//   enc_quantize_kernel  one thread per (coefficient, batch entry): SingleFloat64ToFixedPointCRT of the value that lands on that
//                        coefficient after the Y = X^gap spreading (0 elsewhere), for every Q row and P row; canonical + MForm folded in
//                        on the NTT path, the reference's literal (possibly non-canonical) word otherwise. The NTT launchers follow.
//   dec_nocrt_kernel     level 0: polyToComplexNoCRT / polyToFloatNoCRT literally (uint64 wrap of Q - c included)
//   dec_crt_kernel<W>    level >= 1: exact X mod Q_level in W 64-bit words per thread, centred, rounded to double half-to-even
//                        (big.Float.SetInt(.).Float64(), +-Inf past 2^1024), divided by the scale
//   dec_round_kernel     math.Round(x 2^logprec) / 2^logprec per part
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "capi_common.h"
#include "composite.h"
#include "crt.cuh"
#include "modarith.cuh"

namespace lgpu {

constexpr int kEncThreads = 256;

// ---- encoding --------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kEncThreads) enc_load_kernel(const double2* __restrict__ in, size_t in_stride, int n_values, int slots,
                                                               double2* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= slots) return;
    const size_t b = blockIdx.y;
    out[b * slots + i] = i < n_values ? in[b * in_stride + i] : make_double2(0.0, 0.0);
}

// SingleFloat64ToFixedPointCRT (schemes/ckks/utils.go:171-234) for one modulus; v = value * (+-scale) already formed, neg = value < 0.
// For v >= 2^64 the word is (m 2^e) mod q of the exact integer v (big.NewFloat(v).Add(0.5).Int() keeps v: its ulp is >= 2^12).
__device__ __forceinline__ u64 quantize_word(double v, bool neg, u64 q, u64 bhi) {
    if (v >= 18446744073709551616.0) {
        u64 r = 0;
        if (!isinf(v)) {                                     // +Inf: Float.Int returns nil and leaves xInt = 0
            int e;
            const double f = frexp(v, &e);                   // v = f 2^e, f in [0.5, 1)
            r = bred_add((u64)scalbn(f, 53), q, bhi);        // 53-bit mantissa m, v = m 2^(e-53)
            for (int k = 0; k < e - 53; k++) { r <<= 1; r = r >= q ? r - q : r; }
        }
        return neg ? q - r : r;
    }
    const u64 c = __double2ull_rz(__dadd_rn(v, 0.5));       // uint64(value + 0.5)
    if (neg) return c > q ? q - bred_add(c, q, bhi) : q - c;
    return c > 0x1fffffffffffffffull ? bred_add(c, q, bhi) : c;
}

// grid (ceil(N / 256), batch). Coefficient `col` holds real part j (j < slots) or imaginary part j - slots of the IFFT output when
// col = j * gap (NTTSparseAndMontgomery's Y = X^gap), and 0 otherwise. coeffs = 1: float64 values, n_values of them at gap 1.
__global__ void __launch_bounds__(kEncThreads) enc_quantize_kernel(const double* __restrict__ vals, size_t vals_stride, int coeffs, int n_values,
                                                                   int slots, int log_gap, double scale, int canon, int mont,
                                                                   const LimbConst* __restrict__ limbs, int nrows_q, int limb_p0, int nrows_p,
                                                                   u64* __restrict__ out_q, size_t sq, u64* __restrict__ out_p, size_t sp, int N) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= N) return;
    const size_t b = blockIdx.y;
    double value = 0.0;
    if (coeffs) {
        if (col < n_values) value = vals[b * vals_stride + col];
    } else if ((col & ((1 << log_gap) - 1)) == 0) {
        const int j = col >> log_gap;
        value = j < slots ? vals[b * vals_stride + 2 * (size_t)j] : vals[b * vals_stride + 2 * (size_t)(j - slots) + 1];
    }
    const bool zero = value == 0.0;                          // also -0
    const bool neg = value < 0.0;
    const double v = __dmul_rn(value, neg ? -scale : scale);
    for (int r = 0; r < nrows_q + nrows_p; r++) {
        const bool isq = r < nrows_q;
        const LimbConst& L = limbs[isq ? r : limb_p0 + r - nrows_q];
        u64 w = zero ? 0 : quantize_word(v, neg, L.q, L.bred_hi);
        if (canon) w = bred_add(w, L.q, L.bred_hi);
        if (mont) w = mform(w, L.q, L.bred_hi, L.bred_lo);
        if (isq) out_q[b * sq + (size_t)r * N + col] = w;
        else out_p[b * sp + (size_t)(r - nrows_q) * N + col] = w;
    }
}

// ---- decoding --------------------------------------------------------------------------------------------------------

// where decoded coefficient j goes: the float64 coefficient j (coeffs), or part j / slots of complex value j mod slots
__device__ __forceinline__ size_t dec_pos(int j, int slots, int coeffs) {
    return coeffs ? (size_t)j : (j < slots ? 2 * (size_t)j : 2 * (size_t)(j - slots) + 1);
}

// polyToComplexNoCRT (encoder.go:823-860) / polyToFloatNoCRT (:1119-1160). Complex: values[i] = complex(x, 0), values[i] += complex(0, y),
// then /= complex(scale, 0); Go's complex division by (s, 0) is e = (a + b 0) / s, f = (b - a 0) / s, equal to the per-part quotient here
// because neither part is -0 after the += and both are finite. Float: x / scale directly, so c = Q gives -0.
__global__ void __launch_bounds__(kEncThreads) dec_nocrt_kernel(const u64* __restrict__ pt, size_t pt_stride, int count, int log_gap, int slots,
                                                                int coeffs, u64 Q, double scale, double* __restrict__ out, size_t out_stride) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const size_t b = blockIdx.y;
    const u64 c = pt[b * pt_stride + ((size_t)j << log_gap)];
    const double x = c >= (Q >> 1) ? -__ull2double_rn(Q - c) : __ull2double_rn(c);
    double y;
    if (coeffs) y = x;
    else y = j < slots ? __dadd_rn(x, 0.0) : __dadd_rn(0.0, x);
    out[b * out_stride + dec_pos(j, slots, coeffs)] = __ddiv_rn(y, scale);
}

// round-half-to-even of the W-word magnitude m to double (big.Float.Float64 of an exact integer), +Inf past the largest double
template <int W>
__device__ __forceinline__ double words_to_double(const u64 (&m)[W + 1]) {
    int top = -1;
    u64 mtop = 0;                                                 // m[top], kept out of a dynamic index (the words stay in registers)
#pragma unroll
    for (int w = W - 1; w >= 0; w--)
        if (top < 0 && m[w] != 0) { top = w; mtop = m[w]; }
    if (top < 0) return 0.0;
    const int bl = 64 * top + 64 - __clzll((long long)mtop);     // bit length
    if (bl <= 64) return __ull2double_rn(m[0]);
    // the 64 bits below the top one, plus a sticky bit for everything lower
    const int s = bl - 64;                                        // shift: window = m >> s
    const int ws = s >> 6, bs = s & 63;
    u64 win = 0, sticky = 0;
#pragma unroll
    for (int w = 0; w < W; w++) {
        if (w < ws) sticky |= m[w];
        else if (w == ws) { win = bs ? (m[w] >> bs) : m[w]; sticky |= bs ? (m[w] << (64 - bs)) : 0; }
        else if (w == ws + 1 && bs) win |= m[w] << (64 - bs);
    }
    // win has its top bit set; keep 53 bits, round bit 10, sticky bits 0..9 and below
    u64 mant = win >> 11;
    const bool rnd = (win >> 10) & 1;
    const bool st = (win & 0x3ff) != 0 || sticky != 0;
    if (rnd && (st || (mant & 1))) mant++;                        // may reach 2^53: still exact below
    const int e = s + 11;                                         // value = mant 2^e, mant in [2^52, 2^53]
    if (e >= 972 || (e == 971 && (mant >> 53))) return __longlong_as_double(0x7ff0000000000000ll);   // >= 2^1024: +Inf
    return scalbn((double)mant, e);
}

// polyToComplexCRT (encoder.go:924-971) / polyToFloatCRT (:1033-1082): coefficient j << log_gap of rows 0..L-1 (never above `level`: the
// reference's X mod Q_level depends on those rows only), centred (>= Q >> 1 gives X - Q), scaleDown = Float64(X) / scale. Complex: the
// imaginary part arrives through values[i] += complex(0, .), i.e. 0 + y and x + 0.
template <int W>
__global__ void __launch_bounds__(kEncThreads) dec_crt_kernel(const u64* __restrict__ pt, size_t pt_stride, size_t row_stride, int count, int log_gap,
                                                              int slots, int coeffs, CrtTab T, double scale, double* __restrict__ out, size_t out_stride) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    const size_t b = blockIdx.y;
    u64 acc[W + 1];
    crt_exact<W>(pt + b * pt_stride + ((size_t)j << log_gap), row_stride, T, acc);
    const bool ge = mw_ge<W>(acc, T.Qh);                         // acc >= floor(Q/2)
    if (ge) {                                                    // |X - Q| = Q - X
        u64 br = 0;
#pragma unroll
        for (int w = 0; w < W; w++) {
            const u64 a = T.Q[w], x = acc[w];
            acc[w] = a - x - br;
            br = (a < x) || (a - x < br);
        }
    }
    acc[W] = 0;
    double x = words_to_double<W>(acc);
    if (ge) x = -x;
    double y = __ddiv_rn(x, scale);
    if (!coeffs) y = j < slots ? __dadd_rn(y, 0.0) : __dadd_rn(0.0, y);
    out[b * out_stride + dec_pos(j, slots, coeffs)] = y;
}

// math.Round(x * s) / s per double (decodePublic, encoder.go:536-549); round() is half away from zero like math.Round
__global__ void __launch_bounds__(kEncThreads) dec_round_kernel(double* __restrict__ v, size_t stride, int count, double s) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    double* p = v + (size_t)blockIdx.y * stride + i;
    *p = __ddiv_rn(round(__dmul_rn(*p, s)), s);
}

// ---- host side -------------------------------------------------------------------------------------------------------

template <int W>
static void launch_crt(dim3 grid, cudaStream_t st, const u64* pt, size_t pt_stride, size_t N, int count, int log_gap, int slots, int coeffs,
                       const CrtTab& T, double scale, double* out, size_t out_stride) {
    dec_crt_kernel<W><<<grid, kEncThreads, 0, st>>>(pt, pt_stride, N, count, log_gap, slots, coeffs, T, scale, out, out_stride);
}

}  // namespace lgpu

using namespace lgpu;

static bool aligned_to(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

static const char* kSparseCoeffMsg =
    "coefficient-domain batched encoding with slots < N/2 is not supported: the reference's spreading loop (core/rlwe/utils.go:234-241, "
    "NTTSparseAndMontgomery) reuses j in its inner loop and either indexes past N or zeroes inputs before they are moved, so it has no "
    "defined output";

extern "C" int lgpu_ckks_encode(lgpu_ctx* ctx, const double* values, int n_values, int log_slots, double scale, int flags, const int64_t* rot_group,
                                const double* roots, int level_q, uint64_t* out_q, int level_p, uint64_t* out_p, int batch, size_t values_stride,
                                size_t out_q_stride, size_t out_p_stride, void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "CKKS encoding is only supported on the Standard ring (the ConjugateInvariant ring is not)");
    REQUIRE((flags & ~(LGPU_ENC_NTT | LGPU_ENC_MONTGOMERY | LGPU_ENC_COEFFS)) == 0, "unknown encoder flags");
    const bool coeffs = flags & LGPU_ENC_COEFFS, ntt = flags & LGPU_ENC_NTT, mont = !coeffs && (flags & LGPU_ENC_MONTGOMERY);
    REQUIRE(std::isfinite(scale) && scale > 0, "scale must be finite and positive");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(level_q >= 0 && level_q < c.nQ, "level_q out of range");
    REQUIRE(level_p >= -1 && level_p < c.nP, c.nP ? "level_p out of range" : "level_p out of range: the context has no P moduli");
    const int N = c.N;
    int slots = 0;
    if (coeffs) {
        REQUIRE(n_values >= 0 && n_values <= N, "cannot Encode: maximum number of values is N");
        REQUIRE(level_p == -1, "coefficient encoding (IsBatched = false) writes a ring.Poly: level_p must be -1");
    } else {
        REQUIRE(log_slots >= 0 && log_slots <= c.logN - 1, "cannot Embed: logSlots must be in [0, LogN - 1]");
        slots = 1 << log_slots;
        REQUIRE(n_values >= 0 && n_values <= slots, "cannot Embed: ensure that #values <= slots");
        REQUIRE(ntt || slots == N / 2, kSparseCoeffMsg);
        REQUIRE(rot_group && roots, "null rot_group / roots");
        REQUIRE(aligned_to(rot_group, 8) && aligned_to(roots, 16), "rot_group must be 8-byte and roots 16-byte aligned");
    }
    REQUIRE(n_values == 0 || values, "null values");
    REQUIRE(aligned_to(values, coeffs ? 8 : 16), "values must be 8-byte (float64) or 16-byte (complex128) aligned");
    REQUIRE(out_q && aligned_to(out_q, 8), "null or misaligned out_q");
    REQUIRE(level_p < 0 || (out_p && aligned_to(out_p, 8)), "null or misaligned out_p");
    REQUIRE(batch == 1 || (values_stride >= (size_t)n_values && out_q_stride >= (size_t)(level_q + 1) * N &&
                           (level_p < 0 || out_p_stride >= (size_t)(level_p + 1) * N)), "batch strides smaller than one entry");
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    const double* vals = values;
    size_t vstride = values_stride;
    Scratch buf;
    if (!coeffs) {
        if (buf.alloc((size_t)2 * slots * batch, st)) return -1;
        count_launch(1);
        enc_load_kernel<<<dim3((slots + kEncThreads - 1) / kEncThreads, batch), kEncThreads, 0, st>>>(
            reinterpret_cast<const double2*>(values), values_stride, n_values, slots, reinterpret_cast<double2*>(buf.p));
        LGPU_CUDA_OK(cudaGetLastError());
        if (lgpu_ckks_special_fft(ctx, reinterpret_cast<double*>(buf.p), slots, 2 * N, rot_group, roots, 1, batch, slots, stream)) return -1;
        vals = reinterpret_cast<const double*>(buf.p);
        vstride = (size_t)2 * slots;                              // in doubles
    }
    int log_gap = 0;
    if (!coeffs) while ((slots << (log_gap + 1)) < N) log_gap++;
    count_launch(1);
    enc_quantize_kernel<<<dim3((N + kEncThreads - 1) / kEncThreads, batch), kEncThreads, 0, st>>>(
        vals, vstride, coeffs, n_values, slots, log_gap, scale, ntt, mont, c.d_limbs, level_q + 1, c.nQ, level_p + 1, (u64*)out_q, out_q_stride,
        (u64*)out_p, out_p_stride, N);
    LGPU_CUDA_OK(cudaGetLastError());
    if (ntt) {
        RowMap rm;
        if (make_rowmap(c, LGPU_RING_Q, level_q, rm)) return -1;
        if (launch_ntt(&c, rm, CSpan{(const u64*)out_q, (size_t)N, out_q_stride}, Span{(u64*)out_q, (size_t)N, out_q_stride}, batch, NTT_CANONICAL, st))
            return -1;
        if (level_p >= 0) {
            if (make_rowmap(c, LGPU_RING_P, level_p, rm)) return -1;
            if (launch_ntt(&c, rm, CSpan{(const u64*)out_p, (size_t)N, out_p_stride}, Span{(u64*)out_p, (size_t)N, out_p_stride}, batch,
                           NTT_CANONICAL, st))
                return -1;
        }
    }
    return 0;
}

extern "C" int lgpu_ckks_decode(lgpu_ctx* ctx, const uint64_t* pt, int level, int log_slots, double scale, int flags, double logprec,
                                const int64_t* rot_group, const double* roots, double* values, int batch, size_t pt_stride, size_t values_stride,
                                void* stream) {
    REQUIRE(ctx, "null context");
    const Ctx& c = ctx->c;
    REQUIRE(c.ring_type == 0, "CKKS decoding is only supported on the Standard ring (the ConjugateInvariant ring is not)");
    REQUIRE((flags & ~(LGPU_ENC_NTT | LGPU_ENC_MONTGOMERY | LGPU_ENC_COEFFS)) == 0, "unknown encoder flags");
    const bool coeffs = flags & LGPU_ENC_COEFFS, ntt = flags & LGPU_ENC_NTT;
    REQUIRE(std::isfinite(scale) && scale > 0, "scale must be finite and positive");
    REQUIRE(batch >= 1 && batch <= 65535, "batch out of range");
    REQUIRE(level >= 0 && level < c.nQ, "level out of range");
    REQUIRE(log_slots >= 0 && log_slots <= c.logN - 1, "cannot Decode: logSlots must be in [0, LogN - 1]");
    const int N = c.N, slots = 1 << log_slots;
    const bool round_prec = !coeffs && logprec != 0;
    if (round_prec)
        REQUIRE(logprec == std::floor(logprec) && logprec >= -1022 && logprec <= 1023,
                "logprec must be an integer in [-1022, 1023] (math.Exp2 of other values is not reproduced)");
    if (!coeffs) {
        REQUIRE(rot_group && roots, "null rot_group / roots");
        REQUIRE(aligned_to(rot_group, 8) && aligned_to(roots, 16), "rot_group must be 8-byte and roots 16-byte aligned");
    }
    REQUIRE(pt && aligned_to(pt, 8), "null or misaligned plaintext");
    REQUIRE(values && aligned_to(values, coeffs ? 8 : 16), "null or misaligned values (8-byte float64, 16-byte complex128)");
    REQUIRE(batch == 1 || (pt_stride >= (size_t)(level + 1) * N && values_stride >= (size_t)(coeffs ? N : slots)), "batch strides smaller than one entry");
    const int words = level ? crt_words(c, level) : 0;
    REQUIRE(words <= kMaxCrtWords, "the bit lengths of q_0..q_level sum past 4096: the CRT accumulator exceeds 4096 bits");
    REQUIRE_DEVICE(ctx);
    const cudaStream_t st = (cudaStream_t)stream;
    const size_t rows = (size_t)level + 1, poly = rows * N;
    const int count = coeffs ? N : 2 * slots;
    int log_gap = 0;
    if (!coeffs) while ((slots << (log_gap + 1)) < N) log_gap++;
    const size_t ostride = coeffs ? values_stride : 2 * values_stride;   // in doubles
    // CRT constants
    Scratch tab;
    CrtTab T{};
    const int W = level ? crt_width(words) : 0;
    if (level) {
        std::vector<u64> blob = build_crt(c, level, W);
        if (tab.alloc(blob.size(), st)) return -1;
        // pageable source: the call returns once `blob` is staged, so it may die with this function
        LGPU_CUDA_OK(cudaMemcpyAsync(tab.p, blob.data(), blob.size() * 8, cudaMemcpyHostToDevice, st));
        const int L = level + 1;
        T.q = tab.p; T.bhi = tab.p + L; T.blo = tab.p + 2 * L; T.inv = tab.p + 3 * L; T.rq = reinterpret_cast<const double*>(tab.p + 4 * L);
        T.qhat = tab.p + 5 * L; T.Q = T.qhat + (size_t)L * W; T.Qh = T.Q + W; T.L = L;
    }
    // INTT into scratch in sub-batches of at most ~256 MB (the plaintext is never written)
    const int ch = ntt ? (int)std::max<size_t>(1, std::min<size_t>(batch, ((size_t)256 << 20) / (poly * 8))) : batch;
    Scratch buf;
    if (ntt && buf.alloc(poly * ch, st)) return -1;
    RowMap rm;
    if (make_rowmap(c, LGPU_RING_Q, level, rm)) return -1;
    for (int k = 0; k < batch; k += ch) {
        const int nb = std::min(ch, batch - k);
        const u64* src = (const u64*)pt + (size_t)k * pt_stride;
        size_t sstride = pt_stride;
        if (ntt) {
            if (launch_intt(&c, rm, CSpan{src, (size_t)N, pt_stride}, Span{buf.p, (size_t)N, poly}, nb, NTT_CANONICAL, st)) return -1;
            src = buf.p; sstride = poly;
        }
        double* out = values + (size_t)k * ostride;
        const dim3 grid((count + kEncThreads - 1) / kEncThreads, nb);
        count_launch(1);
        if (!level) {
            dec_nocrt_kernel<<<grid, kEncThreads, 0, st>>>(src, sstride, count, log_gap, slots, coeffs, c.Q[0], scale, out, ostride);
        } else {
            switch (W) {
                case 16: launch_crt<16>(grid, st, src, sstride, N, count, log_gap, slots, coeffs, T, scale, out, ostride); break;
                case 32: launch_crt<32>(grid, st, src, sstride, N, count, log_gap, slots, coeffs, T, scale, out, ostride); break;
                default: launch_crt<64>(grid, st, src, sstride, N, count, log_gap, slots, coeffs, T, scale, out, ostride); break;
            }
        }
        LGPU_CUDA_OK(cudaGetLastError());
    }
    if (!coeffs) {
        if (lgpu_ckks_special_fft(ctx, values, slots, 2 * N, rot_group, roots, 0, batch, values_stride, stream)) return -1;
        if (round_prec) {
            count_launch(1);
            dec_round_kernel<<<dim3((2 * slots + kEncThreads - 1) / kEncThreads, batch), kEncThreads, 0, st>>>(values, ostride, 2 * slots,
                                                                                                             std::ldexp(1.0, (int)logprec));
            LGPU_CUDA_OK(cudaGetLastError());
        }
    }
    return 0;
}

// xpow.cuh -- in-thread monomial products and automorphism indices in the NTT domain (ringpacking.cu, blindrot.cu).
#pragma once
#include "engine.h"
#include "modarith.cuh"

namespace lgpu {

// slot j of NTT(X^k) is psi^(k * (2 brev(j) + 1)) (the evaluation order of the forward transform): psi^e = tw_fwd[brev(e)] for
// e < N and -psi^(e - N) past it. x * that, canonical; k is taken mod 2N (k = 2N - n for X^-n).
__device__ __forceinline__ u64 mul_xpow(u64 x, u64 k, u64 slot_odd, const LimbConst& L, int lg, u64 mask2n) {
    u64 e = (k * slot_odd) & mask2n;
    const u64 n = (mask2n + 1) >> 1, q = L.q;
    const bool neg = e >= n;
    if (neg) e -= n;
    const ulonglong2 w = L.tw_fwd[__brevll(e) >> (64 - lg)];
    const u64 r = cred(x * w.x - __umul64hi(x, w.y) * q, q);
    return neg ? (r ? q - r : 0) : r;
}
__device__ __forceinline__ size_t auto_index(int j, u64 galEl, u64 mask2n, int lg) {     // ring/automorphism.go:12-34
    const u64 tmp1 = 2 * (__brevll((u64)j) >> (64 - lg)) + 1;
    return (size_t)(__brevll(((galEl * tmp1 & mask2n) - 1) >> 1) >> (64 - lg));
}

}  // namespace lgpu

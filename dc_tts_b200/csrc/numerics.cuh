// numerics.cuh -- the kernels' shared arithmetic: the split-fp16 operand format, its power-of-two scales, the warp sum and
// the accurate sigmoid.  Every kernel, the weight packers included, uses these definitions; none restates them.
//
// Split-fp16 operands ("split planes"): every fp32 value x that feeds the fp16 tensor cores is held as two fp16 tensors
// hi = fp16(s x), lo = fp16(s x - hi) (22 significand bits together, 4 bytes per element like fp32) with a power-of-two
// scale s.  A product is three wgmma passes per k-step, hi*hi' + hi*lo' + lo*hi', accumulated in fp32 registers --
// fp32-grade results on the fp16 tensor pipe (the dropped lo*lo' term is 2^-22 relative).  Single-pass fp16 / tf32
// operands miss the 1e-3 parity budget (DESIGN.md section 5).  s x is exact in fp32: s only moves the values into fp16's
// normal range and is undone on the fp32 accumulator.  Hidden activations are LayerNorm outputs, O(1) per row, and
// unscaled (s = 1).  Each kind of operand has its own window for s below; they differ on purpose.
#pragma once
#include <cmath>
#include <cuda_fp16.h>
#include <stdint.h>
#include <type_traits>

namespace dctts {

__host__ __device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
    hi = __float2half_rn(v);
    lo = __float2half_rn(v - __half2float(hi));
}
__host__ __device__ __forceinline__ float join_f16(__half hi, __half lo) { return __half2float(hi) + __half2float(lo); }

// two adjacent elements as one __half2 of each plane (both hi halves first)
__host__ __device__ __forceinline__ void split_f16x2(float2 v, __half2& hi, __half2& lo) {
    const __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y);
    hi = __halves2half2(h0, h1);
    lo = __halves2half2(__float2half_rn(v.x - __half2float(h0)), __float2half_rn(v.y - __half2float(h1)));
}

// N = 4, 8 or 16 consecutive values -> N consecutive halfs at hi and at lo (8- or 16-byte aligned): vector stores,
// all of the hi plane first
template <int N>
__device__ __forceinline__ void split_store_f16(const float* v, __half* hi, __half* lo) {
    static_assert(N == 4 || N == 8 || N == 16, "one 8-byte, one 16-byte or two 16-byte stores per plane");
    using V = typename std::conditional<N == 4, uint2, uint4>::type;
    constexpr int NV = N * (int)sizeof(__half) / (int)sizeof(V);
    __align__(16) __half h[N];
    __align__(16) __half l[N];
#pragma unroll
    for (int i = 0; i < N; ++i) split_f16(v[i], h[i], l[i]);
#pragma unroll
    for (int i = 0; i < NV; ++i) reinterpret_cast<V*>(hi)[i] = reinterpret_cast<const V*>(h)[i];
#pragma unroll
    for (int i = 0; i < NV; ++i) reinterpret_cast<V*>(lo)[i] = reinterpret_cast<const V*>(l)[i];
}

// ---- the scales s, one rule per kind of operand ----
// Weights of the block kernels and of the persistent decode's pre-pass (kernels_pack.cu; the host computes s from the
// device abs-max): max|W| s in [2^10, 2^11), so that the lo plane stays in fp16's normal range; the kernel multiplies the
// accumulator by 1 / s.
inline float weight_scale(float maxabs) {
    float s = 1.f;
    if (maxabs > 0.f) { int e; std::frexp(maxabs, &e); s = std::ldexp(1.f, 11 - e); }
    return s;
}

// The audio-level input of AudioEnc, AudioDec and SSRN, per utterance from its abs-max m: m s in [2^14, 2^15) (1 for an
// all-zero or non-finite utterance).  Unscaled, silence at 1e-8 flushes to zero and 1e-6 .. 1e-4 keep a few bits.
__device__ __forceinline__ float utterance_scale(float m) {
    float s = 1.f;
    if (m > 0.f && isfinite(m)) {
        int e;
        frexpf(m, &e);                                     // m in [2^(e-1), 2^e)
        s = ldexpf(1.f, min(15 - e, 100));                 // 1/s stays a normal float
    }
    return s;
}

// The operands of the training conv-GEMMs, per tensor from the abs-max in `slot` (float bits): max s in [2^13, 2^14), so
// that gradients of 1e-7 and weights of 1e-2 both use fp16's normal range.  The biased exponent is clamped to [1, 254]:
// s is a normal float.
__device__ __forceinline__ float slot_scale(const unsigned* slot) {
    const float m = __uint_as_float(*slot);
    if (!(m > 0.f) || !(m < 3.0e38f)) return 1.0f;
    int e = 127 + 13 - ilogbf(m);
    e = e < 1 ? 1 : (e > 254 ? 254 : e);
    return __uint_as_float((unsigned)e << 23);
}

// ---- reductions and activations whose bits the parity tests pin ----
// butterfly sum over the warp: every lane ends with the same value, summed in this order
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// expf, not __expf: the accurate sigmoid of the LayerNorm epilogues and the highway gate
__device__ __forceinline__ float sigmoid_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

}  // namespace dctts

// Shared helpers for the lt_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/lt_b200.h"

namespace lt {

// ---- error reporting ------------------------------------------------------------------------
char* err_buf();  // thread-local 512-byte buffer (capi.cu)
int fail(int code, const char* fmt, ...);

#define LT_REQUIRE(cond, ...)                                   \
  do {                                                          \
    if (!(cond)) return ::lt::fail(LT_ERR_INVALID, __VA_ARGS__); \
  } while (0)

#define LT_CHECK_LAUNCH(name)                                                                  \
  do {                                                                                         \
    cudaError_t e__ = cudaGetLastError();                                                      \
    if (e__ != cudaSuccess) return ::lt::fail(LT_ERR_CUDA, "%s: %s", name, cudaGetErrorString(e__)); \
  } while (0)

const lt_options& opts();   // process-wide kernel-selection options (capi.cu; lt_set_options)
int sm_count();  // cached cudaDevAttrMultiProcessorCount of the current device

// One-time per-DEVICE setup (cudaFuncSetAttribute is a per-device property): `first()` is true exactly once per device ordinal
// for each DeviceOnce object, from whichever host thread gets there first.
struct DeviceOnce {
  unsigned long long done = 0;
  bool first() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev > 63) return true;
    const unsigned long long bit = 1ull << dev;
    return (__atomic_fetch_or(&done, bit, __ATOMIC_ACQ_REL) & bit) == 0;
  }
};

static inline int ceil_div(long a, long b) { return (int)((a + b - 1) / b); }

// ---- split-fp16 ("S32") format ----------------------------------------------------------------
// x ~= hi + lo with hi = fp16_rn(x), lo = fp16_rn(x - hi): two fp16 tensor-core operands carrying ~22 significand bits.
// The low part is stored UNSCALED (round 2; it was pre-scaled by 2^11 in round 1), so the three products hi*hi, hi*lo,
// lo*hi of a K slice are commensurable and may share an fp32 accumulator (the conv kernels keep the cross products in a second
// one).  Price: for |x| < ~0.125 the low part is an fp16 subnormal, i.e. the representation error is
// max(2^-22 |x|, 2^-25) absolute -- 3e-8, far below the 1e-3 contract for BatchNorm-scaled activations and Kaiming-scaled
// weights (CPU emulation on the calibrated test model: per-layer relative error 1.9e-7..9.0e-7;
// checked on the GPU by tests/test_gpu_tc.py / test_gpu_forward.py).  |x| is saturated at the fp16 maximum (65504).
typedef __half sh_t;
constexpr float kLoScale = 1.0f;   // kept as named constants: the two-accumulator kernels (conv_tc.cu, conv_tc_fold.cu) form D1 + kLoInv * D2
constexpr float kLoInv = 1.0f;

__device__ __forceinline__ void split_s32(float x, sh_t& hi, sh_t& lo) {
  x = fminf(fmaxf(x, -65504.0f), 65504.0f);
  hi = __float2half_rn(x);
  lo = __float2half_rn((x - __half2float(hi)) * kLoScale);
}
__device__ __forceinline__ float join_s32(sh_t hi, sh_t lo) {
  return fmaf(__half2float(lo), kLoInv, __half2float(hi));
}
// element offset (in 2-byte units) of the high part of channel c of a pixel whose row starts at 0;
// low part is +32.
__device__ __host__ __forceinline__ int s32_off(int c) { return ((c >> 5) << 6) + (c & 31); }

// 4 consecutive channels (c % 4 == 0) <-> split storage
__device__ __forceinline__ void store_s32x4(sh_t* row, int c, float4 v) {
  sh_t h[4], l[4];
  split_s32(v.x, h[0], l[0]);
  split_s32(v.y, h[1], l[1]);
  split_s32(v.z, h[2], l[2]);
  split_s32(v.w, h[3], l[3]);
  sh_t* p = row + s32_off(c);
  *reinterpret_cast<uint2*>(p) = *reinterpret_cast<uint2*>(h);
  *reinterpret_cast<uint2*>(p + 32) = *reinterpret_cast<uint2*>(l);
}
__device__ __forceinline__ float4 load_s32x4(const sh_t* row, int c) {
  const sh_t* p = row + s32_off(c);
  uint2 hu = *reinterpret_cast<const uint2*>(p);
  uint2 lu = *reinterpret_cast<const uint2*>(p + 32);
  const sh_t* h = reinterpret_cast<const sh_t*>(&hu);
  const sh_t* l = reinterpret_cast<const sh_t*>(&lu);
  return make_float4(join_s32(h[0], l[0]), join_s32(h[1], l[1]), join_s32(h[2], l[2]), join_s32(h[3], l[3]));
}

// Power-of-two pre-scale of a layer's filter (tensor-core path): S = 2^(9 - floor(log2 max|w|)) puts max|w| * S into
// [512, 1024), so that the UNSCALED low parts of every weight down to 2^-13 of the largest stay normal fp16 numbers (full
// ~22-bit operands); Kaiming-sized filters (|w| ~ 0.03) would otherwise keep only ~2^-20 relative precision, which a
// 152-layer trunk amplifies to ~1.5e-4 at the features (measured).  1 / S is folded into the
// epilogue scale (exact).  absmax_bits: the float bit pattern of max|w| (lt_absmax_fwd), or null for "no scaling".
__device__ __forceinline__ float weight_pow2_scale(const unsigned* absmax_bits) {
  if (!absmax_bits) return 1.0f;
  const unsigned b = *absmax_bits;
  const int e = (int)(b >> 23) - 127;     // floor(log2(max)) for normal floats
  if (b == 0u || e < -100 || e > 100) return 1.0f;
  return exp2f((float)(9 - e));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace lt

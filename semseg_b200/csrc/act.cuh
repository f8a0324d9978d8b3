// Activation storage forms shared by the elementwise / pooling kernels.
//
//   plain : one bf16 NHWC tensor (the speed configuration, "bf16").
//   split : two bf16 NHWC planes (hi, lo) with the same pitch whose fp32 sum is the value: hi = bf16(v),
//           lo = bf16(v - hi) -> 16 mantissa bits. The convolution kernels consume the planes as extra K segments
//           (x_hi*w_hi + x_lo*w_hi + x_hi*w_lo, fp32 accumulation in registers: the error-compensated "bf16x3" operand
//           mode, SURVEY.md §7 hard part 1), which is what lets the path meet north_star's 1e-3 / exact-argmax
//           parity with the fp32 reference (model/resnet.py:63-92 computes in fp32 / TF32).
//
// Every kernel is templated on `S` (split or not); with S = false the lo pointers are never dereferenced and the code
// is the plain bf16 kernel.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

#include "ptx.cuh"

namespace sb {

typedef __nv_bfloat16 bf16_t;

__device__ __forceinline__ void act_unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float2 t = __bfloat1622float2(h[q]);
    f[2 * q] = t.x;
    f[2 * q + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 act_pack8(const float (&f)[8]) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  return o;
}

// Eight consecutive channels as raw 16-byte words (so that several loads can be issued before the first unpack).
template <bool S>
struct Raw8 {
  uint4 h;
  uint4 l;  // untouched when !S
};
template <bool S>
__device__ __forceinline__ Raw8<S> act_ldraw(const bf16_t* hi, const bf16_t* lo, long long off) {
  Raw8<S> r;
  r.h = *reinterpret_cast<const uint4*>(hi + off);
  if constexpr (S) r.l = *reinterpret_cast<const uint4*>(lo + off);
  return r;
}
template <bool S>
__device__ __forceinline__ void act_unpack(const Raw8<S>& r, float (&f)[8]) {
  act_unpack8(r.h, f);
  if constexpr (S) {
    float g[8];
    act_unpack8(r.l, g);
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] += g[q];
  }
}
template <bool S>
__device__ __forceinline__ void act_ld8(const bf16_t* hi, const bf16_t* lo, long long off, float (&f)[8]) {
  act_unpack<S>(act_ldraw<S>(hi, lo, off), f);
}
template <bool S>
__device__ __forceinline__ void act_st8(bf16_t* hi, bf16_t* lo, long long off, const float (&f)[8]) {
  const uint4 h = act_pack8(f);
  *reinterpret_cast<uint4*>(hi + off) = h;
  if constexpr (S) {
    float hf[8], r[8];
    act_unpack8(h, hf);
#pragma unroll
    for (int q = 0; q < 8; ++q) r[q] = f[q] - hf[q];
    *reinterpret_cast<uint4*>(lo + off) = act_pack8(r);
  }
}
// single element
__device__ __forceinline__ void act_split1(float v, bf16_t& hi, bf16_t& lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Launch helper: KERNEL<true>/<false> chosen by whether lo planes were passed.
#define SB_ACT_DISPATCH(split, ...)            \
  do {                                         \
    if (split) {                               \
      constexpr bool kS = true;                \
      __VA_ARGS__;                             \
    } else {                                   \
      constexpr bool kS = false;               \
      __VA_ARGS__;                             \
    }                                          \
  } while (0)

}  // namespace sb

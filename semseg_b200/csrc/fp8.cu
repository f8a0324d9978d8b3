// FP8 (e4m3) eval support: activation quantisation, calibration amax, and the per-output-channel weight pack.
// One formula everywhere (the conv epilogue's e4m3 output included): q = cvt.rn.satfinite.e4m3(v * qscale).
#include <cuda_bf16.h>

#include "host_common.h"
#include "ptx.cuh"

namespace sb {

// 16 channels per thread: two 16-byte loads of bf16, one 16-byte store of e4m3.
__global__ void fp8_quantize_kernel(const __nv_bfloat16* __restrict__ x, int x_pitch, uint8_t* __restrict__ y,
                                    int y_pitch, long long M, int C, float qscale) {
  const int groups = C / 16;
  const long long total = M * groups;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long m = i / groups;
    const int c = static_cast<int>(i - m * groups) * 16;
    const uint4* src = reinterpret_cast<const uint4*>(x + m * x_pitch + c);
    uint4 v[2] = {__ldg(src), __ldg(src + 1)};
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(v);
    uint32_t out[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = __bfloat1622float2(h[2 * k]), b = __bfloat1622float2(h[2 * k + 1]);
      out[k] = static_cast<uint32_t>(pack_e4m3x2(a.x * qscale, a.y * qscale)) |
               (static_cast<uint32_t>(pack_e4m3x2(b.x * qscale, b.y * qscale)) << 16);
    }
    *reinterpret_cast<uint4*>(y + m * y_pitch + c) = make_uint4(out[0], out[1], out[2], out[3]);
  }
}

// max |x| as fp32 bits (= bf16 bits << 16 with the sign cleared); NaN (bits > 0x7f80_0000) is skipped.
__global__ void fp8_amax_kernel(const __nv_bfloat16* __restrict__ x, int x_pitch, long long M, int C,
                                unsigned int* __restrict__ amax_bits) {
  const int groups = C / 8;
  const long long total = M * groups;
  uint32_t best = 0;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long m = i / groups;
    const int c = static_cast<int>(i - m * groups) * 8;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + m * x_pitch + c));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t lo = (w[k] & 0x7fffu) << 16, hi = w[k] & 0x7fff0000u;
      if (lo <= 0x7f800000u) best = max(best, lo);
      if (hi <= 0x7f800000u) best = max(best, hi);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0) atomicMax(amax_bits, best);
}

// One block per output channel: amax over the channel's Cin * taps weights, then the e4m3 slab row of every tap.
__global__ void fp8_pack_weights_kernel(const float* __restrict__ w, int Cin, int taps, uint8_t* __restrict__ wf,
                                        float* __restrict__ scale_w, int Cout) {
  const int co = blockIdx.x;
  const float* row = w + static_cast<long long>(co) * Cin * taps;
  const int n = Cin * taps;
  uint32_t best = 0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) best = max(best, __float_as_uint(row[i]) & 0x7fffffffu);
  __shared__ uint32_t red[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x < 32) {
    best = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (threadIdx.x == 0) red[0] = best;
  }
  __syncthreads();
  const float amax = red[0] == 0u ? 448.f : __uint_as_float(red[0]);
  const float qscale = 448.f / amax;
  if (threadIdx.x == 0) scale_w[co] = amax / 448.f;
  // slab element (t, co, ci) <- w[co][ci][t]; two channels per store
  for (int i = threadIdx.x; i < n / 2; i += blockDim.x) {
    const int t = i / (Cin / 2), ci = 2 * (i - t * (Cin / 2));
    const uint16_t q = pack_e4m3x2(row[ci * taps + t] * qscale, row[(ci + 1) * taps + t] * qscale);
    *reinterpret_cast<uint16_t*>(wf + (static_cast<long long>(t) * Cout + co) * Cin + ci) = q;
  }
}

static int elementwise_grid(long long work) {
  const long long blocks = (work + 255) / 256;
  const long long cap = 8LL * num_sms();
  return static_cast<int>(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

}  // namespace sb

extern "C" int semseg_fp8_quantize(const void* x, int x_pitch, void* y, int y_pitch, long long M, int C, float qscale,
                                   void* stream) {
  using namespace sb;
  SB_CHECK_ARG(x != nullptr && y != nullptr, "fp8_quantize: null x / y");
  SB_CHECK_ARG(M > 0 && C > 0 && C % 16 == 0, "fp8_quantize: need M > 0 and C %% 16 == 0 (C = %d)", C);
  SB_CHECK_ARG(x_pitch >= C && x_pitch % 16 == 0 && y_pitch >= C && y_pitch % 16 == 0,
               "fp8_quantize: pitches (%d, %d) must be >= C and multiples of 16", x_pitch, y_pitch);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0,
               "fp8_quantize: x / y must be 16-byte aligned");
  SB_CHECK_ARG(qscale > 0.f && qscale < 3.0e38f, "fp8_quantize: qscale must be finite and > 0");
  fp8_quantize_kernel<<<elementwise_grid(M * (C / 16)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), x_pitch, static_cast<uint8_t*>(y), y_pitch, M, C, qscale);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_fp8_amax(const void* x, int x_pitch, long long M, int C, unsigned int* amax_bits, void* stream) {
  using namespace sb;
  SB_CHECK_ARG(x != nullptr && amax_bits != nullptr, "fp8_amax: null x / amax_bits");
  SB_CHECK_ARG(M > 0 && C > 0 && C % 8 == 0 && x_pitch >= C && x_pitch % 8 == 0,
               "fp8_amax: need M > 0, C %% 8 == 0 and a pitch >= C, multiple of 8 (C = %d, pitch = %d)", C, x_pitch);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15) == 0, "fp8_amax: x must be 16-byte aligned");
  fp8_amax_kernel<<<elementwise_grid(M * (C / 8)), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(x), x_pitch, M, C, amax_bits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_fp8_pack_weights(const float* w, int Cout, int Cin, int taps, void* wf, float* scale_w,
                                       void* stream) {
  using namespace sb;
  SB_CHECK_ARG(w != nullptr && wf != nullptr && scale_w != nullptr, "fp8_pack_weights: null w / wf / scale_w");
  SB_CHECK_ARG(Cout > 0 && Cin > 0 && Cin % 16 == 0 && taps >= 1 && taps <= SEMSEG_MAX_TAPS,
               "fp8_pack_weights: need Cout > 0, Cin %% 16 == 0, 1 <= taps <= 9 (Cout %d Cin %d taps %d)", Cout, Cin,
               taps);
  fp8_pack_weights_kernel<<<Cout, 256, 0, static_cast<cudaStream_t>(stream)>>>(w, Cin, taps, static_cast<uint8_t*>(wf),
                                                                               scale_w, Cout);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

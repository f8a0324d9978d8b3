// MaxPool2d(kernel 3, stride 2, padding 1) on NHWC bf16 (model/resnet.py:115, used as layer0[9]).
// Forward: one thread per (output pixel, 8 channels); it also records the window position (0..8) of the arg-max
// (first maximum in row-major window order, the tie rule of ATen's max_pool2d_with_indices; NaN propagates and the last
// NaN of the window is recorded, as in ATen) as one byte per element.
// Backward is a deterministic gather: every input pixel checks the (up to four) windows that contain it and sums the
// dy of those whose recorded arg-max is this pixel. No atomics, every dx element written once.
#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

template <bool S>
__global__ void maxpool3x3s2_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo,
                                        __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ y_lo,
                                        unsigned char* __restrict__ argcode, int N, int H, int W, int C, int Ho,
                                        int Wo) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * Ho * Wo * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(idx % groups) << 3;
    long long p = idx / groups;
    const int wo = static_cast<int>(p % Wo);
    p /= Wo;
    const int ho = static_cast<int>(p % Ho);
    const int n = static_cast<int>(p / Ho);
    float m[8];
    unsigned code[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      m[q] = -INFINITY;
      code[q] = 255u;
    }
    for (int kh = 0; kh < 3; ++kh) {
      const int h = 2 * ho - 1 + kh;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int w = 2 * wo - 1 + kw;
        if (w < 0 || w >= W) continue;
        float f[8];
        act_ld8<S>(x, x_lo, ((static_cast<long long>(n) * H + h) * W + w) * C + c0, f);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          // ATen's rule: the first maximum in row-major window order, but the last NaN (a NaN always replaces the
          // running maximum; an all -inf window keeps its first in-bounds tap)
          if (f[q] > m[q] || isnan(f[q]) || code[q] == 255u) {
            m[q] = f[q];
            code[q] = static_cast<unsigned>(kh * 3 + kw);
          }
        }
      }
    }
    const long long o = ((static_cast<long long>(n) * Ho + ho) * Wo + wo) * C + c0;
    act_st8<S>(y, y_lo, o, m);
    if (argcode) {
      uint2 pk;
      pk.x = code[0] | (code[1] << 8) | (code[2] << 16) | (code[3] << 24);
      pk.y = code[4] | (code[5] << 8) | (code[6] << 16) | (code[7] << 24);
      *reinterpret_cast<uint2*>(argcode + o) = pk;
    }
  }
}

template <bool S>
__global__ void maxpool3x3s2_bwd_kernel(const unsigned char* __restrict__ argcode, const __nv_bfloat16* __restrict__ dy,
                                        const __nv_bfloat16* __restrict__ dy_lo, __nv_bfloat16* __restrict__ dx,
                                        __nv_bfloat16* __restrict__ dx_lo, int N, int H, int W, int C, int Ho, int Wo) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * H * W * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(idx % groups) << 3;
    long long p = idx / groups;
    const int w = static_cast<int>(p % W);
    p /= W;
    const int h = static_cast<int>(p % H);
    const int n = static_cast<int>(p / H);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // windows containing (h, w): ho with 2*ho-1 <= h <= 2*ho+1
    const int ho_lo = h / 2, ho_hi = min((h + 1) / 2, Ho - 1);
    const int wo_lo = w / 2, wo_hi = min((w + 1) / 2, Wo - 1);
    for (int ho = ho_lo; ho <= ho_hi; ++ho) {
      for (int wo = wo_lo; wo <= wo_hi; ++wo) {
        const unsigned me = static_cast<unsigned>((h - (2 * ho - 1)) * 3 + (w - (2 * wo - 1)));  // my code in this window
        const long long o = ((static_cast<long long>(n) * Ho + ho) * Wo + wo) * C + c0;
        const uint2 pk = *reinterpret_cast<const uint2*>(argcode + o);
        float g[8];
        act_ld8<S>(dy, dy_lo, o, g);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const unsigned cq = ((q < 4 ? pk.x : pk.y) >> ((q & 3) * 8)) & 0xffu;
          if (cq == me) acc[q] += g[q];
        }
      }
    }
    act_st8<S>(dx, dx_lo, ((static_cast<long long>(n) * H + h) * W + w) * C + c0, acc);
  }
}

static int mp_blocks(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace sb

using namespace sb;

extern "C" int semseg_maxpool3x3s2_fwd(const void* x, const void* x_lo, void* y, void* y_lo, void* argcode, int N,
                                       int H, int W, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && y && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "maxpool3x3s2_fwd: bad args");
  SB_CHECK_ARG((x_lo != nullptr) == (y_lo != nullptr), "maxpool3x3s2_fwd: input and output must use the same storage form");
  if (const int r = check_vec_acts("maxpool3x3s2_fwd", C, {{x, x_lo, C}, {y, y_lo, C}})) return r;
  if (const int r = check_vec_acts("maxpool3x3s2_fwd", C, {{argcode, nullptr, C}}, 8)) return r;  // uint2 stores
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const long long total = static_cast<long long>(N) * Ho * Wo * (C / 8);
  typedef __nv_bfloat16 bf16;
  SB_ACT_DISPATCH(x_lo != nullptr, maxpool3x3s2_fwd_kernel<kS><<<mp_blocks(total), 256, 0, stream>>>(
                                       static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo),
                                       static_cast<bf16*>(y), static_cast<bf16*>(y_lo),
                                       static_cast<unsigned char*>(argcode), N, H, W, C, Ho, Wo));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_maxpool3x3s2_bwd(const void* argcode, const void* dy, const void* dy_lo, void* dx, void* dx_lo,
                                       int N, int H, int W, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(argcode && dy && dx && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "maxpool3x3s2_bwd: bad args");
  SB_CHECK_ARG((dy_lo != nullptr) == (dx_lo != nullptr), "maxpool3x3s2_bwd: dy and dx must use the same storage form");
  if (const int r = check_vec_acts("maxpool3x3s2_bwd", C, {{dy, dy_lo, C}, {dx, dx_lo, C}})) return r;
  if (const int r = check_vec_acts("maxpool3x3s2_bwd", C, {{argcode, nullptr, C}}, 8)) return r;  // uint2 loads
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const long long total = static_cast<long long>(N) * H * W * (C / 8);
  typedef __nv_bfloat16 bf16;
  SB_ACT_DISPATCH(dy_lo != nullptr, maxpool3x3s2_bwd_kernel<kS><<<mp_blocks(total), 256, 0, stream>>>(
                                        static_cast<const unsigned char*>(argcode), static_cast<const bf16*>(dy),
                                        static_cast<const bf16*>(dy_lo), static_cast<bf16*>(dx),
                                        static_cast<bf16*>(dx_lo), N, H, W, C, Ho, Wo));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

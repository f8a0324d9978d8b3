// Bilinear resize (align_corners=True) of NHWC activations, forward and adjoint: F.interpolate(..., mode='bilinear',
// align_corners=True) at model/psanet.py:61,97 (59x59 <-> 30x30 around the attention block). Arithmetic follows ATen's
// upsample_bilinear2d (SURVEY.md Appendix C): scale = (in-1)/(out-1) in fp32, src = scale*dst, i0 = floor(src),
// i1 = min(i0+1, in-1), l1 = src - i0; out = l0h*(l0w*v00 + l1w*v01) + l1h*(l0w*v10 + l1w*v11).
// The backward is a deterministic GATHER (ATen's scatters with atomicAdd): every input pixel sums, in a fixed order, the
// output pixels whose 2x2 support contains it.
#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

__device__ __forceinline__ void rs_src(int o, float scale, int in, int& i0, int& i1, float& l1) {
  const float f = scale * static_cast<float>(o);
  i0 = min(static_cast<int>(f), in - 1);
  i1 = min(i0 + 1, in - 1);
  l1 = f - static_cast<float>(i0);
}

template <bool S>
__global__ void __launch_bounds__(256)
resize_bilinear_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo, int x_pitch, int N,
                           int Hi, int Wi, int C, int Ho, int Wo, __nv_bfloat16* __restrict__ y,
                           __nv_bfloat16* __restrict__ y_lo, int y_pitch) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * Ho * Wo * groups;
  const float sh = Ho > 1 ? static_cast<float>(Hi - 1) / static_cast<float>(Ho - 1) : 0.f;
  const float sw = Wo > 1 ? static_cast<float>(Wi - 1) / static_cast<float>(Wo - 1) : 0.f;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(idx % groups) << 3;
    long long p = idx / groups;
    const int ox = static_cast<int>(p % Wo);
    p /= Wo;
    const int oy = static_cast<int>(p % Ho);
    const int n = static_cast<int>(p / Ho);
    int i0, i1, j0, j1;
    float l1h, l1w;
    rs_src(oy, sh, Hi, i0, i1, l1h);
    rs_src(ox, sw, Wi, j0, j1, l1w);
    const float l0h = 1.f - l1h, l0w = 1.f - l1w;
    const long long base = static_cast<long long>(n) * Hi * Wi;
    float v00[8], v01[8], v10[8], v11[8], o[8];
    act_ld8<S>(x, x_lo, (base + static_cast<long long>(i0) * Wi + j0) * x_pitch + c0, v00);
    act_ld8<S>(x, x_lo, (base + static_cast<long long>(i0) * Wi + j1) * x_pitch + c0, v01);
    act_ld8<S>(x, x_lo, (base + static_cast<long long>(i1) * Wi + j0) * x_pitch + c0, v10);
    act_ld8<S>(x, x_lo, (base + static_cast<long long>(i1) * Wi + j1) * x_pitch + c0, v11);
#pragma unroll
    for (int q = 0; q < 8; ++q) o[q] = l0h * (l0w * v00[q] + l1w * v01[q]) + l1h * (l0w * v10[q] + l1w * v11[q]);
    act_st8<S>(y, y_lo, ((static_cast<long long>(n) * Ho + oy) * Wo + ox) * y_pitch + c0, o);
  }
}

// dx[n, iy, ix, :] = sum over output pixels (oy, ox) whose support contains (iy, ix) of weight * dy[n, oy, ox, :].
template <bool S>
__global__ void __launch_bounds__(256)
resize_bilinear_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dy_lo, int dy_pitch,
                           int N, int Hi, int Wi, int C, int Ho, int Wo, __nv_bfloat16* __restrict__ dx,
                           __nv_bfloat16* __restrict__ dx_lo, int dx_pitch) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * Hi * Wi * groups;
  const float sh = Ho > 1 ? static_cast<float>(Hi - 1) / static_cast<float>(Ho - 1) : 0.f;
  const float sw = Wo > 1 ? static_cast<float>(Wi - 1) / static_cast<float>(Wo - 1) : 0.f;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c0 = static_cast<int>(idx % groups) << 3;
    long long p = idx / groups;
    const int ix = static_cast<int>(p % Wi);
    p /= Wi;
    const int iy = static_cast<int>(p % Hi);
    const int n = static_cast<int>(p / Hi);
    // candidate output rows / columns: those with src in (iy-1, iy+1); a margin of one covers fp32 rounding of src
    int oy_lo = 0, oy_hi = Ho - 1, ox_lo = 0, ox_hi = Wo - 1;
    if (sh > 0.f) {
      oy_lo = max(0, static_cast<int>(ceilf(static_cast<float>(iy - 1) / sh)) - 1);
      oy_hi = min(Ho - 1, static_cast<int>(floorf(static_cast<float>(iy + 1) / sh)) + 1);
    }
    if (sw > 0.f) {
      ox_lo = max(0, static_cast<int>(ceilf(static_cast<float>(ix - 1) / sw)) - 1);
      ox_hi = min(Wo - 1, static_cast<int>(floorf(static_cast<float>(ix + 1) / sw)) + 1);
    }
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      int i0, i1;
      float l1h;
      rs_src(oy, sh, Hi, i0, i1, l1h);
      const float wy = (i0 == iy ? 1.f - l1h : 0.f) + (i1 == iy ? l1h : 0.f);
      if (wy == 0.f) continue;
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        int j0, j1;
        float l1w;
        rs_src(ox, sw, Wi, j0, j1, l1w);
        const float wgt = wy * ((j0 == ix ? 1.f - l1w : 0.f) + (j1 == ix ? l1w : 0.f));
        if (wgt == 0.f) continue;
        float g[8];
        act_ld8<S>(dy, dy_lo, ((static_cast<long long>(n) * Ho + oy) * Wo + ox) * dy_pitch + c0, g);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = fmaf(wgt, g[q], acc[q]);
      }
    }
    act_st8<S>(dx, dx_lo, ((static_cast<long long>(n) * Hi + iy) * Wi + ix) * dx_pitch + c0, acc);
  }
}

static int rs_blocks(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace sb

using namespace sb;
typedef __nv_bfloat16 bf16;

extern "C" int semseg_resize_bilinear_fwd(const void* x, const void* x_lo, int x_pitch, int N, int Hi, int Wi, int C,
                                          int Ho, int Wo, void* y, void* y_lo, int y_pitch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && y && N > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0 && x_pitch % 8 == 0 &&
                   y_pitch % 8 == 0,
               "resize_bilinear_fwd: bad args");
  SB_CHECK_ARG((x_lo != nullptr) == (y_lo != nullptr), "resize_bilinear_fwd: x and y must use the same storage form");
  if (const int r = check_vec_acts("resize_bilinear_fwd", C, {{x, x_lo, x_pitch}, {y, y_lo, y_pitch}})) return r;
  const long long total = static_cast<long long>(N) * Ho * Wo * (C / 8);
  SB_ACT_DISPATCH(x_lo != nullptr, resize_bilinear_fwd_kernel<kS><<<rs_blocks(total), 256, 0, stream>>>(
                                       static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, N, Hi, Wi, C,
                                       Ho, Wo, static_cast<bf16*>(y), static_cast<bf16*>(y_lo), y_pitch));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_resize_bilinear_bwd(const void* dy, const void* dy_lo, int dy_pitch, int N, int Hi, int Wi, int C,
                                          int Ho, int Wo, void* dx, void* dx_lo, int dx_pitch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dy && dx && N > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0 && dy_pitch % 8 == 0 &&
                   dx_pitch % 8 == 0,
               "resize_bilinear_bwd: bad args");
  SB_CHECK_ARG((dy_lo != nullptr) == (dx_lo != nullptr), "resize_bilinear_bwd: dy and dx must use the same storage form");
  if (const int r = check_vec_acts("resize_bilinear_bwd", C, {{dy, dy_lo, dy_pitch}, {dx, dx_lo, dx_pitch}})) return r;
  const long long total = static_cast<long long>(N) * Hi * Wi * (C / 8);
  SB_ACT_DISPATCH(dy_lo != nullptr, resize_bilinear_bwd_kernel<kS><<<rs_blocks(total), 256, 0, stream>>>(
                                        static_cast<const bf16*>(dy), static_cast<const bf16*>(dy_lo), dy_pitch, N, Hi, Wi,
                                        C, Ho, Wo, static_cast<bf16*>(dx), static_cast<bf16*>(dx_lo), dx_pitch));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

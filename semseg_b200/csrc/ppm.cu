// Pyramid pooling module data movement (model/pspnet.py:8-26) on NHWC bf16:
//   ppm_pool            : AdaptiveAvgPool2d(b) for all bins in one launch (window [floor(i*H/b), ceil((i+1)*H/b)))
//   ppm_upsample_concat : bilinear (align_corners=True) upsample of the per-bin features to H x W, written straight
//                         into the channel slices of the 4096-channel concat buffer, plus the copy of x into slice 0
//   and the adjoints of both. All accumulation in fp32, deterministic (fixed reduction order, no atomics).
// These are pure HBM-bandwidth kernels: x is read once per bin for pooling and the concat buffer is written once.
#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

constexpr int kMaxBins = 8;

struct BinSet {
  int nb;
  int b[kMaxBins];
  int cell_off[kMaxBins + 1];  // prefix sum of b*b
  void* ptr[kMaxBins];         // per-bin tensor [N][b][b][C*]
  void* ptr_lo[kMaxBins];      // its lo plane (split storage) or NULL
};

// block = 8 channel groups (64 channels) x 32 pixel lanes. grid = (total cells * N, C/64).
template <bool S>
__global__ void __launch_bounds__(256)
ppm_pool_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo, int pitch, int N, int H,
                int W, int C, BinSet bs) {
  __shared__ float red[32][65];
  const int gl = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + gl * 8;
  const int total_cells = bs.cell_off[bs.nb];
  const int n = blockIdx.x / total_cells;
  int cell = blockIdx.x - n * total_cells;
  int k = 0;
  while (cell >= bs.cell_off[k + 1]) ++k;
  cell -= bs.cell_off[k];
  const int b = bs.b[k];
  const int ci = cell / b, cj = cell - ci * b;
  const int hs = (ci * H) / b, he = ((ci + 1) * H + b - 1) / b;
  const int ws = (cj * W) / b, we = ((cj + 1) * W + b - 1) / b;
  const int ww = we - ws, npix = (he - hs) * ww;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c0 < C) {
    for (int p = pl; p < npix; p += 32) {
      const int hh = hs + p / ww, wx = ws + p % ww;
      float f[8];
      act_ld8<S>(x, x_lo, (static_cast<long long>(n) * H * W + static_cast<long long>(hh) * W + wx) * pitch + c0, f);
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[q] += f[q];
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) red[pl][gl * 8 + q] = acc[q];
  __syncthreads();
  if (pl == 0 && c0 < C) {
    const float inv = 1.f / static_cast<float>(npix);
    float o[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float t = 0.f;
      for (int i = 0; i < 32; ++i) t += red[i][gl * 8 + q];
      o[q] = t * inv;
    }
    act_st8<S>(static_cast<__nv_bfloat16*>(bs.ptr[k]), static_cast<__nv_bfloat16*>(bs.ptr_lo[k]),
               (static_cast<long long>(n) * b * b + cell) * C + c0, o);
  }
}

// Windows of one bin along one dimension of extent L that contain coordinate x: window i spans [floor(i*L/b),
// ceil((i+1)*L/b)), both ends non-decreasing in i, so they are the contiguous range [lo, hi]. lo = floor(x*b/L) always
// contains x (x < (lo+1)*L/b), and so does every later window that starts at or before x. While b <= L a coordinate lies
// in at most 2 windows; when the bin is larger than the map, in about b/L + 1.
__device__ __forceinline__ void ppm_window_range(int x, int L, int b, int& lo, int& hi) {
  lo = (x * b) / L;
  hi = lo;
  while (hi + 1 < b && ((hi + 1) * L) / b <= x) ++hi;
}

__device__ __forceinline__ int ppm_window_size(int i, int L, int b) {
  return ((i + 1) * L + b - 1) / b - (i * L) / b;
}

// dx[n,h,w,c] = add[n,h,w,c] + sum over bins, over cells whose window contains (h,w): dpooled[n,cell,c] / window_size,
// in the fixed order add, bins ascending, ci ascending, cj ascending, one fmaf each with the window's fl(1/size).
// One warp per pixel: the pixel's windows are the ranges [ci_lo, ci_hi] x [cj_lo, cj_hi] of every bin, derived once;
// then the lanes sweep the channels. Up to kMaxCells windows (every pixel while no bin is larger than the map) are listed
// as (cell, 1/size) first, so the channel loop streams through the list and its loads overlap; a pixel with more windows
// walks the ranges in the channel loop instead, in the same order, so both forms give the same bits.
template <bool S>
__global__ void __launch_bounds__(256)
ppm_pool_bwd_kernel(__nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dx_lo, int pitch,
                    const __nv_bfloat16* __restrict__ add, const __nv_bfloat16* __restrict__ add_lo, int add_pitch, int N,
                    int H, int W, int C, BinSet bs) {
  const int lane = threadIdx.x & 31;
  const long long npix = static_cast<long long>(N) * H * W;
  const int groups = C >> 3;
  constexpr int kMaxCells = 4 * kMaxBins;
  for (long long p = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); p < npix;
       p += static_cast<long long>(gridDim.x) * (blockDim.x >> 5)) {
    const int wx = static_cast<int>(p % W);
    const int hh = static_cast<int>((p / W) % H);
    const int n = static_cast<int>(p / (static_cast<long long>(W) * H));
    int4 rng[kMaxBins];  // (ci_lo, ci_hi, cj_lo, cj_hi) per bin
    int total = 0;
    for (int k = 0; k < bs.nb; ++k) {
      ppm_window_range(hh, H, bs.b[k], rng[k].x, rng[k].y);
      ppm_window_range(wx, W, bs.b[k], rng[k].z, rng[k].w);
      total += (rng[k].y - rng[k].x + 1) * (rng[k].w - rng[k].z + 1);
    }
    if (total <= kMaxCells) {
      const __nv_bfloat16* src[kMaxCells];
      const __nv_bfloat16* src_lo[kMaxCells];
      float inv[kMaxCells];
      int cnt = 0;
      for (int k = 0; k < bs.nb; ++k) {
        const int b = bs.b[k];
        const size_t base = static_cast<size_t>(n) * b * b * C;
        for (int ci = rng[k].x; ci <= rng[k].y; ++ci) {
          for (int cj = rng[k].z; cj <= rng[k].w; ++cj) {
            const size_t off = base + static_cast<size_t>(ci * b + cj) * C;
            src[cnt] = static_cast<const __nv_bfloat16*>(bs.ptr[k]) + off;
            src_lo[cnt] = S ? static_cast<const __nv_bfloat16*>(bs.ptr_lo[k]) + off : nullptr;
            inv[cnt] = 1.f / static_cast<float>(ppm_window_size(ci, H, b) * ppm_window_size(cj, W, b));
            ++cnt;
          }
        }
      }
      for (int g = lane; g < groups; g += 32) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (add) act_ld8<S>(add, add_lo, p * add_pitch + g * 8, acc);  // the other gradient branch of x (identity part of the concat)
        for (int i = 0; i < cnt; ++i) {
          float f[8];
          act_ld8<S>(src[i], src_lo[i], g * 8, f);
#pragma unroll
          for (int q = 0; q < 8; ++q) acc[q] = fmaf(f[q], inv[i], acc[q]);
        }
        act_st8<S>(dx, dx_lo, p * pitch + g * 8, acc);
      }
      continue;
    }
    for (int g = lane; g < groups; g += 32) {
      float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (add) act_ld8<S>(add, add_lo, p * add_pitch + g * 8, acc);
      for (int k = 0; k < bs.nb; ++k) {
        const int b = bs.b[k];
        const size_t base = static_cast<size_t>(n) * b * b * C + g * 8;
        for (int ci = rng[k].x; ci <= rng[k].y; ++ci) {
          for (int cj = rng[k].z; cj <= rng[k].w; ++cj) {
            const float inv = 1.f / static_cast<float>(ppm_window_size(ci, H, b) * ppm_window_size(cj, W, b));
            float f[8];
            act_ld8<S>(static_cast<const __nv_bfloat16*>(bs.ptr[k]), static_cast<const __nv_bfloat16*>(bs.ptr_lo[k]),
                       base + static_cast<size_t>(ci * b + cj) * C, f);
#pragma unroll
            for (int q = 0; q < 8; ++q) acc[q] = fmaf(f[q], inv, acc[q]);
          }
        }
      }
      act_st8<S>(dx, dx_lo, p * pitch + g * 8, acc);
    }
  }
}

// out[n,h,w, 0:C] = x ; out[n,h,w, C + k*Cr + c] = bilinear(feat_k)[n,h,w,c]
template <bool S>
__global__ void __launch_bounds__(256)
ppm_upsample_concat_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo, int x_pitch, int N,
                           int H, int W, int C, int Cr, BinSet bs, __nv_bfloat16* __restrict__ out,
                           __nv_bfloat16* __restrict__ out_lo, int out_pitch) {
  const int gx = C >> 3, gf = Cr >> 3;
  const int groups = gx + bs.nb * gf;
  const long long total = static_cast<long long>(N) * H * W * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int g = static_cast<int>(idx - p * groups);
    if (g < gx) {
      *reinterpret_cast<uint4*>(out + p * out_pitch + g * 8) =
          *reinterpret_cast<const uint4*>(x + p * x_pitch + g * 8);
      if constexpr (S)
        *reinterpret_cast<uint4*>(out_lo + p * out_pitch + g * 8) =
            *reinterpret_cast<const uint4*>(x_lo + p * x_pitch + g * 8);
      continue;
    }
    const int k = (g - gx) / gf;
    const int c0 = ((g - gx) - k * gf) << 3;
    const int b = bs.b[k];
    const int wx = static_cast<int>(p % W);
    const int hh = static_cast<int>((p / W) % H);
    const int n = static_cast<int>(p / (static_cast<long long>(W) * H));
    // ATen upsample_bilinear2d, align_corners=True: scale = (in-1)/(out-1) (0 when out == 1)
    const float sh = H > 1 ? static_cast<float>(b - 1) / static_cast<float>(H - 1) : 0.f;
    const float sw = W > 1 ? static_cast<float>(b - 1) / static_cast<float>(W - 1) : 0.f;
    const float fy = sh * hh, fx = sw * wx;
    const int i0 = static_cast<int>(fy), j0 = static_cast<int>(fx);
    const int i1 = min(i0 + 1, b - 1), j1 = min(j0 + 1, b - 1);
    const float l1h = fy - i0, l0h = 1.f - l1h, l1w = fx - j0, l0w = 1.f - l1w;
    const __nv_bfloat16* f = static_cast<const __nv_bfloat16*>(bs.ptr[k]);
    const __nv_bfloat16* f_lo = static_cast<const __nv_bfloat16*>(bs.ptr_lo[k]);
    const long long fb = static_cast<long long>(n) * b * b * Cr + c0;
    float v00[8], v01[8], v10[8], v11[8], o[8];
    act_ld8<S>(f, f_lo, fb + (i0 * b + j0) * Cr, v00);
    act_ld8<S>(f, f_lo, fb + (i0 * b + j1) * Cr, v01);
    act_ld8<S>(f, f_lo, fb + (i1 * b + j0) * Cr, v10);
    act_ld8<S>(f, f_lo, fb + (i1 * b + j1) * Cr, v11);
#pragma unroll
    for (int q = 0; q < 8; ++q) o[q] = l0h * (l0w * v00[q] + l1w * v01[q]) + l1h * (l0w * v10[q] + l1w * v11[q]);
    act_st8<S>(out, out_lo, p * out_pitch + C + k * Cr + c0, o);
  }
}

// dfeat_k[n, ci, cj, c] = sum_p w(p; ci, cj) * dout[n, p, c_off + k*Cr + c]
// block = 8 channel groups x 32 pixel lanes; grid = (N * total cells, Cr / 64).
template <bool S>
__global__ void __launch_bounds__(256)
ppm_upsample_bwd_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ dout_lo, int pitch,
                        int c_off, int N, int H, int W, int Cr, BinSet bs) {
  __shared__ float red[32][65];
  const int gl = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int c0 = blockIdx.y * 64 + gl * 8;
  const int total_cells = bs.cell_off[bs.nb];
  const int n = blockIdx.x / total_cells;
  int cell = blockIdx.x - n * total_cells;
  int k = 0;
  while (cell >= bs.cell_off[k + 1]) ++k;
  cell -= bs.cell_off[k];
  const int b = bs.b[k];
  const int ci = cell / b, cj = cell - ci * b;
  const float sh = H > 1 ? static_cast<float>(b - 1) / static_cast<float>(H - 1) : 0.f;
  const float sw = W > 1 ? static_cast<float>(b - 1) / static_cast<float>(W - 1) : 0.f;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c0 < Cr) {
    const long long src = static_cast<long long>(n) * H * W * pitch + c_off + k * Cr + c0;
    for (int hh = 0; hh < H; ++hh) {
      const float fy = sh * hh;
      const int i0 = static_cast<int>(fy);
      const int i1 = min(i0 + 1, b - 1);
      const float l1h = fy - i0;
      const float wy = (i0 == ci ? 1.f - l1h : 0.f) + (i1 == ci ? l1h : 0.f);
      if (wy == 0.f) continue;
      for (int wx = pl; wx < W; wx += 32) {
        const float fx = sw * wx;
        const int j0 = static_cast<int>(fx);
        const int j1 = min(j0 + 1, b - 1);
        const float l1w = fx - j0;
        const float wgt = wy * ((j0 == cj ? 1.f - l1w : 0.f) + (j1 == cj ? l1w : 0.f));
        if (wgt == 0.f) continue;
        float f[8];
        act_ld8<S>(dout, dout_lo, src + (static_cast<long long>(hh) * W + wx) * pitch, f);
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = fmaf(wgt, f[q], acc[q]);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) red[pl][gl * 8 + q] = acc[q];
  __syncthreads();
  if (pl == 0 && c0 < Cr) {
    float o[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float t = 0.f;
      for (int i = 0; i < 32; ++i) t += red[i][gl * 8 + q];
      o[q] = t;
    }
    act_st8<S>(static_cast<__nv_bfloat16*>(bs.ptr[k]), static_cast<__nv_bfloat16*>(bs.ptr_lo[k]),
               (static_cast<long long>(n) * b * b + cell) * Cr + c0, o);
  }
}

static int make_binset(const int* bins, void* const* ptrs, void* const* ptrs_lo, int nb, BinSet* bs) {
  SB_CHECK_ARG(bins && ptrs && nb >= 1 && nb <= kMaxBins, "ppm: 1..%d bins", kMaxBins);
  bs->nb = nb;
  bs->cell_off[0] = 0;
  for (int i = 0; i < nb; ++i) {
    SB_CHECK_ARG(bins[i] >= 1 && ptrs[i], "ppm: bad bin %d", i);
    SB_CHECK_ARG(!ptrs_lo || ptrs_lo[i], "ppm: missing lo plane of bin %d", i);
    bs->b[i] = bins[i];
    bs->ptr[i] = ptrs[i];
    bs->ptr_lo[i] = ptrs_lo ? ptrs_lo[i] : nullptr;
    bs->cell_off[i + 1] = bs->cell_off[i] + bins[i] * bins[i];
  }
  return SEMSEG_OK;
}

// The per-bin tensors are dense [N][b][b][C] and accessed in 8-channel vectors: their bases must be 16-byte aligned.
static int check_bins(const char* fn, const BinSet& bs) {
  for (int k = 0; k < bs.nb; ++k)
    if (const int r = check_vec_acts(fn, 0, {{bs.ptr[k], bs.ptr_lo[k], 0}})) return r;
  return SEMSEG_OK;
}

static int ew_blocks(long long total) {
  long long b = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(b > cap ? cap : (b < 1 ? 1 : b));
}

}  // namespace sb

using namespace sb;
typedef __nv_bfloat16 bf16;

extern "C" int semseg_ppm_pool(const void* x, const void* x_lo, int x_pitch, int N, int H, int W, int C,
                               const int* bins, void* const* pooled, void* const* pooled_lo, int nb, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && x_pitch % 8 == 0, "ppm_pool: bad args");
  SB_CHECK_ARG((x_lo != nullptr) == (pooled_lo != nullptr), "ppm_pool: input and outputs must use the same storage form");
  BinSet bs;
  int r = make_binset(bins, pooled, pooled_lo, nb, &bs);
  if (r) return r;
  if ((r = check_vec_acts("ppm_pool", C, {{x, x_lo, x_pitch}}))) return r;
  if ((r = check_bins("ppm_pool", bs))) return r;
  dim3 grid(N * bs.cell_off[nb], cdiv(C, 64));
  SB_ACT_DISPATCH(x_lo != nullptr, ppm_pool_kernel<kS><<<grid, 256, 0, stream>>>(
                                       static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, N, H, W, C,
                                       bs));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_ppm_pool_bwd(void* const* dpooled, void* const* dpooled_lo, const int* bins, int nb, int N, int H,
                                   int W, int C, void* dx, void* dx_lo, int dx_pitch, const void* add,
                                   const void* add_lo, int add_pitch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dx && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && dx_pitch % 8 == 0, "ppm_pool_bwd: bad args");
  SB_CHECK_ARG(!add || (add_pitch % 8 == 0 && add_pitch >= C), "ppm_pool_bwd: bad add pitch %d", add_pitch);
  const bool split = dx_lo != nullptr;
  SB_CHECK_ARG((dpooled_lo != nullptr) == split && (!add || (add_lo != nullptr) == split),
               "ppm_pool_bwd: all tensors must use the same storage form");
  BinSet bs;
  int r = make_binset(bins, dpooled, dpooled_lo, nb, &bs);
  if (r) return r;
  if ((r = check_vec_acts("ppm_pool_bwd", C, {{dx, dx_lo, dx_pitch}, {add, add_lo, add_pitch}}))) return r;
  if ((r = check_bins("ppm_pool_bwd", bs))) return r;
  const long long warps = static_cast<long long>(N) * H * W;
  SB_ACT_DISPATCH(split, ppm_pool_bwd_kernel<kS><<<ew_blocks(warps * 32), 256, 0, stream>>>(
                             static_cast<bf16*>(dx), static_cast<bf16*>(dx_lo), dx_pitch, static_cast<const bf16*>(add),
                             static_cast<const bf16*>(add_lo), add_pitch, N, H, W, C, bs));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_ppm_upsample_concat(const void* x, const void* x_lo, int x_pitch, void* const* feats,
                                          void* const* feats_lo, const int* bins, int nb, int N, int H, int W, int C,
                                          int Cr, void* out, void* out_lo, int out_pitch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && out && N > 0 && H > 0 && W > 0 && C % 8 == 0 && Cr % 8 == 0 && x_pitch % 8 == 0 &&
                   out_pitch % 8 == 0 && out_pitch >= C + nb * Cr,
               "ppm_upsample_concat: bad args");
  const bool split = x_lo != nullptr;
  SB_CHECK_ARG((feats_lo != nullptr) == split && (out_lo != nullptr) == split,
               "ppm_upsample_concat: all tensors must use the same storage form");
  BinSet bs;
  int r = make_binset(bins, feats, feats_lo, nb, &bs);
  if (r) return r;
  if ((r = check_vec_acts("ppm_upsample_concat", C, {{x, x_lo, x_pitch}, {out, out_lo, out_pitch}}))) return r;
  if ((r = check_bins("ppm_upsample_concat", bs))) return r;
  const long long total = static_cast<long long>(N) * H * W * (C / 8 + nb * (Cr / 8));
  SB_ACT_DISPATCH(split, ppm_upsample_concat_kernel<kS><<<ew_blocks(total), 256, 0, stream>>>(
                             static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, N, H, W, C, Cr, bs,
                             static_cast<bf16*>(out), static_cast<bf16*>(out_lo), out_pitch));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_ppm_upsample_bwd(const void* dout, const void* dout_lo, int dout_pitch, int c_off,
                                       void* const* dfeats, void* const* dfeats_lo, const int* bins, int nb, int N,
                                       int H, int W, int Cr, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dout && N > 0 && H > 0 && W > 0 && Cr % 8 == 0 && dout_pitch % 8 == 0 && c_off % 8 == 0 && c_off >= 0,
               "ppm_upsample_bwd: bad args");
  SB_CHECK_ARG((dout_lo != nullptr) == (dfeats_lo != nullptr),
               "ppm_upsample_bwd: all tensors must use the same storage form");
  BinSet bs;
  int r = make_binset(bins, dfeats, dfeats_lo, nb, &bs);
  if (r) return r;
  SB_CHECK_ARG(static_cast<long long>(c_off) + static_cast<long long>(nb) * Cr <= dout_pitch,
               "ppm_upsample_bwd: channels c_off + nb*Cr = %d + %d*%d exceed the pitch %d", c_off, nb, Cr, dout_pitch);
  if ((r = check_vec_acts("ppm_upsample_bwd", 0, {{dout, dout_lo, dout_pitch}}))) return r;
  if ((r = check_bins("ppm_upsample_bwd", bs))) return r;
  dim3 grid(N * bs.cell_off[nb], cdiv(Cr, 64));
  SB_ACT_DISPATCH(dout_lo != nullptr, ppm_upsample_bwd_kernel<kS><<<grid, 256, 0, stream>>>(
                                          static_cast<const bf16*>(dout), static_cast<const bf16*>(dout_lo), dout_pitch,
                                          c_off, N, H, W, Cr, bs));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

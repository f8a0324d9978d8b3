// Layout conversion at the module boundary and weight packing.
//   - NCHW fp32 <-> NHWC bf16 / fp32 (model/pspnet.py:80-105 takes and returns NCHW fp32)
//   - fp32 OIHW master weights -> bf16 [tap][row][col] operand slabs for the implicit-GEMM kernels
#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

// 32x32 tiled transpose between [C][HW] (NCHW plane) and [HW][pitch] (NHWC) per image.
template <typename TIn, typename TOut>
__global__ void nchw_to_nhwc_kernel(const TIn* __restrict__ in, TOut* __restrict__ out, TOut* __restrict__ out_lo, int C,
                                    int HW, int out_pitch) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const TIn* src = in + static_cast<size_t>(n) * C * HW;
  TOut* dst = out + static_cast<size_t>(n) * HW * out_pitch;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = c0 + r, p = p0 + threadIdx.x;
    tile[r][threadIdx.x] = (c < C && p < HW) ? static_cast<float>(src[static_cast<size_t>(c) * HW + p]) : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int p = p0 + r, c = c0 + threadIdx.x;
    if (p < HW && c < C) {
      const float v = tile[threadIdx.x][r];
      const TOut hi = static_cast<TOut>(v);
      dst[static_cast<size_t>(p) * out_pitch + c] = hi;
      if (out_lo)   // split storage: lo = v - hi
        out_lo[static_cast<size_t>(n) * HW * out_pitch + static_cast<size_t>(p) * out_pitch + c] =
            static_cast<TOut>(v - static_cast<float>(hi));
    }
  }
}

template <typename TIn, typename TOut>
__global__ void nhwc_to_nchw_kernel(const TIn* __restrict__ in, const TIn* __restrict__ in_lo, TOut* __restrict__ out,
                                    int C, int HW, int in_pitch) {
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const TIn* src = in + static_cast<size_t>(n) * HW * in_pitch;
  TOut* dst = out + static_cast<size_t>(n) * C * HW;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int p = p0 + r, c = c0 + threadIdx.x;
    float v = 0.f;
    if (p < HW && c < C) {
      v = static_cast<float>(src[static_cast<size_t>(p) * in_pitch + c]);
      if (in_lo) v += static_cast<float>(in_lo[static_cast<size_t>(n) * HW * in_pitch + static_cast<size_t>(p) * in_pitch + c]);
    }
    tile[r][threadIdx.x] = v;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = c0 + r, p = p0 + threadIdx.x;
    if (c < C && p < HW) dst[static_cast<size_t>(c) * HW + p] = static_cast<TOut>(tile[threadIdx.x][r]);
  }
}

// dst[o] = bf16(v) (round to nearest); split != 0: dst[lo + o] = bf16(v - hi), the lo slab behind the hi slab.
__device__ __forceinline__ void store_hi_lo(__nv_bfloat16* dst, size_t o, size_t lo, float v, int split) {
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  dst[o] = hi;
  if (split) dst[lo + o] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// Every operand slab of every conv of a model in ONE launch (per-layer packing would be 2 x 63 launch-latency-bound
// launches per step for PSPNet50). A block owns one 32 (co) x 32 (ci) tile of one layer with all of its taps: the fp32
// OIHW rows are read once (32*taps contiguous floats per output channel), parked in shared memory, and written out as
// the bf16 operand slabs the item asks for, zero padded to the slab widths: wf[t][co][ci], wd[t][ci][co] and the stem's
// patch slab wp[co][t*Cin + ci] (Cin <= 3, so the one ci0 == 0 tile of a row holds all 9*Cin values). items[] lives in
// device memory and is sorted by tile0; the block finds its layer by binary search.
__global__ void __launch_bounds__(256) pack_multi_kernel(const semseg_pack_item* __restrict__ items, int n_items) {
  extern __shared__ float pk_tile[];  // [32][32 * taps + 1]
  __shared__ int s_item;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n_items - 1;
    const int b = static_cast<int>(blockIdx.x);
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (items[mid].tile0 <= b) lo = mid; else hi = mid - 1;
    }
    s_item = lo;
  }
  __syncthreads();
  const semseg_pack_item it = items[s_item];
  const int lt = static_cast<int>(blockIdx.x) - it.tile0;
  const int co0 = (lt / it.tiles_ci) * 32, ci0 = (lt % it.tiles_ci) * 32;
  const int taps = it.taps, rowlen = 32 * taps, pitch = rowlen + 1;
  const int nci = max(0, min(32, it.Cin - ci0)), nco = max(0, min(32, it.Cout - co0));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < 32; r += 8) {
    const float* src = it.w + (static_cast<size_t>(co0 + r) * it.Cin + ci0) * taps;
    for (int e = lane; e < rowlen; e += 32) pk_tile[r * pitch + e] = (r < nco && e < nci * taps) ? src[e] : 0.f;
  }
  __syncthreads();
  const int total = taps * 1024;
  if (it.wf) {
    __nv_bfloat16* wf = static_cast<__nv_bfloat16*>(it.wf);
    const size_t lo = static_cast<size_t>(taps) * it.Cout * it.cols_f;
    for (int idx = threadIdx.x; idx < total; idx += 256) {
      const int ci_l = idx & 31, co_l = (idx >> 5) & 31, t = idx >> 10;
      if (co_l < nco && ci0 + ci_l < it.cols_f)
        store_hi_lo(wf, (static_cast<size_t>(t) * it.Cout + co0 + co_l) * it.cols_f + ci0 + ci_l, lo,
                    pk_tile[co_l * pitch + ci_l * taps + t], it.split);
    }
  }
  if (it.wd) {
    __nv_bfloat16* wd = static_cast<__nv_bfloat16*>(it.wd);
    const size_t lo = static_cast<size_t>(taps) * it.Cin * it.cols_d;
    for (int idx = threadIdx.x; idx < total; idx += 256) {
      const int co_l = idx & 31, ci_l = (idx >> 5) & 31, t = idx >> 10;
      if (ci_l < nci && co0 + co_l < it.cols_d)
        store_hi_lo(wd, (static_cast<size_t>(t) * it.Cin + ci0 + ci_l) * it.cols_d + co0 + co_l, lo,
                    pk_tile[co_l * pitch + ci_l * taps + t], it.split);
    }
  }
  if (it.wp && ci0 == 0) {
    __nv_bfloat16* wp = static_cast<__nv_bfloat16*>(it.wp);
    const int real = taps * it.Cin;   // columns real..31 are zero
    for (int idx = threadIdx.x; idx < 1024; idx += 256) {
      const int col = idx & 31, co_l = idx >> 5;
      if (co_l < nco)
        store_hi_lo(wp, static_cast<size_t>(co0 + co_l) * 32 + col, static_cast<size_t>(it.Cout) * 32,
                    col < real ? pk_tile[co_l * pitch + (col % it.Cin) * taps + col / it.Cin] : 0.f, it.split);
    }
  }
}

// Stem conv (3x3, stride 2, pad 1, <= 3 input channels; model/resnet.py:106-108): patches of the input, so the conv
// becomes ONE 64-wide K block (27 real values) per output pixel instead of 9 taps x 64-wide K blocks that are 7/8 zero
// fill fetched in 16-byte pieces:  P[n, ho, wo, (r*3+s)*3 + c] = x[n, 2ho-1+r, 2wo-1+s, c]  (zero outside, 27..31 zero).
__global__ void __launch_bounds__(256) im2col3x3s2_kernel(const __nv_bfloat16* __restrict__ x, int pitch, int N, int H,
                                                          int W, int Cin, int Ho, int Wo, __nv_bfloat16* __restrict__ out) {
  const long long total = static_cast<long long>(N) * Ho * Wo;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int wo = static_cast<int>(idx % Wo);
    const int ho = static_cast<int>((idx / Wo) % Ho);
    const int n = static_cast<int>(idx / (static_cast<long long>(Wo) * Ho));
    __align__(16) __nv_bfloat16 v[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) v[i] = __float2bfloat16_rn(0.f);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = 2 * ho - 1 + r;
#pragma unroll
      for (int sx = 0; sx < 3; ++sx) {
        const int wi = 2 * wo - 1 + sx;
        if (hi >= 0 && hi < H && wi >= 0 && wi < W) {
          const uint2 px = *reinterpret_cast<const uint2*>(x + ((static_cast<size_t>(n) * H + hi) * W + wi) * pitch);
          const __nv_bfloat16* pc = reinterpret_cast<const __nv_bfloat16*>(&px);   // 4 channels, Cin <= 3 are real
#pragma unroll
          for (int c = 0; c < 3; ++c)
            if (c < Cin) v[(r * 3 + sx) * Cin + c] = pc[c];
        }
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(out + idx * 32);
    const uint4* src = reinterpret_cast<const uint4*>(v);
#pragma unroll
    for (int q = 0; q < 4; ++q) dst[q] = src[q];
  }
}

// Input gradient of the stem conv (the adjoint of im2col3x3s2 + the patch-slab product), written as fp32 NCHW:
//   dx[n, c, y, x] = sum over (r, s, ho, wo) with 2ho-1+r = y, 2wo-1+s = x of  sum_k dy[n, ho, wo, k] * w[k, c, r, s]
// A thread owns the 2x2 input pixels (2i..2i+1, 2j..2j+1), which only the four conv-output pixels (i..i+1, j..j+1)
// reach, each through its own taps:
//   dy(i, j)    : (2i, 2j) tap 4, (2i, 2j+1) tap 5, (2i+1, 2j) tap 7, (2i+1, 2j+1) tap 8
//   dy(i, j+1)  : (2i, 2j+1) tap 3, (2i+1, 2j+1) tap 6
//   dy(i+1, j)  : (2i+1, 2j) tap 1, (2i+1, 2j+1) tap 2
//   dy(i+1, j+1): (2i+1, 2j+1) tap 0
// so all 9 taps are used once per k. The weights w[k][tap][c] (fp32 copies of the bf16 slab values, lo slab behind) sit
// in shared memory as one float4 per (k, tap) and are read warp-uniformly (broadcast). bf16x3 sums the conv kernels'
// three products hi*hi + lo*hi + hi*lo. Each output is one fp32 chain in a fixed order (k ascending, then the dy pixel,
// then the product): deterministic, no atomics.
constexpr int kStemCout = 64;

template <int CIN, bool SPLIT>
__global__ void __launch_bounds__(256) stem_dgrad3x3s2_kernel(const __nv_bfloat16* __restrict__ dy,
                                                              const __nv_bfloat16* __restrict__ dy_lo, int pitch, int N,
                                                              int H, int W, int Ho, int Wo,
                                                              const __nv_bfloat16* __restrict__ wp,
                                                              float* __restrict__ dx) {
  __shared__ float4 ws[SPLIT ? 2 : 1][kStemCout * 9];
  for (int e = threadIdx.x; e < kStemCout * 9; e += blockDim.x) {
    const int k = e / 9, t = e % 9;
#pragma unroll
    for (int part = 0; part < (SPLIT ? 2 : 1); ++part) {
      const __nv_bfloat16* row = wp + static_cast<size_t>(part) * kStemCout * 32 + k * 32 + t * CIN;
      float v[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < CIN; ++c) v[c] = __bfloat162float(row[c]);
      ws[part][e] = make_float4(v[0], v[1], v[2], 0.f);
    }
  }
  __syncthreads();
  const size_t plane = static_cast<size_t>(H) * W;
  const long long total = static_cast<long long>(N) * Ho * Wo;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(idx % Wo);
    const int i = static_cast<int>((idx / Wo) % Ho);
    const int n = static_cast<int>(idx / (static_cast<long long>(Wo) * Ho));
    // the four dy pixels (i, j), (i, j+1), (i+1, j), (i+1, j+1); those outside the conv output contribute zero
    const bool ok[4] = {true, j + 1 < Wo, i + 1 < Ho, i + 1 < Ho && j + 1 < Wo};
    size_t off[4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
      off[q] = ((static_cast<size_t>(n) * Ho + i + (q >> 1)) * Wo + j + (q & 1)) * pitch;
    float acc[4][CIN];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int c = 0; c < CIN; ++c) acc[p][c] = 0.f;
    for (int k0 = 0; k0 < kStemCout; k0 += 8) {
      float dh[4][8], dl[4][8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint4 hv = make_uint4(0, 0, 0, 0), lv = make_uint4(0, 0, 0, 0);
        if (ok[q]) {
          hv = __ldg(reinterpret_cast<const uint4*>(dy + off[q] + k0));
          if (SPLIT) lv = __ldg(reinterpret_cast<const uint4*>(dy_lo + off[q] + k0));
        }
        const __nv_bfloat16* hb = reinterpret_cast<const __nv_bfloat16*>(&hv);
        const __nv_bfloat16* lb = reinterpret_cast<const __nv_bfloat16*>(&lv);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          dh[q][e] = __bfloat162float(hb[e]);
          dl[q][e] = SPLIT ? __bfloat162float(lb[e]) : 0.f;
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int k = k0 + e;
        // (dy pixel q, output pixel p, tap t) in the order the chains are summed
        constexpr int kq[9] = {0, 0, 0, 0, 1, 1, 2, 2, 3};
        constexpr int kp[9] = {0, 1, 2, 3, 1, 3, 2, 3, 3};
        constexpr int kt[9] = {4, 5, 7, 8, 3, 6, 1, 2, 0};
#pragma unroll
        for (int u = 0; u < 9; ++u) {
          const float4 wh = ws[0][k * 9 + kt[u]];
          const float whc[3] = {wh.x, wh.y, wh.z};
          float wlc[3] = {0.f, 0.f, 0.f};
          if (SPLIT) {
            const float4 wl = ws[SPLIT ? 1 : 0][k * 9 + kt[u]];
            wlc[0] = wl.x; wlc[1] = wl.y; wlc[2] = wl.z;
          }
#pragma unroll
          for (int c = 0; c < CIN; ++c) {
            float a = fmaf(dh[kq[u]][e], whc[c], acc[kp[u]][c]);
            if (SPLIT) {
              a = fmaf(dl[kq[u]][e], whc[c], a);
              a = fmaf(dh[kq[u]][e], wlc[c], a);
            }
            acc[kp[u]][c] = a;
          }
        }
      }
    }
    const int y0 = 2 * i, x0 = 2 * j;
#pragma unroll
    for (int c = 0; c < CIN; ++c) {
      float* base = dx + (static_cast<size_t>(n) * CIN + c) * plane;
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        const int y = y0 + (p >> 1), x = x0 + (p & 1);
        if (y < H && x < W) base[static_cast<size_t>(y) * W + x] = acc[p][c];
      }
    }
  }
}

// Stride-2 convolutions run on the stride-1 tensor-core kernel through a 2x2 phase decomposition:
//   xp[(ph*2+pw)*N + n][i][j][c] = x[n][2i+ph][2j+pw][c]   (zero where 2i+ph >= H or 2j+pw >= W)
// so tap (r, s) of a stride-2 conv reads phase ((r+1)&1, (s+1)&1) at a shift of -1 or 0.
__global__ void space_to_phases_kernel(const __nv_bfloat16* __restrict__ x, int pitch, int N, int H, int W, int C,
                                       __nv_bfloat16* __restrict__ xp, int Hh, int Wh) {
  const int groups = C >> 3;
  const long long total = 4LL * N * Hh * Wh * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    long long p = idx / groups;
    const int j = static_cast<int>(p % Wh);
    p /= Wh;
    const int i = static_cast<int>(p % Hh);
    p /= Hh;
    const int n = static_cast<int>(p % N);
    const int q = static_cast<int>(p / N);
    const int h = 2 * i + (q >> 1), w = 2 * j + (q & 1);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (h < H && w < W)
      v = *reinterpret_cast<const uint4*>(x + ((static_cast<size_t>(n) * H + h) * W + w) * pitch + g * 8);
    *reinterpret_cast<uint4*>(xp + (idx / groups) * C + g * 8) = v;
  }
}

__global__ void phases_to_space_kernel(const __nv_bfloat16* __restrict__ xp, int N, int H, int W, int C, int Hh,
                                       int Wh, __nv_bfloat16* __restrict__ x) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * H * W * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx % groups);
    long long p = idx / groups;
    const int w = static_cast<int>(p % W);
    p /= W;
    const int h = static_cast<int>(p % H);
    const int n = static_cast<int>(p / H);
    const int q = (h & 1) * 2 + (w & 1);
    const size_t src = (((static_cast<size_t>(q) * N + n) * Hh + (h >> 1)) * Wh + (w >> 1)) * C + g * 8;
    *reinterpret_cast<uint4*>(x + (idx / groups) * C + g * 8) = *reinterpret_cast<const uint4*>(xp + src);
  }
}

}  // namespace sb

using namespace sb;
typedef __nv_bfloat16 bf16;

extern "C" int semseg_space_to_phases(const void* x, int x_pitch, int N, int H, int W, int C, void* xp,
                                      void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && xp && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && x_pitch % 8 == 0,
               "space_to_phases: bad args");
  if (const int r = check_vec_acts("space_to_phases", C, {{x, nullptr, x_pitch}, {xp, nullptr, C}})) return r;
  const int Hh = (H + 1) / 2, Wh = (W + 1) / 2;
  const long long total = 4LL * N * Hh * Wh * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 148 * 16) blocks = 148 * 16;
  space_to_phases_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(static_cast<const bf16*>(x), x_pitch, N, H,
                                                                           W, C, static_cast<bf16*>(xp), Hh, Wh);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_phases_to_space(const void* xp, int N, int H, int W, int C, void* x, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && xp && N > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "phases_to_space: bad args");
  if (const int r = check_vec_acts("phases_to_space", C, {{xp, nullptr, C}, {x, nullptr, C}})) return r;
  const int Hh = (H + 1) / 2, Wh = (W + 1) / 2;
  const long long total = static_cast<long long>(N) * H * W * (C / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > 148 * 16) blocks = 148 * 16;
  phases_to_space_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(static_cast<const bf16*>(xp), N, H, W, C,
                                                                           Hh, Wh, static_cast<bf16*>(x));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_im2col3x3s2(const void* x, int x_pitch, int N, int H, int W, int Cin, void* out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && out && N > 0 && H > 0 && W > 0 && Cin >= 1 && Cin <= 3 && x_pitch >= 4 && x_pitch % 4 == 0,
               "im2col3x3s2: needs 1..3 input channels in a pitch that is a multiple of 4 (got Cin=%d pitch=%d)", Cin,
               x_pitch);
  // one uint2 (4 channels) per input pixel, 16-byte stores of 32 patch values
  if (const int r = check_vec_acts("im2col3x3s2", Cin, {{x, nullptr, x_pitch}}, 8)) return r;
  if (const int r = check_vec_acts("im2col3x3s2", 0, {{out, nullptr, 32}})) return r;
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long total = static_cast<long long>(N) * Ho * Wo;
  long long blocks = (total + 255) / 256;
  if (blocks > 148 * 16) blocks = 148 * 16;
  sb::im2col3x3s2_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(static_cast<const bf16*>(x), x_pitch, N, H, W,
                                                                           Cin, Ho, Wo, static_cast<bf16*>(out));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_stem_dgrad3x3s2(const void* dy, const void* dy_lo, int dy_pitch, int N, int Ho, int Wo, int H,
                                      int W, int Cin, int Cout, const void* wp, int wp_split, float* dx_nchw,
                                      void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dy && wp && dx_nchw, "stem_dgrad3x3s2: null pointer (dy, wp and dx are required)");
  SB_CHECK_ARG(Cin >= 1 && Cin <= 3, "stem_dgrad3x3s2: needs 1..3 input channels (got Cin=%d)", Cin);
  SB_CHECK_ARG(Cout == kStemCout, "stem_dgrad3x3s2: needs Cout=%d (got %d)", kStemCout, Cout);
  SB_CHECK_ARG(N > 0 && H > 0 && W > 0 && Ho == (H - 1) / 2 + 1 && Wo == (W - 1) / 2 + 1,
               "stem_dgrad3x3s2: Ho=(H-1)/2+1 and Wo=(W-1)/2+1 required (got N=%d H=%d W=%d Ho=%d Wo=%d)", N, H, W, Ho,
               Wo);
  SB_CHECK_ARG(dy_pitch >= Cout && dy_pitch % 8 == 0,
               "stem_dgrad3x3s2: dy pitch must be >= Cout and a multiple of 8 (got %d)", dy_pitch);
  SB_CHECK_ARG(wp_split == 0 || wp_split == 1, "stem_dgrad3x3s2: wp_split must be 0 or 1 (got %d)", wp_split);
  SB_CHECK_ARG((dy_lo != nullptr) == (wp_split == 1),
               "stem_dgrad3x3s2: dy_lo and a split weight slab go together (bf16x3), got dy_lo=%s wp_split=%d",
               dy_lo ? "set" : "null", wp_split);
  SB_CHECK_ARG(reinterpret_cast<uintptr_t>(dy) % 16 == 0 && reinterpret_cast<uintptr_t>(dy_lo) % 16 == 0,
               "stem_dgrad3x3s2: dy and dy_lo must be 16-byte aligned");
  const long long total = static_cast<long long>(N) * Ho * Wo;
  long long blocks = (total + 255) / 256;
  if (blocks > 148 * 16) blocks = 148 * 16;
  const dim3 grid(static_cast<unsigned>(blocks));
  const bf16 *d = static_cast<const bf16*>(dy), *dl = static_cast<const bf16*>(dy_lo), *w = static_cast<const bf16*>(wp);
#define SB_STEM_DGRAD(CIN, SPLIT) \
  sb::stem_dgrad3x3s2_kernel<CIN, SPLIT><<<grid, 256, 0, stream>>>(d, dl, dy_pitch, N, H, W, Ho, Wo, w, dx_nchw)
  if (wp_split) {
    if (Cin == 1) SB_STEM_DGRAD(1, true); else if (Cin == 2) SB_STEM_DGRAD(2, true); else SB_STEM_DGRAD(3, true);
  } else {
    if (Cin == 1) SB_STEM_DGRAD(1, false); else if (Cin == 2) SB_STEM_DGRAD(2, false); else SB_STEM_DGRAD(3, false);
  }
#undef SB_STEM_DGRAD
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_pack_weights_multi(const semseg_pack_item* items_dev, int n_items, int n_tiles, int max_taps,
                                         void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(items_dev && n_items > 0 && n_tiles > 0 && max_taps > 0 && max_taps <= SEMSEG_MAX_TAPS,
               "pack_weights_multi: bad args");
  const size_t smem = static_cast<size_t>(32) * (32 * max_taps + 1) * sizeof(float);
  sb::pack_multi_kernel<<<static_cast<unsigned>(n_tiles), 256, smem, stream>>>(items_dev, n_items);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_nchw_f32_to_nhwc_bf16(const float* in, void* out, void* out_lo, int N, int C, int H, int W,
                                            int out_pitch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(in && out && N > 0 && C > 0 && H > 0 && W > 0 && out_pitch >= C, "nchw_f32_to_nhwc_bf16: bad args");
  dim3 grid(cdiv(H * W, 32), cdiv(C, 32), N);
  nchw_to_nhwc_kernel<float, bf16><<<grid, dim3(32, 8), 0, stream>>>(in, static_cast<bf16*>(out),
                                                                     static_cast<bf16*>(out_lo), C, H * W, out_pitch);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_nhwc_bf16_to_nchw_f32(const void* in, const void* in_lo, float* out, int N, int C, int H, int W,
                                            int in_pitch, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(in && out && N > 0 && C > 0 && H > 0 && W > 0 && in_pitch >= C, "nhwc_bf16_to_nchw_f32: bad args");
  dim3 grid(cdiv(H * W, 32), cdiv(C, 32), N);
  nhwc_to_nchw_kernel<bf16, float><<<grid, dim3(32, 8), 0, stream>>>(
      static_cast<const bf16*>(in), static_cast<const bf16*>(in_lo), out, C, H * W, in_pitch);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_nhwc_f32_to_nchw_f32(const float* in, float* out, int N, int C, int H, int W, int in_pitch,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(in && out && N > 0 && C > 0 && H > 0 && W > 0 && in_pitch >= C, "nhwc_f32_to_nchw_f32: bad args");
  dim3 grid(cdiv(H * W, 32), cdiv(C, 32), N);
  nhwc_to_nchw_kernel<float, float><<<grid, dim3(32, 8), 0, stream>>>(in, nullptr, out, C, H * W, in_pitch);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

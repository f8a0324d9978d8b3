// Active Boundary Loss (Wang et al., AAAI 2022; semseg_b200/losses.py ActiveBoundaryLoss) on the grid of the fused
// tail's output, and Boundary IoU (Cheng et al., CVPR 2021; semseg_b200/metrics.py boundaryIoUGPU).
//
// ABL forward, every pass on the device and graph-capturable (include/semseg_b200.h states the contract):
//   1. GT boundary and its exact squared Euclidean distance transform, separable (Meijster et al., 2000) in integers:
//      a column pass (one thread per image column, coalesced) finds the vertical distance to the nearest boundary pixel
//      of the column, a row pass (one thread per image row) takes the lower envelope of the parabolas (x - i)^2 + g(i)^2
//      with integer separators. D = max(sqrt(e) - 1, 0) in fp64, rounded once.
//   2. The boundary score k = KL(p|p_down) + KL(p|p_right): one CTA per 16 x 16 grid tile, the tile and a one-pixel
//      halo staged one chunk of 16 classes at a time (logit and probability), recomputed from the 1/8 logits (the
//      tail's bilinear xZ) and the tail's lse, so no full-resolution probability tensor exists. Each pixel's highest
//      exceeded threshold level goes into an integer count histogram.
//   3. One thread turns the histogram's suffix sums into the threshold level j*, left in device memory.
//   4. Dilation of {k > t_j*}, the direction target argmin D over the 8 neighbours and the pixel itself, the
//      8-neighbour KL logits z and the label-smoothed CE l: the same tiles; a tile without a selected pixel stages
//      nothing. Each selected pixel keeps w dl/dz (8 floats) for the backward; per-CTA (sum w l, M) partials go through
//      the tail's fp64 reduce.
// ABL backward: the same tiles, the selected pixels' w sum_j g_j (p - p_nj) scaled by abl_weight grad / M into the
// output-grid gradient (at zoom 1: straight into dlogits), then the bilinear adjoint of csrc/crf.cu.
//
// KL(a|b) is evaluated as sum_c p_a d_c / sum_c p_a - log1p(sum_c p_b expm1(d_c) / sum_c p_b) with d = s_a - s_b: both
// terms are O(|d|), so the result keeps its relative accuracy where neighbouring distributions nearly agree, and the
// normalisation by the staged sums cancels the rounding of the lse.
//
// Integer atomics count the histograms; every float is written by one thread in a fixed order: deterministic.
#include <cmath>

#include "host_common.h"

namespace sb {

constexpr int kAblTile = 16;
constexpr int kAblThreads = kAblTile * kAblTile;
constexpr int kAblHalo = kAblTile + 2;
constexpr int kAblHP = kAblHalo * kAblHalo;   // halo pixels of a tile
constexpr int kAblCC = 16;                    // classes per staged chunk
constexpr int kAblLevels = 256;               // threshold levels t_j = 1e-5 * 1.2^j
constexpr int kAblMaxClasses = 256;
constexpr int kBiouThreads = 256;
constexpr int kBiouMaxClasses = 4096;

struct AblGeom {
  const float* logits;  // fp32 NHWC [N, h, w, pitch]
  int pitch, N, h, w, C, zshift;
  int Hg, Wg;           // loss grid: zoom (h-1)+1 x zoom (w-1)+1
  const float* lse;     // [N, Hg, Wg]
};

struct AblLevels {
  float t[kAblLevels];  // (float) t_j, t_j in fp64
};

// The logit of class c at grid pixel (gy, gx): the tail's bilinear xZ interpolation (align_corners, Z = 1 << zshift).
__device__ __forceinline__ float abl_logit(const AblGeom& g, int n, int gy, int gx, int c) {
  const int Z = 1 << g.zshift;
  const float step = 1.f / Z;
  const int i0 = gy >> g.zshift, j0 = gx >> g.zshift;
  const int i1 = min(i0 + 1, g.h - 1), j1 = min(j0 + 1, g.w - 1);
  const float l1w = static_cast<float>(gx & (Z - 1)) * step, l0w = 1.f - l1w;
  const float l1h = static_cast<float>(gy & (Z - 1)) * step, l0h = 1.f - l1h;
  const size_t row0 = (static_cast<size_t>(n) * g.h + i0) * g.w, row1 = (static_cast<size_t>(n) * g.h + i1) * g.w;
  const float top = l0w * g.logits[(row0 + j0) * g.pitch + c] + l1w * g.logits[(row0 + j1) * g.pitch + c];
  if (g.zshift == 0) return top;
  const float bot = l0w * g.logits[(row1 + j0) * g.pitch + c] + l1w * g.logits[(row1 + j1) * g.pitch + c];
  return l0h * top + l1h * bot;
}

// Halo pixel hp of the tile at (ty0, tx0), clamped into the grid: out-of-grid neighbours replicate the edge.
__device__ __forceinline__ void abl_halo_pos(const AblGeom& g, int ty0, int tx0, int hp, int& gy, int& gx) {
  gy = min(max(ty0 - 1 + hp / kAblHalo, 0), g.Hg - 1);
  gx = min(max(tx0 - 1 + hp % kAblHalo, 0), g.Wg - 1);
}

__device__ __forceinline__ void abl_stage_lse(const AblGeom& g, int n, int ty0, int tx0, float* slse) {
  for (int hp = threadIdx.x; hp < kAblHP; hp += kAblThreads) {
    int gy, gx;
    abl_halo_pos(g, ty0, tx0, hp, gy, gx);
    slse[hp] = g.lse[(static_cast<size_t>(n) * g.Hg + gy) * g.Wg + gx];
  }
}

// ss[cl][hp] = logit, sp[cl][hp] = exp(logit - lse) of classes c0 + cl; padded classes stage 0 and 0.
__device__ __forceinline__ void abl_stage_chunk(const AblGeom& g, int n, int ty0, int tx0, int c0, const float* slse,
                                                float* ss, float* sp) {
  for (int idx = threadIdx.x; idx < kAblHP * kAblCC; idx += kAblThreads) {
    const int hp = idx / kAblCC, cl = idx - hp * kAblCC;
    const int c = c0 + cl;
    float s = 0.f, p = 0.f;
    if (c < g.C) {
      int gy, gx;
      abl_halo_pos(g, ty0, tx0, hp, gy, gx);
      s = abl_logit(g, n, gy, gx, c);
      p = expf(s - slse[hp]);
    }
    ss[cl * kAblHP + hp] = s;
    sp[cl * kAblHP + hp] = p;
  }
}

// p_b (e^d - 1) with d = s_a - s_b and p_b = exp(s_b - lse_b): expm1 where it is accurate, the exact product elsewhere.
__device__ __forceinline__ float abl_pexpm1(float p_b, float d, float s_a, float lse_b) {
  return fabsf(d) < 1.f ? p_b * expm1f(d) : expf(s_a - lse_b) - p_b;
}

// The sums are ~1 (normalised probabilities), well inside __fdividef's range.
__device__ __forceinline__ float abl_kl(float A, float Sa, float B, float Sb) {
  return __fdividef(A, Sa) - log1pf(__fdividef(B, Sb));
}

// ------------------------------------------------------------------------------------------------ distance transform
// gcol[n][y][x] = vertical distance from (y, x) to the nearest GT-boundary pixel of column x, capped at Hg + Wg (more
// than any in-image distance). A pixel is a GT-boundary pixel if it is ignore_index or differs from the pixel below or
// to its right.
__global__ void __launch_bounds__(256)
abl_edt_cols_kernel(const long long* __restrict__ target, int N, int Hg, int Wg, long long ignore,
                    int* __restrict__ gcol) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(N) * Wg) return;
  const int n = static_cast<int>(i / Wg), x = static_cast<int>(i % Wg);
  const size_t base = static_cast<size_t>(n) * Hg * Wg + x;
  const long long* t = target + base;
  int* gc = gcol + base;
  const int G = Hg + Wg;
  int d = G;
  long long v = t[0];
  for (int y = 0; y < Hg; ++y) {
    const long long below = y + 1 < Hg ? t[static_cast<size_t>(y + 1) * Wg] : v;
    const bool b = v == ignore || v != below || (x + 1 < Wg && v != t[static_cast<size_t>(y) * Wg + 1]);
    d = b ? 0 : min(d + 1, G);
    gc[static_cast<size_t>(y) * Wg] = d;
    v = below;
  }
  for (int y = Hg - 2; y >= 0; --y) {
    d = min(d + 1, G);
    const int cur = gc[static_cast<size_t>(y) * Wg];
    if (cur < d) d = cur;
    else gc[static_cast<size_t>(y) * Wg] = d;
  }
}

__device__ __forceinline__ long long floor_div(long long a, long long b) {  // b > 0
  return a >= 0 ? a / b : -((-a + b - 1) / b);
}

// Per row, e(x) = min_i (x - i)^2 + g(i)^2 (Meijster's lower envelope, integer separators; stacks in the workspace),
// then D = fp32(max(sqrt(e) - 1, 0)), or +inf when the image has no GT-boundary pixel (e >= (Hg + Wg)^2).
__global__ void __launch_bounds__(128)
abl_edt_rows_kernel(const int* __restrict__ gcol, int N, int Hg, int Wg, int* __restrict__ stk_s,
                    int* __restrict__ stk_t, float* __restrict__ D) {
  const long long r = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= static_cast<long long>(N) * Hg) return;
  const int* g = gcol + r * Wg;
  int* s = stk_s + r * Wg;
  int* t = stk_t + r * Wg;
  float* out = D + r * Wg;
  const long long G2 = static_cast<long long>(Hg + Wg) * (Hg + Wg);
  int q = 0;
  s[0] = 0;
  t[0] = 0;
  for (int u = 1; u < Wg; ++u) {
    const long long gu = g[u];
    for (;;) {
      if (q < 0) break;
      const long long xs = t[q], i = s[q], gi = g[i];
      if ((xs - i) * (xs - i) + gi * gi <= (xs - u) * (xs - u) + gu * gu) break;
      --q;
    }
    if (q < 0) {
      q = 0;
      s[0] = u;
    } else {
      const long long i = s[q], gi = g[i];
      const long long wsep = 1 + floor_div(static_cast<long long>(u) * u - i * i + gu * gu - gi * gi, 2 * (u - i));
      if (wsep < Wg) {
        ++q;
        s[q] = u;
        t[q] = static_cast<int>(wsep);
      }
    }
  }
  for (int u = Wg - 1; u >= 0; --u) {
    const long long i = s[q], gi = g[i];
    const long long e = (u - i) * (u - i) + gi * gi;
    out[u] = e >= G2 ? INFINITY : static_cast<float>(fmax(sqrt(static_cast<double>(e)) - 1.0, 0.0));
    if (u == t[q]) --q;
  }
}

// ------------------------------------------------------------------------------------------------ boundary score
// k = KL(p|p_down) + KL(p|p_right) (a term is 0 past the last row / column); hist[j + 1] counts the pixels whose
// highest exceeded level is j (hist[0]: none exceeded).
__global__ void __launch_bounds__(kAblThreads)
abl_kmap_kernel(AblGeom g, AblLevels lv, float* __restrict__ kmap, int* __restrict__ hist) {
  __shared__ float ss[kAblCC * kAblHP], sp[kAblCC * kAblHP], slse[kAblHP];
  __shared__ float sthr[kAblLevels];
  __shared__ int shist[kAblLevels + 1];
  const int n = blockIdx.z, ty0 = blockIdx.y * kAblTile, tx0 = blockIdx.x * kAblTile;
  const int ty = threadIdx.x / kAblTile, tx = threadIdx.x % kAblTile;
  const int gy = ty0 + ty, gx = tx0 + tx;
  const bool inside = gy < g.Hg && gx < g.Wg;
  const int me = (ty + 1) * kAblHalo + tx + 1, rt = me + 1, dn = me + kAblHalo;
  for (int i = threadIdx.x; i < kAblLevels; i += kAblThreads) sthr[i] = lv.t[i];
  for (int i = threadIdx.x; i <= kAblLevels; i += kAblThreads) shist[i] = 0;
  abl_stage_lse(g, n, ty0, tx0, slse);
  float Sa = 0.f, Ar = 0.f, Br = 0.f, Sr = 0.f, Ad = 0.f, Bd = 0.f, Sd = 0.f;
  for (int c0 = 0; c0 < g.C; c0 += kAblCC) {
    __syncthreads();
    abl_stage_chunk(g, n, ty0, tx0, c0, slse, ss, sp);
    __syncthreads();
#pragma unroll 4
    for (int cl = 0; cl < kAblCC; ++cl) {
      const float* s = ss + cl * kAblHP;
      const float* p = sp + cl * kAblHP;
      const float s0 = s[me], p0 = p[me];
      Sa += p0;
      const float d_r = s0 - s[rt], d_d = s0 - s[dn];
      Ar = fmaf(p0, d_r, Ar);
      Ad = fmaf(p0, d_d, Ad);
      Br += abl_pexpm1(p[rt], d_r, s0, slse[rt]);
      Bd += abl_pexpm1(p[dn], d_d, s0, slse[dn]);
      Sr += p[rt];
      Sd += p[dn];
    }
  }
  if (inside) {
    float k = 0.f;
    if (gx + 1 < g.Wg) k += abl_kl(Ar, Sa, Br, Sr);
    if (gy + 1 < g.Hg) k += abl_kl(Ad, Sa, Bd, Sd);
    kmap[(static_cast<size_t>(n) * g.Hg + gy) * g.Wg + gx] = k;
    int cnt = 0;  // levels below k: k > t_j for j < cnt
    for (int b = kAblLevels; b; b >>= 1)
      if (cnt + b <= kAblLevels && k > sthr[cnt + b - 1]) cnt += b;
    atomicAdd(&shist[cnt], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i <= kAblLevels; i += kAblThreads)
    if (shist[i]) atomicAdd(&hist[i], shist[i]);
}

// jstar[0] = j*, the smallest level j < 256 with at most max_n pixels of k > t_j (255 when every level has more);
// jstar[1] = the bits of (float) t_j*.
__global__ void abl_level_kernel(const int* __restrict__ hist, AblLevels lv, double max_n, int* __restrict__ jstar) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  long long above = 0;
  int best = kAblLevels - 1;
  for (int j = kAblLevels - 1; j >= 0; --j) {
    above += hist[j + 1];
    if (static_cast<double>(above) <= max_n) best = j;
  }
  jstar[0] = best;
  jstar[1] = __float_as_int(lv.t[best]);
}

// Neighbour offsets n_0..n_7 (row, col), in the contract's order.
__constant__ int kAblDy[8] = {1, -1, 0, 0, -1, 1, -1, 1};
__constant__ int kAblDx[8] = {0, 0, -1, 1, 1, 1, -1, -1};

// code[pix] = dir (0..8; 15: the image has no GT boundary) | B << 4 | selected << 5; for a selected pixel
// wg[pix][j] = w dl/dz_j; partial[2 b] = sum of w l over the tile's selected pixels, partial[2 b + 1] = their count.
__global__ void __launch_bounds__(kAblThreads)
abl_term_kernel(AblGeom g, const int* __restrict__ jstar, const float* __restrict__ D,
                const float* __restrict__ kmap, float clip, float eps, unsigned char* __restrict__ code,
                float* __restrict__ wg, float* __restrict__ partial) {
  __shared__ float ss[kAblCC * kAblHP], sp[kAblCC * kAblHP], slse[kAblHP];
  __shared__ float red_loss[kAblThreads / 32], red_cnt[kAblThreads / 32];
  const int n = blockIdx.z, ty0 = blockIdx.y * kAblTile, tx0 = blockIdx.x * kAblTile;
  const int ty = threadIdx.x / kAblTile, tx = threadIdx.x % kAblTile;
  const int gy = ty0 + ty, gx = tx0 + tx;
  const bool inside = gy < g.Hg && gx < g.Wg;
  const size_t img = static_cast<size_t>(n) * g.Hg * g.Wg;
  const size_t pix = img + static_cast<size_t>(min(gy, g.Hg - 1)) * g.Wg + min(gx, g.Wg - 1);
  const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  bool sel = false;
  int dir = 15;
  float dc = 0.f;
  if (inside) {
    const float th = __int_as_float(jstar[1]);
    bool B = false;
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int y = gy + dy, x = gx + dx;
        if (y >= 0 && y < g.Hg && x >= 0 && x < g.Wg && kmap[img + static_cast<size_t>(y) * g.Wg + x] > th) B = true;
      }
    dc = D[pix];
    if (dc < INFINITY) {      // argmin over n_0..n_7 (out-of-image: +inf) and the pixel itself, the first on ties
      float best = INFINITY;
      for (int j = 0; j < 9; ++j) {
        const int y = gy + (j < 8 ? kAblDy[j] : 0), x = gx + (j < 8 ? kAblDx[j] : 0);
        const float v = (y >= 0 && y < g.Hg && x >= 0 && x < g.Wg) ? D[img + static_cast<size_t>(y) * g.Wg + x]
                                                                   : INFINITY;
        if (j == 0 || v < best) {
          best = v;
          dir = j;
        }
      }
    }
    sel = B && dir != 8 && dir != 15;
    code[pix] = static_cast<unsigned char>(dir | (B ? 16 : 0) | (sel ? 32 : 0));
  }
  if (!__syncthreads_or(sel)) {
    if (threadIdx.x == 0) {
      partial[2 * b] = 0.f;
      partial[2 * b + 1] = 0.f;
    }
    return;
  }
  abl_stage_lse(g, n, ty0, tx0, slse);
  const int me = (ty + 1) * kAblHalo + tx + 1;
  int nb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) nb[j] = me + kAblDy[j] * kAblHalo + kAblDx[j];
  float A[8], Sn[8], Bc[8], Sp = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) A[j] = Sn[j] = Bc[j] = 0.f;
  for (int c0 = 0; c0 < g.C; c0 += kAblCC) {
    __syncthreads();
    abl_stage_chunk(g, n, ty0, tx0, c0, slse, ss, sp);
    __syncthreads();
    if (!sel) continue;
    const float lse0 = slse[me];
    for (int cl = 0; cl < kAblCC; ++cl) {
      const float* s = ss + cl * kAblHP;
      const float* p = sp + cl * kAblHP;
      const float s0 = s[me], p0 = p[me];
      Sp += p0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float sn = s[nb[j]], pn = p[nb[j]];
        const float d = sn - s0;                  // KL(p_nj | p): a = n_j, b = the centre
        A[j] = fmaf(pn, d, A[j]);
        Sn[j] += pn;
        Bc[j] += abl_pexpm1(p0, d, sn, lse0);
      }
    }
  }
  float loss = 0.f, cnt = 0.f;
  if (sel) {
    float z[8], zmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      z[j] = abl_kl(A[j], Sn[j], Bc[j], Sp);
      zmax = fmaxf(zmax, z[j]);
    }
    float se = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) se += expf(z[j] - zmax);
    const float lz = zmax + logf(se);
    const float y_off = eps / 8.f, y_dir = 1.f - eps, Y = y_dir + 7.f * y_off;
    float yz = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) yz = fmaf(j == dir ? y_dir : y_off, z[j], yz);
    const float w = fminf(dc, clip) / clip;
    loss = w * (Y * lz - yz);
    cnt = 1.f;
    float* o = wg + ((static_cast<size_t>(n) * g.Hg + gy) * g.Wg + gx) * 8;   // recomputed: nothing 64-bit stays live
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = w * (Y * expf(z[j] - lz) - (j == dir ? y_dir : y_off));
  }
  for (int o = 16; o > 0; o >>= 1) {
    loss += __shfl_xor_sync(0xffffffffu, loss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red_loss[threadIdx.x >> 5] = loss;
    red_cnt[threadIdx.x >> 5] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float l = 0.f, c = 0.f;
    for (int i = 0; i < kAblThreads / 32; ++i) {
      l += red_loss[i];
      c += red_cnt[i];
    }
    partial[2 * b] = l;
    partial[2 * b + 1] = c;
  }
}

// For each selected pixel and class: out[pix][c] (accumulate: +=) of abl_weight grad_out / M * sum_j wg_j (p_c -
// p_nj,c). Other pixels are not written.
__global__ void __launch_bounds__(kAblThreads)
abl_bwd_kernel(AblGeom g, const unsigned char* __restrict__ code, const float* __restrict__ wg,
               const float* __restrict__ info, float abl_weight, const float* __restrict__ grad_out,
               float* __restrict__ out, int accumulate) {
  __shared__ float ss[kAblCC * kAblHP], sp[kAblCC * kAblHP], slse[kAblHP];
  const int n = blockIdx.z, ty0 = blockIdx.y * kAblTile, tx0 = blockIdx.x * kAblTile;
  const int ty = threadIdx.x / kAblTile, tx = threadIdx.x % kAblTile;
  const int gy = ty0 + ty, gx = tx0 + tx;
  const bool inside = gy < g.Hg && gx < g.Wg;
  const size_t pix = (static_cast<size_t>(n) * g.Hg + min(gy, g.Hg - 1)) * g.Wg + min(gx, g.Wg - 1);
  const bool sel = inside && (code[pix] & 32);
  if (!__syncthreads_or(sel)) return;
  abl_stage_lse(g, n, ty0, tx0, slse);
  const int me = (ty + 1) * kAblHalo + tx + 1;
  const float scale = abl_weight * grad_out[0] / fmaxf(info[1], 1.f);
  float gw[8], G = 0.f;
  int nb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    gw[j] = sel ? wg[pix * 8 + j] : 0.f;
    G += gw[j];
    nb[j] = me + kAblDy[j] * kAblHalo + kAblDx[j];
  }
  for (int c0 = 0; c0 < g.C; c0 += kAblCC) {
    __syncthreads();
    abl_stage_chunk(g, n, ty0, tx0, c0, slse, ss, sp);
    __syncthreads();
    if (!sel) continue;
    float* o = out + pix * g.C + c0;
    for (int cl = 0; cl < kAblCC && c0 + cl < g.C; ++cl) {
      const float* p = sp + cl * kAblHP;
      float v = G * p[me];
#pragma unroll
      for (int j = 0; j < 8; ++j) v = fmaf(-gw[j], p[nb[j]], v);
      o[cl] = accumulate ? fmaf(scale, v, o[cl]) : scale * v;
    }
  }
}

// ------------------------------------------------------------------------------------------------ Boundary IoU
__device__ __forceinline__ int sat32(long long v) {
  return static_cast<int>(v < INT_MIN ? static_cast<long long>(INT_MIN) : v > INT_MAX ? static_cast<long long>(INT_MAX) : v);
}

// mm[0..3][pix] = min / max of the target, min / max of the prediction over the pixel's row window [x - d, x + d]
// (inside the image; labels saturated to int32).
__global__ void __launch_bounds__(kBiouThreads)
biou_rows_kernel(const long long* __restrict__ pred, const long long* __restrict__ target, long long P, int W, int d,
                 int* __restrict__ mm) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int x = static_cast<int>(i % W);
  const long long row = i - x;
  int tmin = INT_MAX, tmax = INT_MIN, omin = INT_MAX, omax = INT_MIN;
  for (int xx = max(0, x - d); xx <= min(W - 1, x + d); ++xx) {
    const int t = sat32(target[row + xx]), o = sat32(pred[row + xx]);
    tmin = min(tmin, t);
    tmax = max(tmax, t);
    omin = min(omin, o);
    omax = max(omax, o);
  }
  mm[i] = tmin;
  mm[P + i] = tmax;
  mm[2 * P + i] = omin;
  mm[3 * P + i] = omax;
}

// A pixel is in its map's band if its (2d+1)^2 window reaches outside the image or holds another label. Over the pixels
// whose target is not ignore_index: counts[c] = both in band and pred == target == c, counts[K + c] = prediction c in
// band, counts[2K + c] = target c in band.
__global__ void __launch_bounds__(kBiouThreads)
biou_hist_kernel(const long long* __restrict__ pred, const long long* __restrict__ target, const int* __restrict__ mm,
                 long long P, int H, int W, int K, int d, long long ignore, int* __restrict__ counts) {
  extern __shared__ int h[];  // [3 K]
  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x) h[i] = 0;
  __syncthreads();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < P;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long t = target[i];
    if (t == ignore) continue;
    const int x = static_cast<int>(i % W);
    const int y = static_cast<int>((i / W) % H);
    const long long img = i - (static_cast<long long>(y) * W + x);
    bool bt = y < d || y + d > H - 1 || x < d || x + d > W - 1, bo = bt;
    if (!bt) {
      int tmin = INT_MAX, tmax = INT_MIN, omin = INT_MAX, omax = INT_MIN;
      for (int yy = y - d; yy <= y + d; ++yy) {
        const long long q = img + static_cast<long long>(yy) * W + x;
        tmin = min(tmin, mm[q]);
        tmax = max(tmax, mm[P + q]);
        omin = min(omin, mm[2 * P + q]);
        omax = max(omax, mm[3 * P + q]);
      }
      bt = tmin != tmax;
      bo = omin != omax;
    }
    const long long o = pred[i];
    if (bt && t >= 0 && t < K) atomicAdd(&h[2 * K + static_cast<int>(t)], 1);
    if (bo && o >= 0 && o < K) atomicAdd(&h[K + static_cast<int>(o)], 1);
    if (bt && bo && o == t && t >= 0 && t < K) atomicAdd(&h[static_cast<int>(t)], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x)
    if (h[i]) atomicAdd(&counts[i], h[i]);
}

}  // namespace sb

using namespace sb;

namespace {

int abl_grid(int n, int zoom) { return zoom * (n - 1) + 1; }

bool abl_zoom_ok(int zoom) { return zoom == 1 || zoom == 2 || zoom == 4 || zoom == 8; }

long long abl_ctas(int N, int Hg, int Wg) {
  return static_cast<long long>(cdiv(Wg, kAblTile)) * cdiv(Hg, kAblTile) * N;
}

// The forward state, in 4-byte words of P = N Hg Wg pixels and T tiles.
struct AblLayout {
  long long D, k, wg, code, hist, jstar, partial, total;
};

AblLayout abl_layout(int N, int Hg, int Wg) {
  const long long P = static_cast<long long>(N) * Hg * Wg;
  AblLayout l;
  l.D = 0;
  l.k = P;
  l.wg = 2 * P;                 // 8 floats per pixel; the EDT's column distances and stacks (3 P ints) before that
  l.code = 10 * P;              // one byte per pixel
  l.hist = l.code + (P + 3) / 4;
  l.jstar = l.hist + kAblLevels + 1;   // j* and the bits of t_j*
  l.partial = l.jstar + 2;
  l.total = l.partial + 2 * abl_ctas(N, Hg, Wg);
  return l;
}

AblLevels abl_levels() {
  AblLevels lv;
  double t = 1e-5;
  for (int j = 0; j < kAblLevels; ++j) {
    lv.t[j] = static_cast<float>(t);
    t *= 1.2;
  }
  return lv;
}

int check_abl(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse) {
  SB_CHECK_ARG(abl_zoom_ok(zoom), "abl: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(logits && lse, "abl: null pointer");
  SB_CHECK_ARG(N > 0 && N <= 65535 && h > 0 && w > 0 && C > 0 && C <= kAblMaxClasses && pitch >= C,
               "abl: bad sizes (N=%d h=%d w=%d C=%d pitch=%d; C<=%d)", N, h, w, C, pitch, kAblMaxClasses);
  SB_CHECK_ARG(abl_grid(h, zoom) <= 65535LL * kAblTile, "abl: grid height %d too large", abl_grid(h, zoom));
  return SEMSEG_OK;
}

AblGeom abl_geom(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse) {
  AblGeom g;
  g.logits = logits;
  g.pitch = pitch;
  g.N = N;
  g.h = h;
  g.w = w;
  g.C = C;
  g.zshift = zoom == 1 ? 0 : zoom == 2 ? 1 : zoom == 4 ? 2 : 3;
  g.Hg = abl_grid(h, zoom);
  g.Wg = abl_grid(w, zoom);
  g.lse = lse;
  return g;
}

}  // namespace

extern "C" long long semseg_abl_workspace_floats(int N, int h, int w, int C, int zoom, int pass) {
  SB_CHECK_ARG(abl_zoom_ok(zoom) && N > 0 && h > 0 && w > 0 && C > 0 && (pass == 0 || pass == 1),
               "abl: bad zoom %d, size or pass %d", zoom, pass);
  const int Hg = abl_grid(h, zoom), Wg = abl_grid(w, zoom);
  if (pass == 0) return abl_layout(N, Hg, Wg).total;
  if (zoom == 1) return 0;                                 // added straight into dlogits
  return static_cast<long long>(N) * C * Wg * (Hg + h);     // [N][Hg][Wg][C], then its row adjoint [N][h][Wg][C]
}

extern "C" int semseg_abl_fwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse,
                              const void* target, long long ignore_index, double max_n_ratio, float max_clip_dist,
                              float label_smoothing, float* state, float* loss_out, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_abl(logits, pitch, N, h, w, C, zoom, lse);
  if (r) return r;
  SB_CHECK_ARG(target && state && loss_out, "abl_fwd: null pointer");
  SB_CHECK_ARG(std::isfinite(max_n_ratio) && max_n_ratio >= 0.0 && max_n_ratio <= 1.0,
               "abl_fwd: max_n_ratio %g must lie in [0, 1]", max_n_ratio);
  SB_CHECK_ARG(std::isfinite(max_clip_dist) && max_clip_dist > 0.f, "abl_fwd: max_clip_dist %g must be finite and > 0",
               max_clip_dist);
  SB_CHECK_ARG(label_smoothing >= 0.f && label_smoothing <= 1.f, "abl_fwd: label_smoothing %g must lie in [0, 1]",
               label_smoothing);
  const AblGeom g = abl_geom(logits, pitch, N, h, w, C, zoom, lse);
  const AblLayout l = abl_layout(N, g.Hg, g.Wg);
  const long long P = static_cast<long long>(N) * g.Hg * g.Wg;
  const long long* t = static_cast<const long long*>(target);
  float* D = state + l.D;
  int* gcol = reinterpret_cast<int*>(state + l.wg);
  int* hist = reinterpret_cast<int*>(state + l.hist);
  int* jstar = reinterpret_cast<int*>(state + l.jstar);
  const long long cols = static_cast<long long>(N) * g.Wg, rows = static_cast<long long>(N) * g.Hg;
  abl_edt_cols_kernel<<<static_cast<unsigned>((cols + 255) / 256), 256, 0, stream>>>(t, N, g.Hg, g.Wg, ignore_index,
                                                                                      gcol);
  SB_LAUNCHED();
  abl_edt_rows_kernel<<<static_cast<unsigned>((rows + 127) / 128), 128, 0, stream>>>(gcol, N, g.Hg, g.Wg, gcol + P,
                                                                                      gcol + 2 * P, D);
  SB_LAUNCHED();
  SB_CUDA(cudaMemsetAsync(hist, 0, sizeof(int) * (kAblLevels + 1), stream));
  const AblLevels lv = abl_levels();
  const dim3 tiles(cdiv(g.Wg, kAblTile), cdiv(g.Hg, kAblTile), N);
  abl_kmap_kernel<<<tiles, kAblThreads, 0, stream>>>(g, lv, state + l.k, hist);
  SB_LAUNCHED();
  abl_level_kernel<<<1, 32, 0, stream>>>(hist, lv, max_n_ratio * g.Hg * g.Wg, jstar);
  SB_LAUNCHED();
  abl_term_kernel<<<tiles, kAblThreads, 0, stream>>>(g, jstar, D, state + l.k, max_clip_dist, label_smoothing,
                                                     reinterpret_cast<unsigned char*>(state + l.code), state + l.wg,
                                                     state + l.partial);
  SB_LAUNCHED();
  return launch_mean_reduce(state + l.partial, static_cast<int>(abl_ctas(N, g.Hg, g.Wg)), loss_out, stream);
}

extern "C" int semseg_abl_bwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse,
                              const float* state, const float* loss_info, float abl_weight, const float* grad_out,
                              float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_abl(logits, pitch, N, h, w, C, zoom, lse);
  if (r) return r;
  SB_CHECK_ARG(state && loss_info && grad_out && dlogits && (zoom == 1 || workspace), "abl_bwd: null pointer");
  SB_CHECK_ARG(std::isfinite(abl_weight) && abl_weight >= 0.f, "abl_bwd: abl_weight %g must be finite and >= 0",
               abl_weight);
  const AblGeom g = abl_geom(logits, pitch, N, h, w, C, zoom, lse);
  const AblLayout l = abl_layout(N, g.Hg, g.Wg);
  const long long P = static_cast<long long>(N) * g.Hg * g.Wg;
  const dim3 tiles(cdiv(g.Wg, kAblTile), cdiv(g.Hg, kAblTile), N);
  const unsigned char* code = reinterpret_cast<const unsigned char*>(state + l.code);
  if (zoom == 1) {
    abl_bwd_kernel<<<tiles, kAblThreads, 0, stream>>>(g, code, state + l.wg, loss_info, abl_weight, grad_out, dlogits,
                                                      1);
    SB_LAUNCHED();
    return SEMSEG_OK;
  }
  SB_CUDA(cudaMemsetAsync(workspace, 0, sizeof(float) * P * C, stream));
  abl_bwd_kernel<<<tiles, kAblThreads, 0, stream>>>(g, code, state + l.wg, loss_info, abl_weight, grad_out, workspace,
                                                    0);
  SB_LAUNCHED();
  return launch_bilinear_adjoint(workspace, workspace + P * C, N, h, w, g.Hg, g.Wg, C, zoom, dlogits, stream);
}

extern "C" int semseg_boundary_iou_hist(const void* pred, const void* target, int N, int H, int W, int K,
                                        long long ignore_index, int d, int* workspace, int* counts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(pred && target && workspace && counts, "boundary_iou: null pointer");
  SB_CHECK_ARG(N > 0 && H > 0 && W > 0 && K > 0 && K <= kBiouMaxClasses,
               "boundary_iou: bad sizes (N=%d H=%d W=%d K=%d; K<=%d)", N, H, W, K, kBiouMaxClasses);
  SB_CHECK_ARG(d >= 1, "boundary_iou: band width %d must be >= 1", d);
  const long long P = static_cast<long long>(N) * H * W;
  const long long* p = static_cast<const long long*>(pred);
  const long long* t = static_cast<const long long*>(target);
  SB_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 3 * K, stream));
  biou_rows_kernel<<<static_cast<unsigned>((P + kBiouThreads - 1) / kBiouThreads), kBiouThreads, 0, stream>>>(
      p, t, P, W, d, workspace);
  SB_LAUNCHED();
  long long blocks = (P + kBiouThreads * 8 - 1) / (kBiouThreads * 8);
  blocks = blocks > 132 * 8 ? 132 * 8 : blocks < 1 ? 1 : blocks;
  biou_hist_kernel<<<static_cast<unsigned>(blocks), kBiouThreads, sizeof(int) * 3 * K, stream>>>(
      p, t, workspace, P, H, W, K, d, ignore_index, counts);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

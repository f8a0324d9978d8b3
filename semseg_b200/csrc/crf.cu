// Gated CRF loss (Obukhov et al., 2019; semseg_b200/losses.py GatedCRFLoss): an image-gated pairwise term over a local
// window, on the grid of the fused tail's output (the xZ-upsampled logits) or on the 1/8-resolution logits themselves.
//
// Per grid pixel i with p_i = softmax(s_i), window W(i) = the (2r+1)^2 pixels around i inside the image without i, and
//   k_ij = exp(-|pos_i - pos_j|^2 / (2 sigma_xy^2) - |rgb_i - rgb_j|^2 / (2 sigma_rgb^2)),
//   G_ic = sum_{j in W(i)} k_ij p_jc,   S_i = sum_c p_ic G_ic,   K_i = sum_{j in W(i)} k_ij,
//   CRF  = (1/P) sum_i (K_i - S_i),     dCRF/ds_ic = -(2/P) p_ic (G_ic - S_i)      (k and W are symmetric).
//
// One CTA per 16 x 16 grid tile, one thread per pixel. The tile's rgb features and the spatial table are staged once;
// the probabilities of the tile and its radius-r halo are staged in shared memory one chunk of CC classes at a time,
// recomputed from the 1/8 logits (L2 resident: bilinear xZ with the tail's weights) and the per-pixel lse, so neither
// the full-resolution probabilities, the unfolded window nor a gate table ever exists. The gate k_ij is recomputed per
// class chunk (one MUFU per pixel pair and chunk). The halo probabilities are stored class-group major (float4 of four
// classes per halo pixel) so the lanes of a warp, which read neighbouring halo pixels, hit distinct banks.
// Out-of-image halo pixels carry a huge feature (their gate underflows to exactly 0) and the window centre a spatial
// term of -inf, so W(i) needs no branch.
//
// Forward: per-pixel S_i (kept for the backward) and per-CTA (sum of K_i - S_i, pixels) partials, reduced in fp64 by
// the tail's one-CTA reduce. Backward: G per class chunk again, and scale * p_ic (G_ic - S_i) with
// scale = -2 crf_weight grad_out / P. At zoom 1 (the loss grid is the logits grid) it is added into dlogits; at zoom Z > 1
// it goes to an output-resolution workspace and the bilinear adjoint (a rows pass, then a cols pass that adds into
// dlogits) folds it onto the logits. Every output is written by one thread in a fixed order: no atomics, deterministic.
#include <cmath>

#include "host_common.h"

namespace sb {

constexpr int kCrfTile = 16;                   // grid pixels per tile side
constexpr int kCrfThreads = kCrfTile * kCrfTile;
constexpr int kCrfMaxRadius = 8;
constexpr int kCrfMaxClasses = 256;
constexpr float kCrfOutside = 1e18f;           // feature of an out-of-image halo pixel: its gate is exactly 0

__device__ __forceinline__ float crf_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct CrfGeom {
  const float* logits;  // fp32 NHWC [N, h, w, pitch]
  int pitch, N, h, w, C, zshift;
  int Hg, Wg;           // loss grid: zoom (h-1)+1 x zoom (w-1)+1
  const float* lse;     // [N, Hg, Wg]
  const float* image;   // fp32 NCHW [N, 3, H, W], H = istride (Hg-1)+1
  int H, W, istride;
  float fa[3], fb[3];   // feature = x fa + fb = (x std + mean) / 255 * sqrt(log2 e / (2 sigma_rgb^2))
  float spat;           // -log2 e / (2 sigma_xy^2)
  int radius;
};

// The logit of class c at grid pixel (gy, gx): the tail's bilinear xZ interpolation (align_corners, Z = 1 << zshift).
__device__ __forceinline__ float crf_logit(const CrfGeom& g, int n, int gy, int gx, int c) {
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

// Shared memory: [CC/4][HP] float4 probabilities, [HP] float4 features, [(2r+1)^2] spatial log2-gates.
template <int CC>
__device__ __forceinline__ void crf_stage_chunk(const CrfGeom& g, int n, int ty0, int tx0, int HW, int HP, int c0,
                                                float4* sp) {
  float* spf = reinterpret_cast<float*>(sp);
  for (int idx = threadIdx.x; idx < HP * CC; idx += kCrfThreads) {
    const int hp = idx / CC, cl = idx - hp * CC;
    const int gy = ty0 - g.radius + hp / HW, gx = tx0 - g.radius + hp % HW;
    const int c = c0 + cl;
    float p = 0.f;
    if (c < g.C && gy >= 0 && gy < g.Hg && gx >= 0 && gx < g.Wg) {
      const float l = g.lse[(static_cast<size_t>(n) * g.Hg + gy) * g.Wg + gx];
      p = expf(crf_logit(g, n, gy, gx, c) - l);
    }
    spf[((cl >> 2) * HP + hp) * 4 + (cl & 3)] = p;
  }
}

__device__ __forceinline__ void crf_stage_features(const CrfGeom& g, int n, int ty0, int tx0, int HW, int HP,
                                                   float4* sf, float* st) {
  const size_t plane = static_cast<size_t>(g.H) * g.W;
  const float* img = g.image + static_cast<size_t>(n) * 3 * plane;
  for (int hp = threadIdx.x; hp < HP; hp += kCrfThreads) {
    const int gy = ty0 - g.radius + hp / HW, gx = tx0 - g.radius + hp % HW;
    float4 f = make_float4(kCrfOutside, kCrfOutside, kCrfOutside, 0.f);
    if (gy >= 0 && gy < g.Hg && gx >= 0 && gx < g.Wg) {
      const size_t o = static_cast<size_t>(gy) * g.istride * g.W + static_cast<size_t>(gx) * g.istride;
      f.x = fmaf(img[o], g.fa[0], g.fb[0]);
      f.y = fmaf(img[plane + o], g.fa[1], g.fb[1]);
      f.z = fmaf(img[2 * plane + o], g.fa[2], g.fb[2]);
    }
    sf[hp] = f;
  }
  const int D = 2 * g.radius + 1;
  for (int d = threadIdx.x; d < D * D; d += kCrfThreads) {
    const int dy = d / D - g.radius, dx = d % D - g.radius;
    st[d] = (dy == 0 && dx == 0) ? -INFINITY : static_cast<float>(dy * dy + dx * dx) * g.spat;
  }
}

// acc[c] = sum_{j in W(i)} k_ij p_jc for the staged chunk; returns K_i.
template <int CC>
__device__ __forceinline__ float crf_window(const CrfGeom& g, int ty, int tx, int HW, int HP, const float4* sp,
                                            const float4* sf, const float* st, float* acc) {
  const float4 fi = sf[(ty + g.radius) * HW + tx + g.radius];
  float ksum = 0.f;
  const int D = 2 * g.radius + 1;
#pragma unroll
  for (int c = 0; c < CC; ++c) acc[c] = 0.f;
  for (int dy = 0; dy < D; ++dy) {
    const int base = (ty + dy) * HW + tx;
    const float* trow = st + dy * D;
    for (int dx = 0; dx < D; ++dx) {
      const int hp = base + dx;
      const float4 fj = sf[hp];
      const float a = fi.x - fj.x, b = fi.y - fj.y, e = fi.z - fj.z;
      const float k = crf_ex2(trow[dx] - fmaf(a, a, fmaf(b, b, e * e)));
      ksum += k;
#pragma unroll
      for (int q = 0; q < CC / 4; ++q) {
        const float4 p = sp[q * HP + hp];
        acc[4 * q + 0] = fmaf(k, p.x, acc[4 * q + 0]);
        acc[4 * q + 1] = fmaf(k, p.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(k, p.z, acc[4 * q + 2]);
        acc[4 * q + 3] = fmaf(k, p.w, acc[4 * q + 3]);
      }
    }
  }
  return ksum;
}

__device__ __forceinline__ float crf_own_p(const float4* sp, int HP, int hp, int cl) {
  return reinterpret_cast<const float*>(sp)[((cl >> 2) * HP + hp) * 4 + (cl & 3)];
}

template <int CC>
__global__ void __launch_bounds__(kCrfThreads)
gated_crf_fwd_kernel(CrfGeom g, float* __restrict__ s_out, float* __restrict__ partial) {
  extern __shared__ float4 smem4[];
  const int HW = kCrfTile + 2 * g.radius, HP = HW * HW;
  float4* sp = smem4;
  float4* sf = sp + (CC / 4) * HP;
  float* st = reinterpret_cast<float*>(sf + HP);
  __shared__ float red_loss[kCrfThreads / 32];
  __shared__ float red_cnt[kCrfThreads / 32];
  const int n = blockIdx.z, ty0 = blockIdx.y * kCrfTile, tx0 = blockIdx.x * kCrfTile;
  const int ty = threadIdx.x / kCrfTile, tx = threadIdx.x % kCrfTile;
  const int gy = ty0 + ty, gx = tx0 + tx;
  const bool inside = gy < g.Hg && gx < g.Wg;
  const int own = (ty + g.radius) * HW + tx + g.radius;
  crf_stage_features(g, n, ty0, tx0, HW, HP, sf, st);
  float acc[CC];
  float ksum = 0.f, S = 0.f;
  for (int c0 = 0; c0 < g.C; c0 += CC) {
    __syncthreads();  // the previous chunk's readers are done (and, first time, the features are staged)
    crf_stage_chunk<CC>(g, n, ty0, tx0, HW, HP, c0, sp);
    __syncthreads();
    const float k = crf_window<CC>(g, ty, tx, HW, HP, sp, sf, st, acc);
    if (c0 == 0) ksum = k;
#pragma unroll
    for (int c = 0; c < CC; ++c) S = fmaf(crf_own_p(sp, HP, own, c), acc[c], S);  // padded classes have p = 0
  }
  float loss = 0.f, cnt = 0.f;
  if (inside) {
    s_out[(static_cast<size_t>(n) * g.Hg + gy) * g.Wg + gx] = S;
    loss = ksum - S;
    cnt = 1.f;
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
    for (int i = 0; i < kCrfThreads / 32; ++i) {
      l += red_loss[i];
      c += red_cnt[i];
    }
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * b] = l;
    partial[2 * b + 1] = c;
  }
}

// out[(n, gy, gx) * C + c] (accumulate: += into dlogits, pitch C; else =) of scale * grad_out * p (G - S).
template <int CC>
__global__ void __launch_bounds__(kCrfThreads)
gated_crf_bwd_kernel(CrfGeom g, const float* __restrict__ s_in, float scale, const float* __restrict__ grad_out,
                     float* __restrict__ out, int accumulate) {
  extern __shared__ float4 smem4[];
  const int HW = kCrfTile + 2 * g.radius, HP = HW * HW;
  float4* sp = smem4;
  float4* sf = sp + (CC / 4) * HP;
  float* st = reinterpret_cast<float*>(sf + HP);
  const int n = blockIdx.z, ty0 = blockIdx.y * kCrfTile, tx0 = blockIdx.x * kCrfTile;
  const int ty = threadIdx.x / kCrfTile, tx = threadIdx.x % kCrfTile;
  const int gy = ty0 + ty, gx = tx0 + tx;
  const bool inside = gy < g.Hg && gx < g.Wg;
  const int own = (ty + g.radius) * HW + tx + g.radius;
  const size_t pix = (static_cast<size_t>(n) * g.Hg + min(gy, g.Hg - 1)) * g.Wg + min(gx, g.Wg - 1);
  const float S = s_in[pix];
  const float gs = scale * grad_out[0];
  crf_stage_features(g, n, ty0, tx0, HW, HP, sf, st);
  float acc[CC];
  for (int c0 = 0; c0 < g.C; c0 += CC) {
    __syncthreads();
    crf_stage_chunk<CC>(g, n, ty0, tx0, HW, HP, c0, sp);
    __syncthreads();
    crf_window<CC>(g, ty, tx, HW, HP, sp, sf, st, acc);
    if (inside) {
      float* o = out + pix * g.C + c0;
#pragma unroll
      for (int c = 0; c < CC; ++c) {
        if (c0 + c < g.C) {
          const float d = gs * (crf_own_p(sp, HP, own, c) * (acc[c] - S));
          o[c] = accumulate ? o[c] + d : d;
        }
      }
    }
  }
}

// lse of the logits at every node (the loss grid of at='logits'): two class passes, expf / logf.
__global__ void __launch_bounds__(256)
gated_crf_lse_kernel(const float* __restrict__ logits, int pitch, long long M, int C, float* __restrict__ lse) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float* v = logits + i * pitch;
  float m = -INFINITY;
  for (int c = 0; c < C; ++c) m = fmaxf(m, v[c]);
  float s = 0.f;
  for (int c = 0; c < C; ++c) s += expf(v[c] - m);
  lse[i] = m + logf(s);
}

// Bilinear adjoint, rows: T[n][y][X][c] = sum_Y (1 - |Y - yZ| / Z) D[n][Y][X][c] over the output rows of node row y.
__global__ void __launch_bounds__(256)
gated_crf_adjoint_rows_kernel(const float* __restrict__ D, int N, int h, int Hg, int Wg, int C, int Z,
                              float* __restrict__ T) {
  const long long total = static_cast<long long>(N) * h * Wg * C;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long rowlen = static_cast<long long>(Wg) * C;
  const long long xc = i % rowlen;
  const int y = static_cast<int>((i / rowlen) % h);
  const int n = static_cast<int>(i / (rowlen * h));
  const float step = 1.f / Z;
  const int y0 = max(0, (y - 1) * Z + 1), y1 = min(Hg - 1, (y + 1) * Z - 1);
  float acc = 0.f;
  for (int Y = y0; Y <= y1; ++Y)
    acc = fmaf(1.f - static_cast<float>(abs(Y - y * Z)) * step, D[(static_cast<long long>(n) * Hg + Y) * rowlen + xc],
               acc);
  T[i] = acc;
}

// Bilinear adjoint, cols: dlogits[n][y][x][c] += sum_X (1 - |X - xZ| / Z) T[n][y][X][c].
__global__ void __launch_bounds__(256)
gated_crf_adjoint_cols_kernel(const float* __restrict__ T, int N, int h, int w, int Wg, int C, int Z,
                              float* __restrict__ dlogits) {
  const long long total = static_cast<long long>(N) * h * w * C;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % C);
  const int x = static_cast<int>((i / C) % w);
  const long long ny = i / (static_cast<long long>(C) * w);
  const float step = 1.f / Z;
  const int x0 = max(0, (x - 1) * Z + 1), x1 = min(Wg - 1, (x + 1) * Z - 1);
  const float* t = T + ny * Wg * C + c;
  float acc = 0.f;
  for (int X = x0; X <= x1; ++X)
    acc = fmaf(1.f - static_cast<float>(abs(X - x * Z)) * step, t[static_cast<long long>(X) * C], acc);
  dlogits[i] += acc;
}

// The two adjoint passes above, for the other translation units too (csrc/boundary.cu).
int launch_bilinear_adjoint(const float* D, float* T, int N, int h, int w, int Hg, int Wg, int C, int zoom,
                            float* dlogits, cudaStream_t stream) {
  const long long rows = static_cast<long long>(N) * h * Wg * C, cols = static_cast<long long>(N) * h * w * C;
  gated_crf_adjoint_rows_kernel<<<static_cast<unsigned>((rows + 255) / 256), 256, 0, stream>>>(D, N, h, Hg, Wg, C,
                                                                                              zoom, T);
  SB_LAUNCHED();
  gated_crf_adjoint_cols_kernel<<<static_cast<unsigned>((cols + 255) / 256), 256, 0, stream>>>(T, N, h, w, Wg, C,
                                                                                              zoom, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

}  // namespace sb

using namespace sb;

namespace {

int crf_chunk(int C) { return C <= 4 ? 4 : C <= 8 ? 8 : C <= 16 ? 16 : C <= 24 ? 24 : 32; }

size_t crf_smem(int CC, int radius) {
  const size_t HP = static_cast<size_t>(kCrfTile + 2 * radius) * (kCrfTile + 2 * radius);
  const size_t D = 2 * radius + 1;
  return (CC / 4) * HP * sizeof(float4) + HP * sizeof(float4) + D * D * sizeof(float);
}

int grid_size(int n, int zoom) { return zoom * (n - 1) + 1; }

bool finite_pos(float v) { return std::isfinite(v) && v > 0.f; }

int check_crf(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* image, int H, int W,
              int istride, int radius, float sigma_xy, float sigma_rgb, const float* mean, const float* std_) {
  SB_CHECK_ARG(zoom == 1 || zoom == 2 || zoom == 4 || zoom == 8, "gated_crf: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(logits && image, "gated_crf: null pointer");
  SB_CHECK_ARG(N > 0 && h > 0 && w > 0 && C > 0 && C <= kCrfMaxClasses && pitch >= C,
               "gated_crf: bad sizes (N=%d h=%d w=%d C=%d pitch=%d; C<=%d)", N, h, w, C, pitch, kCrfMaxClasses);
  SB_CHECK_ARG(radius >= 1 && radius <= kCrfMaxRadius, "gated_crf: radius %d is not in [1, %d]", radius,
               kCrfMaxRadius);
  SB_CHECK_ARG(finite_pos(sigma_xy) && finite_pos(sigma_rgb), "gated_crf: sigmas must be finite and > 0");
  for (int i = 0; i < 3; ++i)
    SB_CHECK_ARG(std::isfinite(mean[i]) && finite_pos(std_[i]), "gated_crf: mean must be finite and std finite > 0");
  const long long Hg = grid_size(h, zoom), Wg = grid_size(w, zoom);
  SB_CHECK_ARG(Hg <= 65535LL * kCrfTile, "gated_crf: grid height %lld too large", Hg);
  SB_CHECK_ARG(istride >= 1 && H == istride * (Hg - 1) + 1 && W == istride * (Wg - 1) + 1,
               "gated_crf: image %dx%d is not the %lldx%lld grid at stride %d", H, W, Hg, Wg, istride);
  return SEMSEG_OK;
}

CrfGeom make_geom(const float* logits, int pitch, int N, int h, int w, int C, int zoom, const float* lse,
                  const float* image, int H, int W, int istride, int radius, float sigma_xy, float sigma_rgb,
                  const float* mean, const float* std_) {
  CrfGeom g;
  g.logits = logits;
  g.pitch = pitch;
  g.N = N;
  g.h = h;
  g.w = w;
  g.C = C;
  g.zshift = zoom == 1 ? 0 : zoom == 2 ? 1 : zoom == 4 ? 2 : 3;
  g.Hg = grid_size(h, zoom);
  g.Wg = grid_size(w, zoom);
  g.lse = lse;
  g.image = image;
  g.H = H;
  g.W = W;
  g.istride = istride;
  const double f = std::sqrt(1.4426950408889634 / (2.0 * sigma_rgb * sigma_rgb));
  for (int i = 0; i < 3; ++i) {
    g.fa[i] = static_cast<float>(std_[i] / 255.0 * f);
    g.fb[i] = static_cast<float>(mean[i] / 255.0 * f);
  }
  g.spat = static_cast<float>(-1.4426950408889634 / (2.0 * sigma_xy * sigma_xy));
  g.radius = radius;
  return g;
}

long long fwd_ctas(int N, int Hg, int Wg) { return static_cast<long long>(cdiv(Wg, kCrfTile)) * cdiv(Hg, kCrfTile) * N; }

template <int CC, typename Kernel>
int opt_in(Kernel kernel, size_t smem) {
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (smem > 48 * 1024 && (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire))) {
    SB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(crf_smem(CC, kCrfMaxRadius))));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  return SEMSEG_OK;
}

template <int CC>
int launch_crf_fwd(const CrfGeom& g, float* s_out, float* partial, cudaStream_t stream) {
  const size_t smem = crf_smem(CC, g.radius);
  int r = opt_in<CC>(gated_crf_fwd_kernel<CC>, smem);
  if (r) return r;
  gated_crf_fwd_kernel<CC><<<dim3(cdiv(g.Wg, kCrfTile), cdiv(g.Hg, kCrfTile), g.N), kCrfThreads, smem, stream>>>(
      g, s_out, partial);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int CC>
int launch_crf_bwd(const CrfGeom& g, const float* s_in, float scale, const float* grad_out, float* out, int accumulate,
                   cudaStream_t stream) {
  const size_t smem = crf_smem(CC, g.radius);
  int r = opt_in<CC>(gated_crf_bwd_kernel<CC>, smem);
  if (r) return r;
  gated_crf_bwd_kernel<CC><<<dim3(cdiv(g.Wg, kCrfTile), cdiv(g.Hg, kCrfTile), g.N), kCrfThreads, smem, stream>>>(
      g, s_in, scale, grad_out, out, accumulate);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

}  // namespace

extern "C" long long semseg_gated_crf_workspace_floats(int N, int h, int w, int zoom) {
  SB_CHECK_ARG((zoom == 1 || zoom == 2 || zoom == 4 || zoom == 8) && N > 0 && h > 0 && w > 0,
               "gated_crf: bad zoom %d or size", zoom);
  return 2 * fwd_ctas(N, grid_size(h, zoom), grid_size(w, zoom));   // (sum of K - S, pixels) per CTA
}

extern "C" int semseg_gated_crf_fwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom, float* lse,
                                    int compute_lse, const float* image, int H, int W, int istride, int radius,
                                    float sigma_xy, float sigma_rgb, float mean0, float mean1, float mean2, float std0,
                                    float std1, float std2, float* workspace, float* s_out, float* loss_out,
                                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const float mean[3] = {mean0, mean1, mean2}, std_[3] = {std0, std1, std2};
  int r = check_crf(logits, pitch, N, h, w, C, zoom, image, H, W, istride, radius, sigma_xy, sigma_rgb, mean, std_);
  if (r) return r;
  SB_CHECK_ARG(lse && workspace && s_out && loss_out, "gated_crf_fwd: null pointer");
  SB_CHECK_ARG(!compute_lse || zoom == 1, "gated_crf_fwd: the lse is computed only on the logits grid (zoom 1)");
  const CrfGeom g = make_geom(logits, pitch, N, h, w, C, zoom, lse, image, H, W, istride, radius, sigma_xy, sigma_rgb,
                              mean, std_);
  if (compute_lse) {
    const long long M = static_cast<long long>(N) * h * w;
    gated_crf_lse_kernel<<<static_cast<unsigned>((M + 255) / 256), 256, 0, stream>>>(logits, pitch, M, C, lse);
    SB_LAUNCHED();
  }
  switch (crf_chunk(C)) {
    case 4: r = launch_crf_fwd<4>(g, s_out, workspace, stream); break;
    case 8: r = launch_crf_fwd<8>(g, s_out, workspace, stream); break;
    case 16: r = launch_crf_fwd<16>(g, s_out, workspace, stream); break;
    case 24: r = launch_crf_fwd<24>(g, s_out, workspace, stream); break;
    default: r = launch_crf_fwd<32>(g, s_out, workspace, stream); break;
  }
  if (r) return r;
  return launch_mean_reduce(workspace, static_cast<int>(fwd_ctas(N, g.Hg, g.Wg)), loss_out, stream);
}

extern "C" long long semseg_gated_crf_bwd_workspace_floats(int N, int h, int w, int C, int zoom) {
  SB_CHECK_ARG((zoom == 1 || zoom == 2 || zoom == 4 || zoom == 8) && N > 0 && h > 0 && w > 0 && C > 0,
               "gated_crf: bad zoom %d or size", zoom);
  if (zoom == 1) return 0;                               // added straight into dlogits
  const long long Hg = grid_size(h, zoom), Wg = grid_size(w, zoom);
  return static_cast<long long>(N) * C * Wg * (Hg + h);  // D [N][Hg][Wg][C], then T [N][h][Wg][C]
}

extern "C" int semseg_gated_crf_bwd(const float* logits, int pitch, int N, int h, int w, int C, int zoom,
                                    const float* lse, const float* image, int H, int W, int istride, int radius,
                                    float sigma_xy, float sigma_rgb, float mean0, float mean1, float mean2, float std0,
                                    float std1, float std2, const float* s_in, float crf_weight,
                                    const float* grad_out, float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const float mean[3] = {mean0, mean1, mean2}, std_[3] = {std0, std1, std2};
  int r = check_crf(logits, pitch, N, h, w, C, zoom, image, H, W, istride, radius, sigma_xy, sigma_rgb, mean, std_);
  if (r) return r;
  SB_CHECK_ARG(lse && s_in && grad_out && dlogits && (zoom == 1 || workspace), "gated_crf_bwd: null pointer");
  SB_CHECK_ARG(std::isfinite(crf_weight) && crf_weight >= 0.f, "gated_crf_bwd: crf_weight %g must be finite and >= 0",
               crf_weight);
  const CrfGeom g = make_geom(logits, pitch, N, h, w, C, zoom, lse, image, H, W, istride, radius, sigma_xy, sigma_rgb,
                              mean, std_);
  const double P = static_cast<double>(N) * g.Hg * g.Wg;
  const float scale = static_cast<float>(-2.0 * crf_weight / P);
  float* out = zoom == 1 ? dlogits : workspace;
  const int acc = zoom == 1;
  switch (crf_chunk(C)) {
    case 4: r = launch_crf_bwd<4>(g, s_in, scale, grad_out, out, acc, stream); break;
    case 8: r = launch_crf_bwd<8>(g, s_in, scale, grad_out, out, acc, stream); break;
    case 16: r = launch_crf_bwd<16>(g, s_in, scale, grad_out, out, acc, stream); break;
    case 24: r = launch_crf_bwd<24>(g, s_in, scale, grad_out, out, acc, stream); break;
    default: r = launch_crf_bwd<32>(g, s_in, scale, grad_out, out, acc, stream); break;
  }
  if (r || zoom == 1) return r;
  return launch_bilinear_adjoint(workspace, workspace + static_cast<long long>(N) * g.Hg * g.Wg * C, N, h, w, g.Hg,
                                 g.Wg, C, zoom, dlogits, stream);
}

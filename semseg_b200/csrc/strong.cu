// The strong view of mean-teacher training (semseg_b200/augment.py StrongAugment): colour jitter, random grayscale and
// Gaussian blur of a normalised fp32 NCHW batch, each image with its own uniforms u[n, 0..11], as
// include/semseg_b200.h semseg_strong_augment states. The chain runs on the de-normalised image v in [0, 1] in fp32
// with torchvision.transforms.v2.functional's float formulas; an image no operation applies to is copied bit for bit.
// Two kernels, both one CTA per (32x32 output tile, image), no atomics, fixed launch geometry:
//   strong_stats: the tile's fp32 sum of gray(v) of the chain state just before contrast, in a fixed order, into
//                 partial[n][tile]; CTAs of images contrast does not apply to exit at once.
//   strong_apply: the image's contrast mean from its partials (fp64, fixed order), the pointwise chain of the tile and,
//                 for a blurred image, its halo of r = ceil(3 sigma) into shared memory, then the separable blur
//                 (rows, then columns; reflect-101 indices) and the re-normalised, coalesced store.
// The per-image parameters (flags, factors, order, sigma and taps) are derived once per CTA by one thread, in fp64
// with explicit round-to-nearest intrinsics (no contraction), so the host-side oracle reproduces them bit for bit.
#include <algorithm>
#include <atomic>
#include <cmath>

#include "host_common.h"

namespace sb {

constexpr int kStrongTile = 32;
constexpr int kStrongThreads = 256;
constexpr int kStrongMaxR = 15;                      // ceil(3 * 5): sigma_hi <= 5

struct StrongArgs {
  double lo[4], hi[4];       // factor ranges: brightness, contrast, saturation, hue
  int on[4];                 // strength > 0
  double p_jitter, p_gray, p_blur, sig_lo, sig_hi;
  int R;                     // ceil(3 sigma_hi): the largest radius
  float mean[3], std[3];
};

struct StrongImg {
  int any;                   // some operation applies: otherwise the image is copied
  int nops, op[4];           // the jitter operations that apply, in order
  float f[4];                // their factors, by operation
  int contrast, gray, r;     // r: blur radius, 0 = no blur
  float m;                   // contrast mean (strong_apply)
  float taps[kStrongMaxR + 1];
};

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }
__device__ __forceinline__ float gray_of(float r, float g, float b) { return 0.2989f * r + 0.587f * g + 0.114f * b; }

__device__ void strong_image(const float* un, const StrongArgs& a, bool taps, StrongImg* P) {
  P->nops = 0;
  P->contrast = 0;
  if (static_cast<double>(un[0]) < a.p_jitter) {
    for (int k = 0; k < 4; ++k) {
      if (!a.on[k]) continue;
      P->f[k] = __double2float_rn(__dadd_rn(a.lo[k], __dmul_rn(__dsub_rn(a.hi[k], a.lo[k]), static_cast<double>(un[1 + k]))));
      int i = P->nops++;     // insertion by (u[5 + k], k) ascending; k grows, so equal keys stay behind
      while (i > 0 && un[5 + P->op[i - 1]] > un[5 + k]) {
        P->op[i] = P->op[i - 1];
        --i;
      }
      P->op[i] = k;
    }
    P->contrast = a.on[1];
  }
  P->gray = static_cast<double>(un[9]) < a.p_gray;
  P->r = 0;
  if (static_cast<double>(un[10]) < a.p_blur) {
    const float sigma =
        __double2float_rn(__dadd_rn(a.sig_lo, __dmul_rn(__dsub_rn(a.sig_hi, a.sig_lo), static_cast<double>(un[11]))));
    const int r = min(static_cast<int>(ceil(__dmul_rn(3.0, static_cast<double>(sigma)))), a.R);
    P->r = r;
    if (taps) {
      const double s2 = __dmul_rn(2.0, __dmul_rn(sigma, sigma));
      double sum = 1.0;
      for (int k = 1; k <= r; ++k) sum += 2.0 * exp(-static_cast<double>(k * k) / s2);
      for (int k = 0; k <= r; ++k) P->taps[k] = static_cast<float>(exp(-static_cast<double>(k * k) / s2) / sum);
    }
  }
  P->any = P->nops > 0 || P->gray || P->r > 0;
}

// torchvision's _rgb_to_hsv, (h + hue) mod 1, _hsv_to_rgb, on one pixel.
__device__ void strong_hue(float& r, float& g, float& b, float hue) {
  const float maxc = fmaxf(r, fmaxf(g, b)), minc = fminf(r, fminf(g, b));
  const bool eqc = maxc == minc;
  const float cr = maxc - minc;
  const float s = cr / (eqc ? 1.f : maxc);
  const float div = eqc ? 1.f : cr;
  const float rc = (maxc - r) / div, gc = (maxc - g) / div, bc = (maxc - b) / div;
  float h;
  if (maxc == r) {
    h = bc - gc;
  } else if (maxc == g) {
    h = (rc + 2.f) - bc;
  } else {
    h = (gc + 4.f) - rc;
  }
  h = fmodf(h * (1.f / 6.f) + 1.f, 1.f);
  h = h + hue;
  h = h - floorf(h);                                   // torch.remainder(h, 1)
  const float v = maxc;
  const float h6 = h * 6.f;
  const float fi = floorf(h6);
  const float f = h6 - fi;
  const int i = static_cast<int>(fi) % 6;
  const float sxf = s * f;
  const float q = clamp01((1.f - sxf) * v);
  const float t = clamp01((sxf + (1.f - s)) * v);
  const float p = clamp01((1.f - s) * v);
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// The chain on one de-normalised pixel; to_contrast: stop just before contrast (the state strong_stats averages).
__device__ __forceinline__ void strong_chain(float& r, float& g, float& b, const StrongImg& P, bool to_contrast) {
  for (int k = 0; k < P.nops; ++k) {
    const int op = P.op[k];
    const float f = P.f[op];
    if (op == 0) {
      r = clamp01(f * r);
      g = clamp01(f * g);
      b = clamp01(f * b);
    } else if (op == 1) {
      if (to_contrast) return;
      const float mm = (1.f - f) * P.m;
      r = clamp01(f * r + mm);
      g = clamp01(f * g + mm);
      b = clamp01(f * b + mm);
    } else if (op == 2) {
      const float gg = (1.f - f) * gray_of(r, g, b);
      r = clamp01(f * r + gg);
      g = clamp01(f * g + gg);
      b = clamp01(f * b + gg);
    } else {
      strong_hue(r, g, b, f);
    }
  }
  if (P.gray) r = g = b = gray_of(r, g, b);
}

__device__ __forceinline__ float denorm(float x, const StrongArgs& a, int c) {
  return clamp01((x * a.std[c] + a.mean[c]) / 255.f);
}

__device__ __forceinline__ float renorm(float v, const StrongArgs& a, int c) { return (255.f * v - a.mean[c]) / a.std[c]; }

__device__ __forceinline__ int reflect101(int i, int n) {
  i = i < 0 ? -i : i;
  i = i >= n ? 2 * (n - 1) - i : i;
  return min(max(i, 0), n - 1);                        // only halo positions no output reads fall outside
}

__global__ void __launch_bounds__(kStrongThreads)
strong_stats_kernel(const float* __restrict__ x, int H, int W, int tiles_x, const float* __restrict__ u, int ustride,
                    StrongArgs a, float* __restrict__ partial) {
  __shared__ StrongImg P;
  __shared__ float s_w[kStrongThreads / 32];
  const int n = blockIdx.y, tid = threadIdx.x;
  if (tid == 0) strong_image(u + static_cast<size_t>(n) * ustride, a, false, &P);
  __syncthreads();
  if (!P.contrast) return;
  const int ty0 = blockIdx.x / tiles_x * kStrongTile, tx0 = blockIdx.x % tiles_x * kStrongTile;
  const size_t plane = static_cast<size_t>(H) * W;
  const float* xn = x + static_cast<size_t>(n) * 3 * plane;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < kStrongTile * kStrongTile / kStrongThreads; ++k) {
    const int idx = tid + k * kStrongThreads;
    const int gy = ty0 + (idx >> 5), gx = tx0 + (idx & 31);
    if (gy < H && gx < W) {
      const size_t o = static_cast<size_t>(gy) * W + gx;
      float r = denorm(xn[o], a, 0), g = denorm(xn[plane + o], a, 1), b = denorm(xn[2 * plane + o], a, 2);
      strong_chain(r, g, b, P, true);
      acc += gray_of(r, g, b);
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, s);
  if ((tid & 31) == 0) s_w[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
    for (int w = 0; w < kStrongThreads / 32; ++w) t += s_w[w];
    partial[static_cast<size_t>(n) * gridDim.x + blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kStrongThreads)
strong_apply_kernel(const float* __restrict__ x, int H, int W, int tiles_x, const float* __restrict__ u, int ustride,
                    StrongArgs a, const float* __restrict__ partial, float* __restrict__ out) {
  extern __shared__ float S[];                         // [3][SR][SR] chain values, then [3][SR][32] row-blurred
  __shared__ StrongImg P;
  const int n = blockIdx.y, tid = threadIdx.x;
  if (tid == 0) strong_image(u + static_cast<size_t>(n) * ustride, a, true, &P);
  __syncthreads();
  if (P.contrast && tid < 32) {
    const float* pn = partial + static_cast<size_t>(n) * gridDim.x;
    double s = 0.0;
    for (int t = tid; t < static_cast<int>(gridDim.x); t += 32) s += static_cast<double>(pn[t]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (tid == 0) P.m = static_cast<float>(s / (static_cast<double>(H) * W));
  }
  __syncthreads();
  const int ty0 = blockIdx.x / tiles_x * kStrongTile, tx0 = blockIdx.x % tiles_x * kStrongTile;
  const size_t plane = static_cast<size_t>(H) * W;
  const float* xn = x + static_cast<size_t>(n) * 3 * plane;
  float* on = out + static_cast<size_t>(n) * 3 * plane;
  const int r = P.r;
  if (r == 0) {                                        // no blur: pointwise, or a copy
#pragma unroll
    for (int k = 0; k < kStrongTile * kStrongTile / kStrongThreads; ++k) {
      const int idx = tid + k * kStrongThreads;
      const int gy = ty0 + (idx >> 5), gx = tx0 + (idx & 31);
      if (gy < H && gx < W) {
        const size_t o = static_cast<size_t>(gy) * W + gx;
        float r0 = xn[o], g0 = xn[plane + o], b0 = xn[2 * plane + o];
        if (P.any) {
          r0 = denorm(r0, a, 0);
          g0 = denorm(g0, a, 1);
          b0 = denorm(b0, a, 2);
          strong_chain(r0, g0, b0, P, false);
          r0 = renorm(r0, a, 0);
          g0 = renorm(g0, a, 1);
          b0 = renorm(b0, a, 2);
        }
        on[o] = r0;
        on[plane + o] = g0;
        on[2 * plane + o] = b0;
      }
    }
    return;
  }
  const int SR = kStrongTile + 2 * r;
  float* V = S;                                        // [3][SR][SR]
  float* T = S + 3 * SR * SR;                          // [3][SR][32]
  for (int idx = tid; idx < SR * SR; idx += kStrongThreads) {
    const int i = idx / SR, j = idx - i * SR;
    const int gy = reflect101(ty0 - r + i, H), gx = reflect101(tx0 - r + j, W);
    const size_t o = static_cast<size_t>(gy) * W + gx;
    float r0 = denorm(xn[o], a, 0), g0 = denorm(xn[plane + o], a, 1), b0 = denorm(xn[2 * plane + o], a, 2);
    strong_chain(r0, g0, b0, P, false);
    V[idx] = r0;
    V[SR * SR + idx] = g0;
    V[2 * SR * SR + idx] = b0;
  }
  __syncthreads();
  for (int idx = tid; idx < SR * kStrongTile; idx += kStrongThreads) {
    const int i = idx >> 5, j = idx & 31;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float* row = V + c * SR * SR + i * SR + j + r;
      float acc = P.taps[0] * row[0];
      for (int k = 1; k <= r; ++k) acc += P.taps[k] * (row[-k] + row[k]);
      T[c * SR * kStrongTile + idx] = acc;
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kStrongTile * kStrongTile / kStrongThreads; ++k) {
    const int idx = tid + k * kStrongThreads;
    const int i = idx >> 5, j = idx & 31;
    const int gy = ty0 + i, gx = tx0 + j;
    if (gy < H && gx < W) {
      const size_t o = static_cast<size_t>(gy) * W + gx;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float* col = T + c * SR * kStrongTile + (i + r) * kStrongTile + j;
        float acc = P.taps[0] * col[0];
        for (int t = 1; t <= r; ++t) acc += P.taps[t] * (col[-t * kStrongTile] + col[t * kStrongTile]);
        on[c * plane + o] = renorm(acc, a, c);
      }
    }
  }
}

static size_t strong_smem_bytes(int R) {
  const size_t SR = kStrongTile + 2 * R;
  return 3 * (SR * SR + SR * kStrongTile) * sizeof(float);
}

// The opt-in to more than 48 KB of dynamic shared memory is per device: made once for every device this process uses,
// to the largest size (R = 15), before the first launch on that device that needs it.
static std::atomic<bool> g_strong_attr[64];

static int strong_opt_in(size_t smem) {
  if (smem <= 48 * 1024) return SEMSEG_OK;
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !g_strong_attr[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(strong_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(strong_smem_bytes(kStrongMaxR))));
    if (dev >= 0 && dev < 64) g_strong_attr[dev].store(true, std::memory_order_release);
  }
  return SEMSEG_OK;
}

}  // namespace sb

using namespace sb;

extern "C" int semseg_strong_augment(const float* x, int N, int C, int H, int W, const float* uniforms, int ustride,
                                     double brightness, double contrast, double saturation, double hue,
                                     double p_jitter, double p_gray, double p_blur, double sigma_lo, double sigma_hi,
                                     const float* mean3, const float* std3, float* workspace, float* out,
                                     void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && uniforms && mean3 && std3 && workspace && out, "strong_augment: null pointer");
  SB_CHECK_ARG(static_cast<const void*>(x) != static_cast<const void*>(out),
               "strong_augment: the view cannot overwrite its source");
  SB_CHECK_ARG(C == 3, "strong_augment: %d channels, RGB (3) expected", C);
  SB_CHECK_ARG(N > 0 && N <= 65535, "strong_augment: batch of %d images (1..65535)", N);
  SB_CHECK_ARG(ustride >= 12, "strong_augment: uniform row stride %d below 12", ustride);
  const double s[4] = {brightness, contrast, saturation, hue};
  for (int k = 0; k < 4; ++k)
    SB_CHECK_ARG(std::isfinite(s[k]) && s[k] >= 0.0, "strong_augment: strength %g must be finite and >= 0", s[k]);
  SB_CHECK_ARG(hue <= 0.5, "strong_augment: hue %g above 0.5", hue);
  const double p[3] = {p_jitter, p_gray, p_blur};
  for (int k = 0; k < 3; ++k)
    SB_CHECK_ARG(std::isfinite(p[k]) && p[k] >= 0.0 && p[k] <= 1.0, "strong_augment: probability %g outside [0, 1]",
                 p[k]);
  SB_CHECK_ARG(std::isfinite(sigma_lo) && std::isfinite(sigma_hi) && sigma_lo > 0.0 && sigma_lo <= sigma_hi &&
                   sigma_hi <= 5.0,
               "strong_augment: sigma (%g, %g) needs 0 < lo <= hi <= 5", sigma_lo, sigma_hi);
  for (int c = 0; c < 3; ++c) {
    SB_CHECK_ARG(std::isfinite(mean3[c]), "strong_augment: mean[%d] is not finite", c);
    SB_CHECK_ARG(std::isfinite(std3[c]) && std3[c] > 0.f, "strong_augment: std[%d] = %g must be > 0", c,
                 static_cast<double>(std3[c]));
  }
  const int R = static_cast<int>(std::ceil(3.0 * sigma_hi));
  SB_CHECK_ARG(H > R && W > R, "strong_augment: %dx%d image needs H, W > ceil(3 sigma_hi) = %d", H, W, R);
  const long long tiles_x = (W + kStrongTile - 1) / kStrongTile, tiles = tiles_x * ((H + kStrongTile - 1) / kStrongTile);
  SB_CHECK_ARG(tiles < (1LL << 31), "strong_augment: image too large");
  StrongArgs a;
  a.lo[0] = std::max(0.0, 1.0 - brightness);
  a.hi[0] = 1.0 + brightness;
  a.lo[1] = std::max(0.0, 1.0 - contrast);
  a.hi[1] = 1.0 + contrast;
  a.lo[2] = std::max(0.0, 1.0 - saturation);
  a.hi[2] = 1.0 + saturation;
  a.lo[3] = -hue;
  a.hi[3] = hue;
  for (int k = 0; k < 4; ++k) a.on[k] = s[k] > 0.0;
  a.p_jitter = p_jitter;
  a.p_gray = p_gray;
  a.p_blur = p_blur;
  a.sig_lo = sigma_lo;
  a.sig_hi = sigma_hi;
  a.R = R;
  for (int c = 0; c < 3; ++c) {
    a.mean[c] = mean3[c];
    a.std[c] = std3[c];
  }
  const size_t smem = strong_smem_bytes(R);
  if (strong_opt_in(smem) != SEMSEG_OK) return SEMSEG_E_CUDA;
  const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>(N));
  strong_stats_kernel<<<grid, kStrongThreads, 0, stream>>>(x, H, W, static_cast<int>(tiles_x), uniforms, ustride, a,
                                                           workspace);
  SB_LAUNCHED();
  strong_apply_kernel<<<grid, kStrongThreads, smem, stream>>>(x, H, W, static_cast<int>(tiles_x), uniforms, ustride, a,
                                                              workspace, out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

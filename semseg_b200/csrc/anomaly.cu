// Anomaly (out-of-distribution) segmentation on the sliding-window scores (semseg_b200/anomaly.py). Three parts:
//
// Class moments (semseg_anomaly_class_moments): sum ML, sum ML^2 and the pixel count per predicted class, added into a
// caller-owned fp64 [3][C]. One CTA per tile of kMomTile pixels stages the tile's predictions and ML values in shared
// memory; thread c sums class c over the tile in pixel order -> partial[tile][3][C]. One final CTA adds the partials
// per class in tile order. No float atomics: the result does not depend on scheduling.
//
// SML post-processing (semseg_anomaly_sml; standardized max-logit, Jung et al., ICCV 2021, as defined in anomaly.py):
//   standardise : S = (ML - mean[pred]) / std[pred] in fp64;
//   boundaries  : per suppression iteration i, width r_i = r0 - i floor(r0 / n); a pixel is a boundary pixel if the
//                 (2 r_i + 1)^2 window around it, clipped to the image, holds another prediction. Separable: a row pass
//                 (clipped window min / max of pred) and a column pass over its result (-> one flag byte per pixel);
//   suppression : a boundary pixel takes the mean of the previous map over the non-boundary pixels of its clipped 3x3
//                 neighbourhood (row-major order), or keeps its value if there are none; Jacobi, ping-pong between two
//                 fp64 planes;
//   smoothing   : one dilated Gaussian pass, weights exp(-a^2 / 2 sigma^2) exp(-b^2 / 2 sigma^2) passed by value, taps
//                 outside the image dropped and the weights renormalised over the rest; the result is negated and
//                 rounded to fp32 (higher = more anomalous).
// Nothing is read back to the host.
//
// Metrics (semseg_anomaly_metrics): AUROC, AP and FPR at 95 % TPR of scores against 0 / 1 labels, ties grouped.
//   keys    : scores -> order-preserving uint32 keys, complemented so that the ascending radix sort yields descending
//             scores (-0.0 folded into +0.0); payload 0 = inlier, 1 = anomaly, 2 = void. A label other than 0, 1 or
//             ignore_index, or a non-finite score on a non-void pixel, sets an error bit (integer atomicOr);
//   sort    : semseg_segsort_u32_pairs, one segment (csrc/segsort.cu);
//   groups  : the tiled integer scan of csrc/densecrf.cu's unique pass, over three counts at once (group ends,
//             anomalies, inliers): per tile counts, a single-CTA exclusive scan of the tile counts, then each group's
//             inclusive cumulative (TP_g, FP_g), written at its index g by the group's last pixel;
//   terms   : over the groups, in a fixed grid: the Mann-Whitney numerator sum_g (FP_g - FP_g-1)(TP_g-1 + TP_g) exactly
//             in uint64, AP's sum_g (TP_g - TP_g-1) TP_g / (TP_g + FP_g) in fp64 (fixed-order tree per CTA), and the
//             first g with 20 TP_g >= 19 P (integer atomicMin); a single CTA finishes in a fixed order.
// Three doubles (AUROC, AP, FPR95) and three integers (positives, negatives, error bits) are the results; the counts
// are integers throughout, so the metrics are deterministic.
#include <float.h>
#include <limits.h>
#include <math.h>
#include <math_constants.h>

#include "host_common.h"

namespace sb {

constexpr int kMomThreads = 256;
constexpr int kMomTile = 2048;                     // pixels per moments CTA (24 KB of shared memory)
constexpr int kMomMaxClasses = 4096;
constexpr int kSmlThreads = 256;
constexpr int kSmlMaxKernel = 63;                  // smooth_kernel limit: the 1-D weights are passed by value
constexpr int kMetThreads = 256;
constexpr int kMetItems = 16;                      // sorted pixels per thread in the group scan
constexpr int kMetTile = kMetThreads * kMetItems;
constexpr int kMetScanThreads = 1024;
constexpr int kMetTermCtas = 264;                  // fixed grid of the terms pass (2 per SM of an H100 SXM)

// ------------------------------------------------------------------------------------------------ class moments
__global__ void __launch_bounds__(kMomThreads)
anomaly_moments_tile_kernel(const long long* __restrict__ pred, const double* __restrict__ ml, long long P, int C,
                            double* __restrict__ partial) {
  __shared__ int sp[kMomTile];
  __shared__ double sv[kMomTile];
  const long long base = static_cast<long long>(blockIdx.x) * kMomTile;
  const int n = static_cast<int>(min(static_cast<long long>(kMomTile), P - base));
  for (int i = threadIdx.x; i < n; i += kMomThreads) {
    const long long c = pred[base + i];
    sp[i] = (c >= 0 && c < C) ? static_cast<int>(c) : -1;
    sv[i] = ml[base + i];
  }
  __syncthreads();
  double* out = partial + static_cast<size_t>(blockIdx.x) * 3 * C;
  for (int c = threadIdx.x; c < C; c += kMomThreads) {
    double s = 0.0, s2 = 0.0, k = 0.0;
    for (int i = 0; i < n; ++i)
      if (sp[i] == c) {
        const double v = sv[i];
        s += v;
        s2 = fma(v, v, s2);
        k += 1.0;
      }
    out[c] = s;
    out[C + c] = s2;
    out[2 * C + c] = k;
  }
}

__global__ void __launch_bounds__(kMomThreads)
anomaly_moments_final_kernel(const double* __restrict__ partial, int tiles, int C, double* __restrict__ moments) {
  for (int j = blockIdx.x * kMomThreads + threadIdx.x; j < 3 * C; j += gridDim.x * kMomThreads) {
    double s = 0.0;
    for (int t = 0; t < tiles; ++t) s += partial[static_cast<size_t>(t) * 3 * C + j];
    moments[j] += s;
  }
}

// ------------------------------------------------------------------------------------------------ SML
struct SmoothWeights {
  double w[kSmlMaxKernel];   // w[a + k/2] = exp(-a^2 / (2 sigma^2))
};

__global__ void __launch_bounds__(kSmlThreads)
sml_standardise_kernel(const double* __restrict__ ml, const long long* __restrict__ pred, long long P, int C,
                       const double* __restrict__ mean, const double* __restrict__ stdv, double* __restrict__ S) {
  const long long i = static_cast<long long>(blockIdx.x) * kSmlThreads + threadIdx.x;
  if (i >= P) return;
  const long long c = pred[i];
  S[i] = (c >= 0 && c < C) ? (ml[i] - mean[c]) / stdv[c] : CUDART_NAN;
}

// mm[0][p] / mm[1][p] = min / max of pred over the row window [x - r, x + r] clipped to the image.
__global__ void __launch_bounds__(kSmlThreads)
sml_rows_kernel(const long long* __restrict__ pred, long long P, int W, int r, long long* __restrict__ mm) {
  const long long i = static_cast<long long>(blockIdx.x) * kSmlThreads + threadIdx.x;
  if (i >= P) return;
  const int x = static_cast<int>(i % W);
  const long long row = i - x;
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  for (int xx = max(0, x - r); xx <= min(W - 1, x + r); ++xx) {
    const long long v = pred[row + xx];
    lo = min(lo, v);
    hi = max(hi, v);
  }
  mm[i] = lo;
  mm[P + i] = hi;
}

// edge[p] = 1 if the clipped (2r+1)^2 window holds two different predictions: the column window over the row minima and
// maxima.
__global__ void __launch_bounds__(kSmlThreads)
sml_cols_kernel(const long long* __restrict__ mm, long long P, int H, int W, int r, unsigned char* __restrict__ edge) {
  const long long i = static_cast<long long>(blockIdx.x) * kSmlThreads + threadIdx.x;
  if (i >= P) return;
  const int x = static_cast<int>(i % W), y = static_cast<int>(i / W);
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  for (int yy = max(0, y - r); yy <= min(H - 1, y + r); ++yy) {
    const long long q = static_cast<long long>(yy) * W + x;
    lo = min(lo, mm[q]);
    hi = max(hi, mm[P + q]);
  }
  edge[i] = lo != hi;
}

// One Jacobi suppression step: boundary pixels take the mean of `in` over the non-boundary pixels of their clipped 3x3
// neighbourhood (row-major order), or keep their value.
__global__ void __launch_bounds__(kSmlThreads)
sml_suppress_kernel(const double* __restrict__ in, const unsigned char* __restrict__ edge, long long P, int H, int W,
                    double* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * kSmlThreads + threadIdx.x;
  if (i >= P) return;
  double v = in[i];
  if (edge[i]) {
    const int x = static_cast<int>(i % W), y = static_cast<int>(i / W);
    double s = 0.0;
    int n = 0;
    for (int yy = max(0, y - 1); yy <= min(H - 1, y + 1); ++yy)
      for (int xx = max(0, x - 1); xx <= min(W - 1, x + 1); ++xx) {
        const long long q = static_cast<long long>(yy) * W + xx;
        if (!edge[q]) {
          s += in[q];
          ++n;
        }
      }
    if (n) v = s / n;
  }
  out[i] = v;
}

// out = -(sum_ab g(a,b) S(p + d (a, b)) / sum_ab g(a,b)) over the taps inside the image, rounded to fp32.
__global__ void __launch_bounds__(kSmlThreads)
sml_smooth_kernel(const double* __restrict__ S, long long P, int H, int W, int k, int d,
                  const __grid_constant__ SmoothWeights gw, float* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * kSmlThreads + threadIdx.x;
  if (i >= P) return;
  const int x = static_cast<int>(i % W), y = static_cast<int>(i / W);
  const int half = k / 2;
  double num = 0.0, den = 0.0;
  for (int a = -half; a <= half; ++a) {
    const int yy = y + d * a;
    if (yy < 0 || yy >= H) continue;
    const double wa = gw.w[a + half];
    for (int b = -half; b <= half; ++b) {
      const int xx = x + d * b;
      if (xx < 0 || xx >= W) continue;
      const double g = wa * gw.w[b + half];
      num += g * S[static_cast<long long>(yy) * W + xx];
      den += g;
    }
  }
  out[i] = static_cast<float>(-(num / den));
}

// ------------------------------------------------------------------------------------------------ metrics
enum : int { kErrLabel = 1, kErrScore = 2 };

__global__ void __launch_bounds__(kMetThreads)
metrics_keys_kernel(const float* __restrict__ score, const void* __restrict__ label, int label_bytes, int n,
                    long long ignore, unsigned* __restrict__ keys, unsigned* __restrict__ vals, long long* info) {
  const int i = blockIdx.x * kMetThreads + threadIdx.x;
  if (i >= n) return;
  const long long l = label_bytes == 1 ? static_cast<long long>(static_cast<const unsigned char*>(label)[i])
                                       : static_cast<const long long*>(label)[i];
  const float s = score[i];
  unsigned v = 2u;
  int err = 0;
  if (l != ignore) {
    if (l == 0 || l == 1) v = static_cast<unsigned>(l);
    else err |= kErrLabel;
    if (!isfinite(s)) err |= kErrScore;
  }
  if (err) atomicOr(reinterpret_cast<unsigned long long*>(info + 2), static_cast<unsigned long long>(err));
  unsigned b = __float_as_uint(s + 0.0f);               // -0.0 + 0.0 = +0.0
  b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);      // ascending in the score
  keys[i] = ~b;                                         // descending
  vals[i] = v;
}

__device__ __forceinline__ bool met_end(const unsigned* keys, int n, int i) { return i == n - 1 || keys[i + 1] != keys[i]; }

// Per tile of kMetTile sorted pixels: group ends, anomalies, inliers -> cnt[0..2][tile].
__global__ void __launch_bounds__(kMetThreads)
metrics_count_kernel(const unsigned* __restrict__ keys, const unsigned* __restrict__ vals, int n, int nt,
                     unsigned* __restrict__ cnt) {
  __shared__ unsigned tot[3];
  if (threadIdx.x < 3) tot[threadIdx.x] = 0;
  __syncthreads();
  const int base = blockIdx.x * kMetTile, end = min(base + kMetTile, n);
  unsigned e = 0, p = 0, q = 0;
  for (int i = base + threadIdx.x; i < end; i += kMetThreads) {
    e += met_end(keys, n, i);
    p += vals[i] == 1u;
    q += vals[i] == 0u;
  }
  atomicAdd(&tot[0], e);   // integer: the counts do not depend on the order
  atomicAdd(&tot[1], p);
  atomicAdd(&tot[2], q);
  __syncthreads();
  if (threadIdx.x < 3) cnt[static_cast<size_t>(threadIdx.x) * nt + blockIdx.x] = tot[threadIdx.x];
}

// Exclusive scan of each of the three tile-count rows in place (one CTA, csrc/densecrf.cu's dcrf_scan_tiles_kernel);
// the totals (groups, P, N) -> tot[0..2], P and N also -> info[0..1].
__global__ void __launch_bounds__(kMetScanThreads)
metrics_scan_kernel(unsigned* __restrict__ cnt, int nt, unsigned* __restrict__ tot, long long* __restrict__ info) {
  __shared__ unsigned warp_sum[kMetScanThreads / 32];
  const int chunk = (nt + kMetScanThreads - 1) / kMetScanThreads;
  const int b = min(static_cast<int>(threadIdx.x) * chunk, nt), e = min(b + chunk, nt);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int row = 0; row < 3; ++row) {
    unsigned* c = cnt + static_cast<size_t>(row) * nt;
    unsigned s = 0;
    for (int i = b; i < e; ++i) s += c[i];
    unsigned inc = s;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      unsigned v = warp_sum[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
      }
      warp_sum[lane] = v;
    }
    __syncthreads();
    unsigned r = inc - s + (warp ? warp_sum[warp - 1] : 0u);
    for (int i = b; i < e; ++i) {
      const unsigned x = c[i];
      c[i] = r;
      r += x;
    }
    if (threadIdx.x == kMetScanThreads - 1) {
      tot[row] = warp_sum[31];
      if (row) info[row - 1] = warp_sum[31];
    }
    __syncthreads();
  }
}

// Each thread owns kMetItems consecutive sorted pixels of the tile; the last pixel of group g writes the group's
// inclusive cumulative counts: tp[g], fp[g].
__global__ void __launch_bounds__(kMetThreads)
metrics_groups_kernel(const unsigned* __restrict__ keys, const unsigned* __restrict__ vals, int n, int nt,
                      const unsigned* __restrict__ cnt, unsigned* __restrict__ tp, unsigned* __restrict__ fp) {
  __shared__ unsigned warp_sum[3][kMetThreads / 32];
  const int b = blockIdx.x * kMetTile + threadIdx.x * kMetItems, e = min(b + kMetItems, n);
  unsigned s[3] = {0, 0, 0};
  for (int i = b; i < e; ++i) {
    s[0] += met_end(keys, n, i);
    s[1] += vals[i] == 1u;
    s[2] += vals[i] == 0u;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned run[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    unsigned inc = s[k];
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) warp_sum[k][warp] = inc;
    run[k] = inc - s[k];
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    unsigned before = cnt[static_cast<size_t>(k) * nt + blockIdx.x];
    for (int w = 0; w < warp; ++w) before += warp_sum[k][w];
    run[k] += before;
  }
  for (int i = b; i < e; ++i) {
    run[1] += vals[i] == 1u;
    run[2] += vals[i] == 0u;
    if (met_end(keys, n, i)) {
      tp[run[0]] = run[1];
      fp[run[0]] = run[2];
      ++run[0];
    }
  }
}

// Over the groups g < G (G on the device; a fixed grid strides over them): the Mann-Whitney numerator, the AP sum and
// the first group reaching 95 % TPR -> per-CTA partials.
__global__ void __launch_bounds__(kMetThreads)
metrics_terms_kernel(const unsigned* __restrict__ tp, const unsigned* __restrict__ fp, const unsigned* __restrict__ tot,
                     unsigned long long* __restrict__ auc_part, double* __restrict__ ap_part,
                     int* __restrict__ first95) {
  __shared__ unsigned long long su[kMetThreads];
  __shared__ double sd[kMetThreads];
  const int G = static_cast<int>(tot[0]);
  const unsigned long long P = tot[1];
  unsigned long long auc = 0;
  double ap = 0.0;
  int first = INT_MAX;
  for (int g = blockIdx.x * kMetThreads + threadIdx.x; g < G; g += gridDim.x * kMetThreads) {
    const unsigned t1 = tp[g], f1 = fp[g];
    const unsigned t0 = g ? tp[g - 1] : 0u, f0 = g ? fp[g - 1] : 0u;
    auc += static_cast<unsigned long long>(f1 - f0) * (static_cast<unsigned long long>(t0) + t1);
    if (t1 != t0) ap += static_cast<double>(t1 - t0) * (static_cast<double>(t1) / (static_cast<double>(t1) + f1));
    if (first == INT_MAX && 20ull * t1 >= 19ull * P) first = g;
  }
  if (first != INT_MAX) atomicMin(first95, first);
  su[threadIdx.x] = auc;
  sd[threadIdx.x] = ap;
  __syncthreads();
  for (int o = kMetThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      su[threadIdx.x] += su[threadIdx.x + o];
      sd[threadIdx.x] += sd[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    auc_part[blockIdx.x] = su[0];
    ap_part[blockIdx.x] = sd[0];
  }
}

// out[0..2] = AUROC, AP, FPR95 (NaN without positives or without negatives).
__global__ void __launch_bounds__(kMetThreads)
metrics_final_kernel(const unsigned long long* __restrict__ auc_part, const double* __restrict__ ap_part, int parts,
                     const unsigned* __restrict__ fp, const unsigned* __restrict__ tot, const int* __restrict__ first95,
                     double* __restrict__ out) {
  __shared__ unsigned long long su[kMetThreads];
  __shared__ double sd[kMetThreads];
  unsigned long long a = 0;
  double b = 0.0;
  for (int j = threadIdx.x; j < parts; j += kMetThreads) {
    a += auc_part[j];
    b += ap_part[j];
  }
  su[threadIdx.x] = a;
  sd[threadIdx.x] = b;
  __syncthreads();
  for (int o = kMetThreads / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      su[threadIdx.x] += su[threadIdx.x + o];
      sd[threadIdx.x] += sd[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double P = tot[1], N = tot[2];
    if (tot[1] == 0 || tot[2] == 0) {
      out[0] = out[1] = out[2] = CUDART_NAN;
    } else {
      out[0] = static_cast<double>(su[0]) / (2.0 * P * N);
      out[1] = sd[0] / P;
      out[2] = fp[*first95] / N;
    }
  }
}

}  // namespace sb

using namespace sb;

extern "C" long long semseg_anomaly_class_moments_workspace_bytes(long long P, int C) {
  SB_CHECK_ARG(P > 0 && C > 0 && C <= kMomMaxClasses, "anomaly_class_moments: bad sizes P=%lld C=%d (C <= %d)", P, C,
               kMomMaxClasses);
  return ((P + kMomTile - 1) / kMomTile) * 3 * C * static_cast<long long>(sizeof(double));
}

extern "C" int semseg_anomaly_class_moments(const long long* pred, const double* ml, long long P, int C,
                                            void* workspace, double* moments, void* stream_) {
  const long long nb = semseg_anomaly_class_moments_workspace_bytes(P, C);
  if (nb < 0) return static_cast<int>(nb);
  SB_CHECK_ARG(pred && ml && workspace && moments, "anomaly_class_moments: null pointer");
  const long long tiles = (P + kMomTile - 1) / kMomTile;
  SB_CHECK_ARG(tiles < (1LL << 31), "anomaly_class_moments: %lld pixels are too many", P);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  double* partial = static_cast<double*>(workspace);
  anomaly_moments_tile_kernel<<<static_cast<unsigned>(tiles), kMomThreads, 0, stream>>>(pred, ml, P, C, partial);
  SB_LAUNCHED();
  anomaly_moments_final_kernel<<<cdiv(3 * C, kMomThreads), kMomThreads, 0, stream>>>(partial, static_cast<int>(tiles), C,
                                                                                    moments);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_anomaly_sml_workspace_bytes(int H, int W) {
  SB_CHECK_ARG(H > 0 && W > 0, "anomaly_sml: empty image %dx%d", H, W);
  const long long P = static_cast<long long>(H) * W;
  return P * (2 * sizeof(double) + 2 * sizeof(long long) + 8);   // two fp64 planes, row min / max, flags (8-aligned)
}

extern "C" int semseg_anomaly_sml(const double* ml, const long long* pred, int H, int W, int C, const double* mean,
                                  const double* stdv, int boundary_width, int boundary_iterations, int smooth_kernel,
                                  double smooth_sigma, int smooth_dilation, void* workspace, float* out,
                                  void* stream_) {
  const long long nb = semseg_anomaly_sml_workspace_bytes(H, W);
  if (nb < 0) return static_cast<int>(nb);
  SB_CHECK_ARG(ml && pred && mean && stdv && workspace && out, "anomaly_sml: null pointer");
  SB_CHECK_ARG(C > 0 && C <= kMomMaxClasses, "anomaly_sml: bad class count %d (1..%d)", C, kMomMaxClasses);
  SB_CHECK_ARG(boundary_iterations >= 0 && (boundary_iterations == 0 || boundary_width >= 1),
               "anomaly_sml: bad suppression (width %d, iterations %d; width >= 1 when iterations > 0)",
               boundary_width, boundary_iterations);
  SB_CHECK_ARG(smooth_kernel >= 1 && smooth_kernel <= kSmlMaxKernel && smooth_kernel % 2 == 1,
               "anomaly_sml: smooth_kernel %d must be odd and in 1..%d", smooth_kernel, kSmlMaxKernel);
  SB_CHECK_ARG(smooth_sigma > 0.0 && smooth_sigma <= DBL_MAX, "anomaly_sml: smooth_sigma must be finite and > 0");
  SB_CHECK_ARG(smooth_dilation >= 1, "anomaly_sml: smooth_dilation %d must be >= 1", smooth_dilation);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long P = static_cast<long long>(H) * W;
  SB_CHECK_ARG((P + kSmlThreads - 1) / kSmlThreads < (1LL << 31), "anomaly_sml: image too large");
  const unsigned blocks = static_cast<unsigned>((P + kSmlThreads - 1) / kSmlThreads);
  double* a = static_cast<double*>(workspace);
  double* b = a + P;
  long long* mm = reinterpret_cast<long long*>(b + P);
  unsigned char* edge = reinterpret_cast<unsigned char*>(mm + 2 * P);
  sml_standardise_kernel<<<blocks, kSmlThreads, 0, stream>>>(ml, pred, P, C, mean, stdv, a);
  SB_LAUNCHED();
  const int step = boundary_iterations ? boundary_width / boundary_iterations : 0;
  for (int i = 0; i < boundary_iterations; ++i) {
    const int r = boundary_width - i * step;
    sml_rows_kernel<<<blocks, kSmlThreads, 0, stream>>>(pred, P, W, r, mm);
    SB_LAUNCHED();
    sml_cols_kernel<<<blocks, kSmlThreads, 0, stream>>>(mm, P, H, W, r, edge);
    SB_LAUNCHED();
    sml_suppress_kernel<<<blocks, kSmlThreads, 0, stream>>>(a, edge, P, H, W, b);
    SB_LAUNCHED();
    double* t = a;
    a = b;
    b = t;
  }
  SmoothWeights gw{};
  const int half = smooth_kernel / 2;
  for (int j = -half; j <= half; ++j) gw.w[j + half] = exp(-static_cast<double>(j) * j / (2.0 * smooth_sigma * smooth_sigma));
  sml_smooth_kernel<<<blocks, kSmlThreads, 0, stream>>>(a, P, H, W, smooth_kernel, smooth_dilation, gw, out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

namespace {

struct MetricsLayout {
  long long sort_bytes;
  int nt;
  size_t keys, vals, keys_alt, vals_alt, sort_ws, cnt, tot, auc_part, ap_part, first95, total;
};

size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

MetricsLayout metrics_layout(long long n) {
  MetricsLayout l{};
  l.sort_bytes = semseg_segsort_u32_pairs_workspace_bytes(1, n);
  l.nt = static_cast<int>((n + kMetTile - 1) / kMetTile);
  const size_t u = align256(static_cast<size_t>(n) * sizeof(unsigned));
  size_t o = 0;
  l.keys = o; o += u;
  l.vals = o; o += u;
  l.keys_alt = o; o += u;
  l.vals_alt = o; o += u;
  l.sort_ws = o; o += align256(static_cast<size_t>(l.sort_bytes));
  l.cnt = o; o += align256(static_cast<size_t>(3) * l.nt * sizeof(unsigned));
  l.tot = o; o += 256;
  l.auc_part = o; o += align256(kMetTermCtas * sizeof(unsigned long long));
  l.ap_part = o; o += align256(kMetTermCtas * sizeof(double));
  l.first95 = o; o += 256;
  l.total = o;
  return l;
}

}  // namespace

extern "C" long long semseg_anomaly_metrics_workspace_bytes(long long n) {
  SB_CHECK_ARG(n > 0 && n < (1LL << 31), "anomaly_metrics: bad pixel count %lld (1 .. 2^31 - 1)", n);
  return static_cast<long long>(metrics_layout(n).total);
}

extern "C" int semseg_anomaly_metrics(const float* score, const void* label, int label_bytes, long long n,
                                      long long ignore_index, void* workspace, double* out, long long* info,
                                      void* stream_) {
  const long long nb = semseg_anomaly_metrics_workspace_bytes(n);
  if (nb < 0) return static_cast<int>(nb);
  SB_CHECK_ARG(score && label && workspace && out && info, "anomaly_metrics: null pointer");
  SB_CHECK_ARG(label_bytes == 1 || label_bytes == 8, "anomaly_metrics: label_bytes must be 1 (uint8) or 8 (int64), got %d",
               label_bytes);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const MetricsLayout l = metrics_layout(n);
  char* ws = static_cast<char*>(workspace);
  unsigned* keys = reinterpret_cast<unsigned*>(ws + l.keys);
  unsigned* vals = reinterpret_cast<unsigned*>(ws + l.vals);
  unsigned* keys_alt = reinterpret_cast<unsigned*>(ws + l.keys_alt);
  unsigned* vals_alt = reinterpret_cast<unsigned*>(ws + l.vals_alt);
  unsigned* cnt = reinterpret_cast<unsigned*>(ws + l.cnt);
  unsigned* tot = reinterpret_cast<unsigned*>(ws + l.tot);
  unsigned long long* auc_part = reinterpret_cast<unsigned long long*>(ws + l.auc_part);
  double* ap_part = reinterpret_cast<double*>(ws + l.ap_part);
  int* first95 = reinterpret_cast<int*>(ws + l.first95);
  const int ni = static_cast<int>(n);
  SB_CUDA(cudaMemsetAsync(info, 0, 3 * sizeof(long long), stream));
  SB_CUDA(cudaMemsetAsync(first95, 0x7f, sizeof(int), stream));   // 0x7f7f7f7f > any group index
  metrics_keys_kernel<<<cdiv(ni, kMetThreads), kMetThreads, 0, stream>>>(score, label, label_bytes, ni, ignore_index,
                                                                         keys, vals, info);
  SB_LAUNCHED();
  const int r = semseg_segsort_u32_pairs(keys, vals, keys_alt, vals_alt, 1, n, nullptr, ws + l.sort_ws, stream);
  if (r) return r;
  // after the sort keys / vals hold the result; the alternate buffers become the per-group counts
  unsigned* tp = keys_alt;
  unsigned* fp = vals_alt;
  metrics_count_kernel<<<l.nt, kMetThreads, 0, stream>>>(keys, vals, ni, l.nt, cnt);
  SB_LAUNCHED();
  metrics_scan_kernel<<<1, kMetScanThreads, 0, stream>>>(cnt, l.nt, tot, info);
  SB_LAUNCHED();
  metrics_groups_kernel<<<l.nt, kMetThreads, 0, stream>>>(keys, vals, ni, l.nt, cnt, tp, fp);
  SB_LAUNCHED();
  metrics_terms_kernel<<<kMetTermCtas, kMetThreads, 0, stream>>>(tp, fp, tot, auc_part, ap_part, first95);
  SB_LAUNCHED();
  metrics_final_kernel<<<1, kMetThreads, 0, stream>>>(auc_part, ap_part, kMetTermCtas, fp, tot, first95, out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Sliding-window evaluation after the network (tool/test.py:122-199, batched in semseg_b200/inference.py): logit
// upsample + softmax + flip averaging of every crop, overlap accumulation of a scale's crops, and the per-scale resize
// into the image's running total. The ATen chain it replaces materialises [2G, classes, crop, crop] fp32 logits and
// streams them through interpolate / softmax / flip / add / div / cat, then read-modify-writes an fp64 canvas once per
// crop. Here the low-resolution logits (fp32 NHWC, a few MB) are the only input of the scores kernel, every score is
// written once, and every canvas / total element is written once per scale. No tensor cores, no atomics.
//
// semseg_window_scores: same scheme as the fused training tail (tail.cu). Crop = 8(h-1)+1, so the align_corners scale
// is exactly 1/8, source index = x >> 3 and the weights are (x & 7)/8 in ATen's order
//   v = l0h*(l0w*v00 + l1w*v01) + l1h*(l0w*v10 + l1w*v11).
// The mirrored crop's logits are interpolated in their own coordinates at x' = crop-1-x (= F.interpolate of the
// flipped batch followed by .flip(3)); the two softmaxes are averaged as (p + p_mirror) * 0.5.
// The kernel serves every zoom factor of the network: its input is always the 1/8-resolution logits. At zoom Z < 8 the
// reference upsamples them xZ (the module output) and then x(8/Z) to the crop; one x8 upsample is the same function,
// because the xZ grid nests in the x8 grid (align_corners), the xZ result is bilinear on each of its cells, and bilinear
// interpolation of a bilinear function is exact. The two differ only by fp32 rounding.
//
// semseg_window_scores_stats: the same kernel (template flag kStats) writing C + 2 channels per crop: the C scores with
// unchanged arithmetic, then ML = max_c v and LSE = max + log(sum exp(v - max)) of the same upsampled logits, from the
// max and the sum of passes 1 and 2 (the log is taken before the sum is replaced by its reciprocal), flip-averaged as
// (a + a_mirror) * 0.5. The anomaly scores of semseg_b200/anomaly.py are defined on them; the accumulation and the
// resize below are class-count agnostic and carry the two extra channels unchanged.
//
// semseg_window_accumulate: a gather. Every pixel of the un-padded canvas sums in fp64 the scores of the crops that
// cover it in grid (row-major) order, starting from 0.0, and divides by their count: the same fp64 operations in the
// same order as `canvas[:, win] += scores[k]` over the grid followed by `canvas /= hits`, so the result is bit-identical.
//
// semseg_window_resize_add: half-pixel bilinear resize (align_corners=False, no anti-aliasing) of the fp64 canvas with
// ATen's fp64 upsample_bilinear2d arithmetic, added into the fp64 total in the same pass.
#include "host_common.h"

namespace sb {

constexpr int kWinMaxClasses = 256;
constexpr int kWinMaxCrops = 256;                // crops per axis of one scale (semseg_window_accumulate)
constexpr int kScoreCols = 64;                   // output columns per CTA (one per thread)
constexpr int kScoreNodes = kScoreCols / 8 + 2;  // node columns a CTA touches (the mirrored span is not 8-aligned)

// l0*a + l1*b rounded as ATen's fp32 upsample_bilinear2d kernel computes it: fma(l0, a, l1*b). Explicit, so that the
// compiler cannot fuse the other product; with logits in the thousands one ulp of an interpolated logit shows in the
// scores.
__device__ __forceinline__ float lerp_aten(float l0, float a, float l1, float b) { return fmaf(l0, a, __fmul_rn(l1, b)); }

// One CTA per (64 output columns, low-res interval row i0, crop); a thread owns one output column and the 8 output rows
// of the interval. Per class, the horizontal interpolation of the two node rows is done once and shared by the 8 rows.
// Three passes over the classes: max, sum of exp, then the normalised (and flip-averaged) scores. The softmax is ATen's:
// expf(v - max) summed in fp32, times the reciprocal of the sum (ATen divides; the two differ by a few ulp, < 3e-7,
// and an IEEE division per score would cost a slow-path call and register spills). (exp2 of v*log2e - max*log2e, as the training tail does, would cost
// an error proportional to |max| instead of |v - max|: ~1e-4 in the scores of a network with logits in the thousands.)
// Shared memory: [image (original, mirror)][node row (i0, i1)][kScoreNodes][Cs], Cs odd (distinct banks per node).
// kStats: `out` holds C + 2 channels per crop, the last two ML and LSE (see the file comment).
template <bool kFlip, bool kStats>
__global__ void __launch_bounds__(kScoreCols)
window_scores_kernel(const float* __restrict__ logits, int pitch, int G, int h, int w, int C, int Cs, int Ho, int Wo,
                     float* __restrict__ out) {
  extern __shared__ float S[];
  const int g = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kScoreCols;
  const int i1 = min(i0 + 1, h - 1);
  const int x_last = min(x0 + kScoreCols, Wo) - 1;
  const int jb0 = x0 >> 3;                  // first staged node column, original crop
  const int jb1 = (Wo - 1 - x_last) >> 3;   // first staged node column, mirrored crop
  constexpr int kImages = kFlip ? 2 : 1;
  const int tid = threadIdx.x;
  for (int idx = tid; idx < kImages * 2 * kScoreNodes * C; idx += kScoreCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % kScoreNodes, rr = (node / kScoreNodes) & 1, im = node / (2 * kScoreNodes);
    const int j = (im ? jb1 : jb0) + jj;
    if (j < w)
      S[node * Cs + c] =
          logits[((static_cast<size_t>(im * G + g) * h + (rr ? i1 : i0)) * w + j) * static_cast<size_t>(pitch) + c];
  }
  __syncthreads();
  const int x = x0 + tid;
  if (x >= Wo) return;
  const int rows = min(8, Ho - 8 * i0);     // 8, or 1 for the last node row
  const float* P[kImages][4];               // nodes (i0, j0), (i0, j1), (i1, j0), (i1, j1) of each image
  float l0w[kImages], l1w[kImages];
#pragma unroll
  for (int im = 0; im < kImages; ++im) {
    const int xi = im ? Wo - 1 - x : x;
    const int jb = im ? jb1 : jb0;
    const int j0 = xi >> 3, j1 = min(j0 + 1, w - 1);
    l1w[im] = static_cast<float>(xi & 7) * 0.125f;
    l0w[im] = 1.f - l1w[im];
    const float* top = S + (im * 2) * kScoreNodes * Cs;
    P[im][0] = top + (j0 - jb) * Cs;
    P[im][1] = top + (j1 - jb) * Cs;
    P[im][2] = P[im][0] + kScoreNodes * Cs;
    P[im][3] = P[im][1] + kScoreNodes * Cs;
  }
  float mx[kImages][8], sum[kImages][8];
#pragma unroll
  for (int im = 0; im < kImages; ++im)
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      mx[im][r] = -INFINITY;
      sum[im][r] = 0.f;
    }
  // pass 1: max
#pragma unroll 2
  for (int c = 0; c < C; ++c) {
#pragma unroll
    for (int im = 0; im < kImages; ++im) {
      const float top = lerp_aten(l0w[im], P[im][0][c], l1w[im], P[im][1][c]);
      const float bot = lerp_aten(l0w[im], P[im][2][c], l1w[im], P[im][3][c]);
#pragma unroll
      for (int r = 0; r < 8; ++r) mx[im][r] = fmaxf(mx[im][r], lerp_aten(1.f - 0.125f * r, top, 0.125f * r, bot));
    }
  }
  // pass 2: sum of exp(v - max)
#pragma unroll 2
  for (int c = 0; c < C; ++c) {
#pragma unroll
    for (int im = 0; im < kImages; ++im) {
      const float top = lerp_aten(l0w[im], P[im][0][c], l1w[im], P[im][1][c]);
      const float bot = lerp_aten(l0w[im], P[im][2][c], l1w[im], P[im][3][c]);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float v = lerp_aten(1.f - 0.125f * r, top, 0.125f * r, bot);
        sum[im][r] += expf(v - mx[im][r]);
      }
    }
  }
  const size_t plane = static_cast<size_t>(Ho) * Wo;
  const int Co = kStats ? C + 2 : C;   // channels per crop in `out`
  float* o = out + static_cast<size_t>(g) * Co * plane + static_cast<size_t>(8 * i0) * Wo + x;
  if constexpr (kStats) {
    float* oml = o + static_cast<size_t>(C) * plane;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      float ml = mx[0][r], lse = mx[0][r] + logf(sum[0][r]);
      if (kFlip) {
        ml = (ml + mx[1][r]) * 0.5f;
        lse = (lse + (mx[1][r] + logf(sum[1][r]))) * 0.5f;
      }
      if (r < rows) {
        oml[static_cast<size_t>(r) * Wo] = ml;
        oml[plane + static_cast<size_t>(r) * Wo] = lse;
      }
    }
  }
#pragma unroll
  for (int im = 0; im < kImages; ++im)
#pragma unroll
    for (int r = 0; r < 8; ++r) sum[im][r] = __fdividef(1.f, sum[im][r]);   // sum in [1, C]: now its reciprocal
  // pass 3: scores
#pragma unroll 2
  for (int c = 0; c < C; ++c) {
    float p[8];
#pragma unroll
    for (int im = 0; im < kImages; ++im) {
      const float top = lerp_aten(l0w[im], P[im][0][c], l1w[im], P[im][1][c]);
      const float bot = lerp_aten(l0w[im], P[im][2][c], l1w[im], P[im][3][c]);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float v = lerp_aten(1.f - 0.125f * r, top, 0.125f * r, bot);
        const float q = expf(v - mx[im][r]) * sum[im][r];
        p[r] = im ? (p[r] + q) * 0.5f : q;
      }
    }
    float* oc = o + static_cast<size_t>(c) * plane;
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (r < rows) oc[static_cast<size_t>(r) * Wo] = p[r];
  }
}

constexpr int kMcRows = 2;                       // output rows per CTA (same node interval: 8 is even)
constexpr int kMcThreads = kScoreCols * kMcRows; // one thread per output pixel
constexpr int kMcMaxDraws = 128;

// Monte Carlo dropout scores: T draws of a batch's low-resolution logits -> per crop the draw mean of the flip-averaged
// softmax and of the flip-averaged sample entropy. One CTA per (64 output columns, 2 output rows, crop); a thread owns
// one output pixel. Per draw the two node rows of each image are staged as in window_scores_kernel, and the three passes
// over the classes (max, sum of exp, then q = exp(v - max) / sum) use its arithmetic, so each draw's flip-averaged score
// is the bits window_scores_kernel writes. Pass 3 also forms the sample entropy from the max-shifted logits,
// H = log S - sum_c q_c (v_c - max), taken as log S - (1/S) sum_c e_c (v_c - max) with e = exp(v - max): both terms
// are >= 0, so a confident pixel keeps a small H accurate (log-sum-exp minus sum q v would cancel). The running draw
// sums live in shared memory, [C][kMcThreads] (thread-contiguous: no bank conflicts, no atomics), the entropy sum in a
// register; every element of `out` is written once, after the last draw, as sum * (1/T) (the sums start from draw 0's
// value, so T = 1 writes window_scores' bits).
// Shared memory: the node stage [image][node row][kScoreNodes][Cs], then the accumulators: <= 169 KB at C = 256.
template <bool kFlip>
__global__ void __launch_bounds__(kMcThreads)
window_scores_mc_kernel(const float* __restrict__ logits, int pitch, int T, int G, int h, int w, int C, int Cs, int Ho,
                        int Wo, float inv_t, float* __restrict__ out) {
  extern __shared__ float S[];
  constexpr int kImages = kFlip ? 2 : 1;
  float* acc = S + kImages * 2 * kScoreNodes * Cs;
  const int g = blockIdx.z, x0 = blockIdx.x * kScoreCols;
  const int tid = threadIdx.x;
  const int x = x0 + (tid % kScoreCols), y = kMcRows * blockIdx.y + tid / kScoreCols;
  const int i0 = (kMcRows * blockIdx.y) >> 3;     // both rows of the CTA lie in this node interval
  const int i1 = min(i0 + 1, h - 1);
  const int x_last = min(x0 + kScoreCols, Wo) - 1;
  const int jb0 = x0 >> 3;
  const int jb1 = (Wo - 1 - x_last) >> 3;
  const bool valid = x < Wo && y < Ho;
  const int r = y & 7;
  const float l1h = 0.125f * r, l0h = 1.f - 0.125f * r;
  const float* P[kImages][4];
  float l0w[kImages], l1w[kImages];
#pragma unroll
  for (int im = 0; im < kImages; ++im) {
    const int xi = valid ? (im ? Wo - 1 - x : x) : x0;
    const int jb = im ? jb1 : jb0;
    const int j0 = xi >> 3, j1 = min(j0 + 1, w - 1);
    l1w[im] = static_cast<float>(xi & 7) * 0.125f;
    l0w[im] = 1.f - l1w[im];
    const float* top = S + (im * 2) * kScoreNodes * Cs;
    P[im][0] = top + (j0 - jb) * Cs;
    P[im][1] = top + (j1 - jb) * Cs;
    P[im][2] = P[im][0] + kScoreNodes * Cs;
    P[im][3] = P[im][1] + kScoreNodes * Cs;
  }
  const size_t draw_stride = static_cast<size_t>(kImages) * G * h * w * pitch;
  float hsum = 0.f;
  for (int t = 0; t < T; ++t) {
    const float* lt = logits + t * draw_stride;
    __syncthreads();                            // the previous draw's stage is no longer read
    for (int idx = tid; idx < kImages * 2 * kScoreNodes * C; idx += kMcThreads) {
      const int c = idx % C;
      const int node = idx / C;
      const int jj = node % kScoreNodes, rr = (node / kScoreNodes) & 1, im = node / (2 * kScoreNodes);
      const int j = (im ? jb1 : jb0) + jj;
      if (j < w)
        S[node * Cs + c] =
            lt[((static_cast<size_t>(im * G + g) * h + (rr ? i1 : i0)) * w + j) * static_cast<size_t>(pitch) + c];
    }
    __syncthreads();
    if (!valid) continue;
    float mx[kImages], sum[kImages];
#pragma unroll
    for (int im = 0; im < kImages; ++im) {
      mx[im] = -INFINITY;
      sum[im] = 0.f;
    }
    // pass 1: max
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
#pragma unroll
      for (int im = 0; im < kImages; ++im) {
        const float top = lerp_aten(l0w[im], P[im][0][c], l1w[im], P[im][1][c]);
        const float bot = lerp_aten(l0w[im], P[im][2][c], l1w[im], P[im][3][c]);
        mx[im] = fmaxf(mx[im], lerp_aten(l0h, top, l1h, bot));
      }
    }
    // pass 2: sum of exp(v - max)
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
#pragma unroll
      for (int im = 0; im < kImages; ++im) {
        const float top = lerp_aten(l0w[im], P[im][0][c], l1w[im], P[im][1][c]);
        const float bot = lerp_aten(l0w[im], P[im][2][c], l1w[im], P[im][3][c]);
        sum[im] += expf(lerp_aten(l0h, top, l1h, bot) - mx[im]);
      }
    }
    float ent[kImages], rs[kImages];
#pragma unroll
    for (int im = 0; im < kImages; ++im) {
      ent[im] = logf(sum[im]);
      rs[im] = __fdividef(1.f, sum[im]);
    }
    // pass 3: scores into the draw sums, and sum_c exp(v - max) (v - max) per image. The flip average is rounded as
    // the compiler contracts window_scores_kernel's (q + q_mirror) * 0.5: the mirror's product fused into the sum,
    // fma(e_mirror, 1/S_mirror, q) * 0.5, written out so that it cannot contract otherwise here.
    float ed[kImages];
#pragma unroll
    for (int im = 0; im < kImages; ++im) ed[im] = 0.f;
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      float e[kImages];
#pragma unroll
      for (int im = 0; im < kImages; ++im) {
        const float top = lerp_aten(l0w[im], P[im][0][c], l1w[im], P[im][1][c]);
        const float bot = lerp_aten(l0w[im], P[im][2][c], l1w[im], P[im][3][c]);
        const float d = lerp_aten(l0h, top, l1h, bot) - mx[im];
        e[im] = expf(d);
        ed[im] = fmaf(e[im], d, ed[im]);
      }
      const float p = kFlip ? fmaf(e[kImages - 1], rs[kImages - 1], __fmul_rn(e[0], rs[0])) * 0.5f
                            : __fmul_rn(e[0], rs[0]);
      float* a = acc + c * kMcThreads + tid;
      *a = t ? *a + p : p;
    }
    // H = log S - (1/S) sum_c e_c d_c, both terms >= 0
    float hs = ent[0] - rs[0] * ed[0];
    if (kFlip) hs = (hs + (ent[kImages - 1] - rs[kImages - 1] * ed[kImages - 1])) * 0.5f;
    hsum = t ? hsum + hs : hs;
  }
  if (!valid) return;
  const size_t plane = static_cast<size_t>(Ho) * Wo;
  float* o = out + static_cast<size_t>(g) * (C + 1) * plane + static_cast<size_t>(y) * Wo + x;
  for (int c = 0; c < C; ++c) o[c * plane] = acc[c * kMcThreads + tid] * inv_t;
  o[C * plane] = hsum * inv_t;
}

// Crop origins of one scale, per axis, ascending; passed by value (2 KB of kernel parameters).
struct WindowGrid {
  int ny, nx;
  int ys[kWinMaxCrops];
  int xs[kWinMaxCrops];
};

constexpr int kAccCols = 128;
constexpr int kAccClasses = 8;  // classes per CTA

// One CTA per (128 canvas columns, canvas row, 8 classes). The crops covering a pixel form a contiguous index range per
// axis (origins ascending); they are visited row-major, i.e. in grid order.
__global__ void __launch_bounds__(kAccCols)
window_accumulate_kernel(const float* __restrict__ scores, int C, int ch, int cw, const __grid_constant__ WindowGrid wg,
                         int top, int left, int img_h, int img_w, double* __restrict__ canvas) {
  const int yy = blockIdx.y, xx = blockIdx.x * kAccCols + threadIdx.x;
  if (xx >= img_w) return;
  const int y = yy + top, x = xx + left;
  int ky0 = 0;
  while (wg.ys[ky0] + ch <= y) ++ky0;
  int ky1 = ky0;
  while (ky1 + 1 < wg.ny && wg.ys[ky1 + 1] <= y) ++ky1;
  int kx0 = 0;
  while (wg.xs[kx0] + cw <= x) ++kx0;
  int kx1 = kx0;
  while (kx1 + 1 < wg.nx && wg.xs[kx1 + 1] <= x) ++kx1;
  const double count = static_cast<double>((ky1 - ky0 + 1) * (kx1 - kx0 + 1));
  const size_t plane = static_cast<size_t>(ch) * cw;
  const int c_end = min(C, static_cast<int>(blockIdx.z + 1) * kAccClasses);
  for (int c = blockIdx.z * kAccClasses; c < c_end; ++c) {
    double acc = 0.0;
    for (int ky = ky0; ky <= ky1; ++ky) {
      const float* row = scores + (static_cast<size_t>(ky) * wg.nx * C + c) * plane + static_cast<size_t>(y - wg.ys[ky]) * cw;
      for (int kx = kx0; kx <= kx1; ++kx)
        acc += static_cast<double>(row[static_cast<size_t>(kx) * C * plane + (x - wg.xs[kx])]);
    }
    canvas[(static_cast<size_t>(c) * img_h + yy) * img_w + xx] = acc / count;
  }
}

constexpr int kResizeCols = 128;
constexpr int kResizeClasses = 8;

__device__ __forceinline__ void half_pixel_src(int o, double scale, int in, int& i0, int& di, double& l1) {
  double f = scale * (o + 0.5) - 0.5;  // ATen's area_pixel_compute_source_index, align_corners=False
  f = f < 0.0 ? 0.0 : f;
  i0 = static_cast<int>(f);
  di = i0 < in - 1 ? 1 : 0;
  l1 = f - i0;
}

// One CTA per (128 output columns, output row, 8 classes): total[c, y, x] += bilinear(canvas)[c, y, x].
__global__ void __launch_bounds__(kResizeCols)
window_resize_add_kernel(const double* __restrict__ canvas, int C, int Hi, int Wi, double rh, double rw,
                         double* __restrict__ total, int Ho, int Wo) {
  const int y = blockIdx.y, x = blockIdx.x * kResizeCols + threadIdx.x;
  if (x >= Wo) return;
  int h1, dh, w1, dw;
  double l1h, l1w;
  half_pixel_src(y, rh, Hi, h1, dh, l1h);
  half_pixel_src(x, rw, Wi, w1, dw, l1w);
  const double l0h = 1.0 - l1h, l0w = 1.0 - l1w;
  const size_t in_plane = static_cast<size_t>(Hi) * Wi, out_plane = static_cast<size_t>(Ho) * Wo;
  const size_t i00 = static_cast<size_t>(h1) * Wi + w1;
  const size_t i10 = i00 + static_cast<size_t>(dh) * Wi;
  const int c_end = min(C, static_cast<int>(blockIdx.z + 1) * kResizeClasses);
  for (int c = blockIdx.z * kResizeClasses; c < c_end; ++c) {
    const double* s = canvas + c * in_plane;
    const double v = l0h * (l0w * s[i00] + l1w * s[i00 + dw]) + l1h * (l0w * s[i10] + l1w * s[i10 + dw]);
    total[c * out_plane + static_cast<size_t>(y) * Wo + x] += v;
  }
}

}  // namespace sb

using namespace sb;

template <bool kStats>
static int window_scores(const char* fn, const float* logits, int pitch, int G, int h, int w, int C, int flip,
                         float* out, int crop_h, int crop_w, cudaStream_t stream) {
  SB_CHECK_ARG(logits && out, "%s: null pointer", fn);
  SB_CHECK_ARG(G > 0 && h > 1 && w > 1 && h <= 65535 && G <= 65535 && C > 0 && C <= kWinMaxClasses && pitch >= C &&
                   (flip == 0 || flip == 1),
               "%s: bad sizes (G=%d h=%d w=%d C=%d pitch=%d flip=%d; C<=%d, pitch>=C)", fn, G, h, w, C, pitch, flip,
               kWinMaxClasses);
  SB_CHECK_ARG(crop_h == 8 * (h - 1) + 1 && crop_w == 8 * (w - 1) + 1,
               "%s: crop must be 8(h-1)+1 x 8(w-1)+1 of the %dx%d logits (got %dx%d)", fn, h, w, crop_h, crop_w);
  const int Cs = C | 1;
  const size_t smem = static_cast<size_t>(flip ? 2 : 1) * 2 * kScoreNodes * Cs * sizeof(float);  // <= 41 KB
  dim3 grid(cdiv(crop_w, kScoreCols), h, G);
  if (flip)
    window_scores_kernel<true, kStats><<<grid, kScoreCols, smem, stream>>>(logits, pitch, G, h, w, C, Cs, crop_h,
                                                                           crop_w, out);
  else
    window_scores_kernel<false, kStats><<<grid, kScoreCols, smem, stream>>>(logits, pitch, G, h, w, C, Cs, crop_h,
                                                                            crop_w, out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_window_scores(const float* logits, int pitch, int G, int h, int w, int C, int flip, float* out,
                                    int crop_h, int crop_w, void* stream) {
  return window_scores<false>("window_scores", logits, pitch, G, h, w, C, flip, out, crop_h, crop_w,
                              static_cast<cudaStream_t>(stream));
}

extern "C" int semseg_window_scores_stats(const float* logits, int pitch, int G, int h, int w, int C, int flip,
                                          float* out, int crop_h, int crop_w, void* stream) {
  return window_scores<true>("window_scores_stats", logits, pitch, G, h, w, C, flip, out, crop_h, crop_w,
                             static_cast<cudaStream_t>(stream));
}

extern "C" int semseg_window_scores_mc(const float* logits, int pitch, int T, int G, int h, int w, int C, int flip,
                                       float* out, int crop_h, int crop_w, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(logits && out, "window_scores_mc: null pointer");
  SB_CHECK_ARG(T >= 1 && T <= kMcMaxDraws, "window_scores_mc: draws T=%d not in 1..%d", T, kMcMaxDraws);
  SB_CHECK_ARG(G > 0 && h > 1 && w > 1 && h <= 65535 && G <= 65535 && C > 0 && C <= kWinMaxClasses && pitch >= C &&
                   (flip == 0 || flip == 1),
               "window_scores_mc: bad sizes (G=%d h=%d w=%d C=%d pitch=%d flip=%d; C<=%d, pitch>=C)", G, h, w, C, pitch,
               flip, kWinMaxClasses);
  SB_CHECK_ARG(crop_h == 8 * (h - 1) + 1 && crop_w == 8 * (w - 1) + 1,
               "window_scores_mc: crop must be 8(h-1)+1 x 8(w-1)+1 of the %dx%d logits (got %dx%d)", h, w, crop_h,
               crop_w);
  const int Cs = C | 1;
  const size_t smem = (static_cast<size_t>(flip ? 2 : 1) * 2 * kScoreNodes * Cs + static_cast<size_t>(C) * kMcThreads) *
                      sizeof(float);   // <= 169 KB
  const float inv_t = 1.f / static_cast<float>(T);
  dim3 grid(cdiv(crop_w, kScoreCols), cdiv(crop_h, kMcRows), G);
  if (flip) {
    SB_CUDA(cudaFuncSetAttribute(window_scores_mc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem)));
    window_scores_mc_kernel<true><<<grid, kMcThreads, smem, stream>>>(logits, pitch, T, G, h, w, C, Cs, crop_h, crop_w,
                                                                      inv_t, out);
  } else {
    SB_CUDA(cudaFuncSetAttribute(window_scores_mc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem)));
    window_scores_mc_kernel<false><<<grid, kMcThreads, smem, stream>>>(logits, pitch, T, G, h, w, C, Cs, crop_h,
                                                                       crop_w, inv_t, out);
  }
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Origins must start at 0, ascend strictly, end at extent - crop and leave no gap (every pixel covered).
static int check_origins(const int* o, int n, int crop, int extent, const char* axis) {
  SB_CHECK_ARG(o && n > 0 && n <= kWinMaxCrops, "window_accumulate: %s origins: null or count %d not in 1..%d", axis, n,
               kWinMaxCrops);
  SB_CHECK_ARG(o[0] == 0 && o[n - 1] == extent - crop,
               "window_accumulate: %s origins out of range (first %d, last %d; crop %d, padded extent %d)", axis, o[0],
               o[n - 1], crop, extent);
  for (int k = 1; k < n; ++k)
    SB_CHECK_ARG(o[k] > o[k - 1] && o[k] - o[k - 1] <= crop,
                 "window_accumulate: %s origins must ascend with gaps <= crop (%d after %d)", axis, o[k], o[k - 1]);
  return SEMSEG_OK;
}

extern "C" int semseg_window_accumulate(const float* scores, int C, int crop_h, int crop_w, const int* ys, int ny,
                                        const int* xs, int nx, int full_h, int full_w, int top, int left, int img_h,
                                        int img_w, double* canvas, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(scores && canvas, "window_accumulate: null pointer");
  SB_CHECK_ARG(C > 0 && crop_h > 0 && crop_w > 0 && img_h > 0 && img_w > 0 && img_h <= 65535 &&
                   full_h >= crop_h && full_w >= crop_w && top >= 0 && left >= 0 && top + img_h <= full_h &&
                   left + img_w <= full_w,
               "window_accumulate: bad sizes (C=%d crop %dx%d, padded %dx%d, image %dx%d at (%d, %d))", C, crop_h, crop_w,
               full_h, full_w, img_h, img_w, top, left);
  int r = check_origins(ys, ny, crop_h, full_h, "row");
  if (r) return r;
  r = check_origins(xs, nx, crop_w, full_w, "column");
  if (r) return r;
  WindowGrid wg;
  wg.ny = ny;
  wg.nx = nx;
  for (int k = 0; k < kWinMaxCrops; ++k) {
    wg.ys[k] = k < ny ? ys[k] : 0;
    wg.xs[k] = k < nx ? xs[k] : 0;
  }
  dim3 grid(cdiv(img_w, kAccCols), img_h, cdiv(C, kAccClasses));
  window_accumulate_kernel<<<grid, kAccCols, 0, stream>>>(scores, C, crop_h, crop_w, wg, top, left, img_h, img_w,
                                                          canvas);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_window_resize_add(const double* canvas, int C, int Hi, int Wi, double* total, int Ho, int Wo,
                                        void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(canvas && total, "window_resize_add: null pointer");
  SB_CHECK_ARG(C > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && Ho <= 65535,
               "window_resize_add: bad sizes (C=%d, %dx%d -> %dx%d)", C, Hi, Wi, Ho, Wo);
  // ATen's area_pixel_compute_scale for align_corners=False without a scale factor: in / out in fp64
  const double rh = static_cast<double>(Hi) / Ho, rw = static_cast<double>(Wi) / Wo;
  dim3 grid(cdiv(Wo, kResizeCols), Ho, cdiv(C, kResizeClasses));
  window_resize_add_kernel<<<grid, kResizeCols, 0, stream>>>(canvas, C, Hi, Wi, rh, rw, total, Ho, Wo);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

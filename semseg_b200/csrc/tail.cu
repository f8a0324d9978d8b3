// Fused logit upsample (bilinear, align_corners=True, xZ for zoom_factor Z in {1, 2, 4, 8}) + cross-entropy(ignore_index)
// + argmax.
//
// Replaces F.interpolate -> CrossEntropyLoss -> max(1) at model/pspnet.py:94-103 (same in model/psanet.py:168-177),
// which materialise an [N, classes, H, W] fp32 tensor (2.15 GB at bs16 / 150 classes / 473x473, zoom 8) and stream it
// ~9 times per head. Here the low-resolution logits (fp32 NHWC, a few MB, L2 resident) are staged in shared
// memory and every output pixel's class vector is interpolated on the fly; the only full-resolution tensors
// are the int64 argmax and an fp32 log-sum-exp map kept for the backward pass.
//
// The kernels are templated on the zoom factor Z and require Ho = Z*(h-1)+1 and Wo = Z*(w-1)+1. For a power-of-two Z
// the align_corners scale (h-1)/(Ho-1) is exactly 1/Z in fp32, so the source index is x / Z and the weights (x % Z)/Z
// are exact — the same fp32 values ATen computes. Interpolation order follows ATen's upsample_bilinear2d:
//   v = l0h*(l0w*v00 + l1w*v01) + l1h*(l0w*v10 + l1w*v11).
// Z = 1 is plain cross-entropy + argmax + lse on the NHWC logits (model/pspnet.py:94 skips the interpolation): one node
// row is staged and v is the logit itself. Every shipped config uses Z = 8; the Z = 8 instance is the kernel the
// original x8-only entry points ran, instruction for instruction.
//
// Backward is a deterministic, separable gather (rows kernel + cols kernel, see below). No atomics, every dlogits
// element is written exactly once.
//
// Online hard-pixel mining (OHEM cross-entropy, semseg_b200/losses.py) runs on the same kernels in a compile-time form
// (kOhem): the forward also writes each pixel's target probability p_t and nll and leaves the loss to a masked reduce;
// a radix select over the p_t bit patterns finds the k-th smallest p_t on the device; the backward treats every pixel
// with p_t >= threshold as ignored. The kOhem = false instances are the plain cross-entropy kernels, unchanged.
//
// Class weights and label smoothing (nn.CrossEntropyLoss(weight, label_smoothing)) are a second compile-time flag,
// kWeighted. With w the class weights (all ones when none are given), W = sum_c w_c, eps the smoothing and a valid
// pixel's lse = logsumexp_c v_c:
//   loss_pix = (1-eps) w_t (lse - v_t) + (eps/C) sum_c w_c (lse - v_c),   loss = sum loss_pix / D,   D = sum w_t
//   dloss_pix/dv_c = p_c ((1-eps) w_t + (eps/C) W) - [c = t] (1-eps) w_t - (eps/C) w_c
// and loss 0 with an exactly zero gradient when D = 0. Weighted OHEM (kOhem and kWeighted) writes nll = w_t (lse - v_t)
// and scales the pixel's gradient by w_t; its selection and mean over the kept pixels are the OHEM ones. The
// kWeighted = false instances are unchanged.
//
// The soft Dice loss, alone or plus cross-entropy, runs the plain forward instance and its own statistics, reduce and
// gradient kernels (see "Dice" below); no existing instance changes.
//
// The Lovász-Softmax loss, alone or plus cross-entropy, runs the plain forward instance, a key pass, the segmented stable
// radix sort of csrc/segsort.cu and its own scan and gradient kernels (see "Lovász-Softmax" below); no existing
// instance changes.
//
// The RMI loss with its BCE term, optionally plus cross-entropy, runs the plain forward instance and its own pool, moment,
// algebra and gradient kernels (see "RMI" below); no existing instance changes.
//
// The softmax focal loss, with or without class weights, runs sibling forward and rows kernels (see "focal loss" below)
// with the plain reduce and cols kernels; no existing instance changes.
//
// Confidence-masked pseudo-labels from a teacher's logits run a count pass and a two-map forward (see "pseudo-labels"
// below); their backward is the focal backward on the forward's effective targets and weights. No existing instance
// changes.
//
// Entropy minimisation plus cross-entropy (TENT / MinEnt) runs sibling forward and rows kernels (see "entropy" below)
// with the plain reduce and cols kernels; no existing instance changes.
//
// The SegPGD attack loss runs a sibling forward kernel with the plain reduce; its backward is the focal backward on the
// forward's per-pixel weights (see "SegPGD" below). No existing instance changes.
//
// MiB's unbiased cross-entropy is a third compile-time flag of the plain forward and rows kernels, kUnbiased; its unbiased
// distillation runs sibling kernels of the distillation ones with their cols kernel (see "class-incremental" below). The
// kUnbiased = false instances are unchanged.
#include <cmath>

#include "host_common.h"

namespace sb {

constexpr int kMaxClasses = 256;

// ---------------------------------------------------------------------------------------------------- forward
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kLog2e = 1.4426950408889634f;
constexpr int kFwdCols = 128;                    // output columns per CTA (one per thread)
constexpr float kInvalidPt = -1.f;               // p_t of a pixel that is ignored or whose target is out of range

// Compile-time geometry of zoom factor Z (a power of two): source index x >> kShift, fraction (x & kMask) * kStep.
template <int Z>
struct Zoom {
  static_assert(Z == 1 || Z == 2 || Z == 4 || Z == 8, "zoom factor must be 1, 2, 4 or 8");
  static constexpr int kShift = Z == 1 ? 0 : Z == 2 ? 1 : Z == 4 ? 2 : 3;
  static constexpr int kMask = Z - 1;
  static constexpr float kStep = 1.f / Z;                 // exact: Z is a power of two
  static constexpr int kNodes = kFwdCols / Z + 1;         // low-res node columns a forward CTA touches
  static constexpr int kNodeRows = Z == 1 ? 1 : 2;        // node rows a forward CTA stages (Z = 1: no vertical lerp)
};

// Output row r of an interval from its horizontally interpolated node rows, compile-time row weights r/Z.
template <int Z>
__device__ __forceinline__ float row_lerp(float top, float bot, int r) {
  if constexpr (Z == 1) {
    return top;
  } else {
    return (1.f - Zoom<Z>::kStep * r) * top + (Zoom<Z>::kStep * r) * bot;
  }
}

// The C class weights (1 where class_weight is NULL) into s_w[0..C-1] and, after the caller's next __syncthreads(),
// their sum W in s_w[C]: warp 0 sums in a fixed order, so every CTA gets the same bits. Needs blockDim.x >= 32.
__device__ __forceinline__ void stage_class_weights(const float* __restrict__ class_weight, int C, float* s_w) {
  for (int c = threadIdx.x; c < C; c += blockDim.x) s_w[c] = class_weight ? class_weight[c] : 1.f;
  __syncthreads();
  if (threadIdx.x < 32) {
    float a = 0.f;
    for (int c = threadIdx.x; c < C; c += 32) a += s_w[c];
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (threadIdx.x == 0) s_w[C] = a;
  }
}

// One CTA per (128 output columns, low-res interval row i0, image); a thread owns one output column and the Z
// output rows of the interval. Per class the horizontal interpolation of the two node rows (top, bot) is done once
// and shared by the Z rows (v = l0h*top + l1h*bot with compile-time row weights), so at Z = 8 a pixel-class costs ~5
// instructions per pass instead of a full 4-tap interpolation. Two passes over the classes: max/argmax, then
// sum of exp2 — one MUFU per pixel-class, no rescaling branches.
// kOhem: no loss partials; per pixel p_t = exp(v_t - lse) and nll = lse - v_t instead (kInvalidPt / 0 where the target
// is ignored or out of range). The OHEM-only arguments come last, so the plain instances keep their parameter layout.
// kWeighted without kOhem: the partials are (sum of loss_pix, sum of w_t); the class weights and W are staged after the
// node rows and the second class pass also sums w_c (m - v_c) per output row (m: the row's max, so no term cancels).
// kWeighted with kOhem: nll = w_t (lse - v_t). The weighted-only arguments come after the OHEM ones.
// kUnbiased (MiB's unbiased cross-entropy, see "class-incremental" below; neither kOhem nor kWeighted): the first pass
// also keeps the maximum over the old classes [0, c_old), the second their own sum of exp2 against it, and lse_old_out
// gets lse_old per pixel; a pixel labelled with an old class scores lse - lse_old, one labelled with a new class
// lse - v_t. Its arguments come last; the other instances do not read them.
template <int Z, bool kOhem, bool kWeighted = false, bool kUnbiased = false>
__global__ void __launch_bounds__(kFwdCols)
upsample_ce_fwd_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                       const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                       float* __restrict__ partial, long long* __restrict__ argmax_out, float* __restrict__ lse_out,
                       float* __restrict__ pt_out, float* __restrict__ nll_out,
                       const float* __restrict__ class_weight = nullptr, float smoothing = 0.f, int c_old = 0,
                       float* __restrict__ lse_old_out = nullptr) {
  static_assert(!(kUnbiased && (kOhem || kWeighted)), "the unbiased form is plain cross-entropy otherwise");
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  constexpr bool kWeightedCE = kWeighted && !kOhem;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs]; Cs odd -> the node columns a warp reads hit distinct banks
  __shared__ float red_loss[kFwdCols / 32];
  __shared__ float red_cnt[kFwdCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  float* s_w = S + G::kNodeRows * kFwdNodes * Cs;  // kWeightedCE: [C] class weights, then W
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  if constexpr (kWeightedCE) stage_class_weights(class_weight, C, s_w);
  __syncthreads();
  float loss = 0.f, cnt = 0.f;
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);  // Z, or 1 for the last node row (Ho = Z(h-1)+1)
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* A = S + (j0 - j_base) * Cs;   // node (i0, j0)
    const float* B = S + (j1 - j_base) * Cs;   // node (i0, j1)
    const float* Cc = A + kFwdNodes * Cs;      // node (i1, j0); not staged (and not read) at Z = 1
    const float* D = B + kFwdNodes * Cs;       // node (i1, j1)
    float m[Z], sum[Z];
    float mo[Z], so[Z];  // kUnbiased: the old classes' own maximum and sum
    int am[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      m[r] = -INFINITY;
      am[r] = 0;
      sum[r] = 0.f;
      mo[r] = 0.f;
      so[r] = 0.f;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      // the interval's two horizontally interpolated node rows (Z = 1: the logit itself)
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        if (v > m[r]) {
          m[r] = v;
          am[r] = c;
        }
      }
      if constexpr (kUnbiased) {
        if (c == c_old - 1) {   // classes run in order: the maximum so far is the old classes'
#pragma unroll
          for (int r = 0; r < Z; ++r) mo[r] = m[r];
        }
      }
    }
    float m2[Z], sw[Z];  // sw: kWeightedCE, sum_c w_c (m - v_c)
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      m2[r] = m[r] * kLog2e;
      sw[r] = 0.f;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        sum[r] += ex2_approx(fmaf(v, kLog2e, -m2[r]));
        if constexpr (kWeightedCE) sw[r] = fmaf(s_w[c], m[r] - v, sw[r]);
        if constexpr (kUnbiased) {
          if (c < c_old) so[r] += ex2_approx(fmaf(v, kLog2e, -mo[r] * kLog2e));
        }
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        const long long t = target[pix];
        const float lse = m[r] + __logf(sum[r]);
        if (argmax_out) argmax_out[pix] = am[r];
        lse_out[pix] = lse;
        float lse_old = 0.f;
        if constexpr (kUnbiased) {
          lse_old = mo[r] + __logf(so[r]);
          lse_old_out[pix] = lse_old;
        }
        if (kUnbiased && t != ignore_index && t >= 0 && t < c_old) {
          loss += lse - lse_old;   // an old-class label counts as background: every old class is the target
          cnt += 1.f;
        } else if (t != ignore_index && t >= 0 && t < C) {
          const int tc = static_cast<int>(t);
          const float top = Z == 1 ? A[tc] : l0w * A[tc] + l1w * B[tc];
          const float bot = Z == 1 ? 0.f : l0w * Cc[tc] + l1w * D[tc];
          const float vt = row_lerp<Z>(top, bot, r);
          if constexpr (kOhem) {
            pt_out[pix] = expf(vt - lse);
            nll_out[pix] = kWeighted ? (class_weight ? class_weight[tc] : 1.f) * (lse - vt) : lse - vt;
          } else if constexpr (kWeightedCE) {
            // sum_c w_c (lse - v_c) = W (lse - m) + sum_c w_c (m - v_c): two non-negative terms for positive weights.
            // lse - m rather than a second __logf(sum): lse keeps the plain kernel's bits
            const float wt = s_w[tc];
            const float smooth = fmaf(s_w[C], lse - m[r], sw[r]);
            loss += fmaf((1.f - smoothing) * wt, lse - vt, (smoothing / C) * smooth);
            cnt += wt;
          } else {
            loss += lse - vt;
            cnt += 1.f;
          }
        } else if constexpr (kOhem) {
          pt_out[pix] = kInvalidPt;
          nll_out[pix] = 0.f;
        }
      }
    }
  }
  if constexpr (!kOhem) {
    // deterministic block reduction -> one partial per CTA
    for (int o = 16; o > 0; o >>= 1) {
      loss += __shfl_xor_sync(0xffffffffu, loss, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((tid & 31) == 0) {
      red_loss[tid >> 5] = loss;
      red_cnt[tid >> 5] = cnt;
    }
    __syncthreads();
    if (tid == 0) {
      float l = 0.f, k = 0.f;
      for (int i = 0; i < kFwdCols / 32; ++i) {
        l += red_loss[i];
        k += red_cnt[i];
      }
      const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
      partial[2 * b] = l;
      partial[2 * b + 1] = k;
    }
  }
}

// loss_out[0] = sum / max(count, 1) (mean over non-ignored pixels), loss_out[1] = count. Fixed summation order.
// kWeightedMean: the second partial is D = sum of w_t, and loss_out[0] = sum / D, 0 when D = 0 (the sum need not be 0
// then: label smoothing still scores the pixels of zero-weight classes).
template <bool kWeightedMean = false>
__global__ void upsample_ce_reduce_kernel(const float* __restrict__ partial, int nblocks, float* __restrict__ loss_out) {
  __shared__ double sl[256];
  __shared__ double sc[256];
  double l = 0.0, k = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += 256) {
    l += partial[2 * i];
    k += partial[2 * i + 1];
  }
  sl[threadIdx.x] = l;
  sc[threadIdx.x] = k;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sl[threadIdx.x] += sl[threadIdx.x + o];
      sc[threadIdx.x] += sc[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if constexpr (kWeightedMean) {
      loss_out[0] = sc[0] != 0.0 ? static_cast<float>(sl[0] / sc[0]) : 0.f;
    } else {
      loss_out[0] = static_cast<float>(sl[0] / (sc[0] > 0.0 ? sc[0] : 1.0));
    }
    loss_out[1] = static_cast<float>(sc[0]);
  }
}

// The reduce above for the other translation units (csrc/crf.cu): loss_out[0] = sum / count, loss_out[1] = count.
int launch_mean_reduce(const float* partial, int nblocks, float* loss_out, cudaStream_t stream) {
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(partial, nblocks, loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// ---------------------------------------------------------------------------------------------------- OHEM selection
// The k-th smallest p_t over the valid pixels, exactly: a radix select over the fp32 bit patterns (non-negative floats
// order like their uint32 patterns), four passes of 8 bits from the top. Each pass histograms the digit of the pixels
// whose higher digits equal the prefix found so far (integer counts: the result does not depend on the order of the
// atomics), then one CTA picks the digit that holds the k-th value. Device state only: no host synchronisation, so the
// whole selection is captured into a CUDA graph with the step. Workspace words (zeroed before the first pass):
constexpr int kSelPrefix = 0;     // digits found so far
constexpr int kSelK = 1;          // rank of the wanted value among the pixels matching the prefix
constexpr int kSelValid = 2;      // number of valid pixels n_v (pass 0)
constexpr int kSelHist = 4;       // [4 passes][256] counts
constexpr int kSelWords = kSelHist + 4 * 256;
constexpr int kSelThreads = 256;

__global__ void __launch_bounds__(kSelThreads)
ohem_hist_kernel(const float* __restrict__ pt, long long M, int pass, unsigned* __restrict__ sel) {
  __shared__ unsigned hist[256];
  hist[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const unsigned hi_mask = pass == 0 ? 0u : 0xffffffffu << (shift + 8);
  const unsigned prefix = sel[kSelPrefix];
  const int lane = threadIdx.x & 31;
  // base is CTA-uniform: every lane of a warp runs every iteration (the warp-aggregated add below needs all 32)
  for (long long base = static_cast<long long>(blockIdx.x) * kSelThreads; base < M;
       base += static_cast<long long>(gridDim.x) * kSelThreads) {
    const long long i = base + threadIdx.x;
    unsigned d = 0xffffffffu;
    if (i < M) {
      const float p = pt[i];
      const unsigned u = __float_as_uint(p);
      if (p >= 0.f && (u & hi_mask) == prefix) d = (u >> shift) & 255u;
    }
    // confident pixels share a few digits (every p_t in [0.5, 1] has top byte 0x3f): one add per distinct digit
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (d != 0xffffffffu && lane == __ffs(peers) - 1) atomicAdd(&hist[d], static_cast<unsigned>(__popc(peers)));
  }
  __syncthreads();
  if (hist[threadIdx.x]) atomicAdd(&sel[kSelHist + pass * 256 + threadIdx.x], hist[threadIdx.x]);
}

// One CTA: pass 0 counts n_v and sets k = min(min_kept, n_v - 1); every pass appends the digit whose bin holds rank k.
// After the last pass the prefix is the k-th smallest p_t and thr = max(thresh, it) (thresh when no pixel is valid).
__global__ void __launch_bounds__(kSelThreads)
ohem_select_kernel(unsigned* __restrict__ sel, int pass, float thresh, int min_kept, float* __restrict__ thr) {
  __shared__ unsigned cnt[256];
  cnt[threadIdx.x] = sel[kSelHist + pass * 256 + threadIdx.x];
  __syncthreads();
  if (threadIdx.x != 0) return;
  unsigned k, prefix;
  if (pass == 0) {
    unsigned nv = 0;
    for (int b = 0; b < 256; ++b) nv += cnt[b];
    sel[kSelValid] = nv;
    k = nv == 0 ? 0u : min(static_cast<unsigned>(min_kept), nv - 1u);
    prefix = 0;
  } else {
    k = sel[kSelK];
    prefix = sel[kSelPrefix];
  }
  unsigned d = 0;
  for (; d < 255; ++d) {
    if (k < cnt[d]) break;
    k -= cnt[d];
  }
  prefix |= d << (24 - 8 * pass);
  sel[kSelK] = k;
  sel[kSelPrefix] = prefix;
  if (pass == 3) thr[0] = sel[kSelValid] ? fmaxf(thresh, __uint_as_float(prefix)) : thresh;
}

// Kept pixels (p_t >= 0, i.e. valid, and p_t < thr): one (sum of nll, count) partial per kMaskPix pixels, fixed order;
// upsample_ce_reduce_kernel turns them into (mean, kept count).
constexpr int kMaskPix = 4096;

__global__ void __launch_bounds__(kSelThreads)
ohem_masked_sum_kernel(const float* __restrict__ pt, const float* __restrict__ nll, long long M,
                       const float* __restrict__ thr, float* __restrict__ partial) {
  __shared__ float red_loss[kSelThreads / 32];
  __shared__ float red_cnt[kSelThreads / 32];
  const float t = thr[0];
  const long long base = static_cast<long long>(blockIdx.x) * kMaskPix;
  float loss = 0.f, cnt = 0.f;
  for (int j = threadIdx.x; j < kMaskPix; j += kSelThreads) {
    const long long i = base + j;
    if (i < M) {
      const float p = pt[i];
      if (p >= 0.f && p < t) {
        loss += nll[i];
        cnt += 1.f;
      }
    }
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
    float l = 0.f, k = 0.f;
    for (int i = 0; i < kSelThreads / 32; ++i) {
      l += red_loss[i];
      k += red_cnt[i];
    }
    partial[2 * blockIdx.x] = l;
    partial[2 * blockIdx.x + 1] = k;
  }
}

// ---------------------------------------------------------------------------------------------------- backward
// Separable, deterministic, no atomics. With g[y,x,c] = softmax_{y,x}[c] - [c == t_{y,x}] (0 for ignored pixels):
//   dL[i,j,c] = gs * sum_y wy(y,i) * sum_x wx(x,j) * g[y,x,c].
// Phase 1 (rows): one CTA per (image, low-res interval row i0), one thread per class. The thread walks x = 0..Wo-1
// with the four node values of its class in registers; per column the horizontal interpolation (top, bot) is shared
// by the interval's Z output rows and the rows are folded immediately with their compile-time vertical weights, so at
// Z = 8 a pixel-class costs ~10 instructions and one MUFU. (lse*log2e, target) of the Z rows are staged in shared memory as
// one 8-byte word per pixel and read as warp-uniform broadcasts. Output: T2[n][i0][s][j][c], s = 0: the interval's
// contribution to node row i0, s = 1: to node row i0+1 (fp32 workspace, 68 MB at bs16 / 150 classes; at Z = 1 slot 1
// is all zeros).
// Phase 2 (cols): dL[i] = gs * (T2[i][0] + T2[i-1][1]).
// kOhem: a pixel is also ignored when its stored p_t is not below the device threshold, the forward's kept set bit for
// bit; the cols kernel then divides by the kept count in loss_info[1].
// kWeighted: the class weights and W are staged after the pixel words (the width limit of the staged rows is the plain
// one); a thread's own w_c is a register, a pixel's w_t a warp-uniform read of the table. g above becomes
// p_c ((1-eps) w_t + (eps/C) W) - [c = t] (1-eps) w_t - (eps/C) w_c, or w_t (p_c - [c = t]) with kOhem, and the
// weighted cols kernel divides by D = loss_info[1] (0 when D = 0).
struct __align__(8) PixInfo {
  float lse2;  // log-sum-exp * log2(e)
  int t;       // target class, -1 = ignored
};

// One pixel-class term g of the backward (see above) from p = softmax_c at the pixel.
template <bool kOhem, bool kWeighted>
__device__ __forceinline__ float pix_grad(float p, int c, int t, const float* s_w, float k1, float k2, float gam) {
  if constexpr (!kWeighted) {
    return p - (c == t ? 1.f : 0.f);
  } else if constexpr (kOhem) {
    return s_w[t] * (p - (c == t ? 1.f : 0.f));
  } else {
    const float beta = k1 * s_w[t];
    return fmaf(p, beta + k2, -(c == t ? beta + gam : gam));
  }
}

// kUnbiased (neither kOhem nor kWeighted): a pixel labelled with an old class (t < c_old) is staged with t = C, which no
// class matches, and its lse_old * log2(e) in a float array after the pixel words (12 bytes per pixel in all); the old
// classes' threads subtract exp(v_c - lse_old) from its p_c - [c = t] = p_c.
template <int Z, bool kOhem, bool kWeighted = false, bool kUnbiased = false>
__global__ void __launch_bounds__(256)
upsample_ce_bwd_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                            const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                            const float* __restrict__ lse, float* __restrict__ T2, const float* __restrict__ pt,
                            const float* __restrict__ thr, const float* __restrict__ class_weight = nullptr,
                            float smoothing = 0.f, int c_old = 0, const float* __restrict__ lse_old = nullptr) {
  using G = Zoom<Z>;
  extern __shared__ PixInfo s_pix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  float* s_w = reinterpret_cast<float*>(s_pix + Z * Wo);   // kWeighted: [C] class weights, then W
  float* s_lso = s_w;                                      // kUnbiased: [Z][Wo] lse_old * log2(e)
  if constexpr (kWeighted) stage_class_weights(class_weight, C, s_w);
  float thr_v = 0.f;
  if constexpr (kOhem) thr_v = thr[0];
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const long long t = target[rowbase + x];
      PixInfo pi;
      pi.t = (t == ignore_index || t < 0 || t >= C) ? -1 : static_cast<int>(t);
      if constexpr (kOhem) {
        if (!(pt[rowbase + x] < thr_v)) pi.t = -1;
      }
      if constexpr (kUnbiased) {
        if (pi.t >= 0 && pi.t < c_old) pi.t = C;
        s_lso[r * Wo + x] = lse_old[rowbase + x] * kLog2e;
      }
      pi.lse2 = lse[rowbase + x] * kLog2e;
      s_pix[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  float k1 = 0.f, k2 = 0.f, gam = 0.f;  // kWeighted, not kOhem: 1-eps, (eps/C) W, (eps/C) w_c
  if constexpr (kWeighted && !kOhem) {
    k1 = 1.f - smoothing;
    k2 = (smoothing / C) * s_w[C];
    gam = (smoothing / C) * s_w[c];
  }
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];      // left node column of the current interval (rows i0 / i1)
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;  // right-node contributions of the previous interval (node rows i0 / i1)
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;     // right node column (j1 = min(j0+1, w-1))
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];          // prefetch the next interval's right column
    nd = L1[static_cast<size_t>(jn) * pitch];
    float accL0 = 0.f, accR0 = 0.f, accL1 = 0.f, accR1 = 0.f;
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);   // Z, or 1 for the last node column
    if (rows == Z && nx == Z) {
#pragma unroll
      for (int k = 0; k < Z; ++k) {
        const float l1w = G::kStep * k, l0w = 1.f - l1w;
        const float top = l0w * a + l1w * b;
        const float bot = l0w * cc + l1w * d;
        float g0 = 0.f, g1 = 0.f;
#pragma unroll
        for (int r = 0; r < Z; ++r) {
          const PixInfo pi = s_pix[r * Wo + xb + k];
          if (pi.t < 0) continue;  // warp-uniform
          const float v = row_lerp<Z>(top, bot, r);
          float g = pix_grad<kOhem, kWeighted>(ex2_approx(fmaf(v, kLog2e, -pi.lse2)), c, pi.t, s_w, k1, k2, gam);
          if constexpr (kUnbiased) {
            if (c < c_old && pi.t == C) g -= ex2_approx(fmaf(v, kLog2e, -s_lso[r * Wo + xb + k]));
          }
          g0 = fmaf(1.f - G::kStep * r, g, g0);
          g1 = fmaf(G::kStep * r, g, g1);
        }
        accL0 = fmaf(l0w, g0, accL0);
        accR0 = fmaf(l1w, g0, accR0);
        accL1 = fmaf(l0w, g1, accL1);
        accR1 = fmaf(l1w, g1, accR1);
      }
    } else {
      for (int k = 0; k < nx; ++k) {
        const float l1w = G::kStep * k, l0w = 1.f - l1w;
        const float top = l0w * a + l1w * b;
        const float bot = l0w * cc + l1w * d;
        float g0 = 0.f, g1 = 0.f;
        for (int r = 0; r < rows; ++r) {
          const PixInfo pi = s_pix[r * Wo + xb + k];
          if (pi.t < 0) continue;
          const float l1h = G::kStep * r, l0h = 1.f - l1h;
          const float v = l0h * top + l1h * bot;
          float g = pix_grad<kOhem, kWeighted>(ex2_approx(fmaf(v, kLog2e, -pi.lse2)), c, pi.t, s_w, k1, k2, gam);
          if constexpr (kUnbiased) {
            if (c < c_old && pi.t == C) g -= ex2_approx(fmaf(v, kLog2e, -s_lso[r * Wo + xb + k]));
          }
          g0 = fmaf(l0h, g, g0);
          g1 = fmaf(l1h, g, g1);
        }
        accL0 = fmaf(l0w, g0, accL0);
        accR0 = fmaf(l1w, g0, accR0);
        accL1 = fmaf(l0w, g1, accL1);
        accR1 = fmaf(l1w, g1, accR1);
      }
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + accL0;
    T1[static_cast<size_t>(j0) * C] = carry1 + accL1;
    carry0 = accR0;
    carry1 = accR1;
    a = b;
    cc = d;
  }
}

template <bool kWeightedMean = false>
__global__ void __launch_bounds__(256)
upsample_ce_bwd_cols_kernel(const float* __restrict__ T2, int N, int h, int w, int C,
                            const float* __restrict__ loss_info, const float* __restrict__ grad_out,
                            float* __restrict__ dlogits) {
  const int i = blockIdx.x, n = blockIdx.y;
  const float cntv = loss_info[1];
  float gs;
  if constexpr (kWeightedMean) {
    gs = cntv != 0.f ? grad_out[0] / cntv : 0.f;   // D = sum of w_t; T2 need not be 0 when D = 0
  } else {
    gs = grad_out[0] / (cntv > 0.f ? cntv : 1.f);
  }
  const int wc = w * C;
  const float* own = T2 + ((static_cast<size_t>(n) * h + i) * 2 + 0) * wc;                 // interval i, top slot
  const float* prev = i > 0 ? T2 + ((static_cast<size_t>(n) * h + (i - 1)) * 2 + 1) * wc : nullptr;  // interval i-1, bottom
  for (int idx = threadIdx.x; idx < wc; idx += blockDim.x) {
    float acc = own[idx];
    if (prev) acc += prev[idx];
    dlogits[(static_cast<size_t>(n) * h + i) * wc + idx] = acc * gs;
  }
}

// ---------------------------------------------------------------------------------------------------- Dice
// Soft Dice loss (segmentation_models_pytorch's multiclass DiceLoss from logits, with ignore_index), alone or plus
// ce_weight * cross-entropy, summed over every pixel of every image of the call. With p = softmax(v), valid pixels i:
//   n_c = #{t_i = c},  I_c = sum p_ic [t_i = c],  S_c = sum p_ic + n_c,  D_c = max(S_c + smooth, eps)
//   L = (1/C) sum_{c: n_c > 0} (1 - (2 I_c + smooth) / D_c) + ce_weight * CE
//   dL/dv_ic = p_ic (beta_c + lam - G_i) - [c = t_i] (p_ic alpha_c + lam),   G_i = sum_c p_ic beta_c - p_it alpha_t
//   alpha_c = 2 m_c / (C D_c),  beta_c = m_c (2 I_c + smooth) / (C D_c^2) (0 where D_c is the clamp eps),
//   m_c = [n_c > 0],  lam = ce_weight / n_valid
// A pixel's gradient depends on sums over the whole call, so the criterion is a chain of passes:
//   forward : the plain forward instance (lse, argmax, CE partials: lse and argmax are the plain tail's bits), the
//             statistics pass (rows layout, one thread per class: (sum p, sum p at the target, n) per (interval, image)
//             and class, no cross-thread reduction), a per-class fp64 reduce in a fixed order (the (I, S, n) and
//             alpha / beta tables), and a one-CTA reduce of the loss;
//   backward: G_i in the forward's thread-per-pixel layout, the rows kernel with (lse, t, G) staged per pixel, and the
//             plain cols kernel (which divides by table[5C+1] = 1).
// Device table, 5C + 2 floats: alpha[C], beta[C], I[C], S[C], n[C], lam, 1.
struct DicePix {
  float lse2;  // log-sum-exp * log2(e)
  int t;       // target class, -1 = ignored
  float g;     // G_i (backward only)
};
constexpr int kDiceWords = 5;   // alpha, beta, I, S, n

// One interval (Z columns of Z rows; fewer at the last node row / column when !kFull) of the Dice rows kernel for
// class c. kGrad: acc = the (left, right) x (top, bottom node row) gradient sums as in upsample_ce_bwd_rows_kernel;
// else acc = (sum p, sum p at the target, target count).
template <int Z, bool kGrad, bool kFull>
__device__ __forceinline__ void dice_interval(const DicePix* s, int Wo, int xb, int rows, int nx, int c, float a,
                                              float b, float cc, float d, float ac, float bl, float lam, float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const DicePix pi = s[r * Wo + xb + k];
      if (pi.t < 0) continue;  // warp-uniform
      const float v = row_lerp<Z>(top, bot, r);
      const float p = ex2_approx(fmaf(v, kLog2e, -pi.lse2));
      if constexpr (kGrad) {
        const float q = p * (bl - pi.g);
        const float g = c == pi.t ? q - fmaf(p, ac, lam) : q;
        g0 = fmaf(1.f - G::kStep * r, g, g0);
        g1 = fmaf(G::kStep * r, g, g1);
      } else {
        acc[0] += p;
        if (c == pi.t) {
          acc[1] += p;
          acc[2] += 1.f;
        }
      }
    }
    if constexpr (kGrad) {
      acc[0] = fmaf(l0w, g0, acc[0]);
      acc[1] = fmaf(l1w, g0, acc[1]);
      acc[2] = fmaf(l0w, g1, acc[2]);
      acc[3] = fmaf(l1w, g1, acc[3]);
    }
  }
}

// Rows layout of upsample_ce_bwd_rows_kernel: one CTA per (low-res interval row i0, image), one thread per class,
// (lse, target[, G]) of the interval's Z output rows staged as one 12-byte word per pixel.
// !kGrad (statistics): out = partial[n][i0][3][C] = (sum p, sum p at the target, n) over the interval's valid pixels;
// each thread sums an interval column in fp32 and the columns in fp64, so a partial is rounded once.
// kGrad: out = T2 as in upsample_ce_bwd_rows_kernel, of the Dice (+ CE) gradient; gmap = G_i, table = the Dice table.
template <int Z, bool kGrad>
__global__ void __launch_bounds__(256)
upsample_ce_dice_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                             const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                             const float* __restrict__ lse, const float* __restrict__ gmap,
                             const float* __restrict__ table, float* __restrict__ out) {
  extern __shared__ DicePix s_dpix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const long long t = target[rowbase + x];
      DicePix pi;
      pi.t = (t == ignore_index || t < 0 || t >= C) ? -1 : static_cast<int>(t);
      pi.lse2 = lse[rowbase + x] * kLog2e;
      pi.g = kGrad ? gmap[rowbase + x] : 0.f;
      s_dpix[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  float ac = 0.f, bl = 0.f, lam = 0.f;  // kGrad: alpha_c, beta_c + lam, lam
  if constexpr (kGrad) {
    ac = table[c];
    lam = table[kDiceWords * C];
    bl = table[C + c] + lam;
  }
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = out + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;   // kGrad
  float* T1 = out + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;
  double sp = 0.0, si = 0.0, sn = 0.0;  // !kGrad
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];
    nd = L1[static_cast<size_t>(jn) * pitch];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      dice_interval<Z, kGrad, true>(s_dpix, Wo, xb, rows, nx, c, a, b, cc, d, ac, bl, lam, acc);
    } else {
      dice_interval<Z, kGrad, false>(s_dpix, Wo, xb, rows, nx, c, a, b, cc, d, ac, bl, lam, acc);
    }
    if constexpr (kGrad) {
      T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
      T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
      carry0 = acc[1];
      carry1 = acc[3];
    } else {
      sp += acc[0];
      si += acc[1];
      sn += acc[2];
    }
    a = b;
    cc = d;
  }
  if constexpr (!kGrad) {
    float* P = out + (static_cast<size_t>(n) * h + i0) * 3 * C + c;
    P[0] = static_cast<float>(sp);
    P[C] = static_cast<float>(si);
    P[2 * C] = static_cast<float>(sn);
  }
}

// One CTA per class: the class's statistics partials summed in fp64 in a fixed order, then its table entries and its
// loss term 1 - dice_c (0 for an absent class) into terms[c].
__global__ void __launch_bounds__(256)
dice_class_reduce_kernel(const float* __restrict__ partial, int nparts, int C, float smooth, float eps,
                         float* __restrict__ table, double* __restrict__ terms) {
  __shared__ double red[3][256];
  const int c = blockIdx.x;
  double sp = 0.0, si = 0.0, sn = 0.0;
  for (int i = threadIdx.x; i < nparts; i += 256) {
    const float* P = partial + static_cast<size_t>(i) * 3 * C + c;
    sp += P[0];
    si += P[C];
    sn += P[2 * C];
  }
  red[0][threadIdx.x] = sp;
  red[1][threadIdx.x] = si;
  red[2][threadIdx.x] = sn;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      red[0][threadIdx.x] += red[0][threadIdx.x + o];
      red[1][threadIdx.x] += red[1][threadIdx.x + o];
      red[2][threadIdx.x] += red[2][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double I = red[1][0], nc = red[2][0];
    const double S = red[0][0] + nc;
    const double num = 2.0 * I + smooth;
    const double D = fmax(S + smooth, static_cast<double>(eps));
    double alpha = 0.0, beta = 0.0, term = 0.0;
    if (nc > 0.0) {
      term = 1.0 - num / D;
      alpha = 2.0 / (C * D);
      beta = S + smooth < eps ? 0.0 : num / (C * D * D);   // a clamped denominator does not depend on p
    }
    table[c] = static_cast<float>(alpha);
    table[C + c] = static_cast<float>(beta);
    table[2 * C + c] = static_cast<float>(I);
    table[3 * C + c] = static_cast<float>(S);
    table[4 * C + c] = static_cast<float>(nc);
    terms[c] = term;
  }
}

// One CTA: CE = (sum of the forward's CE partials) / n_valid and sum_c terms[c], both in fp64 in a fixed order ->
// loss_out = (L, n_valid), table[5C] = lam, table[5C+1] = 1.
__global__ void __launch_bounds__(256)
dice_loss_kernel(const float* __restrict__ ce_partial, int nblocks, const double* __restrict__ terms, int C,
                 float ce_weight, float* __restrict__ loss_out, float* __restrict__ table) {
  __shared__ double sl[256];
  __shared__ double sc[256];
  __shared__ double st[256];
  double l = 0.0, k = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += 256) {
    l += ce_partial[2 * i];
    k += ce_partial[2 * i + 1];
  }
  sl[threadIdx.x] = l;
  sc[threadIdx.x] = k;
  st[threadIdx.x] = threadIdx.x < C ? terms[threadIdx.x] : 0.0;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sl[threadIdx.x] += sl[threadIdx.x + o];
      sc[threadIdx.x] += sc[threadIdx.x + o];
      st[threadIdx.x] += st[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double nv = sc[0];
    const double ce = nv > 0.0 ? sl[0] / nv : 0.0;
    loss_out[0] = static_cast<float>(st[0] / C + static_cast<double>(ce_weight) * ce);
    loss_out[1] = static_cast<float>(nv);
    table[kDiceWords * C] = nv > 0.0 ? static_cast<float>(ce_weight / nv) : 0.f;
    table[kDiceWords * C + 1] = 1.f;
  }
}

// G_i = sum_c p_ic beta_c - p_it alpha_t per valid pixel (0 elsewhere), in the forward's layout: one CTA per (128
// output columns, interval row, image), one thread per output column and its Z rows, the node rows and the alpha /
// beta tables staged in shared memory.
template <int Z>
__global__ void __launch_bounds__(kFwdCols)
upsample_ce_dice_g_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                          const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                          const float* __restrict__ lse, const float* __restrict__ table, float* __restrict__ gmap) {
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs], then alpha[C], beta[C]
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  float* s_ab = S + G::kNodeRows * kFwdNodes * Cs;
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  for (int c = tid; c < 2 * C; c += kFwdCols) s_ab[c] = table[c];
  __syncthreads();
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x >= Wo) return;
  const int j0 = x >> G::kShift;
  const int j1 = min(j0 + 1, w - 1);
  const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
  const float* A = S + (j0 - j_base) * Cs;
  const float* B = S + (j1 - j_base) * Cs;
  const float* Cc = A + kFwdNodes * Cs;
  const float* D = B + kFwdNodes * Cs;
  float lse2[Z], g[Z];
#pragma unroll
  for (int r = 0; r < Z; ++r) {
    g[r] = 0.f;
    lse2[r] = r < rows ? lse[(static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x] * kLog2e : 0.f;
  }
#pragma unroll 2
  for (int c = 0; c < C; ++c) {
    const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
    const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
    const float beta = s_ab[C + c];
#pragma unroll
    for (int r = 0; r < Z; ++r) g[r] = fmaf(ex2_approx(fmaf(row_lerp<Z>(top, bot, r), kLog2e, -lse2[r])), beta, g[r]);
  }
#pragma unroll
  for (int r = 0; r < Z; ++r) {
    if (r < rows) {
      const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
      const long long t = target[pix];
      float gv = 0.f;
      if (t != ignore_index && t >= 0 && t < C) {
        const int tc = static_cast<int>(t);
        const float top = Z == 1 ? A[tc] : l0w * A[tc] + l1w * B[tc];
        const float bot = Z == 1 ? 0.f : l0w * Cc[tc] + l1w * D[tc];
        const float pt = ex2_approx(fmaf(row_lerp<Z>(top, bot, r), kLog2e, -lse2[r]));
        gv = fmaf(-pt, s_ab[tc], g[r]);
      }
      gmap[pix] = gv;
    }
  }
}

// ---------------------------------------------------------------------------------------------------- Lovász-Softmax
// Lovász-Softmax (Berman, Triki, Blaschko, CVPR 2018), alone or plus ce_weight * cross-entropy. A segment is one class
// over every valid pixel of the call, or one (image, class) pair with per_image. Per segment, with fg_i = [t_i = c],
// e_i = |fg_i - p_ic| (fp32), G = sum fg_i and the valid pixels sorted by e descending, ties by flat pixel index:
//   A_k, B_k = fg / bg counts among the first k,  J_k = 1 - (G - A_k) / (G + B_k),  J_0 = 0,  g_k = J_k - J_{k-1}
//   loss_seg = sum_k e_(k) g_k,   loss = sum_seg w_seg loss_seg + ce_weight * CE
// w_seg is 1 / (number of segments considered) (per_image: 1 / (N * the image's count)); 'present' considers the
// segments with G > 0, 'all' every segment of a scope that has a valid pixel. With the sort order held fixed:
//   gamma_ic = w_seg g_k sign(p_ic - fg_i),  Gamma_i = sum_c p_ic gamma_ic
//   dL/dv_ic = p_ic (gamma_ic - Gamma_i) + lam (p_ic - fg_i),  lam = ce_weight / n_valid
// Every pass computes p_ic the same way, the interpolation spelled out in explicit fmas (lovasz_v), so the key pass,
// the Gamma pass and the rows kernel see the same bits and agree on every sign, zeros included.
//   forward : the plain forward instance (lse, argmax, CE partials); a target histogram per image; one CTA turns it into
//             the per-segment (skip, G, w) table; the key pass writes key = 0x7FFFFFFF - bits(e) (0xFFFFFFFF for an
//             invalid pixel, sorted last) and payload = (pixel index << 1) | fg for each considered segment, in pixel
//             order; the segmented stable radix sort (csrc/segsort.cu); per sorted tile the fg count, a per-segment
//             scan of those counts, and the gradient pass (J_k in fp64 from integer counts, fp64 partials of e g_k,
//             and the scatter of w_seg g_k into the kept gamma map [P][C]); one CTA reduces the loss in a fixed order.
//   backward: Gamma_i (one warp per pixel, the sign applied from p), the rows kernel with (lse, t, Gamma) staged per
//             pixel and gamma read per pixel-class, then the plain cols kernel.
constexpr int kLovThreads = 256;
constexpr int kLovItems = 16;
constexpr int kLovTile = kLovThreads * kLovItems;   // sorted pairs per CTA of the scan passes
constexpr unsigned kLovInvalidKey = 0xFFFFFFFFu;

// The interpolated logit of output pixel (row r, column k) of an interval from its four node values.
template <int Z>
__device__ __forceinline__ float lovasz_h(float a, float b, int k) {
  if constexpr (Z == 1) {
    return a;
  } else {
    const float l1 = Zoom<Z>::kStep * k;
    return fmaf(1.f - l1, a, __fmul_rn(l1, b));
  }
}
template <int Z>
__device__ __forceinline__ float lovasz_v(float top, float bot, int r) {
  if constexpr (Z == 1) {
    return top;
  } else {
    const float l1 = Zoom<Z>::kStep * r;
    return fmaf(1.f - l1, top, __fmul_rn(l1, bot));
  }
}
__device__ __forceinline__ float lovasz_sign(float p, float fg) { return p > fg ? 1.f : p < fg ? -1.f : 0.f; }

// Valid pixels per (image, class) and per image: hist[n][C + 1] (zeroed by the caller; integer atomics).
__global__ void __launch_bounds__(256)
lovasz_target_hist_kernel(const long long* __restrict__ target, int HW, int C, int ignore_index,
                          int* __restrict__ hist) {
  __shared__ int s[kMaxClasses + 1];
  const int n = blockIdx.y;
  for (int c = threadIdx.x; c <= C; c += 256) s[c] = 0;
  __syncthreads();
  const long long* T = target + static_cast<size_t>(n) * HW;
  const int base = blockIdx.x * kLovTile;
  const int end = min(base + kLovTile, HW);
  for (int i = base + threadIdx.x; i < end; i += 256) {
    const long long t = T[i];
    if (t != ignore_index && t >= 0 && t < C) {
      atomicAdd(&s[t], 1);
      atomicAdd(&s[C], 1);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c <= C; c += 256)
    if (s[c]) atomicAdd(&hist[n * (C + 1) + c], s[c]);
}

// One CTA, one thread per class: skip[seg], G[seg], w[seg] of every segment (seg = c, or n * C + c with per_image).
__global__ void __launch_bounds__(kMaxClasses)
lovasz_segments_kernel(const int* __restrict__ hist, int N, int C, int classes_all, int per_image,
                       int* __restrict__ skip, int* __restrict__ seg_g, double* __restrict__ seg_w) {
  const int c = threadIdx.x;
  const bool cls = c < C;
  if (!per_image) {
    int g = 0, nv = 0;
    for (int n = 0; n < N; ++n) {
      if (cls) g += hist[n * (C + 1) + c];
      nv += hist[n * (C + 1) + C];
    }
    const int cnt = classes_all ? (nv > 0 ? C : 0) : __syncthreads_count(cls && g > 0);
    const bool considered = classes_all ? nv > 0 : g > 0;
    if (cls) {
      skip[c] = !considered;
      seg_g[c] = g;
      seg_w[c] = considered ? 1.0 / cnt : 0.0;
    }
    return;
  }
  for (int n = 0; n < N; ++n) {
    const int g = cls ? hist[n * (C + 1) + c] : 0;
    const int nv = hist[n * (C + 1) + C];
    const int cnt = classes_all ? (nv > 0 ? C : 0) : __syncthreads_count(g > 0);
    const bool considered = classes_all ? nv > 0 : g > 0;
    if (cls) {
      skip[n * C + c] = !considered;
      seg_g[n * C + c] = g;
      seg_w[n * C + c] = considered ? 1.0 / (static_cast<double>(N) * cnt) : 0.0;
    }
  }
}

// Forward layout (one CTA per 128 output columns, interval row, image; one thread per column and its Z rows): for every
// considered segment, each pixel's sort key and payload at its position in the segment (pixel order).
template <int Z>
__global__ void __launch_bounds__(kFwdCols)
lovasz_key_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                  const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                  const float* __restrict__ lse, int per_image, const int* __restrict__ skip,
                  unsigned* __restrict__ keys, unsigned* __restrict__ vals) {
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs], then the skip flags of the image's C segments
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  int* s_skip = reinterpret_cast<int*>(S + G::kNodeRows * kFwdNodes * Cs);
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  for (int c = tid; c < C; c += kFwdCols) s_skip[c] = skip[per_image ? n * C + c : c];
  __syncthreads();
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x >= Wo) return;
  const int j0 = x >> G::kShift;
  const int j1 = min(j0 + 1, w - 1);
  const int k = x & G::kMask;
  const float* A = S + (j0 - j_base) * Cs;
  const float* B = S + (j1 - j_base) * Cs;
  const float* Cc = A + kFwdNodes * Cs;
  const float* D = B + kFwdNodes * Cs;
  const size_t L = per_image ? static_cast<size_t>(Ho) * Wo : static_cast<size_t>(N) * Ho * Wo;
  float lse2[Z];
  int t[Z];
  unsigned pix[Z];
#pragma unroll
  for (int r = 0; r < Z; ++r) {
    const size_t p = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
    pix[r] = static_cast<unsigned>(p);
    t[r] = -1;
    lse2[r] = 0.f;
    if (r < rows) {
      const long long tv = target[p];
      t[r] = (tv == ignore_index || tv < 0 || tv >= C) ? -1 : static_cast<int>(tv);
      lse2[r] = lse[p] * kLog2e;
    }
  }
  const size_t local0 = per_image ? static_cast<size_t>(Z * i0) * Wo + x : pix[0];
  for (int c = 0; c < C; ++c) {
    if (s_skip[c]) continue;   // CTA-uniform
    const float top = lovasz_h<Z>(A[c], B[c], k);
    const float bot = Z == 1 ? 0.f : lovasz_h<Z>(Cc[c], D[c], k);
    const size_t seg = per_image ? static_cast<size_t>(n) * C + c : c;
    unsigned* K = keys + seg * L + local0;
    unsigned* V = vals + seg * L + local0;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const float p = ex2_approx(fmaf(lovasz_v<Z>(top, bot, r), kLog2e, -lse2[r]));
        const bool fg = t[r] == c;
        const float e = fabsf((fg ? 1.f : 0.f) - p);
        K[static_cast<size_t>(r) * Wo] = t[r] < 0 ? kLovInvalidKey : 0x7FFFFFFFu - __float_as_uint(e);
        V[static_cast<size_t>(r) * Wo] = (pix[r] << 1) | (fg ? 1u : 0u);
      }
    }
  }
}

// Block-wide exclusive scan of one value per thread (kLovThreads threads); returns the thread's prefix and, through
// total, the block's sum. Integer adds: the order does not matter.
__device__ __forceinline__ unsigned lovasz_block_scan(unsigned v, unsigned* total) {
  __shared__ unsigned ws[kLovThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) ws[warp] = inc;
  __syncthreads();
  unsigned before = 0, all = 0;
  for (int i = 0; i < kLovThreads / 32; ++i) {
    if (i < warp) before += ws[i];
    all += ws[i];
  }
  __syncthreads();
  *total = all;
  return before + inc - v;
}

// fg pairs per sorted tile -> fgcnt[seg][tile].
__global__ void __launch_bounds__(kLovThreads)
lovasz_fgcount_kernel(const unsigned* __restrict__ vals, int L, int nt, const int* __restrict__ skip,
                      unsigned* __restrict__ fgcnt) {
  const int seg = blockIdx.x / nt, tile = blockIdx.x % nt;
  if (skip[seg]) return;
  const unsigned* V = vals + static_cast<size_t>(seg) * L;
  const int base = tile * kLovTile, end = min(base + kLovTile, L);
  unsigned cnt = 0;
  for (int i = base + threadIdx.x; i < end; i += kLovThreads) cnt += V[i] & 1u;
  unsigned total;
  lovasz_block_scan(cnt, &total);
  if (threadIdx.x == 0) fgcnt[blockIdx.x] = total;
}

// One CTA per segment: the exclusive scan of its tiles' fg counts, in place.
__global__ void __launch_bounds__(kLovThreads)
lovasz_fgscan_kernel(unsigned* __restrict__ fgcnt, int nt, const int* __restrict__ skip) {
  const int seg = blockIdx.x;
  if (skip[seg]) return;
  unsigned* F = fgcnt + static_cast<size_t>(seg) * nt;
  const int chunk = (nt + kLovThreads - 1) / kLovThreads;
  const int b = min(static_cast<int>(threadIdx.x) * chunk, nt), e = min(b + chunk, nt);
  unsigned s = 0;
  for (int i = b; i < e; ++i) s += F[i];
  unsigned total;
  unsigned run = lovasz_block_scan(s, &total);
  for (int i = b; i < e; ++i) {
    const unsigned c = F[i];
    F[i] = run;
    run += c;
  }
}

// One CTA per (segment, sorted tile); thread t owns the tile's pairs t*kLovItems .. +kLovItems-1 (staged through
// shared memory, one padding word per 32). Writes gamma[pix][c] = w_seg g_k for the valid pairs and the tile's fp64
// partial of sum e g_k (a fixed-order reduction) to partial[seg][tile].
__global__ void __launch_bounds__(kLovThreads)
lovasz_grad_kernel(const unsigned* __restrict__ keys, const unsigned* __restrict__ vals, int L, int nt, int C,
                   int per_image, const int* __restrict__ skip, const int* __restrict__ seg_g,
                   const double* __restrict__ seg_w, const unsigned* __restrict__ fgbase, float* __restrict__ gamma,
                   double* __restrict__ partial) {
  __shared__ unsigned sk[kLovTile + kLovTile / 32];
  __shared__ unsigned sv[kLovTile + kLovTile / 32];
  __shared__ double red[kLovThreads / 32];
  const int seg = blockIdx.x / nt, tile = blockIdx.x % nt;
  if (skip[seg]) return;
  const size_t off = static_cast<size_t>(seg) * L;
  const int base = tile * kLovTile;
  const int n = min(kLovTile, L - base);
  for (int i = threadIdx.x; i < kLovTile; i += kLovThreads) {
    sk[i + (i >> 5)] = i < n ? keys[off + base + i] : kLovInvalidKey;
    sv[i + (i >> 5)] = i < n ? vals[off + base + i] : 0u;
  }
  __syncthreads();
  const int i0 = threadIdx.x * kLovItems;
  unsigned cnt = 0;
#pragma unroll
  for (int j = 0; j < kLovItems; ++j) cnt += sv[i0 + j + ((i0 + j) >> 5)] & 1u;
  unsigned total;
  unsigned a = fgbase[blockIdx.x] + lovasz_block_scan(cnt, &total);   // fg pairs before this thread's first
  const double g_all = seg_g[seg], wv = seg_w[seg];
  const int c = per_image ? seg % C : seg;
  double acc = 0.0;
  for (int j = 0; j < kLovItems; ++j) {
    const int i = i0 + j;
    const unsigned key = sk[i + (i >> 5)];
    if (key == kLovInvalidKey) break;   // invalid pixels (and the tile's tail) sort last
    const unsigned v = sv[i + (i >> 5)];
    const unsigned fg = v & 1u;
    const double k = static_cast<double>(base + i + 1);   // rank in the segment, 1-based
    const double a1 = a + fg;
    const double jk = 1.0 - (g_all - a1) / (g_all + (k - a1));
    const double jp = k == 1.0 ? 0.0 : 1.0 - (g_all - a) / (g_all + (k - 1.0 - a));
    const double gk = jk - jp;
    acc += static_cast<double>(__uint_as_float(0x7FFFFFFFu - key)) * gk;
    gamma[static_cast<size_t>(v >> 1) * C + c] = static_cast<float>(wv * gk);
    a += fg;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < kLovThreads / 32; ++i) s += red[i];
    partial[blockIdx.x] = s;
  }
}

// One CTA: CE = (sum of the forward's CE partials) / n_valid and sum over the considered segments' tiles of
// w_seg * partial, both fp64 in a fixed order -> loss_out = (L, n_valid), tail = (lam, 1).
__global__ void __launch_bounds__(256)
lovasz_loss_kernel(const float* __restrict__ ce_partial, int nblocks, const double* __restrict__ partial, int S, int nt,
                   const int* __restrict__ skip, const double* __restrict__ seg_w, float ce_weight,
                   float* __restrict__ loss_out, float* __restrict__ tail) {
  __shared__ double sl[256];
  __shared__ double sc[256];
  __shared__ double st[256];
  double l = 0.0, k = 0.0, t = 0.0;
  for (int i = threadIdx.x; i < nblocks; i += 256) {
    l += ce_partial[2 * i];
    k += ce_partial[2 * i + 1];
  }
  const long long m = static_cast<long long>(S) * nt;
  for (long long i = threadIdx.x; i < m; i += 256) {
    const int seg = static_cast<int>(i / nt);
    if (!skip[seg]) t += seg_w[seg] * partial[i];
  }
  sl[threadIdx.x] = l;
  sc[threadIdx.x] = k;
  st[threadIdx.x] = t;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sl[threadIdx.x] += sl[threadIdx.x + o];
      sc[threadIdx.x] += sc[threadIdx.x + o];
      st[threadIdx.x] += st[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double nv = sc[0];
    const double ce = nv > 0.0 ? sl[0] / nv : 0.0;
    loss_out[0] = static_cast<float>(st[0] + static_cast<double>(ce_weight) * ce);
    loss_out[1] = static_cast<float>(nv);
    tail[0] = nv > 0.0 ? static_cast<float>(ce_weight / nv) : 0.f;
    tail[1] = 1.f;
  }
}

// Gamma_i = sum_c p_ic gamma_ic, one warp per output pixel (0 for an invalid pixel): the lanes read the pixel's four
// node vectors and its gamma row across the classes, a fixed shuffle tree sums them.
template <int Z>
__global__ void __launch_bounds__(256)
lovasz_gamma_sum_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                        const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                        const float* __restrict__ lse, const float* __restrict__ gamma, float* __restrict__ gmap) {
  using G = Zoom<Z>;
  const long long P = static_cast<long long>(N) * Ho * Wo;
  const long long pix = static_cast<long long>(blockIdx.x) * (256 / 32) + (threadIdx.x >> 5);
  if (pix >= P) return;
  const int lane = threadIdx.x & 31;
  const int x = static_cast<int>(pix % Wo);
  const long long ny = pix / Wo;
  const int y = static_cast<int>(ny % Ho), n = static_cast<int>(ny / Ho);
  const long long tv = target[pix];
  if (tv == ignore_index || tv < 0 || tv >= C) {
    if (lane == 0) gmap[pix] = 0.f;
    return;
  }
  const int t = static_cast<int>(tv);
  const int i0 = y >> G::kShift, r = y & G::kMask, j0 = x >> G::kShift, k = x & G::kMask;
  const int i1 = min(i0 + 1, h - 1), j1 = min(j0 + 1, w - 1);
  const float* A = logits + ((static_cast<size_t>(n) * h + i0) * w + j0) * pitch;
  const float* B = logits + ((static_cast<size_t>(n) * h + i0) * w + j1) * pitch;
  const float* Cc = logits + ((static_cast<size_t>(n) * h + i1) * w + j0) * pitch;
  const float* D = logits + ((static_cast<size_t>(n) * h + i1) * w + j1) * pitch;
  const float lse2 = lse[pix] * kLog2e;
  const float* gr = gamma + static_cast<size_t>(pix) * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float top = lovasz_h<Z>(A[c], B[c], k);
    const float bot = Z == 1 ? 0.f : lovasz_h<Z>(Cc[c], D[c], k);
    const float p = ex2_approx(fmaf(lovasz_v<Z>(top, bot, r), kLog2e, -lse2));
    s = fmaf(p, gr[c] * lovasz_sign(p, c == t ? 1.f : 0.f), s);
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) gmap[pix] = s;
}

// One interval of the Lovász rows kernel for class c (the Dice rows kernel's layout and folding):
// g = p (gamma sign - Gamma) + lam (p - fg) per valid pixel.
template <int Z, bool kFull>
__device__ __forceinline__ void lovasz_interval(const DicePix* s, const float* __restrict__ gam_row, int Wo, int C,
                                                int xb, int rows, int nx, int c, float a, float b, float cc, float d,
                                                float lam, float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float top = lovasz_h<Z>(a, b, k);
    const float bot = Z == 1 ? 0.f : lovasz_h<Z>(cc, d, k);
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const DicePix pi = s[r * Wo + xb + k];
      if (pi.t < 0) continue;  // warp-uniform
      const float p = ex2_approx(fmaf(lovasz_v<Z>(top, bot, r), kLog2e, -pi.lse2));
      const float fg = c == pi.t ? 1.f : 0.f;
      const float gm = gam_row[(static_cast<size_t>(r) * Wo + xb + k) * C] * lovasz_sign(p, fg);
      const float g = fmaf(p, gm - pi.g, lam * (p - fg));
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

// The rows kernel of the Lovász backward: one CTA per (interval row, image), one thread per class, (lse, t, Gamma)
// of the interval's Z output rows staged as one 12-byte word per pixel -> T2 as upsample_ce_bwd_rows_kernel's.
template <int Z>
__global__ void __launch_bounds__(256)
lovasz_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                   const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                   const float* __restrict__ lse, const float* __restrict__ gmap, const float* __restrict__ gamma,
                   float* __restrict__ T2) {
  extern __shared__ DicePix s_lpix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const long long t = target[rowbase + x];
      DicePix pi;
      pi.t = (t == ignore_index || t < 0 || t >= C) ? -1 : static_cast<int>(t);
      pi.lse2 = lse[rowbase + x] * kLog2e;
      pi.g = gmap[rowbase + x];
      s_lpix[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const float lam = gamma[static_cast<size_t>(N) * Ho * Wo * C];
  const float* gam_row = gamma + (static_cast<size_t>(n) * Ho + Z * i0) * Wo * C + c;
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];
    nd = L1[static_cast<size_t>(jn) * pitch];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      lovasz_interval<Z, true>(s_lpix, gam_row, Wo, C, xb, rows, nx, c, a, b, cc, d, lam, acc);
    } else {
      lovasz_interval<Z, false>(s_lpix, gam_row, Wo, C, xb, rows, nx, c, a, b, cc, d, lam, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
  }
}

// ---------------------------------------------------------------------------------------------------- distillation
// Pixel-wise knowledge distillation from a frozen teacher: the student logits s and the teacher logits t, both upsampled
// xZ exactly as the cross-entropy forward upsamples (Z = 1: the maps themselves), T the temperature, every pixel of
// every image (no target), P pixels in all:
//   log p_c = (s_c - m_s)/T - log Z_s,  Z_s = sum_c exp((s_c - m_s)/T),  m_s = max_c s_c     (log q_c likewise from t)
//   KL = (1/P) sum_pix sum_c q_c (log q_c - log p_c),   dKL/ds_c = (p_c - q_c) / (T P)
// Each log-probability is formed from its own shifted logit, never as a difference of two large sums, so s = t gives
// log q_c - log p_c = 0 bit for bit: a KL and a gradient of exactly 0.
//   forward : one CTA per (kKdCols output columns, interval row, image), the node rows of both maps staged side by side,
//             three class passes per pixel (max; the two sums of exp; the KL terms: three MUFU per pixel-class), fp32
//             within the CTA, one (sum KL, pixels) partial per CTA and the plain fp64 reduce; (lse_s/T, lse_t/T) saved per
//             pixel. 64 columns at Z <= 2, so that two maps of 256 classes fit in shared memory.
//   backward: the rows layout of upsample_ce_bwd_rows_kernel (one thread per class, both maps' node values in
//             registers, (lse_s/T, lse_t/T) log2(e) staged per pixel, two MUFU per pixel-class), then a cols kernel that
//             ADDS grad_out[0] kd_weight T / P times the adjoint into dlogits, which already holds the CE gradient.
template <int Z>
struct KdGeom {
  static constexpr int kCols = Z <= 2 ? 64 : 128;   // output columns per forward CTA
  static constexpr int kNodes = kCols / Z + 1;
};

template <int Z>
__global__ void __launch_bounds__(KdGeom<Z>::kCols)
upsample_kd_fwd_kernel(const float* __restrict__ sl, int pitch_s, const float* __restrict__ tl, int pitch_t, int N, int h,
                       int w, int C, int Cs, int Ho, int Wo, float inv_t, float* __restrict__ partial,
                       float2* __restrict__ lse_out) {
  using G = Zoom<Z>;
  constexpr int kCols = KdGeom<Z>::kCols, kNodes = KdGeom<Z>::kNodes;
  extern __shared__ float S[];  // [2 maps: student, teacher][kNodeRows][kNodes][Cs]
  __shared__ float red_kl[kCols / 32];
  __shared__ float red_cnt[kCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kNodes, w - j_base);
  const int tid = threadIdx.x;
  const int map_floats = G::kNodeRows * kNodes * Cs;
  for (int idx = tid; idx < 2 * G::kNodeRows * nj * C; idx += kCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = (node / nj) % G::kNodeRows, map = node / (nj * G::kNodeRows);
    const size_t src = (static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj);
    S[map * map_floats + (rr * kNodes + jj) * Cs + c] = map ? tl[src * pitch_t + c] : sl[src * pitch_s + c];
  }
  __syncthreads();
  float kl_sum = 0.f, cnt = 0.f;
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* As = S + (j0 - j_base) * Cs;   // student nodes (i0, j0), (i0, j1), (i1, j0), (i1, j1)
    const float* Bs = S + (j1 - j_base) * Cs;
    const float* Cs_ = As + kNodes * Cs;
    const float* Ds = Bs + kNodes * Cs;
    const float* At = As + map_floats;           // teacher nodes
    const float* Bt = Bs + map_floats;
    const float* Ct = Cs_ + map_floats;
    const float* Dt = Ds + map_floats;
    const float k2 = inv_t * kLog2e;
    float ms[Z], mt[Z], zs[Z], zt[Z], kl[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      ms[r] = -INFINITY;
      mt[r] = -INFINITY;
      zs[r] = 0.f;
      zt[r] = 0.f;
      kl[r] = 0.f;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float ts = Z == 1 ? As[c] : l0w * As[c] + l1w * Bs[c];
      const float bs = Z == 1 ? 0.f : l0w * Cs_[c] + l1w * Ds[c];
      const float tt = Z == 1 ? At[c] : l0w * At[c] + l1w * Bt[c];
      const float bt = Z == 1 ? 0.f : l0w * Ct[c] + l1w * Dt[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        ms[r] = fmaxf(ms[r], row_lerp<Z>(ts, bs, r));
        mt[r] = fmaxf(mt[r], row_lerp<Z>(tt, bt, r));
      }
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float ts = Z == 1 ? As[c] : l0w * As[c] + l1w * Bs[c];
      const float bs = Z == 1 ? 0.f : l0w * Cs_[c] + l1w * Ds[c];
      const float tt = Z == 1 ? At[c] : l0w * At[c] + l1w * Bt[c];
      const float bt = Z == 1 ? 0.f : l0w * Ct[c] + l1w * Dt[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        zs[r] += ex2_approx((row_lerp<Z>(ts, bs, r) - ms[r]) * k2);
        zt[r] += ex2_approx((row_lerp<Z>(tt, bt, r) - mt[r]) * k2);
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      zs[r] = logf(zs[r]);   // log Z_s, log Z_t from here on
      zt[r] = logf(zt[r]);
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float ts = Z == 1 ? As[c] : l0w * As[c] + l1w * Bs[c];
      const float bs = Z == 1 ? 0.f : l0w * Cs_[c] + l1w * Ds[c];
      const float tt = Z == 1 ? At[c] : l0w * At[c] + l1w * Bt[c];
      const float bt = Z == 1 ? 0.f : l0w * Ct[c] + l1w * Dt[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float lp = (row_lerp<Z>(ts, bs, r) - ms[r]) * inv_t - zs[r];
        const float lq = (row_lerp<Z>(tt, bt, r) - mt[r]) * inv_t - zt[r];
        kl[r] = fmaf(ex2_approx(lq * kLog2e), lq - lp, kl[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        lse_out[pix] = make_float2(fmaf(ms[r], inv_t, zs[r]), fmaf(mt[r], inv_t, zt[r]));
        kl_sum += kl[r];
        cnt += 1.f;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    kl_sum += __shfl_xor_sync(0xffffffffu, kl_sum, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((tid & 31) == 0) {
    red_kl[tid >> 5] = kl_sum;
    red_cnt[tid >> 5] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    float l = 0.f, k = 0.f;
    for (int i = 0; i < kCols / 32; ++i) {
      l += red_kl[i];
      k += red_cnt[i];
    }
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * b] = l;
    partial[2 * b + 1] = k;
  }
}

// One interval (Z columns of Z rows; fewer at the last node row / column when !kFull) of the distillation rows kernel
// for class c: acc = the (left, right) x (top, bottom node row) sums of p_c - q_c, as in upsample_ce_bwd_rows_kernel.
template <int Z, bool kFull>
__device__ __forceinline__ void kd_interval(const float2* s, int Wo, int xb, int rows, int nx, float k2, float a,
                                            float b, float cc, float d, float at, float bt, float ct, float dt,
                                            float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    const float topt = l0w * at + l1w * bt;
    const float bott = l0w * ct + l1w * dt;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const float2 l2 = s[r * Wo + xb + k];
      const float p = ex2_approx(fmaf(row_lerp<Z>(top, bot, r), k2, -l2.x));
      const float q = ex2_approx(fmaf(row_lerp<Z>(topt, bott, r), k2, -l2.y));
      const float g = p - q;
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

// One CTA per (low-res interval row i0, image), one thread per class; out = T2[n][i0][2][w][C] of sum (p_c - q_c).
template <int Z>
__global__ void __launch_bounds__(256)
upsample_kd_bwd_rows_kernel(const float* __restrict__ sl, int pitch_s, const float* __restrict__ tl, int pitch_t, int N,
                            int h, int w, int C, int Ho, int Wo, float inv_t, const float2* __restrict__ lse,
                            float* __restrict__ T2) {
  extern __shared__ float2 s_kpix[];  // [Z][Wo]: (lse_s/T, lse_t/T) * log2(e)
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const float2 l = lse[rowbase + x];
      s_kpix[r * Wo + x] = make_float2(l.x * kLog2e, l.y * kLog2e);
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const float k2 = inv_t * kLog2e;
  const float* S0 = sl + (static_cast<size_t>(n) * h + i0) * w * pitch_s + c;
  const float* S1 = sl + (static_cast<size_t>(n) * h + i1) * w * pitch_s + c;
  const float* U0 = tl + (static_cast<size_t>(n) * h + i0) * w * pitch_t + c;
  const float* U1 = tl + (static_cast<size_t>(n) * h + i1) * w * pitch_t + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  const int j1 = min(1, w - 1);
  float a = S0[0], cc = S1[0], at = U0[0], ct = U1[0];   // left node column of the current interval
  float nb = S0[static_cast<size_t>(j1) * pitch_s], nd = S1[static_cast<size_t>(j1) * pitch_s];
  float nbt = U0[static_cast<size_t>(j1) * pitch_t], ndt = U1[static_cast<size_t>(j1) * pitch_t];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd, bt = nbt, dt = ndt;
    const int jn = min(j0 + 2, w - 1);
    nb = S0[static_cast<size_t>(jn) * pitch_s];
    nd = S1[static_cast<size_t>(jn) * pitch_s];
    nbt = U0[static_cast<size_t>(jn) * pitch_t];
    ndt = U1[static_cast<size_t>(jn) * pitch_t];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      kd_interval<Z, true>(s_kpix, Wo, xb, rows, nx, k2, a, b, cc, d, at, bt, ct, dt, acc);
    } else {
      kd_interval<Z, false>(s_kpix, Wo, xb, rows, nx, k2, a, b, cc, d, at, bt, ct, dt, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
    at = bt;
    ct = dt;
  }
}

// dlogits[i] += grad_out[0] * scale * (T2[i][0] + T2[i-1][1]): the cols step of upsample_ce_bwd_cols_kernel, adding to
// the gradient already in dlogits instead of writing it.
__global__ void __launch_bounds__(256)
upsample_kd_bwd_cols_kernel(const float* __restrict__ T2, int N, int h, int w, int C, float scale,
                            const float* __restrict__ grad_out, float* __restrict__ dlogits) {
  const int i = blockIdx.x, n = blockIdx.y;
  const float gs = grad_out[0] * scale;
  const int wc = w * C;
  const float* own = T2 + ((static_cast<size_t>(n) * h + i) * 2 + 0) * wc;
  const float* prev = i > 0 ? T2 + ((static_cast<size_t>(n) * h + (i - 1)) * 2 + 1) * wc : nullptr;
  float* out = dlogits + (static_cast<size_t>(n) * h + i) * wc;
  for (int idx = threadIdx.x; idx < wc; idx += blockDim.x) {
    float acc = own[idx];
    if (prev) acc += prev[idx];
    out[idx] = fmaf(acc, gs, out[idx]);
  }
}

// ---------------------------------------------------------------------------------------------------- class-incremental
// MiB's background-aware losses (Cermelli et al., CVPR 2020) for a student of C classes and the previous step's network,
// the teacher, of C_old < C: class 0 is the background, [0, C_old) the old classes, [C_old, C) the new ones, and
// lse_A(x) = log sum_{c in A} exp(x_c), each subset's sum taken against its own maximum, so a confidently new-class
// pixel labelled background scores a large finite loss, not inf.
// Unbiased cross-entropy: the kUnbiased instances of the plain forward and rows kernels (above) with the plain reduce and
// cols kernels. Per valid pixel, l = lse_all(s) - lse_old(s) for a label t < C_old (an old label counts as background),
// lse_all(s) - s_t otherwise; dl/ds_c = p_c - [t < C_old][c < C_old] exp(s_c - lse_old) - [t >= C_old][c = t].
// Unbiased distillation, every pixel (no target), q = softmax(alpha t) over the C_old teacher classes and
// B = {0} u [C_old, C):
//   k = -(1/C_old) [ q_0 (lse_B(s) - lse_all(s)) + sum_{c=1}^{C_old-1} q_c (s_c - lse_all(s)) ],   KD = mean of k
//   dk/ds_c = (p_c - q_0 exp(s_c - lse_B)) / C_old for c in B,   (p_c - q_c) / C_old for 1 <= c < C_old
//   forward : the distillation forward's layout (KdGeom, both maps' node rows staged side by side; the teacher's C_old
//             channels at the student's stride), three class passes per pixel (the maxima of s over all classes and
//             over B and of t; the three sums; the terms), one (sum k, pixels) partial per CTA and the plain fp64
//             reduce; (lse_all(s), lse_B(s), lse(alpha t)) saved per pixel.
//   backward: the distillation rows layout with those three words log2(e) staged per pixel (12 bytes: the Dice width
//             limit), a thread of a class in B reading the teacher's class 0; then the distillation cols kernel, which
//             ADDS into dlogits.
struct UnkdPix {
  float all2, b2, t2;   // lse_all(s), lse_B(s), lse(alpha t), times log2(e)
};

template <int Z>
__device__ __forceinline__ void node_pair(const float* A, const float* B, const float* Cc, const float* D, int c,
                                          float l0w, float l1w, float& top, float& bot) {
  top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
  bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
}

template <int Z>
__global__ void __launch_bounds__(KdGeom<Z>::kCols)
upsample_unkd_fwd_kernel(const float* __restrict__ sl, int pitch_s, const float* __restrict__ tl, int pitch_t, int N,
                         int h, int w, int C, int c_old, int Cs, int Ho, int Wo, float alpha,
                         float* __restrict__ partial, float* __restrict__ lse_out) {
  using G = Zoom<Z>;
  constexpr int kCols = KdGeom<Z>::kCols, kNodes = KdGeom<Z>::kNodes;
  extern __shared__ float S[];  // [2 maps: student (C), teacher (c_old)][kNodeRows][kNodes][Cs]
  __shared__ float red_k[kCols / 32];
  __shared__ float red_cnt[kCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kNodes, w - j_base);
  const int tid = threadIdx.x;
  const int map_floats = G::kNodeRows * kNodes * Cs;
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    const size_t src = (static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj);
    S[(rr * kNodes + jj) * Cs + c] = sl[src * pitch_s + c];
  }
  for (int idx = tid; idx < G::kNodeRows * nj * c_old; idx += kCols) {
    const int c = idx % c_old;
    const int node = idx / c_old;
    const int jj = node % nj, rr = node / nj;
    const size_t src = (static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj);
    S[map_floats + (rr * kNodes + jj) * Cs + c] = tl[src * pitch_t + c];
  }
  __syncthreads();
  float k_sum = 0.f, cnt = 0.f;
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* As = S + (j0 - j_base) * Cs;   // student nodes (i0, j0), (i0, j1), (i1, j0), (i1, j1)
    const float* Bs = S + (j1 - j_base) * Cs;
    const float* Cs_ = As + kNodes * Cs;
    const float* Ds = Bs + kNodes * Cs;
    const float* At = As + map_floats;           // teacher nodes
    const float* Bt = Bs + map_floats;
    const float* Ct = Cs_ + map_floats;
    const float* Dt = Ds + map_floats;
    const float ka = alpha * kLog2e;
    float ms[Z], mb[Z], mt[Z], zs[Z], zb[Z], zt[Z], acc[Z];
    float ts, bs, tt, bt;
    node_pair<Z>(As, Bs, Cs_, Ds, 0, l0w, l1w, ts, bs);
    node_pair<Z>(At, Bt, Ct, Dt, 0, l0w, l1w, tt, bt);
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      ms[r] = mb[r] = row_lerp<Z>(ts, bs, r);
      mt[r] = row_lerp<Z>(tt, bt, r);
      zs[r] = zb[r] = zt[r] = acc[r] = 0.f;
    }
    // pass 1: the maxima (class 0 above; the old classes; the new classes, which are in B)
#pragma unroll 2
    for (int c = 1; c < c_old; ++c) {
      node_pair<Z>(As, Bs, Cs_, Ds, c, l0w, l1w, ts, bs);
      node_pair<Z>(At, Bt, Ct, Dt, c, l0w, l1w, tt, bt);
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        ms[r] = fmaxf(ms[r], row_lerp<Z>(ts, bs, r));
        mt[r] = fmaxf(mt[r], row_lerp<Z>(tt, bt, r));
      }
    }
#pragma unroll 2
    for (int c = c_old; c < C; ++c) {
      node_pair<Z>(As, Bs, Cs_, Ds, c, l0w, l1w, ts, bs);
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(ts, bs, r);
        ms[r] = fmaxf(ms[r], v);
        mb[r] = fmaxf(mb[r], v);
      }
    }
    // pass 2: the sums, each against its own maximum
    node_pair<Z>(As, Bs, Cs_, Ds, 0, l0w, l1w, ts, bs);
#pragma unroll
    for (int r = 0; r < Z; ++r) zb[r] = ex2_approx((row_lerp<Z>(ts, bs, r) - mb[r]) * kLog2e);
#pragma unroll 2
    for (int c = 0; c < c_old; ++c) {
      node_pair<Z>(As, Bs, Cs_, Ds, c, l0w, l1w, ts, bs);
      node_pair<Z>(At, Bt, Ct, Dt, c, l0w, l1w, tt, bt);
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        zs[r] += ex2_approx((row_lerp<Z>(ts, bs, r) - ms[r]) * kLog2e);
        zt[r] += ex2_approx((row_lerp<Z>(tt, bt, r) - mt[r]) * ka);
      }
    }
#pragma unroll 2
    for (int c = c_old; c < C; ++c) {
      node_pair<Z>(As, Bs, Cs_, Ds, c, l0w, l1w, ts, bs);
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(ts, bs, r);
        zs[r] += ex2_approx((v - ms[r]) * kLog2e);
        zb[r] += ex2_approx((v - mb[r]) * kLog2e);
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      zs[r] = logf(zs[r]);   // log sums from here on
      zb[r] = logf(zb[r]);
      zt[r] = logf(zt[r]);
    }
    // pass 3: q_0 (lse_B - lse_all) + sum_{c >= 1} q_c (s_c - lse_all), log q_c = alpha (t_c - m_t) - log z_t
    node_pair<Z>(At, Bt, Ct, Dt, 0, l0w, l1w, tt, bt);
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      const float q0 = ex2_approx(((row_lerp<Z>(tt, bt, r) - mt[r]) * alpha - zt[r]) * kLog2e);
      acc[r] = q0 * ((mb[r] - ms[r]) + (zb[r] - zs[r]));
    }
#pragma unroll 2
    for (int c = 1; c < c_old; ++c) {
      node_pair<Z>(As, Bs, Cs_, Ds, c, l0w, l1w, ts, bs);
      node_pair<Z>(At, Bt, Ct, Dt, c, l0w, l1w, tt, bt);
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float q = ex2_approx(((row_lerp<Z>(tt, bt, r) - mt[r]) * alpha - zt[r]) * kLog2e);
        acc[r] = fmaf(q, (row_lerp<Z>(ts, bs, r) - ms[r]) - zs[r], acc[r]);
      }
    }
    const float inv_old = 1.f / static_cast<float>(c_old);
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        lse_out[3 * pix + 0] = ms[r] + zs[r];
        lse_out[3 * pix + 1] = mb[r] + zb[r];
        lse_out[3 * pix + 2] = fmaf(mt[r], alpha, zt[r]);
        k_sum -= acc[r] * inv_old;
        cnt += 1.f;
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) {
    k_sum += __shfl_xor_sync(0xffffffffu, k_sum, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((tid & 31) == 0) {
    red_k[tid >> 5] = k_sum;
    red_cnt[tid >> 5] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    float l = 0.f, k = 0.f;
    for (int i = 0; i < kCols / 32; ++i) {
      l += red_k[i];
      k += red_cnt[i];
    }
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * b] = l;
    partial[2 * b + 1] = k;
  }
}

// One interval of the unbiased distillation rows kernel for class c (kd_interval's structure): acc = the (left, right) x
// (top, bottom node row) sums of p_c - q_0 exp(s_c - lse_B) (in_b) or p_c - q_c, the teacher values those of class 0
// (in_b) or c.
template <int Z, bool kFull>
__device__ __forceinline__ void unkd_interval(const UnkdPix* s, int Wo, int xb, int rows, int nx, float ka, bool in_b,
                                              float a, float b, float cc, float d, float at, float bt, float ct,
                                              float dt, float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    const float topt = l0w * at + l1w * bt;
    const float bott = l0w * ct + l1w * dt;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const UnkdPix u = s[r * Wo + xb + k];
      const float v = row_lerp<Z>(top, bot, r);
      const float p = ex2_approx(fmaf(v, kLog2e, -u.all2));
      const float q = ex2_approx(fmaf(row_lerp<Z>(topt, bott, r), ka, -u.t2));
      const float g = in_b ? fmaf(-q, ex2_approx(fmaf(v, kLog2e, -u.b2)), p) : p - q;
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

// One CTA per (low-res interval row i0, image), one thread per student class; out = T2[n][i0][2][w][C] of C_old dk/ds_c.
template <int Z>
__global__ void __launch_bounds__(256)
upsample_unkd_bwd_rows_kernel(const float* __restrict__ sl, int pitch_s, const float* __restrict__ tl, int pitch_t,
                              int N, int h, int w, int C, int c_old, int Ho, int Wo, float alpha,
                              const float* __restrict__ lse, float* __restrict__ T2) {
  extern __shared__ UnkdPix s_upix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const float* l = lse + 3 * (rowbase + x);
      s_upix[r * Wo + x] = UnkdPix{l[0] * kLog2e, l[1] * kLog2e, l[2] * kLog2e};
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const bool in_b = c == 0 || c >= c_old;
  const int tc = in_b ? 0 : c;
  const float ka = alpha * kLog2e;
  const float* S0 = sl + (static_cast<size_t>(n) * h + i0) * w * pitch_s + c;
  const float* S1 = sl + (static_cast<size_t>(n) * h + i1) * w * pitch_s + c;
  const float* U0 = tl + (static_cast<size_t>(n) * h + i0) * w * pitch_t + tc;
  const float* U1 = tl + (static_cast<size_t>(n) * h + i1) * w * pitch_t + tc;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  const int j1 = min(1, w - 1);
  float a = S0[0], cc = S1[0], at = U0[0], ct = U1[0];   // left node column of the current interval
  float nb = S0[static_cast<size_t>(j1) * pitch_s], nd = S1[static_cast<size_t>(j1) * pitch_s];
  float nbt = U0[static_cast<size_t>(j1) * pitch_t], ndt = U1[static_cast<size_t>(j1) * pitch_t];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd, bt = nbt, dt = ndt;
    const int jn = min(j0 + 2, w - 1);
    nb = S0[static_cast<size_t>(jn) * pitch_s];
    nd = S1[static_cast<size_t>(jn) * pitch_s];
    nbt = U0[static_cast<size_t>(jn) * pitch_t];
    ndt = U1[static_cast<size_t>(jn) * pitch_t];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      unkd_interval<Z, true>(s_upix, Wo, xb, rows, nx, ka, in_b, a, b, cc, d, at, bt, ct, dt, acc);
    } else {
      unkd_interval<Z, false>(s_upix, Wo, xb, rows, nx, ka, in_b, a, b, cc, d, at, bt, ct, dt, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
    at = bt;
    ct = dt;
  }
}

// ---------------------------------------------------------------------------------------------------- focal loss
// Softmax focal loss (Lin et al., ICCV 2017) with optional class weights. Per valid pixel, with p = softmax(v),
// q = 1 - p_t and nll = -log p_t:
//   l = w_t q^gamma nll,   loss = sum l / n_valid,
//   dl/dv_c = w_t M (p_c - [c = t]),   M = q^gamma + gamma p_t q^(gamma-1) nll = q^gamma (1 + gamma p_t nll / q)
// with torch.pow's 0^0 = 1: at q = 0, l = 0 and M = [gamma = 0]. The forward is the plain forward plus, per pixel, the
// modulator w_t M (0 where the pixel is not valid) kept for the backward; the backward is the plain one with every
// pixel's term scaled by its modulator, then the plain cols kernel with 1 / n_valid.
// Operation order (q and nll keep their relative accuracy as p_t -> 1): the second class pass sums, next to the plain
// S = sum_c e_c (e_c = ex2((v_c - m) log2e); lse = m + log S is the plain forward's bits), S_o = sum_{c != t} e_c with
// the target's term skipped, not subtracted. Then q = S_o / S, p_t = e_t / S, nll = log1p(S_o / e_t) (lse - v_t once e_t
// has underflowed) and q^gamma = ex2(gamma lg2 q): one MUFU pair per pixel.
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kFocalMinEt = 1e-30f;   // below this S_o / e_t may overflow: nll = lse - v_t, large and well conditioned

template <int Z>
__global__ void __launch_bounds__(kFwdCols)
upsample_ce_focal_fwd_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                             const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                             const float* __restrict__ class_weight, float gamma, float* __restrict__ partial,
                             long long* __restrict__ argmax_out, float* __restrict__ lse_out,
                             float* __restrict__ mod_out) {
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs] as in upsample_ce_fwd_kernel
  __shared__ float red_loss[kFwdCols / 32];
  __shared__ float red_cnt[kFwdCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  __syncthreads();
  float loss = 0.f, cnt = 0.f;
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* A = S + (j0 - j_base) * Cs;
    const float* B = S + (j1 - j_base) * Cs;
    const float* Cc = A + kFwdNodes * Cs;
    const float* D = B + kFwdNodes * Cs;
    float m[Z], sum[Z], so[Z];   // so: S_o, the sum without the target's term
    int am[Z], tc[Z];            // tc: target class, -1 = not valid
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      m[r] = -INFINITY;
      am[r] = 0;
      sum[r] = 0.f;
      so[r] = 0.f;
      tc[r] = -1;
      if (r < rows) {
        const long long t = target[(static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x];
        if (t != ignore_index && t >= 0 && t < C) tc[r] = static_cast<int>(t);
      }
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        if (v > m[r]) {
          m[r] = v;
          am[r] = c;
        }
      }
    }
    float m2[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) m2[r] = m[r] * kLog2e;
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        const float e = ex2_approx(fmaf(v, kLog2e, -m2[r]));
        sum[r] += e;
        so[r] += c == tc[r] ? 0.f : e;
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        const float lse = m[r] + __logf(sum[r]);
        if (argmax_out) argmax_out[pix] = am[r];
        lse_out[pix] = lse;
        float mod = 0.f;
        if (tc[r] >= 0) {
          const int t = tc[r];
          const float top = Z == 1 ? A[t] : l0w * A[t] + l1w * B[t];
          const float bot = Z == 1 ? 0.f : l0w * Cc[t] + l1w * D[t];
          const float vt = row_lerp<Z>(top, bot, r);
          const float et = ex2_approx(fmaf(vt, kLog2e, -m2[r]));
          const float q = so[r] / sum[r];
          const float nll = et > kFocalMinEt ? log1pf(so[r] / et) : lse - vt;
          const float wt = class_weight ? class_weight[t] : 1.f;
          float qg, M;   // q^gamma and the modulator, torch.pow's 0^0 = 1
          if (q > 0.f) {
            qg = ex2_approx(gamma * lg2_approx(q));
            M = qg * fmaf(gamma * (et / sum[r]), nll / q, 1.f);
          } else {
            qg = M = gamma == 0.f ? 1.f : 0.f;
          }
          loss += wt * qg * nll;
          cnt += 1.f;
          mod = wt * M;
        }
        mod_out[pix] = mod;
      }
    }
  }
  // deterministic block reduction -> one (sum of l, valid count) partial per CTA, as upsample_ce_fwd_kernel
  for (int o = 16; o > 0; o >>= 1) {
    loss += __shfl_xor_sync(0xffffffffu, loss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((tid & 31) == 0) {
    red_loss[tid >> 5] = loss;
    red_cnt[tid >> 5] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    float l = 0.f, k = 0.f;
    for (int i = 0; i < kFwdCols / 32; ++i) {
      l += red_loss[i];
      k += red_cnt[i];
    }
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * b] = l;
    partial[2 * b + 1] = k;
  }
}

// One interval of the focal rows kernel for class c: g = modulator (p_c - [c = t]), folded as in
// upsample_ce_bwd_rows_kernel. DicePix::g holds the pixel's modulator.
template <int Z, bool kFull>
__device__ __forceinline__ void focal_interval(const DicePix* s, int Wo, int xb, int rows, int nx, int c, float a,
                                               float b, float cc, float d, float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const DicePix pi = s[r * Wo + xb + k];
      if (pi.t < 0) continue;  // warp-uniform
      const float v = row_lerp<Z>(top, bot, r);
      const float p = ex2_approx(fmaf(v, kLog2e, -pi.lse2));
      const float g = pi.g * (p - (c == pi.t ? 1.f : 0.f));
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

// Rows layout of upsample_ce_bwd_rows_kernel with the Dice rows kernel's 12-byte pixel word (lse, target, modulator);
// a pixel whose modulator is 0 (not valid, a zero-weight class, q = 0) is staged as ignored: its gradient is exactly 0.
template <int Z>
__global__ void __launch_bounds__(256)
upsample_ce_focal_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                              const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                              const float* __restrict__ lse, const float* __restrict__ mod, float* __restrict__ T2) {
  extern __shared__ DicePix s_dpix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const long long t = target[rowbase + x];
      DicePix pi;
      pi.g = mod[rowbase + x];
      pi.t = (t == ignore_index || t < 0 || t >= C || pi.g == 0.f) ? -1 : static_cast<int>(t);
      pi.lse2 = lse[rowbase + x] * kLog2e;
      s_dpix[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];
    nd = L1[static_cast<size_t>(jn) * pitch];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      focal_interval<Z, true>(s_dpix, Wo, xb, rows, nx, c, a, b, cc, d, acc);
    } else {
      focal_interval<Z, false>(s_dpix, Wo, xb, rows, nx, c, a, b, cc, d, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
  }
}

// ---------------------------------------------------------------------------------------------------- SegPGD
// The SegPGD attack loss (Gu et al., ECCV 2022). Per valid pixel (target t in [0, C), t != ignore_index), with pred the
// first-maximum argmax of the same pass and nll = lse - v_t as the plain forward computes it:
//   w = (1 - lambda) if pred == t else lambda,   loss = sum w nll / n_valid.
// The weights are constants (no gradient through the argmax), so dloss/dv_c = w (p_c - [c = t]) / n_valid: the focal
// backward with the modulator map mod = w (0 where the pixel is not valid). The two class passes are the plain
// forward's, so lse, the argmax and nll carry the plain kernel's bits.
template <int Z>
__global__ void __launch_bounds__(kFwdCols)
upsample_segpgd_fwd_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                           const long long* __restrict__ target, int Ho, int Wo, int ignore_index, float lambda,
                           float* __restrict__ partial, long long* __restrict__ argmax_out, float* __restrict__ lse_out,
                           float* __restrict__ mod_out) {
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs] as in upsample_ce_fwd_kernel
  __shared__ float red_loss[kFwdCols / 32];
  __shared__ float red_cnt[kFwdCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  __syncthreads();
  float loss = 0.f, cnt = 0.f;
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* A = S + (j0 - j_base) * Cs;
    const float* B = S + (j1 - j_base) * Cs;
    const float* Cc = A + kFwdNodes * Cs;
    const float* D = B + kFwdNodes * Cs;
    float m[Z], sum[Z];
    int am[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      m[r] = -INFINITY;
      am[r] = 0;
      sum[r] = 0.f;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        if (v > m[r]) {
          m[r] = v;
          am[r] = c;
        }
      }
    }
    float m2[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) m2[r] = m[r] * kLog2e;
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) sum[r] += ex2_approx(fmaf(row_lerp<Z>(top, bot, r), kLog2e, -m2[r]));
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        const long long t = target[pix];
        const float lse = m[r] + __logf(sum[r]);
        if (argmax_out) argmax_out[pix] = am[r];
        lse_out[pix] = lse;
        float wt = 0.f;
        if (t != ignore_index && t >= 0 && t < C) {
          const int tc = static_cast<int>(t);
          const float top = Z == 1 ? A[tc] : l0w * A[tc] + l1w * B[tc];
          const float bot = Z == 1 ? 0.f : l0w * Cc[tc] + l1w * D[tc];
          const float vt = row_lerp<Z>(top, bot, r);
          wt = am[r] == tc ? 1.f - lambda : lambda;
          loss += wt * (lse - vt);
          cnt += 1.f;
        }
        mod_out[pix] = wt;
      }
    }
  }
  // deterministic block reduction -> one (sum of w nll, valid count) partial per CTA, as upsample_ce_fwd_kernel
  for (int o = 16; o > 0; o >>= 1) {
    loss += __shfl_xor_sync(0xffffffffu, loss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((tid & 31) == 0) {
    red_loss[tid >> 5] = loss;
    red_cnt[tid >> 5] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    float l = 0.f, k = 0.f;
    for (int i = 0; i < kFwdCols / 32; ++i) {
      l += red_loss[i];
      k += red_cnt[i];
    }
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * b] = l;
    partial[2 * b + 1] = k;
  }
}

// ---------------------------------------------------------------------------------------------------- pseudo-labels
// Confidence-masked pseudo-label cross-entropy from a teacher (FixMatch / UniMatch self-training), with s and t the
// student and teacher maps after the same xZ upsample:
//   L = {target in [0, C), target != ignore_index},  U = {target == ignore_index}
//   yhat = argmax_c t_c (first maximum),  conf = 1 / sum_c exp(t_c - t_yhat)
//   loss = ce_weight (1/|L|) sum_L (lse - s_target) + pl_weight (1/|U|) sum_{U, conf >= threshold} (lse - s_yhat)
// Both terms are CE against a per-pixel "effective target" with a per-pixel weight, so the gradient is
// w_p (p_c - [c = y_p]): the focal backward (rows kernel staging (lse, target, modulator), plain cols kernel with a
// count of 1) run on the forward's effective-target and weight maps. The weights need |L| and |U| before the forward
// writes them: a count pass over the target runs first (integer atomics: the counts do not depend on their order).
//   count  : |L|, |U| as uint64 into the workspace; also writes loss_out[4] = 0, loss_out[5] = 1 (the cols count).
//   forward: the distillation forward's geometry (both maps' node rows staged), the student's max / argmax / lse with the
//            plain forward's operations (the plain tail's bits), the teacher's max / argmax / sum of exp in the same
//            passes; per pixel the effective target (target on L, yhat on confident U, -1 otherwise) and weight
//            (ce_weight/|L|, pl_weight/|U|, 0); (sum CE over L, |L|) and (sum PL, |U|) per CTA, each reduced in fp64 by
//            the plain reduce kernel.
__global__ void __launch_bounds__(256)
upsample_pl_count_kernel(const long long* __restrict__ target, long long M, int C, int ignore_index,
                         unsigned long long* __restrict__ counts, float* __restrict__ loss_out) {
  unsigned nl = 0, nu = 0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < M;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long t = target[i];
    if (t == ignore_index) ++nu;
    else if (t >= 0 && t < C) ++nl;
  }
  nl = __reduce_add_sync(0xffffffffu, nl);
  nu = __reduce_add_sync(0xffffffffu, nu);
  if ((threadIdx.x & 31) == 0) {
    if (nl) atomicAdd(&counts[0], static_cast<unsigned long long>(nl));
    if (nu) atomicAdd(&counts[1], static_cast<unsigned long long>(nu));
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    loss_out[4] = 0.f;
    loss_out[5] = 1.f;
  }
}

// kMix (CutMix / ClassMix, losses.MixPseudoLabelLoss): the teacher of an output pixel is image n's map or its partner
// (n + 1) mod N's, as the uint8 mix mask [N, 8(h-1)+1, 8(w-1)+1] on the input grid says at the pixel's input position
// (Z i, Z j) * 8/Z (the grids nest under align_corners). The partner's node rows are staged as a third map and each
// output row picks its teacher with the same operations, so a pixel's (yhat, conf) are the bits the plain instance
// computes for its teacher image. The mask argument comes last: the kMix = false instances keep their parameter layout.
template <int Z, bool kMix = false>
__global__ void __launch_bounds__(KdGeom<Z>::kCols)
upsample_pl_fwd_kernel(const float* __restrict__ sl, int pitch_s, const float* __restrict__ tl, int pitch_t, int N, int h,
                       int w, int C, int Cs, const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                       float threshold, float pl_weight, float ce_weight, const unsigned long long* __restrict__ counts,
                       float* __restrict__ partial, long long* __restrict__ argmax_out, float* __restrict__ lse_out,
                       long long* __restrict__ eff_out, float* __restrict__ wt_out,
                       const unsigned char* __restrict__ mix_mask = nullptr) {
  using G = Zoom<Z>;
  constexpr int kCols = KdGeom<Z>::kCols, kNodes = KdGeom<Z>::kNodes;
  constexpr int kMaps = kMix ? 3 : 2;
  extern __shared__ float S[];  // [kMaps: student, teacher, partner's teacher][kNodeRows][kNodes][Cs]
  __shared__ float red[4][kCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kNodes, w - j_base);
  const int tid = threadIdx.x;
  const int map_floats = G::kNodeRows * kNodes * Cs;
  const int pn = kMix ? (n + 1 == N ? 0 : n + 1) : n;
  for (int idx = tid; idx < kMaps * G::kNodeRows * nj * C; idx += kCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = (node / nj) % G::kNodeRows, map = node / (nj * G::kNodeRows);
    const size_t src = (static_cast<size_t>(kMix && map == 2 ? pn : n) * h + (rr ? i1 : i0)) * w + (j_base + jj);
    S[map * map_floats + (rr * kNodes + jj) * Cs + c] = map ? tl[src * pitch_t + c] : sl[src * pitch_s + c];
  }
  __syncthreads();
  float acc[4] = {0.f, 0.f, 0.f, 0.f};   // sum CE over L, |L|, sum PL over confident U, |U|
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* A = S + (j0 - j_base) * Cs;   // student nodes (i0, j0), (i0, j1), (i1, j0), (i1, j1)
    const float* B = S + (j1 - j_base) * Cs;
    const float* Cc = A + kNodes * Cs;
    const float* D = B + kNodes * Cs;
    const float* At = A + map_floats;          // teacher nodes
    const float* Bt = B + map_floats;
    const float* Ct = Cc + map_floats;
    const float* Dt = D + map_floats;
    const float* Ap = At + map_floats;         // kMix: the partner's teacher nodes
    const float* Bp = Bt + map_floats;
    const float* Cp = Ct + map_floats;
    const float* Dp = Dt + map_floats;
    unsigned sel = 0;                          // kMix: bit r set -> output row r takes the partner's teacher
    if constexpr (kMix) {
      const int H = 8 * (h - 1) + 1, W = 8 * (w - 1) + 1;
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        if (r < rows && mix_mask[(static_cast<size_t>(n) * H + (Z * i0 + r) * (8 / Z)) * W + x * (8 / Z)])
          sel |= 1u << r;
      }
    }
    float ms[Z], mt[Z], zs[Z], zt[Z];
    int as[Z], at[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      ms[r] = mt[r] = -INFINITY;
      as[r] = at[r] = 0;
      zs[r] = zt[r] = 0.f;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
      const float topt = Z == 1 ? At[c] : l0w * At[c] + l1w * Bt[c];
      const float bott = Z == 1 ? 0.f : l0w * Ct[c] + l1w * Dt[c];
      float topp = 0.f, botp = 0.f;
      if constexpr (kMix) {
        topp = Z == 1 ? Ap[c] : l0w * Ap[c] + l1w * Bp[c];
        botp = Z == 1 ? 0.f : l0w * Cp[c] + l1w * Dp[c];
      }
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        if (v > ms[r]) {
          ms[r] = v;
          as[r] = c;
        }
        const float u = kMix && ((sel >> r) & 1u) ? row_lerp<Z>(topp, botp, r) : row_lerp<Z>(topt, bott, r);
        if (u > mt[r]) {
          mt[r] = u;
          at[r] = c;
        }
      }
    }
    float m2[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) m2[r] = ms[r] * kLog2e;
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
      const float topt = Z == 1 ? At[c] : l0w * At[c] + l1w * Bt[c];
      const float bott = Z == 1 ? 0.f : l0w * Ct[c] + l1w * Dt[c];
      float topp = 0.f, botp = 0.f;
      if constexpr (kMix) {
        topp = Z == 1 ? Ap[c] : l0w * Ap[c] + l1w * Bp[c];
        botp = Z == 1 ? 0.f : l0w * Cp[c] + l1w * Dp[c];
      }
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        zs[r] += ex2_approx(fmaf(row_lerp<Z>(top, bot, r), kLog2e, -m2[r]));   // the plain forward's sum
        const float u = kMix && ((sel >> r) & 1u) ? row_lerp<Z>(topp, botp, r) : row_lerp<Z>(topt, bott, r);
        zt[r] += ex2_approx((u - mt[r]) * kLog2e);                               // yhat's term is exactly 1
      }
    }
    const unsigned long long nl = counts[0], nu = counts[1];
    const float wl = nl ? ce_weight / static_cast<float>(nl) : 0.f;
    const float wu = nu ? pl_weight / static_cast<float>(nu) : 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        const long long t = target[pix];
        const float lse = ms[r] + __logf(zs[r]);
        if (argmax_out) argmax_out[pix] = as[r];
        lse_out[pix] = lse;
        int y = -1;
        float wt = 0.f;
        if (t == ignore_index) {
          acc[3] += 1.f;
          if (1.f / zt[r] >= threshold) {
            y = at[r];
            wt = wu;
          }
        } else if (t >= 0 && t < C) {
          y = static_cast<int>(t);
          wt = wl;
          acc[1] += 1.f;
        }
        if (y >= 0) {
          const float top = Z == 1 ? A[y] : l0w * A[y] + l1w * B[y];
          const float bot = Z == 1 ? 0.f : l0w * Cc[y] + l1w * D[y];
          acc[t == ignore_index ? 2 : 0] += lse - row_lerp<Z>(top, bot, r);
        }
        eff_out[pix] = y;
        wt_out[pix] = wt;
      }
    }
  }
  // deterministic block reduction -> (sum CE, |L|) and (sum PL, |U|) per CTA, each laid out as the plain partials
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  }
  if ((tid & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) red[k][tid >> 5] = acc[k];
  }
  __syncthreads();
  if (tid < 4) {
    float s = 0.f;
    for (int i = 0; i < kCols / 32; ++i) s += red[tid][i];
    const size_t nb = static_cast<size_t>(gridDim.x) * gridDim.y * gridDim.z;
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[(tid >> 1) * 2 * nb + 2 * b + (tid & 1)] = s;
  }
}

// ---------------------------------------------------------------------------------------------------- RMI
// Region Mutual Information loss (Zhao, Wang, Cai, NeurIPS 2019) with its sigmoid BCE term and ce_weight * CE, in the
// authors' default configuration, fixed here: average pooling 4 (stride 4, no padding), radius 3, lambda_way 1, clip
// 1e-6. With v = [t valid], y_c = [t = c] v, s = sigmoid(z), q = s v + 1e-6, Y / Q the 4x4 average pools of y / q
// (Hp = Ho / 4, Wp = Wo / 4), a_k / b_k the 3x3 neighbourhoods of pooled cell k of Y / Q (K = (Hp-2)(Wp-2)), centred:
//   S_aa, S_bb, S_ab = sums over k of a~a~', b~b~', a~b~'    P = S_bb + alpha I    A = S_aa - S_ab P^-1 S_ab'
//   r[n,c] = 1/2 log det(A + alpha I),   RMI = sum_{n,c} r / (9N),   BCE = sum v (softplus(z) - y z) / (n_valid + 1)
//   loss = bce_weight BCE + (1 - bce_weight) RMI + ce_weight CE
// Backward, M = (A + alpha I)^-1, X = S_ab P^-1: G_ab = -M X, G_bb = 1/2 X' M X, dr/db_k = G_ab' a~_k + 2 G_bb b~_k,
// dr/dQ[cell] = sum over the 9 offsets d with k = cell - d in range of (dr/db_k)[d], and per valid pixel
//   dL/dz_c = (1 - bce_weight)/(9N) [pooled] s(1-s)/16 dr/dQ + bce_weight (s - y_c)/(n_valid + 1) + ce_weight/n_valid (p_c - y_c)
// Chain:
//   forward : the plain forward instance (lse, argmax, CE partials); rmi_pool (the upsampled logits of a band of whole
//             pooled rows, one thread per output column: the pooled Y and Q maps and BCE partials, the 16 values of a
//             cell summed in registers and over 4 lanes in a fixed order); rmi_moments (one CTA per (n, c) and moment
//             group, fp64 sums over the cells, a fixed-order tree); rmi_algebra (one thread per (n, c), the 9x9 fp64
//             Cholesky algebra: r and the [G_ab' | 2 G_bb] table); rmi_loss (one CTA, fp64, fixed order).
//   backward: rmi_dq (dr/dQ per pooled cell from the table and the pooled maps), the rows kernel (one thread per class,
//             (lse, t) staged per pixel, the pixel terms above), then the plain cols kernel.
// No float atomics, no host synchronisation.
constexpr float kRmiClip = 1e-6f;
constexpr int kRmiMoments = 189;   // sum Y[9], sum Q[9], YY upper triangle [45], QQ upper triangle [45], YQ [9][9]
constexpr int kRmiRec = 184;       // table record per (n, c): T[9][18] = [G_ab' | 2 G_bb], mean Y[9], mean Q[9], r, pad
constexpr int kRmiRecUsed = 181;
constexpr int kRmiGroups = 5;      // moment groups: Y (sums, YY), Q (sums, QQ), YQ rows 0-2, 3-5, 6-8
constexpr float kLn2 = 0.6931471805599453f;

// A CTA of the pool kernel: whole pooled rows (4 output rows; 8, one interval, at Z = 8) and kCols output columns.
template <int Z>
struct RmiBand {
  static constexpr int kRows = Z < 4 ? 4 : Z;
  static constexpr int kCols = Z == 1 ? 32 : Z == 2 ? 64 : 128;
  static constexpr int kNodeRows = Z == 1 ? 4 : kRows / Z + 1;
  static constexpr int kNodes = kCols / Z + 1;
};

// e = exp(-|v|), rr = 1 / (1 + e): sigmoid(v) = (v >= 0 ? 1 : e) rr, sigmoid'(v) = e rr^2, softplus(v) = max(v, 0) + log(1 + e)
__device__ __forceinline__ float rmi_exp_neg_abs(float v) { return ex2_approx(-fabsf(v) * kLog2e); }

template <int Z>
__global__ void __launch_bounds__(RmiBand<Z>::kCols)
rmi_pool_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                const long long* __restrict__ target, int Ho, int Wo, int ignore_index, float* __restrict__ pooled,
                float* __restrict__ partial) {
  using G = Zoom<Z>;
  using B = RmiBand<Z>;
  constexpr int kPr = B::kRows / 4;   // pooled rows per band
  extern __shared__ float S[];        // [kNodeRows][kNodes][Cs]
  __shared__ float red[B::kCols / 32];
  const int n = blockIdx.z, y0 = blockIdx.y * B::kRows, x0 = blockIdx.x * B::kCols;
  const int ib = y0 >> G::kShift;
  const int j_base = x0 >> G::kShift;
  const int nj = min(B::kNodes, w - j_base);
  const int tid = threadIdx.x;
  for (int idx = tid; idx < B::kNodeRows * nj * C; idx += B::kCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * B::kNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + min(ib + rr, h - 1)) * w + (j_base + jj)) * pitch + c];
  }
  __syncthreads();
  const int Hp = Ho >> 2, Wp = Wo >> 2;
  const int x = x0 + tid;
  const int xs = min(x, Wo - 1);   // lanes past the image compute a real column; their cells are never written
  const int j0 = xs >> G::kShift;
  const int j1 = min(j0 + 1, w - 1);
  const float l1w = static_cast<float>(xs & G::kMask) * G::kStep, l0w = 1.f - l1w;
  const float* A = S + (j0 - j_base) * Cs;
  const float* Bn = S + (j1 - j_base) * Cs;
  int tg[B::kRows];   // target class per row, -1 where not valid
#pragma unroll
  for (int r = 0; r < B::kRows; ++r) {
    tg[r] = -1;
    if (x < Wo && y0 + r < Ho) {
      const long long t = target[(static_cast<size_t>(n) * Ho + (y0 + r)) * Wo + x];
      if (t != ignore_index && t >= 0 && t < C) tg[r] = static_cast<int>(t);
    }
  }
  const int pc = x >> 2;
  const bool writer = (tid & 3) == 0 && pc < Wp;
  float bce = 0.f;
  for (int c = 0; c < C; ++c) {
    float hv[B::kNodeRows];
#pragma unroll
    for (int k = 0; k < B::kNodeRows; ++k) {
      hv[k] = Z == 1 ? A[k * B::kNodes * Cs + c] : l0w * A[k * B::kNodes * Cs + c] + l1w * Bn[k * B::kNodes * Cs + c];
    }
    float qs[kPr], ys[kPr];
#pragma unroll
    for (int p = 0; p < kPr; ++p) qs[p] = ys[p] = 0.f;
#pragma unroll
    for (int r = 0; r < B::kRows; ++r) {
      float v;
      if constexpr (Z == 1) {
        v = hv[r];
      } else {
        v = row_lerp<Z>(hv[r >> G::kShift], hv[(r >> G::kShift) + 1], r & G::kMask);
      }
      float q = kRmiClip;
      if (tg[r] >= 0) {
        const float e = rmi_exp_neg_abs(v);
        const float rr = __fdividef(1.f, 1.f + e);
        q += (v >= 0.f ? 1.f : e) * rr;
        bce += fmaxf(v, 0.f) + kLn2 * lg2_approx(1.f + e) - (tg[r] == c ? v : 0.f);
        if (tg[r] == c) ys[r >> 2] += 1.f;
      }
      qs[r >> 2] += q;
    }
#pragma unroll
    for (int p = 0; p < kPr; ++p) {
      qs[p] += __shfl_xor_sync(0xffffffffu, qs[p], 1);
      qs[p] += __shfl_xor_sync(0xffffffffu, qs[p], 2);
      ys[p] += __shfl_xor_sync(0xffffffffu, ys[p], 1);
      ys[p] += __shfl_xor_sync(0xffffffffu, ys[p], 2);
      const int pr = (y0 >> 2) + p;
      if (writer && pr < Hp) {
        const size_t cell = static_cast<size_t>(pr) * Wp + pc;
        const size_t plane = static_cast<size_t>(Hp) * Wp;
        pooled[(static_cast<size_t>(n) * C + c) * plane + cell] = ys[p] * (1.f / 16.f);
        pooled[((static_cast<size_t>(N) + n) * C + c) * plane + cell] = qs[p] * (1.f / 16.f);
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) bce += __shfl_xor_sync(0xffffffffu, bce, o);
  if ((tid & 31) == 0) red[tid >> 5] = bce;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < B::kCols / 32; ++i) s += red[i];
    partial[(static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = s;
  }
}

// One CTA per (n, c) and moment group g: g = 0 / 1 the sums and upper-triangle products of the Y / Q neighbourhoods,
// g = 2..4 the Y x Q products of neighbourhood rows 3(g-2)..3(g-2)+2. Each thread sums its cells (stride 256) in fp64
// (the fp32 products are exact), then a fixed xor tree per warp and the 8 warps in order. Raw, uncentred sums.
__global__ void __launch_bounds__(256)
rmi_moments_kernel(const float* __restrict__ pooled, int NC, int Hp, int Wp, double* __restrict__ mom) {
  const int nc = blockIdx.x, g = blockIdx.y;
  const size_t plane = static_cast<size_t>(Hp) * Wp;
  const float* Y = pooled + static_cast<size_t>(nc) * plane;
  const float* Q = pooled + (static_cast<size_t>(NC) + nc) * plane;
  const int Wk = Wp - 2, K = (Hp - 2) * Wk;
  double acc[54];
#pragma unroll
  for (int m = 0; m < 54; ++m) acc[m] = 0.0;
  if (g < 2) {
    const float* M = g == 0 ? Y : Q;
    for (int k = threadIdx.x; k < K; k += 256) {
      const float* P = M + static_cast<size_t>(k / Wk) * Wp + k % Wk;
      double a[9];
#pragma unroll
      for (int d = 0; d < 9; ++d) a[d] = P[(d / 3) * Wp + d % 3];
      int idx = 9;
#pragma unroll
      for (int d1 = 0; d1 < 9; ++d1) {
        acc[d1] += a[d1];
#pragma unroll
        for (int d2 = d1; d2 < 9; ++d2) {
          acc[idx] = fma(a[d1], a[d2], acc[idx]);
          ++idx;
        }
      }
    }
  } else {
    const int dy = g - 2;
    for (int k = threadIdx.x; k < K; k += 256) {
      const size_t base = static_cast<size_t>(k / Wk) * Wp + k % Wk;
      double a[3], b[9];
#pragma unroll
      for (int d = 0; d < 3; ++d) a[d] = Y[base + dy * Wp + d];
#pragma unroll
      for (int d = 0; d < 9; ++d) b[d] = Q[base + (d / 3) * Wp + d % 3];
#pragma unroll
      for (int d1 = 0; d1 < 3; ++d1) {
#pragma unroll
        for (int d2 = 0; d2 < 9; ++d2) acc[d1 * 9 + d2] = fma(a[d1], b[d2], acc[d1 * 9 + d2]);
      }
    }
  }
  __shared__ double red[8][54];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int m = 0; m < 54; ++m) {
    double v = acc[m];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) red[warp][m] = v;
  }
  __syncthreads();
  const int cnt = g < 2 ? 54 : 27;
  if (threadIdx.x < cnt) {
    const int m = threadIdx.x;
    double s = 0.0;
    for (int i = 0; i < 8; ++i) s += red[i][m];
    int o;
    if (g < 2) {
      o = m < 9 ? 9 * g + m : 18 + 45 * g + (m - 9);
    } else {
      o = 108 + 27 * (g - 2) + m;
    }
    mom[static_cast<size_t>(nc) * kRmiMoments + o] = s;
  }
}

// In-place lower Cholesky factor of the symmetric 9x9 matrix a (row-major; the upper triangle is left stale).
__device__ __forceinline__ void rmi_chol9(double* a) {
  for (int j = 0; j < 9; ++j) {
    double d = a[j * 9 + j];
    for (int k = 0; k < j; ++k) d -= a[j * 9 + k] * a[j * 9 + k];
    d = sqrt(d);
    a[j * 9 + j] = d;
    for (int i = j + 1; i < 9; ++i) {
      double s = a[i * 9 + j];
      for (int k = 0; k < j; ++k) s -= a[i * 9 + k] * a[j * 9 + k];
      a[i * 9 + j] = s / d;
    }
  }
}

// x = (L L')^-1 b for the lower Cholesky factor L of rmi_chol9.
__device__ __forceinline__ void rmi_solve9(const double* L, const double* b, double* x) {
  for (int i = 0; i < 9; ++i) {
    double s = b[i];
    for (int k = 0; k < i; ++k) s -= L[i * 9 + k] * x[k];
    x[i] = s / L[i * 9 + i];
  }
  for (int i = 8; i >= 0; --i) {
    double s = x[i];
    for (int k = i + 1; k < 9; ++k) s -= L[k * 9 + i] * x[k];
    x[i] = s / L[i * 9 + i];
  }
}

// One thread per (n, c): the centred 9x9 moments from the raw sums, the Cholesky algebra in fp64, r into rterm and the
// table record (fp32): T[d][e] = G_ab'[d][e], T[d][9 + e] = 2 G_bb[d][e], mean Y, mean Q, r.
__global__ void __launch_bounds__(64)
rmi_algebra_kernel(const double* __restrict__ mom, int NC, int K, float alpha, float* __restrict__ table,
                   double* __restrict__ rterm) {
  const int nc = blockIdx.x * 64 + threadIdx.x;
  if (nc >= NC) return;
  const double* m = mom + static_cast<size_t>(nc) * kRmiMoments;
  const double invK = 1.0 / K, al = alpha;
  double Saa[81], P[81], Sab[81], X[81], MX[81];
  int ia = 18, ib = 63;
  for (int d1 = 0; d1 < 9; ++d1) {
    for (int d2 = d1; d2 < 9; ++d2) {
      Saa[d1 * 9 + d2] = Saa[d2 * 9 + d1] = m[ia++] - m[d1] * m[d2] * invK;
      P[d1 * 9 + d2] = P[d2 * 9 + d1] = m[ib++] - m[9 + d1] * m[9 + d2] * invK + (d1 == d2 ? al : 0.0);
    }
    for (int d2 = 0; d2 < 9; ++d2) Sab[d1 * 9 + d2] = m[108 + d1 * 9 + d2] - m[d1] * m[9 + d2] * invK;
  }
  rmi_chol9(P);
  for (int d = 0; d < 9; ++d) rmi_solve9(P, Sab + d * 9, X + d * 9);   // X = S_ab P^-1 (P symmetric)
  double* Am = Saa;                                                  // A + alpha I, in place of S_aa
  for (int i = 0; i < 9; ++i) {
    for (int j = i; j < 9; ++j) {
      double s = Saa[i * 9 + j];
      for (int e = 0; e < 9; ++e) s -= X[i * 9 + e] * Sab[j * 9 + e];
      Am[i * 9 + j] = Am[j * 9 + i] = s + (i == j ? al : 0.0);
    }
  }
  rmi_chol9(Am);
  double r = 0.0;
  for (int i = 0; i < 9; ++i) r += log(Am[i * 9 + i]);
  double col[9], sol[9];
  for (int e = 0; e < 9; ++e) {   // MX = (A + alpha I)^-1 X, column by column
    for (int i = 0; i < 9; ++i) col[i] = X[i * 9 + e];
    rmi_solve9(Am, col, sol);
    for (int i = 0; i < 9; ++i) MX[i * 9 + e] = sol[i];
  }
  float* T = table + static_cast<size_t>(nc) * kRmiRec;
  for (int d = 0; d < 9; ++d) {
    for (int e = 0; e < 9; ++e) {
      double gbb = 0.0;
      for (int i = 0; i < 9; ++i) gbb += X[i * 9 + d] * MX[i * 9 + e];
      T[d * 18 + e] = static_cast<float>(-MX[e * 9 + d]);
      T[d * 18 + 9 + e] = static_cast<float>(gbb);
    }
    T[162 + d] = static_cast<float>(m[d] * invK);
    T[171 + d] = static_cast<float>(m[9 + d] * invK);
  }
  T[180] = static_cast<float>(r);
  for (int i = kRmiRecUsed; i < kRmiRec; ++i) T[i] = 0.f;
  rterm[nc] = r;
}

// One CTA: CE, BCE and sum r in fp64, fixed order -> loss_out = (loss, n_valid, BCE, RMI, CE) and the backward's
// scalars sc = (ce_weight / n_valid, 1, bce_weight / (n_valid + 1), (1 - bce_weight) / (144 N)).
__global__ void __launch_bounds__(256)
rmi_loss_kernel(const float* __restrict__ ce_partial, int nce, const float* __restrict__ bce_partial, int nbce,
                const double* __restrict__ rterm, int NC, int N, float bce_weight, float ce_weight,
                float* __restrict__ loss_out, float* __restrict__ sc) {
  __shared__ double red[4][256];
  double l = 0.0, k = 0.0, b = 0.0, r = 0.0;
  for (int i = threadIdx.x; i < nce; i += 256) {
    l += ce_partial[2 * i];
    k += ce_partial[2 * i + 1];
  }
  for (int i = threadIdx.x; i < nbce; i += 256) b += bce_partial[i];
  for (int i = threadIdx.x; i < NC; i += 256) r += rterm[i];
  red[0][threadIdx.x] = l;
  red[1][threadIdx.x] = k;
  red[2][threadIdx.x] = b;
  red[3][threadIdx.x] = r;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
#pragma unroll
      for (int j = 0; j < 4; ++j) red[j][threadIdx.x] += red[j][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double nv = red[1][0];
    const double ce = nv > 0.0 ? red[0][0] / nv : 0.0;
    const double bce = red[2][0] / (nv + 1.0);
    const double rmi = red[3][0] / (9.0 * N);
    const double bw = bce_weight;
    loss_out[0] = static_cast<float>(bw * bce + (1.0 - bw) * rmi + static_cast<double>(ce_weight) * ce);
    loss_out[1] = static_cast<float>(nv);
    loss_out[2] = static_cast<float>(bce);
    loss_out[3] = static_cast<float>(rmi);
    loss_out[4] = static_cast<float>(ce);
    sc[0] = nv > 0.0 ? static_cast<float>(ce_weight / nv) : 0.f;
    sc[1] = 1.f;
    sc[2] = static_cast<float>(bw / (nv + 1.0));
    sc[3] = static_cast<float>((1.0 - bw) / (144.0 * N));
  }
}

// dr/dQ per pooled cell: one thread per cell of one (n, c) (blockIdx.x), the 5x5 patch of Y and Q around the cell in
// registers, the table record in shared memory; sum over the neighbourhoods k = cell - d that exist.
__global__ void __launch_bounds__(256)
rmi_dq_kernel(const float* __restrict__ pooled, int NC, int Hp, int Wp, const float* __restrict__ table,
              float* __restrict__ dq) {
  __shared__ float s_t[kRmiRecUsed];
  const int nc = blockIdx.x;
  for (int i = threadIdx.x; i < kRmiRecUsed; i += 256) s_t[i] = table[static_cast<size_t>(nc) * kRmiRec + i];
  __syncthreads();
  const int cell = blockIdx.y * 256 + threadIdx.x;
  if (cell >= Hp * Wp) return;
  const size_t plane = static_cast<size_t>(Hp) * Wp;
  const float* Y = pooled + static_cast<size_t>(nc) * plane;
  const float* Q = pooled + (static_cast<size_t>(NC) + nc) * plane;
  const int i = cell / Wp, j = cell % Wp;
  float yv[25], qv[25];
#pragma unroll
  for (int p = 0; p < 25; ++p) {
    const int yi = i + p / 5 - 2, xj = j + p % 5 - 2;
    const bool in = yi >= 0 && yi < Hp && xj >= 0 && xj < Wp;
    yv[p] = in ? Y[static_cast<size_t>(yi) * Wp + xj] : 0.f;
    qv[p] = in ? Q[static_cast<size_t>(yi) * Wp + xj] : 0.f;
  }
  float g = 0.f;
#pragma unroll
  for (int d = 0; d < 9; ++d) {
    const int ki = i - d / 3, kj = j - d % 3;
    if (ki < 0 || ki >= Hp - 2 || kj < 0 || kj >= Wp - 2) continue;
#pragma unroll
    for (int e = 0; e < 9; ++e) {
      const int p = (e / 3 - d / 3 + 2) * 5 + (e % 3 - d % 3 + 2);
      g = fmaf(s_t[d * 18 + e], yv[p] - s_t[162 + e], g);
      g = fmaf(s_t[d * 18 + 9 + e], qv[p] - s_t[171 + e], g);
    }
  }
  dq[static_cast<size_t>(nc) * plane + cell] = g;
}

// One interval of the RMI rows kernel for class c: the (left, right) x (top, bottom node row) gradient sums as in
// upsample_ce_bwd_rows_kernel, of the pixel terms in the RMI comment above.
// The interval's Z x Z pixels lie in kRmiCells x kRmiCells pooled cells (Z = 8: 2 x 2; Z <= 4: one, since y0 and xb are
// multiples of Z): their kr dr/dQ are loaded once per interval, 0 for cells outside the pooled map.
template <int Z>
constexpr int kRmiCells = Z == 8 ? 2 : 1;

template <int Z, bool kFull>
__device__ __forceinline__ void rmi_interval(const PixInfo* s, int Wo, int xb, int y0, int rows, int nx, int c,
                                             float a, float b, float cc, float d, const float* __restrict__ dqc,
                                             int Hp, int Wp, float kce, float kbce, float kr, float* acc) {
  using G = Zoom<Z>;
  constexpr int kCells = kRmiCells<Z>;
  float dqv[kCells][kCells];
#pragma unroll
  for (int u = 0; u < kCells; ++u) {
#pragma unroll
    for (int v = 0; v < kCells; ++v) {
      const int cy = (y0 >> 2) + u, cx = (xb >> 2) + v;
      dqv[u][v] = cy < Hp && cx < Wp ? kr * __ldg(dqc + static_cast<size_t>(cy) * Wp + cx) : 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const PixInfo pi = s[r * Wo + xb + k];
      if (pi.t < 0) continue;  // warp-uniform
      const float v = row_lerp<Z>(top, bot, r);
      const float p = ex2_approx(fmaf(v, kLog2e, -pi.lse2));
      const float e = rmi_exp_neg_abs(v);
      const float rr = __fdividef(1.f, 1.f + e);
      const float sg = (v >= 0.f ? 1.f : e) * rr;
      const float yc = c == pi.t ? 1.f : 0.f;
      float g = fmaf(kce, p - yc, kbce * (sg - yc));
      g = fmaf(e * rr * rr, dqv[kCells == 2 ? r >> 2 : 0][kCells == 2 ? k >> 2 : 0], g);
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

// Rows layout of upsample_ce_bwd_rows_kernel (one CTA per (interval row, image), one thread per class, (lse, t) of the
// interval's Z output rows staged per pixel): T2 of the RMI + BCE + CE gradient; dq = dr/dQ, sc = the loss scalars.
template <int Z>
__global__ void __launch_bounds__(256)
upsample_ce_rmi_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                            const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                            const float* __restrict__ lse, const float* __restrict__ dq, const float* __restrict__ sc,
                            float* __restrict__ T2) {
  extern __shared__ PixInfo s_rpix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const long long t = target[rowbase + x];
      PixInfo pi;
      pi.t = (t == ignore_index || t < 0 || t >= C) ? -1 : static_cast<int>(t);
      pi.lse2 = lse[rowbase + x] * kLog2e;
      s_rpix[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const float kce = sc[0], kbce = sc[2], kr = sc[3];
  const int Hp = Ho >> 2, Wp = Wo >> 2;
  const float* dqc = dq + (static_cast<size_t>(n) * C + c) * Hp * Wp;
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];
    nd = L1[static_cast<size_t>(jn) * pitch];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      rmi_interval<Z, true>(s_rpix, Wo, xb, Z * i0, rows, nx, c, a, b, cc, d, dqc, Hp, Wp, kce, kbce, kr, acc);
    } else {
      rmi_interval<Z, false>(s_rpix, Wo, xb, Z * i0, rows, nx, c, a, b, cc, d, dqc, Hp, Wp, kce, kbce, kr, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
  }
}

// ---------------------------------------------------------------------------------------------------- entropy
// Entropy minimisation (TENT, ADVENT's MinEnt, entropy regularisation) plus cross-entropy, with s the logits after the
// xZ upsample:
//   L = {target in [0, C), target != ignore_index},  U = {target == ignore_index}
//   p = softmax(s),  lse = logsumexp(s),  H = lse - sum_c p_c s_c = -sum_c p_c log p_c
//   loss = ce_weight (1/|L|) sum_L (lse - s_target) + ent_weight (1/|U|) sum_U H
//   dloss/ds_c = ce_weight/|L| (p_c - [c = t]) on L,   -ent_weight/|U| p_c (s_c - lse + H) on U
// and s_c - lse + H = s_c - mu with mu = sum_c p_c s_c, the softmax-expected logit.
// forward : the plain forward's two class passes (lse and argmax are the plain tail's bits); the second pass also sums,
//           with e_c = exp(s_c - m) (m: the pixel's max, at class a), S_o = sum_{c != a} e_c with a's term skipped, not
//           subtracted, and D = sum_c e_c (s_c - m) <= 0. With S = 1 + S_o (a's term exactly 1): mu = m + D / S and
//           H = log1p(S_o) - D / S, two non-negative terms. So H is >= 0, finite, and keeps its relative accuracy when
//           the logits saturate (a term whose e_c underflowed adds exactly 0; log S is not a rounded log near 1). Per
//           pixel lse and mu are written; per CTA (sum CE over L, |L|) and (sum H over U, |U|), each reduced in fp64 by
//           the plain reduce kernel, as the pseudo-label forward does. Constant logits give D = 0 and mu = s_c exactly.
// backward: the rows kernel stages (lse, class or U marker, mu) per pixel, the Dice 12-byte word, and reads |L| and |U|
//           from the forward's loss words for the two per-pixel weights; the plain cols kernel with a count of 1.
// loss_out: [0] CE mean over L, [1] |L|, [2] H mean over U, [3] |U|, [4] 0, [5] 1 (the cols kernel's count).
constexpr int kEntNone = -1;   // staged target of a pixel with no term (or whose term has weight 0)
constexpr int kEntU = -2;      // staged target of an unlabelled pixel

template <int Z>
__global__ void __launch_bounds__(kFwdCols)
upsample_ce_entropy_fwd_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs,
                               const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                               float* __restrict__ partial, float* __restrict__ loss_out,
                               long long* __restrict__ argmax_out, float* __restrict__ lse_out,
                               float* __restrict__ mu_out) {
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs] as in upsample_ce_fwd_kernel
  __shared__ float red[4][kFwdCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  if ((blockIdx.x | blockIdx.y | blockIdx.z) == 0 && tid == 0) {
    loss_out[4] = 0.f;
    loss_out[5] = 1.f;
  }
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  __syncthreads();
  float acc[4] = {0.f, 0.f, 0.f, 0.f};   // sum CE over L, |L|, sum H over U, |U|
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* A = S + (j0 - j_base) * Cs;
    const float* B = S + (j1 - j_base) * Cs;
    const float* Cc = A + kFwdNodes * Cs;
    const float* D = B + kFwdNodes * Cs;
    float m[Z], sum[Z], so[Z], sd[Z];   // so: S_o = sum_{c != argmax} e_c; sd: D = sum_c e_c (s_c - m) <= 0
    int am[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      m[r] = -INFINITY;
      am[r] = 0;
      sum[r] = 0.f;
      so[r] = 0.f;
      sd[r] = 0.f;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        if (v > m[r]) {
          m[r] = v;
          am[r] = c;
        }
      }
    }
    float m2[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) m2[r] = m[r] * kLog2e;
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        const float e = ex2_approx(fmaf(v, kLog2e, -m2[r]));   // the plain forward's sum
        sum[r] += e;
        so[r] += c == am[r] ? 0.f : e;
        sd[r] = fmaf(e, v - m[r], sd[r]);
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo + x;
        const long long t = target[pix];
        const float lse = m[r] + __logf(sum[r]);
        const float dm = sd[r] / (1.f + so[r]);   // D / S with the argmax's term taken as exactly 1
        if (argmax_out) argmax_out[pix] = am[r];
        lse_out[pix] = lse;
        mu_out[pix] = m[r] + dm;
        if (t == ignore_index) {
          const float H = log1pf(so[r]) - dm;
          acc[2] += H;
          acc[3] += 1.f;
        } else if (t >= 0 && t < C) {
          const int tc = static_cast<int>(t);
          const float top = Z == 1 ? A[tc] : l0w * A[tc] + l1w * B[tc];
          const float bot = Z == 1 ? 0.f : l0w * Cc[tc] + l1w * D[tc];
          acc[0] += lse - row_lerp<Z>(top, bot, r);
          acc[1] += 1.f;
        }
      }
    }
  }
  // deterministic block reduction -> (sum CE, |L|) and (sum H, |U|) per CTA, each laid out as the plain partials
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
  }
  if ((tid & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) red[k][tid >> 5] = acc[k];
  }
  __syncthreads();
  if (tid < 4) {
    float s = 0.f;
    for (int i = 0; i < kFwdCols / 32; ++i) s += red[tid][i];
    const size_t nb = static_cast<size_t>(gridDim.x) * gridDim.y * gridDim.z;
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[(tid >> 1) * 2 * nb + 2 * b + (tid & 1)] = s;
  }
}

// One interval of the entropy rows kernel for class c, folded as in upsample_ce_bwd_rows_kernel. DicePix::t is the
// target class on L, kEntU on U; DicePix::g holds mu.
template <int Z, bool kFull>
__device__ __forceinline__ void entropy_interval(const DicePix* s, int Wo, int xb, int rows, int nx, int c, float a,
                                                 float b, float cc, float d, float wl, float wu, float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const DicePix pi = s[r * Wo + xb + k];
      if (pi.t == kEntNone) continue;  // warp-uniform
      const float v = row_lerp<Z>(top, bot, r);
      const float p = ex2_approx(fmaf(v, kLog2e, -pi.lse2));
      const float g = pi.t >= 0 ? wl * (p - (c == pi.t ? 1.f : 0.f)) : wu * p * (pi.g - v);
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

// Rows layout of upsample_ce_bwd_rows_kernel with the Dice rows kernel's 12-byte pixel word (lse, target / kEntU, mu).
// The weights ce_weight / |L| and ent_weight / |U| come from the forward's loss words (0 for an empty set); a pixel
// whose term has weight 0 is staged as kEntNone: its gradient is exactly 0.
template <int Z>
__global__ void __launch_bounds__(256)
upsample_ce_entropy_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C,
                                const long long* __restrict__ target, int Ho, int Wo, int ignore_index,
                                float ent_weight, float ce_weight, const float* __restrict__ lse,
                                const float* __restrict__ mu, const float* __restrict__ loss_info,
                                float* __restrict__ T2) {
  extern __shared__ DicePix s_dpix[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  const float nl = loss_info[1], nu = loss_info[3];
  const float wl = nl > 0.f ? ce_weight / nl : 0.f;
  const float wu = nu > 0.f ? ent_weight / nu : 0.f;
  for (int r = 0; r < rows; ++r) {
    const size_t rowbase = (static_cast<size_t>(n) * Ho + (Z * i0 + r)) * Wo;
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const long long t = target[rowbase + x];
      DicePix pi;
      if (t == ignore_index) {
        pi.t = wu != 0.f ? kEntU : kEntNone;
      } else {
        pi.t = (t >= 0 && t < C && wl != 0.f) ? static_cast<int>(t) : kEntNone;
      }
      pi.g = mu[rowbase + x];
      pi.lse2 = lse[rowbase + x] * kLog2e;
      s_dpix[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];
    nd = L1[static_cast<size_t>(jn) * pitch];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      entropy_interval<Z, true>(s_dpix, Wo, xb, rows, nx, c, a, b, cc, d, wl, wu, acc);
    } else {
      entropy_interval<Z, false>(s_dpix, Wo, xb, rows, nx, c, a, b, cc, d, wl, wu, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
  }
}

// ---------------------------------------------------------------------------------------------------- label relaxation
// Boundary label relaxation (Zhu et al., CVPR 2019). S_i is the set of valid labels (target != ignore_index, in [0, C))
// in the (2 border + 1)^2 window of the target grid centred on valid pixel i, clipped to the image; w the class weights
// (all ones when none are given). With p = softmax(v), per valid pixel:
//   l_i = -log sum_{c in S_i} p_c,   omega_i = (1/|S_i|) sum_{c in S_i} w_c,   loss = sum omega l / D,  D = sum omega
//   dl_i/dv_c = p_c - [c in S_i] p_c / (1 - R_i),   R_i = sum_{c not in S_i} p_c
// and loss 0 with an exactly zero gradient when D = 0.
// Three passes:
//   sets    : one thread per target pixel scans its window once and writes a tag (-1: not valid; t: interior, S = {t};
//             kRelaxSet: boundary), omega, and for a boundary pixel its set as a bit mask of ceil(C/32) words. The
//             window costs (2 border + 1)^2 target reads per pixel, hence the cap kRelaxMaxBorder.
//   forward : the plain forward's two class passes (lse and argmax keep its bits); the second also sums the set's mass
//             e_S and its complement e_R (e_c = ex2((v_c - m) log2e)), each term added to one sum, never subtracted. Then
//             l = log1p(e_R / e_S) (= -log1p(-R), no rounded 1 - R: small losses keep their relative accuracy; 0 when
//             S holds every class) and q = R / (1 - R) = e_R / e_S is kept as lq = log2 q for the backward. Where e_S
//             has underflowed, l = lse - lse_S over the set's members and q = expm1(l) = exp(l) in fp32. The partials
//             (sum omega l, sum omega) go to the weighted-mean reduce.
//   backward: the rows layout with a 12-byte pixel word (the Dice width limit) holding the two exponent offsets
//             a = lse log2e - log2 omega and b = a - lq: g = ex2(v log2e - a) = omega p_c outside the set and
//             g = -ex2(v log2e - b) = -omega p_c q inside it (the in-set term p_c - p_c / (1 - R) without its
//             cancellation), then the weighted-mean cols kernel. Membership is c == t for an interior pixel and one
//             warp-uniform mask word (a warp's 32 classes) for a boundary one.
constexpr int kRelaxSet = 1 << 30;    // tag of a boundary pixel (any value >= kMaxClasses)
constexpr int kRelaxMaxBorder = 4;
constexpr int kRelaxThreads = 256;

__global__ void __launch_bounds__(kRelaxThreads)
upsample_relax_sets_kernel(const long long* __restrict__ target, int N, int Ho, int Wo, int C, int ignore_index,
                           int border, const float* __restrict__ class_weight, int* __restrict__ tag,
                           float* __restrict__ omega, unsigned* __restrict__ mask) {
  __shared__ unsigned s_mask[(kMaxClasses / 32) * kRelaxThreads];   // thread-private: word k at [k][tid]
  const long long M = static_cast<long long>(N) * Ho * Wo;
  const long long pix = static_cast<long long>(blockIdx.x) * kRelaxThreads + threadIdx.x;
  if (pix >= M) return;
  const long long t = target[pix];
  if (t == ignore_index || t < 0 || t >= C) {
    tag[pix] = -1;
    omega[pix] = 0.f;
    return;
  }
  const int nw = (C + 31) >> 5;
  const int x = static_cast<int>(pix % Wo);
  const long long ny = pix / Wo;
  const int y = static_cast<int>(ny % Ho);
  const long long* img = target + (ny / Ho) * Ho * Wo;
  unsigned* sm = s_mask + threadIdx.x;
  for (int k = 0; k < nw; ++k) sm[k * kRelaxThreads] = 0u;
  bool interior = true;
  const int ya = max(y - border, 0), yb = min(y + border, Ho - 1);
  const int xa = max(x - border, 0), xb = min(x + border, Wo - 1);
  for (int yy = ya; yy <= yb; ++yy) {
    for (int xx = xa; xx <= xb; ++xx) {
      const long long l = img[static_cast<size_t>(yy) * Wo + xx];
      if (l == ignore_index || l < 0 || l >= C) continue;
      const int li = static_cast<int>(l);
      sm[(li >> 5) * kRelaxThreads] |= 1u << (li & 31);
      interior = interior && l == t;
    }
  }
  const int tc = static_cast<int>(t);
  if (interior) {
    tag[pix] = tc;
    omega[pix] = class_weight ? class_weight[tc] : 1.f;
    return;
  }
  // the weights summed in ascending class order; without weights omega = |S| / |S| = 1 exactly
  unsigned* mk = mask + pix * nw;
  float wsum = 0.f;
  int cnt = 0;
  for (int k = 0; k < nw; ++k) {
    unsigned bits = sm[k * kRelaxThreads];
    mk[k] = bits;
    cnt += __popc(bits);
    while (bits) {
      const int c = 32 * k + __ffs(bits) - 1;
      bits &= bits - 1;
      wsum += class_weight ? class_weight[c] : 1.f;
    }
  }
  tag[pix] = kRelaxSet;
  omega[pix] = wsum / static_cast<float>(cnt);
}

// Mask word k (classes [32k, 32k + 32)) of a pixel's set from its tag: an interior pixel's is its label's bit.
__device__ __forceinline__ unsigned relax_word(int tg, const unsigned* __restrict__ mask, size_t pix, int nw, int k) {
  if (tg == kRelaxSet) return mask[pix * nw + k];
  return tg >= 0 && (tg >> 5) == k ? 1u << (tg & 31) : 0u;
}

template <int Z>
__global__ void __launch_bounds__(kFwdCols)
upsample_relax_fwd_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Cs, int Ho,
                          int Wo, const int* __restrict__ tag, const float* __restrict__ omega,
                          const unsigned* __restrict__ mask, float* __restrict__ partial,
                          long long* __restrict__ argmax_out, float* __restrict__ lse_out, float* __restrict__ lq_out) {
  using G = Zoom<Z>;
  constexpr int kFwdNodes = G::kNodes;
  extern __shared__ float S[];  // [kNodeRows][kFwdNodes][Cs] as in upsample_ce_fwd_kernel
  __shared__ float red_loss[kFwdCols / 32];
  __shared__ float red_cnt[kFwdCols / 32];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kFwdCols;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> G::kShift;
  const int nj = min(kFwdNodes, w - j_base);
  const int tid = threadIdx.x;
  for (int idx = tid; idx < G::kNodeRows * nj * C; idx += kFwdCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kFwdNodes + jj) * Cs + c] =
        logits[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  __syncthreads();
  float loss = 0.f, cnt = 0.f;
  const int x = x0 + tid;
  const int rows = min(Z, Ho - Z * i0);
  if (x < Wo) {
    const int j0 = x >> G::kShift;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & G::kMask) * G::kStep, l0w = 1.f - l1w;
    const float* A = S + (j0 - j_base) * Cs;
    const float* B = S + (j1 - j_base) * Cs;
    const float* Cc = A + kFwdNodes * Cs;
    const float* D = B + kFwdNodes * Cs;
    const size_t pix0 = (static_cast<size_t>(n) * Ho + Z * i0) * Wo + x;   // row r: pix0 + r * Wo
    const int nw = (C + 31) >> 5;
    float m[Z], sum[Z], er[Z], es[Z];   // er, es: the complement's and the set's sums of e_c
    int am[Z], tg[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      m[r] = -INFINITY;
      am[r] = 0;
      sum[r] = 0.f;
      er[r] = 0.f;
      es[r] = 0.f;
      tg[r] = r < rows ? tag[pix0 + static_cast<size_t>(r) * Wo] : -1;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
      const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
      for (int r = 0; r < Z; ++r) {
        const float v = row_lerp<Z>(top, bot, r);
        if (v > m[r]) {
          m[r] = v;
          am[r] = c;
        }
      }
    }
    float m2[Z];
#pragma unroll
    for (int r = 0; r < Z; ++r) m2[r] = m[r] * kLog2e;
    for (int k = 0; k < nw; ++k) {
      unsigned bits[Z];
#pragma unroll
      for (int r = 0; r < Z; ++r) bits[r] = relax_word(tg[r], mask, pix0 + static_cast<size_t>(r) * Wo, nw, k);
      const int c_end = min(C, 32 * k + 32);
#pragma unroll 2
      for (int c = 32 * k; c < c_end; ++c) {
        const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
        const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
#pragma unroll
        for (int r = 0; r < Z; ++r) {
          const float v = row_lerp<Z>(top, bot, r);
          const float e = ex2_approx(fmaf(v, kLog2e, -m2[r]));
          const bool in = bits[r] & 1u;
          bits[r] >>= 1;
          sum[r] += e;
          er[r] += in ? 0.f : e;
          es[r] += in ? e : 0.f;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (r < rows) {
        const size_t pix = pix0 + static_cast<size_t>(r) * Wo;
        const float lse = m[r] + __logf(sum[r]);
        if (argmax_out) argmax_out[pix] = am[r];
        lse_out[pix] = lse;
        float lq = 0.f;
        if (tg[r] >= 0) {
          float nll;
          if (es[r] > kFocalMinEt) {
            const float q = er[r] / es[r];
            nll = log1pf(q);
            lq = log2f(q);      // -inf when S holds all the mass: the in-set gradient is exactly 0
          } else {
            // lse_S over the set's members, against their own maximum
            auto member_v = [&](int c) {
              const float top = Z == 1 ? A[c] : l0w * A[c] + l1w * B[c];
              const float bot = Z == 1 ? 0.f : l0w * Cc[c] + l1w * D[c];
              return row_lerp<Z>(top, bot, r);
            };
            float ms = -INFINITY, ss = 0.f;
            for (int k = 0; k < nw; ++k) {
              for (unsigned b = relax_word(tg[r], mask, pix, nw, k); b; b &= b - 1) {
                ms = fmaxf(ms, member_v(32 * k + __ffs(b) - 1));
              }
            }
            for (int k = 0; k < nw; ++k) {
              for (unsigned b = relax_word(tg[r], mask, pix, nw, k); b; b &= b - 1) {
                ss += __expf(member_v(32 * k + __ffs(b) - 1) - ms);
              }
            }
            nll = lse - (ms + __logf(ss));
            lq = nll * kLog2e;
          }
          const float wgt = omega[pix];
          loss = fmaf(wgt, nll, loss);
          cnt += wgt;
        }
        lq_out[pix] = lq;
      }
    }
  }
  // deterministic block reduction -> one (sum of omega l, sum of omega) partial per CTA, as upsample_ce_fwd_kernel
  for (int o = 16; o > 0; o >>= 1) {
    loss += __shfl_xor_sync(0xffffffffu, loss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((tid & 31) == 0) {
    red_loss[tid >> 5] = loss;
    red_cnt[tid >> 5] = cnt;
  }
  __syncthreads();
  if (tid == 0) {
    float l = 0.f, k = 0.f;
    for (int i = 0; i < kFwdCols / 32; ++i) {
      l += red_loss[i];
      k += red_cnt[i];
    }
    const size_t b = (static_cast<size_t>(blockIdx.z) * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * b] = l;
    partial[2 * b + 1] = k;
  }
}

struct RelaxPix {
  float a;   // lse log2e - log2 omega: the exponent offset outside the set
  int t;     // -1: no gradient; the label of an interior pixel; kRelaxSet: a boundary pixel
  float b;   // a - log2 q: the exponent offset inside the set
};
static_assert(sizeof(RelaxPix) == 12, "the relaxation rows kernel stages the Dice words' 12 bytes per pixel");

// One interval of the relaxation rows kernel for class c, folded as in upsample_ce_bwd_rows_kernel. mk_c points at the
// mask word of class c of pixel 0; pix0 is the interval's first output row's first pixel.
template <int Z, bool kFull>
__device__ __forceinline__ void relax_interval(const RelaxPix* s, int Wo, int xb, int rows, int nx, int c,
                                               const unsigned* __restrict__ mk_c, size_t pix0, int nw, float a,
                                               float b, float cc, float d, float* acc) {
  using G = Zoom<Z>;
#pragma unroll
  for (int k = 0; k < Z; ++k) {
    if (!kFull && k >= nx) break;
    const float l1w = G::kStep * k, l0w = 1.f - l1w;
    const float top = l0w * a + l1w * b;
    const float bot = l0w * cc + l1w * d;
    float g0 = 0.f, g1 = 0.f;
#pragma unroll
    for (int r = 0; r < Z; ++r) {
      if (!kFull && r >= rows) break;
      const RelaxPix pi = s[r * Wo + xb + k];
      if (pi.t < 0) continue;  // warp-uniform
      const bool in = pi.t == kRelaxSet  // warp-uniform; the word is the same for the warp's 32 classes
                          ? (mk_c[(pix0 + static_cast<size_t>(r) * Wo + xb + k) * nw] >> (c & 31)) & 1u
                          : c == pi.t;
      const float v = row_lerp<Z>(top, bot, r);
      const float e = ex2_approx(fmaf(v, kLog2e, -(in ? pi.b : pi.a)));
      const float g = in ? -e : e;
      g0 = fmaf(1.f - G::kStep * r, g, g0);
      g1 = fmaf(G::kStep * r, g, g1);
    }
    acc[0] = fmaf(l0w, g0, acc[0]);
    acc[1] = fmaf(l1w, g0, acc[1]);
    acc[2] = fmaf(l0w, g1, acc[2]);
    acc[3] = fmaf(l1w, g1, acc[3]);
  }
}

template <int Z>
__global__ void __launch_bounds__(256)
upsample_relax_rows_kernel(const float* __restrict__ logits, int pitch, int N, int h, int w, int C, int Ho, int Wo,
                           const float* __restrict__ lse, const int* __restrict__ tag, const float* __restrict__ omega,
                           const unsigned* __restrict__ mask, const float* __restrict__ lq, float* __restrict__ T2) {
  extern __shared__ RelaxPix s_relax[];  // [Z][Wo]
  const int i0 = blockIdx.x, n = blockIdx.y;
  const int i1 = min(i0 + 1, h - 1);
  const int rows = min(Z, Ho - Z * i0);
  const size_t pix0 = (static_cast<size_t>(n) * Ho + Z * i0) * Wo;
  for (int r = 0; r < rows; ++r) {
    for (int x = threadIdx.x; x < Wo; x += blockDim.x) {
      const size_t pix = pix0 + static_cast<size_t>(r) * Wo + x;
      const int tg = tag[pix];
      const float wgt = omega[pix];
      RelaxPix pi;
      pi.t = tg < 0 || wgt == 0.f ? -1 : tg;
      pi.a = pi.t < 0 ? 0.f : lse[pix] * kLog2e - (wgt == 1.f ? 0.f : log2f(wgt));
      pi.b = pi.t < 0 ? 0.f : pi.a - lq[pix];
      s_relax[r * Wo + x] = pi;
    }
  }
  __syncthreads();
  const int c = threadIdx.x;
  if (c >= C) return;
  const int nw = (C + 31) >> 5;
  const unsigned* mk_c = mask + (c >> 5);
  const float* L0 = logits + (static_cast<size_t>(n) * h + i0) * w * pitch + c;
  const float* L1 = logits + (static_cast<size_t>(n) * h + i1) * w * pitch + c;
  float* T0 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 0) * w * C + c;
  float* T1 = T2 + ((static_cast<size_t>(n) * h + i0) * 2 + 1) * w * C + c;
  float a = L0[0], cc = L1[0];
  float nb = L0[static_cast<size_t>(min(1, w - 1)) * pitch], nd = L1[static_cast<size_t>(min(1, w - 1)) * pitch];
  float carry0 = 0.f, carry1 = 0.f;
  for (int j0 = 0; j0 < w; ++j0) {
    const float b = nb, d = nd;
    const int jn = min(j0 + 2, w - 1);
    nb = L0[static_cast<size_t>(jn) * pitch];
    nd = L1[static_cast<size_t>(jn) * pitch];
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    const int xb = j0 * Z;
    const int nx = min(Z, Wo - xb);
    if (rows == Z && nx == Z) {
      relax_interval<Z, true>(s_relax, Wo, xb, rows, nx, c, mk_c, pix0, nw, a, b, cc, d, acc);
    } else {
      relax_interval<Z, false>(s_relax, Wo, xb, rows, nx, c, mk_c, pix0, nw, a, b, cc, d, acc);
    }
    T0[static_cast<size_t>(j0) * C] = carry0 + acc[0];
    T1[static_cast<size_t>(j0) * C] = carry1 + acc[2];
    carry0 = acc[1];
    carry1 = acc[3];
    a = b;
    cc = d;
  }
}

}  // namespace sb

using namespace sb;

static bool valid_zoom(int zoom) { return zoom == 1 || zoom == 2 || zoom == 4 || zoom == 8; }

static int check_tail(const void* logits, int pitch, int N, int h, int w, int C, const void* target, int Ho, int Wo,
                      int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(logits && target, "upsample_ce: null pointer");
  SB_CHECK_ARG(N > 0 && h > 1 && w > 1 && C > 1 && C <= kMaxClasses && pitch >= C, "upsample_ce: bad sizes (C<=%d)",
               kMaxClasses);
  SB_CHECK_ARG(Ho == zoom * (h - 1) + 1 && Wo == zoom * (w - 1) + 1,
               "upsample_ce: fused kernel needs Ho=%d(h-1)+1, Wo=%d(w-1)+1 (got %dx%d -> %dx%d)", zoom, zoom, h, w, Ho,
               Wo);
  return SEMSEG_OK;
}

// The opt-in to more than 48 KB of dynamic shared memory is per device (nn.DataParallel replicas run the same kernels on
// several devices, from several threads): made once for every device this process uses, to the kernel's largest size,
// before the first launch on that device that needs it.
template <typename Kernel>
static int opt_in_smem(Kernel kernel, std::atomic<bool>* attr_set, int max_bytes) {
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_bytes));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  return SEMSEG_OK;
}

constexpr size_t kSmemDefault = 48 * 1024;
constexpr size_t kBwdSmemMax = 160 * 1024;   // staged (lse, target) words of the backward's Z output rows

static int fwd_ctas(int N, int h, int Wo) { return cdiv(Wo, kFwdCols) * h * N; }

template <int Z, bool kOhem, bool kWeighted = false>
static int launch_fwd_kernel(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                             int Wo, int ignore_index, float* partial, int64_t* argmax, float* lse, float* pt,
                             float* nll, cudaStream_t stream, const float* class_weight = nullptr,
                             float smoothing = 0.f) {
  dim3 grid(cdiv(Wo, kFwdCols), h, N);
  const int Cs = C | 1;
  // the weighted cross-entropy form stages the C class weights and W after the node rows
  constexpr size_t kWeightFloats = kWeighted && !kOhem ? kMaxClasses + 1 : 0;
  const size_t weight_floats = kWeighted && !kOhem ? C + 1 : 0;
  // at most 2 * 65 * 257 floats (Z = 2, 256 classes); above 48 KB only at Z <= 4 (Z = 1 and 2 with 150 classes: 78 KB)
  constexpr size_t kMaxSmem =
      (static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) + kWeightFloats) * sizeof(float);
  const size_t smem = (static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs + weight_floats) * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_fwd_kernel<Z, kOhem, kWeighted>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_ce_fwd_kernel<Z, kOhem, kWeighted><<<grid, kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, partial,
      reinterpret_cast<long long*>(argmax), lse, pt, nll, class_weight, smoothing);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z, bool kWeighted = false>
static int launch_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho, int Wo,
                      int ignore_index, float* workspace, float* loss_out, int64_t* argmax, float* lse,
                      cudaStream_t stream, const float* class_weight = nullptr, float smoothing = 0.f) {
  int r = launch_fwd_kernel<Z, false, kWeighted>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace,
                                                 argmax, lse, nullptr, nullptr, stream, class_weight, smoothing);
  if (r) return r;
  upsample_ce_reduce_kernel<kWeighted><<<1, 256, 0, stream>>>(workspace, fwd_ctas(N, h, Wo), loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

static long long ohem_hist_ctas(long long M) { return std::min<long long>((M + kSelThreads - 1) / kSelThreads, 8LL * num_sms()); }
static long long ohem_mask_ctas(long long M) { return (M + kMaskPix - 1) / kMaskPix; }

// Workspace: kSelWords selection words, then (loss, count) per masked-reduce CTA.
template <int Z, bool kWeighted = false>
static int launch_ohem_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                           int Wo, int ignore_index, float thresh, int min_kept, float* workspace, float* loss_out,
                           int64_t* argmax, float* lse, float* pt, float* nll, float* thr, cudaStream_t stream,
                           const float* class_weight = nullptr) {
  const long long M = static_cast<long long>(N) * Ho * Wo;
  unsigned* sel = reinterpret_cast<unsigned*>(workspace);
  float* partial = workspace + kSelWords;
  SB_CUDA(cudaMemsetAsync(sel, 0, kSelWords * sizeof(unsigned), stream));
  int r = launch_fwd_kernel<Z, true, kWeighted>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, nullptr,
                                                argmax, lse, pt, nll, stream, class_weight);
  if (r) return r;
  const int hist_ctas = static_cast<int>(ohem_hist_ctas(M));
  for (int pass = 0; pass < 4; ++pass) {
    ohem_hist_kernel<<<hist_ctas, kSelThreads, 0, stream>>>(pt, M, pass, sel);
    SB_LAUNCHED();
    ohem_select_kernel<<<1, kSelThreads, 0, stream>>>(sel, pass, thresh, min_kept, thr);
    SB_LAUNCHED();
  }
  const int mask_ctas = static_cast<int>(ohem_mask_ctas(M));
  ohem_masked_sum_kernel<<<mask_ctas, kSelThreads, 0, stream>>>(pt, nll, M, thr, partial);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(partial, mask_ctas, loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z, bool kOhem, bool kWeighted = false>
static int launch_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho, int Wo,
                      int ignore_index, const float* lse, const float* loss_info, const float* grad_out,
                      float* workspace, float* dlogits, const float* pt, const float* thr, cudaStream_t stream,
                      const float* class_weight = nullptr, float smoothing = 0.f) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(PixInfo);
  SB_CHECK_ARG(smem <= kBwdSmemMax, "upsample_ce_bwd: output width %d too large for the staged rows", Wo);
  // the weighted forms stage the class weights and W after the pixel words: the width limit stays the plain one
  constexpr size_t kWeightBytes = kWeighted ? (kMaxClasses + 1) * sizeof(float) : 0;
  const size_t smem_all = smem + (kWeighted ? (C + 1) * sizeof(float) : 0);
  static std::atomic<bool> attr_set[64];
  if (smem_all > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_bwd_rows_kernel<Z, kOhem, kWeighted>, attr_set,
                        static_cast<int>(kBwdSmemMax + kWeightBytes));
    if (r) return r;
  }
  upsample_ce_bwd_rows_kernel<Z, kOhem, kWeighted><<<dim3(h, N), threads, smem_all, stream>>>(
      logits, pitch, N, h, w, C, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lse, workspace, pt,
      thr, class_weight, smoothing);
  SB_LAUNCHED();
  upsample_ce_bwd_cols_kernel<kWeighted && !kOhem><<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, loss_info,
                                                                                  grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_zoom_workspace_floats(int N, int Ho, int Wo, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce: zoom %d is not one of 1, 2, 4, 8", zoom);
  return 2LL * N * ((Ho - 1) / zoom + 1) * cdiv(Wo, kFwdCols);  // (loss, count) per forward CTA
}

extern "C" int semseg_upsample_ce_zoom_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                           const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                           float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse, "upsample_ce_fwd: null output");
  switch (zoom) {
    case 1: return launch_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out, argmax,
                                 lse, stream);
    case 2: return launch_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out, argmax,
                                 lse, stream);
    case 4: return launch_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out, argmax,
                                 lse, stream);
    default: return launch_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out, argmax,
                                  lse, stream);
  }
}

extern "C" long long semseg_upsample_ce_zoom_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce: zoom %d is not one of 1, 2, 4, 8", zoom);
  return 2LL * N * ((Ho - 1) / zoom + 1) * w * C;  // T2[N][h][2][w][C]
}

extern "C" int semseg_upsample_ce_zoom_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                           const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                           const float* lse, const float* loss_info, const float* grad_out,
                                           float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  SB_CHECK_ARG(lse && loss_info && grad_out && dlogits && workspace, "upsample_ce_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_bwd<1, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                        grad_out, workspace, dlogits, nullptr, nullptr, stream);
    case 2: return launch_bwd<2, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                        grad_out, workspace, dlogits, nullptr, nullptr, stream);
    case 4: return launch_bwd<4, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                        grad_out, workspace, dlogits, nullptr, nullptr, stream);
    default: return launch_bwd<8, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                         grad_out, workspace, dlogits, nullptr, nullptr, stream);
  }
}

// OHEM cross-entropy at zoom factor `zoom`: the kOhem instances, the selection and the masked reduce.
static int check_ohem(float thresh, int min_kept) {
  SB_CHECK_ARG(thresh >= 0.f && thresh <= 1.f, "upsample_ce_ohem: thresh %g is not in [0, 1]", thresh);
  SB_CHECK_ARG(min_kept >= 0, "upsample_ce_ohem: min_kept %d is negative", min_kept);
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_ohem_workspace_floats(int N, int Ho, int Wo, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_ohem: zoom %d is not one of 1, 2, 4, 8", zoom);
  return kSelWords + 2LL * ohem_mask_ctas(static_cast<long long>(N) * Ho * Wo);
}

extern "C" int semseg_upsample_ce_ohem_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                           const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                           float thresh, int min_kept, float* workspace, float* loss_out,
                                           int64_t* argmax, float* lse, float* pt, float* nll, float* thr,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_ohem(thresh, min_kept);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && pt && nll && thr, "upsample_ce_ohem_fwd: null output");
  switch (zoom) {
    case 1: return launch_ohem_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                      workspace, loss_out, argmax, lse, pt, nll, thr, stream);
    case 2: return launch_ohem_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                      workspace, loss_out, argmax, lse, pt, nll, thr, stream);
    case 4: return launch_ohem_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                      workspace, loss_out, argmax, lse, pt, nll, thr, stream);
    default: return launch_ohem_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                       workspace, loss_out, argmax, lse, pt, nll, thr, stream);
  }
}

extern "C" long long semseg_upsample_ce_ohem_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_ce_ohem_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                           const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                           const float* lse, const float* pt, const float* thr,
                                           const float* loss_info, const float* grad_out, float* workspace,
                                           float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  SB_CHECK_ARG(lse && pt && thr && loss_info && grad_out && dlogits && workspace, "upsample_ce_ohem_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_bwd<1, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                       grad_out, workspace, dlogits, pt, thr, stream);
    case 2: return launch_bwd<2, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                       grad_out, workspace, dlogits, pt, thr, stream);
    case 4: return launch_bwd<4, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                       grad_out, workspace, dlogits, pt, thr, stream);
    default: return launch_bwd<8, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                        grad_out, workspace, dlogits, pt, thr, stream);
  }
}

// Class-weighted and label-smoothed cross-entropy at zoom factor `zoom`: the kWeighted instances. class_weight NULL =
// all ones.
static int check_smoothing(float label_smoothing) {
  SB_CHECK_ARG(label_smoothing >= 0.f && label_smoothing <= 1.f,
               "upsample_ce_weighted: label_smoothing %g is not in [0, 1]", label_smoothing);
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_weighted_workspace_floats(int N, int Ho, int Wo, int zoom) {
  return semseg_upsample_ce_zoom_workspace_floats(N, Ho, Wo, zoom);
}

extern "C" int semseg_upsample_ce_weighted_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                               const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                               const float* class_weight, float label_smoothing, float* workspace,
                                               float* loss_out, int64_t* argmax, float* lse, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_smoothing(label_smoothing);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse, "upsample_ce_weighted_fwd: null output");
  switch (zoom) {
    case 1: return launch_fwd<1, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                       argmax, lse, stream, class_weight, label_smoothing);
    case 2: return launch_fwd<2, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                       argmax, lse, stream, class_weight, label_smoothing);
    case 4: return launch_fwd<4, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                       argmax, lse, stream, class_weight, label_smoothing);
    default: return launch_fwd<8, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                        argmax, lse, stream, class_weight, label_smoothing);
  }
}

extern "C" long long semseg_upsample_ce_weighted_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_ce_weighted_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                               const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                               const float* class_weight, float label_smoothing, const float* lse,
                                               const float* loss_info, const float* grad_out, float* workspace,
                                               float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_smoothing(label_smoothing);
  if (r) return r;
  SB_CHECK_ARG(lse && loss_info && grad_out && dlogits && workspace, "upsample_ce_weighted_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_bwd<1, false, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                              grad_out, workspace, dlogits, nullptr, nullptr, stream, class_weight,
                                              label_smoothing);
    case 2: return launch_bwd<2, false, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                              grad_out, workspace, dlogits, nullptr, nullptr, stream, class_weight,
                                              label_smoothing);
    case 4: return launch_bwd<4, false, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                              grad_out, workspace, dlogits, nullptr, nullptr, stream, class_weight,
                                              label_smoothing);
    default: return launch_bwd<8, false, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse,
                                               loss_info, grad_out, workspace, dlogits, nullptr, nullptr, stream,
                                               class_weight, label_smoothing);
  }
}

// Weighted OHEM: the OHEM entry points with nll = w_t (lse - v_t) and each kept pixel's gradient scaled by w_t. The
// workspaces are the OHEM ones.
extern "C" int semseg_upsample_ce_ohem_weighted_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                                    const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                                    float thresh, int min_kept, const float* class_weight,
                                                    float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                                    float* pt, float* nll, float* thr, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_ohem(thresh, min_kept);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && pt && nll && thr, "upsample_ce_ohem_weighted_fwd: null output");
  switch (zoom) {
    case 1: return launch_ohem_fwd<1, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                            workspace, loss_out, argmax, lse, pt, nll, thr, stream, class_weight);
    case 2: return launch_ohem_fwd<2, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                            workspace, loss_out, argmax, lse, pt, nll, thr, stream, class_weight);
    case 4: return launch_ohem_fwd<4, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                            workspace, loss_out, argmax, lse, pt, nll, thr, stream, class_weight);
    default: return launch_ohem_fwd<8, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, thresh, min_kept,
                                             workspace, loss_out, argmax, lse, pt, nll, thr, stream, class_weight);
  }
}

extern "C" int semseg_upsample_ce_ohem_weighted_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                                    const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                                    const float* class_weight, const float* lse, const float* pt,
                                                    const float* thr, const float* loss_info, const float* grad_out,
                                                    float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  SB_CHECK_ARG(lse && pt && thr && loss_info && grad_out && dlogits && workspace,
               "upsample_ce_ohem_weighted_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_bwd<1, true, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                             grad_out, workspace, dlogits, pt, thr, stream, class_weight);
    case 2: return launch_bwd<2, true, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                             grad_out, workspace, dlogits, pt, thr, stream, class_weight);
    case 4: return launch_bwd<4, true, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                             grad_out, workspace, dlogits, pt, thr, stream, class_weight);
    default: return launch_bwd<8, true, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, loss_info,
                                              grad_out, workspace, dlogits, pt, thr, stream, class_weight);
  }
}

// Dice loss (+ ce_weight * CE) at zoom factor `zoom`. The rows kernels stage 12 bytes per pixel of the interval's Z
// output rows in at most 224 KB of shared memory: Wo <= 2389 at zoom 8 (the plain form's 8-byte words allow 2560).
constexpr size_t kDiceSmemMax = 224 * 1024;

static int check_dice(int zoom, int Wo, float smooth, float eps, float ce_weight) {
  SB_CHECK_ARG(std::isfinite(smooth) && smooth >= 0.f, "upsample_ce_dice: smooth %g is not finite and >= 0", smooth);
  SB_CHECK_ARG(std::isfinite(eps) && eps >= 0.f, "upsample_ce_dice: eps %g is not finite and >= 0", eps);
  SB_CHECK_ARG(std::isfinite(ce_weight) && ce_weight >= 0.f, "upsample_ce_dice: ce_weight %g is not finite and >= 0",
               ce_weight);
  const size_t max_wo = kDiceSmemMax / (static_cast<size_t>(zoom) * sizeof(DicePix));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_ce_dice: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

template <int Z, bool kGrad>
static int launch_dice_rows(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                            int Wo, int ignore_index, const float* lse, const float* gmap, const float* table,
                            float* out, cudaStream_t stream) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(DicePix);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_dice_rows_kernel<Z, kGrad>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  upsample_ce_dice_rows_kernel<Z, kGrad><<<dim3(h, N), threads, smem, stream>>>(
      logits, pitch, N, h, w, C, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lse, gmap, table,
      out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Forward workspace: the CE partials (2 per forward CTA), the statistics partials [N][h][3][C], then (8-byte aligned)
// the C fp64 loss terms.
static long long dice_terms_offset(int N, int h, int Wo, int C) {
  const long long f = 2LL * fwd_ctas(N, h, Wo) + 3LL * N * h * C;
  return (f + 1) & ~1LL;
}

template <int Z>
static int launch_dice_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                           int Wo, int ignore_index, float smooth, float eps, float ce_weight, float* workspace,
                           float* loss_out, int64_t* argmax, float* lse, float* table, cudaStream_t stream) {
  const int ctas = fwd_ctas(N, h, Wo);
  float* stats = workspace + 2LL * ctas;
  double* terms = reinterpret_cast<double*>(workspace + dice_terms_offset(N, h, Wo, C));
  int r = launch_fwd_kernel<Z, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, argmax, lse,
                                      nullptr, nullptr, stream);
  if (r) return r;
  r = launch_dice_rows<Z, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, nullptr, nullptr, stats,
                                 stream);
  if (r) return r;
  dice_class_reduce_kernel<<<C, 256, 0, stream>>>(stats, N * h, C, smooth, eps, table, terms);
  SB_LAUNCHED();
  dice_loss_kernel<<<1, 256, 0, stream>>>(workspace, ctas, terms, C, ce_weight, loss_out, table);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Backward workspace: T2 [N][h][2][w][C] of the rows kernel, then the G map [N][Ho][Wo].
template <int Z>
static int launch_dice_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                           int Wo, int ignore_index, const float* lse, const float* table, const float* grad_out,
                           float* workspace, float* dlogits, cudaStream_t stream) {
  float* gmap = workspace + 2LL * N * h * w * C;
  const int Cs = C | 1;
  const size_t smem = (static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs + 2 * C) * sizeof(float);
  constexpr size_t kMaxSmem =
      (static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) + 2 * kMaxClasses) * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_dice_g_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_ce_dice_g_kernel<Z><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lse, table,
      gmap);
  SB_LAUNCHED();
  int r = launch_dice_rows<Z, true>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, gmap, table,
                                    workspace, stream);
  if (r) return r;
  // table[5C + 1] = 1: the plain cols kernel's count, so dlogits = grad_out[0] * T2 sums
  upsample_ce_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, table + kDiceWords * C, grad_out,
                                                             dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_dice_workspace_floats(int N, int Ho, int Wo, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_dice: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && C > 0, "upsample_ce_dice: bad sizes");
  return dice_terms_offset(N, (Ho - 1) / zoom + 1, Wo, C) + 2LL * C;
}

extern "C" int semseg_upsample_ce_dice_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                           const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                           float smooth, float eps, float ce_weight, float* workspace,
                                           float* loss_out, int64_t* argmax, float* lse, float* table,
                                           void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_dice(zoom, Wo, smooth, eps, ce_weight);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && table, "upsample_ce_dice_fwd: null output");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "upsample_ce_dice_fwd: workspace not 8-byte aligned");
  switch (zoom) {
    case 1: return launch_dice_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, smooth, eps, ce_weight,
                                      workspace, loss_out, argmax, lse, table, stream);
    case 2: return launch_dice_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, smooth, eps, ce_weight,
                                      workspace, loss_out, argmax, lse, table, stream);
    case 4: return launch_dice_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, smooth, eps, ce_weight,
                                      workspace, loss_out, argmax, lse, table, stream);
    default: return launch_dice_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, smooth, eps,
                                       ce_weight, workspace, loss_out, argmax, lse, table, stream);
  }
}

extern "C" long long semseg_upsample_ce_dice_bwd_workspace_floats(int N, int Ho, int Wo, int w, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_dice: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && w > 0 && C > 0, "upsample_ce_dice: bad sizes");
  return 2LL * N * ((Ho - 1) / zoom + 1) * w * C + static_cast<long long>(N) * Ho * Wo;
}

extern "C" int semseg_upsample_ce_dice_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                           const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                           const float* lse, const float* table, const float* grad_out,
                                           float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_dice(zoom, Wo, 0.f, 0.f, 0.f);
  if (r) return r;
  SB_CHECK_ARG(lse && table && grad_out && workspace && dlogits, "upsample_ce_dice_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_dice_bwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, table, grad_out,
                                      workspace, dlogits, stream);
    case 2: return launch_dice_bwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, table, grad_out,
                                      workspace, dlogits, stream);
    case 4: return launch_dice_bwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, table, grad_out,
                                      workspace, dlogits, stream);
    default: return launch_dice_bwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, table, grad_out,
                                       workspace, dlogits, stream);
  }
}

// RMI loss (+ bce_weight * BCE + ce_weight * CE) at zoom factor `zoom`. The rows kernel stages 8-byte (lse, target)
// words of the interval's Z output rows in at most 224 KB of shared memory: Wo <= 3584 at zoom 8.
constexpr size_t kRmiSmemMax = 224 * 1024;

static int check_rmi(int Ho, int Wo, int zoom, float bce_weight, float pos_alpha, float ce_weight) {
  SB_CHECK_ARG(Ho >= 12 && Wo >= 12, "upsample_ce_rmi: target %dx%d is smaller than 12x12 (3x3 pooled cells)", Ho, Wo);
  SB_CHECK_ARG(bce_weight >= 0.f && bce_weight <= 1.f, "upsample_ce_rmi: bce_weight %g is not in [0, 1]", bce_weight);
  SB_CHECK_ARG(std::isfinite(pos_alpha) && pos_alpha > 0.f, "upsample_ce_rmi: pos_alpha %g is not finite and > 0",
               pos_alpha);
  SB_CHECK_ARG(std::isfinite(ce_weight) && ce_weight >= 0.f, "upsample_ce_rmi: ce_weight %g is not finite and >= 0",
               ce_weight);
  const size_t max_wo = kRmiSmemMax / (static_cast<size_t>(zoom) * sizeof(PixInfo));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_ce_rmi: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  SB_CHECK_ARG(cdiv((Ho / 4) * (Wo / 4), 256) <= 65535, "upsample_ce_rmi: target %dx%d has too many pooled cells", Ho,
               Wo);
  return SEMSEG_OK;
}

static int rmi_pool_ctas(int N, int Ho, int Wo, int zoom) {
  const int rows = zoom < 4 ? 4 : zoom, cols = zoom == 1 ? 32 : zoom == 2 ? 64 : 128;
  return cdiv(Wo, cols) * cdiv(Ho, rows) * N;
}

// Forward workspace (8-byte aligned): the raw moments fp64 [N*C][189], r fp64 [N*C], then the CE partials (2 per
// forward CTA) and the BCE partials (1 per pool CTA).
static long long rmi_ws_floats(int N, int Ho, int Wo, int C, int zoom) {
  const long long nc = static_cast<long long>(N) * C;
  return 2LL * nc * (kRmiMoments + 1) + 2LL * fwd_ctas(N, (Ho - 1) / zoom + 1, Wo) + rmi_pool_ctas(N, Ho, Wo, zoom);
}

template <int Z>
static int launch_rmi_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                          int Wo, int ignore_index, float bce_weight, float pos_alpha, float ce_weight,
                          float* workspace, float* loss_out, int64_t* argmax, float* lse, float* pooled, float* table,
                          cudaStream_t stream) {
  using B = RmiBand<Z>;
  const int NC = N * C, Hp = Ho / 4, Wp = Wo / 4;
  double* mom = reinterpret_cast<double*>(workspace);
  double* rterm = mom + static_cast<size_t>(NC) * kRmiMoments;
  float* ce_part = reinterpret_cast<float*>(rterm + NC);
  const int ctas = fwd_ctas(N, h, Wo);
  float* bce_part = ce_part + 2LL * ctas;
  int r = launch_fwd_kernel<Z, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, ce_part, argmax, lse,
                                      nullptr, nullptr, stream);
  if (r) return r;
  const int Cs = C | 1;
  const size_t smem = static_cast<size_t>(B::kNodeRows) * B::kNodes * Cs * sizeof(float);
  constexpr size_t kMaxSmem = static_cast<size_t>(B::kNodeRows) * B::kNodes * (kMaxClasses | 1) * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    r = opt_in_smem(rmi_pool_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  const dim3 pgrid(cdiv(Wo, B::kCols), cdiv(Ho, B::kRows), N);
  rmi_pool_kernel<Z><<<pgrid, B::kCols, smem, stream>>>(logits, pitch, N, h, w, C, Cs,
                                                        reinterpret_cast<const long long*>(target), Ho, Wo,
                                                        ignore_index, pooled, bce_part);
  SB_LAUNCHED();
  rmi_moments_kernel<<<dim3(NC, kRmiGroups), 256, 0, stream>>>(pooled, NC, Hp, Wp, mom);
  SB_LAUNCHED();
  rmi_algebra_kernel<<<cdiv(NC, 64), 64, 0, stream>>>(mom, NC, (Hp - 2) * (Wp - 2), pos_alpha, table, rterm);
  SB_LAUNCHED();
  rmi_loss_kernel<<<1, 256, 0, stream>>>(ce_part, ctas, bce_part, static_cast<int>(pgrid.x * pgrid.y * pgrid.z), rterm,
                                         NC, N, bce_weight, ce_weight, loss_out,
                                         table + static_cast<size_t>(NC) * kRmiRec);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Backward workspace: T2 [N][h][2][w][C] of the rows kernel, then dr/dQ [N][C][Hp][Wp].
template <int Z>
static int launch_rmi_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                          int Wo, int ignore_index, const float* lse, const float* pooled, const float* table,
                          const float* grad_out, float* workspace, float* dlogits, cudaStream_t stream) {
  const int NC = N * C, Hp = Ho / 4, Wp = Wo / 4;
  float* dq = workspace + 2LL * N * h * w * C;
  const float* sc = table + static_cast<size_t>(NC) * kRmiRec;
  rmi_dq_kernel<<<dim3(NC, cdiv(Hp * Wp, 256)), 256, 0, stream>>>(pooled, NC, Hp, Wp, table, dq);
  SB_LAUNCHED();
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(PixInfo);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_rmi_rows_kernel<Z>, attr_set, static_cast<int>(kRmiSmemMax));
    if (r) return r;
  }
  upsample_ce_rmi_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(
      logits, pitch, N, h, w, C, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lse, dq, sc,
      workspace);
  SB_LAUNCHED();
  // sc[1] = 1: the plain cols kernel's count, so dlogits = grad_out[0] * T2 sums
  upsample_ce_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, sc, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_rmi_workspace_floats(int N, int Ho, int Wo, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_rmi: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && C > 0, "upsample_ce_rmi: bad sizes");
  return rmi_ws_floats(N, Ho, Wo, C, zoom);
}

extern "C" long long semseg_upsample_ce_rmi_table_floats(int N, int C) {
  SB_CHECK_ARG(N > 0 && C > 0, "upsample_ce_rmi: bad sizes");
  return static_cast<long long>(N) * C * kRmiRec + 4;
}

extern "C" int semseg_upsample_ce_rmi_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                          const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                          float bce_weight, float pos_alpha, float ce_weight, float* workspace,
                                          float* loss_out, int64_t* argmax, float* lse, float* pooled, float* table,
                                          void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_rmi(Ho, Wo, zoom, bce_weight, pos_alpha, ce_weight);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && pooled && table, "upsample_ce_rmi_fwd: null output");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "upsample_ce_rmi_fwd: workspace not 8-byte aligned");
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(pooled) | reinterpret_cast<uintptr_t>(table)) & 3) == 0,
               "upsample_ce_rmi_fwd: pooled or table not 4-byte aligned");
  switch (zoom) {
    case 1: return launch_rmi_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, bce_weight, pos_alpha,
                                     ce_weight, workspace, loss_out, argmax, lse, pooled, table, stream);
    case 2: return launch_rmi_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, bce_weight, pos_alpha,
                                     ce_weight, workspace, loss_out, argmax, lse, pooled, table, stream);
    case 4: return launch_rmi_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, bce_weight, pos_alpha,
                                     ce_weight, workspace, loss_out, argmax, lse, pooled, table, stream);
    default: return launch_rmi_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, bce_weight, pos_alpha,
                                      ce_weight, workspace, loss_out, argmax, lse, pooled, table, stream);
  }
}

extern "C" long long semseg_upsample_ce_rmi_bwd_workspace_floats(int N, int Ho, int Wo, int w, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_rmi: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && w > 0 && C > 0, "upsample_ce_rmi: bad sizes");
  return 2LL * N * ((Ho - 1) / zoom + 1) * w * C + static_cast<long long>(N) * C * (Ho / 4) * (Wo / 4);
}

extern "C" int semseg_upsample_ce_rmi_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                          const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                          const float* lse, const float* pooled, const float* table,
                                          const float* grad_out, float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_rmi(Ho, Wo, zoom, 0.f, 1.f, 0.f);
  if (r) return r;
  SB_CHECK_ARG(lse && pooled && table && grad_out && workspace && dlogits, "upsample_ce_rmi_bwd: null pointer");
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(pooled) | reinterpret_cast<uintptr_t>(table)) & 3) == 0,
               "upsample_ce_rmi_bwd: pooled or table not 4-byte aligned");
  switch (zoom) {
    case 1: return launch_rmi_bwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, pooled, table,
                                     grad_out, workspace, dlogits, stream);
    case 2: return launch_rmi_bwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, pooled, table,
                                     grad_out, workspace, dlogits, stream);
    case 4: return launch_rmi_bwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, pooled, table,
                                     grad_out, workspace, dlogits, stream);
    default: return launch_rmi_bwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, pooled, table,
                                      grad_out, workspace, dlogits, stream);
  }
}

// Focal loss at zoom factor `zoom`: its own forward and rows kernels, the plain reduce and cols kernels. The rows kernel
// stages the Dice rows kernel's 12-byte words: the Dice width limit. class_weight NULL = all ones.
static int check_focal(int zoom, int Wo, float gamma, const void* class_weight, const void* mod) {
  SB_CHECK_ARG(std::isfinite(gamma) && gamma >= 0.f, "upsample_ce_focal: gamma %g is not finite and >= 0", gamma);
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(class_weight) | reinterpret_cast<uintptr_t>(mod)) & 3) == 0,
               "upsample_ce_focal: class_weight or modulator map not 4-byte aligned");
  const size_t max_wo = kDiceSmemMax / (static_cast<size_t>(zoom) * sizeof(DicePix));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_ce_focal: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

template <int Z>
static int launch_focal_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                            int Wo, int ignore_index, const float* class_weight, float gamma, float* workspace,
                            float* loss_out, int64_t* argmax, float* lse, float* mod, cudaStream_t stream) {
  const int Cs = C | 1;
  constexpr size_t kMaxSmem =
      static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_focal_fwd_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_ce_focal_fwd_kernel<Z><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, class_weight,
      gamma, workspace, reinterpret_cast<long long*>(argmax), lse, mod);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace, fwd_ctas(N, h, Wo), loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z>
static int launch_focal_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                            int Wo, int ignore_index, const float* lse, const float* mod, const float* loss_info,
                            const float* grad_out, float* workspace, float* dlogits, cudaStream_t stream) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(DicePix);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_focal_rows_kernel<Z>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  upsample_ce_focal_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(
      logits, pitch, N, h, w, C, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lse, mod, workspace);
  SB_LAUNCHED();
  // loss_info[1] = n_valid: the plain cols kernel's 1 / count
  upsample_ce_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, loss_info, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_focal_workspace_floats(int N, int Ho, int Wo, int zoom) {
  return semseg_upsample_ce_zoom_workspace_floats(N, Ho, Wo, zoom);
}

extern "C" int semseg_upsample_ce_focal_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                            const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                            const float* class_weight, float gamma, float* workspace,
                                            float* loss_out, int64_t* argmax, float* lse, float* mod, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_focal(zoom, Wo, gamma, class_weight, mod);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && mod, "upsample_ce_focal_fwd: null output");
  switch (zoom) {
    case 1: return launch_focal_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, class_weight, gamma,
                                       workspace, loss_out, argmax, lse, mod, stream);
    case 2: return launch_focal_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, class_weight, gamma,
                                       workspace, loss_out, argmax, lse, mod, stream);
    case 4: return launch_focal_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, class_weight, gamma,
                                       workspace, loss_out, argmax, lse, mod, stream);
    default: return launch_focal_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, class_weight, gamma,
                                        workspace, loss_out, argmax, lse, mod, stream);
  }
}

extern "C" long long semseg_upsample_ce_focal_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_ce_focal_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                            const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                            const float* lse, const float* mod, const float* loss_info,
                                            const float* grad_out, float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_focal(zoom, Wo, 0.f, nullptr, mod);
  if (r) return r;
  SB_CHECK_ARG(lse && mod && loss_info && grad_out && workspace && dlogits, "upsample_ce_focal_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_focal_bwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, mod, loss_info,
                                       grad_out, workspace, dlogits, stream);
    case 2: return launch_focal_bwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, mod, loss_info,
                                       grad_out, workspace, dlogits, stream);
    case 4: return launch_focal_bwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, mod, loss_info,
                                       grad_out, workspace, dlogits, stream);
    default: return launch_focal_bwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, mod, loss_info,
                                        grad_out, workspace, dlogits, stream);
  }
}

// SegPGD at zoom factor `zoom`: its own forward kernel, the plain reduce; the backward is semseg_upsample_ce_focal_bwd.
template <int Z>
static int launch_segpgd_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                             int Wo, int ignore_index, float lambda, float* workspace, float* loss_out, int64_t* argmax,
                             float* lse, float* mod, cudaStream_t stream) {
  const int Cs = C | 1;
  constexpr size_t kMaxSmem =
      static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_segpgd_fwd_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_segpgd_fwd_kernel<Z><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lambda,
      workspace, reinterpret_cast<long long*>(argmax), lse, mod);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace, fwd_ctas(N, h, Wo), loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_upsample_segpgd_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                          const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                          float lambda, float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                          float* mod, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  SB_CHECK_ARG(std::isfinite(lambda) && lambda >= 0.f && lambda <= 1.f,
               "upsample_segpgd_fwd: lambda %g is not in [0, 1]", lambda);
  // the focal backward's rows kernel stages this map: its width limit and alignment
  r = check_focal(zoom, Wo, 0.f, nullptr, mod);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && mod, "upsample_segpgd_fwd: null output");
  switch (zoom) {
    case 1: return launch_segpgd_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lambda, workspace,
                                        loss_out, argmax, lse, mod, stream);
    case 2: return launch_segpgd_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lambda, workspace,
                                        loss_out, argmax, lse, mod, stream);
    case 4: return launch_segpgd_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lambda, workspace,
                                        loss_out, argmax, lse, mod, stream);
    default: return launch_segpgd_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lambda, workspace,
                                         loss_out, argmax, lse, mod, stream);
  }
}

// Lovász-Softmax (+ ce_weight * CE) at zoom factor `zoom`. The rows kernel stages the Dice rows kernel's 12-byte words:
// the Dice width limit. Payloads hold the flat pixel index in 31 bits: N * Ho * Wo < 2^31.
static int check_lovasz(int N, int Ho, int Wo, int C, int zoom, int classes_all, int per_image, float ce_weight) {
  SB_CHECK_ARG(classes_all == 0 || classes_all == 1, "upsample_ce_lovasz: classes_all %d is not 0 or 1", classes_all);
  SB_CHECK_ARG(per_image == 0 || per_image == 1, "upsample_ce_lovasz: per_image %d is not 0 or 1", per_image);
  SB_CHECK_ARG(static_cast<long long>(N) * Ho * Wo < (1LL << 31), "upsample_ce_lovasz: %d x %d x %d pixels exceed 2^31",
               N, Ho, Wo);
  int r = check_dice(zoom, Wo, 0.f, 0.f, ce_weight);
  if (r) return r;
  const int S = per_image ? N * C : C;
  const long long L = per_image ? static_cast<long long>(Ho) * Wo : static_cast<long long>(N) * Ho * Wo;
  return semseg_segsort_u32_pairs_workspace_bytes(S, L) < 0 ? SEMSEG_E_INVALID : SEMSEG_OK;
}

// Forward workspace, in 4-byte words (8-byte aligned base): sorted keys [S][L] at 0, payloads [S][L] at S*L, the sort's
// second key / payload buffers, the sort workspace, the target histogram [N][C+1], skip[S], G[S], w[S] (fp64), the fg
// tile counts [S][nt], the fp64 tile partials [S][nt], then the CE partials (2 per forward CTA).
struct LovaszWs {
  int S, nt;
  long long L, sort, hist, skip, g, w, fgcnt, partial, ce, total;
  LovaszWs(int N, int Ho, int Wo, int C, int zoom, int per_image) {
    S = per_image ? N * C : C;
    L = per_image ? static_cast<long long>(Ho) * Wo : static_cast<long long>(N) * Ho * Wo;
    nt = static_cast<int>((L + kLovTile - 1) / kLovTile);
    const long long SL = static_cast<long long>(S) * L;
    auto even = [](long long v) { return (v + 1) & ~1LL; };
    sort = even(4 * SL);
    hist = sort + even(semseg_segsort_u32_pairs_workspace_bytes(S, L) / 4);
    skip = hist + static_cast<long long>(N) * (C + 1);
    g = skip + S;
    w = even(g + S);
    fgcnt = w + 2LL * S;
    partial = even(fgcnt + static_cast<long long>(S) * nt);
    ce = partial + 2LL * S * nt;
    total = ce + 2LL * fwd_ctas(N, (Ho - 1) / zoom + 1, Wo);
  }
};

template <int Z>
static int launch_lovasz_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                             int Wo, int ignore_index, int classes_all, int per_image, float ce_weight,
                             float* workspace, float* loss_out, int64_t* argmax, float* lse, float* gamma,
                             cudaStream_t stream) {
  const LovaszWs ws(N, Ho, Wo, C, Z, per_image);
  const long long SL = static_cast<long long>(ws.S) * ws.L;
  const long long P = static_cast<long long>(N) * Ho * Wo;
  unsigned* keys = reinterpret_cast<unsigned*>(workspace);
  unsigned* vals = keys + SL;
  int* hist = reinterpret_cast<int*>(workspace + ws.hist);
  int* skip = reinterpret_cast<int*>(workspace + ws.skip);
  int* seg_g = reinterpret_cast<int*>(workspace + ws.g);
  double* seg_w = reinterpret_cast<double*>(workspace + ws.w);
  unsigned* fgcnt = reinterpret_cast<unsigned*>(workspace + ws.fgcnt);
  double* partial = reinterpret_cast<double*>(workspace + ws.partial);
  float* ce = workspace + ws.ce;
  const long long* tgt = reinterpret_cast<const long long*>(target);
  int r = launch_fwd_kernel<Z, false>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, ce, argmax, lse,
                                      nullptr, nullptr, stream);
  if (r) return r;
  SB_CUDA(cudaMemsetAsync(hist, 0, sizeof(int) * N * (C + 1), stream));
  lovasz_target_hist_kernel<<<dim3(cdiv(Ho * Wo, kLovTile), N), 256, 0, stream>>>(tgt, Ho * Wo, C, ignore_index, hist);
  SB_LAUNCHED();
  lovasz_segments_kernel<<<1, kMaxClasses, 0, stream>>>(hist, N, C, classes_all, per_image, skip, seg_g, seg_w);
  SB_LAUNCHED();
  SB_CUDA(cudaMemsetAsync(gamma, 0, sizeof(float) * P * C, stream));
  const int Cs = C | 1;
  const size_t smem = (static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs + C) * sizeof(float);
  constexpr size_t kMaxSmem =
      (static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) + kMaxClasses) * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    r = opt_in_smem(lovasz_key_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  lovasz_key_kernel<Z><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, tgt, Ho, Wo, ignore_index, lse, per_image, skip, keys, vals);
  SB_LAUNCHED();
  r = semseg_segsort_u32_pairs(keys, vals, keys + 2 * SL, keys + 3 * SL, ws.S, ws.L, skip, workspace + ws.sort,
                               stream);
  if (r) return r;
  const int ctas = ws.S * ws.nt;
  const int Li = static_cast<int>(ws.L);
  lovasz_fgcount_kernel<<<ctas, kLovThreads, 0, stream>>>(vals, Li, ws.nt, skip, fgcnt);
  SB_LAUNCHED();
  lovasz_fgscan_kernel<<<ws.S, kLovThreads, 0, stream>>>(fgcnt, ws.nt, skip);
  SB_LAUNCHED();
  lovasz_grad_kernel<<<ctas, kLovThreads, 0, stream>>>(keys, vals, Li, ws.nt, C, per_image, skip, seg_g, seg_w, fgcnt,
                                                       gamma, partial);
  SB_LAUNCHED();
  lovasz_loss_kernel<<<1, 256, 0, stream>>>(ce, fwd_ctas(N, h, Wo), partial, ws.S, ws.nt, skip, seg_w, ce_weight,
                                            loss_out, gamma + P * C);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Backward workspace: T2 [N][h][2][w][C] of the rows kernel, then the Gamma map [N][Ho][Wo] (the Dice backward's).
template <int Z>
static int launch_lovasz_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                             int Wo, int ignore_index, const float* lse, const float* gamma, const float* grad_out,
                             float* workspace, float* dlogits, cudaStream_t stream) {
  float* gmap = workspace + 2LL * N * h * w * C;
  const long long P = static_cast<long long>(N) * Ho * Wo;
  const long long* tgt = reinterpret_cast<const long long*>(target);
  lovasz_gamma_sum_kernel<Z><<<static_cast<unsigned>((P + 7) / 8), 256, 0, stream>>>(
      logits, pitch, N, h, w, C, tgt, Ho, Wo, ignore_index, lse, gamma, gmap);
  SB_LAUNCHED();
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(DicePix);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(lovasz_rows_kernel<Z>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  lovasz_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(logits, pitch, N, h, w, C, tgt, Ho, Wo, ignore_index,
                                                               lse, gmap, gamma, workspace);
  SB_LAUNCHED();
  // gamma[P*C + 1] = 1: the plain cols kernel's count, so dlogits = grad_out[0] * T2 sums
  upsample_ce_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, gamma + P * C, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_lovasz_workspace_floats(int N, int Ho, int Wo, int C, int zoom,
                                                                int per_image) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_lovasz: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && C > 0 && C <= kMaxClasses, "upsample_ce_lovasz: bad sizes");
  int r = check_lovasz(N, Ho, Wo, C, zoom, 0, per_image, 0.f);
  if (r) return r;
  return LovaszWs(N, Ho, Wo, C, zoom, per_image).total;
}

extern "C" int semseg_upsample_ce_lovasz_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                             const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                             int classes_all, int per_image, float ce_weight, float* workspace,
                                             float* loss_out, int64_t* argmax, float* lse, float* gamma,
                                             void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_lovasz(N, Ho, Wo, C, zoom, classes_all, per_image, ce_weight);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && gamma, "upsample_ce_lovasz_fwd: null output");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0,
               "upsample_ce_lovasz_fwd: workspace not 8-byte aligned");
  switch (zoom) {
    case 1: return launch_lovasz_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, classes_all,
                                        per_image, ce_weight, workspace, loss_out, argmax, lse, gamma, stream);
    case 2: return launch_lovasz_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, classes_all,
                                        per_image, ce_weight, workspace, loss_out, argmax, lse, gamma, stream);
    case 4: return launch_lovasz_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, classes_all,
                                        per_image, ce_weight, workspace, loss_out, argmax, lse, gamma, stream);
    default: return launch_lovasz_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, classes_all,
                                         per_image, ce_weight, workspace, loss_out, argmax, lse, gamma, stream);
  }
}

extern "C" long long semseg_upsample_ce_lovasz_bwd_workspace_floats(int N, int Ho, int Wo, int w, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_lovasz: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && w > 0 && C > 0, "upsample_ce_lovasz: bad sizes");
  return 2LL * N * ((Ho - 1) / zoom + 1) * w * C + static_cast<long long>(N) * Ho * Wo;
}

extern "C" int semseg_upsample_ce_lovasz_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                             const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                             const float* lse, const float* gamma, const float* grad_out,
                                             float* workspace, float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_lovasz(N, Ho, Wo, C, zoom, 0, 0, 0.f);
  if (r) return r;
  SB_CHECK_ARG(lse && gamma && grad_out && workspace && dlogits, "upsample_ce_lovasz_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_lovasz_bwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, gamma, grad_out,
                                        workspace, dlogits, stream);
    case 2: return launch_lovasz_bwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, gamma, grad_out,
                                        workspace, dlogits, stream);
    case 4: return launch_lovasz_bwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, gamma, grad_out,
                                        workspace, dlogits, stream);
    default: return launch_lovasz_bwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, lse, gamma,
                                         grad_out, workspace, dlogits, stream);
  }
}

// Knowledge distillation at zoom factor `zoom` (student and teacher maps upsampled alike). The backward stages one
// 8-byte word per pixel of the interval's Z output rows, as the plain backward does: Wo <= 2560 at zoom 8.
static int check_kd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w, int C,
                    int Ho, int Wo, int zoom, float temperature) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_kd: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(student && teacher, "upsample_kd: null pointer");
  SB_CHECK_ARG(N > 0 && h > 1 && w > 1 && C > 1 && C <= kMaxClasses, "upsample_kd: bad sizes (C<=%d)", kMaxClasses);
  SB_CHECK_ARG(pitch_s >= C && pitch_t >= C, "upsample_kd: pitch %d / %d below C = %d", pitch_s, pitch_t, C);
  SB_CHECK_ARG(Ho == zoom * (h - 1) + 1 && Wo == zoom * (w - 1) + 1,
               "upsample_kd: needs Ho=%d(h-1)+1, Wo=%d(w-1)+1 (got %dx%d -> %dx%d)", zoom, zoom, h, w, Ho, Wo);
  SB_CHECK_ARG(std::isfinite(temperature) && temperature > 0.f, "upsample_kd: temperature %g is not finite and > 0",
               temperature);
  const size_t max_wo = kBwdSmemMax / (static_cast<size_t>(zoom) * sizeof(float2));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_kd: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

template <int Z>
static int kd_fwd_ctas(int N, int h, int Wo) { return cdiv(Wo, KdGeom<Z>::kCols) * h * N; }

static long long kd_fwd_partials(int N, int h, int Wo, int zoom) {
  const int cols = zoom <= 2 ? KdGeom<1>::kCols : KdGeom<8>::kCols;
  return 2LL * N * h * cdiv(Wo, cols);
}

template <int Z>
static int launch_kd_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                         int C, int Ho, int Wo, float temperature, float* workspace, float* kl_out, float* lse,
                         cudaStream_t stream) {
  using K = KdGeom<Z>;
  const int Cs = C | 1;
  // two maps of 256 classes: 133 KB at Z = 1 (65 node columns), 136 KB at Z = 2 and 4 (2 x 33), 70 KB at Z = 8
  constexpr size_t kMaxSmem = 2ull * Zoom<Z>::kNodeRows * K::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = 2ull * Zoom<Z>::kNodeRows * K::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_kd_fwd_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_kd_fwd_kernel<Z><<<dim3(cdiv(Wo, K::kCols), h, N), K::kCols, smem, stream>>>(
      student, pitch_s, teacher, pitch_t, N, h, w, C, Cs, Ho, Wo, 1.f / temperature, workspace,
      reinterpret_cast<float2*>(lse));
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace, kd_fwd_ctas<Z>(N, h, Wo), kl_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z>
static int launch_kd_bwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                         int C, int Ho, int Wo, float temperature, float kd_weight, const float* lse,
                         const float* grad_out, float* workspace, float* dlogits, cudaStream_t stream) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(float2);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_kd_bwd_rows_kernel<Z>, attr_set, static_cast<int>(kBwdSmemMax));
    if (r) return r;
  }
  upsample_kd_bwd_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(
      student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, 1.f / temperature, reinterpret_cast<const float2*>(lse),
      workspace);
  SB_LAUNCHED();
  // d(kd_weight T^2 KL)/ds_c = kd_weight T (p_c - q_c) / P
  const double P = static_cast<double>(N) * Ho * Wo;
  const float scale = static_cast<float>(static_cast<double>(kd_weight) * temperature / P);
  upsample_kd_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, scale, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_kd_workspace_floats(int N, int Ho, int Wo, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_kd: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0, "upsample_kd: bad sizes");
  return kd_fwd_partials(N, (Ho - 1) / zoom + 1, Wo, zoom);   // (sum KL, pixels) per forward CTA
}

extern "C" int semseg_upsample_kd_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N,
                                      int h, int w, int C, int Ho, int Wo, int zoom, float temperature,
                                      float* workspace, float* kl_out, float* lse, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_kd(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, zoom, temperature);
  if (r) return r;
  SB_CHECK_ARG(workspace && kl_out && lse, "upsample_kd_fwd: null output");
  switch (zoom) {
    case 1: return launch_kd_fwd<1>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, workspace,
                                    kl_out, lse, stream);
    case 2: return launch_kd_fwd<2>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, workspace,
                                    kl_out, lse, stream);
    case 4: return launch_kd_fwd<4>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, workspace,
                                    kl_out, lse, stream);
    default: return launch_kd_fwd<8>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, workspace,
                                     kl_out, lse, stream);
  }
}

extern "C" long long semseg_upsample_kd_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_kd: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && w > 0 && C > 0, "upsample_kd: bad sizes");
  return 2LL * N * ((Ho - 1) / zoom + 1) * w * C;  // T2[N][h][2][w][C]
}

extern "C" int semseg_upsample_kd_bwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N,
                                      int h, int w, int C, int Ho, int Wo, int zoom, float temperature,
                                      float kd_weight, const float* lse, const float* grad_out, float* workspace,
                                      float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_kd(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, zoom, temperature);
  if (r) return r;
  SB_CHECK_ARG(std::isfinite(kd_weight) && kd_weight >= 0.f, "upsample_kd_bwd: kd_weight %g is not finite and >= 0",
               kd_weight);
  SB_CHECK_ARG(lse && grad_out && workspace && dlogits, "upsample_kd_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_kd_bwd<1>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, kd_weight,
                                    lse, grad_out, workspace, dlogits, stream);
    case 2: return launch_kd_bwd<2>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, kd_weight,
                                    lse, grad_out, workspace, dlogits, stream);
    case 4: return launch_kd_bwd<4>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, kd_weight,
                                    lse, grad_out, workspace, dlogits, stream);
    default: return launch_kd_bwd<8>(student, pitch_s, teacher, pitch_t, N, h, w, C, Ho, Wo, temperature, kd_weight,
                                     lse, grad_out, workspace, dlogits, stream);
  }
}

// Class-incremental (MiB) losses at zoom factor `zoom`. Both backward rows kernels stage 12 bytes per pixel of the
// interval's Z output rows in kDiceSmemMax: the Dice width limit, Wo <= 2389 at zoom 8.
static int check_incremental(int C, int c_old, int zoom, int Wo) {
  SB_CHECK_ARG(c_old >= 2 && c_old < C, "upsample_incremental: C_old = %d must lie in [2, C = %d)", c_old, C);
  const size_t max_wo = kDiceSmemMax / (static_cast<size_t>(zoom) * 12);
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_incremental: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

template <int Z>
static int launch_unbiased_fwd(const float* logits, int pitch, int N, int h, int w, int C, int c_old,
                               const int64_t* target, int Ho, int Wo, int ignore_index, float* workspace,
                               float* loss_out, int64_t* argmax, float* lse, float* lse_old, cudaStream_t stream) {
  const int Cs = C | 1;
  constexpr size_t kMaxSmem = static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_fwd_kernel<Z, false, false, true>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_ce_fwd_kernel<Z, false, false, true><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, workspace,
      reinterpret_cast<long long*>(argmax), lse, nullptr, nullptr, nullptr, 0.f, c_old, lse_old);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace, fwd_ctas(N, h, Wo), loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z>
static int launch_unbiased_bwd(const float* logits, int pitch, int N, int h, int w, int C, int c_old,
                               const int64_t* target, int Ho, int Wo, int ignore_index, const float* lse,
                               const float* lse_old, const float* loss_info, const float* grad_out, float* workspace,
                               float* dlogits, cudaStream_t stream) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * (sizeof(PixInfo) + sizeof(float));
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_bwd_rows_kernel<Z, false, false, true>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  upsample_ce_bwd_rows_kernel<Z, false, false, true><<<dim3(h, N), threads, smem, stream>>>(
      logits, pitch, N, h, w, C, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, lse, workspace,
      nullptr, nullptr, nullptr, 0.f, c_old, lse_old);
  SB_LAUNCHED();
  upsample_ce_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, loss_info, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_unbiased_workspace_floats(int N, int Ho, int Wo, int zoom) {
  return semseg_upsample_ce_zoom_workspace_floats(N, Ho, Wo, zoom);
}

extern "C" int semseg_upsample_ce_unbiased_fwd(const float* logits, int pitch, int N, int h, int w, int C, int c_old,
                                               const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                               float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                               float* lse_old, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_incremental(C, c_old, zoom, Wo);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && lse_old, "upsample_ce_unbiased_fwd: null output");
  switch (zoom) {
    case 1: return launch_unbiased_fwd<1>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, workspace,
                                          loss_out, argmax, lse, lse_old, stream);
    case 2: return launch_unbiased_fwd<2>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, workspace,
                                          loss_out, argmax, lse, lse_old, stream);
    case 4: return launch_unbiased_fwd<4>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, workspace,
                                          loss_out, argmax, lse, lse_old, stream);
    default: return launch_unbiased_fwd<8>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, workspace,
                                           loss_out, argmax, lse, lse_old, stream);
  }
}

extern "C" long long semseg_upsample_ce_unbiased_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_ce_unbiased_bwd(const float* logits, int pitch, int N, int h, int w, int C, int c_old,
                                               const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                               const float* lse, const float* lse_old, const float* loss_info,
                                               const float* grad_out, float* workspace, float* dlogits,
                                               void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_incremental(C, c_old, zoom, Wo);
  if (r) return r;
  SB_CHECK_ARG(lse && lse_old && loss_info && grad_out && dlogits && workspace, "upsample_ce_unbiased_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_unbiased_bwd<1>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, lse, lse_old,
                                          loss_info, grad_out, workspace, dlogits, stream);
    case 2: return launch_unbiased_bwd<2>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, lse, lse_old,
                                          loss_info, grad_out, workspace, dlogits, stream);
    case 4: return launch_unbiased_bwd<4>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, lse, lse_old,
                                          loss_info, grad_out, workspace, dlogits, stream);
    default: return launch_unbiased_bwd<8>(logits, pitch, N, h, w, C, c_old, target, Ho, Wo, ignore_index, lse,
                                           lse_old, loss_info, grad_out, workspace, dlogits, stream);
  }
}

static int check_unkd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w, int C,
                      int c_old, int Ho, int Wo, int zoom, float alpha) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_unkd: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(student && teacher, "upsample_unkd: null pointer");
  SB_CHECK_ARG(N > 0 && h > 1 && w > 1 && C > 1 && C <= kMaxClasses, "upsample_unkd: bad sizes (C<=%d)", kMaxClasses);
  SB_CHECK_ARG(pitch_s >= C && pitch_t >= c_old, "upsample_unkd: pitch %d / %d below C = %d / C_old = %d", pitch_s,
               pitch_t, C, c_old);
  SB_CHECK_ARG(Ho == zoom * (h - 1) + 1 && Wo == zoom * (w - 1) + 1,
               "upsample_unkd: needs Ho=%d(h-1)+1, Wo=%d(w-1)+1 (got %dx%d -> %dx%d)", zoom, zoom, h, w, Ho, Wo);
  SB_CHECK_ARG(std::isfinite(alpha) && alpha > 0.f, "upsample_unkd: alpha %g is not finite and > 0", alpha);
  return check_incremental(C, c_old, zoom, Wo);
}

template <int Z>
static int launch_unkd_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                           int C, int c_old, int Ho, int Wo, float alpha, float* workspace, float* loss_out,
                           float* lse, cudaStream_t stream) {
  using K = KdGeom<Z>;
  const int Cs = C | 1;
  // the distillation forward's shared memory: two maps at the student's stride
  constexpr size_t kMaxSmem = 2ull * Zoom<Z>::kNodeRows * K::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = 2ull * Zoom<Z>::kNodeRows * K::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_unkd_fwd_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_unkd_fwd_kernel<Z><<<dim3(cdiv(Wo, K::kCols), h, N), K::kCols, smem, stream>>>(
      student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Cs, Ho, Wo, alpha, workspace, lse);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace, kd_fwd_ctas<Z>(N, h, Wo), loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z>
static int launch_unkd_bwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                           int C, int c_old, int Ho, int Wo, float alpha, float kd_weight, const float* lse,
                           const float* grad_out, float* workspace, float* dlogits, cudaStream_t stream) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(UnkdPix);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_unkd_bwd_rows_kernel<Z>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  upsample_unkd_bwd_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(student, pitch_s, teacher, pitch_t, N, h, w,
                                                                          C, c_old, Ho, Wo, alpha, lse, workspace);
  SB_LAUNCHED();
  // d(kd_weight KD)/ds_c = kd_weight (C_old dk/ds_c) / (C_old P)
  const double P = static_cast<double>(N) * Ho * Wo;
  const float scale = static_cast<float>(static_cast<double>(kd_weight) / (static_cast<double>(c_old) * P));
  upsample_kd_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, scale, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_unkd_workspace_floats(int N, int Ho, int Wo, int zoom) {
  return semseg_upsample_kd_workspace_floats(N, Ho, Wo, zoom);
}

extern "C" int semseg_upsample_unkd_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N,
                                        int h, int w, int C, int c_old, int Ho, int Wo, int zoom, float alpha,
                                        float* workspace, float* loss_out, float* lse, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_unkd(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, zoom, alpha);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse, "upsample_unkd_fwd: null output");
  switch (zoom) {
    case 1: return launch_unkd_fwd<1>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, workspace,
                                      loss_out, lse, stream);
    case 2: return launch_unkd_fwd<2>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, workspace,
                                      loss_out, lse, stream);
    case 4: return launch_unkd_fwd<4>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, workspace,
                                      loss_out, lse, stream);
    default: return launch_unkd_fwd<8>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, workspace,
                                       loss_out, lse, stream);
  }
}

extern "C" long long semseg_upsample_unkd_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  return semseg_upsample_kd_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_unkd_bwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N,
                                        int h, int w, int C, int c_old, int Ho, int Wo, int zoom, float alpha,
                                        float kd_weight, const float* lse, const float* grad_out, float* workspace,
                                        float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_unkd(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, zoom, alpha);
  if (r) return r;
  SB_CHECK_ARG(std::isfinite(kd_weight) && kd_weight >= 0.f, "upsample_unkd_bwd: kd_weight %g is not finite and >= 0",
               kd_weight);
  SB_CHECK_ARG(lse && grad_out && workspace && dlogits, "upsample_unkd_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_unkd_bwd<1>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, kd_weight,
                                      lse, grad_out, workspace, dlogits, stream);
    case 2: return launch_unkd_bwd<2>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, kd_weight,
                                      lse, grad_out, workspace, dlogits, stream);
    case 4: return launch_unkd_bwd<4>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha, kd_weight,
                                      lse, grad_out, workspace, dlogits, stream);
    default: return launch_unkd_bwd<8>(student, pitch_s, teacher, pitch_t, N, h, w, C, c_old, Ho, Wo, alpha,
                                       kd_weight, lse, grad_out, workspace, dlogits, stream);
  }
}

// Pseudo-label cross-entropy at zoom factor `zoom`: the count pass, the two-map forward and the plain reduce; the
// backward is semseg_upsample_ce_focal_bwd on the effective targets and weights, so Wo has the Dice limit.
// Workspace: the two uint64 counts (4 floats), then 2 x (value, count) partials per forward CTA.
static int check_pl(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w, int C,
                    const void* target, int Ho, int Wo, int zoom, float threshold, float pl_weight, float ce_weight) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_pl: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(student && teacher && target, "upsample_pl: null pointer");
  SB_CHECK_ARG(N > 0 && h > 1 && w > 1 && C > 1 && C <= kMaxClasses, "upsample_pl: bad sizes (C<=%d)", kMaxClasses);
  SB_CHECK_ARG(pitch_s >= C && pitch_t >= C, "upsample_pl: pitch %d / %d below C = %d", pitch_s, pitch_t, C);
  SB_CHECK_ARG(Ho == zoom * (h - 1) + 1 && Wo == zoom * (w - 1) + 1,
               "upsample_pl: needs Ho=%d(h-1)+1, Wo=%d(w-1)+1 (got %dx%d -> %dx%d)", zoom, zoom, h, w, Ho, Wo);
  SB_CHECK_ARG(std::isfinite(threshold), "upsample_pl: threshold %g is not finite", threshold);
  SB_CHECK_ARG(std::isfinite(pl_weight) && pl_weight >= 0.f, "upsample_pl: pl_weight %g is not finite and >= 0",
               pl_weight);
  SB_CHECK_ARG(std::isfinite(ce_weight) && ce_weight >= 0.f, "upsample_pl: ce_weight %g is not finite and >= 0",
               ce_weight);
  const size_t max_wo = kDiceSmemMax / (static_cast<size_t>(zoom) * sizeof(DicePix));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_pl: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

template <int Z, bool kMix = false>
static int launch_pl_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N, int h, int w,
                         int C, const int64_t* target, int Ho, int Wo, int ignore_index, float threshold,
                         float pl_weight, float ce_weight, float* workspace, float* loss_out, int64_t* argmax,
                         float* lse, int64_t* eff, float* wt, cudaStream_t stream,
                         const uint8_t* mix_mask = nullptr) {
  using K = KdGeom<Z>;
  unsigned long long* counts = reinterpret_cast<unsigned long long*>(workspace);
  float* partial = workspace + 4;
  const int ctas = kd_fwd_ctas<Z>(N, h, Wo);
  const long long M = static_cast<long long>(N) * Ho * Wo;
  SB_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(unsigned long long), stream));
  const int count_ctas = static_cast<int>(std::min<long long>((M + 255) / 256, 4LL * num_sms()));
  upsample_pl_count_kernel<<<count_ctas, 256, 0, stream>>>(reinterpret_cast<const long long*>(target), M, C,
                                                           ignore_index, counts, loss_out);
  SB_LAUNCHED();
  const int Cs = C | 1;
  constexpr unsigned long long kMaps = kMix ? 3 : 2;    // kMix: the partner's teacher rows as a third map
  constexpr size_t kMaxSmem = kMaps * Zoom<Z>::kNodeRows * K::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = kMaps * Zoom<Z>::kNodeRows * K::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_pl_fwd_kernel<Z, kMix>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_pl_fwd_kernel<Z, kMix><<<dim3(cdiv(Wo, K::kCols), h, N), K::kCols, smem, stream>>>(
      student, pitch_s, teacher, pitch_t, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo,
      ignore_index, threshold, pl_weight, ce_weight, counts, partial, reinterpret_cast<long long*>(argmax), lse,
      reinterpret_cast<long long*>(eff), wt, mix_mask);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(partial, ctas, loss_out);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(partial + 2LL * ctas, ctas, loss_out + 2);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_pl_workspace_floats(int N, int Ho, int Wo, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_pl: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0, "upsample_pl: bad sizes");
  return 4 + 2 * kd_fwd_partials(N, (Ho - 1) / zoom + 1, Wo, zoom);
}

extern "C" int semseg_upsample_pl_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N,
                                      int h, int w, int C, const int64_t* target, int Ho, int Wo, int zoom,
                                      int ignore_index, float threshold, float pl_weight, float ce_weight,
                                      float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                      int64_t* eff_target, float* weight, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_pl(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, zoom, threshold, pl_weight,
                   ce_weight);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && eff_target && weight, "upsample_pl_fwd: null output");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "upsample_pl_fwd: workspace not 8-byte aligned");
  switch (zoom) {
    case 1: return launch_pl_fwd<1>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                    threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                    weight, stream);
    case 2: return launch_pl_fwd<2>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                    threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                    weight, stream);
    case 4: return launch_pl_fwd<4>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                    threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                    weight, stream);
    default: return launch_pl_fwd<8>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                     threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                     weight, stream);
  }
}

// The mixed form (CutMix / ClassMix): semseg_upsample_pl_fwd with each output pixel's teacher taken from image n or its
// partner (n + 1) mod N by the input-grid mix mask; the same workspace.
extern "C" int semseg_upsample_pl_mix_fwd(const float* student, int pitch_s, const float* teacher, int pitch_t, int N,
                                          int h, int w, int C, const int64_t* target, int Ho, int Wo, int zoom,
                                          int ignore_index, float threshold, float pl_weight, float ce_weight,
                                          const uint8_t* mix_mask, float* workspace, float* loss_out, int64_t* argmax,
                                          float* lse, int64_t* eff_target, float* weight, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_pl(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, zoom, threshold, pl_weight,
                   ce_weight);
  if (r) return r;
  SB_CHECK_ARG(mix_mask, "upsample_pl_mix_fwd: null mix mask");
  SB_CHECK_ARG(workspace && loss_out && lse && eff_target && weight, "upsample_pl_mix_fwd: null output");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "upsample_pl_mix_fwd: workspace not 8-byte aligned");
  switch (zoom) {
    case 1: return launch_pl_fwd<1, true>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                          threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                          weight, stream, mix_mask);
    case 2: return launch_pl_fwd<2, true>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                          threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                          weight, stream, mix_mask);
    case 4: return launch_pl_fwd<4, true>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo, ignore_index,
                                          threshold, pl_weight, ce_weight, workspace, loss_out, argmax, lse, eff_target,
                                          weight, stream, mix_mask);
    default: return launch_pl_fwd<8, true>(student, pitch_s, teacher, pitch_t, N, h, w, C, target, Ho, Wo,
                                           ignore_index, threshold, pl_weight, ce_weight, workspace, loss_out, argmax,
                                           lse, eff_target, weight, stream, mix_mask);
  }
}

// Entropy (+ CE) at zoom factor `zoom`: its own forward and rows kernels, the plain reduce (twice) and cols kernels. The
// rows kernel stages the Dice rows kernel's 12-byte words: the Dice width limit, checked by both directions.
// Forward workspace: 2 x (value, count) partials per forward CTA.
static int check_entropy(int zoom, int Wo, const void* lse, const void* mu) {
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(lse) | reinterpret_cast<uintptr_t>(mu)) & 3) == 0,
               "upsample_ce_entropy: lse or mu map not 4-byte aligned");
  const size_t max_wo = kDiceSmemMax / (static_cast<size_t>(zoom) * sizeof(DicePix));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_ce_entropy: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

template <int Z>
static int launch_entropy_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                              int Ho, int Wo, int ignore_index, float* workspace, float* loss_out, int64_t* argmax,
                              float* lse, float* mu, cudaStream_t stream) {
  const int Cs = C | 1;
  const int ctas = fwd_ctas(N, h, Wo);
  constexpr size_t kMaxSmem =
      static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_entropy_fwd_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_ce_entropy_fwd_kernel<Z><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, workspace,
      loss_out, reinterpret_cast<long long*>(argmax), lse, mu);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace, ctas, loss_out);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<<<1, 256, 0, stream>>>(workspace + 2LL * ctas, ctas, loss_out + 2);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z>
static int launch_entropy_bwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target,
                              int Ho, int Wo, int ignore_index, float ent_weight, float ce_weight, const float* lse,
                              const float* mu, const float* loss_info, const float* grad_out, float* workspace,
                              float* dlogits, cudaStream_t stream) {
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(DicePix);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_ce_entropy_rows_kernel<Z>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  upsample_ce_entropy_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(
      logits, pitch, N, h, w, C, reinterpret_cast<const long long*>(target), Ho, Wo, ignore_index, ent_weight,
      ce_weight, lse, mu, loss_info, workspace);
  SB_LAUNCHED();
  // loss_info[5] = 1: the per-pixel weights are in T2 already
  upsample_ce_bwd_cols_kernel<<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, loss_info + 4, grad_out, dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_entropy_workspace_floats(int N, int Ho, int Wo, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_entropy: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0, "upsample_ce_entropy: bad sizes");
  return 2 * semseg_upsample_ce_zoom_workspace_floats(N, Ho, Wo, zoom);
}

extern "C" int semseg_upsample_ce_entropy_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                              const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                              float* workspace, float* loss_out, int64_t* argmax, float* lse,
                                              float* mu, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_entropy(zoom, Wo, lse, mu);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && mu, "upsample_ce_entropy_fwd: null output");
  switch (zoom) {
    case 1: return launch_entropy_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                         argmax, lse, mu, stream);
    case 2: return launch_entropy_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                         argmax, lse, mu, stream);
    case 4: return launch_entropy_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace, loss_out,
                                         argmax, lse, mu, stream);
    default: return launch_entropy_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, workspace,
                                          loss_out, argmax, lse, mu, stream);
  }
}

extern "C" long long semseg_upsample_ce_entropy_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  SB_CHECK_ARG(valid_zoom(zoom), "upsample_ce_entropy: zoom %d is not one of 1, 2, 4, 8", zoom);
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_ce_entropy_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                              const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                              float ent_weight, float ce_weight, const float* lse, const float* mu,
                                              const float* loss_info, const float* grad_out, float* workspace,
                                              float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_entropy(zoom, Wo, lse, mu);
  if (r) return r;
  SB_CHECK_ARG(std::isfinite(ent_weight) && ent_weight >= 0.f,
               "upsample_ce_entropy: ent_weight %g is not finite and >= 0", ent_weight);
  SB_CHECK_ARG(std::isfinite(ce_weight) && ce_weight >= 0.f,
               "upsample_ce_entropy: ce_weight %g is not finite and >= 0", ce_weight);
  SB_CHECK_ARG(lse && mu && loss_info && grad_out && workspace && dlogits, "upsample_ce_entropy_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_entropy_bwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, ent_weight,
                                         ce_weight, lse, mu, loss_info, grad_out, workspace, dlogits, stream);
    case 2: return launch_entropy_bwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, ent_weight,
                                         ce_weight, lse, mu, loss_info, grad_out, workspace, dlogits, stream);
    case 4: return launch_entropy_bwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, ent_weight,
                                         ce_weight, lse, mu, loss_info, grad_out, workspace, dlogits, stream);
    default: return launch_entropy_bwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, ent_weight,
                                          ce_weight, lse, mu, loss_info, grad_out, workspace, dlogits, stream);
  }
}

// Boundary label relaxation at zoom factor `zoom`: the sets pass, its own forward and rows kernels, the weighted-mean
// reduce and cols kernels. The rows kernel stages 12 bytes per pixel: the Dice width limit, Wo <= 2389 at zoom 8.
// The per-pixel record `sets` (int32 words, M = N*Ho*Wo): tag[M], omega[M] (fp32), then ceil(C/32) mask words per pixel.
static int check_relax(int zoom, int Wo, int border, const void* class_weight, const void* sets, const void* lq) {
  SB_CHECK_ARG(border >= 0 && border <= kRelaxMaxBorder, "upsample_ce_relax: border %d is not in [0, %d]", border,
               kRelaxMaxBorder);
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(class_weight) | reinterpret_cast<uintptr_t>(sets) |
                 reinterpret_cast<uintptr_t>(lq)) & 3) == 0,
               "upsample_ce_relax: class_weight, sets or lq not 4-byte aligned");
  const size_t max_wo = kDiceSmemMax / (static_cast<size_t>(zoom) * sizeof(RelaxPix));
  SB_CHECK_ARG(static_cast<size_t>(Wo) <= max_wo,
               "upsample_ce_relax: output width %d too large for the staged rows (at most %d at zoom %d)", Wo,
               static_cast<int>(max_wo), zoom);
  return SEMSEG_OK;
}

struct RelaxSets {
  int* tag;
  float* omega;
  unsigned* mask;
};

static RelaxSets relax_sets(int32_t* sets, int N, int Ho, int Wo) {
  const size_t M = static_cast<size_t>(N) * Ho * Wo;
  return {reinterpret_cast<int*>(sets), reinterpret_cast<float*>(sets + M), reinterpret_cast<unsigned*>(sets + 2 * M)};
}

template <int Z>
static int launch_relax_fwd(const float* logits, int pitch, int N, int h, int w, int C, const int64_t* target, int Ho,
                            int Wo, int ignore_index, int border, const float* class_weight, float* workspace,
                            float* loss_out, int64_t* argmax, float* lse, int32_t* sets, float* lq,
                            cudaStream_t stream) {
  const RelaxSets rs = relax_sets(sets, N, Ho, Wo);
  const long long M = static_cast<long long>(N) * Ho * Wo;
  upsample_relax_sets_kernel<<<static_cast<unsigned>((M + kRelaxThreads - 1) / kRelaxThreads), kRelaxThreads, 0,
                               stream>>>(reinterpret_cast<const long long*>(target), N, Ho, Wo, C, ignore_index, border,
                                         class_weight, rs.tag, rs.omega, rs.mask);
  SB_LAUNCHED();
  const int Cs = C | 1;
  constexpr size_t kMaxSmem =
      static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * (kMaxClasses | 1) * sizeof(float);
  const size_t smem = static_cast<size_t>(Zoom<Z>::kNodeRows) * Zoom<Z>::kNodes * Cs * sizeof(float);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_relax_fwd_kernel<Z>, attr_set, static_cast<int>(kMaxSmem));
    if (r) return r;
  }
  upsample_relax_fwd_kernel<Z><<<dim3(cdiv(Wo, kFwdCols), h, N), kFwdCols, smem, stream>>>(
      logits, pitch, N, h, w, C, Cs, Ho, Wo, rs.tag, rs.omega, rs.mask, workspace, reinterpret_cast<long long*>(argmax),
      lse, lq);
  SB_LAUNCHED();
  upsample_ce_reduce_kernel<true><<<1, 256, 0, stream>>>(workspace, fwd_ctas(N, h, Wo), loss_out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int Z>
static int launch_relax_bwd(const float* logits, int pitch, int N, int h, int w, int C, int Ho, int Wo,
                            const float* lse, const int32_t* sets, const float* lq, const float* loss_info,
                            const float* grad_out, float* workspace, float* dlogits, cudaStream_t stream) {
  const RelaxSets rs = relax_sets(const_cast<int32_t*>(sets), N, Ho, Wo);
  const int threads = (C + 31) / 32 * 32;
  const size_t smem = static_cast<size_t>(Z) * Wo * sizeof(RelaxPix);
  static std::atomic<bool> attr_set[64];
  if (smem > kSmemDefault) {
    int r = opt_in_smem(upsample_relax_rows_kernel<Z>, attr_set, static_cast<int>(kDiceSmemMax));
    if (r) return r;
  }
  upsample_relax_rows_kernel<Z><<<dim3(h, N), threads, smem, stream>>>(logits, pitch, N, h, w, C, Ho, Wo, lse, rs.tag,
                                                                       rs.omega, rs.mask, lq, workspace);
  SB_LAUNCHED();
  // loss_info[1] = D = sum of omega: the weighted cols kernel's 1 / D, 0 when D = 0
  upsample_ce_bwd_cols_kernel<true><<<dim3(h, N), 256, 0, stream>>>(workspace, N, h, w, C, loss_info, grad_out,
                                                                    dlogits);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_upsample_ce_relax_workspace_floats(int N, int Ho, int Wo, int zoom) {
  return semseg_upsample_ce_zoom_workspace_floats(N, Ho, Wo, zoom);
}

extern "C" long long semseg_upsample_ce_relax_sets_words(int N, int Ho, int Wo, int C) {
  SB_CHECK_ARG(N > 0 && Ho > 0 && Wo > 0 && C > 1 && C <= kMaxClasses, "upsample_ce_relax: bad sizes (C<=%d)",
               kMaxClasses);
  return (2LL + (C + 31) / 32) * N * Ho * Wo;
}

extern "C" int semseg_upsample_ce_relax_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                            const int64_t* target, int Ho, int Wo, int zoom, int ignore_index,
                                            int border, const float* class_weight, float* workspace, float* loss_out,
                                            int64_t* argmax, float* lse, int32_t* sets, float* lq, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, target, Ho, Wo, zoom);
  if (r) return r;
  r = check_relax(zoom, Wo, border, class_weight, sets, lq);
  if (r) return r;
  SB_CHECK_ARG(workspace && loss_out && lse && sets && lq, "upsample_ce_relax_fwd: null output");
  switch (zoom) {
    case 1: return launch_relax_fwd<1>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, border, class_weight,
                                       workspace, loss_out, argmax, lse, sets, lq, stream);
    case 2: return launch_relax_fwd<2>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, border, class_weight,
                                       workspace, loss_out, argmax, lse, sets, lq, stream);
    case 4: return launch_relax_fwd<4>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, border, class_weight,
                                       workspace, loss_out, argmax, lse, sets, lq, stream);
    default: return launch_relax_fwd<8>(logits, pitch, N, h, w, C, target, Ho, Wo, ignore_index, border, class_weight,
                                        workspace, loss_out, argmax, lse, sets, lq, stream);
  }
}

extern "C" long long semseg_upsample_ce_relax_bwd_workspace_floats(int N, int Ho, int w, int C, int zoom) {
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, zoom);
}

extern "C" int semseg_upsample_ce_relax_bwd(const float* logits, int pitch, int N, int h, int w, int C, int Ho, int Wo,
                                            int zoom, const float* lse, const int32_t* sets, const float* lq,
                                            const float* loss_info, const float* grad_out, float* workspace,
                                            float* dlogits, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int r = check_tail(logits, pitch, N, h, w, C, sets, Ho, Wo, zoom);
  if (r) return r;
  r = check_relax(zoom, Wo, 0, nullptr, sets, lq);
  if (r) return r;
  SB_CHECK_ARG(lse && lq && loss_info && grad_out && workspace && dlogits, "upsample_ce_relax_bwd: null pointer");
  switch (zoom) {
    case 1: return launch_relax_bwd<1>(logits, pitch, N, h, w, C, Ho, Wo, lse, sets, lq, loss_info, grad_out,
                                       workspace, dlogits, stream);
    case 2: return launch_relax_bwd<2>(logits, pitch, N, h, w, C, Ho, Wo, lse, sets, lq, loss_info, grad_out,
                                       workspace, dlogits, stream);
    case 4: return launch_relax_bwd<4>(logits, pitch, N, h, w, C, Ho, Wo, lse, sets, lq, loss_info, grad_out,
                                       workspace, dlogits, stream);
    default: return launch_relax_bwd<8>(logits, pitch, N, h, w, C, Ho, Wo, lse, sets, lq, loss_info, grad_out,
                                        workspace, dlogits, stream);
  }
}

// The x8 entry points (zoom_factor 8, every shipped config): the Z = 8 instances above.
extern "C" long long semseg_upsample_ce_workspace_floats(int N, int Ho, int Wo) {
  return semseg_upsample_ce_zoom_workspace_floats(N, Ho, Wo, 8);
}

extern "C" int semseg_upsample_ce_fwd(const float* logits, int pitch, int N, int h, int w, int C,
                                      const int64_t* target, int Ho, int Wo, int ignore_index, float* workspace,
                                      float* loss_out, int64_t* argmax, float* lse, void* stream_) {
  return semseg_upsample_ce_zoom_fwd(logits, pitch, N, h, w, C, target, Ho, Wo, 8, ignore_index, workspace, loss_out,
                                     argmax, lse, stream_);
}

extern "C" long long semseg_upsample_ce_bwd_workspace_floats(int N, int Ho, int w, int C) {
  return semseg_upsample_ce_zoom_bwd_workspace_floats(N, Ho, w, C, 8);
}

extern "C" int semseg_upsample_ce_bwd(const float* logits, int pitch, int N, int h, int w, int C,
                                      const int64_t* target, int Ho, int Wo, int ignore_index, const float* lse,
                                      const float* loss_info, const float* grad_out, float* workspace,
                                      float* dlogits, void* stream_) {
  return semseg_upsample_ce_zoom_bwd(logits, pitch, N, h, w, C, target, Ho, Wo, 8, ignore_index, lse, loss_info,
                                     grad_out, workspace, dlogits, stream_);
}

// Mixed-sample perturbation for mean-teacher training (semseg_b200/losses.py MixPseudoLabelLoss): CutMix (French et
// al., BMVC 2020, UniMatch's box) and ClassMix (Olsson et al., WACV 2021) masks on the input grid, and the mixed input
// and target batches.
//
// Image n is mixed with its partner (n + 1) mod N; M(n, i, j) = 1 means input pixel (i, j) comes from the partner. The
// draws are one uniform row per image, u[n, 0..4] = (apply, area, ratio, row, column) and, for ClassMix, u[n, 5 + c] =
// class priorities; image n is mixed iff double(u[n, 0]) < p.
//   CutMix  : the box of include/semseg_b200.h semseg_mix_apply, in fp64 with every operation correctly rounded
//             (explicit __d*_rn intrinsics: no contraction), so numpy reproduces it bit for bit.
//   ClassMix: A[m] = the teacher's argmax of image m after the x8 bilinear (align_corners) upsample to the input grid,
//             with the operations and the strict > of the pseudo-label forward's teacher pass at zoom 8
//             (csrc/tail.cu upsample_pl_fwd_kernel<8>), so A is that kernel's yhat bit for bit; S_m = the ceil(k/2) of
//             the k classes present in A[m] with the smallest (u[m, 5 + c], c). M(n, i, j) = mixed(n) and
//             A[pi(n)][i, j] in S_pi(n).
// Three kernels:
//   mix_argmax_x8: the plain forward's geometry (128 input columns per CTA, the two node rows staged, the horizontal
//                  interpolation shared by the 8 rows of an interval); A as uint8, and each image's present classes as
//                  256 bits (shared then global atomicOr: the bits do not depend on the order).
//   mix_select   : one CTA per image, one thread per class: a class's rank among the present ones by (u, c); a warp
//                  ballot gives each 32-class word of S.
//   mix_apply    : one CTA per (1024 input pixels, image), 4 consecutive pixels per thread; the CutMix box is computed
//                  once per CTA. M, then x_m (fp32 NCHW, float4 where a plane's 4 pixels are 16-byte aligned), the mask
//                  and, at the input pixels that lie on the target grid (both coordinates multiples of 8/Z), y_m. Every
//                  output element is written once, no atomics.
#include <cmath>

#include "host_common.h"

namespace sb {

constexpr int kMixCols = 128;          // argmax: input columns per CTA (the plain forward's kFwdCols at zoom 8)
constexpr int kMixNodes = kMixCols / 8 + 1;
constexpr int kMixApplyThreads = 256;
constexpr int kMixApplyPix = 4 * kMixApplyThreads;

// ------------------------------------------------------------------------------------------------ ClassMix argmax
__global__ void __launch_bounds__(kMixCols)
mix_argmax_x8_kernel(const float* __restrict__ tl, int pitch, int h, int w, int C, int Cs,
                     unsigned char* __restrict__ amap, unsigned* __restrict__ present) {
  extern __shared__ float S[];  // [2 node rows][kMixNodes][Cs], as upsample_ce_fwd_kernel<8, ...>
  __shared__ unsigned s_bits[8];
  const int n = blockIdx.z, i0 = blockIdx.y, x0 = blockIdx.x * kMixCols;
  const int H = 8 * (h - 1) + 1, W = 8 * (w - 1) + 1;
  const int i1 = min(i0 + 1, h - 1);
  const int j_base = x0 >> 3;
  const int nj = min(kMixNodes, w - j_base);
  const int tid = threadIdx.x;
  if (tid < 8) s_bits[tid] = 0u;
  for (int idx = tid; idx < 2 * nj * C; idx += kMixCols) {
    const int c = idx % C;
    const int node = idx / C;
    const int jj = node % nj, rr = node / nj;
    S[(rr * kMixNodes + jj) * Cs + c] = tl[((static_cast<size_t>(n) * h + (rr ? i1 : i0)) * w + (j_base + jj)) * pitch + c];
  }
  __syncthreads();
  const int x = x0 + tid;
  const int rows = min(8, H - 8 * i0);
  if (x < W) {
    const int j0 = x >> 3;
    const int j1 = min(j0 + 1, w - 1);
    const float l1w = static_cast<float>(x & 7) * 0.125f, l0w = 1.f - l1w;
    const float* At = S + (j0 - j_base) * Cs;
    const float* Bt = S + (j1 - j_base) * Cs;
    const float* Ct = At + kMixNodes * Cs;
    const float* Dt = Bt + kMixNodes * Cs;
    float mt[8];
    int at[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      mt[r] = -INFINITY;
      at[r] = 0;
    }
#pragma unroll 2
    for (int c = 0; c < C; ++c) {
      const float topt = l0w * At[c] + l1w * Bt[c];
      const float bott = l0w * Ct[c] + l1w * Dt[c];
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const float u = (1.f - 0.125f * r) * topt + (0.125f * r) * bott;   // tail.cu row_lerp<8>
        if (u > mt[r]) {
          mt[r] = u;
          at[r] = c;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if (r < rows) {
        amap[(static_cast<size_t>(n) * H + (8 * i0 + r)) * W + x] = static_cast<unsigned char>(at[r]);
        atomicOr(&s_bits[at[r] >> 5], 1u << (at[r] & 31));
      }
    }
  }
  __syncthreads();
  if (tid < 8 && s_bits[tid]) atomicOr(&present[n * 8 + tid], s_bits[tid]);
}

// ------------------------------------------------------------------------------------------------ ClassMix selection
__global__ void __launch_bounds__(256)
mix_select_kernel(const float* __restrict__ u, int ustride, const unsigned* __restrict__ present, int C,
                  unsigned* __restrict__ selected) {
  __shared__ float s_u[256];
  __shared__ unsigned s_p[8];
  const int m = blockIdx.x, c = threadIdx.x;
  s_u[c] = c < C ? u[static_cast<size_t>(m) * ustride + 5 + c] : 0.f;
  if (c < 8) s_p[c] = present[m * 8 + c];
  __syncthreads();
  int k = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) k += __popc(s_p[i]);
  const bool here = c < C && ((s_p[c >> 5] >> (c & 31)) & 1u);
  bool sel = false;
  if (here) {
    const float uc = s_u[c];
    int rank = 0;
    for (int d = 0; d < C; ++d) {
      if (((s_p[d >> 5] >> (d & 31)) & 1u) && (s_u[d] < uc || (s_u[d] == uc && d < c))) ++rank;
    }
    sel = rank < (k + 1) / 2;
  }
  const unsigned b = __ballot_sync(0xffffffffu, sel);
  if ((c & 31) == 0) selected[m * 8 + (c >> 5)] = b;
}

// ------------------------------------------------------------------------------------------------ mask and mixed batch
// The CutMix box of one image from its uniforms: (x0, y0, bw, bh).
__device__ void cutmix_box(const float* un, int H, int W, double alo, double ahi, double rlo, double rhi, int* box) {
  const double u1 = un[1], u2 = un[2], u3 = un[3], u4 = un[4];
  const double a = __dmul_rn(__dmul_rn(__dadd_rn(alo, __dmul_rn(__dsub_rn(ahi, alo), u1)), static_cast<double>(H)),
                             static_cast<double>(W));
  const double rho = __dadd_rn(rlo, __dmul_rn(__dsub_rn(rhi, rlo), u2));
  const int bw = min(W, max(1, static_cast<int>(floor(__dsqrt_rn(__ddiv_rn(a, rho))))));
  const int bh = min(H, max(1, static_cast<int>(floor(__dsqrt_rn(__dmul_rn(a, rho))))));
  box[0] = min(W - bw, static_cast<int>(floor(__dmul_rn(u4, static_cast<double>(W - bw + 1)))));
  box[1] = min(H - bh, static_cast<int>(floor(__dmul_rn(u3, static_cast<double>(H - bh + 1)))));
  box[2] = bw;
  box[3] = bh;
}

__global__ void __launch_bounds__(kMixApplyThreads)
mix_apply_kernel(int mode, const float* __restrict__ x, int N, int Cin, int H, int W, const long long* __restrict__ y,
                 int Ho, int Wo, int step, const float* __restrict__ u, int ustride, double p, double alo, double ahi,
                 double rlo, double rhi, const unsigned char* __restrict__ amap, const unsigned* __restrict__ selected,
                 unsigned char* __restrict__ mask, float* __restrict__ xm, long long* __restrict__ ym, int vec) {
  __shared__ int s_box[5];       // mixed, x0, y0, bw, bh
  __shared__ unsigned s_sel[8];  // ClassMix: S of the partner
  const int n = blockIdx.y, pn = n + 1 == N ? 0 : n + 1;
  const int tid = threadIdx.x;
  if (tid == 0) {
    const float* un = u + static_cast<size_t>(n) * ustride;
    s_box[0] = static_cast<double>(un[0]) < p;
    if (mode == SEMSEG_MIX_CUTMIX) cutmix_box(un, H, W, alo, ahi, rlo, rhi, s_box + 1);
  }
  if (mode == SEMSEG_MIX_CLASSMIX && tid < 8) s_sel[tid] = selected[pn * 8 + tid];
  __syncthreads();
  const long long HW = static_cast<long long>(H) * W;
  const long long p0 = (static_cast<long long>(blockIdx.x) * kMixApplyThreads + tid) * 4;
  if (p0 >= HW) return;
  const int cnt = static_cast<int>(min(4LL, HW - p0));
  const bool mixed = s_box[0] != 0;
  unsigned m4 = 0;
  for (int k = 0; k < cnt; ++k) {
    const long long pix = p0 + k;
    const int iy = static_cast<int>(pix / W), ix = static_cast<int>(pix - static_cast<long long>(iy) * W);
    bool m = false;
    if (mixed) {
      if (mode == SEMSEG_MIX_CUTMIX) {
        m = iy >= s_box[2] && iy < s_box[2] + s_box[4] && ix >= s_box[1] && ix < s_box[1] + s_box[3];
      } else {
        const int c = amap[static_cast<size_t>(pn) * HW + pix];
        m = (s_sel[c >> 5] >> (c & 31)) & 1u;
      }
    }
    m4 |= static_cast<unsigned>(m) << k;
    if (iy % step == 0 && ix % step == 0) {
      const size_t t = (static_cast<size_t>(n) * Ho + iy / step) * Wo + ix / step;
      const size_t tp = (static_cast<size_t>(pn) * Ho + iy / step) * Wo + ix / step;
      ym[t] = y[m ? tp : t];
    }
  }
  const size_t mo = static_cast<size_t>(n) * HW + p0;
  if (cnt == 4 && vec && (mo & 3) == 0) {
    *reinterpret_cast<uchar4*>(mask + mo) = make_uchar4(m4 & 1u, (m4 >> 1) & 1u, (m4 >> 2) & 1u, (m4 >> 3) & 1u);
  } else {
    for (int k = 0; k < cnt; ++k) mask[mo + k] = (m4 >> k) & 1u;
  }
  for (int c = 0; c < Cin; ++c) {
    const size_t o = (static_cast<size_t>(n) * Cin + c) * HW + p0;
    const size_t op = (static_cast<size_t>(pn) * Cin + c) * HW + p0;
    if (cnt == 4 && vec && (o & 3) == 0) {
      float4 v = *reinterpret_cast<const float4*>(x + o);
      if (m4) {
        if (m4 & 1u) v.x = x[op];
        if (m4 & 2u) v.y = x[op + 1];
        if (m4 & 4u) v.z = x[op + 2];
        if (m4 & 8u) v.w = x[op + 3];
      }
      *reinterpret_cast<float4*>(xm + o) = v;
    } else {
      for (int k = 0; k < cnt; ++k) xm[o + k] = ((m4 >> k) & 1u) ? x[op + k] : x[o + k];
    }
  }
}

}  // namespace sb

using namespace sb;

static bool mix_zoom_ok(int zoom) { return zoom == 1 || zoom == 2 || zoom == 4 || zoom == 8; }

extern "C" int semseg_mix_argmax_x8(const float* teacher, int pitch, int N, int h, int w, int C, uint8_t* argmax,
                                    uint32_t* present, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(teacher && argmax && present, "mix_argmax_x8: null pointer");
  SB_CHECK_ARG(N > 0 && h > 1 && w > 1 && C > 1 && C <= 256, "mix_argmax_x8: bad sizes (N=%d h=%d w=%d C=%d, C<=256)",
               N, h, w, C);
  SB_CHECK_ARG(pitch >= C, "mix_argmax_x8: pitch %d below C = %d", pitch, C);
  const int W = 8 * (w - 1) + 1;
  const int Cs = C | 1;
  const size_t smem = 2ull * kMixNodes * Cs * sizeof(float);     // <= 34,952 bytes: no opt-in
  SB_CUDA(cudaMemsetAsync(present, 0, static_cast<size_t>(N) * 8 * sizeof(uint32_t), stream));
  mix_argmax_x8_kernel<<<dim3(cdiv(W, kMixCols), h, N), kMixCols, smem, stream>>>(teacher, pitch, h, w, C, Cs, argmax,
                                                                                   present);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_mix_select(const float* uniforms, int ustride, const uint32_t* present, int N, int C,
                                 uint32_t* selected, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(uniforms && present && selected, "mix_select: null pointer");
  SB_CHECK_ARG(N > 0 && C > 1 && C <= 256, "mix_select: bad sizes (N=%d C=%d, C<=256)", N, C);
  SB_CHECK_ARG(ustride >= 5 + C, "mix_select: uniform row stride %d below 5 + C = %d", ustride, 5 + C);
  mix_select_kernel<<<N, 256, 0, stream>>>(uniforms, ustride, present, C, selected);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_mix_apply(int mode, const float* x, int N, int Cin, int H, int W, const int64_t* y, int Ho,
                                int Wo, int zoom, const float* uniforms, int ustride, double p, double area_lo,
                                double area_hi, double ratio_lo, double ratio_hi, const uint8_t* argmax,
                                const uint32_t* selected, uint8_t* mask, float* x_mixed, int64_t* y_mixed,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(mode == SEMSEG_MIX_CUTMIX || mode == SEMSEG_MIX_CLASSMIX, "mix_apply: mode %d is not CutMix or ClassMix",
               mode);
  SB_CHECK_ARG(mix_zoom_ok(zoom), "mix_apply: zoom %d is not one of 1, 2, 4, 8", zoom);
  SB_CHECK_ARG(x && y && uniforms && mask && x_mixed && y_mixed, "mix_apply: null pointer");
  SB_CHECK_ARG(mode == SEMSEG_MIX_CUTMIX || (argmax && selected), "mix_apply: ClassMix needs argmax and selected");
  SB_CHECK_ARG(N > 0 && Cin > 0 && H > 1 && W > 1 && (H - 1) % 8 == 0 && (W - 1) % 8 == 0,
               "mix_apply: bad sizes (N=%d Cin=%d H=%d W=%d; H-1 and W-1 multiples of 8)", N, Cin, H, W);
  SB_CHECK_ARG(Ho == (H - 1) / 8 * zoom + 1 && Wo == (W - 1) / 8 * zoom + 1,
               "mix_apply: needs Ho = %d(H-1)/8+1, Wo = %d(W-1)/8+1 (got %dx%d -> %dx%d)", zoom, zoom, H, W, Ho, Wo);
  SB_CHECK_ARG(ustride >= 5, "mix_apply: uniform row stride %d below 5", ustride);
  SB_CHECK_ARG(std::isfinite(p) && p >= 0.0 && p <= 1.0, "mix_apply: p %g outside [0, 1]", p);
  SB_CHECK_ARG(std::isfinite(area_lo) && std::isfinite(area_hi) && area_lo > 0.0 && area_lo <= area_hi &&
                   area_hi <= 1.0,
               "mix_apply: area (%g, %g) needs 0 < lo <= hi <= 1", area_lo, area_hi);
  SB_CHECK_ARG(std::isfinite(ratio_lo) && std::isfinite(ratio_hi) && ratio_lo > 0.0 && ratio_lo <= ratio_hi,
               "mix_apply: ratio (%g, %g) needs 0 < lo <= hi, finite", ratio_lo, ratio_hi);
  SB_CHECK_ARG(static_cast<const void*>(x) != static_cast<const void*>(x_mixed) &&
                   static_cast<const void*>(y) != static_cast<const void*>(y_mixed),
               "mix_apply: the mixed batch cannot overwrite its source");
  const long long HW = static_cast<long long>(H) * W;
  SB_CHECK_ARG(HW / kMixApplyPix < (1LL << 30), "mix_apply: image too large");
  const int vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_mixed)) & 15) == 0 &&
                  (reinterpret_cast<uintptr_t>(mask) & 3) == 0;
  mix_apply_kernel<<<dim3(static_cast<unsigned>((HW + kMixApplyPix - 1) / kMixApplyPix), N), kMixApplyThreads, 0,
                     stream>>>(mode, x, N, Cin, H, W, reinterpret_cast<const long long*>(y), Ho, Wo, 8 / zoom,
                               uniforms, ustride, p, area_lo, area_hi, ratio_lo, ratio_hi, argmax, selected, mask,
                               x_mixed, reinterpret_cast<long long*>(y_mixed), vec);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

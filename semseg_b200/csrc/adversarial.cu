// The L-infinity projected sign step of PGD / SegPGD attacks and their random start (semseg_b200/adversarial.py), on the
// network's fp32 NCHW input [N, 3, H, W] in the normalised space the network sees. With the per-channel constants of
// semseg_adv_box (step a, budget e, pixel box [lo, hi]) and x0 the clean input:
//   step : v = x + a sign(g);  v = min(max(v, x0 - e), x0 + e);  x' = min(max(v, lo), hi)
//   start: x = min(max(min(max(x0 + e (2u - 1), x0 - e), x0 + e), lo), hi)
// Every operation is one fp32 round-to-nearest in this order, so the results are bit-identical to the same formula in
// torch fp32. The products go through __fmul_rn / the sums through __fadd_rn: no FMA contraction. In the step a sign(g)
// is exact (sign in {-1, 0, 1}), so a contraction would be harmless there; in the start e (2u - 1) is not.
// One CTA row per (image, channel) plane: the channel's constants are read once per CTA from the launch parameters.
#include <algorithm>
#include <cmath>

#include "host_common.h"

namespace sb {

constexpr int kAdvThreads = 256;
constexpr int kAdvPerThread = 4;

__device__ __forceinline__ float adv_clamp(float v, float lo, float hi) { return fminf(fmaxf(v, lo), hi); }

__global__ void __launch_bounds__(kAdvThreads)
adv_step_kernel(const float* x, const float* __restrict__ g, const float* __restrict__ x0, float* out, long long hw,
                const semseg_adv_box box) {   // x and out may be one tensor: the step runs in place
  const int c = blockIdx.y % 3;
  const float a = box.step[c], e = box.eps[c], lo = box.lo[c], hi = box.hi[c];
  const size_t base = static_cast<size_t>(blockIdx.y) * hw;
  for (long long i = static_cast<long long>(blockIdx.x) * kAdvThreads + threadIdx.x; i < hw;
       i += static_cast<long long>(gridDim.x) * kAdvThreads) {
    const float gi = g[base + i];
    const float s = gi > 0.f ? 1.f : (gi < 0.f ? -1.f : 0.f);     // torch.sign: sign(0) = 0
    const float xi = x0[base + i];
    const float v = __fadd_rn(x[base + i], __fmul_rn(a, s));
    out[base + i] = adv_clamp(adv_clamp(v, __fsub_rn(xi, e), __fadd_rn(xi, e)), lo, hi);
  }
}

__global__ void __launch_bounds__(kAdvThreads)
adv_start_kernel(const float* __restrict__ x0, const float* __restrict__ u, float* __restrict__ out, long long hw,
                 const semseg_adv_box box) {
  const int c = blockIdx.y % 3;
  const float e = box.eps[c], lo = box.lo[c], hi = box.hi[c];
  const size_t base = static_cast<size_t>(blockIdx.y) * hw;
  for (long long i = static_cast<long long>(blockIdx.x) * kAdvThreads + threadIdx.x; i < hw;
       i += static_cast<long long>(gridDim.x) * kAdvThreads) {
    const float xi = x0[base + i];
    const float r = __fsub_rn(__fmul_rn(2.f, u[base + i]), 1.f);
    const float v = __fadd_rn(xi, __fmul_rn(e, r));
    out[base + i] = adv_clamp(adv_clamp(v, __fsub_rn(xi, e), __fadd_rn(xi, e)), lo, hi);
  }
}

}  // namespace sb

using namespace sb;

static int check_adv(const char* name, std::initializer_list<const void*> ptrs, int N, int H, int W,
                     const semseg_adv_box* box) {
  SB_CHECK_ARG(box != nullptr, "%s: null constants", name);
  for (const void* p : ptrs) {
    SB_CHECK_ARG(p != nullptr, "%s: null pointer", name);
    SB_CHECK_ARG((reinterpret_cast<uintptr_t>(p) & 3) == 0, "%s: tensor not 4-byte aligned", name);
  }
  SB_CHECK_ARG(N > 0 && H > 0 && W > 0 && 3LL * N <= 65535, "%s: bad shape [%d, 3, %d, %d]", name, N, H, W);
  for (int c = 0; c < 3; ++c) {
    SB_CHECK_ARG(std::isfinite(box->step[c]) && box->step[c] >= 0.f, "%s: step[%d] = %g is not finite and >= 0", name,
                 c, box->step[c]);
    SB_CHECK_ARG(std::isfinite(box->eps[c]) && box->eps[c] >= 0.f, "%s: eps[%d] = %g is not finite and >= 0", name, c,
                 box->eps[c]);
    SB_CHECK_ARG(std::isfinite(box->lo[c]) && std::isfinite(box->hi[c]) && box->lo[c] <= box->hi[c],
                 "%s: pixel box [%g, %g] of channel %d is not finite and ordered", name, box->lo[c], box->hi[c], c);
  }
  return SEMSEG_OK;
}

static dim3 adv_grid(int N, long long hw) {
  const long long per_cta = static_cast<long long>(kAdvThreads) * kAdvPerThread;
  return dim3(static_cast<unsigned>(std::min<long long>((hw + per_cta - 1) / per_cta, 65535)), 3 * N);
}

extern "C" int semseg_adv_step(const float* x, const float* grad, const float* x0, float* out, int N, int H, int W,
                               const semseg_adv_box* box, void* stream) {
  int r = check_adv("adv_step", {x, grad, x0, out}, N, H, W, box);
  if (r) return r;
  const long long hw = static_cast<long long>(H) * W;
  adv_step_kernel<<<adv_grid(N, hw), kAdvThreads, 0, static_cast<cudaStream_t>(stream)>>>(x, grad, x0, out, hw, *box);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_adv_start(const float* x0, const float* u, float* out, int N, int H, int W,
                                const semseg_adv_box* box, void* stream) {
  int r = check_adv("adv_start", {x0, u, out}, N, H, W, box);
  if (r) return r;
  const long long hw = static_cast<long long>(H) * W;
  adv_start_kernel<<<adv_grid(N, hw), kAdvThreads, 0, static_cast<cudaStream_t>(stream)>>>(x0, u, out, hw, *box);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

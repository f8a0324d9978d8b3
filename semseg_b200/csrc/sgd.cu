// Multi-tensor SGD with momentum and weight decay in ONE launch (SURVEY.md §8 f4; torch.optim.SGD as configured at
// tool/train.py:140,274-276 runs ~33 foreach kernels over the 161 parameter tensors):
//   g' = g + wd * w;   buf = first ? g' : momentum * buf + (1 - dampening) * g';   w -= lr * (nesterov ? g' + momentum*buf : buf)
// and, in a group whose momentum is 0, w -= lr * g' without reading or writing the buffer (torch leaves it as it is).
// Hyper-parameters are per parameter GROUP (the trainer rewrites the 8 group learning rates every iteration,
// tool/train.py:299-304; nesterov is bit `group` of h.nesterov) and travel by value in the launch parameters; tensors
// are described by a device-resident item table (built once) plus a device array of gradient pointers (gradients are
// fresh tensors every step).
#include "host_common.h"

namespace sb {

constexpr int kSgdChunk = 4096;   // elements per block

__global__ void __launch_bounds__(256)
sgd_multi_kernel(const semseg_sgd_item* __restrict__ items, const unsigned long long* __restrict__ grads, int n_items,
                 const semseg_sgd_hyper h) {
  __shared__ int s_item;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n_items - 1;
    const int b = static_cast<int>(blockIdx.x);
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (items[mid].chunk0 <= b) lo = mid; else hi = mid - 1;
    }
    s_item = lo;
  }
  __syncthreads();
  const semseg_sgd_item it = items[s_item];
  const float* __restrict__ g = reinterpret_cast<const float*>(grads[s_item]);
  if (g == nullptr) return;                      // parameter without a gradient this step (torch skips it too)
  const float lr = h.lr[it.group], mom = h.momentum[it.group], wd = h.weight_decay[it.group], damp = h.dampening[it.group];
  const bool nesterov = (h.nesterov >> it.group) & 1;
  const bool use_buf = mom != 0.f;               // without momentum the buffer (possibly none: buf == 0) is not touched
  const bool read_buf = use_buf && !it.first;
  const long long base = static_cast<long long>(static_cast<int>(blockIdx.x) - it.chunk0) * kSgdChunk;
  const long long end = min(base + kSgdChunk, it.n);
  auto upd = [&](float w, float gg, float b) -> float2 {
    gg = fmaf(wd, w, gg);
    if (!use_buf) return make_float2(w - lr * gg, b);
    b = it.first ? gg : fmaf(mom, b, (1.f - damp) * gg);
    const float step = nesterov ? fmaf(mom, b, gg) : b;
    return make_float2(w - lr * step, b);
  };
  const bool vec = ((reinterpret_cast<uintptr_t>(it.w) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(it.buf)) & 15) == 0;
  long long tail = base;
  if (vec) {
    for (long long i = base + 4LL * threadIdx.x; i + 3 < end; i += 4LL * blockDim.x) {
      float4 w = *reinterpret_cast<const float4*>(it.w + i);
      const float4 gg = *reinterpret_cast<const float4*>(g + i);
      float4 b = read_buf ? *reinterpret_cast<const float4*>(it.buf + i) : make_float4(0, 0, 0, 0);
      float2 r;
      r = upd(w.x, gg.x, b.x); w.x = r.x; b.x = r.y;
      r = upd(w.y, gg.y, b.y); w.y = r.x; b.y = r.y;
      r = upd(w.z, gg.z, b.z); w.z = r.x; b.z = r.y;
      r = upd(w.w, gg.w, b.w); w.w = r.x; b.w = r.y;
      *reinterpret_cast<float4*>(it.w + i) = w;
      if (use_buf) *reinterpret_cast<float4*>(it.buf + i) = b;
    }
    tail = base + ((end - base) & ~3LL);
  }
  for (long long i = tail + threadIdx.x; i < end; i += blockDim.x) {
    const float2 r = upd(it.w[i], g[i], read_buf ? it.buf[i] : 0.f);
    it.w[i] = r.x;
    if (use_buf) it.buf[i] = r.y;
  }
}

// Exponential moving average of a model's weights (semseg_b200/optim.py ModelEMA) in one launch, on the item-table and
// chunk layout of sgd_multi_kernel. fp32 items: e <- lerp(e, w, weight), weight = 1 - decay, in the two-branch form of
// torch.lerp (ATen's Lerp.h), so the result is the bits torch._foreach_lerp_(shadow, source, 1 - decay) gives:
//   weight < 0.5: e + weight (w - e)      else: w - (w - e) (1 - weight)
// (weight 1, decay 0, is an exact copy; weight 0 leaves e as it is). int64 items are copied. Element-wise, no atomics.
__device__ __forceinline__ float ema_lerp(float e, float w, float weight) {
  return fabsf(weight) < 0.5f ? fmaf(weight, w - e, e) : fmaf(-(w - e), 1.f - weight, w);
}

__global__ void __launch_bounds__(256)
ema_multi_kernel(const semseg_ema_item* __restrict__ items, int n_items, float weight) {
  __shared__ int s_item;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n_items - 1;
    const int b = static_cast<int>(blockIdx.x);
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (items[mid].chunk0 <= b) lo = mid; else hi = mid - 1;
    }
    s_item = lo;
  }
  __syncthreads();
  const semseg_ema_item it = items[s_item];
  const long long base = static_cast<long long>(static_cast<int>(blockIdx.x) - it.chunk0) * kSgdChunk;
  const long long end = min(base + kSgdChunk, it.n);
  if (it.kind == SEMSEG_EMA_COPY_I64) {
    long long* __restrict__ e = static_cast<long long*>(it.shadow);
    const long long* __restrict__ w = static_cast<const long long*>(it.source);
    for (long long i = base + threadIdx.x; i < end; i += blockDim.x) e[i] = w[i];
    return;
  }
  float* __restrict__ e = static_cast<float*>(it.shadow);
  const float* __restrict__ w = static_cast<const float*>(it.source);
  const bool vec = ((reinterpret_cast<uintptr_t>(e) | reinterpret_cast<uintptr_t>(w)) & 15) == 0;
  long long tail = base;
  if (vec) {
    for (long long i = base + 4LL * threadIdx.x; i + 3 < end; i += 4LL * blockDim.x) {
      float4 a = *reinterpret_cast<const float4*>(e + i);
      const float4 b = *reinterpret_cast<const float4*>(w + i);
      a.x = ema_lerp(a.x, b.x, weight);
      a.y = ema_lerp(a.y, b.y, weight);
      a.z = ema_lerp(a.z, b.z, weight);
      a.w = ema_lerp(a.w, b.w, weight);
      *reinterpret_cast<float4*>(e + i) = a;
    }
    tail = base + ((end - base) & ~3LL);
  }
  for (long long i = tail + threadIdx.x; i < end; i += blockDim.x) e[i] = ema_lerp(e[i], w[i], weight);
}

}  // namespace sb

extern "C" int semseg_ema_multi(const semseg_ema_item* items_dev, int n_items, int n_chunks, double decay,
                                void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(items_dev, "ema_multi: null item table");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(items_dev) & 7) == 0, "ema_multi: item table not 8-byte aligned");
  SB_CHECK_ARG(n_items > 0 && n_chunks > 0, "ema_multi: bad counts (%d items, %d chunks)", n_items, n_chunks);
  SB_CHECK_ARG(decay >= 0.0 && decay <= 1.0, "ema_multi: decay %g outside [0, 1]", decay);
  sb::ema_multi_kernel<<<static_cast<unsigned>(n_chunks), 256, 0, stream>>>(items_dev, n_items,
                                                                            static_cast<float>(1.0 - decay));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_sgd_chunk_elems(void) { return sb::kSgdChunk; }

extern "C" int semseg_sgd_multi(const semseg_sgd_item* items_dev, const void* grad_ptrs_dev, int n_items, int n_chunks,
                                const semseg_sgd_hyper* hyper, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(items_dev && grad_ptrs_dev && hyper && n_items > 0 && n_chunks > 0, "sgd_multi: bad args");
  sb::sgd_multi_kernel<<<static_cast<unsigned>(n_chunks), 256, 0, stream>>>(
      items_dev, static_cast<const unsigned long long*>(grad_ptrs_dev), n_items, *hyper);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

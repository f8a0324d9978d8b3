// Device-side segmentation metrics (SURVEY §8 f4): intersection / union / target areas per class in ONE pass.
//
// Replaces util/util.py:55-67 of the reference (intersectionAndUnionGPU: a masked in-place write, a boolean-mask gather
// and three torch.histc passes over N*H*W int64 elements, each with its own temporaries) as called from
// tool/train.py:286 and :375. Counts are integers accumulated with integer atomics -> exact and order-independent.
#include "host_common.h"

namespace sb {

// counts[0:K] = |pred == target, target valid|, counts[K:2K] = |pred == k| (pred forced to `ignore` where the target is
// ignored, like the reference's in-place masking), counts[2K:3K] = |target == k|. Values outside [0, K) are not
// counted (torch.histc(min=0, max=K-1) drops them).
__global__ void __launch_bounds__(256) iou_hist_kernel(long long* __restrict__ pred, const long long* __restrict__ target,
                                                       long long n, int K, long long ignore, int write_back,
                                                       int* __restrict__ counts) {
  extern __shared__ int h[];  // [3 * K]
  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x) h[i] = 0;
  __syncthreads();
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long t = target[i];
    long long p = pred[i];
    if (t == ignore) {
      if (write_back && p != ignore) pred[i] = ignore;
      p = ignore;
    }
    if (p >= 0 && p < K) {
      atomicAdd(&h[K + static_cast<int>(p)], 1);
      if (p == t) atomicAdd(&h[static_cast<int>(p)], 1);
    }
    if (t >= 0 && t < K) atomicAdd(&h[2 * K + static_cast<int>(t)], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 3 * K; i += blockDim.x)
    if (h[i]) atomicAdd(&counts[i], h[i]);
}

}  // namespace sb

extern "C" int semseg_iou_hist(void* pred, const void* target, long long n, int K, long long ignore_index,
                               int write_back, int* counts, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // an empty batch (n == 0, whose tensors may have no storage) gives zero counts, as the reference's histc does
  SB_CHECK_ARG(counts && n >= 0 && K > 0 && K <= 4096 && (n == 0 || (pred && target)),
               "iou_hist: bad args (n=%lld, K=%d)", n, K);
  SB_CUDA(cudaMemsetAsync(counts, 0, sizeof(int) * 3 * K, stream));
  if (n == 0) return SEMSEG_OK;
  long long blocks = (n + 256 * 8 - 1) / (256 * 8);
  if (blocks > 148 * 8) blocks = 148 * 8;
  if (blocks < 1) blocks = 1;
  sb::iou_hist_kernel<<<static_cast<unsigned>(blocks), 256, sizeof(int) * 3 * K, stream>>>(
      static_cast<long long*>(pred), static_cast<const long long*>(target), n, K, ignore_index, write_back, counts);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

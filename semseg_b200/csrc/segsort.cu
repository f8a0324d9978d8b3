// Segmented stable radix sort of (uint32 key, uint32 payload) pairs: S segments of one common length L, each sorted by
// key ascending, pairs with equal keys keeping their input order. The Lovász-Softmax loss (csrc/tail.cu) sorts one
// segment of pixel errors per class (or per image and class) with it; it is exported so that it can be tested alone.
//
// LSD radix sort, kSortBits bits per pass from the lowest digit, ping-pong between the caller's two buffers (an even
// number of passes: the result lands back in the input buffers). Each pass is three launches:
//   hist   : one CTA per (segment, tile of kSortTile pairs): the tile's digit histogram in shared memory (integer
//            atomics: the counts do not depend on their order) -> counts[seg][digit][tile];
//   scan   : one CTA per segment: an exclusive scan of counts[seg] in (digit, tile) order, in place -> the position of
//            the first pair of each (digit, tile) in the segment's output;
//   scatter: one CTA per (segment, tile): the tile's pairs in input order, kSortThreads at a time; a pair's output
//            position is its (digit, tile) base plus the number of pairs with the same digit before it in the tile
//            (warp match-any within a round, a per-digit scan over the round's warps, a running count across rounds).
// Tiles never straddle a segment, the launch geometry depends only on (S, L), nothing is read back to the host, and
// every write position is a function of the input alone: the sort captures into a CUDA graph and is deterministic.
// A segment whose skip flag is non-zero is not read or written by any pass.
#include <utility>

#include "host_common.h"

namespace sb {

constexpr int kSortBits = 8;                       // digit width: 4 passes over 32-bit keys
constexpr int kSortDigits = 1 << kSortBits;
constexpr int kSortPasses = 32 / kSortBits;
constexpr int kSortThreads = 256;
constexpr int kSortItems = 16;                     // pairs per thread per tile
constexpr int kSortTile = kSortThreads * kSortItems;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kScanThreads = 1024;
static_assert(kSortPasses % 2 == 0, "the result must land in the input buffers");
static_assert(kSortDigits == kSortThreads, "one thread per digit in the per-round scan");

__global__ void __launch_bounds__(kSortThreads)
segsort_hist_kernel(const unsigned* __restrict__ keys, int L, int nt, int shift, const int* __restrict__ skip,
                    unsigned* __restrict__ counts) {
  __shared__ unsigned hist[kSortDigits];
  const int seg = blockIdx.x / nt, tile = blockIdx.x % nt;
  if (skip && skip[seg]) return;
  hist[threadIdx.x] = 0;
  __syncthreads();
  const unsigned* K = keys + static_cast<size_t>(seg) * L;
  const int base = tile * kSortTile;
  const int end = min(base + kSortTile, L);
  for (int i = base + threadIdx.x; i < end; i += kSortThreads) atomicAdd(&hist[(K[i] >> shift) & (kSortDigits - 1)], 1u);
  __syncthreads();
  counts[(static_cast<size_t>(seg) * kSortDigits + threadIdx.x) * nt + tile] = hist[threadIdx.x];
}

// Exclusive scan of one segment's kSortDigits * nt counts, in place: each thread owns a contiguous chunk.
__global__ void __launch_bounds__(kScanThreads)
segsort_scan_kernel(unsigned* __restrict__ counts, int nt, const int* __restrict__ skip) {
  __shared__ unsigned warp_sum[kScanThreads / 32];
  const int seg = blockIdx.x;
  if (skip && skip[seg]) return;
  unsigned* C = counts + static_cast<size_t>(seg) * kSortDigits * nt;
  const int M = kSortDigits * nt;
  const int chunk = (M + kScanThreads - 1) / kScanThreads;
  const int b = min(threadIdx.x * chunk, M), e = min(b + chunk, M);
  unsigned s = 0;
  for (int i = b; i < e; ++i) s += C[i];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
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
    warp_sum[lane] = v;   // inclusive over warps
  }
  __syncthreads();
  unsigned run = inc - s + (warp ? warp_sum[warp - 1] : 0u);
  for (int i = b; i < e; ++i) {
    const unsigned c = C[i];
    C[i] = run;
    run += c;
  }
}

__global__ void __launch_bounds__(kSortThreads)
segsort_scatter_kernel(const unsigned* __restrict__ keys_in, const unsigned* __restrict__ vals_in,
                       unsigned* __restrict__ keys_out, unsigned* __restrict__ vals_out, int L, int nt, int shift,
                       const int* __restrict__ skip, const unsigned* __restrict__ counts) {
  __shared__ unsigned run[kSortDigits];                 // output position of the next pair of each digit
  __shared__ unsigned wbase[kSortWarps][kSortDigits];   // per round: the warps' pair counts, then their bases
  const int seg = blockIdx.x / nt, tile = blockIdx.x % nt;
  if (skip && skip[seg]) return;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  run[tid] = counts[(static_cast<size_t>(seg) * kSortDigits + tid) * nt + tile];
  const size_t off = static_cast<size_t>(seg) * L;
  const int base = tile * kSortTile;
  const int n = min(kSortTile, L - base);
  const unsigned lt = (1u << lane) - 1u;
  for (int r = 0; r * kSortThreads < n; ++r) {
#pragma unroll
    for (int w = 0; w < kSortWarps; ++w) wbase[w][tid] = 0;
    const int i = r * kSortThreads + tid;
    const bool in = i < n;
    unsigned k = 0, v = 0, d = kSortDigits;   // kSortDigits: no pair (the tile's tail)
    if (in) {
      k = keys_in[off + base + i];
      v = vals_in[off + base + i];
      d = (k >> shift) & (kSortDigits - 1);
    }
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const unsigned rank = __popc(peers & lt);
    __syncthreads();
    if (in && rank == 0) wbase[warp][d] = __popc(peers);
    __syncthreads();
    {
      unsigned s = run[tid];
#pragma unroll
      for (int w = 0; w < kSortWarps; ++w) {
        const unsigned c = wbase[w][tid];
        wbase[w][tid] = s;
        s += c;
      }
      run[tid] = s;
    }
    __syncthreads();
    if (in) {
      const size_t pos = off + wbase[warp][d] + rank;
      keys_out[pos] = k;
      vals_out[pos] = v;
    }
    __syncthreads();
  }
}

static int check_segsort(int S, long long L) {
  SB_CHECK_ARG(S > 0 && L > 0 && L < (1LL << 31), "segsort: bad sizes S=%d L=%lld", S, L);
  const long long nt = (L + kSortTile - 1) / kSortTile;
  SB_CHECK_ARG(nt * S < (1LL << 31), "segsort: %d segments of %lld pairs are too many tiles", S, L);
  return SEMSEG_OK;
}

}  // namespace sb

using namespace sb;

extern "C" long long semseg_segsort_u32_pairs_workspace_bytes(int S, long long L) {
  int r = check_segsort(S, L);
  if (r) return r;
  return static_cast<long long>(S) * kSortDigits * ((L + kSortTile - 1) / kSortTile) * sizeof(unsigned);
}

extern "C" int semseg_segsort_u32_pairs(unsigned* keys, unsigned* vals, unsigned* keys_alt, unsigned* vals_alt, int S,
                                        long long L, const int* skip, void* workspace, void* stream_) {
  int r = check_segsort(S, L);
  if (r) return r;
  SB_CHECK_ARG(keys && vals && keys_alt && vals_alt && workspace, "segsort: null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const int nt = static_cast<int>((L + kSortTile - 1) / kSortTile);
  const int Li = static_cast<int>(L);
  unsigned* counts = static_cast<unsigned*>(workspace);
  unsigned* src_k = keys;
  unsigned* src_v = vals;
  unsigned* dst_k = keys_alt;
  unsigned* dst_v = vals_alt;
  for (int pass = 0; pass < kSortPasses; ++pass) {
    const int shift = pass * kSortBits;
    segsort_hist_kernel<<<nt * S, kSortThreads, 0, stream>>>(src_k, Li, nt, shift, skip, counts);
    SB_LAUNCHED();
    segsort_scan_kernel<<<S, kScanThreads, 0, stream>>>(counts, nt, skip);
    SB_LAUNCHED();
    segsort_scatter_kernel<<<nt * S, kSortThreads, 0, stream>>>(src_k, src_v, dst_k, dst_v, Li, nt, shift, skip,
                                                                counts);
    SB_LAUNCHED();
    std::swap(src_k, dst_k);
    std::swap(src_v, dst_v);
  }
  return SEMSEG_OK;
}

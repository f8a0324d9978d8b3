// Dense CRF refinement (Krähenbühl & Koltun, NeurIPS 2011) of one image's class probabilities: Potts mean-field
// inference with a smoothness kernel (d = 2 features: x, y over pos_xy_std) and an appearance kernel (d = 5: x, y over
// bi_xy_std, r, g, b over bi_rgb_std), each filter approximated on a permutohedral lattice (Adams, Baek & Davis,
// Eurographics 2010) and symmetrically normalised (K~ v = n * K (n * v), n = (K 1 + 1e-20)^-1/2).
//
// One lattice code path, templated on d, serves both kernels.
//   build (once per image and kernel):
//     keys      : one thread per pixel. The features are elevated onto the d-dimensional hyperplane of Z^{d+1} (scaled
//                 by (d+1) sqrt(2/3)), the enclosing simplex is found by rounding and ranking, all in fp64 with explicit
//                 round-to-nearest operations (no FMA contraction: the keys equal a float64 numpy restatement's). Each
//                 of the d+1 vertices' first d coordinates is packed into one 64-bit key, coordinate i offset by off[i]
//                 into bits [shift[i], shift[i] + bits[i]); the widths come from the coordinate ranges on the host.
//     sort      : the (key, entry) pairs, entry = pixel (d+1) + k, by the stable segmented radix sort of csrc/segsort.cu
//                 with S = 1: on the low key word, then (the high words gathered in that order) on the high word.
//     unique    : vertex ids from a tiled scan of the key changes -> each entry's vertex, each vertex's run of sorted
//                 entries and its key; V lands in the lattice header on the device.
//     neighbours: per vertex and lattice direction j, the vertices at key -+ (1, .., 1) with coordinate j replaced by
//                 +-d (binary search in the sorted keys), -1 where there is none.
//     norm      : the filter of a ones vector, n = (K 1 + 1e-20)^-1/2.
//   filter (per kernel and mean-field iteration): splat (a fixed-order sum over each vertex's run of sorted entries),
//   d+1 blur passes ([1 2 1] / 2 along each direction, gathered through the neighbour table, ping-pong), slice.
//   update (per iteration): one warp per pixel computes the unary, slices both kernels' lattices, scales by n and the
//   kernel weights and takes the softmax over C.
// Values are fp32 and class-contiguous ([V][C] on the lattice, [N][C] on the pixels). No float atomics, every result is
// written once: the whole CRF is deterministic.
#include <float.h>
#include <math.h>

#include <algorithm>
#include <cmath>
#include <utility>

#include "host_common.h"

namespace sb {
namespace {

typedef unsigned long long u64;

constexpr int kDcrfThreads = 256;
constexpr int kDcrfItems = 16;                      // entries per thread in the unique scan
constexpr int kDcrfTile = kDcrfThreads * kDcrfItems;
constexpr int kDcrfScanThreads = 1024;
constexpr int kDcrfMaxBlocks = 1 << 20;             // grid-stride cap of the element-wise kernels

struct KeyPack {
  long long off[5];
  int shift[5];
  int bits[5];
};

struct Scales {
  double s[5];   // (d+1) sqrt(2/3) / sqrt((i+1)(i+2))
};

// ------------------------------------------------------------------------------------------------ build kernels
template <int D>
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_keys_kernel(const float* __restrict__ image, int H, int W, double sxy, double srgb, Scales sc, KeyPack pk,
                 u64* __restrict__ key64, unsigned* __restrict__ lo, unsigned* __restrict__ idx, float* __restrict__ wts) {
  const int N = H * W;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) {
    double f[D];
    f[0] = static_cast<double>(i % W) / sxy;
    f[1] = static_cast<double>(i / W) / sxy;
    if constexpr (D == 5) {
#pragma unroll
      for (int c = 0; c < 3; ++c) f[2 + c] = static_cast<double>(fminf(fmaxf(image[3 * static_cast<size_t>(i) + c], 0.f), 255.f)) / srgb;
    }
    double el[D + 1];
    double sm = 0.0;
#pragma unroll
    for (int j = D; j > 0; --j) {
      const double cf = __dmul_rn(f[j - 1], sc.s[j - 1]);
      el[j] = __dsub_rn(sm, __dmul_rn(static_cast<double>(j), cf));
      sm = __dadd_rn(sm, cf);
    }
    el[0] = sm;
    const double down = 1.0 / (D + 1);
    long long rem0[D + 1];
    int rank[D + 1];
    long long sum = 0;
#pragma unroll
    for (int k = 0; k <= D; ++k) {
      const long long rd = static_cast<long long>(floor(__dadd_rn(__dmul_rn(el[k], down), 0.5)));
      rem0[k] = rd * (D + 1);
      sum += rd;
      rank[k] = 0;
    }
#pragma unroll
    for (int a = 0; a < D; ++a)
#pragma unroll
      for (int b = a + 1; b <= D; ++b) {
        if (__dsub_rn(el[a], static_cast<double>(rem0[a])) < __dsub_rn(el[b], static_cast<double>(rem0[b]))) ++rank[a];
        else ++rank[b];
      }
    if (sum > 0) {
#pragma unroll
      for (int k = 0; k <= D; ++k) {
        if (rank[k] >= D + 1 - sum) {
          rem0[k] -= D + 1;
          rank[k] += static_cast<int>(sum) - (D + 1);
        } else {
          rank[k] += static_cast<int>(sum);
        }
      }
    } else if (sum < 0) {
#pragma unroll
      for (int k = 0; k <= D; ++k) {
        if (rank[k] < -sum) {
          rem0[k] += D + 1;
          rank[k] += D + 1 + static_cast<int>(sum);
        } else {
          rank[k] += static_cast<int>(sum);
        }
      }
    }
    double bary[D + 2];
#pragma unroll
    for (int k = 0; k < D + 2; ++k) bary[k] = 0.0;
#pragma unroll
    for (int k = 0; k <= D; ++k) {
      const double v = __dmul_rn(__dsub_rn(el[k], static_cast<double>(rem0[k])), down);
      bary[D - rank[k]] += v;
      bary[D - rank[k] + 1] -= v;
    }
    bary[0] += 1.0 + bary[D + 1];
#pragma unroll
    for (int r = 0; r <= D; ++r) {
      u64 key = 0;
#pragma unroll
      for (int k = 0; k < D; ++k) {
        const long long coord = rem0[k] + (rank[k] <= D - r ? r : r - (D + 1));
        key |= static_cast<u64>(coord + pk.off[k]) << pk.shift[k];
      }
      const size_t e = static_cast<size_t>(i) * (D + 1) + r;
      key64[e] = key;
      lo[e] = static_cast<unsigned>(key);
      idx[e] = static_cast<unsigned>(e);
      wts[e] = static_cast<float>(bary[r]);
    }
  }
}

__global__ void dcrf_gather_hi_kernel(const u64* __restrict__ key64, const unsigned* __restrict__ idx, int L,
                                      unsigned* __restrict__ hi) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L; i += gridDim.x * blockDim.x)
    hi[i] = static_cast<unsigned>(key64[idx[i]] >> 32);
}

__device__ __forceinline__ bool dcrf_starts(const u64* key64, const unsigned* idx, int i) {
  return i == 0 || key64[idx[i]] != key64[idx[i - 1]];
}

// Number of vertex starts (key changes) in each tile of kDcrfTile sorted entries.
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_unique_count_kernel(const u64* __restrict__ key64, const unsigned* __restrict__ idx, int L,
                         unsigned* __restrict__ tile_count) {
  __shared__ unsigned total;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  const int base = blockIdx.x * kDcrfTile, end = min(base + kDcrfTile, L);
  unsigned n = 0;
  for (int i = base + threadIdx.x; i < end; i += kDcrfThreads) n += dcrf_starts(key64, idx, i);
  atomicAdd(&total, n);   // integer: the count does not depend on the order
  __syncthreads();
  if (threadIdx.x == 0) tile_count[blockIdx.x] = total;
}

// Exclusive scan of the tile counts in place (one CTA); V = the total -> Vout, run[V] = L.
__global__ void __launch_bounds__(kDcrfScanThreads)
dcrf_scan_tiles_kernel(unsigned* __restrict__ c, int nt, int L, int* __restrict__ Vout, int* __restrict__ run) {
  __shared__ unsigned warp_sum[kDcrfScanThreads / 32];
  const int chunk = (nt + kDcrfScanThreads - 1) / kDcrfScanThreads;
  const int b = min(static_cast<int>(threadIdx.x) * chunk, nt), e = min(b + chunk, nt);
  unsigned s = 0;
  for (int i = b; i < e; ++i) s += c[i];
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
    warp_sum[lane] = v;
  }
  __syncthreads();
  unsigned r = inc - s + (warp ? warp_sum[warp - 1] : 0u);
  for (int i = b; i < e; ++i) {
    const unsigned x = c[i];
    c[i] = r;
    r += x;
  }
  if (threadIdx.x == kDcrfScanThreads - 1) {
    *Vout = static_cast<int>(warp_sum[31]);
    run[warp_sum[31]] = L;
  }
}

// Each thread owns kDcrfItems consecutive sorted entries of the tile: vertex ids in sorted order, scattered back to the
// entries; each vertex's first sorted entry and key.
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_unique_write_kernel(const u64* __restrict__ key64, const unsigned* __restrict__ idx, int L,
                         const unsigned* __restrict__ tile_base, int* __restrict__ vid, int* __restrict__ run,
                         u64* __restrict__ vkey) {
  __shared__ unsigned warp_sum[kDcrfThreads / 32];
  const int b = blockIdx.x * kDcrfTile + threadIdx.x * kDcrfItems, e = min(b + kDcrfItems, L);
  unsigned s = 0;
  for (int i = b; i < e; ++i) s += dcrf_starts(key64, idx, i);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned inc = s;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  unsigned before = 0;
  for (int w = 0; w < warp; ++w) before += warp_sum[w];
  int v = static_cast<int>(tile_base[blockIdx.x] + before + inc - s) - 1;   // the vertex of the entry before b
  for (int i = b; i < e; ++i) {
    const unsigned p = idx[i];
    if (dcrf_starts(key64, idx, i)) {
      ++v;
      run[v] = i;
      vkey[v] = key64[p];
    }
    vid[p] = v;
  }
}

template <int D>
__device__ __forceinline__ int dcrf_find(const u64* __restrict__ vkey, int V, u64 key) {
  int lo = 0, hi = V;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (vkey[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return (lo < V && vkey[lo] == key) ? lo : -1;
}

// nbr[v][j][0] = the vertex at key - 1 (coordinate j: + d), nbr[v][j][1] at key + 1 (coordinate j: - d); for j = d
// every stored coordinate moves by -1 / +1 (the implied coordinate d takes the +-d).
template <int D>
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_neighbours_kernel(const u64* __restrict__ vkey, const int* __restrict__ Vp, int Vcap, KeyPack pk,
                       int* __restrict__ nbr) {
  const int V = min(*Vp, Vcap);
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
    const u64 key = vkey[v];
    long long u[D];
#pragma unroll
    for (int k = 0; k < D; ++k) u[k] = static_cast<long long>((key >> pk.shift[k]) & ((1ull << pk.bits[k]) - 1));
#pragma unroll
    for (int j = 0; j <= D; ++j)
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        u64 nk = 0;
        bool ok = true;
#pragma unroll
        for (int k = 0; k < D; ++k) {
          const long long x = u[k] + (k == j ? (s ? -D : D) : (s ? 1 : -1));
          ok = ok && x >= 0 && x < (1ll << pk.bits[k]);
          nk |= static_cast<u64>(x) << pk.shift[k];
        }
        nbr[(static_cast<size_t>(v) * (D + 1) + j) * 2 + s] = ok ? dcrf_find<D>(vkey, V, nk) : -1;
      }
  }
}

template <int D>
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_unpack_kernel(const u64* __restrict__ vkey, const int* __restrict__ Vp, int Vcap, KeyPack pk, int* __restrict__ out) {
  const int V = min(*Vp, Vcap);
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
    const u64 key = vkey[v];
#pragma unroll
    for (int k = 0; k < D; ++k)
      out[static_cast<size_t>(v) * D + k] =
          static_cast<int>(static_cast<long long>((key >> pk.shift[k]) & ((1ull << pk.bits[k]) - 1)) - pk.off[k]);
  }
}

// ------------------------------------------------------------------------------------------------ filter kernels
// lat[v][c] = sum over the vertex's sorted entries e (pixel p) of w[e] * norm[p] * in[p][c]; in == null: ones (C = 1),
// norm == null: 1.
template <int D>
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_splat_kernel(const unsigned* __restrict__ idx, const int* __restrict__ run, const float* __restrict__ wts,
                  const float* __restrict__ norm, const float* __restrict__ in, int C, const int* __restrict__ Vp,
                  int Vcap, float* __restrict__ lat) {
  const long long total = static_cast<long long>(min(*Vp, Vcap)) * C;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(t / C), c = static_cast<int>(t - static_cast<long long>(v) * C);
    const int b = run[v], e = run[v + 1];
    float acc = 0.f;
    for (int j = b; j < e; ++j) {
      const unsigned p = idx[j];
      const unsigned pix = p / (D + 1);
      float x = in ? in[static_cast<size_t>(pix) * C + c] : 1.f;
      if (norm) x *= norm[pix];
      acc += wts[p] * x;
    }
    lat[t] = acc;
  }
}

template <int D>
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_blur_kernel(const int* __restrict__ nbr, int j, int C, const int* __restrict__ Vp, int Vcap,
                 const float* __restrict__ in, float* __restrict__ out) {
  const int V = min(*Vp, Vcap);
  const long long total = static_cast<long long>(V) * C;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(t / C), c = static_cast<int>(t - static_cast<long long>(v) * C);
    const int n1 = nbr[(static_cast<size_t>(v) * (D + 1) + j) * 2], n2 = nbr[(static_cast<size_t>(v) * (D + 1) + j) * 2 + 1];
    const float a = (n1 >= 0 && n1 < V) ? in[static_cast<size_t>(n1) * C + c] : 0.f;
    const float b = (n2 >= 0 && n2 < V) ? in[static_cast<size_t>(n2) * C + c] : 0.f;
    out[t] = in[t] + 0.5f * (a + b);
  }
}

template <int D>
__device__ __forceinline__ float dcrf_slice_one(const int* __restrict__ vid, const float* __restrict__ wts,
                                                const float* __restrict__ lat, int V, int C, size_t i, int c) {
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k <= D; ++k) {
    const int v = vid[i * (D + 1) + k];
    if (v >= 0 && v < V) acc += wts[i * (D + 1) + k] * lat[static_cast<size_t>(v) * C + c];
  }
  return acc;
}

// out[i][c] = norm[i] * slice (norm == null: 1); finish_norm: out[i] = (slice + 1e-20)^-1/2 (C = 1).
template <int D>
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_slice_kernel(const int* __restrict__ vid, const float* __restrict__ wts, const float* __restrict__ lat,
                  const int* __restrict__ Vp, int Vcap, int N, int C, const float* __restrict__ norm, int finish_norm,
                  float* __restrict__ out) {
  const int V = min(*Vp, Vcap);
  const long long total = static_cast<long long>(N) * C;
  for (long long t = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; t < total;
       t += static_cast<long long>(gridDim.x) * blockDim.x) {
    const size_t i = static_cast<size_t>(t / C);
    const int c = static_cast<int>(t - static_cast<long long>(i) * C);
    const float s = dcrf_slice_one<D>(vid, wts, lat, V, C, i, c);
    out[t] = finish_norm ? 1.f / sqrtf(s + 1e-20f) : (norm ? norm[i] * s : s);
  }
}

struct Lattice {
  float* w;       // [L] barycentric weight of entry pixel (d+1) + k
  int* vid;       // [L] vertex of the entry
  unsigned* idx;  // [L] entries in key order
  int* run;       // [Vmax + 1] first sorted entry of each vertex, run[V] = L
  int* nbr;       // [Vmax][d+1][2]
  u64* vkey;      // [Vmax] packed keys, ascending
  float* norm;    // [N]
};

struct Message {
  const int* vid;
  const float* w;
  const float* norm;
  const float* lat;
  int V;
  float weight;
};

__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// One warp per pixel: Q[i][c] = softmax_c(log max(P[i][c], clip) + w_s n_s[i] slice_s + w_a n_a[i] slice_a); a
// message whose lat is null is left out.
__global__ void __launch_bounds__(kDcrfThreads)
dcrf_update_kernel(const float* __restrict__ prob, int N, int C, float clip, Message ms, Message ma,
                   float* __restrict__ Q) {
  const int lane = threadIdx.x & 31;
  const int warps = gridDim.x * (blockDim.x >> 5);
  for (int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < N; i += warps) {
    const size_t row = static_cast<size_t>(i) * C;
    const float gs = ms.lat ? ms.weight * ms.norm[i] : 0.f;
    const float ga = ma.lat ? ma.weight * ma.norm[i] : 0.f;
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) {
      float z = logf(fmaxf(prob[row + c], clip));
      if (ms.lat) z += gs * dcrf_slice_one<2>(ms.vid, ms.w, ms.lat, ms.V, C, i, c);
      if (ma.lat) z += ga * dcrf_slice_one<5>(ma.vid, ma.w, ma.lat, ma.V, C, i, c);
      Q[row + c] = z;
      m = fmaxf(m, z);
    }
    m = warp_max(m);
    float s = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float e = expf(Q[row + c] - m);
      Q[row + c] = e;
      s += e;
    }
    const float inv = 1.f / warp_sum(s);
    for (int c = lane; c < C; c += 32) Q[row + c] *= inv;
  }
}

// ------------------------------------------------------------------------------------------------ host side
int grid_for(long long n) { return static_cast<int>(std::max(1LL, std::min<long long>((n + kDcrfThreads - 1) / kDcrfThreads, kDcrfMaxBlocks))); }

Scales scales_for(int d) {
  Scales sc{};
  for (int i = 0; i < d; ++i) sc.s[i] = std::sqrt(2.0 / 3.0) * (d + 1) / std::sqrt(static_cast<double>((i + 1) * (i + 2)));
  return sc;
}

// Key layout of kernel d on an H x W image: each stored coordinate's range from the elevation's linear form over the
// feature ranges (x in [0, W-1], y in [0, H-1], colour in [0, 255]), widened by 4(d+1) for the rounding, the simplex
// vertices and the blur neighbours. Returns the total bit count (> 64: does not fit). A coordinate whose range leaves
// [-2^52, 2^52] counts as at least 53 bits without any integer conversion: beyond it the device's fp64 elevation no
// longer rounds to exact integers and the int64 arithmetic of the keys could overflow, so such a layout is rejected
// (1024 bits for an infinite or NaN range, from standard deviations so small that the features overflow).
int key_layout(int d, int H, int W, double sxy, double srgb, KeyPack* pk) {
  const double kRange = 4503599627370496.0;   // 2^52
  const Scales sc = scales_for(d);
  double fmax[5] = {(W - 1) / sxy, (H - 1) / sxy, 255.0 / srgb, 255.0 / srgb, 255.0 / srgb};
  int shift = 0;
  for (int i = 0; i < d; ++i) {
    // el[i] = sum_{k >= i} s_k f_k - i s_{i-1} f_{i-1}   (el[0] = sum_k s_k f_k)
    double lo = 0.0, hi = 0.0;
    for (int k = i; k < d; ++k) hi += sc.s[k] * fmax[k];
    if (i > 0) lo -= i * sc.s[i - 1] * fmax[i - 1];
    const double margin = 4.0 * (d + 1) + 2.0;
    const double fa = std::floor(lo - margin), fb = std::ceil(hi + margin);
    if (!(fa >= -kRange && fb <= kRange)) {
      const double span = fb - fa + 1.0;
      shift += std::isfinite(span) ? std::max(53, static_cast<int>(std::ceil(std::log2(span)))) : 1024;
      pk->off[i] = 0;
      pk->shift[i] = 0;
      pk->bits[i] = 1;
      continue;
    }
    const long long a = static_cast<long long>(fa), b = static_cast<long long>(fb);
    const unsigned long long span = static_cast<unsigned long long>(b - a + 1);
    int bits = 1;
    while (bits < 63 && (1ull << bits) < span) ++bits;
    pk->off[i] = -a;
    pk->shift[i] = shift < 64 ? shift : 63;
    pk->bits[i] = bits;
    shift += bits;
  }
  return shift;
}

struct Carve {
  char* base;
  size_t off;
  template <typename T>
  T* take(size_t n) {
    off = (off + 255) & ~static_cast<size_t>(255);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
};

struct Scratch {
  u64* key64;
  unsigned* lo;
  unsigned* alt_k;
  unsigned* alt_v;
  unsigned* tiles;
  void* sort_ws;
};

// The lattice buffer: int V[2] (smoothness, appearance), both lattices at their worst case V = N (d+1), then the
// build's scratch sized for d = 5. Returns the byte size.
size_t carve_lattice(void* base, int H, int W, int** V, Lattice* ls, Lattice* la, Scratch* sc) {
  const size_t N = static_cast<size_t>(H) * W;
  Carve cv{static_cast<char*>(base), 0};
  *V = cv.take<int>(2);
  Lattice* lats[2] = {ls, la};
  const int ds[2] = {2, 5};
  for (int k = 0; k < 2; ++k) {
    const size_t L = N * (ds[k] + 1);
    Lattice& l = *lats[k];
    l.w = cv.take<float>(L);
    l.vid = cv.take<int>(L);
    l.idx = cv.take<unsigned>(L);
    l.run = cv.take<int>(L + 1);
    l.nbr = cv.take<int>(L * (ds[k] + 1) * 2);
    l.vkey = cv.take<u64>(L);
    l.norm = cv.take<float>(N);
  }
  const size_t L5 = N * 6;
  sc->key64 = cv.take<u64>(L5);
  sc->lo = cv.take<unsigned>(L5);
  sc->alt_k = cv.take<unsigned>(L5);
  sc->alt_v = cv.take<unsigned>(L5);
  sc->tiles = cv.take<unsigned>((L5 + kDcrfTile - 1) / kDcrfTile);
  sc->sort_ws = cv.take<char>(static_cast<size_t>(semseg_segsort_u32_pairs_workspace_bytes(1, static_cast<long long>(L5))));
  return cv.off;
}

bool bad_std(double s) { return !(std::isfinite(s) && s > 0.0); }

int check_image(const char* fn, int H, int W) {
  SB_CHECK_ARG(H > 0 && W > 0, "%s: empty image %dx%d", fn, H, W);
  SB_CHECK_ARG(static_cast<long long>(H) * W * 6 < (1LL << 31), "%s: image %dx%d too large (N*6 >= 2^31)", fn, H, W);
  return SEMSEG_OK;
}

int check_stds(const char* fn, int H, int W, double pos_xy_std, double bi_xy_std, double bi_rgb_std, KeyPack* ps,
               KeyPack* pa) {
  SB_CHECK_ARG(!bad_std(pos_xy_std) && !bad_std(bi_xy_std) && !bad_std(bi_rgb_std),
               "%s: standard deviations must be finite and positive (pos_xy_std=%g bi_xy_std=%g bi_rgb_std=%g)", fn,
               pos_xy_std, bi_xy_std, bi_rgb_std);
  const int bs = key_layout(2, H, W, pos_xy_std, 1.0, ps);
  const int ba = key_layout(5, H, W, bi_xy_std, bi_rgb_std, pa);
  SB_CHECK_ARG(bs <= 64 && ba <= 64, "%s: lattice keys need %d (smoothness) and %d (appearance) bits, more than 64",
               fn, bs, ba);
  return SEMSEG_OK;
}

int check_V(const char* fn, int H, int W, int Vs, int Va) {
  const long long N = static_cast<long long>(H) * W;
  SB_CHECK_ARG(Vs >= 1 && Vs <= 3 * N && Va >= 1 && Va <= 6 * N, "%s: vertex counts Vs=%d Va=%d out of range", fn, Vs,
               Va);
  return SEMSEG_OK;
}

template <int D>
int build_one(const float* image, int H, int W, double sxy, double srgb, const KeyPack& pk, const Lattice& l,
              const Scratch& sc, int* Vdev, cudaStream_t stream) {
  const int N = H * W, L = N * (D + 1);
  dcrf_keys_kernel<D><<<grid_for(N), kDcrfThreads, 0, stream>>>(image, H, W, sxy, srgb, scales_for(D), pk, sc.key64,
                                                               sc.lo, l.idx, l.w);
  SB_LAUNCHED();
  int r = semseg_segsort_u32_pairs(sc.lo, l.idx, sc.alt_k, sc.alt_v, 1, L, nullptr, sc.sort_ws, stream);
  if (r) return r;
  dcrf_gather_hi_kernel<<<grid_for(L), kDcrfThreads, 0, stream>>>(sc.key64, l.idx, L, sc.lo);
  SB_LAUNCHED();
  r = semseg_segsort_u32_pairs(sc.lo, l.idx, sc.alt_k, sc.alt_v, 1, L, nullptr, sc.sort_ws, stream);
  if (r) return r;
  const int nt = cdiv(L, kDcrfTile);
  dcrf_unique_count_kernel<<<nt, kDcrfThreads, 0, stream>>>(sc.key64, l.idx, L, sc.tiles);
  SB_LAUNCHED();
  dcrf_scan_tiles_kernel<<<1, kDcrfScanThreads, 0, stream>>>(sc.tiles, nt, L, Vdev, l.run);
  SB_LAUNCHED();
  dcrf_unique_write_kernel<<<nt, kDcrfThreads, 0, stream>>>(sc.key64, l.idx, L, sc.tiles, l.vid, l.run, l.vkey);
  SB_LAUNCHED();
  dcrf_neighbours_kernel<D><<<grid_for(L), kDcrfThreads, 0, stream>>>(l.vkey, Vdev, L, pk, l.nbr);
  SB_LAUNCHED();
  // n = (K 1 + 1e-20)^-1/2, with the sort's scratch as the blur's ping-pong buffers
  float* a = reinterpret_cast<float*>(sc.lo);
  float* b = reinterpret_cast<float*>(sc.alt_k);
  dcrf_splat_kernel<D><<<grid_for(L), kDcrfThreads, 0, stream>>>(l.idx, l.run, l.w, nullptr, nullptr, 1, Vdev, L, a);
  SB_LAUNCHED();
  for (int j = 0; j <= D; ++j) {
    dcrf_blur_kernel<D><<<grid_for(L), kDcrfThreads, 0, stream>>>(l.nbr, j, 1, Vdev, L, a, b);
    SB_LAUNCHED();
    std::swap(a, b);
  }
  dcrf_slice_kernel<D><<<grid_for(N), kDcrfThreads, 0, stream>>>(l.vid, l.w, a, Vdev, L, N, 1, nullptr, 1, l.norm);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// The normalised filter's lattice part: lat_out = blur(splat(norm * in)); returns the buffer holding the result.
template <int D>
int filter_lattice(const Lattice& l, const int* Vdev, int V, const float* in, int C, float* a, float* b, float** res,
                   cudaStream_t stream) {
  const long long VC = static_cast<long long>(V) * C;
  dcrf_splat_kernel<D><<<grid_for(VC), kDcrfThreads, 0, stream>>>(l.idx, l.run, l.w, l.norm, in, C, Vdev, V, a);
  SB_LAUNCHED();
  for (int j = 0; j <= D; ++j) {
    dcrf_blur_kernel<D><<<grid_for(VC), kDcrfThreads, 0, stream>>>(l.nbr, j, C, Vdev, V, a, b);
    SB_LAUNCHED();
    std::swap(a, b);
  }
  *res = a;
  return SEMSEG_OK;
}

}  // namespace
}  // namespace sb

using namespace sb;

extern "C" long long semseg_densecrf_lattice_bytes(int H, int W) {
  int r = check_image("densecrf_lattice_bytes", H, W);
  if (r) return r;
  int* V;
  Lattice ls, la;
  Scratch sc;
  return static_cast<long long>(carve_lattice(nullptr, H, W, &V, &ls, &la, &sc));
}

extern "C" int semseg_densecrf_build(const float* image, int H, int W, double pos_xy_std, double bi_xy_std,
                                     double bi_rgb_std, void* lattice, void* stream_) {
  int r = check_image("densecrf_build", H, W);
  if (r) return r;
  KeyPack ps, pa;
  r = check_stds("densecrf_build", H, W, pos_xy_std, bi_xy_std, bi_rgb_std, &ps, &pa);
  if (r) return r;
  SB_CHECK_ARG(image && lattice, "densecrf_build: null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int* V;
  Lattice ls, la;
  Scratch sc;
  carve_lattice(lattice, H, W, &V, &ls, &la, &sc);
  r = build_one<2>(image, H, W, pos_xy_std, 1.0, ps, ls, sc, V, stream);
  if (r) return r;
  return build_one<5>(image, H, W, bi_xy_std, bi_rgb_std, pa, la, sc, V + 1, stream);
}

extern "C" long long semseg_densecrf_values_floats(int H, int W, int Vs, int Va, int C) {
  int r = check_image("densecrf_values_floats", H, W);
  if (r) return r;
  r = check_V("densecrf_values_floats", H, W, Vs, Va);
  if (r) return r;
  SB_CHECK_ARG(C >= 1, "densecrf_values_floats: C=%d", C);
  return 2LL * (static_cast<long long>(Vs) + Va) * C;
}

extern "C" int semseg_densecrf_filter(const void* lattice, int H, int W, int Vs, int Va, int kernel, const float* in,
                                      int C, float* values, float* out, void* stream_) {
  int r = check_image("densecrf_filter", H, W);
  if (r) return r;
  r = check_V("densecrf_filter", H, W, Vs, Va);
  if (r) return r;
  SB_CHECK_ARG(kernel == 0 || kernel == 1, "densecrf_filter: kernel %d (0 = smoothness, 1 = appearance)", kernel);
  SB_CHECK_ARG(C >= 1, "densecrf_filter: C=%d", C);
  SB_CHECK_ARG(lattice && in && values && out, "densecrf_filter: null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int* V;
  Lattice ls, la;
  Scratch sc;
  carve_lattice(const_cast<void*>(lattice), H, W, &V, &ls, &la, &sc);
  const int N = H * W;
  float* res;
  if (kernel == 0) {
    float* a = values;
    r = filter_lattice<2>(ls, V, Vs, in, C, a, a + static_cast<size_t>(Vs) * C, &res, stream);
    if (r) return r;
    dcrf_slice_kernel<2><<<grid_for(static_cast<long long>(N) * C), kDcrfThreads, 0, stream>>>(
        ls.vid, ls.w, res, V, Vs, N, C, ls.norm, 0, out);
  } else {
    float* a = values + 2 * static_cast<size_t>(Vs) * C;
    r = filter_lattice<5>(la, V + 1, Va, in, C, a, a + static_cast<size_t>(Va) * C, &res, stream);
    if (r) return r;
    dcrf_slice_kernel<5><<<grid_for(static_cast<long long>(N) * C), kDcrfThreads, 0, stream>>>(
        la.vid, la.w, res, V + 1, Va, N, C, la.norm, 0, out);
  }
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_densecrf_meanfield(const void* lattice, int H, int W, int Vs, int Va, const float* prob, int C,
                                         double clip, int iterations, double pos_weight, double bi_weight,
                                         float* values, float* Q, void* stream_) {
  int r = check_image("densecrf_meanfield", H, W);
  if (r) return r;
  r = check_V("densecrf_meanfield", H, W, Vs, Va);
  if (r) return r;
  SB_CHECK_ARG(C >= 1, "densecrf_meanfield: C=%d", C);
  SB_CHECK_ARG(iterations >= 0, "densecrf_meanfield: iterations=%d must be >= 0", iterations);
  SB_CHECK_ARG(clip >= static_cast<double>(FLT_MIN) && clip < 1.0,
               "densecrf_meanfield: clip=%g must lie in [FLT_MIN, 1) (the update takes log max(p, clip) in fp32)", clip);
  SB_CHECK_ARG(std::isfinite(pos_weight) && pos_weight >= 0.0 && std::isfinite(bi_weight) && bi_weight >= 0.0,
               "densecrf_meanfield: weights must be finite and non-negative (pos_weight=%g bi_weight=%g)", pos_weight,
               bi_weight);
  SB_CHECK_ARG(lattice && prob && values && Q, "densecrf_meanfield: null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int* V;
  Lattice ls, la;
  Scratch sc;
  carve_lattice(const_cast<void*>(lattice), H, W, &V, &ls, &la, &sc);
  const int N = H * W;
  const int update_grid = static_cast<int>(std::min<long long>(cdiv(N, kDcrfThreads / 32), kDcrfMaxBlocks));
  Message none{nullptr, nullptr, nullptr, nullptr, 0, 0.f};
  dcrf_update_kernel<<<update_grid, kDcrfThreads, 0, stream>>>(prob, N, C, static_cast<float>(clip), none, none, Q);
  SB_LAUNCHED();
  float* vs = values;
  float* va = values + 2 * static_cast<size_t>(Vs) * C;
  for (int it = 0; it < iterations; ++it) {
    Message ms = none, ma = none;
    if (pos_weight > 0.0) {
      float* res;
      r = filter_lattice<2>(ls, V, Vs, Q, C, vs, vs + static_cast<size_t>(Vs) * C, &res, stream);
      if (r) return r;
      ms = Message{ls.vid, ls.w, ls.norm, res, Vs, static_cast<float>(pos_weight)};
    }
    if (bi_weight > 0.0) {
      float* res;
      r = filter_lattice<5>(la, V + 1, Va, Q, C, va, va + static_cast<size_t>(Va) * C, &res, stream);
      if (r) return r;
      ma = Message{la.vid, la.w, la.norm, res, Va, static_cast<float>(bi_weight)};
    }
    dcrf_update_kernel<<<update_grid, kDcrfThreads, 0, stream>>>(prob, N, C, static_cast<float>(clip), ms, ma, Q);
    SB_LAUNCHED();
  }
  return SEMSEG_OK;
}

extern "C" int semseg_densecrf_keys(const void* lattice, int H, int W, int Vs, int Va, int kernel, double pos_xy_std,
                                    double bi_xy_std, double bi_rgb_std, int* out, void* stream_) {
  int r = check_image("densecrf_keys", H, W);
  if (r) return r;
  KeyPack ps, pa;
  r = check_stds("densecrf_keys", H, W, pos_xy_std, bi_xy_std, bi_rgb_std, &ps, &pa);
  if (r) return r;
  r = check_V("densecrf_keys", H, W, Vs, Va);
  if (r) return r;
  SB_CHECK_ARG(kernel == 0 || kernel == 1, "densecrf_keys: kernel %d (0 = smoothness, 1 = appearance)", kernel);
  SB_CHECK_ARG(lattice && out, "densecrf_keys: null pointer");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int* V;
  Lattice ls, la;
  Scratch sc;
  carve_lattice(const_cast<void*>(lattice), H, W, &V, &ls, &la, &sc);
  if (kernel == 0) dcrf_unpack_kernel<2><<<grid_for(Vs), kDcrfThreads, 0, stream>>>(ls.vkey, V, Vs, ps, out);
  else dcrf_unpack_kernel<5><<<grid_for(Va), kDcrfThreads, 0, stream>>>(la.vkey, V + 1, Va, pa, out);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// BatchNorm (training statistics, apply, backward), ReLU and residual kernels on NHWC bf16 tensors.
// All statistics are fp32; per-tile / per-chunk partials are merged with Chan's parallel-variance
// formula in a fixed order, so results are run-to-run deterministic.
// Mirrors nn.BatchNorm2d / nn.SyncBatchNorm + ReLU + residual add as used at model/resnet.py:77-92
// (biased variance for normalisation, unbiased for running_var, eps 1e-5, momentum 0.1).
#include <initializer_list>

#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

struct Moments {
  float n, mean, m2;
};
__device__ __forceinline__ Moments merge(const Moments& a, const Moments& b) {
  if (b.n == 0.f) return a;
  if (a.n == 0.f) return b;
  Moments r;
  r.n = a.n + b.n;
  const float d = b.mean - a.mean;
  r.mean = a.mean + d * (b.n / r.n);
  r.m2 = a.m2 + b.m2 + d * d * (a.n * b.n / r.n);
  return r;
}

// The conv epilogue's statistics buffer is [rows][3][C] = (sum, sum of squares, count) per epilogue warp.

// Block-wide merge of the conv statistics rows for CH channels starting at c0. A block is 1024 threads = CH channels x
// (1024 / CH) row lanes; narrow channel groups (CH = 8) spread a layer over more blocks / SMs, which is what bounds this
// kernel (each block pulls rows * 3 * CH floats out of L2). Every thread issues all of its row loads (up to 8 rows = 24
// loads) before the first add; raw (sum, sum of squares, count) are added over a thread's rows and over the row lanes of
// its warp (butterfly), converted once to (mean, M2, n) and the 32 warps are merged with Chan's formula by a shuffle tree.
// Result: valid in lane 0 of warp w < CH for channel c0 + w.
template <int CH>
__device__ __forceinline__ Moments block_conv_moments(const float* __restrict__ part, int T, int C, int c0,
                                                      Moments (*sm)[CH + 1]) {
  constexpr int RL = 1024 / CH;  // row lanes per block
  constexpr int U = 8;
  const int cl = threadIdx.x % CH;
  const int rl = threadIdx.x / CH;
  const int c = c0 + cl;
  float S = 0.f, Q = 0.f, n = 0.f;
  if (c < C) {
    for (int t0 = rl; t0 < T; t0 += RL * U) {
      float s[U], q[U], m[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = t0 + RL * u;
        const bool ok = t < T;
        const float* row = part + static_cast<size_t>(ok ? t : 0) * 3 * C;
        s[u] = ok ? row[c] : 0.f;
        q[u] = ok ? row[C + c] : 0.f;
        m[u] = ok ? row[2 * C + c] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        S += s[u];
        Q += q[u];
        n += m[u];
      }
    }
  }
#pragma unroll
  for (int o = CH; o < 32; o <<= 1) {  // lanes cl, cl + CH, ... of a warp hold the same channel
    S += __shfl_xor_sync(0xffffffffu, S, o);
    Q += __shfl_xor_sync(0xffffffffu, Q, o);
    n += __shfl_xor_sync(0xffffffffu, n, o);
  }
  Moments acc = {0.f, 0.f, 0.f};
  if (n > 0.f) {
    acc.n = n;
    acc.mean = S / n;
    acc.m2 = fmaxf(Q - S * acc.mean, 0.f);
  }
  if ((threadIdx.x & 31) < CH) sm[threadIdx.x >> 5][cl] = acc;
  __syncthreads();
  // warp w (< CH) merges channel c0 + w: lane i holds warp i's partial, 5-step shuffle tree in a fixed order
  Moments r = {0.f, 0.f, 0.f};
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (w < CH) {
    r = sm[lane][w];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      Moments other;
      other.mean = __shfl_down_sync(0xffffffffu, r.mean, o);
      other.m2 = __shfl_down_sync(0xffffffffu, r.m2, o);
      other.n = __shfl_down_sync(0xffffffffu, r.n, o);
      r = merge(r, other);
    }
  }
  return r;  // valid in lane 0 of warps 0..CH-1
}

// Channels per block such that a layer needs at most 128 blocks (one wave). The peer exchange does not rely on that:
// its blocks only wait for words the peers push, which needs none of this GPU's SMs (st_ll / ld_ll below).
static int stats_group_channels(int C) { return C <= 1024 ? 8 : (C <= 2048 ? 16 : 32); }

// Launch helper: KERNEL<kCH> with kCH = stats_group_channels(C) channels per block.
#define SB_STATS_GROUP_DISPATCH(C, ...)  \
  do {                                   \
    switch (stats_group_channels(C)) {   \
      case 8: {                          \
        constexpr int kCH = 8;           \
        __VA_ARGS__;                     \
      } break;                           \
      case 16: {                         \
        constexpr int kCH = 16;          \
        __VA_ARGS__;                     \
      } break;                           \
      default: {                         \
        constexpr int kCH = 32;          \
        __VA_ARGS__;                     \
      } break;                           \
    }                                    \
  } while (0)

template <int CH>
__global__ void __launch_bounds__(1024) bn_merge_conv_partials_kernel(const float* __restrict__ part, int T, int C,
                                                                      float* __restrict__ out) {
  __shared__ Moments sm[32][CH + 1];
  const Moments r = block_conv_moments<CH>(part, T, C, blockIdx.x * CH, sm);
  const int c = blockIdx.x * CH + (threadIdx.x >> 5);
  if ((threadIdx.x & 31) == 0 && (threadIdx.x >> 5) < CH && c < C) {
    out[c] = r.mean;
    out[C + c] = r.m2;
    out[2 * C + c] = r.n;
  }
}

// ------------------------------------------------------------------------------------------------
// SyncBatchNorm statistics exchange over NVLink peer memory (torch symmetric memory): fused into the finalise and the
// backward's final reduction (their PEER form), no NCCL call, no stream hop; the protocol is described at st_ll / ld_ll
// below. The cross-rank merge is done in rank order on every rank, so all ranks compute bit-identical statistics.
// Kernels take it as a `const __grid_constant__` parameter: buf[p] with a run-time p is then read from the parameter
// bank instead of from a copy of the whole struct in local memory.
struct PeerArgs {
  float* buf[8];        // peer-mapped data buffers (buf[rank] is local): 8-byte {value, seq} words, [slot][src rank][slot_floats]
  int world, rank, slot, slot_floats;
  const unsigned* seq_ptr;  // device-resident step counter = the sequence number of this exchange (read at run time, so
                            // a captured CUDA graph with the slot baked in can be replayed)
  long long timeout_ticks;
};

// Exchange protocol ("LL", flag-in-data): a value travels as ONE 8-byte word {fp32 bits, sequence number}. The sender
// stores the word straight into sub-block `rank` of the slot in EVERY peer's buffer (posted NVLink stores); the receiver
// polls the word in its OWN memory until the sequence number matches. 8-byte stores are single transactions, so there is
// no separate flag, no system-scope fence, no cross-block counter: every thread that finishes a channel exchanges that
// channel on its own, the latency is one NVLink store, and a block only ever waits for data that peers push without
// needing any of this GPU's SMs (no co-residency requirement, nothing an NCCL kernel sharing the SMs can dead-lock with).
// A peer that never arrives trips the watchdog (default 10 minutes, SEMSEG_B200_P2P_TIMEOUT_S) instead of hanging the GPU.
__device__ __forceinline__ void st_ll(unsigned long long* p, float v, unsigned seq) {
  const unsigned long long w = (static_cast<unsigned long long>(seq) << 32) | __float_as_uint(v);
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ float ld_ll(const unsigned long long* p, unsigned seq, const PeerArgs& pa, int peer) {
  unsigned long long w;
  const long long t0 = clock64();
  for (;;) {
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
    if (static_cast<unsigned>(w >> 32) == seq) break;
    if (clock64() - t0 > pa.timeout_ticks) {
      printf("semseg_b200: SyncBN peer exchange timed out (rank %d waiting for rank %d, slot %d, seq %u)\n", pa.rank, peer,
             pa.slot, seq);
      __trap();
    }
  }
  return __uint_as_float(static_cast<unsigned>(w & 0xffffffffu));
}

// Finalise channel c from its moments over all ranks: mean_invstd [3][C] = (mean, invstd, samples per channel over all
// ranks — the backward's 1/count), scale_shift [2][C] = (gamma*invstd, beta - mean*scale), and the running statistics
// (momentum, unbiased variance) when given. Every finalise kernel ends here, so equal moments give equal bits.
__device__ __forceinline__ void finalize_channel(const Moments& r, int c, int C, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, float eps, float momentum,
                                                 float* __restrict__ running_mean, float* __restrict__ running_var,
                                                 float* __restrict__ mean_invstd, float* __restrict__ scale_shift) {
  const float var = r.n > 0.f ? r.m2 / r.n : 0.f;
  const float invstd = rsqrtf(var + eps);
  mean_invstd[c] = r.mean;
  mean_invstd[C + c] = invstd;
  mean_invstd[2 * C + c] = r.n;
  const float sc = (gamma ? gamma[c] : 1.f) * invstd;
  scale_shift[c] = sc;
  scale_shift[C + c] = (beta ? beta[c] : 0.f) - r.mean * sc;
  if (running_mean) running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * r.mean;
  if (running_var) {
    const float unb = r.n > 1.f ? r.m2 / (r.n - 1.f) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unb;
  }
}

// Merge this rank's conv partials and finalise in one launch. PEER: exchange the channel's (mean, M2, n) with every
// rank and merge the ranks' moments in rank order before finalising.
template <int CH, bool PEER>
__global__ void __launch_bounds__(1024) bn_finalize_partials_kernel(const float* __restrict__ part, int T, int C,
                                            const float* __restrict__ gamma, const float* __restrict__ beta,
                                            float eps, float momentum, float* __restrict__ running_mean,
                                            float* __restrict__ running_var, float* __restrict__ mean_invstd,
                                            float* __restrict__ scale_shift, const __grid_constant__ PeerArgs pa) {
  __shared__ Moments sm[32][CH + 1];
  Moments r = block_conv_moments<CH>(part, T, C, blockIdx.x * CH, sm);
  const int c = blockIdx.x * CH + (threadIdx.x >> 5);
  if (!((threadIdx.x & 31) == 0 && (threadIdx.x >> 5) < CH && c < C)) return;   // this thread finishes channel c
  if constexpr (PEER) {
    const unsigned seq = *pa.seq_ptr;
    const size_t slot0 = static_cast<size_t>(pa.slot) * pa.world * pa.slot_floats;
    const size_t off = slot0 + static_cast<size_t>(pa.rank) * pa.slot_floats;
    for (int p = 0; p < pa.world; ++p) {
      unsigned long long* dst = reinterpret_cast<unsigned long long*>(pa.buf[p]) + off;
      st_ll(dst + c, r.mean, seq);
      st_ll(dst + C + c, r.m2, seq);
      st_ll(dst + 2 * C + c, r.n, seq);
    }
    r = Moments{0.f, 0.f, 0.f};
    for (int p = 0; p < pa.world; ++p) {
      const unsigned long long* b = reinterpret_cast<const unsigned long long*>(pa.buf[pa.rank]) + slot0 +
                                    static_cast<size_t>(p) * pa.slot_floats;
      Moments m;
      m.mean = ld_ll(b + c, seq, pa, p);
      m.m2 = ld_ll(b + C + c, seq, pa, p);
      m.n = ld_ll(b + 2 * C + c, seq, pa, p);
      r = merge(r, m);
    }
  }
  finalize_channel(r, c, C, gamma, beta, eps, momentum, running_mean, running_var, mean_invstd, scale_shift);
}

// NCCL form: rank_stats [R][3][C] (every rank's merged conv partials, gathered) -> merged in rank order, finalised.
__global__ void bn_finalize_kernel(const float* __restrict__ rs, int R, int C, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum,
                                   float* __restrict__ running_mean, float* __restrict__ running_var,
                                   float* __restrict__ mean_invstd, float* __restrict__ scale_shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  Moments acc = {0.f, 0.f, 0.f};
  for (int r = 0; r < R; ++r) {
    const float* b = rs + static_cast<size_t>(r) * 3 * C;
    Moments m;
    m.mean = b[c];
    m.m2 = b[C + c];
    m.n = b[2 * C + c];
    acc = merge(acc, m);
  }
  finalize_channel(acc, c, C, gamma, beta, eps, momentum, running_mean, running_var, mean_invstd, scale_shift);
}

// Running-statistics folding of channel c: invstd, scale = gamma*invstd, shift = beta - mean*scale. Shared by the eval
// fold and the frozen-BN backward, so that the backward's ReLU mask fma(raw, scale, shift) > 0 sees the forward's bits.
__device__ __forceinline__ void fold_running(const float* __restrict__ gamma, const float* __restrict__ beta,
                                             const float* __restrict__ rm, const float* __restrict__ rv, float eps, int c,
                                             float& invstd, float& sc, float& sh) {
  invstd = rsqrtf(rv[c] + eps);
  sc = (gamma ? gamma[c] : 1.f) * invstd;
  sh = (beta ? beta[c] : 0.f) - rm[c] * sc;
}

__global__ void bn_fold_eval_kernel(const float* __restrict__ gamma, const float* __restrict__ beta,
                                    const float* __restrict__ rm, const float* __restrict__ rv, float eps, int C,
                                    float* __restrict__ scale_shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float invstd, sc, sh;
  fold_running(gamma, beta, rm, rv, eps, c, invstd, sc, sh);
  scale_shift[c] = sc;
  scale_shift[C + c] = sh;
}

// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float2 t = __bfloat1622float2(h[q]);
    f[2 * q] = t.x;
    f[2 * q + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  return o;
}

// Grid sizing guarantees (gridDim.x * blockDim.x) % (C/8) == 0, so a thread keeps the same 8 channels for its
// whole grid-stride loop and the per-channel coefficients are loaded once.
template <bool S>
__global__ void bn_apply_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo, int x_pitch,
                                const float* __restrict__ ss, const __nv_bfloat16* __restrict__ res,
                                const __nv_bfloat16* __restrict__ res_lo, int res_pitch, __nv_bfloat16* __restrict__ y,
                                __nv_bfloat16* __restrict__ y_lo, int y_pitch, long long M, int C, int relu) {
  const int groups = C >> 3;
  long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const int c0 = static_cast<int>(idx % groups) << 3;
  float sc[8], sh[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    sc[q] = ss[c0 + q];
    sh[q] = ss[C + c0 + q];
  }
  // stride is a multiple of groups, so pixel p advances by pstride each iteration; 4 pixels are kept in flight.
  const long long pstride = stride / groups;
  long long p = idx / groups;
  constexpr int U = 4;
  for (; p + (U - 1) * pstride < M; p += U * pstride) {
    Raw8<S> xv[U], rv[U];
#pragma unroll
    for (int u = 0; u < U; ++u) xv[u] = act_ldraw<S>(x, x_lo, (p + u * pstride) * x_pitch + c0);
    if (res) {
#pragma unroll
      for (int u = 0; u < U; ++u) rv[u] = act_ldraw<S>(res, res_lo, (p + u * pstride) * res_pitch + c0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float f[8], r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      act_unpack<S>(xv[u], f);
      if (res) act_unpack<S>(rv[u], r);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        float v = fmaf(f[q], sc[q], sh[q]) + r[q];
        if (relu) v = fmaxf(v, 0.f);
        f[q] = v;
      }
      act_st8<S>(y, y_lo, (p + u * pstride) * y_pitch + c0, f);
    }
  }
  for (; p < M; p += pstride) {
    float f[8], r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    act_ld8<S>(x, x_lo, p * x_pitch + c0, f);
    if (res) act_ld8<S>(res, res_lo, p * res_pitch + c0, r);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float v = fmaf(f[q], sc[q], sh[q]) + r[q];
      if (relu) v = fmaxf(v, 0.f);
      f[q] = v;
    }
    act_st8<S>(y, y_lo, p * y_pitch + c0, f);
  }
}

// Backward reduce, stage 1: per-chunk sums of dz and dz*xhat. block = 8 groups x 32 pixel lanes.
template <bool S>
__global__ void bn_bwd_reduce_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dy_lo,
                                     int dy_pitch, const __nv_bfloat16* __restrict__ y,
                                     const __nv_bfloat16* __restrict__ y_lo, int y_pitch,
                                     const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo,
                                     int x_pitch, const float* __restrict__ mean_invstd, const float* __restrict__ ss,
                                     int M, int C, int relu, int rows_per_chunk, float* __restrict__ part) {
  __shared__ float s_a[32][65];
  __shared__ float s_b[32][65];
  const int gl = threadIdx.x & 7;
  const int pl = threadIdx.x >> 3;
  const int c0 = blockIdx.x * 64 + gl * 8;
  const int chunk = blockIdx.y;
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(M, r0 + rows_per_chunk);
  const bool active = c0 < C;
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (active) {
    float mean[8], invstd[8], msc[8], msh[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      mean[q] = mean_invstd[c0 + q];
      invstd[q] = mean_invstd[C + c0 + q];
      msc[q] = ss ? ss[c0 + q] : 0.f;       // ReLU mask recomputed from the raw conv output when y is not given:
      msh[q] = ss ? ss[C + c0 + q] : 0.f;   // y > 0  <=>  fma(x, scale, shift) > 0 (same fma as bn_apply, no residual)
    }
    const bool mask_from_y = relu && y != nullptr;
    const bool mask_from_x = relu && y == nullptr;
    constexpr int U = S ? 2 : 4;  // rows in flight per thread
    auto accumulate = [&](float (&d)[8], const float (&xv)[8], const float (&yv)[8]) {
      if (mask_from_y) {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (!(yv[q] > 0.f)) d[q] = 0.f;
      } else if (mask_from_x) {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (!(fmaf(xv[q], msc[q], msh[q]) > 0.f)) d[q] = 0.f;
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        a[q] += d[q];
        b[q] = fmaf(d[q], (xv[q] - mean[q]) * invstd[q], b[q]);
      }
    };
    int r = r0 + pl;
    for (; r + (U - 1) * 32 < r1; r += U * 32) {
      Raw8<S> dv[U], xr[U], yr[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        dv[u] = act_ldraw<S>(dy, dy_lo, static_cast<long long>(r + u * 32) * dy_pitch + c0);
        xr[u] = act_ldraw<S>(x, x_lo, static_cast<long long>(r + u * 32) * x_pitch + c0);
      }
      if (mask_from_y) {
#pragma unroll
        for (int u = 0; u < U; ++u) yr[u] = act_ldraw<S>(y, y_lo, static_cast<long long>(r + u * 32) * y_pitch + c0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float d[8], xv[8], yv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        act_unpack<S>(dv[u], d);
        act_unpack<S>(xr[u], xv);
        if (mask_from_y) act_unpack<S>(yr[u], yv);
        accumulate(d, xv, yv);
      }
    }
    for (; r < r1; r += 32) {
      float d[8], xv[8], yv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      act_ld8<S>(dy, dy_lo, static_cast<long long>(r) * dy_pitch + c0, d);
      act_ld8<S>(x, x_lo, static_cast<long long>(r) * x_pitch + c0, xv);
      if (mask_from_y) act_ld8<S>(y, y_lo, static_cast<long long>(r) * y_pitch + c0, yv);
      accumulate(d, xv, yv);
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    s_a[pl][gl * 8 + q] = a[q];
    s_b[pl][gl * 8 + q] = b[q];
  }
  __syncthreads();
  if (pl < 2 && active) {
    // pl 0 reduces the dz sums, pl 1 the dz*xhat sums
    float(*src)[65] = pl == 0 ? s_a : s_b;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float t = 0.f;
      for (int i = 0; i < 32; ++i) t += src[i][gl * 8 + q];
      if (c0 + q < C) part[(static_cast<size_t>(chunk) * 2 + pl) * C + c0 + q] = t;
    }
  }
}

// stage 2: sums[2][C] = sum over chunks (fixed order). PEER: also exchange this rank's sums with every rank and add
// them in rank order into sums_total[2][C] (sums, the local ones, feed dgamma/dbeta, which DDP averages later).
template <bool PEER>
__global__ void __launch_bounds__(1024) bn_bwd_reduce_final_kernel(const float* __restrict__ part, int chunks, int C,
                                           float* __restrict__ sums, float* __restrict__ sums_total,
                                           const __grid_constant__ PeerArgs pa) {
  __shared__ float sm[32][33];
  const int cl = threadIdx.x & 31;
  const int tl = threadIdx.x >> 5;
  const int idx = blockIdx.x * 32 + cl;  // over 2*C: [which][c]
  float acc = 0.f;
  if (idx < 2 * C) {
    const int which = idx / C, c = idx - which * C;
    constexpr int U = 8;
    for (int t0 = tl; t0 < chunks; t0 += 32 * U) {
      float v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int t = t0 + 32 * u;
        v[u] = t < chunks ? part[(static_cast<size_t>(t) * 2 + which) * C + c] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) acc += v[u];
    }
  }
  sm[tl][cl] = acc;
  __syncthreads();
  if (!(tl == 0 && idx < 2 * C)) return;
  float own = 0.f;
  for (int i = 0; i < 32; ++i) own += sm[i][cl];
  sums[idx] = own;
  if constexpr (PEER) {
    const unsigned seq = *pa.seq_ptr;
    const size_t slot0 = static_cast<size_t>(pa.slot) * pa.world * pa.slot_floats;
    const size_t off = slot0 + static_cast<size_t>(pa.rank) * pa.slot_floats + idx;
    for (int p = 0; p < pa.world; ++p) st_ll(reinterpret_cast<unsigned long long*>(pa.buf[p]) + off, own, seq);
    float r = 0.f;
    for (int p = 0; p < pa.world; ++p)
      r += ld_ll(reinterpret_cast<const unsigned long long*>(pa.buf[pa.rank]) + slot0 + static_cast<size_t>(p) * pa.slot_floats + idx,
                 seq, pa, p);
    sums_total[idx] = r;
  }
}

template <bool S>
__global__ void bn_bwd_apply_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dy_lo,
                                    int dy_pitch, const __nv_bfloat16* __restrict__ y,
                                    const __nv_bfloat16* __restrict__ y_lo, int y_pitch,
                                    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo,
                                    int x_pitch, const float* __restrict__ mean_invstd, const float* __restrict__ gamma,
                                    const float* __restrict__ ss, const float* __restrict__ sums, float inv_count,
                                    long long M, int C, int relu, __nv_bfloat16* __restrict__ dx,
                                    __nv_bfloat16* __restrict__ dx_lo, int dx_pitch, __nv_bfloat16* __restrict__ dres,
                                    __nv_bfloat16* __restrict__ dres_lo, int dres_pitch,
                                    float* __restrict__ dgamma_dbeta) {
  const int groups = C >> 3;
  if (dgamma_dbeta && blockIdx.x == 0) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      dgamma_dbeta[c] = sums[C + c];
      dgamma_dbeta[C + c] = sums[c];
    }
  }
  long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const int c0 = static_cast<int>(idx % groups) << 3;
  // dx = g*invstd*(dz - s1/M - xhat*s2/M) = ka*dz + kx*x + kb  with xhat = (x - mean)*invstd
  float ka[8], kx[8], kb[8], msc[8], msh[8];
  const bool mask_from_y = relu && y != nullptr;
  const bool mask_from_x = relu && y == nullptr;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int c = c0 + q;
    msc[q] = ss ? ss[c] : 0.f;
    msh[q] = ss ? ss[C + c] : 0.f;
    const float mean = mean_invstd[c], invstd = mean_invstd[C + c];
    const float g = gamma ? gamma[c] : 1.f;
    ka[q] = g * invstd;
    const float ic = inv_count > 0.f ? inv_count : 1.f / mean_invstd[2 * C + c];   // count <= 0: the exchanged total
    kx[q] = -ka[q] * invstd * sums[C + c] * ic;
    kb[q] = -ka[q] * sums[c] * ic - kx[q] * mean;
  }
  auto finish = [&](float (&d)[8], const float (&xv)[8], const float (&yv)[8], long long pp) {
    if (mask_from_y) {
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (!(yv[q] > 0.f)) d[q] = 0.f;
    } else if (mask_from_x) {
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (!(fmaf(xv[q], msc[q], msh[q]) > 0.f)) d[q] = 0.f;
    }
    if (dres) act_st8<S>(dres, dres_lo, pp * dres_pitch + c0, d);
    float o[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) o[q] = fmaf(ka[q], d[q], fmaf(kx[q], xv[q], kb[q]));
    act_st8<S>(dx, dx_lo, pp * dx_pitch + c0, o);
  };
  const long long pstride = stride / groups;
  long long p = idx / groups;
  constexpr int U = 2;
  for (; p + (U - 1) * pstride < M; p += U * pstride) {
    Raw8<S> dv[U], xr[U], yr[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      dv[u] = act_ldraw<S>(dy, dy_lo, (p + u * pstride) * dy_pitch + c0);
      xr[u] = act_ldraw<S>(x, x_lo, (p + u * pstride) * x_pitch + c0);
    }
    if (mask_from_y) {
#pragma unroll
      for (int u = 0; u < U; ++u) yr[u] = act_ldraw<S>(y, y_lo, (p + u * pstride) * y_pitch + c0);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float d[8], xv[8], yv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      act_unpack<S>(dv[u], d);
      act_unpack<S>(xr[u], xv);
      if (mask_from_y) act_unpack<S>(yr[u], yv);
      finish(d, xv, yv, p + u * pstride);
    }
  }
  for (; p < M; p += pstride) {
    float d[8], xv[8], yv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    act_ld8<S>(dy, dy_lo, p * dy_pitch + c0, d);
    act_ld8<S>(x, x_lo, p * x_pitch + c0, xv);
    if (mask_from_y) act_ld8<S>(y, y_lo, p * y_pitch + c0, yv);
    finish(d, xv, yv, p);
  }
}

// Frozen BatchNorm backward (eval-mode BN inside a network that trains): the forward normalised with the running
// statistics, so nothing global is needed before d_raw and the whole backward is ONE pass. With dz = dy * (y > 0 if relu):
//   d_raw = dz * scale, dres = dz (optional), and per-chunk partials of (sum dz, sum dz*xhat), xhat = (raw - mean)*invstd,
// in the bn_bwd_reduce workspace layout (bn_bwd_reduce_final_kernel finishes them in a fixed order). The ReLU mask comes
// from y, or — y == nullptr, forward without residual — from fma(raw, scale, shift) > 0 like bn_bwd_reduce_kernel.
// part == nullptr: no sums. raw == nullptr: the dz*xhat row is zero. block = 8 channel groups x 32 pixel lanes.
template <bool S>
__global__ void __launch_bounds__(256, 2)
bn_bwd_frozen_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ dy_lo, int dy_pitch,
                     const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ y_lo, int y_pitch,
                     const __nv_bfloat16* __restrict__ raw, const __nv_bfloat16* __restrict__ raw_lo, int raw_pitch,
                     const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ rm,
                     const float* __restrict__ rv, float eps, int M, int C, int relu, int rows_per_chunk,
                     __nv_bfloat16* __restrict__ d_raw, __nv_bfloat16* __restrict__ d_raw_lo, int d_raw_pitch,
                     __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dres_lo, int dres_pitch,
                     float* __restrict__ part) {
  __shared__ float s_a[32][65];
  __shared__ float s_b[32][65];
  const int gl = threadIdx.x & 7;
  const int pl = threadIdx.x >> 3;
  const int c0 = blockIdx.x * 64 + gl * 8;
  const int chunk = blockIdx.y;
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(M, r0 + rows_per_chunk);
  const bool active = c0 < C;
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (active) {
    float mean[8], invstd[8], sc[8], sh[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      fold_running(gamma, beta, rm, rv, eps, c0 + q, invstd[q], sc[q], sh[q]);
      mean[q] = rm[c0 + q];
    }
    const bool mask_from_y = relu && y != nullptr;
    const bool mask_from_x = relu && y == nullptr;
    const bool load_x = raw != nullptr && (mask_from_x || part != nullptr);
    constexpr int U = S ? 2 : 4;  // rows in flight per thread
    auto finish = [&](float (&d)[8], const float (&xv)[8], const float (&yv)[8], long long rr) {
      if (mask_from_y) {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (!(yv[q] > 0.f)) d[q] = 0.f;
      } else if (mask_from_x) {
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (!(fmaf(xv[q], sc[q], sh[q]) > 0.f)) d[q] = 0.f;
      }
      if (dres) act_st8<S>(dres, dres_lo, rr * dres_pitch + c0, d);
      float o[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        a[q] += d[q];
        if (load_x) b[q] = fmaf(d[q], (xv[q] - mean[q]) * invstd[q], b[q]);
        o[q] = d[q] * sc[q];
      }
      act_st8<S>(d_raw, d_raw_lo, rr * d_raw_pitch + c0, o);
    };
    int r = r0 + pl;
    for (; r + (U - 1) * 32 < r1; r += U * 32) {
      Raw8<S> dv[U], xr[U], yr[U];
#pragma unroll
      for (int u = 0; u < U; ++u) dv[u] = act_ldraw<S>(dy, dy_lo, static_cast<long long>(r + u * 32) * dy_pitch + c0);
      if (load_x) {
#pragma unroll
        for (int u = 0; u < U; ++u)
          xr[u] = act_ldraw<S>(raw, raw_lo, static_cast<long long>(r + u * 32) * raw_pitch + c0);
      }
      if (mask_from_y) {
#pragma unroll
        for (int u = 0; u < U; ++u) yr[u] = act_ldraw<S>(y, y_lo, static_cast<long long>(r + u * 32) * y_pitch + c0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float d[8], xv[8] = {0, 0, 0, 0, 0, 0, 0, 0}, yv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        act_unpack<S>(dv[u], d);
        if (load_x) act_unpack<S>(xr[u], xv);
        if (mask_from_y) act_unpack<S>(yr[u], yv);
        finish(d, xv, yv, r + u * 32);
      }
    }
    for (; r < r1; r += 32) {
      float d[8], xv[8] = {0, 0, 0, 0, 0, 0, 0, 0}, yv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      act_ld8<S>(dy, dy_lo, static_cast<long long>(r) * dy_pitch + c0, d);
      if (load_x) act_ld8<S>(raw, raw_lo, static_cast<long long>(r) * raw_pitch + c0, xv);
      if (mask_from_y) act_ld8<S>(y, y_lo, static_cast<long long>(r) * y_pitch + c0, yv);
      finish(d, xv, yv, r);
    }
  }
  if (part == nullptr) return;  // uniform over the grid: no thread is left waiting at the barrier
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    s_a[pl][gl * 8 + q] = a[q];
    s_b[pl][gl * 8 + q] = b[q];
  }
  __syncthreads();
  if (pl < 2 && active) {
    // pl 0 reduces the dz sums, pl 1 the dz*xhat sums (same order as bn_bwd_reduce_kernel)
    float(*src)[65] = pl == 0 ? s_a : s_b;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float t = 0.f;
      for (int i = 0; i < 32; ++i) t += src[i][gl * 8 + q];
      if (c0 + q < C) part[(static_cast<size_t>(chunk) * 2 + pl) * C + c0 + q] = t;
    }
  }
}

// out = a + b
template <bool S>
__global__ void add_act_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ a_lo, int a_pitch,
                               const __nv_bfloat16* __restrict__ b, const __nv_bfloat16* __restrict__ b_lo, int b_pitch,
                               __nv_bfloat16* __restrict__ out, __nv_bfloat16* __restrict__ out_lo, int out_pitch,
                               long long M, int C) {
  const int groups = C >> 3;
  const long long total = M * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int c0 = static_cast<int>(idx - p * groups) << 3;
    float x[8], z[8];
    act_ld8<S>(a, a_lo, p * a_pitch + c0, x);
    act_ld8<S>(b, b_lo, p * b_pitch + c0, z);
#pragma unroll
    for (int q = 0; q < 8; ++q) x[q] += z[q];
    act_st8<S>(out, out_lo, p * out_pitch + c0, x);
  }
}

// out[n, p, c] = x[n, p, c] * s[n, c]  (Dropout2d: one Bernoulli-derived factor per (image, channel)).
template <bool S>
__global__ void scale_nc_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo, int x_pitch,
                                const float* __restrict__ s, __nv_bfloat16* __restrict__ out,
                                __nv_bfloat16* __restrict__ out_lo, int out_pitch, int N, long long HW, int C) {
  const int groups = C >> 3;
  const long long total = static_cast<long long>(N) * HW * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int c0 = static_cast<int>(idx - p * groups) << 3;
    const int n = static_cast<int>(p / HW);
    float f[8];
    act_ld8<S>(x, x_lo, p * x_pitch + c0, f);
    const float4 s0 = *reinterpret_cast<const float4*>(s + static_cast<size_t>(n) * C + c0);
    const float4 s1 = *reinterpret_cast<const float4*>(s + static_cast<size_t>(n) * C + c0 + 4);
    f[0] *= s0.x; f[1] *= s0.y; f[2] *= s0.z; f[3] *= s0.w;
    f[4] *= s1.x; f[5] *= s1.y; f[6] *= s1.z; f[7] *= s1.w;
    act_st8<S>(out, out_lo, p * out_pitch + c0, f);
  }
}

// Feature-perturbation fork: x [M, HW, C] -> out [M + N, HW, C] with out[m] = x[m] and out[M + n] = x[n] * s[n, c] for
// the first N <= M images (M = N: UniMatch's FP batch; M = 2N: its two strong streams, the first one perturbed). The
// perturbed part is scale_nc's arithmetic (bit-equal to scale_nc(x[:N], s)); the copy is stored through the same
// act_st8, so s = 1 gives bit-equal copies in either storage form.
template <bool S>
__global__ void fp_fork_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ x_lo, int x_pitch,
                               const float* __restrict__ s, __nv_bfloat16* __restrict__ out,
                               __nv_bfloat16* __restrict__ out_lo, int out_pitch, int M, int N, long long HW, int C) {
  const int groups = C >> 3;
  const long long first = static_cast<long long>(M) * HW;
  const long long total = first * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int c0 = static_cast<int>(idx - p * groups) << 3;
    const int n = static_cast<int>(p / HW);
    float f[8];
    act_ld8<S>(x, x_lo, p * x_pitch + c0, f);
    act_st8<S>(out, out_lo, p * out_pitch + c0, f);
    if (n < N) {
      const float4 s0 = *reinterpret_cast<const float4*>(s + static_cast<size_t>(n) * C + c0);
      const float4 s1 = *reinterpret_cast<const float4*>(s + static_cast<size_t>(n) * C + c0 + 4);
      f[0] *= s0.x; f[1] *= s0.y; f[2] *= s0.z; f[3] *= s0.w;
      f[4] *= s1.x; f[5] *= s1.y; f[6] *= s1.z; f[7] *= s1.w;
      act_st8<S>(out, out_lo, (p + first) * out_pitch + c0, f);
    }
  }
}

// Its backward: out[m] = d[m], plus s[n, c] * d[M + n] for the first N images, in fp32 (the product and the sum each
// rounded to nearest, never contracted to an fma) and rounded once to the activation form.
template <bool S>
__global__ void fp_fold_kernel(const __nv_bfloat16* __restrict__ d, const __nv_bfloat16* __restrict__ d_lo, int d_pitch,
                               const float* __restrict__ s, __nv_bfloat16* __restrict__ out,
                               __nv_bfloat16* __restrict__ out_lo, int out_pitch, int M, int N, long long HW, int C) {
  const int groups = C >> 3;
  const long long first = static_cast<long long>(M) * HW;
  const long long total = first * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int c0 = static_cast<int>(idx - p * groups) << 3;
    const int n = static_cast<int>(p / HW);
    const Raw8<S> ra = act_ldraw<S>(d, d_lo, p * d_pitch + c0);
    float a[8];
    act_unpack<S>(ra, a);
    if (n < N) {
      const Raw8<S> rb = act_ldraw<S>(d, d_lo, (p + first) * d_pitch + c0);
      const float4 s0 = *reinterpret_cast<const float4*>(s + static_cast<size_t>(n) * C + c0);
      const float4 s1 = *reinterpret_cast<const float4*>(s + static_cast<size_t>(n) * C + c0 + 4);
      const float sv[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      float b[8];
      act_unpack<S>(rb, b);
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] = __fadd_rn(a[q], __fmul_rn(sv[q], b[q]));
    }
    act_st8<S>(out, out_lo, p * out_pitch + c0, a);
  }
}

// K-sliced conv finish: y = epilogue(sum_s partial[s]) for a chunk of pixels x 64 channels per block (8 channel groups
// x 32 pixel lanes), plus the chunk's per-channel (sum, sum of squares, count) row in the conv-epilogue statistics format.
template <bool S>
__global__ void __launch_bounds__(256)
conv_splitk_finish_kernel(const float* __restrict__ part, int k_slices, long long slice_stride, int part_pitch, int M, int C,
                          int affine, int relu, const float* __restrict__ scale, const float* __restrict__ shift,
                          const __nv_bfloat16* __restrict__ res, const __nv_bfloat16* __restrict__ res_lo, int res_pitch,
                          __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ y_lo, int y_pitch,
                          int rows_per_chunk, float* __restrict__ stats) {
  __shared__ float s_a[32][65];
  __shared__ float s_b[32][65];
  const int gl = threadIdx.x & 7;
  const int pl = threadIdx.x >> 3;
  const int c0 = blockIdx.x * 64 + gl * 8;
  const int chunk = blockIdx.y;
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(M, r0 + rows_per_chunk);
  float a[8] = {0, 0, 0, 0, 0, 0, 0, 0}, b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  float sc[8], sh[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    sc[q] = (affine && scale) ? scale[c0 + q] : 1.f;
    sh[q] = (affine && shift) ? shift[c0 + q] : 0.f;
  }
  for (int r = r0 + pl; r < r1; r += 32) {
    float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const float* src = part + static_cast<long long>(r) * part_pitch + c0;
    for (int s = 0; s < k_slices; ++s) {   // fixed order, fp32 round-to-nearest adds
      const float4 p0 = *reinterpret_cast<const float4*>(src + s * slice_stride);
      const float4 p1 = *reinterpret_cast<const float4*>(src + s * slice_stride + 4);
      v[0] += p0.x; v[1] += p0.y; v[2] += p0.z; v[3] += p0.w;
      v[4] += p1.x; v[5] += p1.y; v[6] += p1.z; v[7] += p1.w;
    }
    if (affine) {
      float rr[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (res) act_ld8<S>(res, res_lo, static_cast<long long>(r) * res_pitch + c0, rr);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        float t = fmaf(v[q], sc[q], sh[q]) + rr[q];
        v[q] = relu ? fmaxf(t, 0.f) : t;
      }
    }
    act_st8<S>(y, y_lo, static_cast<long long>(r) * y_pitch + c0, v);
    if (stats) {   // statistics of the values as stored (hi + lo / bf16), like the conv epilogue
      float w[8];
      act_ld8<S>(y, y_lo, static_cast<long long>(r) * y_pitch + c0, w);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        a[q] += w[q];
        b[q] = fmaf(w[q], w[q], b[q]);
      }
    }
  }
  if (!stats) return;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    s_a[pl][gl * 8 + q] = a[q];
    s_b[pl][gl * 8 + q] = b[q];
  }
  __syncthreads();
  if (pl < 3) {
    float* row = stats + static_cast<size_t>(chunk) * 3 * C;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      float t = 0.f;
      if (pl < 2) {
        float(*src)[65] = pl == 0 ? s_a : s_b;
        for (int i = 0; i < 32; ++i) t += src[i][gl * 8 + q];
      } else {
        t = static_cast<float>(r1 - r0);
      }
      row[pl * C + c0 + q] = t;
    }
  }
}

// fp32 [M][in_pitch] (first C columns) -> activation [M][out_pitch] with columns C..Cp-1 zero filled (Cp % 8 == 0).
template <bool S>
__global__ void f32_to_act_kernel(const float* __restrict__ in, int in_pitch, __nv_bfloat16* __restrict__ out,
                                  __nv_bfloat16* __restrict__ out_lo, int out_pitch, long long M, int C, int Cp) {
  const int groups = Cp >> 3;
  const long long total = M * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int c0 = static_cast<int>(idx - p * groups) << 3;
    float f[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) f[q] = (c0 + q < C) ? in[p * in_pitch + c0 + q] : 0.f;
    act_st8<S>(out, out_lo, p * out_pitch + c0, f);
  }
}

// activation [M][in_pitch] -> fp32 [M][out_pitch] (C % 8 == 0 columns).
template <bool S>
__global__ void act_to_f32_kernel(const __nv_bfloat16* __restrict__ in, const __nv_bfloat16* __restrict__ in_lo,
                                  int in_pitch, float* __restrict__ out, int out_pitch, long long M, int C) {
  const int groups = C >> 3;
  const long long total = M * groups;
  for (long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long p = idx / groups;
    const int c0 = static_cast<int>(idx - p * groups) << 3;
    float f[8];
    act_ld8<S>(in, in_lo, p * in_pitch + c0, f);
#pragma unroll
    for (int q = 0; q < 8; ++q) out[p * out_pitch + c0 + q] = f[q];
  }
}

static int ew_grid(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

// Grid whose total thread count is a multiple of `groups` (= C/8), so each thread owns fixed channels.
static int ew_grid_fixed_channels(long long total, int threads, int groups) {
  long long b = ew_grid(total, threads);
  // smallest m with (m * threads) % groups == 0
  long long m = 1;
  while ((m * threads) % groups != 0) ++m;
  b = (b + m - 1) / m * m;
  return static_cast<int>(b);
}

static int chunk_rows(int M) {
  int rows = cdiv(M, 1024);
  if (rows < 256) rows = 256;
  return (rows + 31) & ~31;
}

}  // namespace sb

using namespace sb;
typedef __nv_bfloat16 bf16;

extern "C" long long semseg_bn_workspace_floats(int M, int C) {
  if (M <= 0 || C <= 0) return 0;
  const int rows = chunk_rows(M);
  const long long chunks = cdiv(M, rows);
  return chunks * 2 * C;
}

// The exchange arguments of semseg_bn_finalize_partials / semseg_bn_bwd_reduce with a peer table: `need_floats` words
// of this rank's block must fit in a slot.
static int fill_peer_args(sb::PeerArgs* pa, void* const* peer_bufs, int world, int rank, int slot, int slot_floats,
                          const void* seq_ptr, int need_floats) {
  SB_CHECK_ARG(world >= 1 && world <= 8 && rank >= 0 && rank < world, "p2p: world %d rank %d unsupported", world, rank);
  SB_CHECK_ARG(slot >= 0 && need_floats <= slot_floats, "p2p: slot too small (%d > %d floats)", need_floats,
               slot_floats);
  SB_CHECK_ARG(seq_ptr, "p2p: null sequence-number pointer");
  for (int i = 0; i < world; ++i) {
    SB_CHECK_ARG(peer_bufs[i], "p2p: null peer pointer %d", i);
    pa->buf[i] = static_cast<float*>(peer_bufs[i]);
  }
  pa->world = world;
  pa->rank = rank;
  pa->slot = slot;
  pa->slot_floats = slot_floats;
  pa->seq_ptr = static_cast<const unsigned*>(seq_ptr);
  static long long ticks = 0;
  if (ticks == 0) {
    const char* e = getenv("SEMSEG_B200_P2P_TIMEOUT_S");
    double sec = e ? atof(e) : 600.0;
    if (!(sec > 0.0)) sec = 600.0;
    ticks = static_cast<long long>(sec * 2.0e9);
  }
  pa->timeout_ticks = ticks;
  return SEMSEG_OK;
}

extern "C" int semseg_bn_merge_partials(const float* stats_partial, int rows, int C, float* out_stats, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(stats_partial && out_stats && rows > 0 && C > 0, "bn_merge_partials: bad args");
  SB_STATS_GROUP_DISPATCH(C, bn_merge_conv_partials_kernel<kCH><<<cdiv(C, kCH), 1024, 0, stream>>>(stats_partial, rows,
                                                                                                   C, out_stats));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_finalize_partials(const float* stats_partial, int rows, int C, const float* gamma,
                                           const float* beta, float eps, float momentum, float* running_mean,
                                           float* running_var, float* mean_invstd, float* scale_shift,
                                           void* const* peer_bufs, int world, int rank, int slot, int slot_floats,
                                           const void* seq_ptr, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(stats_partial && mean_invstd && scale_shift && rows > 0 && C > 0, "bn_finalize_partials: bad args");
  sb::PeerArgs pa = {};
  if (peer_bufs) {
    const int r = fill_peer_args(&pa, peer_bufs, world, rank, slot, slot_floats, seq_ptr, 3 * C);
    if (r) return r;
  }
  SB_STATS_GROUP_DISPATCH(C, {
    auto kernel = peer_bufs ? bn_finalize_partials_kernel<kCH, true> : bn_finalize_partials_kernel<kCH, false>;
    kernel<<<cdiv(C, kCH), 1024, 0, stream>>>(stats_partial, rows, C, gamma, beta, eps, momentum, running_mean,
                                             running_var, mean_invstd, scale_shift, pa);
  });
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_finalize(const float* rank_stats, int R, int C, const float* gamma, const float* beta,
                                  float eps, float momentum, float* running_mean, float* running_var,
                                  float* mean_invstd, float* scale_shift, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(rank_stats && mean_invstd && scale_shift && R > 0 && C > 0, "bn_finalize: bad args");
  bn_finalize_kernel<<<cdiv(C, 128), 128, 0, stream>>>(rank_stats, R, C, gamma, beta, eps, momentum, running_mean,
                                                      running_var, mean_invstd, scale_shift);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_fold_eval(const float* gamma, const float* beta, const float* running_mean,
                                   const float* running_var, float eps, int C, float* scale_shift, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(running_mean && running_var && scale_shift && C > 0, "bn_fold_eval: bad args");
  bn_fold_eval_kernel<<<cdiv(C, 128), 128, 0, stream>>>(gamma, beta, running_mean, running_var, eps, C, scale_shift);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_apply(const void* x, const void* x_lo, int x_pitch, const float* scale_shift,
                               const void* residual, const void* residual_lo, int res_pitch, void* y, void* y_lo,
                               int y_pitch, int M, int C, int relu, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && scale_shift && y && M > 0 && C > 0, "bn_apply: bad args");
  SB_CHECK_ARG(C % 8 == 0 && x_pitch % 8 == 0 && y_pitch % 8 == 0 && (!residual || res_pitch % 8 == 0),
               "bn_apply: channels and pitches must be multiples of 8");
  const bool split = x_lo != nullptr;
  SB_CHECK_ARG((y_lo != nullptr) == split && (!residual || (residual_lo != nullptr) == split),
               "bn_apply: all tensors must use the same storage form (plain or split)");
  if (const int r = check_vec_acts("bn_apply", C, {{x, x_lo, x_pitch}, {residual, residual_lo, res_pitch},
                                                   {y, y_lo, y_pitch}}))
    return r;
  const long long total = static_cast<long long>(M) * (C / 8);
  const int grid = ew_grid_fixed_channels(total, 256, C / 8);
  SB_ACT_DISPATCH(split, bn_apply_kernel<kS><<<grid, 256, 0, stream>>>(
                             static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, scale_shift,
                             static_cast<const bf16*>(residual), static_cast<const bf16*>(residual_lo), res_pitch,
                             static_cast<bf16*>(y), static_cast<bf16*>(y_lo), y_pitch, M, C, relu));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_bwd_reduce(const void* dy, const void* dy_lo, int dy_pitch, const void* y, const void* y_lo,
                                    int y_pitch, const void* x, const void* x_lo, int x_pitch,
                                    const float* mean_invstd, const float* scale_shift, int M, int C, int relu,
                                    float* workspace, long long workspace_floats, float* sums, float* sums_total,
                                    void* const* peer_bufs, int world, int rank, int slot, int slot_floats,
                                    const void* seq_ptr, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dy && x && mean_invstd && workspace && sums && M > 0 && C > 0, "bn_bwd_reduce: bad args");
  SB_CHECK_ARG(!relu || y || scale_shift, "bn_bwd_reduce: relu needs y or scale_shift");
  SB_CHECK_ARG(C % 8 == 0 && dy_pitch % 8 == 0 && x_pitch % 8 == 0 && (!(relu && y) || y_pitch % 8 == 0),
               "bn_bwd_reduce: channels and pitches must be multiples of 8");
  SB_CHECK_ARG(workspace_floats >= semseg_bn_workspace_floats(M, C), "bn_bwd_reduce: workspace too small");
  const bool split = dy_lo != nullptr;
  SB_CHECK_ARG((x_lo != nullptr) == split && (!(relu && y) || (y_lo != nullptr) == split),
               "bn_bwd_reduce: all tensors must use the same storage form (plain or split)");
  if (const int r = check_vec_acts("bn_bwd_reduce", C, {{dy, dy_lo, dy_pitch}, {x, x_lo, x_pitch},
                                                        {relu ? y : nullptr, y_lo, y_pitch}}))
    return r;
  sb::PeerArgs pa = {};
  if (peer_bufs) {
    SB_CHECK_ARG(sums_total, "bn_bwd_reduce: the peer exchange needs sums_total");
    const int r = fill_peer_args(&pa, peer_bufs, world, rank, slot, slot_floats, seq_ptr, 2 * C);
    if (r) return r;
  }
  const int rows = chunk_rows(M);
  const int chunks = cdiv(M, rows);
  dim3 grid(cdiv(C, 64), chunks);
  SB_ACT_DISPATCH(split, bn_bwd_reduce_kernel<kS><<<grid, 256, 0, stream>>>(
                             static_cast<const bf16*>(dy), static_cast<const bf16*>(dy_lo), dy_pitch,
                             static_cast<const bf16*>(y), static_cast<const bf16*>(y_lo), y_pitch,
                             static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, mean_invstd,
                             scale_shift, M, C, relu, rows, workspace));
  SB_LAUNCHED();
  auto final_kernel = peer_bufs ? bn_bwd_reduce_final_kernel<true> : bn_bwd_reduce_final_kernel<false>;
  final_kernel<<<cdiv(2 * C, 32), 1024, 0, stream>>>(workspace, chunks, C, sums, sums_total, pa);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_bwd_apply(const void* dy, const void* dy_lo, int dy_pitch, const void* y, const void* y_lo,
                                   int y_pitch, const void* x, const void* x_lo, int x_pitch,
                                   const float* mean_invstd, const float* gamma, const float* scale_shift,
                                   const float* sums, float count, int M, int C, int relu, void* dx, void* dx_lo,
                                   int dx_pitch, void* dres, void* dres_lo, int dres_pitch, float* dgamma_dbeta,
                                   void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dy && x && mean_invstd && sums && dx && M > 0 && C > 0, "bn_bwd_apply: bad args");
  SB_CHECK_ARG(!relu || y || scale_shift, "bn_bwd_apply: relu needs y or scale_shift");
  SB_CHECK_ARG(C % 8 == 0 && dy_pitch % 8 == 0 && x_pitch % 8 == 0 && dx_pitch % 8 == 0 &&
                   (!(relu && y) || y_pitch % 8 == 0) && (!dres || dres_pitch % 8 == 0),
               "bn_bwd_apply: channels and pitches must be multiples of 8");
  const bool split = dy_lo != nullptr;
  SB_CHECK_ARG((x_lo != nullptr) == split && (dx_lo != nullptr) == split &&
                   (!(relu && y) || (y_lo != nullptr) == split) && (!dres || (dres_lo != nullptr) == split),
               "bn_bwd_apply: all tensors must use the same storage form (plain or split)");
  if (const int r = check_vec_acts("bn_bwd_apply", C, {{dy, dy_lo, dy_pitch}, {x, x_lo, x_pitch},
                                                       {relu ? y : nullptr, y_lo, y_pitch}, {dx, dx_lo, dx_pitch},
                                                       {dres, dres_lo, dres_pitch}}))
    return r;
  const long long total = static_cast<long long>(M) * (C / 8);
  const int grid = ew_grid_fixed_channels(total, 256, C / 8);
  SB_ACT_DISPATCH(split, bn_bwd_apply_kernel<kS><<<grid, 256, 0, stream>>>(
                             static_cast<const bf16*>(dy), static_cast<const bf16*>(dy_lo), dy_pitch,
                             static_cast<const bf16*>(y), static_cast<const bf16*>(y_lo), y_pitch,
                             static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, mean_invstd, gamma,
                             scale_shift, sums, count > 0.f ? 1.f / count : 0.f, M, C, relu, static_cast<bf16*>(dx),
                             static_cast<bf16*>(dx_lo), dx_pitch, static_cast<bf16*>(dres),
                             static_cast<bf16*>(dres_lo), dres_pitch, dgamma_dbeta));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_bn_bwd_frozen(const void* dy, const void* dy_lo, int dy_pitch, const void* y, const void* y_lo,
                                    int y_pitch, const void* raw, const void* raw_lo, int raw_pitch, const float* gamma,
                                    const float* beta, const float* running_mean, const float* running_var, float eps,
                                    int M, int C, int relu, void* d_raw, void* d_raw_lo, int d_raw_pitch, void* dres,
                                    void* dres_lo, int dres_pitch, float* workspace, long long workspace_floats,
                                    float* sums, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dy && d_raw && running_mean && running_var, "bn_bwd_frozen: null dy, d_raw or running statistics");
  SB_CHECK_ARG(M > 0 && C > 0 && C % 8 == 0, "bn_bwd_frozen: need M > 0 and C > 0, C %% 8 == 0 (M %d, C %d)", M, C);
  SB_CHECK_ARG(!relu || y || raw, "bn_bwd_frozen: relu needs y or raw for the mask");
  const bool use_y = relu && y, use_raw = raw != nullptr;
  SB_CHECK_ARG(dy_pitch >= C && dy_pitch % 8 == 0 && d_raw_pitch >= C && d_raw_pitch % 8 == 0 &&
                   (!use_y || (y_pitch >= C && y_pitch % 8 == 0)) &&
                   (!use_raw || (raw_pitch >= C && raw_pitch % 8 == 0)) &&
                   (!dres || (dres_pitch >= C && dres_pitch % 8 == 0)),
               "bn_bwd_frozen: pitches must be multiples of 8 and at least C");
  SB_CHECK_ARG(!sums || (workspace && workspace_floats >= semseg_bn_workspace_floats(M, C)),
               "bn_bwd_frozen: sums need a workspace of semseg_bn_workspace_floats(M, C) floats");
  const bool split = dy_lo != nullptr;
  SB_CHECK_ARG((d_raw_lo != nullptr) == split && (!use_y || (y_lo != nullptr) == split) &&
                   (!use_raw || (raw_lo != nullptr) == split) && (!dres || (dres_lo != nullptr) == split),
               "bn_bwd_frozen: all tensors must use the same storage form (plain or split)");
  if (const int r = check_vec_acts("bn_bwd_frozen", C, {{dy, dy_lo, dy_pitch}, {use_y ? y : nullptr, y_lo, y_pitch},
                                                        {raw, raw_lo, raw_pitch}, {d_raw, d_raw_lo, d_raw_pitch},
                                                        {dres, dres_lo, dres_pitch}}))
    return r;
  const int rows = chunk_rows(M);
  const int chunks = cdiv(M, rows);
  dim3 grid(cdiv(C, 64), chunks);
  SB_ACT_DISPATCH(split, bn_bwd_frozen_kernel<kS><<<grid, 256, 0, stream>>>(
                             static_cast<const bf16*>(dy), static_cast<const bf16*>(dy_lo), dy_pitch,
                             static_cast<const bf16*>(use_y ? y : nullptr), static_cast<const bf16*>(y_lo), y_pitch,
                             static_cast<const bf16*>(raw), static_cast<const bf16*>(raw_lo), raw_pitch, gamma, beta,
                             running_mean, running_var, eps, M, C, relu, rows, static_cast<bf16*>(d_raw),
                             static_cast<bf16*>(d_raw_lo), d_raw_pitch, static_cast<bf16*>(dres),
                             static_cast<bf16*>(dres_lo), dres_pitch, sums ? workspace : nullptr));
  SB_LAUNCHED();
  if (sums) {
    bn_bwd_reduce_final_kernel<false><<<cdiv(2 * C, 32), 1024, 0, stream>>>(workspace, chunks, C, sums, nullptr,
                                                                         sb::PeerArgs{});
    SB_LAUNCHED();
  }
  return SEMSEG_OK;
}

extern "C" int semseg_add_act(const void* a, const void* a_lo, int a_pitch, const void* b, const void* b_lo,
                              int b_pitch, void* out, void* out_lo, int out_pitch, int M, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(a && b && out && M > 0 && C > 0 && C % 8 == 0 && a_pitch % 8 == 0 && b_pitch % 8 == 0 &&
                   out_pitch % 8 == 0,
               "add_act: bad args");
  const bool split = a_lo != nullptr;
  SB_CHECK_ARG((b_lo != nullptr) == split && (out_lo != nullptr) == split,
               "add_act: all tensors must use the same storage form (plain or split)");
  if (const int r = check_vec_acts("add_act", C, {{a, a_lo, a_pitch}, {b, b_lo, b_pitch}, {out, out_lo, out_pitch}}))
    return r;
  const long long total = static_cast<long long>(M) * (C / 8);
  SB_ACT_DISPATCH(split, add_act_kernel<kS><<<ew_grid(total, 256), 256, 0, stream>>>(
                             static_cast<const bf16*>(a), static_cast<const bf16*>(a_lo), a_pitch,
                             static_cast<const bf16*>(b), static_cast<const bf16*>(b_lo), b_pitch,
                             static_cast<bf16*>(out), static_cast<bf16*>(out_lo), out_pitch, M, C));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_scale_nc(const void* x, const void* x_lo, int x_pitch, const float* scale, void* out,
                               void* out_lo, int out_pitch, int N, int HW, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(x && scale && out && N > 0 && HW > 0 && C > 0 && C % 8 == 0 && x_pitch % 8 == 0 && out_pitch % 8 == 0,
               "scale_nc: bad args");
  const bool split = x_lo != nullptr;
  SB_CHECK_ARG((out_lo != nullptr) == split, "scale_nc: input and output must use the same storage form");
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(scale) & 15) == 0, "scale_nc: scale %p is not 16-byte aligned", scale);
  if (const int r = check_vec_acts("scale_nc", C, {{x, x_lo, x_pitch}, {out, out_lo, out_pitch}})) return r;
  const long long total = static_cast<long long>(N) * HW * (C / 8);
  SB_ACT_DISPATCH(split, scale_nc_kernel<kS><<<ew_grid(total, 256), 256, 0, stream>>>(
                             static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, scale,
                             static_cast<bf16*>(out), static_cast<bf16*>(out_lo), out_pitch, N, HW, C));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// The fork and the fold share their argument rules: the fork's `x` holds M images and `out` M + N, the fold's the
// other way round; the first N <= M images are the perturbed ones.
static int check_fp_args(const char* fn, const void* x, const void* x_lo, int x_pitch, const float* scale,
                         const void* out, const void* out_lo, int out_pitch, int M, int N, int HW, int C) {
  SB_CHECK_ARG(x && scale && out, "%s: null x, scale or out", fn);
  SB_CHECK_ARG(N > 0 && HW > 0 && C > 0 && C % 8 == 0, "%s: need N, HW, C > 0 and C %% 8 == 0 (N %d, HW %d, C %d)", fn,
               N, HW, C);
  SB_CHECK_ARG(M >= N, "%s: need M >= N (M %d, N %d)", fn, M, N);
  SB_CHECK_ARG(x_pitch >= C && x_pitch % 8 == 0 && out_pitch >= C && out_pitch % 8 == 0,
               "%s: pitches must be multiples of 8 and at least C (x %d, out %d, C %d)", fn, x_pitch, out_pitch, C);
  SB_CHECK_ARG((out_lo != nullptr) == (x_lo != nullptr), "%s: input and output must use the same storage form", fn);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(scale) & 15) == 0, "%s: scale %p is not 16-byte aligned", fn, scale);
  return check_vec_acts(fn, C, {{x, x_lo, x_pitch}, {out, out_lo, out_pitch}});
}

static int fp_fork_launch(const char* fn, const void* x, const void* x_lo, int x_pitch, const float* scale, void* out,
                          void* out_lo, int out_pitch, int M, int N, int HW, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (const int r = check_fp_args(fn, x, x_lo, x_pitch, scale, out, out_lo, out_pitch, M, N, HW, C)) return r;
  const long long total = static_cast<long long>(M) * HW * (C / 8);
  SB_ACT_DISPATCH(x_lo != nullptr, fp_fork_kernel<kS><<<ew_grid(total, 256), 256, 0, stream>>>(
                                       static_cast<const bf16*>(x), static_cast<const bf16*>(x_lo), x_pitch, scale,
                                       static_cast<bf16*>(out), static_cast<bf16*>(out_lo), out_pitch, M, N, HW, C));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

static int fp_fold_launch(const char* fn, const void* d, const void* d_lo, int d_pitch, const float* scale, void* out,
                          void* out_lo, int out_pitch, int M, int N, int HW, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (const int r = check_fp_args(fn, d, d_lo, d_pitch, scale, out, out_lo, out_pitch, M, N, HW, C)) return r;
  const long long total = static_cast<long long>(M) * HW * (C / 8);
  SB_ACT_DISPATCH(d_lo != nullptr, fp_fold_kernel<kS><<<ew_grid(total, 256), 256, 0, stream>>>(
                                       static_cast<const bf16*>(d), static_cast<const bf16*>(d_lo), d_pitch, scale,
                                       static_cast<bf16*>(out), static_cast<bf16*>(out_lo), out_pitch, M, N, HW, C));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_fp_fork(const void* x, const void* x_lo, int x_pitch, const float* scale, void* out, void* out_lo,
                              int out_pitch, int N, int HW, int C, void* stream) {
  return fp_fork_launch("fp_fork", x, x_lo, x_pitch, scale, out, out_lo, out_pitch, N, N, HW, C, stream);
}

extern "C" int semseg_fp_fold(const void* d, const void* d_lo, int d_pitch, const float* scale, void* out, void* out_lo,
                              int out_pitch, int N, int HW, int C, void* stream) {
  return fp_fold_launch("fp_fold", d, d_lo, d_pitch, scale, out, out_lo, out_pitch, N, N, HW, C, stream);
}

extern "C" int semseg_fp_fork_prefix(const void* x, const void* x_lo, int x_pitch, const float* scale, void* out,
                                     void* out_lo, int out_pitch, int M, int N, int HW, int C, void* stream) {
  return fp_fork_launch("fp_fork_prefix", x, x_lo, x_pitch, scale, out, out_lo, out_pitch, M, N, HW, C, stream);
}

extern "C" int semseg_fp_fold_prefix(const void* d, const void* d_lo, int d_pitch, const float* scale, void* out,
                                     void* out_lo, int out_pitch, int M, int N, int HW, int C, void* stream) {
  return fp_fold_launch("fp_fold_prefix", d, d_lo, d_pitch, scale, out, out_lo, out_pitch, M, N, HW, C, stream);
}

static int splitk_chunk_rows(int M) {
  int rows = cdiv(M, 2048);
  if (rows < 128) rows = 128;
  return (rows + 31) & ~31;
}

extern "C" int semseg_conv_splitk_rows(int M) { return M > 0 ? cdiv(M, splitk_chunk_rows(M)) : SEMSEG_E_INVALID; }

extern "C" int semseg_conv_splitk_finish(const float* partial, int k_slices, long long slice_stride, int part_pitch,
                                         int M, int C, int epi_mode, int relu, const float* scale, const float* shift,
                                         const void* residual, const void* residual_lo, int res_pitch, void* y,
                                         void* y_lo, int y_pitch, float* stats_partial, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(partial && y && k_slices >= 1 && M > 0 && C > 0 && C % 64 == 0, "conv_splitk_finish: bad args");
  SB_CHECK_ARG(part_pitch % 4 == 0 && part_pitch >= C && slice_stride % 4 == 0 && y_pitch % 8 == 0 &&
                   (!residual || res_pitch % 8 == 0),
               "conv_splitk_finish: pitches must keep 16-byte alignment");
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(partial) | reinterpret_cast<uintptr_t>(y) |
                 reinterpret_cast<uintptr_t>(y_lo) | reinterpret_cast<uintptr_t>(residual) |
                 reinterpret_cast<uintptr_t>(residual_lo)) & 15) == 0,
               "conv_splitk_finish: partial, y and residual must be 16-byte aligned");
  SB_CHECK_ARG(epi_mode == SEMSEG_EPI_RAW || epi_mode == SEMSEG_EPI_AFFINE, "conv_splitk_finish: RAW or AFFINE only");
  SB_CHECK_ARG(!stats_partial || epi_mode == SEMSEG_EPI_RAW, "conv_splitk_finish: statistics only in RAW mode");
  const bool split = y_lo != nullptr;
  SB_CHECK_ARG(!residual || (residual_lo != nullptr) == split, "conv_splitk_finish: residual / y storage forms differ");
  const int rows = splitk_chunk_rows(M);
  dim3 grid(C / 64, cdiv(M, rows));
  SB_ACT_DISPATCH(split, conv_splitk_finish_kernel<kS><<<grid, 256, 0, stream>>>(
                             partial, k_slices, slice_stride, part_pitch, M, C, epi_mode == SEMSEG_EPI_AFFINE ? 1 : 0,
                             relu, scale, shift, static_cast<const bf16*>(residual),
                             static_cast<const bf16*>(residual_lo), res_pitch, static_cast<bf16*>(y),
                             static_cast<bf16*>(y_lo), y_pitch, rows, stats_partial));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_f32_to_act(const float* in, int in_pitch, void* out, void* out_lo, int out_pitch, long long M,
                                 int C, int Cp, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(in && out && M > 0 && C > 0 && Cp >= C && Cp % 8 == 0 && out_pitch % 8 == 0 && in_pitch >= C,
               "f32_to_act: bad args");
  if (const int r = check_vec_acts("f32_to_act", Cp, {{out, out_lo, out_pitch}})) return r;
  const long long total = M * (Cp / 8);
  SB_ACT_DISPATCH(out_lo != nullptr, f32_to_act_kernel<kS><<<ew_grid(total, 256), 256, 0, stream>>>(
                                         in, in_pitch, static_cast<bf16*>(out), static_cast<bf16*>(out_lo), out_pitch,
                                         M, C, Cp));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_act_to_f32(const void* in, const void* in_lo, int in_pitch, float* out, int out_pitch,
                                 long long M, int C, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(in && out && M > 0 && C > 0 && C % 8 == 0 && in_pitch % 8 == 0 && out_pitch >= C,
               "act_to_f32: bad args");
  if (const int r = check_vec_acts("act_to_f32", C, {{in, in_lo, in_pitch}})) return r;
  const long long total = M * (C / 8);
  SB_ACT_DISPATCH(in_lo != nullptr, act_to_f32_kernel<kS><<<ew_grid(total, 256), 256, 0, stream>>>(
                                        static_cast<const bf16*>(in), static_cast<const bf16*>(in_lo), in_pitch, out,
                                        out_pitch, M, C));
  SB_LAUNCHED();
  return SEMSEG_OK;
}

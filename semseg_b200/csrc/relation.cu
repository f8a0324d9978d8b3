// Cross-image relational distillation (CIRKD's mini-batch pixel-to-pixel term, losses.DistillationLoss's
// relation_weight), flash-attention style: the [B M, B M] similarity maps of the student and the teacher never exist
// in memory, only two log-sum-exps per (row image, column image, row).
//
//   nodes      : NHWC feature [B, h, w, 512] (plain or split) -> max-pool p x p (ceil mode) -> L2-normalise (fp32, a node
//                with norm < 1e-12 is the zero vector) -> bf16 operand [B, M, 512] (hi, and lo in bf16x3), 1024-byte
//                K-major rows for TMA. The student's also keeps the window offset of every (node, channel) maximum
//                (uint8, first maximum in row-major window order) and 1/|x| per node (0 for a zero node).
//   kl_fwd     : CTA = (image i, 64 rows of i, image j). The rows' X_i / Y_i chunks and the keys' X_j / Y_j chunks stream
//                through a TMA / mbarrier ring as [64 rows x 64 channels] boxes; one consumer warpgroup accumulates
//                S = X_i X_j^T and T = Y_i Y_j^T for 64 keys at a time (two m64n64 wgmma chains over K = 512) and keeps
//                per row the running (max, sum) of both maps and the rescaled cross term sum exp(t - m_t) (t - s), so
//                KL(Q_row || P_row) = cross / l_t - lse_t + lse_s. Writes (lse_s, lse_t) per (i, j, row) and one fp64
//                partial per CTA; a one-CTA kernel reduces the partials in a fixed order. No atomics.
//   kl_bwd     : CTA = (image n, 64 rows of n, channel half). For every partner j and key tile it recomputes S and T of
//                (n, j) once and forms G = (P_nj - Q_nj) + (P_jn - Q_jn)^T elementwise: the row statistics of n's rows
//                for the first term, those of j's rows (the keys) for the second, so both roles of X_n in the loss are
//                one GEMM, dX_n += coef G X_j, on a 64 x 256 fp32 accumulator in registers. Each CTA owns the rows and
//                channels it writes. The two channel halves recompute S and T each: 2 recomputes of the forward's GEMMs.
//   nodes_bwd  : (dx^ - x^ (x^ . dx^)) / |x| (0 for a zero node) routed to each window's saved maximum; the rest of the
//                window is written with zeros, so the NHWC gradient needs no memset.
// bf16x3 (split operands): every GEMM runs three K segments, hi*hi + lo*hi + hi*lo, into the same accumulator, the
// backward's G split into hi + lo like the nodes.
#include <math.h>

#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

constexpr int kRlC = 512;                         // node channels (the cls[0] width of every PSPNet / PSANet)
constexpr int kRlRows = 64;                       // rows (and keys) per tile
constexpr int kRlBox = kRlRows * 128;             // one [64 rows x 64 channels] bf16 box, 8 KB
constexpr int kRlStage = 4 * kRlBox;              // four boxes per ring stage
constexpr int kRlChunks = kRlC / 64;
constexpr int kRlFwdStages = 3;
constexpr int kRlFwdSmem = kRlFwdStages * kRlStage + 256 + kRlRows * 8 + 1024;
constexpr int kRlBwdStages = 4;
constexpr int kRlBwdSmem = kRlBwdStages * kRlStage + 2 * kRlBox + 256 + 1024;
constexpr int kRlMaxPool = 16;                    // window offsets are stored as uint8

struct RelKLParams {
  float* lse;             // [B][B][M][2] (lse_s, lse_t) per (row image, column image, row)
  double* partial;        // [grid] fp64 KL sum of the CTA's rows (forward)
  const float* grad;      // [1] dL/dR (backward)
  float* dnodes;          // [B][M][512] fp32 gradient of the student nodes (backward)
  int B, M, tiles, nseg;
  float inv_tau;
  float coef;             // tau / (B^2 M) (backward)
};

__device__ __forceinline__ uint64_t rl_desc_kmajor(uint32_t addr) { return make_wgmma_desc_sw128(addr, 16, 1024); }

// S and T of one (64 rows, 64 keys) tile over K = 512 (nseg segments) from the ring; `it` is the ring position.
template <int kStages>
__device__ __forceinline__ void rl_tile_st(uint8_t* smem, uint64_t* full, uint64_t* empty, int& it, int nseg,
                                           float (&as)[32], float (&at)[32]) {
  int prev_s = -1;
  const int n = nseg * kRlChunks;
  for (int q = 0; q < n; ++q, ++it) {
    const int s = it % kStages;
    mbar_wait(&full[s], (it / kStages) & 1);
    const uint32_t base = smem_u32(smem + s * kRlStage);
    const uint64_t ax = rl_desc_kmajor(base), ay = rl_desc_kmajor(base + kRlBox);
    const uint64_t bx = rl_desc_kmajor(base + 2 * kRlBox), by = rl_desc_kmajor(base + 3 * kRlBox);
    wgmma_fence_operand(as);
    wgmma_fence_operand(at);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t acc = (q > 0 || k > 0) ? 1u : 0u;
      wgmma_bf16<64, 0, 0>(as, ax + static_cast<uint64_t>(2 * k), bx + static_cast<uint64_t>(2 * k), acc);
      wgmma_bf16<64, 0, 0>(at, ay + static_cast<uint64_t>(2 * k), by + static_cast<uint64_t>(2 * k), acc);
    }
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_operand(as);
    wgmma_fence_operand(at);
    if (prev_s >= 0) mbar_arrive(&empty[prev_s]);
    prev_s = s;
  }
  wgmma_wait<0>();
  wgmma_fence_operand(as);
  wgmma_fence_operand(at);
  mbar_arrive(&empty[prev_s]);
}

// producer side of rl_tile_st: chunk c of rows (image ri, row r0) and keys (image kj, row k0) of both networks
__device__ __forceinline__ void rl_load_st(uint8_t* smem, uint64_t* full, uint64_t* empty, int& it, int stages, int nseg,
                                           const CUtensorMap* tx, const CUtensorMap* txl, const CUtensorMap* ty,
                                           const CUtensorMap* tyl, int ri, int r0, int kj, int k0) {
  for (int seg = 0; seg < nseg; ++seg) {
    for (int c = 0; c < kRlChunks; ++c, ++it) {
      const int s = it % stages;
      mbar_wait(&empty[s], ((it / stages) & 1) ^ 1);
      uint8_t* dst = smem + s * kRlStage;
      mbar_expect_tx(&full[s], kRlStage);
      tma_load_3d(dst, seg == 1 ? txl : tx, &full[s], c * 64, r0, ri);
      tma_load_3d(dst + kRlBox, seg == 1 ? tyl : ty, &full[s], c * 64, r0, ri);
      tma_load_3d(dst + 2 * kRlBox, seg == 2 ? txl : tx, &full[s], c * 64, k0, kj);
      tma_load_3d(dst + 3 * kRlBox, seg == 2 ? tyl : ty, &full[s], c * 64, k0, kj);
    }
  }
}

__global__ void __launch_bounds__(256, 2)
relation_kl_fwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmXlo,
                       const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmYlo,
                       const RelKLParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* misc = smem + kRlFwdStages * kRlStage;
  uint64_t* full = reinterpret_cast<uint64_t*>(misc);
  uint64_t* empty = full + kRlFwdStages;
  double* s_kl = reinterpret_cast<double*>(misc + 256);      // [64] per-row KL

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x % p.B;
  const int rt = (blockIdx.x / p.B) % p.tiles;
  const int i = blockIdx.x / (p.B * p.tiles);
  const int num_kt = p.tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < kRlFwdStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 128);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && elect_one()) {
      int it = 0;
      for (int kt = 0; kt < num_kt; ++kt)
        rl_load_st(smem, full, empty, it, kRlFwdStages, p.nseg, &tmX, &tmXlo, &tmY, &tmYlo, i, rt * kRlRows, j,
                   kt * kRlRows);
    }
    return;
  }
  const int ct = threadIdx.x - 128, wq = ct >> 5;
  // the sums and the rescale factors in fp64: a row's KL is a small difference of O(log M) quantities when Q and P are
  // near uniform (large tau), so the fp32 rounding of the sums would swamp it
  float ms[2], mt[2];
  double ls[2], lt[2], cr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    ms[r] = mt[r] = -INFINITY;
    ls[r] = lt[r] = cr[r] = 0.0;
  }
  int it = 0;
  for (int kt = 0; kt < num_kt; ++kt) {
    float as[32], at[32];
    rl_tile_st<kRlFwdStages>(smem, full, empty, it, p.nseg, as, at);
    // online update of the thread's two rows over its 16 columns; the four lanes of a row share its maximum
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float tms = -INFINITY, tmt = -INFINITY;
#pragma unroll
      for (int q = 0; q < 8; ++q)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int k = kt * kRlRows + 8 * q + 2 * (lane & 3) + e;
          if (k < p.M) {
            tms = fmaxf(tms, as[4 * q + 2 * r + e] * p.inv_tau);
            tmt = fmaxf(tmt, at[4 * q + 2 * r + e] * p.inv_tau);
          }
        }
      tms = fmaxf(tms, __shfl_xor_sync(0xffffffffu, tms, 1));
      tms = fmaxf(tms, __shfl_xor_sync(0xffffffffu, tms, 2));
      tmt = fmaxf(tmt, __shfl_xor_sync(0xffffffffu, tmt, 1));
      tmt = fmaxf(tmt, __shfl_xor_sync(0xffffffffu, tmt, 2));
      const float nms = fmaxf(ms[r], tms), nmt = fmaxf(mt[r], tmt);
      const double fs = exp(static_cast<double>(ms[r]) - nms), ft = exp(static_cast<double>(mt[r]) - nmt);
      float sl = 0.f, tl = 0.f, cx = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int k = kt * kRlRows + 8 * q + 2 * (lane & 3) + e;
          if (k < p.M) {
            const float s = as[4 * q + 2 * r + e] * p.inv_tau, t = at[4 * q + 2 * r + e] * p.inv_tau;
            const float et = expf(t - nmt);
            sl += expf(s - nms);
            tl += et;
            cx = fmaf(et, t - s, cx);
          }
        }
      ls[r] = ls[r] * fs + static_cast<double>(sl);
      lt[r] = lt[r] * ft + static_cast<double>(tl);
      cr[r] = cr[r] * ft + static_cast<double>(cx);
      ms[r] = nms;
      mt[r] = nmt;
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      ls[r] += __shfl_xor_sync(0xffffffffu, ls[r], o);
      lt[r] += __shfl_xor_sync(0xffffffffu, lt[r], o);
      cr[r] += __shfl_xor_sync(0xffffffffu, cr[r], o);
    }
    const int row = wq * 16 + (lane >> 2) + 8 * r;
    const int grow = rt * kRlRows + row;
    double kl = 0.0;
    if (grow < p.M) {
      const float lse_s = static_cast<float>(ms[r] + log(ls[r])), lse_t = static_cast<float>(mt[r] + log(lt[r]));
      // sum q (t - s) - lse_t + lse_s, with lse_t - lse_s = (m_t - m_s) + log(l_t / l_s)
      kl = cr[r] / lt[r] - (static_cast<double>(mt[r]) - ms[r]) - log(lt[r] / ls[r]);
      if ((lane & 3) == 0)
        *reinterpret_cast<float2*>(p.lse + ((static_cast<size_t>(i) * p.B + j) * p.M + grow) * 2) =
            make_float2(lse_s, lse_t);
    }
    if ((lane & 3) == 0) s_kl[row] = kl;
  }
  named_bar_sync(1, 128);
  if (ct == 0) {
    double sum = 0.0;
    for (int r = 0; r < kRlRows; ++r) sum += s_kl[r];
    p.partial[blockIdx.x] = sum;
  }
}

// loss[0] = scale * sum of the CTA partials, fp64 in a fixed order
__global__ void __launch_bounds__(256) relation_reduce_kernel(const double* __restrict__ partial, int n, double scale,
                                                              float* __restrict__ loss) {
  __shared__ double sd[256];
  double a = 0.0;
  for (int k = threadIdx.x; k < n; k += 256) a += partial[k];
  sd[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sd[threadIdx.x] += sd[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = static_cast<float>(sd[0] * scale);
}

__global__ void __launch_bounds__(256, 1)
relation_kl_bwd_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmXlo,
                       const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmYlo,
                       const RelKLParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* g_st = smem + kRlBwdStages * kRlStage;             // G as K-major A operand: hi box, lo box
  uint64_t* full = reinterpret_cast<uint64_t*>(g_st + 2 * kRlBox);
  uint64_t* empty = full + kRlBwdStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = blockIdx.x & 1;
  const int rt = (blockIdx.x >> 1) % p.tiles;
  const int n = (blockIdx.x >> 1) / p.tiles;
  const int num_kt = p.tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < kRlBwdStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 128);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    if (warp == 0 && elect_one()) {
      int it = 0;
      for (int j = 0; j < p.B; ++j)
        for (int kt = 0; kt < num_kt; ++kt) {
          rl_load_st(smem, full, empty, it, kRlBwdStages, p.nseg, &tmX, &tmXlo, &tmY, &tmYlo, n, rt * kRlRows, j,
                     kt * kRlRows);
          // the keys' channel half as the MN-major B operand of G X_j
          for (int seg = 0; seg < p.nseg; ++seg, ++it) {
            const int s = it % kRlBwdStages;
            mbar_wait(&empty[s], ((it / kRlBwdStages) & 1) ^ 1);
            uint8_t* dst = smem + s * kRlStage;
            mbar_expect_tx(&full[s], kRlStage);
            for (int b = 0; b < 4; ++b)
              tma_load_3d(dst + b * kRlBox, seg == 2 ? &tmXlo : &tmX, &full[s], (4 * half + b) * 64, kt * kRlRows, j);
          }
        }
    }
    return;
  }
  const int ct = threadIdx.x - 128, wq = ct >> 5;
  const float coef = p.coef * p.grad[0];
  float acc[128];
#pragma unroll
  for (int k = 0; k < 128; ++k) acc[k] = 0.f;
  int row[2];
  bool row_ok[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    row[r] = rt * kRlRows + wq * 16 + (lane >> 2) + 8 * r;
    row_ok[r] = row[r] < p.M;
  }
  int it = 0;
  for (int j = 0; j < p.B; ++j) {
    float2 rs[2];
#pragma unroll
    for (int r = 0; r < 2; ++r)
      rs[r] = row_ok[r] ? *reinterpret_cast<const float2*>(p.lse + ((static_cast<size_t>(n) * p.B + j) * p.M + row[r]) * 2)
                        : make_float2(0.f, 0.f);
    const float* cs_base = p.lse + (static_cast<size_t>(j) * p.B + n) * p.M * 2;
    for (int kt = 0; kt < num_kt; ++kt) {
      float as[32], at[32];
      rl_tile_st<kRlBwdStages>(smem, full, empty, it, p.nseg, as, at);
      // G = coef ((P - Q)_nj + (P - Q)_jn^T) -> bf16 (hi, lo) K-major swizzled A tile
#pragma unroll
      for (int q = 0; q < 8; ++q)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int kl = 8 * q + 2 * (lane & 3) + e;
          const int k = kt * kRlRows + kl;
          float2 cs = make_float2(0.f, 0.f);
          if (k < p.M) cs = *reinterpret_cast<const float2*>(cs_base + static_cast<size_t>(k) * 2);
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float g = 0.f;
            if (k < p.M && row_ok[r]) {
              const float s = as[4 * q + 2 * r + e] * p.inv_tau, t = at[4 * q + 2 * r + e] * p.inv_tau;
              g = coef * ((expf(s - rs[r].x) - expf(t - rs[r].y)) + (expf(s - cs.x) - expf(t - cs.y)));
            }
            const int lr = wq * 16 + (lane >> 2) + 8 * r;
            const int off = lr * 128 + (((kl >> 3) ^ (lr & 7)) << 4) + (kl & 7) * 2;
            const __nv_bfloat16 hi = __float2bfloat16_rn(g);
            *reinterpret_cast<__nv_bfloat16*>(g_st + off) = hi;
            if (p.nseg > 1) *reinterpret_cast<__nv_bfloat16*>(g_st + kRlBox + off) = __float2bfloat16_rn(g - __bfloat162float(hi));
          }
        }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
      const uint32_t ga = smem_u32(g_st);
      for (int seg = 0; seg < p.nseg; ++seg, ++it) {
        const int s = it % kRlBwdStages;
        mbar_wait(&full[s], (it / kRlBwdStages) & 1);
        const uint64_t adesc = rl_desc_kmajor(ga + (seg == 1 ? kRlBox : 0));
        const uint64_t bdesc = make_wgmma_desc_sw128(smem_u32(smem + s * kRlStage), kRlBox, 1024);
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_bf16<256, 0, 1>(acc, adesc + static_cast<uint64_t>(2 * k), bdesc + static_cast<uint64_t>(128 * k), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_operand(acc);
        mbar_arrive(&empty[s]);
      }
      named_bar_sync(1, 128);      // every warp's wgmma has read G before the next tile overwrites it
    }
  }
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (!row_ok[r]) continue;
    float* out = p.dnodes + (static_cast<size_t>(n) * p.M + row[r]) * kRlC + half * 256 + cq;
#pragma unroll
    for (int q = 0; q < 32; ++q) *reinterpret_cast<float2*>(out + 8 * q) = make_float2(acc[4 * q + 2 * r], acc[4 * q + 2 * r + 1]);
  }
}

// one warp per node, 16 channels per lane
template <bool kSIn, bool kSOut>
__global__ void __launch_bounds__(128, 1)
relation_nodes_kernel(const bf16_t* __restrict__ f, const bf16_t* __restrict__ f_lo, int pitch, int B, int h, int w,
                      int pool, int gh, int gw, bf16_t* __restrict__ out, bf16_t* __restrict__ out_lo,
                      uint8_t* __restrict__ arg, float* __restrict__ inv_norm) {
  const int node = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int M = gh * gw;
  if (node >= B * M) return;
  const int b = node / M, m = node - b * M, a = m / gw, c = m - a * gw;
  const int y0 = a * pool, x0 = c * pool, y1 = min(y0 + pool, h), x1 = min(x0 + pool, w);
  float v[16];
  uint8_t off[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    v[q] = -INFINITY;
    off[q] = 0;
  }
  for (int y = y0; y < y1; ++y)
    for (int x = x0; x < x1; ++x) {
      const long long base = ((static_cast<long long>(b) * h + y) * w + x) * pitch + 16 * lane;
      float u[16];
      act_ld8<kSIn>(f, f_lo, base, *reinterpret_cast<float(*)[8]>(u));
      act_ld8<kSIn>(f, f_lo, base + 8, *reinterpret_cast<float(*)[8]>(u + 8));
      const uint8_t o = static_cast<uint8_t>((y - y0) * pool + (x - x0));
#pragma unroll
      for (int q = 0; q < 16; ++q)
        if (u[q] > v[q]) {
          v[q] = u[q];
          off[q] = o;
        }
    }
  float ss = 0.f;
#pragma unroll
  for (int q = 0; q < 16; ++q) ss = fmaf(v[q], v[q], ss);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float nrm = sqrtf(ss);
  const float inv = nrm < 1e-12f ? 0.f : 1.f / nrm;
  float xh[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) xh[q] = v[q] * inv;
  const long long ob = static_cast<long long>(node) * kRlC + 16 * lane;
  act_st8<kSOut>(out, out_lo, ob, *reinterpret_cast<float(*)[8]>(xh));
  act_st8<kSOut>(out, out_lo, ob + 8, *reinterpret_cast<float(*)[8]>(xh + 8));
  if (arg) {
    uint4 pk;
    uint32_t* pw = reinterpret_cast<uint32_t*>(&pk);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      pw[q] = off[4 * q] | (off[4 * q + 1] << 8) | (off[4 * q + 2] << 16) | (static_cast<uint32_t>(off[4 * q + 3]) << 24);
    *reinterpret_cast<uint4*>(arg + ob) = pk;
    if (lane == 0) inv_norm[node] = inv;
  }
}

template <bool kSIn, bool kSOut>
__global__ void __launch_bounds__(128)
relation_nodes_bwd_kernel(const bf16_t* __restrict__ f, const bf16_t* __restrict__ f_lo, int pitch, int B, int h,
                          int w, int pool, int gh, int gw, const uint8_t* __restrict__ arg,
                          const float* __restrict__ inv_norm, const float* __restrict__ dnodes,
                          bf16_t* __restrict__ df, bf16_t* __restrict__ df_lo, int df_pitch) {
  const int node = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int M = gh * gw;
  if (node >= B * M) return;
  const int b = node / M, m = node - b * M, a = m / gw, c = m - a * gw;
  const int y0 = a * pool, x0 = c * pool, y1 = min(y0 + pool, h), x1 = min(x0 + pool, w);
  const long long ob = static_cast<long long>(node) * kRlC + 16 * lane;
  const float inv = inv_norm[node];
  uint8_t off[16];
  {
    const uint4 pk = *reinterpret_cast<const uint4*>(arg + ob);
    const uint32_t* pw = reinterpret_cast<const uint32_t*>(&pk);
#pragma unroll
    for (int q = 0; q < 16; ++q) off[q] = static_cast<uint8_t>(pw[q >> 2] >> (8 * (q & 3)));
  }
  float xh[16], d[16], dot = 0.f;
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int y = y0 + off[q] / pool, x = x0 + off[q] % pool;
    const long long e = ((static_cast<long long>(b) * h + y) * w + x) * pitch + 16 * lane + q;
    float xv = __bfloat162float(f[e]);
    if (kSIn) xv += __bfloat162float(f_lo[e]);
    xh[q] = xv * inv;
    d[q] = dnodes[ob + q];
    dot = fmaf(xh[q], d[q], dot);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
  float dx[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) dx[q] = (d[q] - xh[q] * dot) * inv;
  for (int y = y0; y < y1; ++y)
    for (int x = x0; x < x1; ++x) {
      const uint8_t o = static_cast<uint8_t>((y - y0) * pool + (x - x0));
      float u[16];
#pragma unroll
      for (int q = 0; q < 16; ++q) u[q] = off[q] == o ? dx[q] : 0.f;
      const long long base = ((static_cast<long long>(b) * h + y) * w + x) * df_pitch + 16 * lane;
      act_st8<kSOut>(df, df_lo, base, *reinterpret_cast<float(*)[8]>(u));
      act_st8<kSOut>(df, df_lo, base + 8, *reinterpret_cast<float(*)[8]>(u + 8));
    }
}

template <typename K>
static int set_smem_once(K kernel, int bytes, std::atomic<bool> (&flags)[64]) {
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !flags[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (dev >= 0 && dev < 64) flags[dev].store(true, std::memory_order_release);
  }
  return SEMSEG_OK;
}

static int check_grid(const char* fn, int B, int h, int w, int C, int pool) {
  SB_CHECK_ARG(B > 0 && h > 0 && w > 0, "%s: bad shape B=%d h=%d w=%d", fn, B, h, w);
  SB_CHECK_ARG(C == kRlC, "%s: the feature width must be %d (got %d)", fn, kRlC, C);
  SB_CHECK_ARG(pool >= 1 && pool <= kRlMaxPool, "%s: pool must lie in [1, %d] (got %d)", fn, kRlMaxPool, pool);
  const long long M = static_cast<long long>(cdiv(h, pool)) * cdiv(w, pool);
  SB_CHECK_ARG(static_cast<long long>(B) * M < (1LL << 24) && static_cast<long long>(B) * B * M < (1LL << 30),
               "%s: too many nodes (B=%d, M=%lld)", fn, B, M);
  return SEMSEG_OK;
}

static int check_nodes_ptr(const char* fn, const void* x, const void* x_lo) {
  SB_CHECK_ARG(x != nullptr, "%s: null node operand", fn);
  SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(x_lo)) & 15) == 0,
               "%s: node operand %p (lo %p) is not 16-byte aligned", fn, x, x_lo);
  return SEMSEG_OK;
}

static int check_kl(const char* fn, const void* xs, const void* xs_lo, const void* xt, const void* xt_lo, int B, int M,
                    int C, float tau) {
  SB_CHECK_ARG(B > 0 && M > 0 && static_cast<long long>(B) * B * M < (1LL << 30), "%s: bad shape B=%d M=%d", fn, B, M);
  SB_CHECK_ARG(C == kRlC, "%s: the node width must be %d (got %d)", fn, kRlC, C);
  SB_CHECK_ARG(isfinite(tau) && tau > 0.f, "%s: temperature must be finite and > 0 (got %g)", fn,
               static_cast<double>(tau));
  SB_CHECK_ARG((xs_lo != nullptr) == (xt_lo != nullptr), "%s: student and teacher nodes must share one operand form",
               fn);
  if (const int r = check_nodes_ptr(fn, xs, xs_lo)) return r;
  if (const int r = check_nodes_ptr(fn, xt, xt_lo)) return r;
  return SEMSEG_OK;
}

static int encode_nodes(CUtensorMap* m, const void* x, int B, int M) {
  uint64_t dims[3] = {(uint64_t)kRlC, (uint64_t)M, (uint64_t)B};
  uint64_t str[2] = {(uint64_t)kRlC * 2, (uint64_t)kRlC * 2 * M};
  uint32_t box[3] = {64u, (uint32_t)kRlRows, 1u};
  return encode_tmap_bf16(m, x, 3, dims, str, box);
}

static int encode_pair(CUtensorMap* m, CUtensorMap* ml, const void* x, const void* x_lo, int B, int M) {
  if (const int r = encode_nodes(m, x, B, M)) return r;
  *ml = *m;
  if (x_lo) return encode_nodes(ml, x_lo, B, M);
  return SEMSEG_OK;
}

}  // namespace sb

extern "C" int semseg_relation_nodes(const void* feat, const void* feat_lo, int pitch, int B, int h, int w, int C,
                                     int pool, void* nodes, void* nodes_lo, unsigned char* argmax, float* inv_norm,
                                     void* stream_) {
  using namespace sb;
  const char* fn = "relation_nodes";
  SB_CHECK_ARG(feat && nodes, "%s: null feature or node pointer", fn);
  if (const int r = check_grid(fn, B, h, w, C, pool)) return r;
  SB_CHECK_ARG(pitch % 8 == 0, "%s: pitch %d is not a multiple of 8", fn, pitch);
  SB_CHECK_ARG((argmax != nullptr) == (inv_norm != nullptr), "%s: argmax and inv_norm go together", fn);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(argmax) & 15) == 0 && (reinterpret_cast<uintptr_t>(inv_norm) & 3) == 0,
               "%s: argmax must be 16-byte and inv_norm 4-byte aligned", fn);
  if (const int r = check_vec_acts(fn, C, {{feat, feat_lo, pitch}})) return r;
  if (const int r = check_nodes_ptr(fn, nodes, nodes_lo)) return r;
  const int gh = cdiv(h, pool), gw = cdiv(w, pool);
  const int nn = B * gh * gw;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bf16_t* fi = static_cast<const bf16_t*>(feat);
  const bf16_t* fl = static_cast<const bf16_t*>(feat_lo);
  bf16_t* o = static_cast<bf16_t*>(nodes);
  bf16_t* ol = static_cast<bf16_t*>(nodes_lo);
  const dim3 grid(cdiv(nn, 4));
  if (feat_lo) {
    if (nodes_lo) relation_nodes_kernel<true, true><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, o, ol, argmax, inv_norm);
    else relation_nodes_kernel<true, false><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, o, ol, argmax, inv_norm);
  } else {
    if (nodes_lo) relation_nodes_kernel<false, true><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, o, ol, argmax, inv_norm);
    else relation_nodes_kernel<false, false><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, o, ol, argmax, inv_norm);
  }
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" long long semseg_relation_workspace_floats(int B, int M) {
  if (B <= 0 || M <= 0 || static_cast<long long>(B) * B * M >= (1LL << 30)) return -1;
  return 2LL * B * B * sb::cdiv(M, sb::kRlRows);
}

extern "C" int semseg_relation_kl_fwd(const void* xs, const void* xs_lo, const void* xt, const void* xt_lo, int B,
                                      int M, int C, float temperature, float* workspace, float* lse, float* loss,
                                      void* stream_) {
  using namespace sb;
  const char* fn = "relation_kl_fwd";
  if (const int r = check_kl(fn, xs, xs_lo, xt, xt_lo, B, M, C, temperature)) return r;
  SB_CHECK_ARG(workspace && lse && loss, "%s: null workspace, lse or loss", fn);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 7) == 0 && (reinterpret_cast<uintptr_t>(lse) & 7) == 0,
               "%s: workspace and lse must be 8-byte aligned", fn);
  RelKLParams p;
  memset(&p, 0, sizeof(p));
  p.lse = lse;
  p.partial = reinterpret_cast<double*>(workspace);
  p.B = B; p.M = M; p.tiles = cdiv(M, kRlRows); p.nseg = xs_lo ? 3 : 1;
  p.inv_tau = 1.f / temperature;
  CUtensorMap tx, txl, ty, tyl;
  if (const int r = encode_pair(&tx, &txl, xs, xs_lo, B, M)) return r;
  if (const int r = encode_pair(&ty, &tyl, xt, xt_lo, B, M)) return r;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static std::atomic<bool> attr[64];
  if (const int r = set_smem_once(relation_kl_fwd_kernel, kRlFwdSmem, attr)) return r;
  const int grid = B * B * p.tiles;
  relation_kl_fwd_kernel<<<grid, 256, kRlFwdSmem, stream>>>(tx, txl, ty, tyl, p);
  SB_LAUNCHED();
  const double t = static_cast<double>(temperature);
  relation_reduce_kernel<<<1, 256, 0, stream>>>(p.partial, grid, t * t / (static_cast<double>(B) * B * M), loss);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_relation_kl_bwd(const void* xs, const void* xs_lo, const void* xt, const void* xt_lo, int B,
                                      int M, int C, float temperature, const float* lse, const float* grad_out,
                                      float* dnodes, void* stream_) {
  using namespace sb;
  const char* fn = "relation_kl_bwd";
  if (const int r = check_kl(fn, xs, xs_lo, xt, xt_lo, B, M, C, temperature)) return r;
  SB_CHECK_ARG(lse && grad_out && dnodes, "%s: null lse, grad_out or dnodes", fn);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(lse) & 7) == 0 && (reinterpret_cast<uintptr_t>(dnodes) & 7) == 0,
               "%s: lse and dnodes must be 8-byte aligned", fn);
  RelKLParams p;
  memset(&p, 0, sizeof(p));
  p.lse = const_cast<float*>(lse);
  p.grad = grad_out;
  p.dnodes = dnodes;
  p.B = B; p.M = M; p.tiles = cdiv(M, kRlRows); p.nseg = xs_lo ? 3 : 1;
  p.inv_tau = 1.f / temperature;
  p.coef = static_cast<float>(static_cast<double>(temperature) / (static_cast<double>(B) * B * M));
  CUtensorMap tx, txl, ty, tyl;
  if (const int r = encode_pair(&tx, &txl, xs, xs_lo, B, M)) return r;
  if (const int r = encode_pair(&ty, &tyl, xt, xt_lo, B, M)) return r;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static std::atomic<bool> attr[64];
  if (const int r = set_smem_once(relation_kl_bwd_kernel, kRlBwdSmem, attr)) return r;
  relation_kl_bwd_kernel<<<B * p.tiles * 2, 256, kRlBwdSmem, stream>>>(tx, txl, ty, tyl, p);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_relation_nodes_bwd(const void* feat, const void* feat_lo, int pitch, int B, int h, int w, int C,
                                         int pool, const unsigned char* argmax, const float* inv_norm,
                                         const float* dnodes, void* dfeat, void* dfeat_lo, int dfeat_pitch,
                                         void* stream_) {
  using namespace sb;
  const char* fn = "relation_nodes_bwd";
  SB_CHECK_ARG(feat && argmax && inv_norm && dnodes && dfeat, "%s: null pointer", fn);
  if (const int r = check_grid(fn, B, h, w, C, pool)) return r;
  SB_CHECK_ARG(pitch % 8 == 0 && dfeat_pitch % 8 == 0, "%s: pitches must be multiples of 8", fn);
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(argmax) & 15) == 0, "%s: argmax must be 16-byte aligned", fn);
  if (const int r = check_vec_acts(fn, C, {{feat, feat_lo, pitch}, {dfeat, dfeat_lo, dfeat_pitch}})) return r;
  const int gh = cdiv(h, pool), gw = cdiv(w, pool);
  const int nn = B * gh * gw;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bf16_t* fi = static_cast<const bf16_t*>(feat);
  const bf16_t* fl = static_cast<const bf16_t*>(feat_lo);
  bf16_t* o = static_cast<bf16_t*>(dfeat);
  bf16_t* ol = static_cast<bf16_t*>(dfeat_lo);
  const dim3 grid(cdiv(nn, 4));
  if (feat_lo) {
    if (dfeat_lo) relation_nodes_bwd_kernel<true, true><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, argmax, inv_norm, dnodes, o, ol, dfeat_pitch);
    else relation_nodes_bwd_kernel<true, false><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, argmax, inv_norm, dnodes, o, ol, dfeat_pitch);
  } else {
    if (dfeat_lo) relation_nodes_bwd_kernel<false, true><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, argmax, inv_norm, dnodes, o, ol, dfeat_pitch);
    else relation_nodes_bwd_kernel<false, false><<<grid, 128, 0, stream>>>(fi, fl, pitch, B, h, w, pool, gh, gw, argmax, inv_norm, dnodes, o, ol, dfeat_pitch);
  }
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// Fused point-wise spatial attention (SURVEY.md §8 f2): mask gather -> softmax -> aggregation in ONE kernel, so that
// the [N, HW, HW] attention map of model/psanet.py:81-91 (psa_mask -> F.softmax(dim=1) -> torch.bmm, three fp32 round
// trips of a 3.24 MB/image/branch tensor plus an NHWC->NCHW copy of the 12.5 MB logits) never exists in HBM.
//
// Per image:   out[t, :] = (1/norm) * sum_s P[t, s] * feat[s, :],   P[t, :] = softmax_s( L[t, s] )
//   collect    (psa_type 0): L[t, s] = A[t, idx(s - t)]   (the TARGET pixel's own 59x59 attention vector)
//   distribute (psa_type 1): L[t, s] = A[s, idx(t - s)]   (one entry of every SOURCE pixel's vector)
//   idx(d) = (d.y + hh) * mW + (d.x + hw); positions outside the mask window contribute logit 0 (the reference zero-fills
//   psa_mask's output BEFORE the softmax, lib/psa/functions/psamask.py:17).
// Two more forms of the same gather (template parameters; the window + softmax instances are the original kernels):
//   dense (compact=True, model/psanet.py:76-79): mH*mW == HW and the owner's vector is indexed by the other pixel's flat
//     position, L[t, s] = A[t, s] (collect) or A[s, t] (distribute: the reference's view(n,hw,hw).transpose(1,2));
//   no softmax (psa_softmax=False): P = L, no statistics are computed or read.
// A = attention logits fp32 NHWC [N, HW, a_pitch] straight from the 1x1 conv's F32 epilogue (no NCHW copy).
//
// One kernel template covers the forward aggregation AND the feature gradient of the backward pass, which is the same
// contraction with rows and reduction index swapped:  dfeat[s, :] = (1/norm) * sum_t P[t, s] * dout[t, :].
//   kRowOwner : the attention vector of element (row, k) belongs to the row pixel (else to the k pixel)
//   kStatsRow : the softmax statistics (max, 1/sum) of element (row, k) belong to the row (else to k)
//     forward  collect: (1,1)   forward distribute: (0,1)   dfeat collect: (0,0)   dfeat distribute: (1,0)
//
// CTA = a run of <= 64 consecutive pixel positions (rows) of one image. 64 rows x 512 fp32 accumulator columns is half
// of the register file, so the tile is 64 rows rather than 128.
//   warpgroup 0    : TMA producer of the B operand (one elected thread): feat/dout K blocks [64 pixels x 512 channels]
//                    bf16 as eight [64 ch, 64 px] boxes = MN-major SWIZZLE_128B operand (the wgrad kernel's operand form)
//   warpgroups 1-2 : (a) softmax statistics of the CTA's rows (forward), (b) per K block: gather 64 x 64 logits, exp,
//                    normalise, bf16 -> K-major SWIZZLE_128B A-operand stage in shared memory, then warpgroup w issues
//                    wgmma D[64 x 256 fp32 registers] += P[64 x 64] * B[64 x columns 256w..256w+255],
//                    (c) epilogue: registers -> scale -> bf16 (or hi/lo pair) -> global.
// bf16x3 (split feat / out): the K loop runs three times (P_hi*B_hi, P_lo*B_hi, P_hi*B_lo) into the same accumulator.
#include "host_common.h"
#include "ptx.cuh"
#include "act.cuh"

namespace sb {

constexpr int kPfRows = 64;
constexpr int kPfK = 64;
constexpr int kPfC = 512;                         // channels of feat / out (mid_channels of the PSA module)
constexpr int kPfBoxBytes = kPfK * 128;           // one [64 ch, 64 px] box
constexpr int kPfBBytes = (kPfC / 64) * kPfBoxBytes;   // 64 KB
constexpr int kPfABytes = kPfRows * 128;          // 8 KB
constexpr int kPfStageBytes = kPfABytes + kPfBBytes;
constexpr int kPfStages = 2;
constexpr int kPfWorkers = 256;                   // warpgroups 1, 2
constexpr int kPfThreads = 128 + kPfWorkers;
constexpr int kPfMisc = 256 + 2 * kPfRows * 4 + 2 * 8 * kPfRows * 4;   // barriers, row stats, per-warp partial stats
constexpr int kPfSmem = kPfStages * kPfStageBytes + kPfMisc + 1024;

struct PsaFusedParams {
  const float* A;       // [N][Q][a_pitch]
  float2* stats;        // [N][Q] (max, 1/sum) per target; written when kStatsRow (forward), read otherwise
  __nv_bfloat16* out;   // [N][Q][out_pitch]
  __nv_bfloat16* out_lo;
  int out_pitch;
  int N, H, W, mH, mW, a_pitch;
  int tile_rows;        // pixel positions per CTA tile (<= kPfRows)
  int tiles_per_img;
  int nseg;             // 1 (bf16) or 3 (bf16x3)
  float scale;          // 1 / normalization_factor
};

// logit of attention element (own, other): window form = the owner's mask entry at offset other - own, zero outside the
// window; dense form = the owner's entry at the other pixel's flat position `oth`
template <bool kDense>
__device__ __forceinline__ float pf_logit(const float* __restrict__ An, int a_pitch, int own, int own_i, int own_j,
                                          int oth, int oth_i, int oth_j, int hh, int hw, int mH, int mW) {
  if (kDense) return __ldg(An + static_cast<size_t>(own) * a_pitch + oth);
  const int a = oth_i - own_i + hh, b = oth_j - own_j + hw;
  return (a >= 0 && a < mH && b >= 0 && b < mW) ? __ldg(An + static_cast<size_t>(own) * a_pitch + a * mW + b) : 0.f;
}

template <bool kRowOwner, bool kStatsRow, bool kDense, bool kSoftmax>
__global__ void __launch_bounds__(kPfThreads, 1)
psa_attend_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmB_lo,
                  const PsaFusedParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* misc = smem + kPfStages * kPfStageBytes;
  uint64_t* full_b = reinterpret_cast<uint64_t*>(misc);       // TMA bytes of the B tile landed
  uint64_t* empty = full_b + kPfStages;                       // MMAs that read the stage completed
  float* s_m = reinterpret_cast<float*>(misc + 256);          // [64] row max
  float* s_inv = s_m + kPfRows;                               // [64] row 1/sum

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x / p.tiles_per_img;
  const int tile = blockIdx.x - n * p.tiles_per_img;
  const int Q = p.H * p.W;
  const int pos0 = tile * p.tile_rows;                                   // first pixel position of this tile
  const int live_rows = min(p.tile_rows, Q - pos0);                      // rows of the tile that exist
  const int hh = (p.mH - 1) / 2, hw = (p.mW - 1) / 2;
  const int num_kb = (Q + kPfK - 1) / kPfK;
  const int total_kb = num_kb * p.nseg;
  const float* An = p.A + static_cast<size_t>(n) * Q * p.a_pitch;
  float2* stats_n = p.stats + static_cast<size_t>(n) * Q;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmB);
    if (p.nseg > 1) tma_prefetch_desc(&tmB_lo);
    for (int i = 0; i < kPfStages; ++i) {
      mbar_init(&full_b[i], 1);
      mbar_init(&empty[i], kPfWorkers);
    }
    fence_barrier_init();
  }
  // rows of the 64-row A tile that do not exist in this CTA's tile stay zero for the whole kernel
  for (int s = 0; s < kPfStages; ++s) {
    uint4* a4 = reinterpret_cast<uint4*>(smem + s * kPfStageBytes);
    for (int i = threadIdx.x; i < kPfABytes / 16; i += kPfThreads) a4[i] = make_uint4(0, 0, 0, 0);
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp < 4) {
    // ===================================================================== TMA producer (B operand)
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      for (int it = 0; it < total_kb; ++it) {
        const int s = it % kPfStages;
        const uint32_t par = (it / kPfStages) & 1;
        mbar_wait(&empty[s], par ^ 1);
        const int seg = it / num_kb, kb = it - seg * num_kb;
        const CUtensorMap* m = (seg == 2) ? &tmB_lo : &tmB;
        uint8_t* dst = smem + s * kPfStageBytes + kPfABytes;
        mbar_expect_tx(&full_b[s], kPfBBytes);
#pragma unroll
        for (int bx = 0; bx < kPfC / 64; ++bx) tma_load_3d(dst + bx * kPfBoxBytes, m, &full_b[s], bx * 64, kb * kPfK, n);
      }
    }
    return;
  }
  // ===================================================================== workers: statistics, P tiles, MMA, epilogue
  setmaxnreg_inc<232>();
  const int wt = threadIdx.x - 128;         // 0..255
  const int ww = wt >> 5;                    // worker warp 0..7
  // ---- (a) softmax statistics of the tile's rows (forward kernels)
  if (kSoftmax && kStatsRow) {
    if (kRowOwner) {
      // collect: row = target, its own attention vector, contiguous along the source column -> one warp per row
      for (int r = ww; r < kPfRows; r += kPfWorkers / 32) {
        float m = -INFINITY, sum = 0.f;
        if (r < live_rows) {
          const int own = pos0 + r, ri = own / p.W, rj = own - ri * p.W;
          for (int q = lane; q < Q; q += 32)
            m = fmaxf(m, pf_logit<kDense>(An, p.a_pitch, own, ri, rj, q, q / p.W, q % p.W, hh, hw, p.mH, p.mW));
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
          for (int q = lane; q < Q; q += 32)
            sum += __expf(pf_logit<kDense>(An, p.a_pitch, own, ri, rj, q, q / p.W, q % p.W, hh, hw, p.mH, p.mW) - m);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
          if (lane == 0) stats_n[own] = make_float2(m, 1.f / sum);
        }
        if (lane == 0) {
          s_m[r] = m;
          s_inv[r] = (r < live_rows) ? 1.f / sum : 0.f;
        }
      }
    } else {
      // distribute: row = target, one entry of every source vector; consecutive rows read consecutive addresses ->
      // lanes along rows, the sources split over the 8 worker warps (online softmax), partials merged through smem
      float* pm = reinterpret_cast<float*>(misc + 256 + 2 * kPfRows * 4);   // [8][64] partial max
      float* ps = pm + 8 * kPfRows;                                           // [8][64] partial sum
      const int q_per = (Q + 7) / 8, q0 = ww * q_per, q1 = min(Q, q0 + q_per);
      for (int r = lane; r < kPfRows; r += 32) {
        float m = -INFINITY, sum = 0.f;
        if (r < live_rows) {
          const int pos = pos0 + r, ri = pos / p.W, rj = pos - ri * p.W;
          for (int q = q0; q < q1; ++q) {
            const float l = pf_logit<kDense>(An, p.a_pitch, q, q / p.W, q % p.W, pos, ri, rj, hh, hw, p.mH, p.mW);
            const float mn = fmaxf(m, l);
            sum = sum * __expf(m - mn) + __expf(l - mn);
            m = mn;
          }
        }
        pm[ww * kPfRows + r] = m;
        ps[ww * kPfRows + r] = sum;
      }
      named_bar_sync(1, kPfWorkers);
      if (wt < kPfRows) {
        const int r = wt;
        float m = -INFINITY, sum = 0.f;
        if (r < live_rows) {
#pragma unroll
          for (int k = 0; k < 8; ++k) m = fmaxf(m, pm[k * kPfRows + r]);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float mk = pm[k * kPfRows + r];
            if (mk > -INFINITY) sum += ps[k * kPfRows + r] * __expf(mk - m);
          }
          stats_n[pos0 + r] = make_float2(m, 1.f / sum);
        }
        s_m[r] = m;
        s_inv[r] = (r < live_rows) ? 1.f / sum : 0.f;
      }
    }
    named_bar_sync(1, kPfWorkers);
  }
  // ---- (b) P tiles and MMAs
  const int wg = wt >> 7;                    // accumulator columns [256 wg, 256 wg + 256)
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  int prev_s = -1;
  for (int it = 0; it < total_kb; ++it) {
    const int s = it % kPfStages;
    const uint32_t par = (it / kPfStages) & 1;
    const int seg = it / num_kb, kb = it - seg * num_kb;
    mbar_wait(&empty[s], par ^ 1);
    uint8_t* a_st = smem + s * kPfStageBytes;
    const bool want_lo = seg == 1;
    if (kRowOwner) {
      // the row pixel owns the attention vector -> addresses are contiguous along k: one warp per (row, 32-column
      // half), lanes along k; the live (row, half) items are dealt round-robin to the 8 worker warps
      // [forward collect, dfeat distribute]
      for (int item = ww; item < 2 * live_rows; item += kPfWorkers / 32) {
        const int r = item >> 1, half = item & 1;
        const int rpos = pos0 + r, ri = rpos / p.W, rj = rpos - ri * p.W;
        const int kl = half * 32 + lane, q = kb * kPfK + kl;
        float pv = 0.f;
        if (q < Q) {
          const int qi = q / p.W, qj = q - qi * p.W;
          const float l = pf_logit<kDense>(An, p.a_pitch, rpos, ri, rj, q, qi, qj, hh, hw, p.mH, p.mW);
          if (!kSoftmax) {
            pv = l;
          } else if (kStatsRow) {
            pv = __expf(l - s_m[r]) * s_inv[r];
          } else {
            const float2 st = stats_n[q];
            pv = __expf(l - st.x) * st.y;
          }
        }
        __nv_bfloat16 hi = __float2bfloat16_rn(pv);
        if (want_lo) hi = __float2bfloat16_rn(pv - __bfloat162float(hi));
        *reinterpret_cast<__nv_bfloat16*>(a_st + r * 128 + (((kl >> 3) ^ (r & 7)) << 4) + (kl & 7) * 2) = hi;
      }
    } else {
      // the k pixel owns the vector -> addresses are contiguous along the row index: lanes along rows; the
      // (32-row group, k column) items are dealt round-robin to the 8 worker warps  [forward distribute, dfeat collect]
      const int row_groups = (live_rows + 31) >> 5;
      for (int item = ww; item < row_groups * kPfK; item += kPfWorkers / 32) {
        const int rg = item % row_groups, kl = item / row_groups;
        const int r = rg * 32 + lane, q = kb * kPfK + kl;
        if (r >= live_rows) continue;
        float pv = 0.f;
        if (q < Q) {
          const int pos = pos0 + r, ri = pos / p.W, rj = pos - ri * p.W;
          const int qi = q / p.W, qj = q - qi * p.W;
          const float l = pf_logit<kDense>(An, p.a_pitch, q, qi, qj, pos, ri, rj, hh, hw, p.mH, p.mW);
          if (!kSoftmax) {
            pv = l;
          } else if (kStatsRow) {
            pv = __expf(l - s_m[r]) * s_inv[r];
          } else {
            const float2 st = stats_n[q];
            pv = __expf(l - st.x) * st.y;
          }
        }
        __nv_bfloat16 hi = __float2bfloat16_rn(pv);
        if (want_lo) hi = __float2bfloat16_rn(pv - __bfloat162float(hi));
        *reinterpret_cast<__nv_bfloat16*>(a_st + r * 128 + (((kl >> 3) ^ (r & 7)) << 4) + (kl & 7) * 2) = hi;
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(1, kPfWorkers);           // the whole P tile is in shared memory
    mbar_wait(&full_b[s], par);
    const uint32_t a_addr = smem_u32(a_st);
    const uint64_t adesc = make_wgmma_desc_sw128(a_addr, 16, 1024);
    const uint64_t bdesc = make_wgmma_desc_sw128(a_addr + kPfABytes + wg * 4 * kPfBoxBytes, kPfBoxBytes, 1024);
    wgmma_fence_operand(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kPfK / 16; ++k)
      wgmma_bf16<256, 0, 1>(acc, adesc + static_cast<uint64_t>(k * 2), bdesc + static_cast<uint64_t>(k * 128),
                            (it > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_operand(acc);
    if (prev_s >= 0) mbar_arrive(&empty[prev_s]);
    prev_s = s;
  }
  wgmma_wait<0>();
  wgmma_fence_operand(acc);
  // ---- (c) epilogue: registers -> scale -> bf16 (hi/lo) -> global
  const int wq = (wt >> 5) & 3;
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = wq * 16 + (lane >> 2) + 8 * i;
    if (r >= live_rows) continue;
    const long long orow = (static_cast<long long>(n) * Q + pos0 + r) * p.out_pitch + wg * 256 + cq;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const float v0 = acc[4 * j + 2 * i] * p.scale, v1 = acc[4 * j + 2 * i + 1] * p.scale;
      const uint32_t h = pack_bf16x2(v0, v1);
      *reinterpret_cast<uint32_t*>(p.out + orow + 8 * j) = h;
      if (p.out_lo) {
        const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&h));
        *reinterpret_cast<uint32_t*>(p.out_lo + orow + 8 * j) = pack_bf16x2(v0 - hf.x, v1 - hf.y);
      }
    }
  }
}

template <bool kRowOwner, bool kStatsRow, bool kDense, bool kSoftmax>
static int launch_attend(const CUtensorMap& tmB, const CUtensorMap& tmB_lo, const PsaFusedParams& p, int grid,
                         cudaStream_t stream) {
  static std::atomic<bool> attr_set[64];
  const auto kernel = psa_attend_kernel<kRowOwner, kStatsRow, kDense, kSoftmax>;
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPfSmem));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  kernel<<<grid, kPfThreads, kPfSmem, stream>>>(tmB, tmB_lo, p);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

// (row owner, stats on row): forward collect (1,1), forward distribute (0,1), dfeat collect (0,0), dfeat distribute (1,0).
// Without softmax there are no statistics, so only the owner side differs between the four.
template <bool kDense, bool kSoftmax>
static int launch_attend_form(int mode, int psa_type, const CUtensorMap& tmB, const CUtensorMap& tmB_lo,
                              const PsaFusedParams& p, int grid, cudaStream_t stream) {
  if (!kSoftmax)
    return (mode == 0) == (psa_type == 0) ? launch_attend<true, false, kDense, false>(tmB, tmB_lo, p, grid, stream)
                                          : launch_attend<false, false, kDense, false>(tmB, tmB_lo, p, grid, stream);
  if (mode == 0) return psa_type == 0 ? launch_attend<true, true, kDense, true>(tmB, tmB_lo, p, grid, stream)
                                      : launch_attend<false, true, kDense, true>(tmB, tmB_lo, p, grid, stream);
  return psa_type == 0 ? launch_attend<false, false, kDense, true>(tmB, tmB_lo, p, grid, stream)
                       : launch_attend<true, false, kDense, true>(tmB, tmB_lo, p, grid, stream);
}

// Pixel positions per CTA tile: `max_rows`, fewer when that leaves SMs idle (`blocks_per_tile` CTAs share a tile).
static int psa_tile_rows(int N, int Q, int max_rows, int blocks_per_tile) {
  const long long want = static_cast<long long>(N) * Q * blocks_per_tile / num_sms();
  if (want >= max_rows) return max_rows;
  return want < 8 ? 8 : static_cast<int>(want);
}

}  // namespace sb

namespace sb {

// form bits of the _ex entry points: the mask form and the softmax switch shared by the forward and backward checks.
// Both kernels read (and the forward writes) stats as float2.
static int check_psa_form(const char* fn, int form, int H, int W, int mH, int mW, int a_pitch, const float* stats) {
  const bool has_stats = stats != nullptr;
  SB_CHECK_ARG((reinterpret_cast<uintptr_t>(stats) & 7) == 0, "%s: stats %p is not 8-byte aligned", fn,
               static_cast<const void*>(stats));
  SB_CHECK_ARG((form & ~(SEMSEG_PSA_DENSE | SEMSEG_PSA_NO_SOFTMAX)) == 0, "%s: unknown form bits 0x%x", fn, form);
  if (form & SEMSEG_PSA_DENSE)
    SB_CHECK_ARG(mH > 0 && mW > 0 && mH * mW == H * W && a_pitch >= H * W,
                 "%s: bad mask geometry: the dense form needs mH*mW == H*W (%d x %d for %d x %d) and a_pitch >= H*W", fn,
                 mH, mW, H, W);
  else
    SB_CHECK_ARG(mH > 0 && mW > 0 && (mH & 1) && (mW & 1) && a_pitch >= mH * mW, "%s: bad mask geometry", fn);
  SB_CHECK_ARG(has_stats || (form & SEMSEG_PSA_NO_SOFTMAX), "%s: stats are required with softmax", fn);
  return SEMSEG_OK;
}

}  // namespace sb

// mode 0: out = P * feat (forward; writes stats)      mode 1: dfeat = P^T * dout (backward; reads stats)
extern "C" int semseg_psa_attend(int mode, int psa_type, const float* attn, int a_pitch, const void* feat,
                                 const void* feat_lo, int feat_pitch, float* stats, void* out, void* out_lo, int out_pitch,
                                 int N, int H, int W, int mH, int mW, int C, float scale, void* stream_) {
  return semseg_psa_attend_ex(mode, psa_type, 0, attn, a_pitch, feat, feat_lo, feat_pitch, stats, out, out_lo, out_pitch,
                              N, H, W, mH, mW, C, scale, stream_);
}

extern "C" int semseg_psa_attend_ex(int mode, int psa_type, int form, const float* attn, int a_pitch, const void* feat,
                                    const void* feat_lo, int feat_pitch, float* stats, void* out, void* out_lo,
                                    int out_pitch, int N, int H, int W, int mH, int mW, int C, float scale, void* stream_) {
  using namespace sb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(attn && feat && out && N > 0 && H > 0 && W > 0, "psa_attend: bad args");
  SB_CHECK_ARG(mode == 0 || mode == 1, "psa_attend: mode must be 0 (forward) or 1 (feature gradient)");
  SB_CHECK_ARG(psa_type == 0 || psa_type == 1, "psa_attend: psa_type must be 0 (collect) or 1 (distribute)");
  if (const int r = check_psa_form("psa_attend", form, H, W, mH, mW, a_pitch, stats)) return r;
  SB_CHECK_ARG(C == kPfC, "psa_attend: feature width must be %d (got %d)", kPfC, C);
  SB_CHECK_ARG(W <= 128, "psa_attend: feature maps wider than %d are not supported", 128);
  SB_CHECK_ARG(feat_pitch % 8 == 0 && out_pitch % 8 == 0 && feat_pitch >= C && out_pitch >= C, "psa_attend: bad pitch");
  SB_CHECK_ARG((feat_lo != nullptr) == (out_lo != nullptr), "psa_attend: feat and out must use the same storage form");
  // feat through TMA (16-byte global addresses), out stored as bf16 pairs
  if (const int r = check_vec_acts("psa_attend", C, {{feat, feat_lo, feat_pitch}})) return r;
  if (const int r = check_vec_acts("psa_attend", C, {{out, out_lo, out_pitch}}, 4)) return r;
  PsaFusedParams p;
  memset(&p, 0, sizeof(p));
  p.A = attn; p.stats = reinterpret_cast<float2*>(stats);
  p.out = static_cast<__nv_bfloat16*>(out); p.out_lo = static_cast<__nv_bfloat16*>(out_lo); p.out_pitch = out_pitch;
  p.N = N; p.H = H; p.W = W; p.mH = mH; p.mW = mW; p.a_pitch = a_pitch;
  // the tensor-core work is negligible, the per-row gather / exp work of the workers is what takes the time: tiles
  // shrink below 64 rows when 64 would leave SMs idle
  p.tile_rows = psa_tile_rows(N, H * W, kPfRows, 1);
  p.tiles_per_img = cdiv(H * W, p.tile_rows);
  p.nseg = feat_lo ? 3 : 1;
  p.scale = scale;
  CUtensorMap tmB, tmB_lo;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)H * W, (uint64_t)N};
    uint64_t str[2] = {(uint64_t)feat_pitch * 2, (uint64_t)feat_pitch * 2 * H * W};
    uint32_t box[3] = {64u, (uint32_t)kPfK, 1u};
    int r = encode_tmap_bf16(&tmB, feat, 3, dims, str, box);
    if (r) return r;
    tmB_lo = tmB;
    if (feat_lo && (r = encode_tmap_bf16(&tmB_lo, feat_lo, 3, dims, str, box))) return r;
  }
  const int grid = N * p.tiles_per_img;
  switch (form) {
    case 0: return launch_attend_form<false, true>(mode, psa_type, tmB, tmB_lo, p, grid, stream);
    case SEMSEG_PSA_DENSE: return launch_attend_form<true, true>(mode, psa_type, tmB, tmB_lo, p, grid, stream);
    case SEMSEG_PSA_NO_SOFTMAX: return launch_attend_form<false, false>(mode, psa_type, tmB, tmB_lo, p, grid, stream);
    default: return launch_attend_form<true, false>(mode, psa_type, tmB, tmB_lo, p, grid, stream);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Attention-logit gradient of the fused op (the softmax backward, flash-attention style: nothing [HW x HW] is stored):
//   dP[t, s] = scale * sum_c dout[t, c] * feat[s, c]                       (GEMM on wgmma: M = targets, N = sources, K = C)
//   D[t]     = sum_c dout[t, c] * out[t, c]            (= sum_s P[t, s] * dP[t, s])
//   dL[t, s] = P[t, s] * (dP[t, s] - D[t])             P recomputed from the logits and the saved (max, 1/sum)
//   dA[owner][idx(other - owner)] = dL[t, s]           owner = t (collect) or s (distribute); dA is zero elsewhere (caller
//                                                      zero-fills it: 74 % of a full 59x59 mask never receives gradient)
// Dense form: dA[owner][other] = dL[t, s], every entry is written. Without softmax: dL[t, s] = dP[t, s], so D, out and the
// statistics are not read.
// CTA = <= 128 consecutive target positions x one block of 256 sources; warpgroup 0 = TMA producer, warpgroup 1 + w
// computes targets [64w, 64w + 64) with wgmma into registers; operands K-major from TMA ([64 c, 128 rows] of dout,
// [64 c, 256 rows] of feat), 4-stage ring.
namespace sb {

constexpr int kPgBlockN = 256;
constexpr int kPgABytes = 128 * 128;             // [128 rows][64 c] bf16
constexpr int kPgBBytes = kPgBlockN * 128;       // [256 rows][64 c]
constexpr int kPgStageBytes = kPgABytes + kPgBBytes;   // 48 KB
constexpr int kPgStages = 4;
constexpr int kPgThreads = 384;
constexpr int kPgSmem = kPgStages * kPgStageBytes + 1024 + 1024;

struct PsaGradParams {
  const float* A;
  const float2* stats;
  float* dA;
  const __nv_bfloat16* dout;
  const __nv_bfloat16* dout_lo;
  const __nv_bfloat16* out;
  const __nv_bfloat16* out_lo;
  int dout_pitch, out_pitch;
  int N, H, W, mH, mW, a_pitch, C;
  int tile_rows, tiles_per_img, nseg;
  float scale;
};

template <bool kCollect, bool kDense, bool kSoftmax>
__global__ void __launch_bounds__(kPgThreads, 1)
psa_attn_grad_kernel(const __grid_constant__ CUtensorMap tmDO, const __grid_constant__ CUtensorMap tmDO_lo,
                     const __grid_constant__ CUtensorMap tmF, const __grid_constant__ CUtensorMap tmF_lo,
                     const PsaGradParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* misc = smem + kPgStages * kPgStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(misc);
  uint64_t* empty = full + kPgStages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x / p.tiles_per_img;
  const int tile = blockIdx.x - n * p.tiles_per_img;
  const int Q = p.H * p.W;
  const int q_row0 = tile * p.tile_rows;                                 // first target position of the tile
  const int live_rows = min(p.tile_rows, Q - q_row0);
  const int hh = (p.mH - 1) / 2, hw = (p.mW - 1) / 2;
  const int k_blocks = p.C / 64;
  // one 256-source block per CTA (blockIdx.y): the per-element epilogue (recompute P, scatter) dominates, so the source
  // blocks of a target tile run on different SMs
  const int nb = blockIdx.y;
  const int per_nb = k_blocks * p.nseg;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmDO);
    tma_prefetch_desc(&tmF);
    for (int i = 0; i < kPgStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 256);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      for (int kk = 0; kk < per_nb; ++kk) {
        const int s = kk % kPgStages;
        const uint32_t par = (kk / kPgStages) & 1;
        mbar_wait(&empty[s], par ^ 1);
        const int seg = kk / k_blocks, kb = kk - seg * k_blocks;   // 0: do_hi*f_hi, 1: do_lo*f_hi, 2: do_hi*f_lo
        const CUtensorMap* mA = seg == 1 ? &tmDO_lo : &tmDO;
        const CUtensorMap* mB = seg == 2 ? &tmF_lo : &tmF;
        uint8_t* a_dst = smem + s * kPgStageBytes;
        mbar_expect_tx(&full[s], kPgStageBytes);
        tma_load_3d(a_dst, mA, &full[s], kb * 64, q_row0, n);
        tma_load_3d(a_dst + kPgABytes, mB, &full[s], kb * 64, nb * kPgBlockN, n);
      }
    }
    return;
  }
  setmaxnreg_inc<232>();
  const int ct = threadIdx.x - 128;
  const int wg = ct >> 7, wq = (ct >> 5) & 3;
  const int cq = 2 * (lane & 3);
  const float* An = p.A + static_cast<size_t>(n) * Q * p.a_pitch;
  float* dAn = p.dA + static_cast<size_t>(n) * Q * p.a_pitch;
  // the thread's two target rows r = 64 wg + 16 wq + lane / 4 + 8 i; D[t] = <dout[t, :], out[t, :]> (the four lanes
  // that share a row take a quarter of the channels each) and the row's softmax statistics
  bool r_ok[2];
  int tpos[2];
  float D[2], rm[2], rinv[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
    r_ok[i] = r < live_rows;
    tpos[i] = q_row0 + (r_ok[i] ? r : 0);
    float d = 0.f;
    rm[i] = 0.f;
    rinv[i] = 0.f;
    if (kSoftmax && r_ok[i]) {
      const long long o1 = (static_cast<long long>(n) * Q + tpos[i]) * p.dout_pitch;
      const long long o2 = (static_cast<long long>(n) * Q + tpos[i]) * p.out_pitch;
      const int cpl = p.C / 4;
      for (int c = (lane & 3) * cpl; c < (lane & 3) * cpl + cpl; c += 8) {
        float a[8], b[8];
        if (p.dout_lo) {
          act_ld8<true>(p.dout, p.dout_lo, o1 + c, a);
          act_ld8<true>(p.out, p.out_lo, o2 + c, b);
        } else {
          act_ld8<false>(p.dout, nullptr, o1 + c, a);
          act_ld8<false>(p.out, nullptr, o2 + c, b);
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) d = fmaf(a[q], b[q], d);
      }
      const float2 st = p.stats[static_cast<size_t>(n) * Q + tpos[i]];
      rm[i] = st.x;
      rinv[i] = st.y;
    }
    if (kSoftmax) {
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
    }
    D[i] = d;
  }

  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  int prev_s = -1;
  for (int kk = 0; kk < per_nb; ++kk) {
    const int s = kk % kPgStages;
    const uint32_t par = (kk / kPgStages) & 1;
    mbar_wait(&full[s], par);
    const uint32_t a_addr = smem_u32(smem + s * kPgStageBytes);
    const uint64_t adesc = make_wgmma_desc_sw128(a_addr + wg * 64 * 128, 16, 1024);
    const uint64_t bdesc = make_wgmma_desc_sw128(a_addr + kPgABytes, 16, 1024);
    wgmma_fence_operand(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_bf16<kPgBlockN, 0, 0>(acc, adesc + static_cast<uint64_t>(k * 2), bdesc + static_cast<uint64_t>(k * 2),
                                  (kk > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_operand(acc);
    if (prev_s >= 0) mbar_arrive(&empty[prev_s]);
    prev_s = s;
  }
  wgmma_wait<0>();
  wgmma_fence_operand(acc);

#pragma unroll
  for (int i = 0; i < 2; ++i) {
    if (!r_ok[i]) continue;
    const int tp = tpos[i], ti = tp / p.W, tj = tp - ti * p.W;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int s = nb * kPgBlockN + 8 * j + cq + e;
        if (s >= Q) continue;
        const int si = s / p.W, sj = s - si * p.W;
        // owner / other of the attention entry
        const int oi = kCollect ? ti : si, oj = kCollect ? tj : sj, own = kCollect ? tp : s;
        const int a = (kCollect ? si : ti) - oi + hh, b = (kCollect ? sj : tj) - oj + hw;
        if (kDense || (a >= 0 && a < p.mH && b >= 0 && b < p.mW)) {
          const size_t off = kDense ? static_cast<size_t>(own) * p.a_pitch + (kCollect ? s : tp)
                                    : static_cast<size_t>(own) * p.a_pitch + a * p.mW + b;
          if (kSoftmax) {
            const float pv = __expf(__ldg(An + off) - rm[i]) * rinv[i];
            dAn[off] = pv * (p.scale * acc[4 * j + 2 * i + e] - D[i]);
          } else {
            dAn[off] = p.scale * acc[4 * j + 2 * i + e];
          }
        }
      }
    }
  }
}

template <bool kCollect, bool kDense, bool kSoftmax>
static int launch_attn_grad(const CUtensorMap& a, const CUtensorMap& al, const CUtensorMap& b, const CUtensorMap& bl,
                            const PsaGradParams& p, int grid, cudaStream_t stream) {
  static std::atomic<bool> attr_set[64];
  const auto kernel = psa_attn_grad_kernel<kCollect, kDense, kSoftmax>;
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPgSmem));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  const dim3 g(grid, cdiv(p.H * p.W, kPgBlockN));
  kernel<<<g, kPgThreads, kPgSmem, stream>>>(a, al, b, bl, p);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <bool kDense, bool kSoftmax>
static int launch_attn_grad_form(int psa_type, const CUtensorMap& a, const CUtensorMap& al, const CUtensorMap& b,
                                 const CUtensorMap& bl, const PsaGradParams& p, int grid, cudaStream_t stream) {
  return psa_type == 0 ? launch_attn_grad<true, kDense, kSoftmax>(a, al, b, bl, p, grid, stream)
                       : launch_attn_grad<false, kDense, kSoftmax>(a, al, b, bl, p, grid, stream);
}

}  // namespace sb

extern "C" int semseg_psa_attend_bwd_attn(int psa_type, const float* attn, int a_pitch, const float* stats,
                                          const void* feat, const void* feat_lo, int feat_pitch, const void* out,
                                          const void* out_lo, int out_pitch, const void* dout, const void* dout_lo,
                                          int dout_pitch, float* dattn, int N, int H, int W, int mH, int mW, int C,
                                          float scale, void* stream_) {
  return semseg_psa_attend_bwd_attn_ex(psa_type, 0, attn, a_pitch, stats, feat, feat_lo, feat_pitch, out, out_lo,
                                       out_pitch, dout, dout_lo, dout_pitch, dattn, N, H, W, mH, mW, C, scale, stream_);
}

extern "C" int semseg_psa_attend_bwd_attn_ex(int psa_type, int form, const float* attn, int a_pitch, const float* stats,
                                             const void* feat, const void* feat_lo, int feat_pitch, const void* out,
                                             const void* out_lo, int out_pitch, const void* dout, const void* dout_lo,
                                             int dout_pitch, float* dattn, int N, int H, int W, int mH, int mW, int C,
                                             float scale, void* stream_) {
  using namespace sb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const bool softmax = !(form & SEMSEG_PSA_NO_SOFTMAX);
  SB_CHECK_ARG(attn && feat && dout && dattn && N > 0 && H > 0 && W > 0, "psa_attend_bwd_attn: bad args");
  SB_CHECK_ARG(psa_type == 0 || psa_type == 1, "psa_attend_bwd_attn: psa_type must be 0 or 1");
  if (const int r = check_psa_form("psa_attend_bwd_attn", form, H, W, mH, mW, a_pitch, stats)) return r;
  SB_CHECK_ARG(out || !softmax, "psa_attend_bwd_attn: out is required with softmax");
  SB_CHECK_ARG(C > 0 && C % 64 == 0 && W <= 128, "psa_attend_bwd_attn: C %% 64 == 0 and W <= 128 required");
  SB_CHECK_ARG(feat_pitch % 8 == 0 && out_pitch % 8 == 0 && dout_pitch % 8 == 0, "psa_attend_bwd_attn: bad pitch");
  const bool split = feat_lo != nullptr;
  SB_CHECK_ARG(((out_lo != nullptr) == split || (!softmax && !out)) && (dout_lo != nullptr) == split,
               "psa_attend_bwd_attn: all activations must use the same storage form");
  // feat and dout through TMA, dout and out (read only with softmax) as 16-byte vectors in the D term: every check
  // comes before the dattn memset, so a rejected call makes no CUDA call
  if (const int r = check_vec_acts("psa_attend_bwd_attn", C, {{feat, feat_lo, feat_pitch}, {dout, dout_lo, dout_pitch},
                                                              {softmax ? out : nullptr, out_lo, out_pitch}}))
    return r;
  PsaGradParams p;
  memset(&p, 0, sizeof(p));
  p.A = attn; p.stats = reinterpret_cast<const float2*>(stats); p.dA = dattn;
  p.dout = static_cast<const __nv_bfloat16*>(dout); p.dout_lo = static_cast<const __nv_bfloat16*>(dout_lo);
  p.out = static_cast<const __nv_bfloat16*>(out); p.out_lo = static_cast<const __nv_bfloat16*>(out_lo);
  p.dout_pitch = dout_pitch; p.out_pitch = out_pitch;
  p.N = N; p.H = H; p.W = W; p.mH = mH; p.mW = mW; p.a_pitch = a_pitch; p.C = C;
  p.tile_rows = psa_tile_rows(N, H * W, 128, cdiv(H * W, kPgBlockN));   // keep every SM busy
  p.tiles_per_img = cdiv(H * W, p.tile_rows);
  p.nseg = split ? 3 : 1;
  p.scale = scale;
  // the caller's dattn must be zero where no gradient lands: outside the mask windows, and in the dense form the padding
  // columns of a pitch wider than H*W
  if (!(form & SEMSEG_PSA_DENSE) || a_pitch != H * W)
    SB_CUDA(cudaMemsetAsync(dattn, 0, sizeof(float) * static_cast<size_t>(N) * H * W * a_pitch, stream));
  CUtensorMap tmDO, tmDO_lo, tmF, tmF_lo;
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)H * W, (uint64_t)N};
    uint64_t str[2] = {(uint64_t)dout_pitch * 2, (uint64_t)dout_pitch * 2 * H * W};
    uint32_t box[3] = {64u, 128u, 1u};
    int r = encode_tmap_bf16(&tmDO, dout, 3, dims, str, box);
    if (r) return r;
    tmDO_lo = tmDO;
    if (split && (r = encode_tmap_bf16(&tmDO_lo, dout_lo, 3, dims, str, box))) return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)C, (uint64_t)H * W, (uint64_t)N};
    uint64_t str[2] = {(uint64_t)feat_pitch * 2, (uint64_t)feat_pitch * 2 * H * W};
    uint32_t box[3] = {64u, (uint32_t)kPgBlockN, 1u};
    int r = encode_tmap_bf16(&tmF, feat, 3, dims, str, box);
    if (r) return r;
    tmF_lo = tmF;
    if (split && (r = encode_tmap_bf16(&tmF_lo, feat_lo, 3, dims, str, box))) return r;
  }
  const int grid = N * p.tiles_per_img;
  switch (form) {
    case 0: return launch_attn_grad_form<false, true>(psa_type, tmDO, tmDO_lo, tmF, tmF_lo, p, grid, stream);
    case SEMSEG_PSA_DENSE: return launch_attn_grad_form<true, true>(psa_type, tmDO, tmDO_lo, tmF, tmF_lo, p, grid, stream);
    case SEMSEG_PSA_NO_SOFTMAX:
      return launch_attn_grad_form<false, false>(psa_type, tmDO, tmDO_lo, tmF, tmF_lo, p, grid, stream);
    default: return launch_attn_grad_form<true, false>(psa_type, tmDO, tmDO_lo, tmF, tmF_lo, p, grid, stream);
  }
}

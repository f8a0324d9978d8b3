// Weight-gradient implicit GEMM on sm_90a tensor cores (wgmma):
//
//   dw[t][co][ci] = sum_p dy[p, co] * x[p + off(t), ci]
//
// GEMM view: M = Cout (128-channel tile), N = Cin (BLOCK_N-channel tile), K = pixels. Both operands are
// "MN-major" for the tensor core: a TMA box [64 ch, bw, bh, 1] lands as (pixels x 128 bytes) rows in
// 128B-swizzled smem, which is exactly the canonical MN-major SWIZZLE_128B layout
// ((8,n),(8,k)):((1,LBO),(8,SBO)) with LBO = bytes per 64-channel box and SBO = 1024 (8 pixels).
// Replaces cuDNN's wgrad behind autograd for every nn.Conv2d on the path (model/resnet.py:63-69).
//
// Work unit = (split, tap, co-tile, ci-tile); a split owns a contiguous range of pixel boxes.
// K block = one pixel box of <= 64 pixels; the smem rows a box does not cover are zeroed once at kernel
// start and never written again, so they contribute exact zeros.
// Warpgroup 0 is the TMA producer; warpgroup 1 + w (w = 0, 1) owns output channels [64w, 64w + 64) of the co tile:
// wgmma M = 64 x N = BLOCK_N into fp32 registers, then fp32 partials straight from the registers to global memory.
#include "host_common.h"
#include "ptx.cuh"

namespace sb {

constexpr int kWgThreads = 384;
constexpr int kWgConsumerThreads = 256;
constexpr int kWgBoxPixels = 64;
constexpr int kWgBoxBytes = kWgBoxPixels * 128;  // one 64-channel x 64-pixel box
constexpr int kWgABoxes = 2;                      // 128 Cout channels

// N tile (Cin channels per work unit): 256 for wide layers, 128 / 64 for the narrow ones (stem, layer1/2).
template <int BN>
struct WgCfg {
  static constexpr int kBBoxes = BN / 64;
  static constexpr int kStageBytes = (kWgABoxes + kBBoxes) * kWgBoxBytes;  // 48 / 32 / 24 KB
  static constexpr int kStages = BN == 256 ? 4 : (BN == 128 ? 6 : 8);
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 1024;
};

struct WgradKParams {
  int N, H, W, Cin, Cout, taps;
  int bh, bw, tiles_h, tiles_w, num_boxes;
  int co_tiles, ci_tiles, n_splits, boxes_per_split, block_n;
  // Multi-tap units for narrow inputs (Cin <= 128, 3x3): the 256-wide N tile holds `tu` taps x (cin_boxes*64) channels,
  // so the dy tile is loaded once for `tu` taps instead of once per tap (the narrow layers are L2->SM bound).
  int tu, cin_boxes, unit_taps, oob_img;
  int dh[SEMSEG_MAX_TAPS], dw[SEMSEG_MAX_TAPS], img_add[SEMSEG_MAX_TAPS];
  int img_mul;
  int nseg;    // 1 = bf16 operands; 3 = bf16x3 (dy_hi*x_hi, dy_lo*x_hi, dy_hi*x_lo accumulated in registers)
  float* out;  // [n_splits][taps][Cout][Cin]
};

template <int kWgBlockN>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX,
                  const __grid_constant__ CUtensorMap tmDY_lo, const __grid_constant__ CUtensorMap tmX_lo,
                  const WgradKParams p) {
  constexpr int kWgBBoxes = WgCfg<kWgBlockN>::kBBoxes;
  constexpr int kWgStageBytes = WgCfg<kWgBlockN>::kStageBytes;
  constexpr int kWgStages = WgCfg<kWgBlockN>::kStages;
  constexpr int kAcc = kWgBlockN / 2;
  static_assert(kWgStages <= 16, "barrier area sized for <= 16 stages");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* misc = smem + kWgStages * kWgStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(misc);
  uint64_t* empty_bar = full_bar + 16;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int units_per_split = p.unit_taps * p.co_tiles * p.ci_tiles;
  const int num_units = units_per_split * p.n_splits;
  const uint32_t box_bytes = static_cast<uint32_t>(p.bh * p.bw) * 128u;
  const uint32_t stage_tx = box_bytes * (kWgABoxes + kWgBBoxes);   // bytes credited to a full barrier per stage

  // Zero all operand stages once: rows beyond the pixel box stay zero for the whole kernel.
  {
    uint4 z = make_uint4(0, 0, 0, 0);
    uint4* s4 = reinterpret_cast<uint4*>(smem);
    for (int i = threadIdx.x; i < kWgStages * kWgStageBytes / 16; i += kWgThreads) s4[i] = z;
  }
  fence_proxy_async_smem();

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX);
    if (p.nseg > 1) {
      tma_prefetch_desc(&tmDY_lo);
      tma_prefetch_desc(&tmX_lo);
    }
    for (int i = 0; i < kWgStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kWgConsumerThreads);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // unit -> (split, tap, co_tile, ci_tile); ci fastest so concurrent CTAs share the dy boxes in L2
  auto decode = [&](int unit, int& split, int& tap, int& co_t, int& ci_t) {
    ci_t = unit % p.ci_tiles;
    int r = unit / p.ci_tiles;
    co_t = r % p.co_tiles;
    r /= p.co_tiles;
    tap = r % p.unit_taps;   // tap, or tap group when p.tu > 1
    split = r / p.unit_taps;
  };

  if (warp < 4) {
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int it = 0;
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        int split, tap, co_t, ci_t;
        decode(unit, split, tap, co_t, ci_t);
        const int b0 = split * p.boxes_per_split;
        const int b1 = min(b0 + p.boxes_per_split, p.num_boxes);
        const int tiles_per_img = p.tiles_h * p.tiles_w;
        for (int bs = b0 * p.nseg; bs < b1 * p.nseg; ++bs, ++it) {
          const int b = bs / p.nseg;
          const int seg = bs - b * p.nseg;   // split storage: every pixel box is issued as three operand segments
          const CUtensorMap* mDY = seg == 1 ? &tmDY_lo : &tmDY;
          const CUtensorMap* mX = seg == 2 ? &tmX_lo : &tmX;
          const int s = it % kWgStages;
          const uint32_t par = (it / kWgStages) & 1;
          mbar_wait(&empty_bar[s], par ^ 1);
          const int img = b / tiles_per_img;
          const int rem = b - img * tiles_per_img;
          const int h0 = (rem / p.tiles_w) * p.bh;
          const int w0 = (rem % p.tiles_w) * p.bw;
          uint8_t* st = smem + s * kWgStageBytes;
          mbar_expect_tx(&full_bar[s], stage_tx);
#pragma unroll
          for (int i = 0; i < kWgABoxes; ++i)
            tma_load_4d(st + i * kWgBoxBytes, mDY, &full_bar[s], co_t * 128 + i * 64, w0, h0, img);
          if (p.tu > 1) {
#pragma unroll
            for (int i = 0; i < kWgBBoxes; ++i) {   // box i = (tap of the group, 64-channel block)
              const int ti = tap * p.tu + i / p.cin_boxes;
              const bool live = ti < p.taps;        // dead taps of the last group: fully out-of-range box -> zeros
              const int tt = live ? ti : 0;
              tma_load_4d(st + (kWgABoxes + i) * kWgBoxBytes, mX, &full_bar[s], (i % p.cin_boxes) * 64,
                          w0 + p.dw[tt], h0 + p.dh[tt], live ? img * p.img_mul + p.img_add[tt] : p.oob_img);
            }
          } else {
#pragma unroll
            for (int i = 0; i < kWgBBoxes; ++i)
              tma_load_4d(st + (kWgABoxes + i) * kWgBoxBytes, mX, &full_bar[s], ci_t * kWgBlockN + i * 64,
                          w0 + p.dw[tap], h0 + p.dh[tap], img * p.img_mul + p.img_add[tap]);
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int ct = threadIdx.x - 128;
    const int wg = ct >> 7;                 // dy box (64 output channels) of this warpgroup
    const int wq = (ct >> 5) & 3;
    const int cq = 2 * (lane & 3);
    float acc[kAcc];
    int it = 0;
    for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
      int split, tap, co_t, ci_t;
      decode(unit, split, tap, co_t, ci_t);
      const int b0 = split * p.boxes_per_split;
      const int b1 = min(b0 + p.boxes_per_split, p.num_boxes);
#pragma unroll
      for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
      int prev_s = -1;
      for (int b = b0 * p.nseg; b < b1 * p.nseg; ++b, ++it) {
        const int s = it % kWgStages;
        const uint32_t par = (it / kWgStages) & 1;
        mbar_wait(&full_bar[s], par);
        const uint32_t st = smem_u32(smem + s * kWgStageBytes);
        // MN-major SW128: LBO = next 64-channel box, SBO = next 8 pixels (1024 B)
        const uint64_t adesc = make_wgmma_desc_sw128(st + wg * kWgBoxBytes, kWgBoxBytes, 1024);
        const uint64_t bdesc = make_wgmma_desc_sw128(st + kWgABoxes * kWgBoxBytes, kWgBoxBytes, 1024);
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kWgBoxPixels / 16; ++k)   // 16 pixels along K = 2048 bytes -> +128 in 16-byte units
          wgmma_bf16<kWgBlockN, 1, 1>(acc, adesc + static_cast<uint64_t>(k * 128),
                                      bdesc + static_cast<uint64_t>(k * 128), (b > b0 * p.nseg || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_operand(acc);
        if (prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      if (prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);

      const int ci0 = ci_t * kWgBlockN;
      const bool pairs = (p.Cin & 1) == 0;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int co = co_t * 128 + wg * 64 + wq * 16 + (lane >> 2) + 8 * i;
        if (co >= p.Cout) continue;
#pragma unroll
        for (int j = 0; j < kWgBlockN / 8; ++j) {
          const int col = 8 * j + cq;          // column of the N tile (even)
          int tap_o = tap, ci = ci0 + col;
          if (p.tu > 1) {                      // destination of the column: (tap of the group, input channel)
            const int box = col >> 6;
            tap_o = tap * p.tu + box / p.cin_boxes;
            ci = (box % p.cin_boxes) * 64 + (col & 63);
            if (tap_o >= p.taps) continue;
          }
          if (ci >= p.Cin) continue;
          float* o = p.out + ((static_cast<size_t>(split) * p.taps + tap_o) * p.Cout + co) * p.Cin + ci;
          const float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
          if (pairs && ci + 1 < p.Cin) {
            *reinterpret_cast<float2*>(o) = make_float2(v0, v1);
          } else {
            o[0] = v0;
            if (ci + 1 < p.Cin) o[1] = v1;
          }
        }
      }
    }
  }
}

// part[s][t][co][ci] -> dw[co][ci][t], splits added in order s = 0, 1, ... (fixed order => deterministic).
// block = (32 plane lanes, taps, G groups): every lane owns W consecutive plane elements (W = 4: one 16-byte load per
// split, four splits in flight), so even the single-split layers (cls head: a 75 MB transposing copy) keep enough bytes
// in flight; the [tap][lane] tile is turned through shared memory so the OIHW writes are contiguous too.
constexpr int kRedMaxTaps = 9;
template <int W>
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int n_splits, int taps, size_t plane,
                                    float* __restrict__ dw, int accumulate) {
  extern __shared__ __align__(16) float red_tile[];  // [G][taps][32 * W + 4]
  constexpr int kRow = 32 * W + 4;
  const int lane = threadIdx.x, t = threadIdx.y, grp = threadIdx.z;
  float* tile = red_tile + grp * taps * kRow;
  const size_t idx0 = (static_cast<size_t>(blockIdx.x) * blockDim.z + grp) * (32 * W);
  const size_t idx = idx0 + static_cast<size_t>(lane) * W;
  float s[W];
#pragma unroll
  for (int q = 0; q < W; ++q) s[q] = 0.f;
  if (idx < plane) {  // plane % W == 0: the whole vector is inside
    const size_t stride = static_cast<size_t>(taps) * plane;
    const float* p = part + static_cast<size_t>(t) * plane + idx;
    auto ld = [&](const float* q, float (&v)[W]) {
      if constexpr (W == 4) {
        const float4 f = *reinterpret_cast<const float4*>(q);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
      } else {
        v[0] = *q;
      }
    };
    int sp = 0;
    for (; sp + 4 <= n_splits; sp += 4) {
      float a[W], b[W], c[W], d[W];
      ld(p, a);
      ld(p + stride, b);
      ld(p + 2 * stride, c);
      ld(p + 3 * stride, d);
#pragma unroll
      for (int q = 0; q < W; ++q) {
        s[q] += a[q];
        s[q] += b[q];
        s[q] += c[q];
        s[q] += d[q];
      }
      p += 4 * stride;
    }
    for (; sp < n_splits; ++sp) {
      float a[W];
      ld(p, a);
#pragma unroll
      for (int q = 0; q < W; ++q) s[q] += a[q];
      p += stride;
    }
  }
#pragma unroll
  for (int q = 0; q < W; ++q) tile[t * kRow + lane * W + q] = s[q];
  __syncthreads();
  // this group's 32*W*taps outputs are contiguous in dw; thread (t, lane) writes W of them, 32*taps apart
  const int per = 32 * taps;
#pragma unroll
  for (int k = 0; k < W; ++k) {
    const int j = k * per + t * 32 + lane;
    const int l = j / taps, tt = j - l * taps;
    if (idx0 + l < plane) {
      float* d = dw + idx0 * taps + j;
      const float v = tile[tt * kRow + l];
      *d = accumulate ? (*d + v) : v;
    }
  }
}

template <int BN>
static int launch_wgrad(const CUtensorMap& tmDY, const CUtensorMap& tmX, const CUtensorMap& tmDY_lo,
                        const CUtensorMap& tmX_lo, const WgradKParams& kp, int grid, cudaStream_t stream) {
  // per-device opt-in to > 48 KB dynamic shared memory (see conv_igemm.cu)
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(conv_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 WgCfg<BN>::kSmemBytes));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  conv_wgrad_kernel<BN><<<grid, kWgThreads, WgCfg<BN>::kSmemBytes, stream>>>(tmDY, tmX, tmDY_lo, tmX_lo, kp);
  return SEMSEG_OK;
}

static void wgrad_geometry(const semseg_wgrad_desc* d, WgradKParams* kp) {
  kp->N = d->N; kp->H = d->H; kp->W = d->W; kp->Cin = d->Cin; kp->Cout = d->Cout; kp->taps = d->taps;
  choose_box(d->H, d->W, kWgBoxPixels, &kp->bh, &kp->bw);
  kp->tiles_h = cdiv(d->H, kp->bh);
  kp->tiles_w = cdiv(d->W, kp->bw);
  kp->num_boxes = d->N * kp->tiles_h * kp->tiles_w;
  kp->co_tiles = cdiv(d->Cout, 128);
  kp->block_n = d->Cin > 128 ? 256 : (d->Cin > 64 ? 128 : 64);
  kp->ci_tiles = cdiv(d->Cin, kp->block_n);
  kp->tu = 1;
  kp->cin_boxes = cdiv(d->Cin, 64);
  kp->unit_taps = d->taps;
  kp->oob_img = d->Nin;
  if (d->taps > 1 && d->Cin <= 128) {   // narrow 3x3: several taps share one dy tile (N tile = 256)
    kp->tu = 4 / kp->cin_boxes;
    kp->unit_taps = cdiv(d->taps, kp->tu);
    kp->block_n = 256;
    kp->ci_tiles = 1;
  }
  const int units = kp->unit_taps * kp->co_tiles * kp->ci_tiles;
  int splits = d->n_splits;
  if (splits <= 0) {
    // Split-K factor: the work units (units x splits) run on `slots` CTAs in whole rounds, so the last round should be
    // (nearly) full, while every unit keeps enough K blocks to amortise its pipeline fill / drain (~8 blocks).
    const int slots = num_sms();
    const int max_by_k = kp->num_boxes / 16 > 0 ? kp->num_boxes / 16 : 1;
    const int max_s = max_by_k < 64 ? max_by_k : 64;
    double best = -1.0;
    splits = 1;
    for (int sp = 1; sp <= max_s; ++sp) {
      const double waves = static_cast<double>(units) * sp / slots;
      const double rounds = ceil(waves);
      const double kb = static_cast<double>(kp->num_boxes) / sp;
      const double score = (waves / rounds) * (kb / (kb + 8.0)) * (waves >= 1.0 ? 1.0 : waves);
      if (score > best + 1e-9) {
        best = score;
        splits = sp;
      }
    }
    if (d->x_lo != nullptr) {
      // bf16x3: bound one accumulation chain to 21 pixel boxes (21 x 4 MMA steps x 3 segments = 252 steps): the tensor
      // core's fp32 accumulation truncates (~2^-24 per step towards zero); the fixed-order fp32 reduction of the split
      // partials rounds to nearest.
      const int need = cdiv(kp->num_boxes, 21);
      if (splits < need) splits = need;
    }
  }
  kp->boxes_per_split = cdiv(kp->num_boxes, splits);
  kp->n_splits = cdiv(kp->num_boxes, kp->boxes_per_split);  // no empty splits
}

}  // namespace sb

extern "C" int semseg_conv_wgrad_splits(const semseg_wgrad_desc* d) {
  if (!d || d->N <= 0 || d->H <= 0 || d->W <= 0 || d->Cin <= 0 || d->Cout <= 0) return SEMSEG_E_INVALID;
  sb::WgradKParams kp;
  sb::wgrad_geometry(d, &kp);
  return kp.n_splits;
}

extern "C" int semseg_conv_wgrad(const semseg_wgrad_desc* d, void* stream_) {
  using namespace sb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(d != nullptr, "wgrad: null descriptor");
  SB_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0 && d->Cin > 0 && d->Cout > 0, "wgrad: bad sizes");
  SB_CHECK_ARG(d->taps >= 1 && d->taps <= SEMSEG_MAX_TAPS, "wgrad: taps out of range");
  SB_CHECK_ARG(d->x && d->dy && d->dw_partial, "wgrad: null pointer");
  SB_CHECK_ARG(d->x_pitch % 8 == 0 && d->dy_pitch % 8 == 0, "wgrad: pitches must be multiples of 8");
  WgradKParams kp;
  memset(&kp, 0, sizeof(kp));
  wgrad_geometry(d, &kp);
  if (d->n_splits > 0)
    SB_CHECK_ARG(kp.n_splits == d->n_splits, "wgrad: n_splits %d not realisable (library would use %d)",
                 d->n_splits, kp.n_splits);
  for (int t = 0; t < d->taps; ++t) {
    kp.dh[t] = d->dh[t]; kp.dw[t] = d->dw[t]; kp.img_add[t] = d->img_add[t];
  }
  kp.img_mul = d->img_mul;
  kp.out = d->dw_partial;
  const bool split = d->x_lo != nullptr;
  SB_CHECK_ARG((d->dy_lo != nullptr) == split, "wgrad: x and dy must use the same storage form (plain or split)");
  kp.nseg = split ? 3 : 1;

  CUtensorMap tmDY, tmX, tmDY_lo, tmX_lo;
  {
    uint64_t dims[4] = {(uint64_t)d->Cout, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->N};
    uint64_t str[3] = {(uint64_t)d->dy_pitch * 2, (uint64_t)d->dy_pitch * 2 * d->W,
                       (uint64_t)d->dy_pitch * 2 * d->W * d->H};
    uint32_t box[4] = {64u, (uint32_t)kp.bw, (uint32_t)kp.bh, 1};
    int r = encode_tmap_bf16(&tmDY, d->dy, 4, dims, str, box);
    if (r) return r;
    tmDY_lo = tmDY;
    if (split && (r = encode_tmap_bf16(&tmDY_lo, d->dy_lo, 4, dims, str, box))) return r;
  }
  {
    uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)d->Win, (uint64_t)d->Hin, (uint64_t)d->Nin};
    uint64_t str[3] = {(uint64_t)d->x_pitch * 2, (uint64_t)d->x_pitch * 2 * d->Win,
                       (uint64_t)d->x_pitch * 2 * d->Win * d->Hin};
    uint32_t box[4] = {64u, (uint32_t)kp.bw, (uint32_t)kp.bh, 1};
    int r = encode_tmap_bf16(&tmX, d->x, 4, dims, str, box);
    if (r) return r;
    tmX_lo = tmX;
    if (split && (r = encode_tmap_bf16(&tmX_lo, d->x_lo, 4, dims, str, box))) return r;
  }
  const int units = kp.unit_taps * kp.co_tiles * kp.ci_tiles * kp.n_splits;
  int rc = SEMSEG_OK;
  const int grid = units < num_sms() ? units : num_sms();
  switch (kp.block_n) {
    case 256: rc = launch_wgrad<256>(tmDY, tmX, tmDY_lo, tmX_lo, kp, grid, stream); break;
    case 128: rc = launch_wgrad<128>(tmDY, tmX, tmDY_lo, tmX_lo, kp, grid, stream); break;
    default: rc = launch_wgrad<64>(tmDY, tmX, tmDY_lo, tmX_lo, kp, grid, stream); break;
  }
  if (rc) return rc;
  SB_LAUNCHED();
  return SEMSEG_OK;
}

extern "C" int semseg_wgrad_reduce(const float* dw_partial, int n_splits, int taps, int Cout, int Cin,
                                   float* dw_oihw, int accumulate, void* stream_) {
  using namespace sb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(dw_partial && dw_oihw && n_splits > 0 && taps > 0 && Cout > 0 && Cin > 0, "wgrad_reduce: bad args");
  SB_CHECK_ARG(taps <= kRedMaxTaps, "wgrad_reduce: at most 9 taps");
  const size_t plane = static_cast<size_t>(Cout) * Cin;
  const int groups = taps >= 8 ? 1 : 8 / taps;
  const dim3 block(32, taps, groups);
  if (plane % 4 == 0) {
    const size_t per_block = static_cast<size_t>(128) * groups;
    const unsigned blocks = static_cast<unsigned>((plane + per_block - 1) / per_block);
    const size_t smem = static_cast<size_t>(groups) * taps * (128 + 4) * sizeof(float);
    wgrad_reduce_kernel<4><<<blocks, block, smem, stream>>>(dw_partial, n_splits, taps, plane, dw_oihw, accumulate);
  } else {
    const size_t per_block = static_cast<size_t>(32) * groups;
    const unsigned blocks = static_cast<unsigned>((plane + per_block - 1) / per_block);
    const size_t smem = static_cast<size_t>(groups) * taps * (32 + 4) * sizeof(float);
    wgrad_reduce_kernel<1><<<blocks, block, smem, stream>>>(dw_partial, n_splits, taps, plane, dw_oihw, accumulate);
  }
  SB_LAUNCHED();
  return SEMSEG_OK;
}

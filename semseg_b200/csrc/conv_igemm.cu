// Implicit-GEMM convolution (fprop and dgrad) for NHWC bf16 activations on sm_90a tensor cores (wgmma).
//
//   out[p, co] = sum_t sum_ci x[p + off(t), ci] * w[t][co][ci]
//
// GEMM view: M = pixels (tiles of a bh x bw pixel rectangle inside one image, <= 128 rows),
// N = Cout (BLOCK_N columns per tile), K = taps * Cin in blocks of 64 channels.
//
// Replaces the cuDNN convolutions behind nn.Conv2d in the reference (model/resnet.py:63-69,
// model/pspnet.py:49-58,65-69,73-77). One persistent CTA per SM, warp-specialised:
//   warpgroup 0   : TMA producer (one elected thread) — A tile = 4-D box [64 ch, bw, bh, 1] at the tap-shifted pixel
//                   (TMA zero-fills the halo), B tile = 3-D box [64, BLOCK_N, 1] of the packed weights; both land in
//                   128B-swizzled shared memory.
//   warpgroups 1-2: MMA + epilogue — warpgroup w issues wgmma (M=64, N=BLOCK_N, K=16) on pixel rows [64w, 64w+64) of
//                   the tile into fp32 register accumulators, then runs the epilogue straight from the registers:
//                   (affine / ReLU / residual) -> bf16 -> swizzled smem -> TMA store; running BatchNorm statistics
//                   (sum, sum of squares, count per channel) of the stored bf16 values, one statistics row per
//                   32 pixel rows of the tile.
#include "host_common.h"
#include "ptx.cuh"

namespace sb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 bf16 = 128 bytes = one swizzle span
constexpr int kConvThreads = 384;   // producer warpgroup + two MMA / epilogue warpgroups
constexpr int kConsumerThreads = 256;
constexpr int kATileBytes = kBlockM * kBlockK * 2;  // 16 KB
constexpr int kStageOutBytes = kBlockM * 64 * 2;    // 16 KB epilogue staging chunk (64 columns)
constexpr int kMiscBytes = 2048;

template <int BLOCK_N>
struct ConvCfg {
  static constexpr int kBTileBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = kATileBytes + kBTileBytes;
  static constexpr int kStages = (BLOCK_N == 256) ? 4 : (BLOCK_N == 128 ? 6 : 8);
  static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kStageOutBytes + kMiscBytes + 1024;
};

struct ConvKParams {
  int N, H, W;
  int Cin, Cout;
  int taps;
  int bh, bw, tiles_h, tiles_w;
  int n_tiles, num_m_tiles;
  int k_chunks;  // ceil(Cin / 64)
  int dh[SEMSEG_MAX_TAPS], dw[SEMSEG_MAX_TAPS], wtap[SEMSEG_MAX_TAPS], img_add[SEMSEG_MAX_TAPS];
  int img_mul;
  int epi_mode, relu;
  const float* scale;
  const float* shift;
  const __nv_bfloat16* residual;
  const __nv_bfloat16* residual_lo;  // split storage: lo plane of the residual
  int res_pitch;
  int nseg;  // operand segments per K block: 1 = bf16, 3 = bf16x3 (x_hi*w_hi, x_lo*w_hi, x_hi*w_lo)
  // K slicing (F32 epilogue only): work item = (pixel tile, channel tile, K slice); slice s accumulates K blocks
  // [s*kb_per_slice, (s+1)*kb_per_slice) and writes its fp32 partial to out_f32 + s*slice_stride. Bounds the length of
  // one tensor-core accumulation chain: the tensor core accumulates in fp32 with truncation, a bias of ~2^-24 per MMA
  // step towards zero, negligible for bf16 but not at the 1e-5 level the bf16x3 mode works at.
  int k_slices, kb_per_slice;
  long long slice_stride;
  float* out_f32;
  int out_pitch;
  float* stats_partial;  // [gridDim.x * 4][3][Cout]: per 32 pixel rows of the tile (sum, sum of squares, count)
  // e4m3 operand mode (kFp8): which outputs the AFFINE epilogue writes, and the factor its e4m3 output is multiplied by
  // before the saturating round (1 / s_out, where s_out is the consumer's dequantisation scale)
  int out_bf16, out_e4m3;
  float y8_qscale;
};

// kFp8 (e4m3 operand mode, eval only): x and w are e4m3 bytes, a K block is 128 channels (still one 128-byte swizzle
// span, so the stage bytes, TMA boxes and barrier ring are those of bf16) and takes four m64nNk32 e4m3 wgmmas. With
// kPromote each stage accumulates into a fresh register tile that is then added into the fp32 master accumulator (the
// FP8 tensor-core accumulation loses precision over long K, measured in DESIGN §4), so BLOCK_N <= 128; without it the
// wgmmas accumulate straight into acc like bf16 (kept for that measurement). The AFFINE epilogue writes the bf16 output,
// an e4m3 copy of it scaled by y8_qscale (staged in the second buffer with a 64-byte swizzle, TMA store through the
// tmC_lo slot), or both.
//
// kSplit (bf16x3 operand mode, activations stored as hi/lo bf16 planes — act.cuh): every K block is issued three times,
// (x_hi, w_hi), (x_lo, w_hi), (x_hi, w_lo), into the same fp32 accumulator; the producer just picks the hi or lo
// tensor map per segment, the MMA loop is unchanged. The epilogue splits its fp32 result into (hi, lo) again and stores
// both planes (two staging tiles, two TMA stores); BatchNorm statistics are taken from hi + lo.
template <int BLOCK_N, bool kSplit, bool kFp8, bool kPromote>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmA_lo,
                  const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmC_lo,
                  const ConvKParams p) {
  using Cfg = ConvCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kStageBytes = Cfg::kStageBytes;
  constexpr int kAcc = BLOCK_N / 2;   // fp32 accumulator registers per thread
  constexpr int kKElems = kFp8 ? 2 * kBlockK : kBlockK;   // channels per K block (128 bytes either way)
  static_assert(!(kSplit && kFp8), "bf16x3 and e4m3 operand modes are exclusive");
  const int num_items = p.num_m_tiles * p.n_tiles * p.k_slices;
  auto decode_item = [&](int item, int& m_tile, int& n_tile, int& k_slice) {
    k_slice = item % p.k_slices;
    item /= p.k_slices;
    n_tile = item % p.n_tiles;
    m_tile = item / p.n_tiles;
  };

  auto tile_origin = [&](int m_tile, int& img, int& h0, int& w0) {   // image and first pixel of a pixel tile
    const int tiles_per_img = p.tiles_h * p.tiles_w;
    img = m_tile / tiles_per_img;
    const int rem = m_tile - img * tiles_per_img;
    h0 = (rem / p.tiles_w) * p.bh;
    w0 = (rem % p.tiles_w) * p.bw;
  };

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // aligned by an offset from smem_raw (not through an integer), so that the compiler still knows every pointer below
  // is in shared memory: the epilogue's staging stores and statistics loads become st.shared / ld.shared with 32-bit
  // addresses instead of generic accesses with 64-bit address arithmetic
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* stage_base = smem;
  uint8_t* out_stage = smem + kStages * kStageBytes;  // 2 x 16 KB
  uint8_t* misc = out_stage + 2 * kStageOutBytes;
  static_assert(kStages <= 16, "barrier area sized for <= 16 stages");
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(misc);
  uint64_t* empty_bar = full_bar + 16;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nseg = kSplit ? p.nseg : 1;
  const int total_kblk = p.taps * p.k_chunks;   // K blocks = (64-channel block, tap) pairs
  auto slice_range = [&](int k_slice, int& kblk0, int& kblk1) {
    kblk0 = k_slice * p.kb_per_slice;
    kblk1 = min(kblk0 + p.kb_per_slice, total_kblk);
  };
  const uint32_t stage_tx = static_cast<uint32_t>(p.bh * p.bw) * 128u + static_cast<uint32_t>(Cfg::kBTileBytes);

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
    if (kSplit) {
      tma_prefetch_desc(&tmA_lo);
      tma_prefetch_desc(&tmB_lo);
      tma_prefetch_desc(&tmC_lo);
    }
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kConsumerThreads);
    }
    fence_barrier_init();
  }
  if (p.stats_partial != nullptr) {  // four statistics rows per CTA: one per 32 pixel rows of the tile
    float* row = p.stats_partial + static_cast<size_t>(blockIdx.x) * 4 * 3 * p.Cout;
    for (int i = threadIdx.x; i < 4 * 3 * p.Cout; i += kConvThreads) row[i] = 0.f;
  }
  __syncthreads();

  if (warp < 4) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int it = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        int m_tile, n_tile, k_slice, kblk0, kblk1;
        decode_item(item, m_tile, n_tile, k_slice);
        slice_range(k_slice, kblk0, kblk1);
        const int tiles_per_img = p.tiles_h * p.tiles_w;
        const int img = m_tile / tiles_per_img;
        const int rem = m_tile - img * tiles_per_img;
        const int h0 = (rem / p.tiles_w) * p.bh;
        const int w0 = (rem % p.tiles_w) * p.bw;
        const int n0 = n_tile * BLOCK_N;
        for (int kb = kblk0 * nseg; kb < kblk1 * nseg; ++kb, ++it) {
          const int s = it % kStages;
          const uint32_t par = (it / kStages) & 1;
          mbar_wait(&empty_bar[s], par ^ 1);
          const int ks = kb / nseg;          // (channel block, tap)
          const int seg = kb - ks * nseg;    // 0: x_hi*w_hi, 1: x_lo*w_hi, 2: x_hi*w_lo
          const int cb = ks / p.taps;
          const int t = ks - cb * p.taps;
          const CUtensorMap* mA = (kSplit && seg == 1) ? &tmA_lo : &tmA;
          const CUtensorMap* mB = (kSplit && seg == 2) ? &tmB_lo : &tmB;
          uint8_t* a_dst = stage_base + s * kStageBytes;
          uint8_t* b_dst = a_dst + kATileBytes;
          mbar_expect_tx(&full_bar[s], stage_tx);
          tma_load_4d(a_dst, mA, &full_bar[s], cb * kKElems, w0 + p.dw[t], h0 + p.dh[t],
                      img * p.img_mul + p.img_add[t]);
          // 3-D weights [taps][rows][cols]: coordinates (k, row, tap)
          tma_load_3d(b_dst, mB, &full_bar[s], cb * kKElems, n0, p.wtap[t]);
        }
      }
    }
  } else {
    // ===================================================================== MMA + epilogue (warpgroups 1, 2)
    setmaxnreg_inc<232>();
    const int ct = threadIdx.x - 128;      // 0..255
    const int wg = ct >> 7;                // pixel rows [64*wg, 64*wg + 64) of the tile
    const int wq = (ct >> 5) & 3;          // warp inside the warpgroup
    const int r_base = wg * 64 + wq * 16 + (lane >> 2);   // accumulator rows r_base and r_base + 8
    const int cq = 2 * (lane & 3);         // first of the thread's column pair inside every 8 columns
    int it = 0;
    int store_buf = 0;
    float acc[kAcc];
    constexpr int kChunks = BLOCK_N / 64;
    const bool stats = !kFp8 && p.stats_partial != nullptr && p.epi_mode == SEMSEG_EPI_RAW;
    // running sum and sum of squares of this thread's statistics column in every chunk, and the running pixel count
    // of its 32 rows (the same for every chunk), added to the CTA's statistics row in global memory only when the
    // CTA's next item is in another channel tile (or there is none)
    float st_acc[kChunks][2], st_n = 0.f;
#pragma unroll
    for (int ch = 0; ch < kChunks; ++ch) st_acc[ch][0] = st_acc[ch][1] = 0.f;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      int m_tile, n_tile, k_slice, kblk0, kblk1;
      decode_item(item, m_tile, n_tile, k_slice);
      slice_range(k_slice, kblk0, kblk1);
      const int num_kb = (kblk1 - kblk0) * nseg;
      if (p.epi_mode == SEMSEG_EPI_AFFINE && p.residual != nullptr && (lane & 3) < kChunks) {
        // pull the tile's residual into L2 while the main loop runs (the epilogue reads it chunk by chunk): lane & 3
        // picks the 128-byte line (one 64-column chunk) of each of the thread's two pixel rows
        const int c = n_tile * BLOCK_N + 64 * (lane & 3);
        int img, h0, w0;
        tile_origin(m_tile, img, h0, w0);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = r_base + 8 * i, hi = r / p.bw, wi = r - hi * p.bw;
          if (c < p.Cout && r < p.bh * p.bw && h0 + hi < p.H && w0 + wi < p.W) {
            const long long ro = ((static_cast<long long>(img) * p.H + (h0 + hi)) * p.W + (w0 + wi)) * p.res_pitch + c;
            prefetch_l2(p.residual + ro);
            if (kSplit) prefetch_l2(p.residual_lo + ro);
          }
        }
      }
      // ---- main loop: one wgmma batch (K = 64) per stage; a stage is released once the next batch was issued and
      // the one reading it has completed
      int prev_s = -1;
#pragma unroll
      for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
      if constexpr (kFp8 && kPromote) {
        // promoted accumulation: each stage's four wgmmas start a fresh tile, which is added into acc in fp32 once they
        // completed; the other warpgroup's wgmmas keep the tensor core busy meanwhile
        float part[kAcc];
        for (int kb = 0; kb < num_kb; ++kb, ++it) {
          const int s = it % kStages;
          const uint32_t par = (it / kStages) & 1;
          mbar_wait(&full_bar[s], par);
          const uint32_t a_addr = smem_u32(stage_base + s * kStageBytes) + static_cast<uint32_t>(wg * 64 * 128);
          const uint32_t b_addr = smem_u32(stage_base + s * kStageBytes + kATileBytes);
          const uint64_t adesc = make_wgmma_desc_sw128(a_addr, 16, 1024);
          const uint64_t bdesc = make_wgmma_desc_sw128(b_addr, 16, 1024);
          wgmma_fence_operand(part);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)   // advance 32 bytes (32 e4m3) along K inside the 128-byte swizzle span
            wgmma_e4m3<BLOCK_N>(part, adesc + static_cast<uint64_t>(k * 2), bdesc + static_cast<uint64_t>(k * 2),
                                k > 0 ? 1u : 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_operand(part);
          mbar_arrive(&empty_bar[s]);
#pragma unroll
          for (int i = 0; i < kAcc; ++i) acc[i] += part[i];
        }
      } else {
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % kStages;
        const uint32_t par = (it / kStages) & 1;
        mbar_wait(&full_bar[s], par);
        const uint32_t a_addr = smem_u32(stage_base + s * kStageBytes) + static_cast<uint32_t>(wg * 64 * 128);
        const uint32_t b_addr = smem_u32(stage_base + s * kStageBytes + kATileBytes);
        const uint64_t adesc = make_wgmma_desc_sw128(a_addr, 16, 1024);
        const uint64_t bdesc = make_wgmma_desc_sw128(b_addr, 16, 1024);
        wgmma_fence_operand(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k)   // advance 32 bytes (16 bf16) along K inside the 128-byte swizzle span
          if constexpr (kFp8)   // (32 e4m3 per step)
            wgmma_e4m3<BLOCK_N>(acc, adesc + static_cast<uint64_t>(k * 2), bdesc + static_cast<uint64_t>(k * 2),
                                (kb > 0 || k > 0) ? 1u : 0u);
          else
            wgmma_bf16<BLOCK_N, 0, 0>(acc, adesc + static_cast<uint64_t>(k * 2), bdesc + static_cast<uint64_t>(k * 2),
                                      (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_operand(acc);
        if (prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
        prev_s = s;
      }
      wgmma_wait<0>();
      wgmma_fence_operand(acc);
      if (prev_s >= 0) mbar_arrive(&empty_bar[prev_s]);
      }

      // ---- epilogue
      int img, h0, w0;
      tile_origin(m_tile, img, h0, w0);
      const int n0 = n_tile * BLOCK_N;
      auto row_ok = [&](int r) {
        const int hi = r / p.bw, wi = r - (r / p.bw) * p.bw;
        return (r < p.bh * p.bw) && (h0 + hi < p.H) && (w0 + wi < p.W);
      };
      auto row_pix = [&](int r) {
        const int hi = r / p.bw, wi = r - hi * p.bw;
        return (static_cast<long long>(img) * p.H + (h0 + hi)) * p.W + (w0 + wi);
      };
      bool rv[2];
      long long pix[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        rv[i] = row_ok(r_base + 8 * i);
        pix[i] = row_pix(r_base + 8 * i);
      }
#pragma unroll
      for (int ch = 0; ch < kChunks; ++ch) {
        const int c0 = n0 + ch * 64;  // first output channel of this chunk
        if (c0 >= p.Cout) break;      // (uniform) nothing to write for padded columns
        float* a = acc + ch * 32;     // this chunk's 32 registers: a[4j + 2i + e] = (row r_base + 8i, col 8j + cq + e)

        if (p.epi_mode == SEMSEG_EPI_F32) {
          const bool bias = p.shift != nullptr && k_slice == 0;
          // float2 stores need 8-byte alignment: an even pitch and slice stride, and an output that starts on an even
          // float (out_f32 may be a channel slice of a wider buffer at any offset)
          const bool pairs = ((p.out_pitch | p.slice_stride) & 1) == 0 &&
                             (reinterpret_cast<uintptr_t>(p.out_f32) & 7) == 0;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            if (!rv[i]) continue;
            float* orow = p.out_f32 + k_slice * p.slice_stride + pix[i] * p.out_pitch;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int c = c0 + 8 * j + cq;
              float v0 = a[4 * j + 2 * i], v1 = a[4 * j + 2 * i + 1];
              if (pairs && c + 1 < p.Cout) {
                if (bias) {
                  v0 += __ldg(p.shift + c);
                  v1 += __ldg(p.shift + c + 1);
                }
                *reinterpret_cast<float2*>(orow + c) = make_float2(v0, v1);
              } else {
                if (c < p.Cout) orow[c] = bias ? v0 + __ldg(p.shift + c) : v0;
                if (c + 1 < p.Cout) orow[c + 1] = bias ? v1 + __ldg(p.shift + c + 1) : v1;
              }
            }
          }
          continue;
        }

        if (p.epi_mode == SEMSEG_EPI_AFFINE) {
          const bool has_res = p.residual != nullptr;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = c0 + 8 * j + cq;
            const float sc0 = p.scale ? __ldg(p.scale + c) : 1.f, sc1 = p.scale ? __ldg(p.scale + c + 1) : 1.f;
            const float sh0 = p.shift ? __ldg(p.shift + c) : 0.f, sh1 = p.shift ? __ldg(p.shift + c + 1) : 0.f;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              float r0 = 0.f, r1 = 0.f;
              if (has_res && rv[i]) {
                const long long ro = pix[i] * p.res_pitch + c;
                float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.residual + ro));
                if constexpr (kSplit) {
                  const float2 fl = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.residual_lo + ro));
                  f.x += fl.x;
                  f.y += fl.y;
                }
                r0 = f.x;
                r1 = f.y;
              }
              float v0 = fmaf(a[4 * j + 2 * i], sc0, sh0) + r0;
              float v1 = fmaf(a[4 * j + 2 * i + 1], sc1, sh1) + r1;
              if (p.relu) {
                v0 = fmaxf(v0, 0.f);
                v1 = fmaxf(v1, 0.f);
              }
              a[4 * j + 2 * i] = v0;
              a[4 * j + 2 * i + 1] = v1;
            }
          }
        }

        // registers -> bf16 -> 128B-swizzled staging tile (row = pixel, 64 channels = 128 bytes); the two staging
        // buffers are used alternately (split storage: buffer 0 = hi plane tile, buffer 1 = lo plane tile)
        // (kFp8: buffer 0 = bf16 tile, buffer 1 = e4m3 tile [row][64 bytes] with the 64-byte swizzle: 16-byte chunk
        // c of row r at chunk c ^ ((r >> 1) & 3), so the 8 rows of a warp's stores hit 8 distinct bank groups)
        uint8_t* obuf = out_stage + ((kSplit || kFp8) ? 0 : store_buf) * kStageOutBytes;
        if (ct == 0) tma_store_wait_read<((kSplit || kFp8) ? 0 : 1)>();  // the store(s) that last read the buffer(s) drained
        named_bar_sync(1, kConsumerThreads);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int r = r_base + 8 * i;
            const float v0 = a[4 * j + 2 * i], v1 = a[4 * j + 2 * i + 1];
            if constexpr (kFp8) {
              if (p.out_bf16)
                *reinterpret_cast<uint32_t*>(obuf + r * 128 + ((j ^ (r & 7)) << 4) + cq * 2) = pack_bf16x2(v0, v1);
              if (p.out_e4m3)
                *reinterpret_cast<uint16_t*>(obuf + kStageOutBytes + r * 64 + ((((j >> 1) ^ (r >> 1)) & 3) << 4) +
                                             8 * (j & 1) + cq) =
                    pack_e4m3x2(v0 * p.y8_qscale, v1 * p.y8_qscale);
              continue;
            }
            const uint32_t h = pack_bf16x2(v0, v1);
            const int off = r * 128 + ((j ^ (r & 7)) << 4) + cq * 2;
            *reinterpret_cast<uint32_t*>(obuf + off) = h;
            if constexpr (kSplit) {   // lo = value - float(hi), staged in the second buffer
              const float2 hf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&h));
              *reinterpret_cast<uint32_t*>(obuf + kStageOutBytes + off) = pack_bf16x2(v0 - hf.x, v1 - hf.y);
            }
          }
        }
        fence_proxy_async_smem();
        named_bar_sync(1, kConsumerThreads);
        if (ct == 0) {
          if constexpr (kFp8) {
            if (p.out_bf16) tma_store_4d(&tmC, obuf, c0, w0, h0, img);
            if (p.out_e4m3) tma_store_4d(&tmC_lo, obuf + kStageOutBytes, c0, w0, h0, img);
          } else {
            tma_store_4d(&tmC, obuf, c0, w0, h0, img);
            if (kSplit) tma_store_4d(&tmC_lo, obuf + kStageOutBytes, c0, w0, h0, img);
          }
          tma_store_commit();
        }
        if (stats) {
          // Per-column statistics of the bf16 values just staged (exactly what BN-apply will read back). Warp g of
          // warpgroup w reduces pixel rows [32g, 32g + 32) of the chunk's columns [32w, 32w + 32), lane = column (two
          // lanes per 4-byte word: conflict-free), one pass of sum and sum of squares in row order, added to the
          // thread's registers: no cross-warp traffic, fixed order -> deterministic. A row outside the image adds
          // +0.f: neither sum is ever -0.f, so that leaves its bits as skipping the row would, and the 32 loads need
          // no branches and can all be in flight together.
          const int g = wq;
          const uint32_t row_msk = __ballot_sync(0xffffffffu, row_ok(g * 32 + lane));
          float sm = 0.f, sq = 0.f;
          const int col = 32 * wg + lane;
          const uint8_t* base = obuf + g * 32 * 128 + (col & 7) * 2;
          const int chunk16 = col >> 3;
#pragma unroll
          for (int r = 0; r < 32; ++r) {   // (32g + r) & 7 = r & 7: the row's swizzle phase
            const uint8_t* src = base + r * 128 + ((chunk16 ^ (r & 7)) << 4);
            float f = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(src));
            if constexpr (kSplit) f += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(src + kStageOutBytes));
            f = ((row_msk >> r) & 1u) ? f : 0.f;
            sm += f;
            sq = fmaf(f, f, sq);
          }
          st_acc[ch][0] += sm;
          st_acc[ch][1] += sq;
          if (ch == 0) st_n += static_cast<float>(__popc(row_msk));   // integer-valued: exact
        }
        store_buf ^= 1;
      }
      // Flush: one read-modify-write of the CTA's statistics row g when the next item is in another channel tile. A
      // CTA's items step by gridDim.x, so its consecutive items either always share the channel tile (then the
      // registers hold the sum over all its tiles, added to the zeroed row once) or never do (then they hold one
      // tile's sum): either way the fp32 additions are those of a per-tile update of the row, in the same order.
      const int next = item + gridDim.x;
      if (stats && (next >= num_items || (next / p.k_slices) % p.n_tiles != n_tile)) {
        float* st_dst = p.stats_partial + (static_cast<size_t>(blockIdx.x) * 4 + wq) * 3 * p.Cout + n0 + 32 * wg + lane;
        float old[kChunks][3];
#pragma unroll
        for (int ch = 0; ch < kChunks; ++ch)   // all loads first: one global round trip per flush
          if (n0 + ch * 64 < p.Cout)
#pragma unroll
            for (int v = 0; v < 3; ++v) old[ch][v] = st_dst[ch * 64 + v * p.Cout];
#pragma unroll
        for (int ch = 0; ch < kChunks; ++ch) {
          if (n0 + ch * 64 < p.Cout) {
            st_dst[ch * 64] = old[ch][0] + st_acc[ch][0];
            st_dst[ch * 64 + p.Cout] = old[ch][1] + st_acc[ch][1];
            st_dst[ch * 64 + 2 * p.Cout] = old[ch][2] + st_n;
          }
          st_acc[ch][0] = st_acc[ch][1] = 0.f;
        }
        st_n = 0.f;
      }
    }
    if (ct == 0) tma_store_wait_all<0>();
  }
}

// Grid (= 1/4 of the rows of the statistics buffer): one persistent CTA per SM at most.
static int conv_grid(int num_m_tiles, int n_tiles) {
  const int sms = num_sms();
  const long long tiles = static_cast<long long>(num_m_tiles) * n_tiles;
  return static_cast<int>(tiles < sms ? tiles : sms);
}

struct ConvMaps {
  CUtensorMap a, b, c, a_lo, b_lo, c_lo;
};

template <int BLOCK_N>
static int launch_conv(const ConvMaps& tm, const ConvKParams& kp, bool split, int grid, cudaStream_t stream) {
  using Cfg = ConvCfg<BLOCK_N>;
  // the opt-in to > 48 KB of dynamic shared memory is per device: set it once for every device this process uses
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(conv_igemm_kernel<BLOCK_N, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 Cfg::kSmemBytes));
    SB_CUDA(cudaFuncSetAttribute(conv_igemm_kernel<BLOCK_N, true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 Cfg::kSmemBytes));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  if (split)
    conv_igemm_kernel<BLOCK_N, true, false, false><<<grid, kConvThreads, Cfg::kSmemBytes, stream>>>(
        tm.a, tm.b, tm.c, tm.a_lo, tm.b_lo, tm.c_lo, kp);
  else
    conv_igemm_kernel<BLOCK_N, false, false, false><<<grid, kConvThreads, Cfg::kSmemBytes, stream>>>(
        tm.a, tm.b, tm.c, tm.a_lo, tm.b_lo, tm.c_lo, kp);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

template <int BLOCK_N, bool kPromote>
static int launch_conv_e4m3(const ConvMaps& tm, const ConvKParams& kp, int grid, cudaStream_t stream) {
  using Cfg = ConvCfg<BLOCK_N>;
  static std::atomic<bool> attr_set[64];
  int dev = 0;
  SB_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
    SB_CUDA(cudaFuncSetAttribute(conv_igemm_kernel<BLOCK_N, false, true, kPromote>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 Cfg::kSmemBytes));
    if (dev >= 0 && dev < 64) attr_set[dev].store(true, std::memory_order_release);
  }
  conv_igemm_kernel<BLOCK_N, false, true, kPromote><<<grid, kConvThreads, Cfg::kSmemBytes, stream>>>(tm.a, tm.b, tm.c, tm.a_lo,
                                                                                          tm.b_lo, tm.c_lo, kp);
  SB_LAUNCHED();
  return SEMSEG_OK;
}

}  // namespace sb

static int conv_block_n(int Cout) {
  if (Cout % 256 == 0 || Cout > 128) return 256;
  return Cout > 64 ? 128 : 64;
}

// Rows of the RAW-epilogue statistics buffer = number of CTAs the kernel will launch for this problem.
// K blocks (64-channel block x tap) of a conv, and the slice count that keeps one accumulation chain <= max_kblocks.
extern "C" int semseg_conv_k_slices(int Cin, int taps, int max_kblocks) {
  if (Cin <= 0 || taps <= 0 || max_kblocks <= 0) return SEMSEG_E_INVALID;
  const int total = taps * sb::cdiv(Cin, sb::kBlockK);
  const int per = sb::cdiv(total, sb::cdiv(total, max_kblocks));
  return sb::cdiv(total, per);
}

extern "C" int semseg_conv_stats_rows(int N, int H, int W, int Cout) {
  if (N <= 0 || H <= 0 || W <= 0 || Cout <= 0) return SEMSEG_E_INVALID;
  int bh, bw;
  sb::choose_box(H, W, sb::kBlockM, &bh, &bw);
  // four statistics rows per CTA (one per 32 pixel rows of the tile)
  return 4 * sb::conv_grid(N * sb::cdiv(H, bh) * sb::cdiv(W, bw), sb::cdiv(Cout, conv_block_n(Cout)));
}

// The e4m3 operand mode (eval convs of semseg_b200/fp8.py): x and w are e4m3 bytes, the AFFINE epilogue writes y (bf16),
// y8 (e4m3, v * y8_qscale rounded and saturated) or both. Everything the mode does not support is rejected here.
static int conv_fprop_e4m3(const semseg_conv_desc* d, cudaStream_t stream) {
  using namespace sb;
  SB_CHECK_ARG(d->e4m3 == 1 || d->e4m3 == 2, "conv: e4m3 must be 0, 1 (promoted) or 2 (unpromoted), got %d", d->e4m3);
  SB_CHECK_ARG(d->Cin % 128 == 0, "conv: e4m3 operands need Cin %% 128 == 0 (got %d)", d->Cin);
  SB_CHECK_ARG(d->Cout % 64 == 0, "conv: e4m3 operands need Cout %% 64 == 0 (got %d)", d->Cout);
  SB_CHECK_ARG(d->epi_mode == SEMSEG_EPI_AFFINE, "conv: e4m3 operands need the AFFINE epilogue");
  SB_CHECK_ARG(d->x_lo == nullptr && d->y_lo == nullptr && d->residual_lo == nullptr && d->w_split == 0,
               "conv: e4m3 operands cannot be split (bf16x3)");
  SB_CHECK_ARG(d->k_slices <= 1, "conv: e4m3 operands cannot be K-sliced");
  SB_CHECK_ARG(d->stats_partial == nullptr, "conv: e4m3 operands take no statistics");
  SB_CHECK_ARG(d->y != nullptr || d->y8 != nullptr, "conv: e4m3 conv without an output (y, y8)");
  SB_CHECK_ARG(d->x_pitch % 16 == 0 && d->x_pitch >= d->Cin,
               "conv: e4m3 x_pitch %d must be a multiple of 16 bytes and >= Cin", d->x_pitch);
  SB_CHECK_ARG(d->w_cols % 16 == 0 && d->w_cols >= d->Cin,
               "conv: e4m3 w_cols %d must be a multiple of 16 bytes and >= Cin", d->w_cols);
  SB_CHECK_ARG(d->y == nullptr || (d->y_pitch % 8 == 0 && d->y_pitch >= d->Cout), "conv: bad y_pitch %d", d->y_pitch);
  SB_CHECK_ARG(d->y8 == nullptr || (d->y8_pitch % 16 == 0 && d->y8_pitch >= d->Cout),
               "conv: y8_pitch %d must be a multiple of 16 bytes and >= Cout", d->y8_pitch);
  SB_CHECK_ARG(d->y8 == nullptr || (d->y8_qscale > 0.f && d->y8_qscale < 3.0e38f),
               "conv: y8_qscale must be finite and > 0");
  SB_CHECK_ARG(d->residual == nullptr || (d->res_pitch % 8 == 0 && (reinterpret_cast<uintptr_t>(d->residual) & 3) == 0),
               "conv: res_pitch must be a multiple of 8 and the residual 4-byte aligned");
  for (int t = 0; t < d->taps; ++t)
    SB_CHECK_ARG(d->wtap[t] >= 0 && d->wtap[t] < d->n_wtaps, "conv: wtap[%d]=%d out of range", t, d->wtap[t]);

  ConvKParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.N = d->N; kp.H = d->H; kp.W = d->W; kp.Cin = d->Cin; kp.Cout = d->Cout; kp.taps = d->taps;
  choose_box(d->H, d->W, kBlockM, &kp.bh, &kp.bw);
  kp.tiles_h = cdiv(d->H, kp.bh);
  kp.tiles_w = cdiv(d->W, kp.bw);
  kp.num_m_tiles = d->N * kp.tiles_h * kp.tiles_w;
  kp.k_chunks = d->Cin / 128;
  for (int t = 0; t < d->taps; ++t) {
    kp.dh[t] = d->dh[t]; kp.dw[t] = d->dw[t]; kp.wtap[t] = d->wtap[t]; kp.img_add[t] = d->img_add[t];
  }
  kp.img_mul = d->img_mul;
  kp.epi_mode = SEMSEG_EPI_AFFINE; kp.relu = d->relu;
  kp.scale = d->scale; kp.shift = d->shift;
  kp.residual = static_cast<const __nv_bfloat16*>(d->residual); kp.res_pitch = d->res_pitch;
  kp.nseg = 1;
  kp.out_bf16 = d->y != nullptr;
  kp.out_e4m3 = d->y8 != nullptr;
  kp.y8_qscale = d->y8_qscale;
  const int block_n = d->Cout % 128 == 0 ? 128 : 64;   // <= 128: the promoted accumulation holds two register tiles
  kp.n_tiles = d->Cout / block_n;
  kp.k_slices = 1;
  kp.kb_per_slice = kp.taps * kp.k_chunks;
  const int grid = conv_grid(kp.num_m_tiles, kp.n_tiles);

  ConvMaps tm;
  {
    uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)d->Win, (uint64_t)d->Hin, (uint64_t)d->Nin};
    uint64_t str[3] = {(uint64_t)d->x_pitch, (uint64_t)d->x_pitch * d->Win, (uint64_t)d->x_pitch * d->Win * d->Hin};
    uint32_t box[4] = {128u, (uint32_t)kp.bw, (uint32_t)kp.bh, 1};
    int r = encode_tmap_u8(&tm.a, d->x, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (r) return r;
    tm.a_lo = tm.a;
  }
  {
    uint64_t dims[3] = {(uint64_t)d->w_cols, (uint64_t)d->w_rows, (uint64_t)d->n_wtaps};
    uint64_t str[2] = {(uint64_t)d->w_cols, (uint64_t)d->w_cols * d->w_rows};
    uint32_t box[3] = {128u, (uint32_t)block_n, 1};
    int r = encode_tmap_u8(&tm.b, d->w, 3, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B);
    if (r) return r;
    tm.b_lo = tm.b;
  }
  {
    uint32_t box[4] = {64u, (uint32_t)kp.bw, (uint32_t)kp.bh, 1};
    int r;
    if (d->y) {
      uint64_t dims[4] = {(uint64_t)d->Cout, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->N};
      uint64_t str[3] = {(uint64_t)d->y_pitch * 2, (uint64_t)d->y_pitch * 2 * d->W, (uint64_t)d->y_pitch * 2 * d->W * d->H};
      if ((r = encode_tmap_bf16(&tm.c, d->y, 4, dims, str, box))) return r;
    }
    if (d->y8) {   // the e4m3 staging tile: [row][64 bytes], 64-byte swizzle
      uint64_t dims[4] = {(uint64_t)d->Cout, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->N};
      uint64_t str[3] = {(uint64_t)d->y8_pitch, (uint64_t)d->y8_pitch * d->W, (uint64_t)d->y8_pitch * d->W * d->H};
      if ((r = encode_tmap_u8(&tm.c_lo, d->y8, 4, dims, str, box, CU_TENSOR_MAP_SWIZZLE_64B))) return r;
    }
    if (!d->y) tm.c = tm.c_lo;
    if (!d->y8) tm.c_lo = tm.c;
  }
  if (d->e4m3 == 2)   // unpromoted accumulation: the measurement form of DESIGN §4
    return block_n == 128 ? launch_conv_e4m3<128, false>(tm, kp, grid, stream)
                          : launch_conv_e4m3<64, false>(tm, kp, grid, stream);
  return block_n == 128 ? launch_conv_e4m3<128, true>(tm, kp, grid, stream)
                        : launch_conv_e4m3<64, true>(tm, kp, grid, stream);
}

extern "C" int semseg_conv_fprop(const semseg_conv_desc* d, void* stream_) {
  using namespace sb;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  SB_CHECK_ARG(d != nullptr, "conv: null descriptor");
  SB_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0 && d->Cin > 0 && d->Cout > 0, "conv: bad sizes");
  SB_CHECK_ARG(d->taps >= 1 && d->taps <= SEMSEG_MAX_TAPS, "conv: taps=%d out of range", d->taps);
  SB_CHECK_ARG(d->x && d->w, "conv: null x/w");
  SB_CHECK_ARG(d->x_pitch % 8 == 0 && d->x_pitch >= d->Cin, "conv: x_pitch %d must be a multiple of 8 and >= Cin",
               d->x_pitch);
  SB_CHECK_ARG(d->w_cols % 8 == 0 && d->w_cols >= d->Cin, "conv: w_cols %d must be a multiple of 8 and >= Cin",
               d->w_cols);
  SB_CHECK_ARG(d->epi_mode >= 0 && d->epi_mode <= 2, "conv: bad epi_mode");
  if (d->e4m3) return conv_fprop_e4m3(d, stream);
  SB_CHECK_ARG(d->y8 == nullptr, "conv: y8 (e4m3 output) needs e4m3 operands");

  ConvKParams kp;
  memset(&kp, 0, sizeof(kp));
  kp.N = d->N; kp.H = d->H; kp.W = d->W; kp.Cin = d->Cin; kp.Cout = d->Cout; kp.taps = d->taps;
  choose_box(d->H, d->W, kBlockM, &kp.bh, &kp.bw);
  kp.tiles_h = cdiv(d->H, kp.bh);
  kp.tiles_w = cdiv(d->W, kp.bw);
  kp.num_m_tiles = d->N * kp.tiles_h * kp.tiles_w;
  kp.k_chunks = cdiv(d->Cin, kBlockK);
  for (int t = 0; t < d->taps; ++t) {
    kp.dh[t] = d->dh[t]; kp.dw[t] = d->dw[t]; kp.wtap[t] = d->wtap[t]; kp.img_add[t] = d->img_add[t];
    SB_CHECK_ARG(d->wtap[t] >= 0 && d->wtap[t] < d->n_wtaps, "conv: wtap[%d]=%d out of range", t, d->wtap[t]);
  }
  kp.img_mul = d->img_mul;
  kp.epi_mode = d->epi_mode; kp.relu = d->relu;
  kp.scale = d->scale; kp.shift = d->shift;
  kp.residual = static_cast<const __nv_bfloat16*>(d->residual); kp.res_pitch = d->res_pitch;
  kp.residual_lo = static_cast<const __nv_bfloat16*>(d->residual_lo);
  const bool split = d->x_lo != nullptr;   // bf16x3 operand mode: hi/lo planes for x, w, y, residual
  kp.nseg = split ? 3 : 1;
  if (split) {
    SB_CHECK_ARG(d->w_split != 0, "conv: split activations need split weights (w_split)");
    SB_CHECK_ARG(d->epi_mode == SEMSEG_EPI_F32 || d->y_lo != nullptr, "conv: split input needs a split output (y_lo)");
    SB_CHECK_ARG(!d->residual || d->residual_lo, "conv: split input needs a split residual (residual_lo)");
  } else {
    SB_CHECK_ARG(!d->y_lo && !d->residual_lo, "conv: lo planes given without x_lo");
  }
  kp.out_f32 = d->out_f32; kp.out_pitch = d->out_pitch;
  kp.stats_partial = d->stats_partial;

  const int block_n = conv_block_n(d->Cout);
  kp.n_tiles = cdiv(d->Cout, block_n);
  kp.k_slices = 1;
  kp.kb_per_slice = kp.taps * kp.k_chunks;
  kp.slice_stride = 0;
  if (d->k_slices > 1) {
    SB_CHECK_ARG(d->epi_mode == SEMSEG_EPI_F32, "conv: K slicing needs the F32 epilogue (partials are fp32)");
    SB_CHECK_ARG(d->slice_stride >= static_cast<long long>(d->N) * d->H * d->W * d->out_pitch,
                 "conv: slice_stride too small for an [N,H,W,out_pitch] partial");
    kp.kb_per_slice = cdiv(kp.taps * kp.k_chunks, d->k_slices);
    kp.k_slices = cdiv(kp.taps * kp.k_chunks, kp.kb_per_slice);   // no empty slices
    SB_CHECK_ARG(kp.k_slices == d->k_slices, "conv: k_slices %d not realisable for %d K blocks (use %d)", d->k_slices,
                 kp.taps * kp.k_chunks, kp.k_slices);
    kp.slice_stride = d->slice_stride;
  }
  const int grid = conv_grid(kp.num_m_tiles, kp.n_tiles * kp.k_slices);

  // A: input activations [Nin][Hin][Win][x_pitch] viewed as (C, W, H, N)
  ConvMaps tm;
  {
    uint64_t dims[4] = {(uint64_t)d->Cin, (uint64_t)d->Win, (uint64_t)d->Hin, (uint64_t)d->Nin};
    uint64_t str[3] = {(uint64_t)d->x_pitch * 2, (uint64_t)d->x_pitch * 2 * d->Win,
                       (uint64_t)d->x_pitch * 2 * d->Win * d->Hin};
    uint32_t box[4] = {(uint32_t)kBlockK, (uint32_t)kp.bw, (uint32_t)kp.bh, 1};
    int r = encode_tmap_bf16(&tm.a, d->x, 4, dims, str, box);
    if (r) return r;
    tm.a_lo = tm.a;
    if (split && (r = encode_tmap_bf16(&tm.a_lo, d->x_lo, 4, dims, str, box))) return r;
  }
  {
    uint64_t dims[3] = {(uint64_t)d->w_cols, (uint64_t)d->w_rows, (uint64_t)d->n_wtaps};
    uint64_t str[2] = {(uint64_t)d->w_cols * 2, (uint64_t)d->w_cols * 2 * d->w_rows};
    uint32_t box[3] = {(uint32_t)kBlockK, (uint32_t)block_n, 1};
    int r = encode_tmap_bf16(&tm.b, d->w, 3, dims, str, box);
    if (r) return r;
    tm.b_lo = tm.b;
    if (split) {   // the lo slab follows the hi slab (semseg_pack_item.split != 0)
      const __nv_bfloat16* w_lo =
          static_cast<const __nv_bfloat16*>(d->w) + static_cast<size_t>(d->n_wtaps) * d->w_rows * d->w_cols;
      if ((r = encode_tmap_bf16(&tm.b_lo, w_lo, 3, dims, str, box))) return r;
    }
  }
  if (d->epi_mode == SEMSEG_EPI_F32) {
    SB_CHECK_ARG(d->out_f32 != nullptr && d->out_pitch >= d->Cout, "conv: F32 epilogue needs out_f32/out_pitch");
    tm.c = tm.a;  // unused
    tm.c_lo = tm.a;
  } else {
    SB_CHECK_ARG(d->y != nullptr, "conv: null y");
    SB_CHECK_ARG(d->Cout % 64 == 0, "conv: bf16 epilogue needs Cout %% 64 == 0 (got %d)", d->Cout);
    SB_CHECK_ARG(d->y_pitch % 8 == 0 && d->y_pitch >= d->Cout, "conv: bad y_pitch %d", d->y_pitch);
    if (d->residual)   // the epilogue reads the residual as bf16 pairs
      SB_CHECK_ARG(d->res_pitch % 8 == 0 && (reinterpret_cast<uintptr_t>(d->residual) & 3) == 0 &&
                       (reinterpret_cast<uintptr_t>(d->residual_lo) & 3) == 0,
                   "conv: res_pitch must be a multiple of 8 and the residual 4-byte aligned");
    uint64_t dims[4] = {(uint64_t)d->Cout, (uint64_t)d->W, (uint64_t)d->H, (uint64_t)d->N};
    uint64_t str[3] = {(uint64_t)d->y_pitch * 2, (uint64_t)d->y_pitch * 2 * d->W,
                       (uint64_t)d->y_pitch * 2 * d->W * d->H};
    uint32_t box[4] = {64u, (uint32_t)kp.bw, (uint32_t)kp.bh, 1};
    int r = encode_tmap_bf16(&tm.c, d->y, 4, dims, str, box);
    if (r) return r;
    tm.c_lo = tm.c;
    if (split && (r = encode_tmap_bf16(&tm.c_lo, d->y_lo, 4, dims, str, box))) return r;
  }
  switch (block_n) {
    case 256: return launch_conv<256>(tm, kp, split, grid, stream);
    case 128: return launch_conv<128>(tm, kp, split, grid, stream);
    default: return launch_conv<64>(tm, kp, split, grid, stream);
  }
}

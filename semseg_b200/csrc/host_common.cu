#include "host_common.h"

#include <cudaTypedefs.h>
#include <stdarg.h>
#include <string.h>

#include <mutex>

namespace sb {

static thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 148;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    cached[dev] = n;
  }
  return cached[dev];
}

int check_vec_acts(const char* fn, int C, std::initializer_list<VecAct> acts, int align) {
  for (const VecAct& a : acts) {
    if (!a.hi) continue;
    SB_CHECK_ARG(((reinterpret_cast<uintptr_t>(a.hi) | reinterpret_cast<uintptr_t>(a.lo)) & (align - 1)) == 0,
                 "%s: activation base %p (lo %p) is not %d-byte aligned", fn, a.hi, a.lo, align);
    SB_CHECK_ARG(a.pitch >= C, "%s: pitch %d is smaller than C = %d", fn, a.pitch, C);
  }
  return SEMSEG_OK;
}

static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box) {
  auto fn = get_encode();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
    return SEMSEG_E_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("tensor base %p not 16-byte aligned", base);
    return SEMSEG_E_INVALID;
  }
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (box[i] == 0 || box[i] > 256) {
      set_error("TMA box dim %d = %u out of range", i, box[i]);
      return SEMSEG_E_INVALID;
    }
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gs[i] = strides_bytes[i];
    if (gs[i] % 16 != 0) {
      set_error("TMA stride %d = %llu not a multiple of 16 bytes", i, (unsigned long long)gs[i]);
      return SEMSEG_E_INVALID;
    }
  }
  auto encode = [&] {
    return fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), gd, gs, bx, es,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  };
  CUresult r = encode();
  if (r == CUDA_ERROR_INVALID_CONTEXT) {
    // a thread that has made no runtime call yet has no current context (autograd's device thread, when the first
    // backward node it runs encodes a tensor map before launching anything): bind the device's primary context, retry
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) r = encode();
  }
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu,%llu box %u,%u,%u)", (int)r,
              rank, (unsigned long long)gd[0], (unsigned long long)gd[1], (unsigned long long)(rank > 2 ? gd[2] : 0),
              bx[0], bx[1], rank > 2 ? bx[2] : 0);
    return SEMSEG_E_CUDA;
  }
  return SEMSEG_OK;
}

void choose_box(int H, int W, int max_pixels, int* bh_out, int* bw_out) {
  double best = -1.0;
  int best_bh = 1, best_bw = 1;
  int wcap = W < max_pixels ? W : max_pixels;
  for (int bw = 1; bw <= wcap; ++bw) {
    int bh = max_pixels / bw;
    if (bh > H) bh = H;
    if (bh > 256) bh = 256;
    if (bh < 1) continue;
    // shrink bh to the smallest value giving the same number of row tiles (less OOB work)
    int th = cdiv(H, bh);
    bh = cdiv(H, th);
    int tw = cdiv(W, bw);
    double util = (double)H * W / ((double)th * tw * max_pixels);
    // prefer higher utilisation, then wider boxes (longer contiguous runs)
    if (util > best + 1e-9 || (util > best - 1e-9 && bw > best_bw)) {
      best = util;
      best_bh = bh;
      best_bw = bw;
    }
  }
  *bh_out = best_bh;
  *bw_out = best_bw;
}

}  // namespace sb

extern "C" const char* semseg_last_error(void) { return sb::g_err; }
extern "C" int semseg_abi_version(void) { return 3; }
extern "C" long long semseg_launch_count(void) { return sb::g_launches.load(); }

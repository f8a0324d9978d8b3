// Host-side helpers shared by the C-ABI translation units: error reporting, launch counting,
// TMA tensor-map encoding through the driver entry point (no link-time dependency on libcuda).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <initializer_list>

#include "../../include/semseg_b200.h"

namespace sb {

void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;
int num_sms();

#define SB_CHECK_ARG(cond, ...)  \
  do {                           \
    if (!(cond)) {               \
      sb::set_error(__VA_ARGS__); \
      return SEMSEG_E_INVALID;   \
    }                            \
  } while (0)

#define SB_CUDA(call)                                                                     \
  do {                                                                                    \
    cudaError_t e__ = (call);                                                             \
    if (e__ != cudaSuccess) {                                                             \
      sb::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return SEMSEG_E_CUDA;                                                               \
    }                                                                                     \
  } while (0)

// Call after every kernel launch: counts it and surfaces launch-configuration errors.
#define SB_LAUNCHED()                                                                        \
  do {                                                                                       \
    sb::g_launches.fetch_add(1, std::memory_order_relaxed);                                  \
    cudaError_t e__ = cudaGetLastError();                                                    \
    if (e__ != cudaSuccess) {                                                                \
      sb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return SEMSEG_E_CUDA;                                                                  \
    }                                                                                        \
  } while (0)

// bf16 tensor map, `rank` dims (innermost first), SWIZZLE_128B, zero OOB fill.
// dims/box in elements, strides_bytes[i] = byte stride of dim i+1 (rank-1 entries).
int encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                     const uint64_t* strides_bytes, const uint32_t* box);

// Pixel box (bh x bw <= max_pixels) maximising tile utilisation of an H x W map.
void choose_box(int H, int W, int max_pixels, int* bh, int* bw);

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// An activation operand of a kernel that accesses it in vector pieces (act_ld8 / act_st8, uint4, uint2): hi and lo
// bases, pitch in elements.
struct VecAct {
  const void* hi;
  const void* lo;
  int pitch;
};

// Rejects before launch an operand such a kernel would access out of line: a hi or lo base that is not `align`-byte
// aligned (16 for 8-channel bf16 vectors: a channel slice starting at a channel that is not a multiple of 8), or a pitch
// below C (rows that overlap). Operands the kernel does not touch are passed with hi == nullptr and skipped.
int check_vec_acts(const char* fn, int C, std::initializer_list<VecAct> acts, int align = 16);

}  // namespace sb

// Host-side helpers shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>

#include "../../include/hero_b200.h"

namespace hero {

// Thread-local error text returned by hero_last_error().
char* error_buffer();
int set_error(int status, const char* fmt, ...);
int sm_count();
// True while hero_gemm_profile_begin/end brackets GEMM launches with timing events (the layer
// runtime then keeps everything on one stream so per-launch durations do not overlap).
bool gemm_profile_active();
// While set (on this host thread), GEMM launches hand out their work items dynamically: the layer
// runtime's backward, whose dgrad chain and weight-gradient stream share the SMs. A grid that has
// the SMs to itself keeps the static stride, which measured faster there. Returns the previous
// setting.
bool gemm_set_shared_sms(bool on);
// HERO_SERIAL_PROFILE=1 (development): no programmatic dependent launch and a single stream, so a
// timeline profiler sees every kernel's own duration (tools/step_profile.py).
bool serial_profiling();

#define HERO_CUDA_CHECK(expr)                                                              \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      return ::hero::set_error(HERO_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,              \
                               cudaGetErrorString(_e), __FILE__, __LINE__);                \
  } while (0)

#define HERO_REQUIRE(cond, ...)                                           \
  do {                                                                    \
    if (!(cond)) return ::hero::set_error(HERO_ERR_INVALID, __VA_ARGS__); \
  } while (0)

#define HERO_LAUNCH_CHECK()                                                                  \
  do {                                                                                       \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess)                                                                   \
      return ::hero::set_error(HERO_ERR_CUDA, "kernel launch failed: %s (%s:%d)",            \
                               cudaGetErrorString(_e), __FILE__, __LINE__);                  \
  } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Launch with programmatic dependent launch enabled (see ptx.cuh pdl_wait): the kernel MUST call
// pdl_wait() before its first access to global memory written by earlier work in the stream.
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                     cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = serial_profiling() ? 0 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// 2-D bf16 tensor map over a row-major [outer, inner] matrix (leading dim `ld` elements) with a
// 128-byte-swizzled box of box_inner (<= 64) x box_outer elements. `map` is a CUtensorMap.
int encode_tmap_2d_bf16(void* map, const void* ptr, long long inner, long long outer, long long ld,
                        int box_inner, int box_outer);

}  // namespace hero

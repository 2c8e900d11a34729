// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma, fences.
// No CUTLASS dependency.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace hero {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 %%rx;\n"
      ".reg .pred %%px;\n"
      "elect.sync %%rx|%%px, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, %%px;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (reported as a CUDA error) after ~4 s of wall clock instead
// of hanging the GPU. try_wait itself suspends for a HW-defined slice, so count time, not spins.
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// The trap sits in a function of its own: inlined, ptxas holds every register live at it to the
// kernel's launch-time register count, which spills the accumulators of a warpgroup that raised
// its count with setmaxnreg.
static __device__ __noinline__ void mbar_wait_timed_out() { __trap(); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) == 0 && global_timer_ns() - t0 > 4000000000ull) mbar_wait_timed_out();
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------- wgmma (sm_90a)
// Shared-memory matrix descriptor for wgmma, 128-byte swizzle:
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type (1 = SWIZZLE_128B)
// K-major operands: 8-row groups SBO = 1024 B apart, LBO unused (encoded 1).
// MN-major operands: 64-element MN atoms LBO bytes apart, 8-k groups SBO = 1024 B apart.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                    uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Warpgroup-collective: every thread of the 128-thread warpgroup executes these.
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs.
template <int R>
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 inputs, fp32 accumulators in registers.
// TA / TB: 0 = K-major, 1 = MN-major operand. Accumulator fragment of thread t of the warpgroup
// (warp w = t / 32, lane l): d[4j + 2h + e] = D[16w + l / 4 + 8h][8j + 2(l % 4) + e].
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t adesc, uint64_t bdesc,
                                                uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %10, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, %11, %12;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc,
                                                uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc,
                                                uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t adesc, uint64_t bdesc,
                                                 uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, %131, %132;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

// ---------------------------------------------------------------- warpgroup registers, named barriers
// setmaxnreg: every thread of the warpgroup executes the same instruction. .dec returns registers
// to the SM's pool; .inc blocks until the pool can grant them. N is a multiple of 8 in [24, 256].
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
// Named barrier `id` (1..15; 0 is __syncthreads) over `count` threads (a multiple of 32): sync
// waits for the barrier to complete, arrive counts towards it without waiting.
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int count) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ---------------------------------------------------------------- programmatic dependent launch
// Kernels launched with the programmatic-stream-serialization attribute may start while the
// previous kernel in the stream is still draining: everything before pdl_wait() (barrier init,
// descriptor prefetch) overlaps that tail; pdl_wait() blocks until the previous
// grid has completed and its writes are visible. pdl_launch_dependents() lets the NEXT kernel
// begin its own prologue early.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// ---------------------------------------------------------------- misc
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

// Counter-based per-element hash used for dropout masks: fwd and bwd regenerate the same
// mask from (key, element index); nothing is stored.
__device__ __forceinline__ uint32_t hash_u32(uint32_t key, uint32_t idx) {
  uint32_t h = idx * 0x9E3779B1u ^ key;
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}
// One 32-bit hash decides TWO consecutive elements (16 bits each): keep iff bits16 >= p * 2^16.
// `threshold` is passed as p * 2^32 (C-ABI) and narrowed here; p = 0.1 -> 6553 / 65536.
__device__ __forceinline__ bool dropout_keep(uint32_t key, uint32_t idx, uint32_t threshold) {
  const uint32_t h = hash_u32(key, idx >> 1);
  const uint32_t bits = (idx & 1u) ? (h >> 16) : (h & 0xFFFFu);
  return bits >= (threshold >> 16);
}
// 8 consecutive elements starting at an even index: 4 hashes. Applies v = keep ? v * scale : 0.
__device__ __forceinline__ void dropout_apply8(float (&v)[8], uint32_t key, uint32_t idx0,
                                               uint32_t threshold, float scale) {
  const uint32_t t16 = threshold >> 16;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint32_t h = hash_u32(key, (idx0 >> 1) + j);
    v[2 * j] = ((h & 0xFFFFu) >= t16) ? v[2 * j] * scale : 0.0f;
    v[2 * j + 1] = ((h >> 16) >= t16) ? v[2 * j + 1] * scale : 0.0f;
  }
}

// ---- attention dropout words. One hash per (query token, head, group of 8 key columns); the
// four pair-words of the group (two 15-bit lanes each, bits [0,15) and [16,31)) are the hash and
// three multiply-xorshift derivations of it (3 instructions instead of 10 per pair: the hash was
// the largest single item of the softmax loops). A lane keeps its probability iff lane15 >= t15,
// t15 = p * 2^15 (p = 0.1 -> 3276 / 32768).
__device__ __forceinline__ uint32_t attn_drop_group(uint32_t key, int tok, int heads, int head,
                                                    int col_group) {
  return hash_u32(key, ((uint32_t)tok * (uint32_t)heads + (uint32_t)head) * 128u +
                           (uint32_t)col_group);
}
__device__ __forceinline__ uint32_t attn_drop_pair(uint32_t h0, int k) {   // k = pair in group
  if (k == 0) return h0;
  uint32_t w = h0 * (k == 1 ? 0x9E3779B1u : (k == 2 ? 0x85EBCA6Bu : 0xC2B2AE35u));
  return w ^ (w >> 15);
}
// both lanes at once: 0xFFFF in each 16-bit half whose lane is kept. `k2` = (0x8000 - t15) in
// both halves: bit 15 of (lane15 + 0x8000 - t15) is set iff lane15 >= t15; PRMT then replicates
// the sign bits of bytes 1 and 3 over their halves.
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
}
__device__ __forceinline__ uint32_t attn_keep_sum(uint32_t w, uint32_t k2) {
  return (w & 0x7FFF7FFFu) + k2;
}
__device__ __forceinline__ uint32_t attn_keep_mask2(uint32_t w, uint32_t k2) {
  return prmt(attn_keep_sum(w, k2), 0u, 0xBB99u);
}
__device__ __forceinline__ uint32_t attn_drop_k2(uint32_t threshold) {   // threshold = p * 2^32
  const uint32_t k = 0x8000u - (threshold >> 17);
  return k | (k << 16);
}
// scalar form (long-row kernels): is key column j of this query kept?
__device__ __forceinline__ bool attn_drop_keep(uint32_t key, uint32_t threshold, int tok, int heads,
                                               int head, int j) {
  const uint32_t w = attn_drop_pair(attn_drop_group(key, tok, heads, head, j >> 3), (j >> 1) & 3);
  const uint32_t lane = (j & 1) ? ((w >> 16) & 0x7FFFu) : (w & 0x7FFFu);
  return lane >= (threshold >> 17);
}

// exp2 on the MUFU unit (one op per element).
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 0.5 * erfc(|x| / sqrt 2) = 2^(|x| P(|x|) - 1): P is the degree-5 polynomial fitted to
// -log2(erfc(t))/t (t = |x|/sqrt 2 in [0, 6]) with the 1/sqrt2 factors, the sign and the factor
// 0.5 folded into its coefficients. Weighted fit: error of gelu < 3e-7 absolute and < 0.4 %
// relative even in the far negative tail, i.e. below bf16 resolution everywhere. One MUFU op, no
// branches, 7 FP32 instructions — CUDA's erff() costs ~2.5x that and was the GEMM epilogue's
// bottleneck.
__device__ __forceinline__ float half_erfc_abs(float x) {
  const float ax = fminf(fabsf(x), 8.4852814f);
  float p = 3.1522031349595636e-05f;
  p = fmaf(p, ax, -0.000753118481952697f);
  p = fmaf(p, ax, 0.00801779329776764f);
  p = fmaf(p, ax, -0.05329384654760361f);
  p = fmaf(p, ax, -0.4588814675807953f);
  p = fmaf(p, ax, -1.1511543989181519f);
  return fast_ex2(fmaf(p, ax, -1.0f));
}

// gelu(x) = 0.5 x (1 + erf(x / sqrt 2)) = relu(x) - |x| * 0.5 erfc(|x| / sqrt 2)
// (model/layers.py:16-25 of the reference)
__device__ __forceinline__ float gelu_erf(float x) {
  return fmaxf(x, 0.f) - fabsf(x * half_erfc_abs(x));
}
// gelu(x) and its derivative together (the forward FFN-up epilogue saves the derivative so the
// backward epilogue is a plain multiply): shares the erfc evaluation, one extra MUFU for the pdf
// (1/sqrt(2 pi) folded into the exponent).
__device__ __forceinline__ float gelu_erf_with_grad(float x, float& dgelu) {
  const float e = half_erfc_abs(x);
  const float pdf = fast_ex2(fmaf(x * x, -0.72134752044448170f, -1.3257480647361592f));
  const float cdf = 0.5f + copysignf(0.5f - e, x);
  dgelu = fmaf(x, pdf, cdf);
  return fmaxf(x, 0.f) - fabsf(x * e);
}
__device__ __forceinline__ float gelu_erf_grad(float x) {
  float d;
  (void)gelu_erf_with_grad(x, d);
  return d;
}

// TMA store of a smem box (bulk async group) and its group bookkeeping.
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(tmap)),
      "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace hero

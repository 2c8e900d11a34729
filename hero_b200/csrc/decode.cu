// Forward-only decoder attention for a few query rows per sequence: the self-attention and the
// decoder-encoder attention of the TVC caption decoder (model/tvc.py:67-154), teacher-forced and
// one greedy step at a time.
//
// Query row i attends to the key / value rows [kv_off[i], kv_off[i] + kv_len[i]) of K and V. That
// one contract covers every use of the decoder: causal self-attention over a packed caption (row
// (n, t) sees keys 0..t of caption n), a decode step (one query per caption against its KV cache)
// and cross-attention (keys are the caption's segment frames). The reference's -10000 additive
// masks underflow to exactly zero weight after the max subtraction in fp32, so a key range is the
// same softmax.
//
// One CTA of 128 threads per (query row, head). With a handful of queries per (caption, head) a
// tensor-core tile would be almost all padding, so the dot products run on CUDA cores in fp32:
// one thread per key for Q.K (16-byte loads of the 64-element key row), then each warp walks a
// quarter of the keys for P.V with every lane owning two output columns (128-byte coalesced rows).
//
// The gather form (hero_dec_attn_gather_fwd) is the same kernel body with key j of query row i read
// from row kv_idx[i * ld_idx + j] instead of kv_off[i] + j: beam search addresses each beam's
// history through its ancestry table and never copies a KV cache. Only the row lookup differs, so
// the range form's arithmetic, and its results, are those of the kernel before the template.
#include <cuda_bf16.h>
#include <math.h>

#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int DA_THREADS = 128;
constexpr int DA_WARPS = DA_THREADS / 32;
constexpr int DA_HEAD_DIM = 64;
constexpr int DA_MAX_KV = 1024;

__device__ __forceinline__ float da_block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : v + w;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < DA_WARPS; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  __syncthreads();   // red is reused by the next reduction
  return r;
}

// GATHER: key j of row i is row kv_idx[i * ld_idx + j] (checked against [0, n_kv)); otherwise
// row kv_off[i] + j (kv_idx, ld_idx and n_kv unused).
template <bool GATHER>
__global__ void __launch_bounds__(DA_THREADS)
    dec_attn_fwd_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq,
                        const __nv_bfloat16* __restrict__ k, int64_t ldk,
                        const __nv_bfloat16* __restrict__ v, int64_t ldv,
                        const int32_t* __restrict__ kv_off, const int32_t* __restrict__ kv_len,
                        const int32_t* __restrict__ kv_idx, int64_t ld_idx, int32_t n_kv,
                        float scale, __nv_bfloat16* __restrict__ out, int64_t ldo) {
  __shared__ float qs[DA_HEAD_DIM];
  __shared__ float p[DA_MAX_KV];
  __shared__ float part[DA_WARPS][DA_HEAD_DIM];
  __shared__ float red[DA_WARPS];
  const int row = blockIdx.x, head = blockIdx.y, tid = threadIdx.x;
  const int col0 = head * DA_HEAD_DIM;
  pdl_wait();
  pdl_launch_dependents();
  const int off = GATHER ? 0 : __ldg(kv_off + row), len = __ldg(kv_len + row);
  const int32_t* idx = GATHER ? kv_idx + (int64_t)row * ld_idx : nullptr;
  __nv_bfloat16* o = out + (int64_t)row * ldo + col0;
  if (len < 1 || len > DA_MAX_KV) {   // outside the contract: NaN, never a stray read
    if (tid < DA_HEAD_DIM) o[tid] = __float2bfloat16(__int_as_float(0x7fc00000));
    return;
  }
  if (tid < DA_HEAD_DIM) qs[tid] = __bfloat162float(q[(int64_t)row * ldq + col0 + tid]) * scale;
  __syncthreads();

  // scores s_j = (q / sqrt(d)) . k_j, one key per thread
  float mx = -INFINITY;
  bool bad = false;
  for (int j = tid; j < len; j += DA_THREADS) {
    int64_t kj = off + j;
    if constexpr (GATHER) {
      kj = __ldg(idx + j);
      if (kj < 0 || kj >= n_kv) {
        bad = true;
        continue;
      }
    }
    const uint4* kr = reinterpret_cast<const uint4*>(k + kj * ldk + col0);
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < DA_HEAD_DIM / 8; ++c) {
      const uint4 u = __ldg(kr + c);
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __bfloat1622float2(h2[e]);
        s = fmaf(qs[c * 8 + 2 * e], f.x, s);
        s = fmaf(qs[c * 8 + 2 * e + 1], f.y, s);
      }
    }
    p[j] = s;
    mx = fmaxf(mx, s);
  }
  if constexpr (GATHER) {
    if (__syncthreads_or(bad)) {         // a key row outside [0, n_kv): NaN, never a stray read
      if (tid < DA_HEAD_DIM) o[tid] = __float2bfloat16(__int_as_float(0x7fc00000));
      return;
    }
  }
  mx = da_block_reduce(mx, red, true);
  float sum = 0.f;
  for (int j = tid; j < len; j += DA_THREADS) {
    const float e = expf(p[j] - mx);
    p[j] = e;
    sum += e;
  }
  sum = da_block_reduce(sum, red, false);   // its barrier also publishes p[]

  // out = (sum_j e_j v_j) / sum_j e_j: warp w takes keys w, w + 4, ...; lane l columns 2l, 2l+1
  const int warp = tid >> 5, lane = tid & 31;
  float a0 = 0.f, a1 = 0.f;
  for (int j = warp; j < len; j += DA_WARPS) {
    const float pj = p[j];
    const int64_t vj = GATHER ? (int64_t)__ldg(idx + j) : (int64_t)(off + j);
    const float2 f = __bfloat1622float2(
        reinterpret_cast<const __nv_bfloat162*>(v + vj * ldv + col0)[lane]);
    a0 = fmaf(pj, f.x, a0);
    a1 = fmaf(pj, f.y, a1);
  }
  part[warp][2 * lane] = a0;
  part[warp][2 * lane + 1] = a1;
  __syncthreads();
  if (tid < DA_HEAD_DIM) {
    float acc = part[0][tid];
#pragma unroll
    for (int w = 1; w < DA_WARPS; ++w) acc += part[w][tid];
    o[tid] = __float2bfloat16(acc / sum);
  }
}

}  // namespace hero

using namespace hero;

namespace {

int dec_attn_launch(bool gather, const void* q, int64_t ldq, const void* k, int64_t ldk,
                    const void* v, int64_t ldv, const int32_t* kv_off, const int32_t* kv_len,
                    const int32_t* kv_idx, int64_t ld_idx, int32_t n_kv, int32_t rows,
                    int32_t heads, int32_t head_dim, float scale, void* out, int64_t ldo,
                    void* stream, const char* name) {
  HERO_REQUIRE(q && k && v && kv_len && out && (gather ? kv_idx != nullptr : kv_off != nullptr),
               "%s: null pointer", name);
  HERO_REQUIRE(head_dim == DA_HEAD_DIM, "%s: head_dim = %d (only %d)", name, head_dim,
               DA_HEAD_DIM);
  HERO_REQUIRE(rows >= 0 && heads >= 1 && heads <= 65535, "%s: rows %d, heads %d", name, rows,
               heads);
  const int64_t width = (int64_t)heads * head_dim;
  HERO_REQUIRE(ldq >= width && ldk >= width && ldv >= width && ldo >= width,
               "%s: a leading dimension is below heads * head_dim = %lld", name,
               (long long)width);
  HERO_REQUIRE(ldk % 8 == 0 && (reinterpret_cast<uintptr_t>(k) & 15) == 0,
               "%s: K needs 16-byte aligned rows (ldk %lld)", name, (long long)ldk);
  HERO_REQUIRE(ldv % 2 == 0 && (reinterpret_cast<uintptr_t>(v) & 3) == 0,
               "%s: V needs 4-byte aligned rows (ldv %lld)", name, (long long)ldv);
  HERO_REQUIRE(!gather || (ld_idx >= 0 && n_kv >= 1), "%s: ld_idx %lld, n_kv %d", name,
               (long long)ld_idx, n_kv);
  if (rows == 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(gather ? dec_attn_fwd_kernel<true> : dec_attn_fwd_kernel<false>,
                             dim3(rows, heads), dim3(DA_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream),
                             static_cast<const __nv_bfloat16*>(q), ldq,
                             static_cast<const __nv_bfloat16*>(k), ldk,
                             static_cast<const __nv_bfloat16*>(v), ldv, kv_off, kv_len, kv_idx,
                             ld_idx, n_kv, scale, static_cast<__nv_bfloat16*>(out), ldo));
  return HERO_OK;
}

}  // namespace

extern "C" int hero_dec_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk,
                                 const void* v, int64_t ldv, const int32_t* kv_off,
                                 const int32_t* kv_len, int32_t rows, int32_t heads,
                                 int32_t head_dim, float scale, void* out, int64_t ldo,
                                 void* stream) {
  return dec_attn_launch(false, q, ldq, k, ldk, v, ldv, kv_off, kv_len, nullptr, 0, 0, rows, heads,
                         head_dim, scale, out, ldo, stream, "dec_attn_fwd");
}

extern "C" int hero_dec_attn_gather_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk,
                                        const void* v, int64_t ldv, const int32_t* kv_idx,
                                        int64_t ld_idx, const int32_t* kv_len, int32_t n_kv,
                                        int32_t rows, int32_t heads, int32_t head_dim, float scale,
                                        void* out, int64_t ldo, void* stream) {
  return dec_attn_launch(true, q, ldq, k, ldk, v, ldv, nullptr, kv_len, kv_idx, ld_idx, n_kv,
                         rows, heads, head_dim, scale, out, ldo, stream, "dec_attn_gather_fwd");
}

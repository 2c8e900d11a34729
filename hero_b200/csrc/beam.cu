// TVC beam search (hero_b200/tvc.py TvcGenerator.beam_search): the two per-step selections that
// follow the vocabulary GEMM, with no host round trip.
//
//   hero_beam_logprob_topk   per row of fp32 logits: log-sum-exp and the top-B (z - lse, column),
//                            one read of the row
//   hero_beam_select         per caption: the next B beams among the <= B * B candidates of its
//                            beams, their scores / finished flags / lengths, the next step's ids,
//                            and the token-history and KV-ancestry rows copied from each parent
//
// Both order candidates by one 64-bit key, the order-preserving uint32 image of the fp32 value
// above the complement of the item index: a larger key is a larger value, and equal values go to
// the lower item (column, or flat candidate index p * B + k). Keys are unique within a selection,
// so a maximum names its item.
#include <math.h>

#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int BEAM_MAX = 16;
constexpr int BT_THREADS = 512;
constexpr int BT_WARPS = BT_THREADS / 32;
constexpr int BS_PER_LANE = BEAM_MAX * BEAM_MAX / 32;   // candidates per lane of hero_beam_select

__device__ __forceinline__ uint32_t beam_ord(float x) {
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float beam_unord(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}
// 0 is below every real key (the image of -inf is 0x007fffff): an empty slot
__device__ __forceinline__ unsigned long long beam_key(float v, uint32_t item) {
  return ((unsigned long long)beam_ord(v) << 32) | (unsigned long long)(0xffffffffu - item);
}
__device__ __forceinline__ uint32_t beam_item(unsigned long long key) {
  return 0xffffffffu - (uint32_t)(key & 0xffffffffu);
}
__device__ __forceinline__ float beam_value(unsigned long long key) {
  return beam_unord((uint32_t)(key >> 32));
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// KB-entry descending list in registers: insert c if it beats the last entry
template <int KB>
__device__ __forceinline__ void list_push(unsigned long long (&l)[KB], unsigned long long c) {
  if (c <= l[KB - 1]) return;
  l[KB - 1] = c;
#pragma unroll
  for (int i = KB - 1; i > 0; --i) {
    const unsigned long long hi = l[i] > l[i - 1] ? l[i] : l[i - 1];
    const unsigned long long lo = l[i] > l[i - 1] ? l[i - 1] : l[i];
    l[i - 1] = hi;
    l[i] = lo;
  }
}
template <int KB>
__device__ __forceinline__ void list_pop(unsigned long long (&l)[KB]) {
#pragma unroll
  for (int i = 0; i < KB - 1; ++i) l[i] = l[i + 1];
  l[KB - 1] = 0ull;
}

// running (max, sum of exp(x - max)); -inf inputs add nothing
__device__ __forceinline__ void lse_push(float& m, float& s, float x) {
  if (x > m) {
    s *= expf(m - x);
    m = x;
  }
  if (m != -INFINITY) s += expf(x - m);
}
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
  const float mm = fmaxf(m, m2);
  if (mm == -INFINITY) return;
  s = (m == -INFINITY ? 0.f : s * expf(m - mm)) + (m2 == -INFINITY ? 0.f : s2 * expf(m2 - mm));
  m = mm;
}

template <int KB>
__device__ __forceinline__ void topk_push(unsigned long long (&l)[KB], float& m, float& s, float x,
                                          int col) {
  lse_push(m, s, x);
  list_push<KB>(l, beam_key(x, (uint32_t)col));
}

// One CTA per row. Each thread keeps an online (max, sum) and a top-KB list of the columns it reads
// (16-byte loads when the row is aligned); the (max, sum) pairs combine in a fixed tree, and the
// lists merge per warp and then across warps by B rounds of a warp-wide maximum of the list heads.
// Only the first `beam` <= KB entries are produced.
template <int KB>
__global__ void __launch_bounds__(BT_THREADS)
    beam_logprob_topk_kernel(const float* __restrict__ x, int64_t ld, int32_t n, int32_t beam,
                             float* __restrict__ lse_out, float* __restrict__ logp,
                             int32_t* __restrict__ cols) {
  __shared__ unsigned long long wl[BT_WARPS][KB];
  __shared__ float wm[BT_WARPS], ws[BT_WARPS];
  __shared__ float lse_sh;
  const int row = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  pdl_wait();
  pdl_launch_dependents();
  const float* xr = x + (int64_t)row * ld;
  unsigned long long l[KB];
#pragma unroll
  for (int i = 0; i < KB; ++i) l[i] = 0ull;
  float m = -INFINITY, s = 0.f;
  int c0 = 0;
  if ((reinterpret_cast<uintptr_t>(xr) & 15) == 0) {
    const float4* x4 = reinterpret_cast<const float4*>(xr);
    const int n4 = n >> 2;
#pragma unroll 2
    for (int q = tid; q < n4; q += BT_THREADS) {
      const float4 u = __ldg(x4 + q);
      topk_push<KB>(l, m, s, u.x, 4 * q);
      topk_push<KB>(l, m, s, u.y, 4 * q + 1);
      topk_push<KB>(l, m, s, u.z, 4 * q + 2);
      topk_push<KB>(l, m, s, u.w, 4 * q + 3);
    }
    c0 = n4 << 2;
  }
  for (int c = c0 + tid; c < n; c += BT_THREADS) topk_push<KB>(l, m, s, __ldg(xr + c), c);

  // log-sum-exp: warp tree, then warp 0 over the warps in order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    lse_merge(m, s, m2, s2);
  }
  if (lane == 0) {
    wm[warp] = m;
    ws[warp] = s;
  }
  // top-B of the warp: `beam` rounds of the maximum list head, popped by its owner
  for (int r = 0; r < beam; ++r) {
    const unsigned long long mx = warp_max_u64(l[0]);
    if (l[0] == mx && mx != 0ull) list_pop<KB>(l);
    if (lane == 0) wl[warp][r] = mx;
  }
  __syncthreads();
  if (warp != 0) return;
  if (lane == 0) {
    float mm = wm[0], ss = ws[0];
    for (int w = 1; w < BT_WARPS; ++w) lse_merge(mm, ss, wm[w], ws[w]);
    lse_sh = mm + logf(ss);
    lse_out[row] = lse_sh;
  }
  __syncwarp();
  const float lse = lse_sh;
  int ptr = 0;
  unsigned long long head = lane < BT_WARPS ? wl[lane][0] : 0ull;
  for (int r = 0; r < beam; ++r) {
    const unsigned long long mx = warp_max_u64(head);
    if (head == mx && mx != 0ull) {
      ++ptr;
      head = ptr < beam ? wl[lane][ptr] : 0ull;
    }
    if (lane == 0) {
      logp[(int64_t)row * beam + r] = beam_value(mx) - lse;
      cols[(int64_t)row * beam + r] = (int32_t)beam_item(mx);
    }
  }
}

// One warp per caption n, rows n * B .. n * B + B - 1. Candidate c = p * B + k of parent row p:
// live p offers (tok[p, k], score[p] + logp[p, k]) for k < B; finished p offers only k = 0,
// (eos, score[p]). B rounds of a warp-wide maximum pick the next beams in descending score, ties to
// the lower c. New beam b' with parent p then writes its score, finished flag, length (its step
// count up to and including the first eos), the next step's id, and its history rows: hist[., j]
// from p for j < step, the new token at j = step; anc[., j] from p for j <= step and, at
// step + 1, the KV-cache row it writes next, (step + 1) * R + its row.
__global__ void __launch_bounds__(32)
    beam_select_kernel(const float* __restrict__ logp, const int32_t* __restrict__ tok,
                       const float* __restrict__ score_in, const int32_t* __restrict__ fin_in,
                       const int32_t* __restrict__ len_in, const int32_t* __restrict__ hist_in,
                       const int32_t* __restrict__ anc_in, int32_t beam, int32_t step,
                       int32_t max_step, int32_t eos, int32_t n_rows, float* __restrict__ score_out,
                       int32_t* __restrict__ fin_out, int32_t* __restrict__ len_out,
                       int32_t* __restrict__ hist_out, int32_t* __restrict__ anc_out,
                       int32_t* __restrict__ next_ids) {
  __shared__ int32_t par[BEAM_MAX];
  const int lane = threadIdx.x;
  const int base = blockIdx.x * beam;
  pdl_wait();
  pdl_launch_dependents();
  unsigned long long key[BS_PER_LANE];
#pragma unroll
  for (int q = 0; q < BS_PER_LANE; ++q) {
    const int c = lane + 32 * q;
    key[q] = 0ull;
    if (c < beam * beam) {
      const int p = c / beam, k = c - p * beam, r = base + p;
      if (fin_in[r]) {
        if (k == 0) key[q] = beam_key(score_in[r], (uint32_t)c);
      } else {
        key[q] = beam_key(score_in[r] + logp[(int64_t)r * beam + k], (uint32_t)c);
      }
    }
  }
  unsigned long long mine = 0ull;   // lane b' keeps the key of new beam b'
  for (int b = 0; b < beam; ++b) {
    unsigned long long best = 0ull;
#pragma unroll
    for (int q = 0; q < BS_PER_LANE; ++q) best = key[q] > best ? key[q] : best;
    const unsigned long long mx = warp_max_u64(best);
#pragma unroll
    for (int q = 0; q < BS_PER_LANE; ++q)
      if (key[q] == mx) key[q] = 0ull;
    if (lane == b) mine = mx;
  }
  if (lane < beam) {
    const int c = (int)beam_item(mine);
    const int p = c / beam, k = c - p * beam, rp = base + p, r = base + lane;
    const bool done = fin_in[rp] != 0;
    const int32_t t = done ? eos : tok[(int64_t)rp * beam + k];
    score_out[r] = beam_value(mine);
    fin_out[r] = (done || t == eos) ? 1 : 0;
    len_out[r] = done ? len_in[rp] : step + 1;
    next_ids[r] = t;
    hist_out[(int64_t)r * max_step + step] = t;
    par[lane] = rp;
  }
  __syncwarp();
  for (int b = 0; b < beam; ++b) {
    const int64_t src = (int64_t)par[b] * max_step, dst = (int64_t)(base + b) * max_step;
    for (int j = lane; j < step; j += 32) hist_out[dst + j] = hist_in[src + j];
    for (int j = lane; j <= step; j += 32) anc_out[dst + j] = anc_in[src + j];
    if (lane == 0 && step + 1 < max_step) anc_out[dst + step + 1] = (step + 1) * n_rows + base + b;
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_beam_logprob_topk(const float* x, int64_t ld, int32_t rows, int32_t n,
                                      int32_t beam, float* lse, float* logp, int32_t* cols,
                                      void* stream) {
  HERO_REQUIRE(x && lse && logp && cols, "beam_logprob_topk: null pointer");
  HERO_REQUIRE(rows >= 0 && n >= 1 && ld >= n, "beam_logprob_topk: rows %d, n %d, ld %lld", rows,
               n, (long long)ld);
  HERO_REQUIRE(beam >= 1 && beam <= BEAM_MAX && beam <= n,
               "beam_logprob_topk: beam %d (1 to %d, and at most n = %d)", beam, BEAM_MAX, n);
  if (rows == 0) return HERO_OK;
  auto kernel = beam <= 1   ? beam_logprob_topk_kernel<1>
                : beam <= 2 ? beam_logprob_topk_kernel<2>
                : beam <= 4 ? beam_logprob_topk_kernel<4>
                : beam <= 8 ? beam_logprob_topk_kernel<8>
                            : beam_logprob_topk_kernel<16>;
  HERO_CUDA_CHECK(launch_pdl(kernel, dim3(rows), dim3(BT_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream), x, ld, n, beam, lse, logp,
                             cols));
  return HERO_OK;
}

extern "C" int hero_beam_select(const float* logp, const int32_t* tok, const float* score_in,
                                const int32_t* fin_in, const int32_t* len_in,
                                const int32_t* hist_in, const int32_t* anc_in, int32_t n_cap,
                                int32_t beam, int32_t step, int32_t max_step, int32_t eos,
                                float* score_out, int32_t* fin_out, int32_t* len_out,
                                int32_t* hist_out, int32_t* anc_out, int32_t* next_ids,
                                void* stream) {
  HERO_REQUIRE(logp && tok && score_in && fin_in && len_in && hist_in && anc_in && score_out &&
                   fin_out && len_out && hist_out && anc_out && next_ids,
               "beam_select: null pointer");
  HERO_REQUIRE(beam >= 1 && beam <= BEAM_MAX, "beam_select: beam %d (1 to %d)", beam, BEAM_MAX);
  HERO_REQUIRE(n_cap >= 0 && max_step >= 1 && step >= 0 && step < max_step,
               "beam_select: n_cap %d, step %d, max_step %d", n_cap, step, max_step);
  HERO_REQUIRE((int64_t)n_cap * beam * max_step < (int64_t)INT32_MAX,
               "beam_select: %d captions x %d beams x %d steps overflow int32 cache rows", n_cap,
               beam, max_step);
  HERO_REQUIRE(score_in != score_out && hist_in != hist_out && anc_in != anc_out &&
                   fin_in != fin_out && len_in != len_out,
               "beam_select: the state is read from one buffer and written to another");
  if (n_cap == 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(beam_select_kernel, dim3(n_cap), dim3(32), 0,
                             reinterpret_cast<cudaStream_t>(stream), logp, tok, score_in, fin_in,
                             len_in, hist_in, anc_in, beam, step, max_step, eos, n_cap * beam,
                             score_out, fin_out, len_out, hist_out, anc_out, next_ids));
  return HERO_OK;
}

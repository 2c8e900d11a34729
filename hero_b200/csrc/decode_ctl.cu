// TVC decoding controls (hero_b200/tvc.py TvcGenerator): the per-step token bans and the sampler
// that sit between the vocabulary GEMM and the next step's ids, with no host round trip.
//
//   hero_dec_ban_tokens    per row: -inf into the logits of the tokens that would repeat an n-gram
//                          of the row's history, and into EOS while the step is below min_length
//   hero_sample_tokens     per row: temperature, top-k and top-p, then one Gumbel-max draw written
//                          straight into the next step's id row
//
// Bans (step t, row r, history y_0 .. y_{t-1} read at hist[j * step_stride + r * row_stride]):
//   s = [bos, y_0, ..., y_{t-1}], L = t + 1. With n >= 1 and L >= n, for every start
//   j in [0, L - n]: if s[j .. j + n - 2] == s[L - n + 1 .. L - 1] then token s[j + n - 1] is banned
//   (n == 1: every token of s). If t < min_length, eos is banned. A banned column c < n_valid gets
//   logits[r, c] = -inf; the other columns are untouched. Masking comes before any normalisation.
//
// Sampling (row r of fp32 logits z over its first n columns, step t):
//   1. x_j = z_j / temperature (fp32 division).
//   2. top-k, 0 < k < n: keep j iff key(x_j) >= the k-th largest key (ties at it kept).
//   3. top-p, p < 1: over the kept columns, w_j = floor(exp(x_j - max x) * 2^32) as an integer
//      (fp32 exp), W = sum w_j, need = max(1, ceil(p * W)) in fp64; keep j iff key(x_j) >= theta,
//      theta the largest key such that the kept columns with key >= theta weigh >= need.
//   4. id = argmax over the kept j with x_j > -inf of (x_j + G_j), ties to the lower j, with
//        rkey = hash_u32(hash_u32(seed, r), t)
//        u_j  = ((hash_u32(rkey, j) >> 9) + 0.5) * 2^-23       (2^-24 .. 1 - 2^-24, exact in fp32)
//        G_j  = -log(-log(u_j))                                 (fp32 logf; finite, at most 16.6)
//      hash_u32 is the dropout hash of ptx.cuh. Gumbel-max draws from softmax(x) over the kept
//      set (up to the 2^-23 resolution of the uniforms): no sort and no stored random state. A
//      -inf column (a banned token) has probability 0 and is never drawn.
// key() is the order-preserving uint32 image of the float (radix_select.cuh ord_key). Both
// thresholds come from the 8-bit radix passes of radix_select.cuh: counts for top-k, integer masses
// for top-p.
//
// Early stop (hero_dec_finished, after each step's selection): fin[r] |= (ids[r] == eos) when ids
// is given (greedy / sampling); fin is read as-is otherwise (beam search: the finished flags
// hero_beam_select just wrote). If every fin[r], r < rows, is set and *stop_dev still holds
// INT32_MAX, the step is stored in *stop_dev and, with a system-scope release store, in the pinned
// host word *stop_host, which the host polls with a plain load before it enqueues the next step.
// The device never reads the host word, and a set step is never moved.
#include <limits.h>
#include <math.h>

#include <atomic>

#include "common.h"
#include "ptx.cuh"
#include "radix_select.cuh"

namespace hero {

constexpr int BAN_THREADS = 256;
constexpr int BAN_MAX_HIST = 1024;             // bos + 1023 steps (TvcGenerator's position table)
constexpr int SAMPLE_THREADS = 1024;
constexpr int SAMPLE_MAX_COLS = 52 * 1024;     // the staged row: 208 KB of the 227 KB per block
constexpr int FIN_THREADS = 256;

// One CTA per row: the history is staged in shared memory, each thread takes start positions j
// and compares the (n - 1)-token window with the suffix. Several threads may write -inf into the
// same column.
__global__ void __launch_bounds__(BAN_THREADS)
    dec_ban_tokens_kernel(float* __restrict__ x, int64_t ld, int32_t n_valid,
                          const int32_t* __restrict__ hist, int64_t step_stride,
                          int64_t row_stride, int32_t bos, int32_t step, int32_t ngram,
                          int32_t min_length, int32_t eos) {
  __shared__ int32_t s[BAN_MAX_HIST];
  const int row = blockIdx.x, tid = threadIdx.x;
  const int L = step + 1;
  pdl_wait();
  pdl_launch_dependents();
  float* xr = x + (int64_t)row * ld;
  if (tid == 0 && step < min_length && eos >= 0 && eos < n_valid) xr[eos] = -INFINITY;
  if (ngram <= 0 || L < ngram) return;
  const int32_t* h = hist + (int64_t)row * row_stride;
  for (int j = tid; j < L; j += BAN_THREADS) s[j] = j == 0 ? bos : h[(int64_t)(j - 1) * step_stride];
  __syncthreads();
  const int m = ngram - 1, suffix = L - m;
  for (int j = tid; j <= L - ngram; j += BAN_THREADS) {
    bool hit = true;
    for (int i = 0; i < m && hit; ++i) hit = s[j + i] == s[suffix + i];
    const int32_t tok = s[j + m];
    if (hit && tok >= 0 && tok < n_valid) xr[tok] = -INFINITY;
  }
}

// The row staged in shared memory as x = z / temperature
struct StagedKeys {
  const float* x;
  __device__ __forceinline__ bool get(int t, uint32_t& k) const {
    k = ord_key(x[t]);
    return true;
  }
};
__device__ __forceinline__ unsigned long long sample_mass(float x, float mx) {
  return __float2ull_rz(expf(x - mx) * 4294967296.f);
}
// The columns kept by top-k (key >= lo), weighted by their integer mass
struct StagedMass {
  const float* x;
  uint32_t lo;
  float mx;
  __device__ __forceinline__ bool get(int t, uint32_t& k) const {
    k = ord_key(x[t]);
    return k >= lo;
  }
  __device__ __forceinline__ unsigned long long weight(int t) const { return sample_mass(x[t], mx); }
};

static_assert(SAMPLE_MAX_COLS * sizeof(float) + 2 * sizeof(RadixSmem<unsigned long long>) +
                      SAMPLE_THREADS * sizeof(unsigned long long) + 64 <=
                  227 * 1024,
              "the staged sampler row exceeds the sm_90 shared memory per block");

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// One CTA per row; the row is read from global memory once and kept in dynamic shared memory for
// the up to 10 passes that follow (max, 4 count passes, total mass, 4 mass passes, the draw).
__global__ void __launch_bounds__(SAMPLE_THREADS, 1)
    sample_tokens_kernel(const float* __restrict__ z, int64_t ld, int32_t n, float temperature,
                         int32_t top_k, float top_p, uint32_t seed, int32_t step,
                         int32_t* __restrict__ ids) {
  extern __shared__ float xs[];
  __shared__ RadixSmem<uint32_t> rc;
  __shared__ RadixSmem<unsigned long long> rm;
  __shared__ unsigned long long scratch[SAMPLE_THREADS];
  __shared__ uint32_t s_max;
  __shared__ unsigned long long s_total, s_best;
  const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  if (tid == 0) {
    s_max = 0u;
    s_total = 0ull;
    s_best = 0ull;
  }
  pdl_wait();
  pdl_launch_dependents();
  const float* zr = z + (int64_t)row * ld;
  uint32_t mk = 0u;
  for (int j = tid; j < n; j += SAMPLE_THREADS) {
    const float v = __ldg(zr + j) / temperature;
    xs[j] = v;
    mk = max(mk, ord_key(v));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mk = max(mk, __shfl_xor_sync(0xffffffffu, mk, o));
  __syncthreads();                                    // xs and the zeroed scalars
  if (lane == 0) atomicMax(&s_max, mk);
  uint32_t thr = 0u;                                  // keep j iff key(x_j) >= thr
  if (top_k > 0 && top_k < n) {
    uint32_t need;
    bool all;
    block_radix_select<SAMPLE_THREADS, false>(StagedKeys{xs}, n, (uint32_t)top_k, rc, thr, need,
                                              all);
    if (all) thr = 0u;
  }
  __syncthreads();                                    // s_max
  if (top_p < 1.f) {
    const float mx = key_to_float(s_max);
    unsigned long long tot = 0ull;
    for (int j = tid; j < n; j += SAMPLE_THREADS)
      if (ord_key(xs[j]) >= thr) tot += sample_mass(xs[j], mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
    if (lane == 0) atomicAdd(&s_total, tot);
    __syncthreads();
    unsigned long long need = (unsigned long long)ceil((double)top_p * (double)s_total);
    if (need < 1ull) need = 1ull;
    uint32_t pthr;
    unsigned long long rest;
    bool all;
    block_radix_select<SAMPLE_THREADS, true>(StagedMass{xs, thr, mx}, n, need, rm, pthr, rest,
                                             all, scratch);
    thr = pthr;                                       // >= thr: only kept columns have weight
  }
  const uint32_t rkey = hash_u32(hash_u32(seed, (uint32_t)row), (uint32_t)step);
  unsigned long long best = 0ull;
  for (int j = tid; j < n; j += SAMPLE_THREADS) {
    const float v = xs[j];
    if (ord_key(v) < thr || v == -INFINITY) continue;
    // 23 bits + 0.5 fit the fp32 significand exactly, so u < 1 and G is finite
    const float u = ((float)(hash_u32(rkey, (uint32_t)j) >> 9) + 0.5f) * 1.1920928955078125e-7f;
    const float g = -logf(-logf(u));
    const unsigned long long c =
        ((unsigned long long)ord_key(v + g) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)j);
    best = c > best ? c : best;
  }
  best = warp_max_u64(best);
  if (lane == 0) atomicMax(&s_best, best);
  __syncthreads();
  if (tid == 0) ids[row] = (int32_t)(0xffffffffu - (uint32_t)(s_best & 0xffffffffu));
}

// One CTA: rows is at most n_captions x 16 beams, a few thousand flags.
__global__ void __launch_bounds__(FIN_THREADS)
    dec_finished_kernel(const int32_t* __restrict__ ids, int32_t* __restrict__ fin, int32_t rows,
                        int32_t eos, int32_t step, int32_t* __restrict__ stop_dev,
                        int32_t* stop_host) {
  const int tid = threadIdx.x;
  pdl_wait();
  pdl_launch_dependents();
  int all = 1;
  for (int r = tid; r < rows; r += FIN_THREADS) {
    int32_t f = fin[r];
    if (ids != nullptr && !f && ids[r] == eos) fin[r] = f = 1;
    all &= f != 0;
  }
  all = __syncthreads_and(all);
  if (tid == 0 && all && *stop_dev == INT_MAX) {
    *stop_dev = step;
    asm volatile("st.release.sys.s32 [%0], %1;" ::"l"(stop_host), "r"(step) : "memory");
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_dec_ban_tokens(float* x, int64_t ld, int32_t rows, int32_t n_valid,
                                   const int32_t* hist, int64_t step_stride, int64_t row_stride,
                                   int32_t bos, int32_t step, int32_t ngram, int32_t min_length,
                                   int32_t eos, void* stream) {
  HERO_REQUIRE(x && (hist || step == 0 || ngram == 0), "dec_ban_tokens: null pointer");
  HERO_REQUIRE(rows >= 0 && n_valid >= 1 && ld >= n_valid,
               "dec_ban_tokens: rows %d, n_valid %d, ld %lld", rows, n_valid, (long long)ld);
  HERO_REQUIRE(step >= 0 && step < BAN_MAX_HIST, "dec_ban_tokens: step %d outside [0, %d)", step,
               BAN_MAX_HIST);
  HERO_REQUIRE(ngram >= 0 && min_length >= 0, "dec_ban_tokens: ngram %d, min_length %d", ngram,
               min_length);
  if (rows == 0 || (ngram == 0 && step >= min_length)) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(dec_ban_tokens_kernel, dim3(rows), dim3(BAN_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream), x, ld, n_valid, hist,
                             step_stride, row_stride, bos, step, ngram, min_length, eos));
  return HERO_OK;
}

extern "C" int hero_sample_tokens(const float* x, int64_t ld, int32_t rows, int32_t n,
                                  float temperature, int32_t top_k, float top_p, uint32_t seed,
                                  int32_t step, int32_t* ids, void* stream) {
  HERO_REQUIRE(x && ids, "sample_tokens: null pointer");
  HERO_REQUIRE(rows >= 0 && n >= 1 && n <= SAMPLE_MAX_COLS && ld >= n,
               "sample_tokens: %d columns (ld %lld) outside [1, %d]", n, (long long)ld,
               SAMPLE_MAX_COLS);
  HERO_REQUIRE(temperature > 0.f && isfinite(temperature) && top_k >= 0 && top_p > 0.f &&
                   top_p <= 1.f && step >= 0,
               "sample_tokens: temperature %g, top_k %d, top_p %g, step %d", (double)temperature,
               top_k, (double)top_p, step);
  if (rows == 0) return HERO_OK;
  const size_t smem = (size_t)n * sizeof(float);
  // The opt-in is set once per device, to the size of the largest row, so it never changes
  // between another host thread's check and launch.
  int dev = 0;
  HERO_CUDA_CHECK(cudaGetDevice(&dev));
  static std::atomic<unsigned long long> configured{0ull};
  const unsigned long long bit = 1ull << (dev & 63);
  if ((configured.load() & bit) == 0ull) {
    HERO_CUDA_CHECK(cudaFuncSetAttribute(sample_tokens_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)(SAMPLE_MAX_COLS * sizeof(float))));
    configured.fetch_or(bit);
  }
  HERO_CUDA_CHECK(launch_pdl(sample_tokens_kernel, dim3(rows), dim3(SAMPLE_THREADS), smem,
                             reinterpret_cast<cudaStream_t>(stream), x, ld, n, temperature, top_k,
                             top_p, seed, step, ids));
  return HERO_OK;
}

extern "C" int hero_dec_finished(const int32_t* ids, int32_t* fin, int32_t rows, int32_t eos,
                                 int32_t step, int32_t* stop_dev, int32_t* stop_host,
                                 void* stream) {
  HERO_REQUIRE((fin || rows == 0) && stop_dev && stop_host, "dec_finished: null pointer");
  HERO_REQUIRE(rows >= 0 && step >= 0, "dec_finished: rows %d, step %d", rows, step);
  // The kernel stores into the host word through its device mapping: a pageable pointer has none.
  cudaPointerAttributes attr;
  HERO_CUDA_CHECK(cudaPointerGetAttributes(&attr, stop_host));
  HERO_REQUIRE(attr.type == cudaMemoryTypeHost && attr.devicePointer != nullptr,
               "dec_finished: stop_host is not pinned, device-mapped host memory");
  HERO_CUDA_CHECK(launch_pdl(dec_finished_kernel, dim3(1), dim3(FIN_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream), ids, fin, rows, eos, step,
                             stop_dev, static_cast<int32_t*>(attr.devicePointer)));
  return HERO_OK;
}

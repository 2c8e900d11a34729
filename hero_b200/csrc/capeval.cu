// TVC caption metrics: the per-clip integer counts and fp64 partials of BLEU-1..4, ROUGE-L and
// CIDEr-D (the reference's eval/pycocoevalcap/{bleu,rouge,cider}, which loop over Python dicts on the
// host). The host finishes the O(clips) arithmetic in the reference's expression order.
//
// Sentences are CSR word ids (1..65535), one hypothesis per clip (sentences 0..n_clips-1) followed by
// the references (clip c owns n_clips + ref_off[c] .. n_clips + ref_off[c + 1] - 1). An n-gram is an
// exact 64-bit key of four 16-bit slots, w0 << 48 | w1 << 32 | w2 << 16 | w3, unused slots 0; keys
// compare as signed 64-bit integers everywhere (that is the order torch.sort gives the df table).
//
//  1. caption_ngrams_kernel, one CTA per sentence: every n-gram key (n = 1..4) in shared memory,
//     bitonic-sorted and run-length counted into the sentence's slice of ukey / ucnt.
//  2. caption_df_keys_kernel, one CTA per clip: each reference n-gram that no earlier reference of
//     the same clip has, so the clip's union of reference n-grams appears once; other slots get 0
//     (never a key). The caller sorts this; df(g) is the length of g's run, found by binary search.
//  3. caption_clip_kernel, one CTA per clip: BLEU clipped matches and the closest reference length,
//     per reference the CIDEr-D similarity of each order in fp64, and a bit-parallel LCS per
//     (hypothesis, reference) pair, one warp per pair. No floating-point atomics: every fp64 sum is
//     a fixed-order reduction, so two runs give the same bits.
#include <limits.h>
#include <stdint.h>

#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int CAP_MAX_LEN = 1024;                 // words per sentence
constexpr int CAP_MAX_GRAMS = 4 * CAP_MAX_LEN;    // >= 4 * len - 6, a power of two
constexpr int CAP_SORT_THREADS = 256;
constexpr int CAP_CLIP_THREADS = 128;
constexpr int CAP_CLIP_WARPS = CAP_CLIP_THREADS / 32;
constexpr double CAP_SIGMA = 6.0;

__device__ __forceinline__ int cap_grams(int len) {
  int g = 0;
#pragma unroll
  for (int n = 1; n <= 4; ++n) g += max(0, len - n + 1);
  return g;
}

// n of an n-gram key: its non-zero slots (the words of an n-gram are all non-zero)
__device__ __forceinline__ int cap_order(long long k) {
  const unsigned long long u = (unsigned long long)k;
  return 1 + (((u >> 32) & 0xFFFF) != 0) + (((u >> 16) & 0xFFFF) != 0) + ((u & 0xFFFF) != 0);
}

// index of key in the ascending a[0, n), or -1
__device__ __forceinline__ int cap_find(const long long* a, int n, long long key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return (lo < n && a[lo] == key) ? lo : -1;
}

// number of entries equal to key in the ascending a[0, n)
__device__ __forceinline__ int cap_count(const long long* a, long long n, long long key) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  long long lo2 = lo, hi2 = n;
  while (lo2 < hi2) {
    const long long mid = (lo2 + hi2) >> 1;
    if (a[mid] <= key) lo2 = mid + 1; else hi2 = mid;
  }
  return (int)(lo2 - lo);
}

__global__ void __launch_bounds__(CAP_SORT_THREADS)
caption_ngrams_kernel(const int32_t* __restrict__ sent_off, const int32_t* __restrict__ gram_off,
                      const int32_t* __restrict__ tok, long long* __restrict__ ukey,
                      int32_t* __restrict__ ucnt, int32_t* __restrict__ nuniq) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ long long key[CAP_MAX_GRAMS];
  __shared__ int warp_sum[CAP_SORT_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int s = blockIdx.x;
  const int t0 = sent_off[s], len = sent_off[s + 1] - t0;
  const int ng = cap_grams(len);
  int p2 = 1;
  while (p2 < ng) p2 <<= 1;
  for (int i = tid; i < p2; i += CAP_SORT_THREADS) {
    long long k = LLONG_MAX;                       // padding sorts last and is never read back
    if (i < ng) {
      int n = 1, pos = i;                          // unigrams first, then bigrams, ...
      while (pos >= len - n + 1) { pos -= len - n + 1; ++n; }
      unsigned long long u = 0;
      for (int j = 0; j < 4; ++j)
        u = (u << 16) | (j < n ? (unsigned long long)(uint16_t)tok[t0 + pos + j] : 0ull);
      k = (long long)u;
    }
    key[i] = k;
  }
  __syncthreads();
  for (int k = 2; k <= p2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < p2; i += CAP_SORT_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const long long a = key[i], b = key[ixj];
          if ((a > b) == ((i & k) == 0)) { key[i] = b; key[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  // run heads in a contiguous chunk per thread, then a block exclusive scan of the chunk counts
  const int chunk = (ng + CAP_SORT_THREADS - 1) / CAP_SORT_THREADS;
  const int c0 = min(ng, tid * chunk), c1 = min(ng, c0 + chunk);
  int heads = 0;
  for (int i = c0; i < c1; ++i) heads += (i == 0 || key[i] != key[i - 1]);
  int incl = heads;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_sum[warp] = incl;
  __syncthreads();
  int base = incl - heads;
  for (int w = 0; w < warp; ++w) base += warp_sum[w];
  long long* uk = ukey + gram_off[s];
  int32_t* uc = ucnt + gram_off[s];
  for (int i = c0; i < c1; ++i) {
    if (i != 0 && key[i] == key[i - 1]) continue;
    int e = i + 1;
    while (e < ng && key[e] == key[i]) ++e;
    uk[base] = key[i];
    uc[base] = e - i;
    ++base;
  }
  if (tid == CAP_SORT_THREADS - 1) nuniq[s] = base;
}

__global__ void __launch_bounds__(CAP_SORT_THREADS)
caption_df_keys_kernel(const int32_t* __restrict__ sent_off, const int32_t* __restrict__ gram_off,
                       const int32_t* __restrict__ ref_off, int n_clips,
                       const long long* __restrict__ ukey, const int32_t* __restrict__ nuniq,
                       long long* __restrict__ dfk) {
  pdl_wait();
  pdl_launch_dependents();
  const int c = blockIdx.x;
  const int r0 = n_clips + ref_off[c], r1 = n_clips + ref_off[c + 1];
  const int base = gram_off[n_clips];
  for (int r = r0; r < r1; ++r) {
    const int cap = gram_off[r + 1] - gram_off[r], nu = nuniq[r];
    const long long* uk = ukey + gram_off[r];
    for (int i = threadIdx.x; i < cap; i += CAP_SORT_THREADS) {
      long long k = 0;
      if (i < nu) {
        k = uk[i];
        for (int q = r0; q < r; ++q)
          if (cap_find(ukey + gram_off[q], nuniq[q], k) >= 0) { k = 0; break; }
      }
      dfk[gram_off[r] - base + i] = k;
    }
  }
}

// v[base + n - 1] += x, branch-free so that v stays in registers (adding 0.0 elsewhere changes
// no sum: the partials are never -0.0 that matters, every weight is >= 0)
template <int V>
__device__ __forceinline__ void cap_add(double (&v)[V], int base, int n, double x) {
#pragma unroll
  for (int j = 0; j < 4; ++j) v[base + j] += n == j + 1 ? x : 0.0;
}

// Fixed-order CTA sum of V doubles per thread: butterfly within each warp, then warp 0..W-1 in
// order. Every thread gets the totals.
template <int V>
__device__ __forceinline__ void cap_block_sum(double (&v)[V], double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < V; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
  __syncthreads();                                  // red is free
  if (lane == 0)
#pragma unroll
    for (int j = 0; j < V; ++j) red[warp * V + j] = v[j];
  __syncthreads();
#pragma unroll
  for (int j = 0; j < V; ++j) {
    double t = red[j];
    for (int w = 1; w < CAP_CLIP_WARPS; ++w) t += red[w * V + j];
    v[j] = t;
  }
}

// LCS length of a (hyp, length m <= 1024, word ids >= 1) and b (length n) by one warp: the
// bit-parallel recurrence V' = (V + (V & M_b)) | (V & ~M_b) (Hyyro 2004) on an m-bit vector, lane l
// holding bits 32l .. 32l + 31; LCS = zero bits of V below m. The 1024-bit add carries across lanes
// by one carry-lookahead step on the lanes' generate / propagate ballots.
__device__ int cap_lcs_warp(const int32_t* __restrict__ a, int m, const int32_t* __restrict__ b,
                            int n) {
  const int lane = threadIdx.x & 31;
  int av[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const int i = lane * 32 + k;
    av[k] = i < m ? a[i] : 0;
  }
  uint32_t v = 0xFFFFFFFFu;
  for (int j = 0; j < n; ++j) {
    const int w = b[j];
    uint32_t mb = 0;
#pragma unroll
    for (int k = 0; k < 32; ++k) mb |= (uint32_t)(av[k] == w) << k;
    const uint32_t u = v & mb;
    const unsigned long long s64 = (unsigned long long)v + u;
    uint32_t s = (uint32_t)s64;
    const uint32_t g = __ballot_sync(0xffffffffu, (s64 >> 32) != 0);
    const uint32_t p = __ballot_sync(0xffffffffu, s == 0xFFFFFFFFu);   // exclusive with g
    const uint32_t carry_in = ((g | p) + g) ^ p;
    s += (carry_in >> lane) & 1u;
    v = s | (v & ~mb);
  }
  const int valid = min(32, max(0, m - lane * 32));
  const uint32_t mask = valid == 32 ? 0xFFFFFFFFu : ((1u << valid) - 1u);
  int zeros = __popc(~v & mask);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) zeros += __shfl_xor_sync(0xffffffffu, zeros, o);
  return zeros;
}

__global__ void __launch_bounds__(CAP_CLIP_THREADS)
caption_clip_kernel(const int32_t* __restrict__ sent_off, const int32_t* __restrict__ gram_off,
                    const int32_t* __restrict__ ref_off, const int32_t* __restrict__ tok,
                    int n_clips, const long long* __restrict__ ukey,
                    const int32_t* __restrict__ ucnt, const int32_t* __restrict__ nuniq,
                    const long long* __restrict__ df, long long n_df,
                    const double* __restrict__ log_n, double* __restrict__ out) {
  pdl_wait();
  pdl_launch_dependents();
  extern __shared__ __align__(16) unsigned char cap_smem[];
  __shared__ double red[CAP_CLIP_WARPS * 8];
  __shared__ int ired[CAP_CLIP_WARPS * 4];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = blockIdx.x;
  const int nh = nuniq[c];
  long long* hkey = reinterpret_cast<long long*>(cap_smem);
  double* hidf = reinterpret_cast<double*>(hkey + nh);
  int32_t* hcnt = reinterpret_cast<int32_t*>(hidf + nh);
  int32_t* hmax = hcnt + nh;
  const int hl = sent_off[c + 1] - sent_off[c];
  const int r0 = n_clips + ref_off[c], r1 = n_clips + ref_off[c + 1];
  const double ref_len = log_n[n_clips];

  // hypothesis: idf of each n-gram, its norm per order
  double nh2[4] = {0.0, 0.0, 0.0, 0.0};
  for (int i = tid; i < nh; i += CAP_CLIP_THREADS) {
    const long long k = ukey[gram_off[c] + i];
    const int cnt = ucnt[gram_off[c] + i];
    const double idf = ref_len - log_n[max(1, cap_count(df, n_df, k))];
    hkey[i] = k;
    hcnt[i] = cnt;
    hidf[i] = idf;
    hmax[i] = 0;
    const double w = (double)cnt * idf;
    cap_add(nh2, 0, cap_order(k), w * w);
  }
  cap_block_sum<4>(nh2, red);                      // its first barrier publishes the arrays
  double norm_h[4];
#pragma unroll
  for (int n = 0; n < 4; ++n) norm_h[n] = sqrt(nh2[n]);
  const int bh = max(0, hl - 1);                   // the reference's "length": bigram count

  double* ref_out = out + 5ll * n_clips;
  for (int r = r0; r < r1; ++r) {
    const int nr = nuniq[r];
    const long long* rk = ukey + gram_off[r];
    const int32_t* rc = ucnt + gram_off[r];
    double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};   // ref norm^2 [4], dot [4]
    for (int i = tid; i < nr; i += CAP_CLIP_THREADS) {
      const long long k = rk[i];
      const double w = (double)rc[i] * (ref_len - log_n[max(1, cap_count(df, n_df, k))]);
      cap_add(acc, 0, cap_order(k), w * w);
    }
    for (int i = tid; i < nh; i += CAP_CLIP_THREADS) {
      const int j = cap_find(rk, nr, hkey[i]);
      if (j < 0) continue;
      const int cr = rc[j];
      hmax[i] = max(hmax[i], cr);
      const double wr = (double)cr * hidf[i], wh = (double)hcnt[i] * hidf[i];
      cap_add(acc, 4, cap_order(hkey[i]), fmin(wh, wr) * wr);
    }
    cap_block_sum<8>(acc, red);
    if (tid == 0) {
      const int rl = sent_off[r + 1] - sent_off[r];
      const double delta = (double)(bh - max(0, rl - 1));
      const double pen = exp(-(delta * delta) / (2.0 * CAP_SIGMA * CAP_SIGMA));
      double* o = ref_out + 5ll * (r - n_clips);
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        double val = acc[4 + n];
        const double nrm = sqrt(acc[n]);
        if (norm_h[n] != 0.0 && nrm != 0.0) val /= norm_h[n] * nrm;
        o[n] = val * pen;
      }
    }
  }
  __syncthreads();                                  // hmax complete

  // BLEU: clipped matches per order
  int corr[4] = {0, 0, 0, 0};
  for (int i = tid; i < nh; i += CAP_CLIP_THREADS) {
    const int n = cap_order(hkey[i]), m = min(hcnt[i], hmax[i]);
#pragma unroll
    for (int j = 0; j < 4; ++j) corr[j] += j == n - 1 ? m : 0;
  }
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) corr[n] += __shfl_xor_sync(0xffffffffu, corr[n], o);
  if (lane == 0)
#pragma unroll
    for (int n = 0; n < 4; ++n) ired[warp * 4 + n] = corr[n];
  __syncthreads();
  if (tid == 0) {
    double* o = out + 5ll * c;
    for (int n = 0; n < 4; ++n) {
      int t = 0;
      for (int w = 0; w < CAP_CLIP_WARPS; ++w) t += ired[w * 4 + n];
      o[n] = (double)t;
    }
    // closest reference length, ties to the shorter: min over (|l - hl|, l)
    int best = -1, best_d = 0;
    for (int r = r0; r < r1; ++r) {
      const int l = sent_off[r + 1] - sent_off[r], d = abs(l - hl);
      if (best < 0 || d < best_d || (d == best_d && l < best)) { best = l; best_d = d; }
    }
    o[4] = (double)best;
  }

  // ROUGE-L: one warp per (hypothesis, reference) pair
  for (int r = r0 + warp; r < r1; r += CAP_CLIP_WARPS) {
    const int lcs = cap_lcs_warp(tok + sent_off[c], hl, tok + sent_off[r],
                                 sent_off[r + 1] - sent_off[r]);
    if (lane == 0) ref_out[5ll * (r - n_clips) + 4] = (double)lcs;
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_caption_ngrams(const int32_t* sent_off, const int32_t* gram_off,
                                   const int32_t* ref_off, const int32_t* tok, int32_t n_clips,
                                   int32_t n_sent, long long* ukey, int32_t* ucnt, int32_t* nuniq,
                                   long long* dfk, void* stream) {
  HERO_REQUIRE(sent_off && gram_off && ref_off && tok && ukey && ucnt && nuniq && dfk,
               "caption_ngrams: null pointer");
  HERO_REQUIRE(n_clips >= 1 && n_sent > n_clips, "caption_ngrams: %d clips, %d sentences", n_clips,
               n_sent);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  HERO_CUDA_CHECK(launch_pdl(caption_ngrams_kernel, dim3(n_sent), dim3(CAP_SORT_THREADS), 0, st,
                             sent_off, gram_off, tok, ukey, ucnt, nuniq));
  HERO_CUDA_CHECK(launch_pdl(caption_df_keys_kernel, dim3(n_clips), dim3(CAP_SORT_THREADS), 0, st,
                             sent_off, gram_off, ref_off, (int)n_clips, (const long long*)ukey,
                             (const int32_t*)nuniq, dfk));
  return HERO_OK;
}

extern "C" int hero_caption_clip_stats(const int32_t* sent_off, const int32_t* gram_off,
                                       const int32_t* ref_off, const int32_t* tok, int32_t n_clips,
                                       int32_t max_hyp_grams, const long long* ukey,
                                       const int32_t* ucnt, const int32_t* nuniq,
                                       const long long* df, int64_t n_df, const double* log_n,
                                       double* out, void* stream) {
  HERO_REQUIRE(sent_off && gram_off && ref_off && tok && ukey && ucnt && nuniq && df && log_n && out,
               "caption_clip_stats: null pointer");
  HERO_REQUIRE(n_clips >= 1, "caption_clip_stats: %d clips", n_clips);
  HERO_REQUIRE(max_hyp_grams >= 0 && max_hyp_grams <= CAP_MAX_GRAMS,
               "caption_clip_stats: max_hyp_grams = %d outside [0, %d]", max_hyp_grams,
               CAP_MAX_GRAMS);
  HERO_REQUIRE(n_df >= 0, "caption_clip_stats: n_df = %lld", (long long)n_df);
  const size_t smem = (size_t)max_hyp_grams * (sizeof(long long) + sizeof(double) + 2 * sizeof(int));
  HERO_CUDA_CHECK(cudaFuncSetAttribute(caption_clip_kernel,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  HERO_CUDA_CHECK(launch_pdl(caption_clip_kernel, dim3(n_clips), dim3(CAP_CLIP_THREADS), smem,
                             reinterpret_cast<cudaStream_t>(stream), sent_off, gram_off, ref_off,
                             tok, (int)n_clips, ukey, ucnt, nuniq, df, (long long)n_df, log_n,
                             out));
  return HERO_OK;
}

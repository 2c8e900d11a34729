// Full-corpus retrieval ranking (eval_vcmr.py:205-418 / eval_vr.py:198-260 of the reference): the
// selections that follow the query-vs-corpus GEMM, with no (Nq, K, L, L) tensor, no full sort and
// no host round trip.
//
//   hero_rank_topk          per-row top-K of an fp32 matrix (video scores), optionally exp(a.x)
//   hero_vcmr_span_probs    start / end probabilities of selected (query, clip) pairs, read from
//                           the p^ . c^ GEMM rows and rescaled by the stored inverse norms
//   hero_vcmr_moment_topn   per-query top-N of st[s] . video_factor . ed[e] over the band-valid
//                           (clip, start, end) triples, enumerated on the fly
//
// Both selections are one CTA per row: an 8-bit radix select on the order-preserving uint32 image
// of the float (radix_select.cuh) finds the N-th largest key, the survivors are gathered (ties at
// the threshold in ascending item order) and bitonic-sorted in shared memory on (key, -item). The
// output order is therefore deterministic: descending value, ties to the lower item index.
#include "common.h"
#include "ptx.cuh"
#include "radix_select.cuh"

namespace hero {

constexpr int RANK_THREADS = 512;
constexpr int RANK_MAX_N = 1024;          // K of hero_rank_topk, N of hero_vcmr_moment_topn
constexpr int RANK_MAX_COLS = 65536;      // columns of hero_rank_topk
constexpr int RANK_MAX_L = 512;           // frames per clip
constexpr int RANK_MAX_KW = 15;           // span convolution width
constexpr int MOMENT_SMEM_MAX = 160 * 1024;   // st / ed / factor staged in shared memory up to this
constexpr float kRankMaskFill = -1e4f;    // mask_logits (model/modeling_utils.py:42-43)

// descending order of the packed value = descending key, then ascending item
__device__ __forceinline__ unsigned long long pack_cand(uint32_t key, uint32_t item) {
  return ((unsigned long long)key << 32) | (unsigned long long)(0xffffffffu - item);
}
__device__ __forceinline__ uint32_t cand_item(unsigned long long c) {
  return 0xffffffffu - (uint32_t)(c & 0xffffffffu);
}

struct SelectSmem {
  RadixSmem<uint32_t> radix;
  uint32_t warp_cnt[RANK_THREADS / 32];
  unsigned long long cand[RANK_MAX_N];
  uint32_t n_atomic;
};
static_assert(MOMENT_SMEM_MAX + sizeof(SelectSmem) <= 227 * 1024,
              "staged moment selection exceeds the sm_90 shared memory per block");

// Top-`n_sel` items of [0, n_items) by key, where src.get(t, key) says whether item t exists and
// gives its key. Leaves smem.cand[0, count) sorted (descending key, ascending item) and returns
// count = min(n_sel, number of existing items). Every thread of the CTA must call it.
template <class Src>
__device__ int block_select_sorted(const Src& src, int n_items, int n_sel, SelectSmem& sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr unsigned kFull = 0xffffffffu;
  uint32_t prefix, need;
  bool take_all;
  // ---- radix select of the n_sel-th largest key (radix_select.cuh)
  block_radix_select<RANK_THREADS, false>(src, n_items, (uint32_t)n_sel, sm.radix, prefix, need,
                                          take_all);
  // ---- gather: keys above the threshold in any order, keys equal to it in item order
  if (tid == 0) sm.n_atomic = 0;
  __syncthreads();
  const uint32_t thr = prefix;
  const uint32_t eq_slot0 = (uint32_t)n_sel - need;   // slots [0, eq_slot0) hold keys > thr
  uint32_t eq_seen = 0;                              // CTA-uniform
  for (int base = 0; base < n_items; base += RANK_THREADS) {
    const int t = base + tid;
    uint32_t k = 0;
    bool eq = false;
    if (t < n_items && src.get(t, k)) {
      if (take_all || k > thr) {
        const uint32_t slot = atomicAdd(&sm.n_atomic, 1u);
        sm.cand[slot] = pack_cand(k, (uint32_t)t);
      } else if (k == thr) {
        eq = true;
      }
    }
    if (take_all || eq_seen >= need) continue;       // CTA-uniform
    const unsigned b = __ballot_sync(kFull, eq);
    if (lane == 0) sm.warp_cnt[warp] = (uint32_t)__popc(b);
    __syncthreads();
    uint32_t before = eq_seen, chunk = 0;
#pragma unroll
    for (int w = 0; w < RANK_THREADS / 32; ++w) {
      const uint32_t cw = sm.warp_cnt[w];
      if (w < warp) before += cw;
      chunk += cw;
    }
    const uint32_t r = before + (uint32_t)__popc(b & ((1u << lane) - 1u));
    if (eq && r < need) sm.cand[eq_slot0 + r] = pack_cand(k, (uint32_t)t);
    __syncthreads();
    eq_seen += chunk;
  }
  __syncthreads();
  const int count = take_all ? (int)sm.n_atomic : n_sel;
  // ---- bitonic sort of the survivors, descending
  int m = 1;
  while (m < count) m <<= 1;
  for (int i = count + tid; i < m; i += RANK_THREADS) sm.cand[i] = 0ull;
  __syncthreads();
  for (int k = 2; k <= m; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < m; i += RANK_THREADS) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = sm.cand[i], b = sm.cand[ixj];
          const bool desc = (i & k) == 0;
          if (desc ? (a < b) : (a > b)) {
            sm.cand[i] = b;
            sm.cand[ixj] = a;
          }
        }
      }
      __syncthreads();
    }
  }
  return count;
}

// ------------------------------------------------------------------ per-row top-K
struct RowSrc {
  const float* row;
  __device__ __forceinline__ bool get(int t, uint32_t& k) const {
    k = ord_key(row[t]);
    return true;
  }
};

__global__ void __launch_bounds__(RANK_THREADS)
rank_topk_kernel(const float* __restrict__ x, long long ld, int n, int k_sel, float alpha,
                 int apply_exp, float* __restrict__ val, int32_t* __restrict__ idx) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ SelectSmem sm;
  const long long r = blockIdx.x;
  const int count = block_select_sorted(RowSrc{x + r * ld}, n, k_sel, sm);
  for (int i = threadIdx.x; i < k_sel; i += RANK_THREADS) {
    if (i < count) {
      const unsigned long long c = sm.cand[i];
      const float v = key_to_float((uint32_t)(c >> 32));
      val[r * k_sel + i] = apply_exp ? expf(alpha * v) : v;
      idx[r * k_sel + i] = (int32_t)cand_item(c);
    } else {
      val[r * k_sel + i] = 0.f;
      idx[r * k_sel + i] = -1;
    }
  }
}

// ------------------------------------------------------------------ span probabilities
// One CTA per (query row, clip) pair: sim[l] = S[row, clip * L + l] / (|inv_row| |inv_frame|)
// (= p . c from the normalised GEMM), both width-K convolutions (zero padded), mask_logits, then a
// softmax over the L frames.
constexpr int SPAN_PROB_THREADS = 128;

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : v + w;
  }
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = red[0];
#pragma unroll
  for (int w = 1; w < SPAN_PROB_THREADS / 32; ++w) t = is_max ? fmaxf(t, red[w]) : t + red[w];
  return t;
}

__global__ void __launch_bounds__(SPAN_PROB_THREADS)
vcmr_span_probs_kernel(const float* __restrict__ S, long long ld_s,
                       const int32_t* __restrict__ pair_row, const int32_t* __restrict__ pair_clip,
                       const float* __restrict__ row_inv, const float* __restrict__ frame_inv,
                       const uint8_t* __restrict__ mask, const float* __restrict__ w_st,
                       const float* __restrict__ w_ed, int nv, int L, int kw,
                       float* __restrict__ st, float* __restrict__ ed) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float s_sim[RANK_MAX_L];
  __shared__ float s_w[2 * RANK_MAX_KW];
  __shared__ float red[2][SPAN_PROB_THREADS / 32];
  const long long b = blockIdx.x;
  const int row = pair_row[b], v = pair_clip[b];
  float* st_out = st + b * L;
  float* ed_out = ed + b * L;
  if (v < 0 || v >= nv) {          // not a clip of the corpus: the pair's output is NaN
    for (int l = threadIdx.x; l < L; l += SPAN_PROB_THREADS) st_out[l] = ed_out[l] = __int_as_float(0x7fc00000);
    return;
  }
  const float sr = fabsf(row_inv[row]);
  const float* srow = S + (long long)row * ld_s + (long long)v * L;
  const float* finv = frame_inv + (long long)v * L;
  for (int l = threadIdx.x; l < L; l += SPAN_PROB_THREADS) s_sim[l] = srow[l] / (sr * fabsf(finv[l]));
  if (threadIdx.x < 2 * kw) s_w[threadIdx.x] = threadIdx.x < kw ? w_st[threadIdx.x] : w_ed[threadIdx.x - kw];
  __syncthreads();
  constexpr int PER = RANK_MAX_L / SPAN_PROB_THREADS;
  float a[PER], e[PER];
  float amax = -INFINITY, emax = -INFINITY;
  const int half = kw / 2;
  const uint8_t* mk = mask + (long long)v * L;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int l = threadIdx.x + i * SPAN_PROB_THREADS;
    a[i] = e[i] = -INFINITY;
    if (l < L) {
      float x = 0.f, y = 0.f;
      for (int k = 0; k < kw; ++k) {
        const int j = l + k - half;
        if (j >= 0 && j < L) {
          x = fmaf(s_w[k], s_sim[j], x);
          y = fmaf(s_w[kw + k], s_sim[j], y);
        }
      }
      const bool on = mk[l] != 0;
      a[i] = on ? x : kRankMaskFill;
      e[i] = on ? y : kRankMaskFill;
      amax = fmaxf(amax, a[i]);
      emax = fmaxf(emax, e[i]);
    }
  }
  amax = block_reduce(amax, true, red[0]);
  emax = block_reduce(emax, true, red[1]);
  float asum = 0.f, esum = 0.f;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    a[i] = expf(a[i] - amax);      // exp(-inf) = 0 past L
    e[i] = expf(e[i] - emax);
    asum += a[i];
    esum += e[i];
  }
  asum = block_reduce(asum, false, red[0]);
  esum = block_reduce(esum, false, red[1]);
  const float ra = 1.f / asum, re = 1.f / esum;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int l = threadIdx.x + i * SPAN_PROB_THREADS;
    if (l < L) {
      st_out[l] = a[i] * ra;
      ed_out[l] = e[i] * re;
    }
  }
}

// ------------------------------------------------------------------ moment top-N
// Item t enumerates the band-valid triples in flat-index order: t = (j * L + s) * W + w with
// e = s + min_l + w, W = the band width clipped to L; items with e >= L do not exist.
struct MomentSrc {
  const float* st;   // [K, L] of this query (shared or global memory)
  const float* ed;
  const float* vf;   // [K] or nullptr (factor 1)
  int L, W, min_l;
  __device__ __forceinline__ void decode(int t, int& j, int& s, int& e) const {
    const int lw = L * W;
    j = t / lw;
    const int r = t - j * lw;
    s = r / W;
    e = s + min_l + (r - s * W);
  }
  __device__ __forceinline__ bool get(int t, uint32_t& k) const {
    int j, s, e;
    decode(t, j, s, e);
    if (e >= L) return false;
    float v = st[j * L + s];
    if (vf != nullptr) v *= vf[j];
    k = ord_key(v * ed[j * L + e]);
    return true;
  }
};

__global__ void __launch_bounds__(RANK_THREADS)
vcmr_moment_topn_kernel(const float* __restrict__ st, const float* __restrict__ ed,
                        const float* __restrict__ vf, int K, int L, int min_l, int W, int n_sel,
                        int stage, float* __restrict__ score, int32_t* __restrict__ jse) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ SelectSmem sm;
  extern __shared__ float dyn[];
  const long long q = blockIdx.x;
  const float* g_st = st + q * K * L;
  const float* g_ed = ed + q * K * L;
  const float* g_vf = vf == nullptr ? nullptr : vf + q * K;
  MomentSrc src{g_st, g_ed, g_vf, L, W, min_l};
  if (stage) {
    float* s_st = dyn;
    float* s_ed = dyn + K * L;
    float* s_vf = dyn + 2 * K * L;
    for (int i = threadIdx.x; i < K * L; i += RANK_THREADS) {
      s_st[i] = g_st[i];
      s_ed[i] = g_ed[i];
    }
    if (g_vf != nullptr)
      for (int i = threadIdx.x; i < K; i += RANK_THREADS) s_vf[i] = g_vf[i];
    __syncthreads();
    src = MomentSrc{s_st, s_ed, g_vf == nullptr ? nullptr : s_vf, L, W, min_l};
  }
  const int n_items = W > 0 ? K * L * W : 0;
  const int count = block_select_sorted(src, n_items, n_sel, sm);
  for (int i = threadIdx.x; i < n_sel; i += RANK_THREADS) {
    const long long o = q * n_sel + i;
    if (i < count) {
      const unsigned long long c = sm.cand[i];
      int j, s, e;
      src.decode((int)cand_item(c), j, s, e);
      score[o] = key_to_float((uint32_t)(c >> 32));
      jse[o * 3 + 0] = j;
      jse[o * 3 + 1] = s;
      jse[o * 3 + 2] = e;
    } else {
      score[o] = 0.f;
      jse[o * 3 + 0] = jse[o * 3 + 1] = jse[o * 3 + 2] = -1;
    }
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_rank_topk(const float* x, int64_t ld, int32_t rows, int32_t n, int32_t k,
                              float alpha, int32_t apply_exp, float* values, int32_t* indices,
                              void* stream) {
  HERO_REQUIRE(x && values && indices, "rank_topk: null pointer");
  HERO_REQUIRE(rows >= 0 && n >= 1 && n <= RANK_MAX_COLS && ld >= n,
               "rank_topk: %d columns (ld %lld) outside [1, %d]", n, (long long)ld, RANK_MAX_COLS);
  HERO_REQUIRE(k >= 1 && k <= RANK_MAX_N && k <= n, "rank_topk: k = %d outside [1, min(%d, %d)]", k,
               RANK_MAX_N, n);
  HERO_REQUIRE(!apply_exp || alpha > 0.f, "rank_topk: exp(alpha * x) needs alpha > 0");
  if (rows == 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(rank_topk_kernel, dim3(rows), dim3(RANK_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream), x, (long long)ld, n, k, alpha,
                             apply_exp, values, indices));
  return HERO_OK;
}

extern "C" int hero_vcmr_span_probs(const float* s, int64_t ld_s, const int32_t* pair_row,
                                    const int32_t* pair_clip, int32_t n_pairs, const float* row_inv,
                                    const float* frame_inv, const uint8_t* mask, const float* w_st,
                                    const float* w_ed, int32_t nv, int32_t len, int32_t kw,
                                    float* st, float* ed, void* stream) {
  HERO_REQUIRE(s && pair_row && pair_clip && row_inv && frame_inv && mask && w_st && w_ed && st && ed,
               "vcmr_span_probs: null pointer");
  HERO_REQUIRE(len >= 1 && len <= RANK_MAX_L && kw >= 1 && kw <= RANK_MAX_KW && (kw & 1) && nv >= 1 &&
                   ld_s >= (int64_t)nv * len,
               "vcmr_span_probs: unsupported shape (len %d, kernel %d, clips %d)", len, kw, nv);
  if (n_pairs <= 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(vcmr_span_probs_kernel, dim3(n_pairs), dim3(SPAN_PROB_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream), s, (long long)ld_s, pair_row,
                             pair_clip, row_inv, frame_inv, mask, w_st, w_ed, nv, len, kw, st, ed));
  return HERO_OK;
}

extern "C" int hero_vcmr_moment_topn(const float* st, const float* ed, const float* video_factor,
                                     int32_t nq, int32_t k, int32_t len, int32_t min_l,
                                     int32_t max_l, int32_t n, float* score, int32_t* jse,
                                     void* stream) {
  HERO_REQUIRE(st && ed && score && jse, "vcmr_moment_topn: null pointer");
  HERO_REQUIRE(k >= 1 && len >= 1 && len <= RANK_MAX_L && (long long)k * len * len < (1ll << 31),
               "vcmr_moment_topn: unsupported shape (k %d, len %d)", k, len);
  HERO_REQUIRE(n >= 1 && n <= RANK_MAX_N, "vcmr_moment_topn: n = %d outside [1, %d]", n, RANK_MAX_N);
  HERO_REQUIRE(min_l >= 0, "vcmr_moment_topn: min_l = %d < 0", min_l);
  if (nq <= 0) return HERO_OK;
  // valid spans: min_l <= e - s < max_l and e < len; W offsets per start after clipping to len
  const int w_hi = max_l < len ? max_l : len;
  const int W = w_hi > min_l ? w_hi - min_l : 0;
  const long long bytes = (2ll * k * len + k) * (long long)sizeof(float);
  const int stage = bytes <= MOMENT_SMEM_MAX ? 1 : 0;
  const size_t smem = stage ? (size_t)bytes : 0;
  // Without the opt-in a launch may request at most 48 KB minus the kernel's static shared memory
  // (SelectSmem). The attribute is per function and outlives this call, so it is set to exactly
  // this launch's size on every staged launch: the result never depends on earlier calls.
  if (stage)
    HERO_CUDA_CHECK(cudaFuncSetAttribute(vcmr_moment_topn_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  HERO_CUDA_CHECK(launch_pdl(vcmr_moment_topn_kernel, dim3(nq), dim3(RANK_THREADS), smem,
                             reinterpret_cast<cudaStream_t>(stream), st, ed, video_factor, k, len,
                             min_l, W, n, stage, score, jse));
  return HERO_OK;
}

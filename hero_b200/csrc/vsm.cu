// Video-subtitle-matching / moment-retrieval head kernels (SURVEY.md §8f rank 1): the small ops
// that follow the encoder in HeroForPretraining / HeroForVcmr (model/pretrain.py:128-166,364-413 of
// the reference), fused so the head is a handful of launches with no host round trip:
//
//   video-level scores   q^ = q / max(|q|, eps), c^ = c / max(|c|, eps)        (l2norm_split)
//                        S[m, (n, l)] = q^_m . c^_{n,l}                          (wgmma GEMM, split-bf16)
//                        score[m, n] = max_l mask_logits(S[m, n, l], mask[n, l]) (masked_max)
//   span logits          sim[b, l] = query_b . ctx_{b,l};  st / ed = conv1d_k(sim) masked
//
// and their backward passes. Everything here is HBM / latency bound and tiny next to the encoder
// (32 .. 256 queries x clips x 100 frames); the point is launch count and the absence of syncs.
#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr float kMaskFill = -1e4f;   // mask_logits (model/modeling_utils.py:42-43)

// ------------------------------------------------------------------ row L2 normalisation
// One warp per row: x^ = x / max(|x|_2, eps) (F.normalize), written as split-bf16 halves (the GEMM
// operands) and optionally as fp32; inv[r] = 1 / max(|x|, eps), negated when the clamp was active
// (the backward then has no projection term).
__global__ void __launch_bounds__(256)
l2norm_split_kernel(const float* __restrict__ x, long long rows, int d, float eps,
                    __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                    float* __restrict__ inv) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* p = x + r * d;
  float ss = 0.f;
  for (int c = lane * 4; c < d; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(p + c);
    ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  ss = warp_sum(ss);
  const float nrm = sqrtf(ss);
  const bool clamped = nrm < eps;
  const float s = 1.0f / fmaxf(nrm, eps);
  if (lane == 0) inv[r] = clamped ? -s : s;
  for (int c = lane * 4; c < d; c += 128) {
    const float4 v = *reinterpret_cast<const float4*>(p + c);
    const float o[4] = {v.x * s, v.y * s, v.z * s, v.w * s};
    uint32_t h[2], l[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      h[j] = pack_bf16x2(o[2 * j], o[2 * j + 1]);
      const float2 back = unpack_bf16x2(h[j]);
      l[j] = pack_bf16x2(o[2 * j] - back.x, o[2 * j + 1] - back.y);
    }
    *reinterpret_cast<uint2*>(hi + r * d + c) = make_uint2(h[0], h[1]);
    *reinterpret_cast<uint2*>(lo + r * d + c) = make_uint2(l[0], l[1]);
  }
}

// ------------------------------------------------------------------ masked max over frames
// S: [nq, ld_s] fp32 with S[m, n * L + l]; one warp per (m, n).
__global__ void __launch_bounds__(256)
vsm_masked_max_kernel(const float* __restrict__ S, long long ld_s, const uint8_t* __restrict__ mask,
                      int nq, int nv, int L, float* __restrict__ scores,
                      int32_t* __restrict__ argmax) {
  pdl_wait();
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const long long w = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= (long long)nq * nv) return;
  const int m = (int)(w / nv), n = (int)(w % nv);
  const float* row = S + (long long)m * ld_s + (long long)n * L;
  const uint8_t* mk = mask + (long long)n * L;
  float best = -INFINITY;
  int arg = 0x7fffffff;
  for (int l = lane; l < L; l += 32) {
    const float v = mk[l] ? row[l] : kMaskFill;
    if (v > best) { best = v; arg = l; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  if (lane == 0) {
    scores[w] = best;
    argmax[w] = arg;
  }
}

__device__ __forceinline__ float bf16_pair_sum(const __nv_bfloat16* hi, const __nv_bfloat16* lo,
                                               long long i) {
  return __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}

// Backward of the normalisation given dx^ (acc): dx = (acc - x^ (x^ . acc)) * inv  (no projection
// when the norm was clamped). 256 threads cooperate on one row held as acc[] in registers.
template <int PER>
__device__ __forceinline__ void normalize_bwd_row(const float (&acc)[PER], const float (&xh)[PER],
                                                  float inv, float* out, int d, float* red) {
  float dot = 0.f;
#pragma unroll
  for (int j = 0; j < PER; ++j) dot += acc[j] * xh[j];
  dot = warp_sum(dot);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[warp] = dot;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[w];
  const bool clamped = inv < 0.f;
  const float s = fabsf(inv);
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int c = threadIdx.x + j * 256;
    if (c < d) out[c] = (clamped ? acc[j] : (acc[j] - xh[j] * tot)) * s;
  }
}

constexpr int VSM_PER = 4;   // feature columns per thread: d <= 1024

// dq[m] = normalize_bwd( sum_n g[m, n] * mask * c^[n, argmax[m, n]] ): one CTA per query.
__global__ void __launch_bounds__(256)
vsm_scores_bwd_q_kernel(const float* __restrict__ g, const int32_t* __restrict__ argmax,
                        const uint8_t* __restrict__ mask, const __nv_bfloat16* __restrict__ c_hi,
                        const __nv_bfloat16* __restrict__ c_lo, const __nv_bfloat16* __restrict__ q_hi,
                        const __nv_bfloat16* __restrict__ q_lo, const float* __restrict__ q_inv,
                        int nv, int L, int d, float* __restrict__ dq) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[8];
  const int m = blockIdx.x;
  float acc[VSM_PER], xh[VSM_PER];
#pragma unroll
  for (int j = 0; j < VSM_PER; ++j) {
    const int c = threadIdx.x + j * 256;
    acc[j] = 0.f;
    xh[j] = c < d ? bf16_pair_sum(q_hi, q_lo, (long long)m * d + c) : 0.f;
  }
  for (int n = 0; n < nv; ++n) {
    const int l = argmax[(long long)m * nv + n];
    if (l < 0 || l >= L || !mask[(long long)n * L + l]) continue;   // CTA-uniform
    const float gv = g[(long long)m * nv + n];
    const long long row = ((long long)n * L + l) * d;
#pragma unroll
    for (int j = 0; j < VSM_PER; ++j) {
      const int c = threadIdx.x + j * 256;
      if (c < d) acc[j] = fmaf(gv, bf16_pair_sum(c_hi, c_lo, row + c), acc[j]);
    }
  }
  normalize_bwd_row<VSM_PER>(acc, xh, q_inv[m], dq + (long long)m * d, d, red);
}

// dctx[n, l] = normalize_bwd( sum_{m: argmax[m, n] == l} g[m, n] * q^[m] ): one CTA per frame.
__global__ void __launch_bounds__(256)
vsm_scores_bwd_ctx_kernel(const float* __restrict__ g, const int32_t* __restrict__ argmax,
                          const uint8_t* __restrict__ mask, const __nv_bfloat16* __restrict__ c_hi,
                          const __nv_bfloat16* __restrict__ c_lo,
                          const __nv_bfloat16* __restrict__ q_hi,
                          const __nv_bfloat16* __restrict__ q_lo, const float* __restrict__ c_inv,
                          int nq, int nv, int L, int d, float* __restrict__ dctx) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[8];
  const int n = blockIdx.x / L, l = blockIdx.x % L;
  const long long row = (long long)n * L + l;
  float acc[VSM_PER], xh[VSM_PER];
#pragma unroll
  for (int j = 0; j < VSM_PER; ++j) acc[j] = xh[j] = 0.f;
  if (!mask[row]) {     // masked frames never carry gradient (mask_logits multiplies by 0)
#pragma unroll
    for (int j = 0; j < VSM_PER; ++j) {
      const int c = threadIdx.x + j * 256;
      if (c < d) dctx[row * d + c] = 0.f;
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < VSM_PER; ++j) {
    const int c = threadIdx.x + j * 256;
    if (c < d) xh[j] = bf16_pair_sum(c_hi, c_lo, row * d + c);
  }
  for (int m = 0; m < nq; ++m) {
    if (argmax[(long long)m * nv + n] != l) continue;               // CTA-uniform
    const float gv = g[(long long)m * nv + n];
#pragma unroll
    for (int j = 0; j < VSM_PER; ++j) {
      const int c = threadIdx.x + j * 256;
      if (c < d) acc[j] = fmaf(gv, bf16_pair_sum(q_hi, q_lo, (long long)m * d + c), acc[j]);
    }
  }
  normalize_bwd_row<VSM_PER>(acc, xh, c_inv[row], dctx + row * d, d, red);
}

// ------------------------------------------------------------------ span logits
// One CTA per (query, clip) pair b: sim[l] = query_b . ctx_{b,l} (a warp per frame), then the two
// width-K convolutions (zero padded, no bias, model/pretrain.py:48-60) and mask_logits.
constexpr int SPAN_MAX_L = 512;
constexpr int SPAN_MAX_K = 15;

__global__ void __launch_bounds__(256)
vsm_span_fwd_kernel(const float* __restrict__ query, const float* __restrict__ ctx,
                    const uint8_t* __restrict__ mask, const float* __restrict__ w_st,
                    const float* __restrict__ w_ed, int L, int d, int K, float* __restrict__ sim,
                    float* __restrict__ st, float* __restrict__ ed) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float s_sim[SPAN_MAX_L];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* q = query + (long long)b * d;
  for (int l = warp; l < L; l += 8) {
    const float* c = ctx + ((long long)b * L + l) * d;
    float acc = 0.f;
    for (int k = lane * 4; k < d; k += 128) {
      const float4 a = *reinterpret_cast<const float4*>(q + k);
      const float4 v = *reinterpret_cast<const float4*>(c + k);
      acc += a.x * v.x + a.y * v.y + a.z * v.z + a.w * v.w;
    }
    acc = warp_sum(acc);
    if (lane == 0) s_sim[l] = acc;
  }
  __syncthreads();
  const int half = K / 2;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    float a = 0.f, e = 0.f;
    for (int k = 0; k < K; ++k) {
      const int j = l + k - half;
      if (j >= 0 && j < L) {
        a = fmaf(w_st[k], s_sim[j], a);
        e = fmaf(w_ed[k], s_sim[j], e);
      }
    }
    const bool on = mask[(long long)b * L + l] != 0;
    sim[(long long)b * L + l] = s_sim[l];
    st[(long long)b * L + l] = on ? a : kMaskFill;
    ed[(long long)b * L + l] = on ? e : kMaskFill;
  }
}

__global__ void __launch_bounds__(256)
vsm_span_bwd_kernel(const float* __restrict__ dst, const float* __restrict__ ded,
                    const uint8_t* __restrict__ mask, const float* __restrict__ w_st,
                    const float* __restrict__ w_ed, const float* __restrict__ sim,
                    const float* __restrict__ query, const float* __restrict__ ctx, int L, int d,
                    int K, float* __restrict__ dquery, float* __restrict__ dctx,
                    float* __restrict__ dw_st, float* __restrict__ dw_ed) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float s_a[SPAN_MAX_L], s_e[SPAN_MAX_L], s_sim[SPAN_MAX_L], s_ds[SPAN_MAX_L];
  __shared__ float s_dw[2 * SPAN_MAX_K];
  const int b = blockIdx.x;
  const int half = K / 2;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    const bool on = mask[(long long)b * L + l] != 0;
    s_a[l] = on ? dst[(long long)b * L + l] : 0.f;     // gradient through mask_logits
    s_e[l] = on ? ded[(long long)b * L + l] : 0.f;
    s_sim[l] = sim[(long long)b * L + l];
  }
  if (threadIdx.x < 2 * SPAN_MAX_K) s_dw[threadIdx.x] = 0.f;
  __syncthreads();
  // dsim[j] = sum_k w[k] * dout[j - k + half];   dw[k] = sum_l dout[l] * sim[l + k - half]
  for (int j = threadIdx.x; j < L; j += blockDim.x) {
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
      const int l = j - k + half;
      if (l >= 0 && l < L) acc += w_st[k] * s_a[l] + w_ed[k] * s_e[l];
    }
    s_ds[j] = acc;
  }
  if (threadIdx.x < 2 * K) {
    const int k = threadIdx.x % K;
    const float* dout = threadIdx.x < K ? s_a : s_e;
    float acc = 0.f;
    for (int l = 0; l < L; ++l) {
      const int j = l + k - half;
      if (j >= 0 && j < L) acc += dout[l] * s_sim[j];
    }
    atomicAdd((threadIdx.x < K ? dw_st : dw_ed) + k, acc);
  }
  __syncthreads();
  const float* q = query + (long long)b * d;
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const float qc = q[c];
    float dq = 0.f;
    for (int l = 0; l < L; ++l) {
      const float ds = s_ds[l];
      const long long i = ((long long)b * L + l) * d + c;
      dq = fmaf(ds, ctx[i], dq);
      dctx[i] = ds * qc;
    }
    dquery[(long long)b * d + c] = dq;
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_l2norm_split_f32(const float* x, int64_t rows, int32_t d, float eps, void* hi,
                                     void* lo, float* inv_norm, void* stream) {
  HERO_REQUIRE(x && hi && lo && inv_norm && d > 0 && d % 4 == 0, "l2norm_split: bad args");
  if (rows <= 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(l2norm_split_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0,
                             reinterpret_cast<cudaStream_t>(stream), x, (long long)rows, d, eps,
                             reinterpret_cast<__nv_bfloat16*>(hi),
                             reinterpret_cast<__nv_bfloat16*>(lo), inv_norm));
  return HERO_OK;
}

extern "C" int hero_vsm_masked_max(const float* s, int64_t ld_s, const uint8_t* mask, int32_t nq,
                                   int32_t nv, int32_t len, float* scores, int32_t* argmax,
                                   void* stream) {
  HERO_REQUIRE(s && mask && scores && argmax && nq >= 0 && nv >= 0 && len > 0, "vsm_masked_max: bad args");
  const long long n = (long long)nq * nv;
  if (n == 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(vsm_masked_max_kernel, dim3((unsigned)((n + 7) / 8)), dim3(256), 0,
                             reinterpret_cast<cudaStream_t>(stream), s, (long long)ld_s, mask, nq,
                             nv, len, scores, argmax));
  return HERO_OK;
}

extern "C" int hero_vsm_scores_bwd(const float* g, const int32_t* argmax, const uint8_t* mask,
                                   const void* q_hi, const void* q_lo, const float* q_inv,
                                   const void* c_hi, const void* c_lo, const float* c_inv,
                                   int32_t nq, int32_t nv, int32_t len, int32_t d, float* dq,
                                   float* dctx, void* stream) {
  HERO_REQUIRE(g && argmax && mask && q_hi && q_lo && q_inv && c_hi && c_lo && c_inv,
               "vsm_scores_bwd: null pointer");
  HERO_REQUIRE(d > 0 && d <= 256 * VSM_PER, "vsm_scores_bwd: feature dim %d > %d", d, 256 * VSM_PER);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  auto bf = [](const void* p) { return reinterpret_cast<const __nv_bfloat16*>(p); };
  if (dq != nullptr && nq > 0)
    HERO_CUDA_CHECK(launch_pdl(vsm_scores_bwd_q_kernel, dim3(nq), dim3(256), 0, st, g, argmax, mask,
                               bf(c_hi), bf(c_lo), bf(q_hi), bf(q_lo), q_inv, nv, len, d, dq));
  if (dctx != nullptr && nv > 0)
    HERO_CUDA_CHECK(launch_pdl(vsm_scores_bwd_ctx_kernel, dim3((unsigned)((long long)nv * len)),
                               dim3(256), 0, st, g, argmax, mask, bf(c_hi), bf(c_lo), bf(q_hi),
                               bf(q_lo), c_inv, nq, nv, len, d, dctx));
  return HERO_OK;
}

extern "C" int hero_vsm_span_fwd(const float* query, const float* ctx, const uint8_t* mask,
                                 const float* w_st, const float* w_ed, int32_t n, int32_t len,
                                 int32_t d, int32_t k, float* sim, float* st, float* ed,
                                 void* stream) {
  HERO_REQUIRE(query && ctx && mask && w_st && w_ed && sim && st && ed, "vsm_span_fwd: null pointer");
  HERO_REQUIRE(len > 0 && len <= SPAN_MAX_L && d % 4 == 0 && k >= 1 && k <= SPAN_MAX_K && (k & 1),
               "vsm_span_fwd: unsupported shape (len %d, d %d, kernel %d)", len, d, k);
  if (n <= 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(vsm_span_fwd_kernel, dim3(n), dim3(256), 0,
                             reinterpret_cast<cudaStream_t>(stream), query, ctx, mask, w_st, w_ed,
                             len, d, k, sim, st, ed));
  return HERO_OK;
}

extern "C" int hero_vsm_span_bwd(const float* dst, const float* ded, const uint8_t* mask,
                                 const float* w_st, const float* w_ed, const float* sim,
                                 const float* query, const float* ctx, int32_t n, int32_t len,
                                 int32_t d, int32_t k, float* dquery, float* dctx, float* dw_st,
                                 float* dw_ed, void* stream) {
  HERO_REQUIRE(dst && ded && mask && w_st && w_ed && sim && query && ctx && dquery && dctx && dw_st &&
                   dw_ed,
               "vsm_span_bwd: null pointer");
  HERO_REQUIRE(len > 0 && len <= SPAN_MAX_L && k >= 1 && k <= SPAN_MAX_K && (k & 1),
               "vsm_span_bwd: unsupported shape (len %d, kernel %d)", len, k);
  if (n <= 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(vsm_span_bwd_kernel, dim3(n), dim3(256), 0,
                             reinterpret_cast<cudaStream_t>(stream), dst, ded, mask, w_st, w_ed, sim,
                             query, ctx, len, d, k, dquery, dctx, dw_st, dw_ed));
  return HERO_OK;
}

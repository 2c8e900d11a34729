// Video QA attention pooling (model/videoQA.py:36-59,90-95): the two learned poolings of the
// temporal transformer's frame outputs, which the reference computes as einsums over a padded
// (Nv, Nq, L, H) tensor.
//
//   a[v,q,l] = softmax_l(mask_logits(w_qa . h[v,q,l], m[v,q,l]))      qa_pooled[v,q] = sum_l a h
//   b[v,q,l] = softmax_q(mask_logits(w_st . h[v,q,l], m[v,q,l]))      st_pooled[v,l] = sum_q b h
//
// h[v,q,l] is row map[(v*Nq+q)*L+l] of the packed fp32 frame outputs, or zeros where map < 0
// (padded frames are never computed in the packed layout). mask_logits(x, m) = x*m + (1-m)*(-1e4)
// is evaluated with every operation rounded in fp32, as torch does. Everything is fp32 with fixed
// reduction orders, so forward and backward are deterministic (no atomics).
#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int QA_MAX_NQ = 16;
constexpr int QA_MAX_L = 512;
constexpr int QA_THREADS = 256;
constexpr int QA_WARPS = QA_THREADS / 32;
constexpr int QA_CHUNK_ROWS = 64;    // rows per partial sum of the weight gradients

__device__ __forceinline__ float qa_mask_logits(float x, float m) {
  return __fadd_rn(__fmul_rn(x, m), __fmul_rn(__fsub_rn(1.f, m), -1e4f));
}

// Block-wide sum / max in a fixed order; `red` holds QA_WARPS floats. Every thread gets the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = lane < QA_WARPS ? red[lane] : 0.f;
  return warp_sum(t);
}

__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = lane < QA_WARPS ? red[lane] : -INFINITY;
  return warp_max(t);
}

// Two dot products of one H-row with two H-vectors, one warp, float4 loads, fixed order.
__device__ __forceinline__ void warp_dot2(const float* __restrict__ row, const float* __restrict__ u,
                                          const float* __restrict__ w, int H, float& du,
                                          float& dw) {
  float su = 0.f, sw = 0.f;
  const int lane = threadIdx.x & 31;
  for (int c = lane * 4; c < H; c += 128) {
    const float4 x = *reinterpret_cast<const float4*>(row + c);
    const float4 a = *reinterpret_cast<const float4*>(u + c);
    const float4 b = *reinterpret_cast<const float4*>(w + c);
    su += x.x * a.x + x.y * a.y + x.z * a.z + x.w * a.w;
    sw += x.x * b.x + x.y * b.y + x.z * b.z + x.w * b.w;
  }
  du = warp_sum(su);
  dw = warp_sum(sw);
}

// ---- forward ------------------------------------------------------------------------------------
// One warp per (v,q,l) row: masked logits of both poolings into la / lb.
__global__ void __launch_bounds__(QA_THREADS)
qa_logits_kernel(const float* __restrict__ h, const int32_t* __restrict__ map,
                 const float* __restrict__ mask, const float* __restrict__ w_qa,
                 const float* __restrict__ w_st, int R, int H, float* __restrict__ la,
                 float* __restrict__ lb) {
  pdl_wait();
  pdl_launch_dependents();
  const int row = blockIdx.x * QA_WARPS + (threadIdx.x >> 5);
  if (row >= R) return;
  const int src = map[row];
  float sa = 0.f, sb = 0.f;
  if (src >= 0) warp_dot2(h + (long long)src * H, w_qa, w_st, H, sa, sb);
  if ((threadIdx.x & 31) == 0) {
    const float m = mask[row];
    la[row] = qa_mask_logits(sa, m);
    lb[row] = qa_mask_logits(sb, m);
  }
}

// Blocks [0, Nv*Nq): softmax over l of one (v,q) and its qa-pooled row. Blocks [Nv*Nq, Nv*Nq +
// Nv*L): softmax over q of one (v,l) and its st/ed-pooled row. la / lb are overwritten in place
// with the probabilities (each element belongs to exactly one block).
__global__ void __launch_bounds__(QA_THREADS)
qa_pool_kernel(const float* __restrict__ h, const int32_t* __restrict__ map, int Nv, int Nq,
               int L, int H, float* __restrict__ pa, float* __restrict__ pb,
               float* __restrict__ qa_out, float* __restrict__ st_out) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float p[QA_MAX_L];
  __shared__ int32_t src[QA_MAX_L];
  __shared__ float red[QA_WARPS];
  const int tid = threadIdx.x;
  const int nvq = Nv * Nq;
  int n;
  float* out;
  if ((int)blockIdx.x < nvq) {
    const int vq = blockIdx.x;
    float* lg = pa + (long long)vq * L;
    float mx = -INFINITY;
    for (int l = tid; l < L; l += QA_THREADS) {
      p[l] = lg[l];
      src[l] = map[(long long)vq * L + l];
      mx = fmaxf(mx, p[l]);
    }
    mx = block_max(mx, red);
    float s = 0.f;
    for (int l = tid; l < L; l += QA_THREADS) {
      p[l] = expf(p[l] - mx);
      s += p[l];
    }
    s = block_sum(s, red);
    for (int l = tid; l < L; l += QA_THREADS) {
      p[l] = p[l] / s;
      lg[l] = p[l];
    }
    n = L;
    out = qa_out + (long long)vq * H;
  } else {
    const int vl = blockIdx.x - nvq;
    const int v = vl / L, l = vl % L;
    if (tid < Nq) {
      const long long r = ((long long)v * Nq + tid) * L + l;
      p[tid] = pb[r];
      src[tid] = map[r];
    }
    __syncthreads();
    float mx = -INFINITY;
    for (int q = 0; q < Nq; ++q) mx = fmaxf(mx, p[q]);
    float s = 0.f;
    for (int q = 0; q < Nq; ++q) s += expf(p[q] - mx);
    __syncthreads();
    if (tid < Nq) {
      const float e = expf(p[tid] - mx) / s;
      p[tid] = e;
      pb[((long long)v * Nq + tid) * L + l] = e;
    }
    n = Nq;
    out = st_out + (long long)vl * H;
  }
  __syncthreads();
  for (int c = tid * 4; c < H; c += QA_THREADS * 4) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = 0; i < n; ++i) {
      if (src[i] < 0) continue;
      const float w = p[i];
      const float4 x = *reinterpret_cast<const float4*>(h + (long long)src[i] * H + c);
      acc.x += w * x.x;
      acc.y += w * x.y;
      acc.z += w * x.z;
      acc.w += w * x.w;
    }
    *reinterpret_cast<float4*>(out + c) = acc;
  }
}

// ---- backward -----------------------------------------------------------------------------------
// One warp per row: da = d qa_pooled[v,q] . h, db = d st_pooled[v,l] . h.
__global__ void __launch_bounds__(QA_THREADS)
qa_bwd_dots_kernel(const float* __restrict__ h, const int32_t* __restrict__ map,
                   const float* __restrict__ dqa, const float* __restrict__ dst, int Nq, int L,
                   int R, int H, float* __restrict__ da, float* __restrict__ db) {
  pdl_wait();
  pdl_launch_dependents();
  const int row = blockIdx.x * QA_WARPS + (threadIdx.x >> 5);
  if (row >= R) return;
  const int src = map[row];
  const int vq = row / L, l = row % L, v = vq / Nq;
  float sa = 0.f, sb = 0.f;
  if (src >= 0)
    warp_dot2(h + (long long)src * H, dqa + (long long)vq * H, dst + ((long long)v * L + l) * H,
              H, sa, sb);
  if ((threadIdx.x & 31) == 0) {
    da[row] = sa;
    db[row] = sb;
  }
}

// One block per (v,q): softmax backward of both poolings (d logit, times the mask_logits slope
// m) into gqa / gst, and d h of its frame rows.
__global__ void __launch_bounds__(QA_THREADS, 1)
qa_bwd_rows_kernel(const int32_t* __restrict__ map, const float* __restrict__ mask,
                   const float* __restrict__ pa, const float* __restrict__ pb,
                   const float* __restrict__ da, const float* __restrict__ db,
                   const float* __restrict__ dqa, const float* __restrict__ dst,
                   const float* __restrict__ w_qa, const float* __restrict__ w_st, int Nq, int L,
                   int H, float* __restrict__ gqa, float* __restrict__ gst, float* __restrict__ dh) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[QA_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int vq = blockIdx.x, v = vq / Nq;
  const long long r0 = (long long)vq * L;
  float s = 0.f;
  for (int l = tid; l < L; l += QA_THREADS) s += pa[r0 + l] * da[r0 + l];
  s = block_sum(s, red);
  for (int l = warp; l < L; l += QA_WARPS) {
    const long long row = r0 + l;
    const float m = mask[row];
    const float a = pa[row], b = pb[row];
    const float ga = a * (da[row] - s) * m;
    float t = 0.f;                          // sum_q' b db over the candidates of (v, l)
    const float* pbl = pb + (long long)v * Nq * L + l;
    const float* dbl = db + (long long)v * Nq * L + l;
#pragma unroll 1
    for (int q = 0; q < Nq; ++q) t += pbl[q * L] * dbl[q * L];
    const float gb = b * (db[row] - t) * m;
    if (lane == 0) {
      gqa[row] = ga;
      gst[row] = gb;
    }
    const int src = map[row];
    if (src < 0) continue;
    const float* dq = dqa + (long long)vq * H;
    const float* ds = dst + ((long long)v * L + l) * H;
    float* out = dh + (long long)src * H;
    for (int c = lane * 4; c < H; c += 128) {
      const float4 x = *reinterpret_cast<const float4*>(dq + c);
      const float4 y = *reinterpret_cast<const float4*>(ds + c);
      const float4 u = *reinterpret_cast<const float4*>(w_qa + c);
      const float4 w = *reinterpret_cast<const float4*>(w_st + c);
      float4 o;
      o.x = a * x.x + ga * u.x + b * y.x + gb * w.x;
      o.y = a * x.y + ga * u.y + b * y.y + gb * w.y;
      o.z = a * x.z + ga * u.z + b * y.z + gb * w.z;
      o.w = a * x.w + ga * u.w + b * y.w + gb * w.w;
      *reinterpret_cast<float4*>(out + c) = o;
    }
  }
}

// Partial weight gradients over QA_CHUNK_ROWS rows: part[chunk][0|1][c] = sum_rows g * h[row][c].
__global__ void __launch_bounds__(QA_THREADS)
qa_bwd_wpart_kernel(const float* __restrict__ h, const int32_t* __restrict__ map,
                    const float* __restrict__ gqa, const float* __restrict__ gst, int R, int H,
                    float* __restrict__ part) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float sg[2][QA_CHUNK_ROWS];
  __shared__ int32_t ssrc[QA_CHUNK_ROWS];
  const int tid = threadIdx.x;
  const int r0 = blockIdx.x * QA_CHUNK_ROWS;
  const int nr = min(QA_CHUNK_ROWS, R - r0);
  if (tid < nr) {
    sg[0][tid] = gqa[r0 + tid];
    sg[1][tid] = gst[r0 + tid];
    ssrc[tid] = map[r0 + tid];
  }
  __syncthreads();
  float* p0 = part + (long long)blockIdx.x * 2 * H;
  for (int c = tid; c < H; c += QA_THREADS) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < nr; ++i) {
      if (ssrc[i] < 0) continue;
      const float x = h[(long long)ssrc[i] * H + c];
      a += sg[0][i] * x;
      b += sg[1][i] * x;
    }
    p0[c] = a;
    p0[H + c] = b;
  }
}

// dw_qa[c] += sum over chunks (in order) of part[chunk][0][c]; dw_st likewise.
__global__ void __launch_bounds__(QA_THREADS)
qa_bwd_wsum_kernel(const float* __restrict__ part, int n_chunks, int H, float* __restrict__ dw_qa,
                   float* __restrict__ dw_st) {
  pdl_wait();
  pdl_launch_dependents();
  const int c = blockIdx.x * QA_THREADS + threadIdx.x;
  if (c >= 2 * H) return;
  float s = 0.f;
  for (int k = 0; k < n_chunks; ++k) s += part[(long long)k * 2 * H + c];
  if (c < H)
    dw_qa[c] += s;
  else
    dw_st[c - H] += s;
}

static bool qa_aligned(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

static int qa_check(const void* h, int Nv, int Nq, int L, int H) {
  HERO_REQUIRE(Nv >= 1, "qa_pool: Nv = %d < 1", Nv);
  HERO_REQUIRE(Nq >= 1 && Nq <= QA_MAX_NQ, "qa_pool: Nq = %d outside [1, %d]", Nq, QA_MAX_NQ);
  HERO_REQUIRE(L >= 1 && L <= QA_MAX_L, "qa_pool: L = %d outside [1, %d]", L, QA_MAX_L);
  HERO_REQUIRE(H >= 8 && H % 8 == 0, "qa_pool: H = %d is not a positive multiple of 8", H);
  HERO_REQUIRE((long long)Nv * Nq * L < (1LL << 31), "qa_pool: too many rows");
  return HERO_OK;
}

}  // namespace hero

using namespace hero;

extern "C" int hero_qa_pool_fwd(const float* h, const int32_t* map, const float* mask,
                                const float* w_qa, const float* w_st, int32_t Nv, int32_t Nq,
                                int32_t L, int32_t H, float* a, float* b, float* qa_pooled,
                                float* st_pooled, void* stream) {
  HERO_REQUIRE(h && map && mask && w_qa && w_st && a && b && qa_pooled && st_pooled,
               "qa_pool_fwd: null pointer");
  int st = qa_check(h, Nv, Nq, L, H);
  if (st != HERO_OK) return st;
  HERO_REQUIRE(qa_aligned(h) && qa_aligned(w_qa) && qa_aligned(w_st) && qa_aligned(qa_pooled) &&
                   qa_aligned(st_pooled),
               "qa_pool_fwd: h, w_qa, w_st and the pooled outputs must be 16-byte aligned");
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int R = Nv * Nq * L;
  HERO_CUDA_CHECK(launch_pdl(qa_logits_kernel, dim3(ceil_div(R, QA_WARPS)), dim3(QA_THREADS), 0, s,
                             h, map, mask, w_qa, w_st, R, (int)H, a, b));
  HERO_CUDA_CHECK(launch_pdl(qa_pool_kernel, dim3(Nv * Nq + Nv * L), dim3(QA_THREADS), 0, s, h, map,
                             (int)Nv, (int)Nq, (int)L, (int)H, a, b, qa_pooled, st_pooled));
  return HERO_OK;
}

extern "C" int64_t hero_qa_pool_bwd_scratch_floats(int32_t Nv, int32_t Nq, int32_t L, int32_t H) {
  const long long R = (long long)Nv * Nq * L;
  return 4 * R + 2LL * H * ((R + QA_CHUNK_ROWS - 1) / QA_CHUNK_ROWS);
}

extern "C" int hero_qa_pool_bwd(const float* h, const int32_t* map, const float* mask,
                                const float* w_qa, const float* w_st, const float* a,
                                const float* b, const float* d_qa_pooled,
                                const float* d_st_pooled, int32_t Nv, int32_t Nq, int32_t L,
                                int32_t H, float* scratch, float* dh, float* dw_qa, float* dw_st,
                                void* stream) {
  HERO_REQUIRE(h && map && mask && w_qa && w_st && a && b && d_qa_pooled && d_st_pooled &&
                   scratch && dh && dw_qa && dw_st,
               "qa_pool_bwd: null pointer");
  int st = qa_check(h, Nv, Nq, L, H);
  if (st != HERO_OK) return st;
  HERO_REQUIRE(qa_aligned(h) && qa_aligned(w_qa) && qa_aligned(w_st) && qa_aligned(d_qa_pooled) &&
                   qa_aligned(d_st_pooled) && qa_aligned(dh),
               "qa_pool_bwd: h, w_qa, w_st, the pooled gradients and dh must be 16-byte aligned");
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int R = Nv * Nq * L;
  const int n_chunks = ceil_div(R, QA_CHUNK_ROWS);
  float* da = scratch;
  float* db = da + R;
  float* gqa = db + R;
  float* gst = gqa + R;
  float* part = gst + R;
  HERO_CUDA_CHECK(launch_pdl(qa_bwd_dots_kernel, dim3(ceil_div(R, QA_WARPS)), dim3(QA_THREADS), 0,
                             s, h, map, d_qa_pooled, d_st_pooled, (int)Nq, (int)L, R, (int)H, da,
                             db));
  HERO_CUDA_CHECK(launch_pdl(qa_bwd_rows_kernel, dim3(Nv * Nq), dim3(QA_THREADS), 0, s, map, mask,
                             a, b, (const float*)da, (const float*)db, d_qa_pooled, d_st_pooled,
                             w_qa, w_st, (int)Nq, (int)L, (int)H, gqa, gst, dh));
  HERO_CUDA_CHECK(launch_pdl(qa_bwd_wpart_kernel, dim3(n_chunks), dim3(QA_THREADS), 0, s, h, map,
                             (const float*)gqa, (const float*)gst, R, (int)H, part));
  HERO_CUDA_CHECK(launch_pdl(qa_bwd_wsum_kernel, dim3(ceil_div(2 * H, QA_THREADS)),
                             dim3(QA_THREADS), 0, s, (const float*)part, n_chunks, (int)H, dw_qa,
                             dw_st));
  return HERO_OK;
}

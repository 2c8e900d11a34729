// Flat-buffer fused AdamW and sum-of-squares (global-norm clipping), HBM-bound.
// Arithmetic follows the reference's optim/adamw.py:80-104: bias-corrected step size computed on
// the host, eps added to sqrt(v) (not inside), decoupled weight decay applied AFTER the Adam
// update on the already-updated parameter with the un-corrected lr.
#include "common.h"
#include "ptx.cuh"

namespace hero {

// The AdamW update of the four consecutive elements [4i, 4i + 4): 16-byte vector accesses on all
// seven streams (p, g, m, v read; p, m, v + bf16 written: 30 B per parameter). Shared by the
// single-range and the segment-table kernels, so both compute bitwise the same values.
__device__ __forceinline__ void adamw_vec4(float* __restrict__ p, const float* __restrict__ g,
                                           float* __restrict__ m, float* __restrict__ v,
                                           __nv_bfloat16* __restrict__ p_bf16, long long i,
                                           float step_size, float beta1, float beta2, float ob1,
                                           float ob2, float eps, float lr_wd, float grad_scale) {
  const float4 g4 = __ldg(reinterpret_cast<const float4*>(g) + i);
  float4 m4 = reinterpret_cast<float4*>(m)[i];
  float4 v4 = reinterpret_cast<float4*>(v)[i];
  float4 p4 = reinterpret_cast<float4*>(p)[i];
  const float gr[4] = {g4.x * grad_scale, g4.y * grad_scale, g4.z * grad_scale, g4.w * grad_scale};
  float mm[4] = {m4.x, m4.y, m4.z, m4.w}, vv[4] = {v4.x, v4.y, v4.z, v4.w};
  float pp[4] = {p4.x, p4.y, p4.z, p4.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    mm[j] = beta1 * mm[j] + ob1 * gr[j];
    vv[j] = beta2 * vv[j] + ob2 * gr[j] * gr[j];
    pp[j] = pp[j] - step_size * (mm[j] / (sqrtf(vv[j]) + eps));
    if (lr_wd > 0.0f) pp[j] = pp[j] - lr_wd * pp[j];
  }
  reinterpret_cast<float4*>(m)[i] = make_float4(mm[0], mm[1], mm[2], mm[3]);
  reinterpret_cast<float4*>(v)[i] = make_float4(vv[0], vv[1], vv[2], vv[3]);
  reinterpret_cast<float4*>(p)[i] = make_float4(pp[0], pp[1], pp[2], pp[3]);
  if (p_bf16 != nullptr) {
    uint2 u;
    u.x = pack_bf16x2(pp[0], pp[1]);
    u.y = pack_bf16x2(pp[2], pp[3]);
    reinterpret_cast<uint2*>(p_bf16)[i] = u;
  }
}

// `clip` (device scalar: sum of squares of ALL gradients) folds global-norm clipping into the
// update without a host round trip.
__global__ void __launch_bounds__(256)
adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
             float* __restrict__ v, __nv_bfloat16* __restrict__ p_bf16, long long n, float step_size,
             float beta1, float beta2, float eps, float lr_wd, float grad_scale,
             const float* __restrict__ clip, float clip_max_norm) {
  if (clip != nullptr) {
    const float norm = sqrtf(__ldg(clip));
    grad_scale *= fminf(1.0f, clip_max_norm / (norm + 1e-6f));
  }
  const long long n4 = n >> 2;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const float ob1 = 1.0f - beta1, ob2 = 1.0f - beta2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride)
    adamw_vec4(p, g, m, v, p_bf16, i, step_size, beta1, beta2, ob1, ob2, eps, lr_wd, grad_scale);
  // tail (n not a multiple of 4)
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float gr = g[i] * grad_scale;
    const float mi = beta1 * m[i] + ob1 * gr;
    const float vi = beta2 * v[i] + ob2 * gr * gr;
    float pi = p[i] - step_size * (mi / (sqrtf(vi) + eps));
    if (lr_wd > 0.0f) pi = pi - lr_wd * pi;
    m[i] = mi;
    v[i] = vi;
    p[i] = pi;
    if (p_bf16 != nullptr) p_bf16[i] = __float2bfloat16(pi);
  }
}

// out[0] += sum of `s` over the 256 threads of the block (one atomic per block).
__device__ __forceinline__ void block_sum_atomic_add(float s, float* __restrict__ out) {
  s = warp_sum(s);
  __shared__ float sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 8) {
    float t = sm[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) t += __shfl_xor_sync(0xffu, t, o);
    if (threadIdx.x == 0) atomicAdd(out, t);
  }
}

__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ x, long long n, float* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  float s = 0.f;
  const long long n4 = n >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(x) + i);
    s = fmaf(t.x, t.x, s); s = fmaf(t.y, t.y, s); s = fmaf(t.z, t.z, s); s = fmaf(t.w, t.w, s);
  }
  for (long long i = (n4 << 2) + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float t = x[i];
    s = fmaf(t, t, s);
  }
  block_sum_atomic_add(s, out);
}

// ---- segment tables: any set of disjoint ranges of the flat buffer, each in one of at most
// HERO_ADAMW_MAX_GROUPS groups. A table is int64 triples (start, length, group), starts and lengths
// multiples of 4 (checked on the host). Work is one grid-stride loop over the float4 index of the
// concatenated segments, so it is spread over the threads as if the segments were one range. A
// thread walks the table once; inside a segment its loop is the plain strided loop of adamw_kernel
// (no per-iteration lookup). Elements outside every segment are never touched.
struct AdamwGroupArgs {
  float step_size[HERO_ADAMW_MAX_GROUPS];
  float lr_wd[HERO_ADAMW_MAX_GROUPS];
};

__global__ void __launch_bounds__(256)
adamw_groups_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                    float* __restrict__ v, __nv_bfloat16* __restrict__ p_bf16,
                    const long long* __restrict__ seg, int n_seg, const AdamwGroupArgs groups,
                    float beta1, float beta2, float eps, float grad_scale,
                    const float* __restrict__ clip, float clip_max_norm) {
  if (clip != nullptr) {
    const float norm = sqrtf(__ldg(clip));
    grad_scale *= fminf(1.0f, clip_max_norm / (norm + 1e-6f));
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  const float ob1 = 1.0f - beta1, ob2 = 1.0f - beta2;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // concatenated float4 index
  long long end4 = 0;
  for (int s = 0; s < n_seg; ++s) {
    const long long delta4 = (__ldg(seg + 3 * s) >> 2) - end4;      // buffer index - concatenated
    end4 += __ldg(seg + 3 * s + 1) >> 2;
    if (i >= end4) continue;
    const int grp = (int)__ldg(seg + 3 * s + 2);
    const float step_size = groups.step_size[grp], lr_wd = groups.lr_wd[grp];
    for (; i < end4; i += stride)
      adamw_vec4(p, g, m, v, p_bf16, i + delta4, step_size, beta1, beta2, ob1, ob2, eps, lr_wd,
                 grad_scale);
  }
}

__global__ void __launch_bounds__(256)
sumsq_segments_kernel(const float* __restrict__ x, const long long* __restrict__ seg, int n_seg,
                      float* __restrict__ out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  float acc = 0.f;
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long end4 = 0;
  for (int s = 0; s < n_seg; ++s) {
    const long long delta4 = (__ldg(seg + 3 * s) >> 2) - end4;
    end4 += __ldg(seg + 3 * s + 1) >> 2;
    for (; i < end4; i += stride) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(x) + i + delta4);
      acc = fmaf(t.x, t.x, acc); acc = fmaf(t.y, t.y, acc);
      acc = fmaf(t.z, t.z, acc); acc = fmaf(t.w, t.w, acc);
    }
  }
  block_sum_atomic_add(acc, out);
}

// Row r of the fused LM-head cross entropy: combines the (max, sum exp) partials of its slabs into
// (row max, log-sum-exp). Shared by ce_finish_kernel and ce_finish_stats_kernel, so both compute
// bitwise the same lse and loss.
__device__ __forceinline__ float2 ce_row_finish(const float2* __restrict__ part, long long ld,
                                                int n_slabs, int r) {
  float mx = -INFINITY;
  for (int t = 0; t < n_slabs; ++t) mx = fmaxf(mx, part[(long long)t * ld + r].x);   // coalesced in r
  float s = 0.f;
  for (int t = 0; t < n_slabs; ++t) {
    const float2 p = part[(long long)t * ld + r];
    s += p.y * __expf(p.x - mx);
  }
  return make_float2(mx, mx + __logf(s));
}

// Finish of the fused LM-head cross entropy: combine the (max, sum exp) partials of a row.
__global__ void __launch_bounds__(128)
ce_finish_kernel(const float2* __restrict__ part, long long ld, int n_slabs,
                 const float* __restrict__ lab, int m, float* __restrict__ loss,
                 float* __restrict__ lse) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const float l = ce_row_finish(part, ld, n_slabs, r).y;
  lse[r] = l;
  loss[r] = l - lab[r];
}

// acc[0] += sum_{r < m} a[r], acc[1] += sum_{r < m} b[r], in an order fixed by m and blockDim
// alone: every CTA has written its rows of a / b; the last CTA to finish (ticket on `done`, zeroed
// before the launch) sums all m rows, thread t taking rows t, t + blockDim, ... in turn, then the
// fixed butterfly of warp_sum and the warps in index order. No float atomics: two runs on the same
// inputs give bitwise the same acc.
template <typename TB>
__device__ __forceinline__ void last_cta_accumulate(const float* a, const TB* b, int m,
                                                    float* __restrict__ acc,
                                                    unsigned* __restrict__ done) {
  __shared__ bool last;
  __shared__ float wsum[2][32];
  __threadfence();                       // this CTA's rows of a / b are visible device-wide
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  float sa = 0.f, sb = 0.f;
  for (int r = threadIdx.x; r < m; r += blockDim.x) {
    sa += __ldcg(a + r);                 // L2: the rows were written by other SMs
    sb += (float)__ldcg(b + r);
  }
  sa = warp_sum(sa);
  sb = warp_sum(sb);
  const int warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
  if ((threadIdx.x & 31) == 0) {
    wsum[0][warp] = sa;
    wsum[1][warp] = sb;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ta = 0.f, tb = 0.f;
    for (int w = 0; w < n_warps; ++w) {
      ta += wsum[0][w];
      tb += wsum[1][w];
    }
    acc[0] += ta;
    acc[1] += tb;
  }
}

// hero_ce_finish plus the top-1 hit of every row and an optional fixed-order accumulation. The
// label logit is the same fp32 register value that entered its slab's max in the GEMM epilogue, so
// label_logit >= (max over slabs) holds exactly when the label column is a top-1 column.
__global__ void __launch_bounds__(128)
ce_finish_stats_kernel(const float2* __restrict__ part, long long ld, int n_slabs,
                       const float* __restrict__ lab, int m, float* __restrict__ loss,
                       float* __restrict__ lse, int* __restrict__ hit, float* __restrict__ acc,
                       unsigned* __restrict__ done) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < m) {
    const float2 f = ce_row_finish(part, ld, n_slabs, r);
    const float v = lab[r];
    lse[r] = f.y;
    loss[r] = f.y - v;
    hit[r] = v >= f.x ? 1 : 0;
  }
  if (acc != nullptr) last_cta_accumulate(loss, hit, m, acc, done);
}

// Per row of x, y (fp32 [m, d], rows ld apart): l2[r] = sqrt(sum (x - y)^2) and
// cos[r] = x.y / (max(|x|, eps) * max(|y|, eps)), F.cosine_similarity as torch 2.x computes it
// (each norm clamped on its own). One warp per row, eight rows per CTA.
template <bool VEC>
__global__ void __launch_bounds__(256)
row_l2_cos_kernel(const float* __restrict__ x, const float* __restrict__ y, int m, int d,
                  long long ldx, long long ldy, float eps, float* __restrict__ l2,
                  float* __restrict__ cos_out, float* __restrict__ acc,
                  unsigned* __restrict__ done) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row < m) {
    const float* xr = x + (long long)row * ldx;
    const float* yr = y + (long long)row * ldy;
    float sdd = 0.f, sxx = 0.f, syy = 0.f, sxy = 0.f;
    if (VEC) {
      for (int i = lane; i < (d >> 2); i += 32) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(xr) + i);
        const float4 b = __ldg(reinterpret_cast<const float4*>(yr) + i);
        const float xa[4] = {a.x, a.y, a.z, a.w}, yb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float t = xa[j] - yb[j];
          sdd = fmaf(t, t, sdd);
          sxx = fmaf(xa[j], xa[j], sxx);
          syy = fmaf(yb[j], yb[j], syy);
          sxy = fmaf(xa[j], yb[j], sxy);
        }
      }
    } else {
      for (int i = lane; i < d; i += 32) {
        const float a = __ldg(xr + i), b = __ldg(yr + i), t = a - b;
        sdd = fmaf(t, t, sdd);
        sxx = fmaf(a, a, sxx);
        syy = fmaf(b, b, syy);
        sxy = fmaf(a, b, sxy);
      }
    }
    sdd = warp_sum(sdd);
    sxx = warp_sum(sxx);
    syy = warp_sum(syy);
    sxy = warp_sum(sxy);
    if (lane == 0) {
      l2[row] = sqrtf(sdd);
      cos_out[row] = sxy / (fmaxf(sqrtf(sxx), eps) * fmaxf(sqrtf(syy), eps));
    }
  }
  if (acc != nullptr) last_cta_accumulate(l2, cos_out, m, acc, done);
}

// dst[i] = (dst[i] + sum_s slots[s * stride + i]) * scale: the reduction step of the copy-engine
// gradient exchange (peers have written their contributions into `slots`).
__global__ void reduce_slots_kernel(float* __restrict__ dst, const float* __restrict__ slots,
                                    int n_slots, long long stride, long long n4, float scale) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 acc = reinterpret_cast<const float4*>(dst)[i];
    for (int s = 0; s < n_slots; ++s) {
      const float4 v = reinterpret_cast<const float4*>(slots + s * stride)[i];
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    acc.x *= scale; acc.y *= scale; acc.z *= scale; acc.w *= scale;
    reinterpret_cast<float4*>(dst)[i] = acc;
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_reduce_slots_f32(float* dst, const float* slots, int32_t n_slots,
                                     int64_t slot_stride, int64_t n, float scale,
                                     int32_t max_ctas, void* stream) {
  HERO_REQUIRE(dst && (slots || n_slots == 0) && n >= 0 && n % 4 == 0 && slot_stride % 4 == 0,
               "reduce_slots: bad args (n and stride must be multiples of 4)");
  if (n == 0) return HERO_OK;
  long long blocks = (n / 4 + 255) / 256;
  const long long cap = max_ctas > 0 ? max_ctas : 64;
  if (blocks > cap) blocks = cap;
  reduce_slots_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      dst, slots, n_slots, slot_stride, n / 4, scale);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_adamw_step(float* p, const float* g, float* m, float* v, void* p_bf16,
                               int64_t n, float step_size, float beta1, float beta2, float eps,
                               float lr_wd, float grad_scale, const float* clip_sumsq,
                               float clip_max_norm, void* stream) {
  HERO_REQUIRE(p && g && m && v && n >= 0, "adamw: bad args");
  HERO_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) |
                 reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15u) == 0 &&
                   (reinterpret_cast<uintptr_t>(p_bf16) & 7u) == 0,
               "adamw: buffers must be 16-byte aligned (bf16 copy 8-byte)");
  if (n == 0) return HERO_OK;
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  long long blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > sms * 8LL) blocks = sms * 8LL;
  adamw_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      p, g, m, v, reinterpret_cast<__nv_bfloat16*>(p_bf16), n, step_size, beta1, beta2, eps, lr_wd,
      grad_scale, clip_sumsq, clip_max_norm);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

// Host-side checks of a segment table; sets *total4 to the float4 count over all segments.
static int check_segments(const int64_t* seg, int32_t n_seg, int64_t n, int32_t n_groups,
                          long long* total4) {
  HERO_REQUIRE(n_groups >= 1 && n_groups <= HERO_ADAMW_MAX_GROUPS,
               "segments: %d groups (1 to %d supported)", n_groups, HERO_ADAMW_MAX_GROUPS);
  HERO_REQUIRE(n_seg >= 0 && (seg != nullptr || n_seg == 0), "segments: bad table");
  long long sum = 0, end = 0;
  for (int32_t s = 0; s < n_seg; ++s) {
    const int64_t st = seg[3 * s], len = seg[3 * s + 1], grp = seg[3 * s + 2];
    HERO_REQUIRE(grp >= 0 && grp < n_groups, "segments: segment %d has group %lld, not in [0, %d)",
                 s, (long long)grp, n_groups);
    HERO_REQUIRE(st >= 0 && len >= 0 && len <= n - st,
                 "segments: segment %d = [%lld, %lld + %lld) is not inside [0, %lld)", s,
                 (long long)st, (long long)st, (long long)len, (long long)n);
    HERO_REQUIRE(st % 4 == 0 && len % 4 == 0,
                 "segments: segment %d: start and length must be multiples of 4", s);
    HERO_REQUIRE(st >= end, "segments: segment %d overlaps or precedes the previous one", s);
    end = st + len;
    sum += len;
  }
  *total4 = sum / 4;
  return HERO_OK;
}

static long long stream_blocks(long long n4, int sms) {
  long long blocks = (n4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > sms * 8LL) blocks = sms * 8LL;
  return blocks;
}

extern "C" int hero_adamw_step_groups(float* p, const float* g, float* m, float* v, void* p_bf16,
                                      int64_t n, const int64_t* segments_host,
                                      const int64_t* segments_dev, int32_t n_segments,
                                      const hero_adamw_groups* groups, float beta1, float beta2,
                                      float eps, float grad_scale, const float* clip_sumsq,
                                      float clip_max_norm, void* stream) {
  HERO_REQUIRE(p && g && m && v && groups && n >= 0, "adamw_groups: bad args");
  HERO_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) |
                 reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15u) == 0 &&
                   (reinterpret_cast<uintptr_t>(p_bf16) & 7u) == 0,
               "adamw_groups: buffers must be 16-byte aligned (bf16 copy 8-byte)");
  long long total4 = 0;
  const int st = check_segments(segments_host, n_segments, n, groups->n_groups, &total4);
  if (st != HERO_OK) return st;
  HERO_REQUIRE(segments_dev != nullptr || n_segments == 0, "adamw_groups: no device table");
  if (total4 == 0) return HERO_OK;
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  AdamwGroupArgs ga;
  for (int k = 0; k < HERO_ADAMW_MAX_GROUPS; ++k) {
    ga.step_size[k] = k < groups->n_groups ? groups->step_size[k] : 0.f;
    ga.lr_wd[k] = k < groups->n_groups ? groups->lr_wd[k] : 0.f;
  }
  adamw_groups_kernel<<<(unsigned)stream_blocks(total4, sms), 256, 0,
                        reinterpret_cast<cudaStream_t>(stream)>>>(
      p, g, m, v, reinterpret_cast<__nv_bfloat16*>(p_bf16),
      reinterpret_cast<const long long*>(segments_dev), n_segments, ga, beta1, beta2, eps,
      grad_scale, clip_sumsq, clip_max_norm);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_sumsq_segments_f32(const float* x, int64_t n, const int64_t* segments_host,
                                       const int64_t* segments_dev, int32_t n_segments,
                                       int32_t n_groups, float* out, void* stream) {
  HERO_REQUIRE(x && out && n >= 0, "sumsq_segments: bad args");
  HERO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15u) == 0,
               "sumsq_segments: x must be 16-byte aligned");
  long long total4 = 0;
  const int st = check_segments(segments_host, n_segments, n, n_groups, &total4);
  if (st != HERO_OK) return st;
  HERO_REQUIRE(segments_dev != nullptr || n_segments == 0, "sumsq_segments: no device table");
  if (total4 == 0) return HERO_OK;
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  sumsq_segments_kernel<<<(unsigned)stream_blocks(total4, sms), 256, 0,
                          reinterpret_cast<cudaStream_t>(stream)>>>(
      x, reinterpret_cast<const long long*>(segments_dev), n_segments, out);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_ce_finish(const void* ce_partial, int64_t ld_partial, int32_t n_slabs,
                              const float* label_logit, int32_t m, float* loss, float* lse,
                              void* stream) {
  HERO_REQUIRE(ce_partial && label_logit && loss && lse && n_slabs > 0 && ld_partial >= m,
               "ce_finish: bad args");
  if (m <= 0) return HERO_OK;
  ce_finish_kernel<<<(m + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float2*>(ce_partial), ld_partial, n_slabs, label_logit, m, loss, lse);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_ce_finish_stats(const void* ce_partial, int64_t ld_partial, int32_t n_slabs,
                                    const float* label_logit, int32_t m, float* loss, float* lse,
                                    int32_t* hit, float* acc, uint32_t* counter, void* stream) {
  HERO_REQUIRE(ce_partial && label_logit && loss && lse && hit && n_slabs > 0 && ld_partial >= m &&
                   m >= 0 && m <= HERO_ROW_STATS_MAX_ROWS,
               "ce_finish_stats: bad args (m = %d, at most %d rows)", m, HERO_ROW_STATS_MAX_ROWS);
  HERO_REQUIRE(acc == nullptr || counter != nullptr, "ce_finish_stats: acc needs a counter");
  if (m == 0) return HERO_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (acc != nullptr) HERO_CUDA_CHECK(cudaMemsetAsync(counter, 0, sizeof(uint32_t), st));
  ce_finish_stats_kernel<<<(m + 127) / 128, 128, 0, st>>>(
      reinterpret_cast<const float2*>(ce_partial), ld_partial, n_slabs, label_logit, m, loss, lse,
      hit, acc, counter);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_row_l2_cos(const float* x, int64_t ldx, const float* y, int64_t ldy, int32_t m,
                               int32_t d, float eps, float* l2, float* cos, float* acc,
                               uint32_t* counter, void* stream) {
  HERO_REQUIRE(m >= 0 && m <= HERO_ROW_STATS_MAX_ROWS && d >= 1 && d <= HERO_ROW_L2_COS_MAX_D,
               "row_l2_cos: (m, d) = (%d, %d); 0 <= m <= %d and 1 <= d <= %d", m, d,
               HERO_ROW_STATS_MAX_ROWS, HERO_ROW_L2_COS_MAX_D);
  HERO_REQUIRE(x && y && l2 && cos && ldx >= d && ldy >= d, "row_l2_cos: bad args");
  HERO_REQUIRE(acc == nullptr || counter != nullptr, "row_l2_cos: acc needs a counter");
  if (m == 0) return HERO_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (acc != nullptr) HERO_CUDA_CHECK(cudaMemsetAsync(counter, 0, sizeof(uint32_t), st));
  const bool vec = d % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 &&
                   ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) == 0;
  const unsigned blocks = (unsigned)((m + 7) / 8);
  if (vec)
    row_l2_cos_kernel<true><<<blocks, 256, 0, st>>>(x, y, m, d, ldx, ldy, eps, l2, cos, acc,
                                                    counter);
  else
    row_l2_cos_kernel<false><<<blocks, 256, 0, st>>>(x, y, m, d, ldx, ldy, eps, l2, cos, acc,
                                                     counter);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_sumsq_f32(const float* x, int64_t n, float* out, void* stream) {
  HERO_REQUIRE(x && out && n >= 0, "sumsq: bad args");
  if (n == 0) return HERO_OK;
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  HERO_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15u) == 0, "sumsq: x must be 16-byte aligned");
  long long blocks = (n / 4 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > sms * 8LL) blocks = sms * 8LL;
  sumsq_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, n, out);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

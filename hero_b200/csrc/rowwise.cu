// HBM-bound row kernels: fused gather+add+LayerNorm(+dropout)+scatter forward/backward, row
// gathers (pack / unpack / frame merge), column sums (bias grads), casts.
// One warp owns one row; 16-byte vector accesses; fp32 statistics via a true two-pass over
// registers (mean, then centred sum of squares) like apex FusedLayerNorm / torch.nn.LayerNorm.
#include <cstdlib>

#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int LN_WARPS = 4;

// Load 8 consecutive elements of the (gathered, summed) pre-LN row into v[8].
__device__ __forceinline__ void ln_load8(const hero_ln_args& a, long long xrow, int add_row, int e0,
                                         float (&v)[8]) {
  if (a.x_is_f32) {
    const float* p = reinterpret_cast<const float*>(a.x) + xrow * a.h + e0;
    const float4 u0 = __ldg(reinterpret_cast<const float4*>(p));
    const float4 u1 = __ldg(reinterpret_cast<const float4*>(p + 4));
    v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w;
    v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
  } else {
    const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(a.x) + xrow * a.h + e0;
    const uint4 u = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      v[2 * j] = f.x;
      v[2 * j + 1] = f.y;
    }
  }
  if (a.add_tab != nullptr) {
    const float* p = a.add_tab + (long long)add_row * a.h + e0;
    const float4 u0 = __ldg(reinterpret_cast<const float4*>(p));
    const float4 u1 = __ldg(reinterpret_cast<const float4*>(p + 4));
    v[0] += u0.x; v[1] += u0.y; v[2] += u0.z; v[3] += u0.w;
    v[4] += u1.x; v[5] += u1.y; v[6] += u1.z; v[7] += u1.w;
  }
  if (a.add_vec != nullptr) {
    const float* p = a.add_vec + e0;
    const float4 u0 = __ldg(reinterpret_cast<const float4*>(p));
    const float4 u1 = __ldg(reinterpret_cast<const float4*>(p + 4));
    v[0] += u0.x; v[1] += u0.y; v[2] += u0.z; v[3] += u0.w;
    v[4] += u1.x; v[5] += u1.y; v[6] += u1.z; v[7] += u1.w;
  }
}

__device__ __forceinline__ void load_f32x8(const float* p, float (&v)[8]) {
  const float4 u0 = __ldg(reinterpret_cast<const float4*>(p));
  const float4 u1 = __ldg(reinterpret_cast<const float4*>(p + 4));
  v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w;
  v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
}

__device__ __forceinline__ void load_bf16x8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}

// 8 consecutive fp32 accumulations as two 16-byte vector reductions (one L2 atomic per 4 floats).
__device__ __forceinline__ void red_add_f32x8(float* p, const float (&v)[8]) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v[0]), "f"(v[1]),
               "f"(v[2]), "f"(v[3])
               : "memory");
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p + 4), "f"(v[4]), "f"(v[5]),
               "f"(v[6]), "f"(v[7])
               : "memory");
}

__device__ __forceinline__ void store_f32x8(float* p, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// bf16(v) to `hi` and the bf16 of what that rounding lost to `lo`: v ~ hi + lo to ~16 mantissa bits
__device__ __forceinline__ void store_bf16x8_split(__nv_bfloat16* hi, __nv_bfloat16* lo,
                                                   const float (&v)[8]) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[j] = pack_bf16x2(v[2 * j], v[2 * j + 1]);
    const float2 back = unpack_bf16x2(h[j]);
    l[j] = pack_bf16x2(v[2 * j] - back.x, v[2 * j + 1] - back.y);
  }
  *reinterpret_cast<uint4*>(hi) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo) = make_uint4(l[0], l[1], l[2], l[3]);
}

__device__ __forceinline__ void store_bf16x8(__nv_bfloat16* p, const float (&v)[8]) {
  uint4 u;
  u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
  u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// ------------------------------------------------------------------ LN forward (generic)
// Every option of hero_ln_args: fp32 or bf16 rows, row gather, table / vector adds, row lengths up
// to MAXJ * 256. One warp per row; ROWS rows per warp iteration (1 in every instantiation: two
// rows in flight per warp measured slower, 25.9 vs 18.4 us at 16.5 k rows). The transformer-layer
// LayerNorms take the fast path below, the 4352-wide rows ln_fwd_wide_kernel.
template <int MAXJ, int ROWS>
__global__ void __launch_bounds__(LN_WARPS * 32)
ln_fwd_kernel(const hero_ln_args a) {
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * LN_WARPS + warp;
  const int stride = gridDim.x * LN_WARPS * ROWS;
  const float inv_h = 1.0f / (float)a.h;
  for (int base = gw * ROWS; base < a.n_rows; base += stride) {
    float v[ROWS][MAXJ][8];
    float sum[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int i = base + r;
      sum[r] = 0.f;
      if (i < a.n_rows) {
        const long long xrow = a.x_rows ? a.x_rows[i] : i;
        const int add_row = a.add_tab ? a.add_idx[i] : 0;
#pragma unroll
        for (int c = 0; c < MAXJ; ++c) {
          const int e0 = (c * 32 + lane) * 8;
          if (e0 < a.h) {
            ln_load8(a, xrow, add_row, e0, v[r][c]);
#pragma unroll
            for (int j = 0; j < 8; ++j) sum[r] += v[r][c][j];
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int i = base + r;
      if (i >= a.n_rows) break;   // warp-uniform
      const float mean = warp_sum(sum[r]) * inv_h;
      float sq = 0.f;
#pragma unroll
      for (int c = 0; c < MAXJ; ++c) {
        const int e0 = (c * 32 + lane) * 8;
        if (e0 < a.h) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float d = v[r][c][j] - mean;
            sq += d * d;
          }
        }
      }
      const float var = warp_sum(sq) * inv_h;
      const float rstd = rsqrtf(var + a.eps);
      if (lane == 0) {
        if (a.mean) a.mean[i] = mean;
        if (a.rstd) a.rstd[i] = rstd;
      }
      const long long yrow = a.y_rows ? a.y_rows[i] : i;
      __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(a.y) + yrow * a.h;
#pragma unroll
      for (int c = 0; c < MAXJ; ++c) {
        const int e0 = (c * 32 + lane) * 8;
        if (e0 < a.h) {
          float g[8], b[8], o[8];
          load_f32x8(a.gamma + e0, g);
          load_f32x8(a.beta + e0, b);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = (v[r][c][j] - mean) * rstd * g[j] + b[j];
          if (a.drop_threshold != 0u)
            dropout_apply8(o, a.drop_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                           a.drop_threshold, a.drop_scale);
          if (a.y_lo)
            store_bf16x8_split(y + e0, reinterpret_cast<__nv_bfloat16*>(a.y_lo) + yrow * a.h + e0, o);
          else
            store_bf16x8(y + e0, o);
          if (a.y_f32) store_f32x8(a.y_f32 + yrow * a.h + e0, o);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ LN fast path (h <= 768)
// The transformer-layer LayerNorms (18 of the 21 per step) read a plain bf16 row: no gather, no
// table add. The one-row-per-warp kernel above re-reads gamma/beta (6 KB of L1 traffic per 1.5 KB
// row) and has one row in flight per warp: 2.8 TB/s. Here warps are persistent, keep the
// parameters in registers, and load row i+1 (raw, packed) before normalising row i.
constexpr int LNF_J = 3;   // 3 x 32 lanes x 8 elements = 768 columns

__device__ __forceinline__ void unpack8(const uint4& u, float (&v)[8]) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}

// A row of <= 768 elements as this lane holds it between the load and its use: packed bf16
// (one uint4 per 8 elements) or fp32 (two float4). The pre-LayerNorm sums of the transformer layers
// are fp32 (the residual stream), embedding-side rows bf16.
template <bool XF32>
struct RowRaw {
  uint4 q[LNF_J][XF32 ? 2 : 1];
  __device__ __forceinline__ void load(const void* base, long long row, int h, int lane) {
#pragma unroll
    for (int c = 0; c < LNF_J; ++c) {
      const int e0 = (c * 32 + lane) * 8;
      if (XF32) {
        const float* p = reinterpret_cast<const float*>(base) + row * h + e0;
        q[c][0] = (e0 < h) ? *reinterpret_cast<const uint4*>(p) : make_uint4(0, 0, 0, 0);
        q[c][XF32 ? 1 : 0] = (e0 < h) ? *reinterpret_cast<const uint4*>(p + 4) : make_uint4(0, 0, 0, 0);
      } else {
        const __nv_bfloat16* p = reinterpret_cast<const __nv_bfloat16*>(base) + row * h + e0;
        q[c][0] = (e0 < h) ? *reinterpret_cast<const uint4*>(p) : make_uint4(0, 0, 0, 0);
      }
    }
  }
  __device__ __forceinline__ void unpack(int c, float (&v)[8]) const {
    if (XF32) {
      const uint4 a = q[c][0], b = q[c][XF32 ? 1 : 0];
      v[0] = __uint_as_float(a.x); v[1] = __uint_as_float(a.y);
      v[2] = __uint_as_float(a.z); v[3] = __uint_as_float(a.w);
      v[4] = __uint_as_float(b.x); v[5] = __uint_as_float(b.y);
      v[6] = __uint_as_float(b.z); v[7] = __uint_as_float(b.w);
    } else {
      unpack8(q[c][0], v);
    }
  }
};

template <bool XF32>
__global__ void __launch_bounds__(LN_WARPS * 32)
ln_fwd_fast_kernel(const hero_ln_args a) {
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int stride = gridDim.x * LN_WARPS;
  const float inv_h = 1.0f / (float)a.h;
  float g[LNF_J][8], b[LNF_J][8];
#pragma unroll
  for (int c = 0; c < LNF_J; ++c) {
    const int e0 = (c * 32 + lane) * 8;
    if (e0 < a.h) {
      load_f32x8(a.gamma + e0, g[c]);
      load_f32x8(a.beta + e0, b[c]);
    }
  }
  int i = blockIdx.x * LN_WARPS + warp;
  RowRaw<XF32> raw;
  if (i < a.n_rows) raw.load(a.x, a.x_rows ? a.x_rows[i] : i, a.h, lane);
  for (; i < a.n_rows; i += stride) {
    float v[LNF_J][8];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < LNF_J; ++c) {
      raw.unpack(c, v[c]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += v[c][j];
    }
    const int nxt = i + stride;
    if (nxt < a.n_rows) raw.load(a.x, a.x_rows ? a.x_rows[nxt] : nxt, a.h, lane);
    const float mean = warp_sum(sum) * inv_h;
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < LNF_J; ++c) {
      if ((c * 32 + lane) * 8 < a.h) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[c][j] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) * inv_h + a.eps);
    if (lane == 0) {
      if (a.mean) a.mean[i] = mean;
      if (a.rstd) a.rstd[i] = rstd;
    }
    const long long yrow = a.y_rows ? a.y_rows[i] : i;
    __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(a.y) + yrow * (long long)a.h;
#pragma unroll
    for (int c = 0; c < LNF_J; ++c) {
      const int e0 = (c * 32 + lane) * 8;
      if (e0 < a.h) {
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * g[c][j] + b[c][j];
        if (a.drop_threshold != 0u)
          dropout_apply8(o, a.drop_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                         a.drop_threshold, a.drop_scale);
        store_bf16x8(y + e0, o);
        if (a.y_f32) store_f32x8(a.y_f32 + yrow * (long long)a.h + e0, o);
      }
    }
  }
}

// Backward fast path: row gradients AND the column reductions (dgamma, dbeta, dbias) in one pass
// over x and dy. Per-lane fp32 accumulators for the lane's 24 columns live in registers for the
// whole kernel; at the end the CTA's warps are summed through shared memory and each CTA issues
// one atomicAdd per column and output. (The split row kernel + column kernel read x and dy twice
// and dx_drop once more: 55 us per 16.5 k-token call against 17 us of HBM time.)
template <bool XF32>
__global__ void __launch_bounds__(LN_WARPS * 32, XF32 ? 1 : 2)
ln_bwd_fast_kernel(const hero_ln_args a) {
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int stride = gridDim.x * LN_WARPS;
  const float inv_h = 1.0f / (float)a.h;
  float g[LNF_J][8], dg[LNF_J][8], db[LNF_J][8], dbi[LNF_J][8];
#pragma unroll
  for (int c = 0; c < LNF_J; ++c) {
    const int e0 = (c * 32 + lane) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) g[c][j] = dg[c][j] = db[c][j] = dbi[c][j] = 0.f;
    if (e0 < a.h) load_f32x8(a.gamma + e0, g[c]);
  }
  int i = blockIdx.x * LN_WARPS + warp;
  RowRaw<XF32> rx;
  RowRaw<false> rd;
  float mean = 0.f, rstd = 0.f;
  if (i < a.n_rows) {
    rx.load(a.x, a.x_rows ? a.x_rows[i] : i, a.h, lane);
    rd.load(a.dy, a.y_rows ? a.y_rows[i] : i, a.h, lane);
    mean = a.mean[i];
    rstd = a.rstd[i];
  }
  for (; i < a.n_rows; i += stride) {
    float xh[LNF_J][8], gy[LNF_J][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int c = 0; c < LNF_J; ++c) {
      float d[8];
      rx.unpack(c, xh[c]);
      rd.unpack(c, d);
      const int e0 = (c * 32 + lane) * 8;
      if (a.drop_threshold != 0u)
        dropout_apply8(d, a.drop_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                       a.drop_threshold, a.drop_scale);
      const bool ok = e0 < a.h;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        xh[c][j] = ok ? (xh[c][j] - mean) * rstd : 0.f;
        gy[c][j] = d[j] * g[c][j];
        s1 += gy[c][j];
        s2 += gy[c][j] * xh[c][j];
        dg[c][j] += d[j] * xh[c][j];
        db[c][j] += d[j];
      }
    }
    const float rstd_i = rstd;
    const int nxt = i + stride;
    if (nxt < a.n_rows) {
      rx.load(a.x, a.x_rows ? a.x_rows[nxt] : nxt, a.h, lane);
      rd.load(a.dy, a.y_rows ? a.y_rows[nxt] : nxt, a.h, lane);
      mean = a.mean[nxt];
      rstd = a.rstd[nxt];
    }
    const float c1 = warp_sum(s1) * inv_h;
    const float c2 = warp_sum(s2) * inv_h;
#pragma unroll
    for (int c = 0; c < LNF_J; ++c) {
      const int e0 = (c * 32 + lane) * 8;
      if (e0 < a.h) {
        float dx[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) dx[j] = rstd_i * (gy[c][j] - c1 - xh[c][j] * c2);
        if (a.dx) store_bf16x8(reinterpret_cast<__nv_bfloat16*>(a.dx) + (long long)i * a.h + e0, dx);
        if (a.dx_drop) {
          if (a.drop2_threshold != 0u)
            dropout_apply8(dx, a.drop2_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                           a.drop2_threshold, a.drop2_scale);
          store_bf16x8(reinterpret_cast<__nv_bfloat16*>(a.dx_drop) + (long long)i * a.h + e0, dx);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) dbi[c][j] += dx[j];
      }
    }
  }
  // CTA reduction of the column accumulators, one output at a time through a [768] smem row
  __shared__ float red[LNF_J * 32 * 8];
  float* outs[3] = {a.dgamma, a.dbeta, a.dbias};
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    if (outs[pass] == nullptr) continue;   // CTA-uniform
    for (int w = 0; w < LN_WARPS; ++w) {
      __syncthreads();
      if (warp == w) {
#pragma unroll
        for (int c = 0; c < LNF_J; ++c) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float val = pass == 0 ? dg[c][j] : (pass == 1 ? db[c][j] : dbi[c][j]);
            float* slot = red + (c * 8 + j) * 32 + lane;   // conflict-free: lanes -> banks
            *slot = (w == 0) ? val : *slot + val;
          }
        }
      }
    }
    __syncthreads();
    for (int col = threadIdx.x; col < a.h; col += LN_WARPS * 32)
      atomicAdd(outs[pass] + col, red[((col >> 8) * 8 + (col & 7)) * 32 + ((col & 255) >> 3)]);
  }
}

// ------------------------------------------------------------------ LN forward, wide rows
// The 4352-d frame-feature LayerNorms (model/embed.py:108-116, model/layers.py:82-90): a 17 KB fp32
// row per warp left 3 200 warps with 136 values each in registers (255 regs, 1 TB/s). Here a
// 256-thread CTA owns a row (<= 3 x 8 elements per thread), CTAs are persistent over rows and
// keep gamma / beta in registers; mean and centred variance are block reductions.
constexpr int LNW_THREADS = 256;
constexpr int LNW_C = 3;   // rows of up to 3 * 256 * 8 = 6144 elements

__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();          // red[] may still be read by the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < LNW_THREADS / 32; ++w) t += red[w];
  return t;
}

// (gamma / beta are re-read per row - 35 KB that stay in L1 - instead of living in 48 registers:
// at 64 registers four CTAs fit per SM, and one row per CTA in flight needs that many to cover
// the HBM latency)
__global__ void __launch_bounds__(LNW_THREADS, 4)
ln_fwd_wide_kernel(const hero_ln_args a) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ float red[LNW_THREADS / 32];
  const float inv_h = 1.0f / (float)a.h;
  for (int i = blockIdx.x; i < a.n_rows; i += gridDim.x) {
    const long long xrow = a.x_rows ? a.x_rows[i] : i;
    const int add_row = a.add_tab ? a.add_idx[i] : 0;
    float v[LNW_C][8];
    float sum = 0.f;
#pragma unroll
    for (int c = 0; c < LNW_C; ++c) {
      const int e0 = (c * LNW_THREADS + threadIdx.x) * 8;
      if (e0 < a.h) {
        ln_load8(a, xrow, add_row, e0, v[c]);
#pragma unroll
        for (int j = 0; j < 8; ++j) sum += v[c][j];
      }
    }
    const float mean = block_sum_256(sum, red) * inv_h;
    float sq = 0.f;
#pragma unroll
    for (int c = 0; c < LNW_C; ++c) {
      if ((c * LNW_THREADS + threadIdx.x) * 8 < a.h) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[c][j] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(block_sum_256(sq, red) * inv_h + a.eps);
    if (threadIdx.x == 0) {
      if (a.mean) a.mean[i] = mean;
      if (a.rstd) a.rstd[i] = rstd;
    }
    const long long yoff = (a.y_rows ? a.y_rows[i] : i) * (long long)a.h;
    __nv_bfloat16* y = reinterpret_cast<__nv_bfloat16*>(a.y) + yoff;
    __nv_bfloat16* ylo = a.y_lo ? reinterpret_cast<__nv_bfloat16*>(a.y_lo) + yoff : nullptr;
#pragma unroll
    for (int c = 0; c < LNW_C; ++c) {
      const int e0 = (c * LNW_THREADS + threadIdx.x) * 8;
      if (e0 < a.h) {
        float o[8], g[8], b[8];
        load_f32x8(a.gamma + e0, g);
        load_f32x8(a.beta + e0, b);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = (v[c][j] - mean) * rstd * g[j] + b[j];
        if (a.drop_threshold != 0u)
          dropout_apply8(o, a.drop_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                         a.drop_threshold, a.drop_scale);
        if (ylo) store_bf16x8_split(y + e0, ylo + e0, o); else store_bf16x8(y + e0, o);
      }
    }
  }
}

// ------------------------------------------------------------------ LN backward, generic (rows)
// dx (and its dropout-masked copy / table scatter-adds) per row, one warp per row. Parameter and
// bias gradients of this path are column reductions done by ln_param_grad_kernel.
template <int MAXJ, int ROWS>
__global__ void __launch_bounds__(LN_WARPS * 32)
ln_bwd_kernel(const hero_ln_args a) {
  pdl_wait();
  pdl_launch_dependents();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gw = blockIdx.x * LN_WARPS + warp;
  const int stride = gridDim.x * LN_WARPS * ROWS;
  const float inv_h = 1.0f / (float)a.h;

  for (int base = gw * ROWS; base < a.n_rows; base += stride) {
    float xh[ROWS][MAXJ][8], gy[ROWS][MAXJ][8];
    float s1[ROWS], s2[ROWS], rs[ROWS];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int i = base + r;
      s1[r] = s2[r] = 0.f;
      rs[r] = 0.f;
      if (i < a.n_rows) {
        const long long xrow = a.x_rows ? a.x_rows[i] : i;
        const int add_row = a.add_tab ? a.add_idx[i] : 0;
        const long long yrow = a.y_rows ? a.y_rows[i] : i;
        const float mean = a.mean[i], rstd = a.rstd[i];
        rs[r] = rstd;
        const __nv_bfloat16* dy = reinterpret_cast<const __nv_bfloat16*>(a.dy) + yrow * a.h;
#pragma unroll
        for (int c = 0; c < MAXJ; ++c) {
          const int e0 = (c * 32 + lane) * 8;
          if (e0 < a.h) {
            ln_load8(a, xrow, add_row, e0, xh[r][c]);
            float d[8], g[8];
            load_bf16x8(dy + e0, d);
            load_f32x8(a.gamma + e0, g);
            if (a.drop_threshold != 0u)
              dropout_apply8(d, a.drop_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                             a.drop_threshold, a.drop_scale);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              xh[r][c][j] = (xh[r][c][j] - mean) * rstd;
              gy[r][c][j] = d[j] * g[j];
              s1[r] += gy[r][c][j];
              s2[r] += gy[r][c][j] * xh[r][c][j];
            }
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
      const int i = base + r;
      if (i >= a.n_rows) break;   // warp-uniform
      const float c1 = warp_sum(s1[r]) * inv_h;
      const float c2 = warp_sum(s2[r]) * inv_h;
      const float rstd = rs[r];
      const long long xrow = a.x_rows ? a.x_rows[i] : i;
      const int add_row = a.add_tab ? a.add_idx[i] : 0;
#pragma unroll
      for (int c = 0; c < MAXJ; ++c) {
        const int e0 = (c * 32 + lane) * 8;
        if (e0 < a.h) {
          float dx[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) dx[j] = rstd * (gy[r][c][j] - c1 - xh[r][c][j] * c2);
          if (a.dx) store_bf16x8(reinterpret_cast<__nv_bfloat16*>(a.dx) + (long long)i * a.h + e0, dx);
          if (a.dx_drop) {
            float dd[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) dd[j] = dx[j];
            if (a.drop2_threshold != 0u)
              dropout_apply8(dd, a.drop2_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)e0,
                             a.drop2_threshold, a.drop2_scale);
            store_bf16x8(reinterpret_cast<__nv_bfloat16*>(a.dx_drop) + (long long)i * a.h + e0, dd);
          }
          if (a.d_x_tab && (int)xrow != a.x_pad_idx) {
            red_add_f32x8(a.d_x_tab + xrow * a.h + e0, dx);
          }
          if (a.d_add_tab && a.add_tab && add_row != a.add_pad_idx) {
            red_add_f32x8(a.d_add_tab + (long long)add_row * a.h + e0, dx);
          }
        }
      }
    }
  }
}

// Column-parallel parameter gradients: dgamma += sum_i dy*xhat, dbeta += sum_i dy, and optionally
// dbias += sum_i dx_drop (the bias gradient of the Linear feeding this LayerNorm). Each thread owns
// 8 consecutive columns (16-byte loads); block = 32 column groups x 8 row lanes; grid.y splits rows.
// Runs after the row kernel, whose dx / dx_drop output is still L2-resident.
__global__ void __launch_bounds__(256)
ln_param_grad_kernel(const hero_ln_args a, int rows_per_block) {
  pdl_wait();
  pdl_launch_dependents();
  const int cg = threadIdx.x & 31;
  const int col = (blockIdx.x * 32 + cg) * 8;
  const int rl = threadIdx.x >> 5;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(a.n_rows, r0 + rows_per_block);
  const bool want_gb = a.dgamma != nullptr || a.dbeta != nullptr;
  const __nv_bfloat16* dsrc = reinterpret_cast<const __nv_bfloat16*>(a.dx_drop ? a.dx_drop : a.dx);
  const bool want_bias = a.dbias != nullptr && dsrc != nullptr;
  float dg[8], db[8], dbi[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) dg[j] = db[j] = dbi[j] = 0.f;
  if (col < a.h) {
    for (int i = r0 + rl; i < r1; i += 8) {
      if (want_gb) {
        const long long xrow = a.x_rows ? a.x_rows[i] : i;
        const long long yrow = a.y_rows ? a.y_rows[i] : i;
        const int add_row = a.add_tab ? a.add_idx[i] : 0;
        float x[8], d[8];
        ln_load8(a, xrow, add_row, col, x);
        load_bf16x8(reinterpret_cast<const __nv_bfloat16*>(a.dy) + yrow * a.h + col, d);
        if (a.drop_threshold != 0u)
          dropout_apply8(d, a.drop_key, (uint32_t)i * (uint32_t)a.h + (uint32_t)col,
                         a.drop_threshold, a.drop_scale);
        const float mean = a.mean[i], rstd = a.rstd[i];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          dg[j] += d[j] * (x[j] - mean) * rstd;
          db[j] += d[j];
        }
      }
      if (want_bias) {
        float v[8];
        load_bf16x8(dsrc + (long long)i * a.h + col, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) dbi[j] += v[j];
      }
    }
  }
  __shared__ float sm[8][32 * 8 + 4];
  float* outs[3] = {a.dgamma, a.dbeta, want_bias ? a.dbias : nullptr};
  for (int pass = 0; pass < 3; ++pass) {
    if (outs[pass] == nullptr) continue;   // block-uniform
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[rl][cg * 8 + j] = pass == 0 ? dg[j] : (pass == 1 ? db[j] : dbi[j]);
    __syncthreads();
    const int c = threadIdx.x;
    const int gcol = blockIdx.x * 256 + c;
    if (gcol < a.h) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) t += sm[w][c];
      atomicAdd(outs[pass] + gcol, t);
    }
  }
}

// ------------------------------------------------------------------ row gathers
__global__ void gather_rows_kernel(const __nv_bfloat16* __restrict__ src,
                                   const int32_t* __restrict__ idx, __nv_bfloat16* __restrict__ dst,
                                   int n, int h8) {
  pdl_wait();
  pdl_launch_dependents();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n * h8) return;
  const int i = (int)(t / h8), c = (int)(t % h8);
  const int s = idx[i];
  uint4 v = make_uint4(0, 0, 0, 0);
  if (s >= 0) v = reinterpret_cast<const uint4*>(src)[(long long)s * h8 + c];
  reinterpret_cast<uint4*>(dst)[(long long)i * h8 + c] = v;
}

__global__ void gather_rows_f32_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx,
                                       float* __restrict__ dst, int n, int h4) {
  pdl_wait();
  pdl_launch_dependents();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n * h4) return;
  const int i = (int)(t / h4), c = (int)(t % h4);
  const int s = idx[i];
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (s >= 0) v = reinterpret_cast<const float4*>(src)[(long long)s * h4 + c];
  reinterpret_cast<float4*>(dst)[(long long)i * h4 + c] = v;
}

// bf16 output: one thread per (row, 8-column chunk) walks the row's (short) CSR list.
__global__ void gather_sum_rows_kernel(const __nv_bfloat16* __restrict__ src,
                                       const int32_t* __restrict__ off,
                                       const int32_t* __restrict__ idx,
                                       __nv_bfloat16* __restrict__ dst, int n, int h8) {
  pdl_wait();
  pdl_launch_dependents();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n * h8) return;
  const int i = (int)(t / h8), c = (int)(t % h8);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  const int e0 = off[i], e1 = off[i + 1];
  for (int e = e0; e < e1; ++e) {
    float v[8];
    load_bf16x8(src + ((long long)idx[e] * h8 + c) * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += v[j];
  }
  store_bf16x8(dst + ((long long)i * h8 + c) * 8, acc);
}

// fp32 accumulate output (embedding-table gradients: few rows, long lists): grid = (row, split);
// each block sums a slice of the row's list with h/8 threads and adds it with fp32 atomics.
__global__ void gather_sum_rows_f32_kernel(const __nv_bfloat16* __restrict__ src,
                                           const int32_t* __restrict__ off,
                                           const int32_t* __restrict__ idx, float* __restrict__ dst,
                                           int h8, int per_split) {
  pdl_wait();
  pdl_launch_dependents();
  const int i = blockIdx.x;
  const int end = off[i + 1];
  for (int e0 = off[i] + blockIdx.y * per_split; e0 < end; e0 += gridDim.y * per_split) {
    const int e1 = min(end, e0 + per_split);
    for (int c = threadIdx.x; c < h8; c += blockDim.x) {
      float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      int e = e0;
      // four independent rows in flight (a serial chain of L2-latency loads made a 64-entry
      // slice cost ~25 us regardless of the data volume)
      for (; e + 4 <= e1; e += 4) {
        float v0[8], v1[8], v2[8], v3[8];
        const int r0 = idx[e], r1 = idx[e + 1], r2 = idx[e + 2], r3 = idx[e + 3];
        load_bf16x8(src + ((long long)r0 * h8 + c) * 8, v0);
        load_bf16x8(src + ((long long)r1 * h8 + c) * 8, v1);
        load_bf16x8(src + ((long long)r2 * h8 + c) * 8, v2);
        load_bf16x8(src + ((long long)r3 * h8 + c) * 8, v3);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += (v0[j] + v1[j]) + (v2[j] + v3[j]);
      }
      for (; e < e1; ++e) {
        float v[8];
        load_bf16x8(src + ((long long)idx[e] * h8 + c) * 8, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
      }
      red_add_f32x8(dst + ((long long)i * h8 + c) * 8, acc);
    }
  }
}

// out[n] += sum_m x[m, n]. Each thread owns 8 consecutive columns (16-byte loads); a block is
// 32 column groups (256 columns = 512 B per row, fully coalesced) x 8 row lanes; grid.y splits rows.
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ x, long long ld, int m, int n,
              float* __restrict__ out, int rows_per_block) {
  pdl_wait();
  pdl_launch_dependents();
  const int cg = threadIdx.x & 31;
  const int col = (blockIdx.x * 32 + cg) * 8;
  const int rl = threadIdx.x >> 5;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(m, r0 + rows_per_block);
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (col < n) {
    int r = r0 + rl;
    // two rows in flight per iteration
    for (; r + 8 < r1; r += 16) {
      float v0[8], v1[8];
      load_bf16x8(x + (long long)r * ld + col, v0);
      load_bf16x8(x + (long long)(r + 8) * ld + col, v1);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v0[j] + v1[j];
    }
    for (; r < r1; r += 8) {
      float v0[8];
      load_bf16x8(x + (long long)r * ld + col, v0);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v0[j];
    }
  }
  __shared__ float sm[8][32 * 8 + 4];
#pragma unroll
  for (int j = 0; j < 8; ++j) sm[rl][cg * 8 + j] = acc[j];
  __syncthreads();
  // thread t sums column t of the block's 256 columns over the 8 row lanes
  const int c = threadIdx.x;
  const int gcol = blockIdx.x * 256 + c;
  if (gcol < n) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += sm[w][c];
    atomicAdd(out + gcol, t);
  }
}

__global__ void relu_bwd_kernel(const __nv_bfloat16* __restrict__ dy,
                                const __nv_bfloat16* __restrict__ pre,
                                __nv_bfloat16* __restrict__ out, long long n8) {
  pdl_wait();
  pdl_launch_dependents();
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n8) return;
  float d[8], p[8];
  load_bf16x8(dy + t * 8, d);
  load_bf16x8(pre + t * 8, p);
#pragma unroll
  for (int j = 0; j < 8; ++j) d[j] = p[j] > 0.f ? d[j] : 0.f;
  store_bf16x8(out + t * 8, d);
}

__global__ void cast_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                            long long n) {
  const long long t = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if (t + 8 <= n) {
    float v[8];
    load_f32x8(src + t, v);
    store_bf16x8(dst + t, v);
  } else {
    for (long long j = t; j < n; ++j) dst[j] = __float2bfloat16(src[j]);
  }
}

// Plain bf16 rows of at most 768 columns (every transformer-layer LayerNorm): fast kernels.
static bool ln_fast_ok(const hero_ln_args* a) {
  return a->h <= LNF_J * 256 && a->add_tab == nullptr && a->add_vec == nullptr &&
         a->y_lo == nullptr;
}

static int check_ln(const hero_ln_args* a) {
  HERO_REQUIRE(a != nullptr, "null ln args");
  HERO_REQUIRE(a->x && a->gamma, "ln: null x/gamma");
  HERO_REQUIRE(a->h > 0 && a->h % 8 == 0 && a->h <= 4352, "ln: unsupported row length %d", a->h);
  HERO_REQUIRE(a->add_tab == nullptr || a->add_idx != nullptr, "ln: add_tab needs add_idx");
  return HERO_OK;
}

}  // namespace hero

using namespace hero;

extern "C" int hero_ln_fwd(const hero_ln_args* a, void* stream) {
  if (int rc = check_ln(a)) return rc;
  HERO_REQUIRE(a->y && a->beta, "ln_fwd: null y/beta");
  HERO_REQUIRE(a->y_f32 == nullptr || a->h <= 768, "ln_fwd: y_f32 needs h <= 768");
  if (a->n_rows <= 0) return HERO_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  if (ln_fast_ok(a)) {
    int grid = ceil_div(a->n_rows, LN_WARPS);
    if (grid > sms * 4) grid = sms * 4;
    if (a->x_is_f32)
      HERO_CUDA_CHECK(launch_pdl(ln_fwd_fast_kernel<true>, dim3(grid), dim3(LN_WARPS * 32), 0, st, *a));
    else
      HERO_CUDA_CHECK(launch_pdl(ln_fwd_fast_kernel<false>, dim3(grid), dim3(LN_WARPS * 32), 0, st, *a));
  } else if (a->h <= 768) {
    HERO_CUDA_CHECK(launch_pdl(ln_fwd_kernel<3, 1>, dim3(ceil_div(a->n_rows, LN_WARPS)),
                               dim3(LN_WARPS * 32), 0, st, *a));
  } else if (a->h <= LNW_C * LNW_THREADS * 8 && a->n_rows >= 64) {
    int grid = a->n_rows < sms * 8 ? a->n_rows : sms * 8;
    HERO_CUDA_CHECK(launch_pdl(ln_fwd_wide_kernel, dim3(grid), dim3(LNW_THREADS), 0, st, *a));
  } else {
    int grid = ceil_div(a->n_rows, LN_WARPS);
    if (grid > sms * 8) grid = sms * 8;
    HERO_CUDA_CHECK(launch_pdl(ln_fwd_kernel<17, 1>, dim3(grid), dim3(LN_WARPS * 32), 0, st, *a));
  }
  return HERO_OK;
}

extern "C" int hero_ln_bwd(const hero_ln_args* a, void* stream) {
  if (int rc = check_ln(a)) return rc;
  HERO_REQUIRE(a->dy && a->mean && a->rstd, "ln_bwd: null dy/mean/rstd");
  if (a->n_rows <= 0) return HERO_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  const bool want_rows = a->dx || a->dx_drop || a->d_x_tab || a->d_add_tab;
  const bool want_cols = a->dgamma || a->dbeta || a->dbias;
  if (want_rows && ln_fast_ok(a) && !a->d_x_tab && !a->d_add_tab) {
    // one pass: row gradients + dgamma / dbeta / dbias
    int grid = ceil_div(a->n_rows, LN_WARPS);
    if (grid > sms * 2) grid = sms * 2;
    if (a->x_is_f32)
      HERO_CUDA_CHECK(launch_pdl(ln_bwd_fast_kernel<true>, dim3(grid), dim3(LN_WARPS * 32), 0, st, *a));
    else
      HERO_CUDA_CHECK(launch_pdl(ln_bwd_fast_kernel<false>, dim3(grid), dim3(LN_WARPS * 32), 0, st, *a));
    return HERO_OK;
  }
  if (want_rows) {
    if (a->h <= 768) {
      HERO_CUDA_CHECK(launch_pdl(ln_bwd_kernel<3, 1>, dim3(ceil_div(a->n_rows, LN_WARPS)),
                                 dim3(LN_WARPS * 32), 0, st, *a));
    } else {
      int grid = ceil_div(a->n_rows, LN_WARPS);
      if (grid > sms * 8) grid = sms * 8;
      HERO_CUDA_CHECK(launch_pdl(ln_bwd_kernel<17, 1>, dim3(grid), dim3(LN_WARPS * 32), 0, st, *a));
    }
  }
  if (want_cols) {
    HERO_REQUIRE(!a->dbias || a->dx || a->dx_drop, "ln_bwd: dbias needs dx or dx_drop");
    const int col_blocks = ceil_div(a->h, 256);
    int row_splits = ceil_div(sms * 8, col_blocks);
    if (row_splits > ceil_div(a->n_rows, 32)) row_splits = ceil_div(a->n_rows, 32);
    if (row_splits < 1) row_splits = 1;
    const int rpb = ceil_div(a->n_rows, row_splits);
    dim3 g(col_blocks, ceil_div(a->n_rows, rpb));
    HERO_CUDA_CHECK(launch_pdl(ln_param_grad_kernel, g, dim3(256), 0, st, *a, rpb));
  }
  return HERO_OK;
}

extern "C" int hero_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) {
  HERO_REQUIRE(src && dst && n >= 0, "cast: bad args");
  if (n == 0) return HERO_OK;
  const long long groups = (n + 7) / 8;
  cast_kernel<<<(unsigned)((groups + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      src, reinterpret_cast<__nv_bfloat16*>(dst), n);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_gather_rows_bf16(const void* src, const int32_t* idx, void* dst, int32_t n,
                                     int32_t h, void* stream) {
  HERO_REQUIRE(src && idx && dst && h % 8 == 0, "gather_rows: bad args");
  if (n <= 0) return HERO_OK;
  const long long total = (long long)n * (h / 8);
  gather_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0,
                       reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), idx, reinterpret_cast<__nv_bfloat16*>(dst), n,
      h / 8);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_gather_rows_f32(const float* src, const int32_t* idx, float* dst, int32_t n,
                                    int32_t h, void* stream) {
  HERO_REQUIRE(src && idx && dst && h % 4 == 0, "gather_rows_f32: bad args");
  if (n <= 0) return HERO_OK;
  const long long total = (long long)n * (h / 4);
  gather_rows_f32_kernel<<<(unsigned)((total + 255) / 256), 256, 0,
                           reinterpret_cast<cudaStream_t>(stream)>>>(src, idx, dst, n, h / 4);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_gather_sum_rows_bf16(const void* src, const int32_t* off, const int32_t* idx,
                                         void* dst, int32_t n, int32_t h, void* stream) {
  HERO_REQUIRE(src && off && dst && h % 8 == 0, "gather_sum_rows: bad args");
  if (n <= 0) return HERO_OK;
  const long long total = (long long)n * (h / 8);
  gather_sum_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0,
                           reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), off, idx, reinterpret_cast<__nv_bfloat16*>(dst),
      n, h / 8);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_gather_sum_rows_f32(const void* src, const int32_t* off, const int32_t* idx,
                                        float* dst, int32_t n, int32_t h, void* stream) {
  HERO_REQUIRE(src && off && dst && h % 8 == 0, "gather_sum_rows_f32: bad args");
  if (n <= 0) return HERO_OK;
  // Lists can be thousands of entries long (every sequence shares a position row): each block
  // sums 32-entry slices (looping when a list has more than 64 * 32 entries) and adds its partial
  // with fp32 atomics; rows with short lists cost one early-exit block each.
  dim3 grid(n, 64);
  gather_sum_rows_f32_kernel<<<grid, 96, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(src), off, idx, dst, h / 8, 32);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

extern "C" int hero_colsum_bf16(const void* x, int64_t ld, int32_t m, int32_t n, float* out,
                                void* stream) {
  HERO_REQUIRE(x && out, "colsum: bad args");
  if (m <= 0 || n <= 0) return HERO_OK;
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  HERO_REQUIRE(n % 8 == 0 && ld % 8 == 0, "colsum: n and ld must be multiples of 8");
  const int col_blocks = ceil_div(n, 256);
  int row_splits = ceil_div(sms * 8, col_blocks);
  if (row_splits > ceil_div(m, 32)) row_splits = ceil_div(m, 32);
  if (row_splits < 1) row_splits = 1;
  const int rpb = ceil_div(m, row_splits);
  dim3 g(col_blocks, ceil_div(m, rpb));
  HERO_CUDA_CHECK(launch_pdl(colsum_kernel, g, dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                             reinterpret_cast<const __nv_bfloat16*>(x), (long long)ld, m, n, out,
                             rpb));
  return HERO_OK;
}

extern "C" int hero_relu_bwd_bf16(const void* dy, const void* pre, void* out, int64_t n,
                                  void* stream) {
  HERO_REQUIRE(dy && pre && out && n % 8 == 0, "relu_bwd: bad args");
  if (n == 0) return HERO_OK;
  const long long n8 = n / 8;
  relu_bwd_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const __nv_bfloat16*>(pre),
      reinterpret_cast<__nv_bfloat16*>(out), n8);
  HERO_LAUNCH_CHECK();
  return HERO_OK;
}

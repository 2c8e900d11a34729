// Variable-length multi-head self-attention on the Hopper tensor cores (wgmma / TMA).
//
// HERO's sequences are short (cross-modal rows ~10-70 tokens, temporal rows <= 100 frames), so a
// 128-row MMA tile would be mostly empty if it held one sequence. Instead the host packs
// CONSECUTIVE sequences of the packed token stream into tiles of <= 128 tokens (a sequence never
// straddles tiles); one CTA handles one (tile, head):
//
//   forward   S = Q K^T (128x128x64)  -> per-row softmax restricted to the row's own sequence
//             (block-diagonal mask = the key-padding mask of model/layers.py:299-302 in the packed
//             layout) -> P (bf16, smem) -> O = P V (128x64x128) -> ctx
//   backward  S = Q K^T, dP = dO V^T -> P, dS rows -> dV = P^T dO, dK = dS^T Q, dQ = dS K
//
// Q/K/V/dO tiles arrive by TMA (128-byte swizzle); every contraction is a warpgroup wgmma with
// fp32 accumulators in registers. The transposed operands (P^T, dS^T, V/dO/Q/K as [k][n]) need no
// copies: the SAME smem tiles are addressed as MN-major operands through the wgmma descriptors.
// Softmax statistics, exp2, dropout masks and the P / dS tiles never touch HBM.
//
// Replaces model/layers.py:129-160 (BertSelfAttention after the QKV projections) and its autograd
// backward. D_i = sum_j P_ij dP_ij is taken as dO_i . O_i from the saved forward output.
#include <cuda.h>

#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int AT_ROWS = 128;           // tokens per tile
constexpr int AT_D = 64;               // head dim
constexpr int AT_TILE_BYTES = AT_ROWS * AT_D * 2;   // 16 KB: one [128 x 64] bf16 operand tile
constexpr int AT_P_BYTES = AT_ROWS * AT_ROWS * 2;   // 32 KB: one [128 x 128] bf16 tile (2 chunks)

// Block-diagonal mask on the tensor core. A fifth K = 16 step of the S = Q K^T MMA multiplies the
// tile's sequence-membership matrix E [128 tokens x 16 sequence ordinals] (128.0 at a token's own
// sequence, else 0) with itself: S'_ij = S_ij + 16384 * [seq(i) == seq(j)]. Softmax is
// shift-invariant per row, so the row's own sequence sees its plain softmax while every other
// column (other sequences of the tile, rows past the tile's end) sits 16384 raw = 2955 log2 units
// lower and its exp2 is exactly 0: the softmax loops need no compares, selects or predicates.
// 16384 is exact in fp32 next to |S| < 2^10 up to an absolute error of 2^-9 (2.4e-4 relative in
// p, an eighth of P's bf16 rounding). The reference adds -10000 to the scaled scores
// (model/layers.py:299-302), i.e. 80000 raw: equally finite. The host plan keeps <= AT_MAX_SEQS
// sequences per tile.
constexpr int AT_MAX_SEQS = 16;
constexpr int AT_MASK_BYTES = 2 * AT_MAX_SEQS * 128;   // [k = ordinal][mn = token], 2 chunks of 64 tokens
constexpr float AT_MASK_BIG = 16384.0f;

// Column i of the membership operand (MN-major: one 128-byte row per ordinal, tokens contiguous,
// two 64-token chunks of 2 KB): thread i owns its token's 16 entries.
template <int K0 = 0, int K1 = AT_MAX_SEQS>
__device__ __forceinline__ void write_membership(uint8_t* sE, int i, int ord) {
  uint8_t* base = sE + (i >> 6) * (AT_MAX_SEQS * 128) + ((i & 7) << 1);
  const int u = (i & 63) >> 3;
#pragma unroll
  for (int k = K0; k < K1; ++k)
    *reinterpret_cast<uint16_t*>(base + k * 128 + ((u ^ (k & 7)) << 4)) =
        (k == ord) ? static_cast<uint16_t>(0x4300) : static_cast<uint16_t>(0);   // bf16 128.0
}

// Ordinal (0-based) of thread i's sequence within the tile, -1 for rows past the tile's end:
// the number of sequence starts at rows <= i, minus one. `warp_starts` is 4 ints of smem; the
// caller synchronises the CTA between the two halves.
__device__ __forceinline__ uint32_t seq_starts_ballot(bool valid, int lo, int i, int* warp_starts) {
  const uint32_t bal = __ballot_sync(0xffffffffu, valid && lo == i);
  // (a 256-thread CTA has two warps per row quadrant: both write the same count)
  if ((threadIdx.x & 31) == 0) warp_starts[(threadIdx.x >> 5) & 3] = __popc(bal);
  return bal;
}
__device__ __forceinline__ int seq_ordinal(bool valid, uint32_t bal, const int* warp_starts) {
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  int ord = __popc(bal & (0xffffffffu >> (31 - lane))) - 1;
  for (int w = 0; w < warp; ++w) ord += warp_starts[w];
  return valid ? ord : -1;
}

// element (row i, col j) of a [128 x 128] bf16 tile stored as two 64-column chunks of
// [128 rows x 128 B] with the 128-byte swizzle: byte offset of the 16-byte unit holding cols
// [8u', 8u'+8) where j = 64*chunk + 8u + (j % 8).
__device__ __forceinline__ uint32_t p_unit_offset(int row, int chunk, int u) {
  return chunk * (AT_ROWS * 128) + row * 128 + ((u ^ (row & 7)) << 4);
}

__device__ __forceinline__ float ex2(float x) { return fast_ex2(x); }

struct AttnTcArgs {
  const int32_t* tile_tok0;
  const int32_t* tile_ntok;
  const int32_t* seq_lo;
  const int32_t* seq_hi;
  int heads;
  int H;
  float scale_log2;      // log2(e) / sqrt(d)
  float scale;           // 1 / sqrt(d)
  uint32_t drop_thr, drop_key;
  float drop_scale;
};

// A warp's part of a [64 x 64] wgmma result (rows 16w + l/4 and + 8, columns 8j + 2(l%4) + {0,1}),
// optionally scaled, parked as bf16 in a swizzled [128 x 128 B] smem tile at tile row row0 + ...
__device__ __forceinline__ void stage_frag64(uint8_t* tile, int row0, const float (&o)[32],
                                             float sa, float sb) {
  const int lane = threadIdx.x & 31;
  const int fc = (lane & 3) * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = row0 + (lane >> 2) + 8 * h;
    const float sc = h ? sb : sa;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      *reinterpret_cast<uint32_t*>(tile + r * 128 + ((j ^ (r & 7)) << 4) + fc * 2) =
          pack_bf16x2(o[4 * j + 2 * h] * sc, o[4 * j + 2 * h + 1] * sc);
  }
}
// ... and the CTA then writes the tile(s) out with every warp covering 4 full 128-byte rows per
// instruction (a lane-per-row store would touch 32 different lines per instruction).
// Rows >= ntok belong to the next tile.
__device__ __forceinline__ void store_tiles(const uint8_t* tiles, int n_parts, __nv_bfloat16* base,
                                            long long row_stride, long long part_stride, int ntok) {
  for (int idx = threadIdx.x; idx < n_parts * AT_ROWS * 8; idx += blockDim.x) {
    const int part = idx >> 10, row = (idx >> 3) & 127, u = idx & 7;
    if (row < ntok) {
      const uint4 v = *reinterpret_cast<const uint4*>(tiles + part * AT_TILE_BYTES + row * 128 +
                                                      ((u ^ (row & 7)) << 4));
      *reinterpret_cast<uint4*>(base + row * row_stride + part * part_stride + u * 8) = v;
    }
  }
}

// S[64 rows from row 64 * g, 128 keys] of the tile = Q K^T + 16384 * [same sequence], issued by one
// warpgroup (Q, K K-major; the membership operand MN-major on both sides)
__device__ __forceinline__ void issue_scores(float (&s)[64], const uint8_t* sQ, const uint8_t* sK,
                                             const uint8_t* sE, int g) {
#pragma unroll
  for (int k = 0; k < AT_D / 16; ++k)
    wgmma_m64n128k16<0, 0>(s, make_sw128_desc(smem_u32(sQ) + g * 8192 + k * 32, 16, 1024),
                           make_sw128_desc(smem_u32(sK) + k * 32, 16, 1024), k > 0 ? 1u : 0u);
  wgmma_m64n128k16<1, 1>(s, make_sw128_desc(smem_u32(sE) + g * 2048, AT_MAX_SEQS * 128, 1024),
                         make_sw128_desc(smem_u32(sE), AT_MAX_SEQS * 128, 1024), 1u);
}

// ------------------------------------------------------------------------------------ forward
// One warpgroup; the 128 query rows are taken as two 64-row halves (S of a half: 64 fp32 registers
// per thread). The softmax runs on the accumulator fragment: a row's 128 scores are spread over
// the four lanes of a quad (32 each), so its max and sum take two shuffles.
__global__ void __launch_bounds__(128)
attn_tc_fwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv, const AttnTcArgs a,
                   __nv_bfloat16* __restrict__ ctx, float* __restrict__ lse) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  // Q, K, V operand tiles, then P (32 KB, two 64-column chunks); the output is staged over Q
  uint8_t* sQ = smem;
  uint8_t* sK = smem + AT_TILE_BYTES;
  uint8_t* sV = smem + 2 * AT_TILE_BYTES;
  uint8_t* sP = smem + 3 * AT_TILE_BYTES;
  uint8_t* sE = sP + AT_P_BYTES;                    // sequence-membership operand (4 KB)
  uint64_t* bars = reinterpret_cast<uint64_t*>(sE + AT_MASK_BYTES);
  uint64_t* tma_bar = bars;
  int* warp_starts = reinterpret_cast<int*>(bars + 3);

  const int tile = blockIdx.x, head = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tok0 = a.tile_tok0[tile];
  const int ntok = a.tile_ntok[tile];
  // (the plan arrays were uploaded long before the previous kernel started: safe before pdl_wait)
  const int i = threadIdx.x;
  const bool valid = i < ntok;
  int lo = 0;
  if (valid) lo = a.seq_lo[tok0 + i] - tok0;
  const uint32_t starts = seq_starts_ballot(valid, lo, i, warp_starts);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    mbar_init(tma_bar, 1);
    fence_barrier_init();
    pdl_wait();
    mbar_arrive_expect_tx(tma_bar, 3 * AT_TILE_BYTES);
    tma_load_2d(sQ, &tmap_qkv, tma_bar, head * AT_D, tok0);
    tma_load_2d(sK, &tmap_qkv, tma_bar, a.H + head * AT_D, tok0);
    tma_load_2d(sV, &tmap_qkv, tma_bar, 2 * a.H + head * AT_D, tok0);
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  {
    const int ord = seq_ordinal(valid, starts, warp_starts);
    if (ord >= AT_MAX_SEQS) __trap();     // the plan packs <= AT_MAX_SEQS sequences per tile
    write_membership(sE, i, ord);
    fence_proxy_async();
  }
  __syncthreads();
  mbar_wait(tma_bar, 0);

  const int fc = (lane & 3) * 2;
  const uint32_t k2 = attn_drop_k2(a.drop_thr);
  float inv[2][2];
#pragma unroll 1
  for (int g = 0; g < 2; ++g) {
    float s[64];
    wgmma_fence();
    issue_scores(s, sQ, sK, sE, g);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(s);
    // ---- softmax of rows r[0], r[1]: the other sequences' columns underflow to exactly 0 ----
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) mx[h] = fmaxf(mx[h], fmaxf(s[4 * j + 2 * h], s[4 * j + 2 * h + 1]));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = g * 64 + warp * 16 + (lane >> 2) + 8 * h;
      const float nmx = -mx[h] * a.scale_log2;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const float p0 = ex2(fmaf(s[4 * j + 2 * h], a.scale_log2, nmx));
        const float p1 = ex2(fmaf(s[4 * j + 2 * h + 1], a.scale_log2, nmx));
        sum[h] += p0 + p1;
        uint32_t pk = pack_bf16x2(p0, p1);
        if (a.drop_thr != 0u)      // the 1 / (1 - p) scale is folded into the output row scale
          pk &= attn_keep_mask2(
              attn_drop_pair(attn_drop_group(a.drop_key, tok0 + r, a.heads, head, j), fc >> 1), k2);
        *reinterpret_cast<uint32_t*>(sP + p_unit_offset(r, j >> 3, j & 7) + fc * 2) = pk;
      }
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
      inv[g][h] = (sum[h] > 0.f ? 1.0f / sum[h] : 0.f) * (a.drop_thr != 0u ? a.drop_scale : 1.0f);
      if (r < ntok && lse != nullptr && (lane & 3) == 0)   // log2-domain log-sum-exp, for the backward
        lse[(long long)(tok0 + r) * a.heads + head] = (mx[h] - AT_MASK_BIG) * a.scale_log2 + log2f(sum[h]);
    }
  }
  fence_proxy_async();
  __syncthreads();

  // O = P V (A = P K-major, B = V MN-major), staged over the dead Q tile
#pragma unroll 1
  for (int g = 0; g < 2; ++g) {
    float o[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_ROWS / 16; ++k)
      wgmma_m64n64k16<0, 1>(
          o, make_sw128_desc(smem_u32(sP) + (k >> 2) * (AT_ROWS * 128) + g * 8192 + (k & 3) * 32, 16, 1024),
          make_sw128_desc(smem_u32(sV) + k * 2048, AT_TILE_BYTES, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o);
    stage_frag64(sQ, g * 64 + warp * 16, o, inv[g][0], inv[g][1]);
  }
  __syncthreads();
  store_tiles(sQ, 1, ctx + (long long)tok0 * a.H + head * AT_D, a.H, 0, ntok);
}

// ------------------------------------------------------------------------------------ backward
// Two warpgroups; warpgroup g owns tile rows [64g, 64g + 64) of every product. S and dP of its
// rows stay in registers (2 x 64 per thread) and become P / dS in smem in ONE pass, the
// probabilities rebuilt from the forward's log-sum-exp. smem (112 KB): Q, K, V, dO tiles;
// P's first 64-column chunk is written over V, its second over the forward output O (both dead
// once every S / dP MMA has retired), dS after them.
constexpr int AT_BWD_THREADS = 256;
__global__ void __launch_bounds__(AT_BWD_THREADS)
attn_tc_bwd_kernel(const __grid_constant__ CUtensorMap tmap_qkv,
                   const __grid_constant__ CUtensorMap tmap_do,
                   const __grid_constant__ CUtensorMap tmap_o, const AttnTcArgs a,
                   const float* __restrict__ lse, __nv_bfloat16* __restrict__ dqkv,
                   float* __restrict__ dbias) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();
  uint8_t* sQ = smem;
  uint8_t* sK = smem + AT_TILE_BYTES;
  uint8_t* sV = smem + 2 * AT_TILE_BYTES;
  uint8_t* sdO = smem + 3 * AT_TILE_BYTES;
  // P chunk 0 over V, chunk 1 after dO: chunk stride = 2 tiles
  uint8_t* sP = sV;
  constexpr uint32_t P_CHUNK = 2 * AT_TILE_BYTES;
  uint8_t* sdS = smem + 5 * AT_TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sdS + AT_P_BYTES);
  uint64_t* tma_bar = bars;
  int* warp_starts = reinterpret_cast<int*>(bars + 3);
  float* sDi = reinterpret_cast<float*>(bars + 8);   // D_i of the tile's rows
  uint8_t* sE = sdS;     // membership operand of the S MMA; dS is written after that MMA retired

  const int tile = blockIdx.x, head = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tok0 = a.tile_tok0[tile];
  const int ntok = a.tile_ntok[tile];
  const int i = threadIdx.x & 127;        // tile row (membership, D_i)
  const int half = threadIdx.x >> 7;      // = the warpgroup
  const bool valid = i < ntok;
  int lo = 0;
  if (valid) lo = a.seq_lo[tok0 + i] - tok0;
  const uint32_t starts = seq_starts_ballot(valid, lo, i, warp_starts);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_qkv);
    tma_prefetch_desc(&tmap_do);
    tma_prefetch_desc(&tmap_o);
    mbar_init(tma_bar, 1);
    fence_barrier_init();
    pdl_wait();
    mbar_arrive_expect_tx(tma_bar, 5 * AT_TILE_BYTES);
    tma_load_2d(sQ, &tmap_qkv, tma_bar, head * AT_D, tok0);
    tma_load_2d(sK, &tmap_qkv, tma_bar, a.H + head * AT_D, tok0);
    tma_load_2d(sV, &tmap_qkv, tma_bar, 2 * a.H + head * AT_D, tok0);
    tma_load_2d(sdO, &tmap_do, tma_bar, head * AT_D, tok0);
    // the forward output O lands where P's second chunk will be written later
    tma_load_2d(sP + P_CHUNK, &tmap_o, tma_bar, head * AT_D, tok0);
  }
  __syncthreads();
  pdl_wait();
  pdl_launch_dependents();

  {
    const int ord = seq_ordinal(valid, starts, warp_starts);
    if (ord >= AT_MAX_SEQS) __trap();
    if (half == 0) write_membership<0, AT_MAX_SEQS / 2>(sE, i, ord);
    else write_membership<AT_MAX_SEQS / 2, AT_MAX_SEQS>(sE, i, ord);
    fence_proxy_async();
  }
  __syncthreads();
  mbar_wait(tma_bar, 0);
  // S = Q K^T (+ membership), dP = dO V^T go first; D_i is computed while they run
  float s[64], dp[64];
  wgmma_fence();
  issue_scores(s, sQ, sK, sE, half);
#pragma unroll
  for (int k = 0; k < AT_D / 16; ++k)
    wgmma_m64n128k16<0, 0>(dp, make_sw128_desc(smem_u32(sdO) + half * 8192 + k * 32, 16, 1024),
                           make_sw128_desc(smem_u32(sV) + k * 32, 16, 1024), k > 0 ? 1u : 0u);
  wgmma_commit();
  // D_i = dO_i . O_i from the swizzled smem tiles (conflict-free 16-byte reads)
  if (half == 0) {
    float Di = 0.f;
    if (valid) {
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        const uint32_t off = i * 128 + ((g ^ (i & 7)) << 4);
        const uint4 o = *reinterpret_cast<const uint4*>(sP + P_CHUNK + off);
        const uint4 d = *reinterpret_cast<const uint4*>(sdO + off);
        const uint32_t ow[4] = {o.x, o.y, o.z, o.w}, dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 x = unpack_bf16x2(ow[j]), y = unpack_bf16x2(dw[j]);
          Di = fmaf(x.x, y.x, Di);
          Di = fmaf(x.y, y.y, Di);
        }
      }
    }
    sDi[i] = Di;
  }
  wgmma_wait<0>();
  wgmma_fence_acc(s);
  wgmma_fence_acc(dp);
  // every S / dP MMA has retired and every O row has been read: V, O and E are dead from here on
  __syncthreads();

  const bool drop = a.drop_thr != 0u;
  const float keep_scale = drop ? a.drop_scale : 1.0f;
  const uint32_t ks_bits = __float_as_uint(keep_scale);
  const uint32_t k2 = attn_drop_k2(a.drop_thr);
  const int fc = (lane & 3) * 2;
  const int wrow0 = half * 64 + (warp & 3) * 16;   // this warp's 16 rows
  // Stored tiles: P = bf16(p) on kept lanes (dV = keep_scale * P^T dO, scaled when dV is staged),
  // dS = p * (dP * keep - D) (dQ, dK scaled by 1 / sqrt(d) when staged; a power of two).
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wrow0 + (lane >> 2) + 8 * h;
    const bool rv = r < ntok;
    // exponent offset of this row: its log-sum-exp plus the membership shift; rows past the
    // tile's end get +inf so that their P and dS rows (which the transposed products sum over)
    // are 0
    const float row_c =
        rv ? fmaf(AT_MASK_BIG, a.scale_log2, lse[(long long)(tok0 + r) * a.heads + head]) : INFINITY;
    const float Di = sDi[r];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      uint32_t m2 = 0xFFFFFFFFu;
      float keep0 = 1.0f, keep1 = 1.0f;
      if (drop) {
        const uint32_t h0 = attn_drop_group(a.drop_key, tok0 + r, a.heads, head, j);
        const uint32_t sg = attn_keep_sum(attn_drop_pair(h0, fc >> 1), k2);
        m2 = prmt(sg, 0u, 0xBB99u);
        keep0 = __uint_as_float(prmt(sg, 0u, 0x9999u) & ks_bits);
        keep1 = __uint_as_float(prmt(sg, 0u, 0xBBBBu) & ks_bits);
      }
      const int q = 4 * j + 2 * h;
      const float p0 = ex2(fmaf(s[q], a.scale_log2, -row_c));
      const float p1 = ex2(fmaf(s[q + 1], a.scale_log2, -row_c));
      const float ds0 = p0 * fmaf(dp[q], keep0, -Di);
      const float ds1 = p1 * fmaf(dp[q + 1], keep1, -Di);
      const uint32_t in_chunk = r * 128 + (((j & 7) ^ (r & 7)) << 4) + fc * 2;
      *reinterpret_cast<uint32_t*>(sP + (j >> 3) * P_CHUNK + in_chunk) = pack_bf16x2(p0, p1) & m2;
      *reinterpret_cast<uint32_t*>(sdS + (j >> 3) * (AT_ROWS * 128) + in_chunk) =
          pack_bf16x2(ds0, ds1);
    }
  }
  fence_proxy_async();
  __syncthreads();

  {
    // dQ[i][d] = sum_j dS[i][j] K[j][d] : A = dS K-major, B = K tile as [k=j][n=d] (MN-major)
    // dK[j][d] = sum_i dS[i][j] Q[i][d], dV[j][d] = sum_i P[i][j] dO[i][d]:
    //   A = dS^T / P^T = the same smem tiles read MN-major, B = Q / dO tiles MN-major
    float dq[32], dk[32], dv[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AT_ROWS / 16; ++k) {
      wgmma_m64n64k16<0, 1>(
          dq, make_sw128_desc(smem_u32(sdS) + (k >> 2) * (AT_ROWS * 128) + half * 8192 + (k & 3) * 32, 16, 1024),
          make_sw128_desc(smem_u32(sK) + k * 2048, AT_TILE_BYTES, 1024), k > 0 ? 1u : 0u);
      wgmma_m64n64k16<1, 1>(
          dk, make_sw128_desc(smem_u32(sdS) + half * (AT_ROWS * 128) + k * 2048, AT_ROWS * 128, 1024),
          make_sw128_desc(smem_u32(sQ) + k * 2048, AT_TILE_BYTES, 1024), k > 0 ? 1u : 0u);
      wgmma_m64n64k16<1, 1>(
          dv, make_sw128_desc(smem_u32(sP) + half * P_CHUNK + k * 2048, P_CHUNK, 1024),
          make_sw128_desc(smem_u32(sdO) + k * 2048, AT_TILE_BYTES, 1024), k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dq);
    wgmma_fence_acc(dk);
    wgmma_fence_acc(dv);
    __syncthreads();     // every operand read has retired: Q / K / V(P) tiles take the results
    // rows of dQ (query r), dK / dV (key r) -> dqkv[tok0 + r, {0, H, 2H} + head * 64 ...]: staged
    // in the Q / K / V tiles, then written with coalesced row stores
    stage_frag64(sQ, wrow0, dq, a.scale, a.scale);
    stage_frag64(sK, wrow0, dk, a.scale, a.scale);
    stage_frag64(sV, wrow0, dv, keep_scale, keep_scale);
  }
  // Bias gradient of the QKV projection = column sums of dqkv over the tile's tokens: one more
  // MMA over the staged tiles. A = [dQ | dK] (then [dV | -]) read MN-major (m = feature,
  // k = token), B = 16 identical rows of the token-validity vector (K-major) -> every column of
  // D holds the column sums: one fp32 atomic per feature replaces a separate pass over dqkv.
  uint8_t* sB = sdS;
  if (dbias != nullptr) {
    const int idx = threadIdx.x;                          // unit (n, chunk, u)
    const int n = idx >> 4, ch = (idx >> 3) & 1, u = idx & 7;
    const int k0 = ch * 64 + u * 8;
    uint32_t w[4];
#pragma unroll
    for (int e = 0; e < 4; ++e)
      w[e] = ((k0 + 2 * e < ntok) ? 0x3F80u : 0u) | ((k0 + 2 * e + 1 < ntok) ? 0x3F800000u : 0u);
    *reinterpret_cast<uint4*>(sB + ch * 2048 + n * 128 + ((u ^ (n & 7)) << 4)) =
        make_uint4(w[0], w[1], w[2], w[3]);
  }
  fence_proxy_async();
  __syncthreads();
  store_tiles(smem, 3, dqkv + (long long)tok0 * (3 * a.H) + head * AT_D, 3LL * a.H, a.H, ntok);
  if (dbias != nullptr) {
    float* db = dbias + head * AT_D;
    // warpgroup g: features [64g, 64g + 64) of [dQ | dK] (tiles 0, 1), then warpgroup 0 alone: dV
#pragma unroll 1
    for (int grp = 0; grp < 2 - half; ++grp) {
      float cs[8];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < AT_ROWS / 16; ++k)
        wgmma_m64n16k16<1, 0>(
            cs, make_sw128_desc(smem_u32(smem) + (grp * 2 + half) * AT_TILE_BYTES + k * 2048, AT_TILE_BYTES, 1024),
            make_sw128_desc(smem_u32(sB) + (k >> 2) * 2048 + (k & 3) * 32, 16, 1024), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(cs);
      if ((lane & 3) == 0) {
        const int f = (warp & 3) * 16 + (lane >> 2);       // feature of d[0]; d[2]: f + 8
        float* dst = db + (grp == 1 ? 2 * a.H : (half ? a.H : 0));
        atomicAdd(dst + f, cs[0]);
        atomicAdd(dst + f + 8, cs[2]);
      }
    }
  }
}


// ------------------------------------------------------------------------------------ long rows
// Sequences longer than one 128-token tile (reference limit: max_position_embeddings = 514;
// cross-modal rows of max_txt_len subtitle tokens + matched frames, model/embed.py:33-41,
// config/train-tv*.json) are rare in HERO batches. They are handled by plain fp32 CUDA-core
// kernels, one CTA per (sequence, head), K / V (forward, dQ) or Q / dO (dK, dV) of the whole
// sequence staged in shared memory as bf16: exact same arithmetic contract as the tile kernels
// (softmax over the row's own sequence, the same dropout words, log2-domain LSE), ~20x slower per
// token, which is irrelevant at their frequency.
constexpr int AL_MAX = 768;            // tokens per long sequence (2 x 768 x 128 B = 192 KB smem)
constexpr int AL_THREADS = 256;

__device__ __forceinline__ void al_load_rows(uint8_t* dst, const __nv_bfloat16* src, long long ld,
                                             int n) {
  // n rows of 64 bf16 (128 B) -> dense [n][128 B] smem, 16-byte units
  for (int idx = threadIdx.x; idx < n * 8; idx += blockDim.x) {
    const int r = idx >> 3, u = idx & 7;
    *reinterpret_cast<uint4*>(dst + r * 128 + u * 16) =
        *reinterpret_cast<const uint4*>(src + (long long)r * ld + u * 8);
  }
}

__device__ __forceinline__ void al_row_f32(const uint8_t* row, float (&v)[64]) {
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const uint4 q = *reinterpret_cast<const uint4*>(row + u * 16);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      v[u * 8 + 2 * j] = f.x;
      v[u * 8 + 2 * j + 1] = f.y;
    }
  }
}

__device__ __forceinline__ void al_global_row_f32(const __nv_bfloat16* p, float (&v)[64]) {
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const uint4 q = *reinterpret_cast<const uint4*>(p + u * 8);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      v[u * 8 + 2 * j] = f.x;
      v[u * 8 + 2 * j + 1] = f.y;
    }
  }
}

__device__ __forceinline__ float al_dot_row(const float (&q)[64], const uint8_t* row) {
  float s = 0.f;
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const uint4 k = *reinterpret_cast<const uint4*>(row + u * 16);   // broadcast read
    const uint32_t w[4] = {k.x, k.y, k.z, k.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      s = fmaf(q[u * 8 + 2 * j], f.x, s);
      s = fmaf(q[u * 8 + 2 * j + 1], f.y, s);
    }
  }
  return s;
}

__device__ __forceinline__ void al_axpy_row(float (&acc)[64], float a, const uint8_t* row) {
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    const uint4 k = *reinterpret_cast<const uint4*>(row + u * 16);
    const uint32_t w[4] = {k.x, k.y, k.z, k.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      acc[u * 8 + 2 * j] = fmaf(a, f.x, acc[u * 8 + 2 * j]);
      acc[u * 8 + 2 * j + 1] = fmaf(a, f.y, acc[u * 8 + 2 * j + 1]);
    }
  }
}

__device__ __forceinline__ void al_store_row(__nv_bfloat16* p, const float (&v)[64], float scale) {
#pragma unroll
  for (int u = 0; u < 8; ++u) {
    uint4 q;
    q.x = pack_bf16x2(v[u * 8] * scale, v[u * 8 + 1] * scale);
    q.y = pack_bf16x2(v[u * 8 + 2] * scale, v[u * 8 + 3] * scale);
    q.z = pack_bf16x2(v[u * 8 + 4] * scale, v[u * 8 + 5] * scale);
    q.w = pack_bf16x2(v[u * 8 + 6] * scale, v[u * 8 + 7] * scale);
    *reinterpret_cast<uint4*>(p + u * 8) = q;
  }
}

// bias-gradient contribution of one stored row (the bf16-rounded values, like the tile kernels)
template <int N>
__device__ __forceinline__ void al_add_row(float* dst, const float (&v)[N]) {
#pragma unroll
  for (int d = 0; d < N; ++d) atomicAdd(dst + d, __bfloat162float(__float2bfloat16(v[d])));
}

// dropout keep factor of probability (query token tok, head, key column j RELATIVE to the tile
// start = the sequence start for a long tile): the same word layout as the tile kernels
__device__ __forceinline__ float al_keep(const AttnTcArgs& a, int tok, int head, int j) {
  if (a.drop_thr == 0u) return 1.0f;
  return attn_drop_keep(a.drop_key, a.drop_thr, tok, a.heads, head, j) ? a.drop_scale : 0.f;
}

// forward (MODE 0): ctx, lse.   dQ (MODE 1): K, V in smem, thread per query row.
template <int MODE>
__global__ void __launch_bounds__(AL_THREADS)
attn_long_q_kernel(const AttnTcArgs a, int first_tile, const __nv_bfloat16* __restrict__ qkv,
                   __nv_bfloat16* __restrict__ ctx, float* __restrict__ lse,
                   const __nv_bfloat16* __restrict__ dctx, __nv_bfloat16* __restrict__ dqkv,
                   float* __restrict__ dbias) {
  extern __shared__ __align__(16) uint8_t smem[];
  pdl_wait();
  pdl_launch_dependents();
  const int tile = first_tile + blockIdx.x, head = blockIdx.y;
  const int tok0 = a.tile_tok0[tile], n = a.tile_ntok[tile];
  uint8_t* sK = smem;
  uint8_t* sV = smem + (size_t)n * 128;
  const long long ld = 3LL * a.H;
  al_load_rows(sK, qkv + (long long)tok0 * ld + a.H + head * AT_D, ld, n);
  al_load_rows(sV, qkv + (long long)tok0 * ld + 2 * a.H + head * AT_D, ld, n);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float q[64];
    al_global_row_f32(qkv + (long long)(tok0 + i) * ld + head * AT_D, q);
    if (MODE == 0) {
      float mx = -INFINITY;
      for (int j = 0; j < n; ++j) mx = fmaxf(mx, al_dot_row(q, sK + j * 128));
      float sum = 0.f, o[64];
#pragma unroll
      for (int d = 0; d < 64; ++d) o[d] = 0.f;
      for (int j = 0; j < n; ++j) {
        const float p = ex2((al_dot_row(q, sK + j * 128) - mx) * a.scale_log2);
        sum += p;
        al_axpy_row(o, p * al_keep(a, tok0 + i, head, j), sV + j * 128);
      }
      if (lse != nullptr) lse[(long long)(tok0 + i) * a.heads + head] = mx * a.scale_log2 + log2f(sum);
      al_store_row(ctx + (long long)(tok0 + i) * a.H + head * AT_D, o, 1.0f / sum);
    } else {
      float dO[64], O[64], dq[64];
      al_global_row_f32(dctx + (long long)(tok0 + i) * a.H + head * AT_D, dO);
      al_global_row_f32(ctx + (long long)(tok0 + i) * a.H + head * AT_D, O);
      float Di = 0.f;
#pragma unroll
      for (int d = 0; d < 64; ++d) {
        Di = fmaf(dO[d], O[d], Di);
        dq[d] = 0.f;
      }
      const float row_lse = lse[(long long)(tok0 + i) * a.heads + head];
      for (int j = 0; j < n; ++j) {
        const float p = ex2(fmaf(al_dot_row(q, sK + j * 128), a.scale_log2, -row_lse));
        const float dp = al_dot_row(dO, sV + j * 128);
        const float ds = p * (dp * al_keep(a, tok0 + i, head, j) - Di) * a.scale;
        al_axpy_row(dq, ds, sK + j * 128);
      }
      al_store_row(dqkv + (long long)(tok0 + i) * ld + head * AT_D, dq, 1.0f);
      if (dbias != nullptr) al_add_row(dbias + head * AT_D, dq);
    }
  }
}

// dK, dV: Q, dO of the sequence in smem (+ per-query LSE and D); a PAIR of threads owns one key
// row, each half of the 64 features (partial dot products are summed with one shuffle).
__global__ void __launch_bounds__(AL_THREADS)
attn_long_kv_kernel(const AttnTcArgs a, int first_tile, const __nv_bfloat16* __restrict__ qkv,
                    const __nv_bfloat16* __restrict__ ctx, const float* __restrict__ lse,
                    const __nv_bfloat16* __restrict__ dctx, __nv_bfloat16* __restrict__ dqkv,
                    float* __restrict__ dbias) {
  extern __shared__ __align__(16) uint8_t smem[];
  pdl_wait();
  pdl_launch_dependents();
  const int tile = first_tile + blockIdx.x, head = blockIdx.y;
  const int tok0 = a.tile_tok0[tile], n = a.tile_ntok[tile];
  uint8_t* sQ = smem;
  uint8_t* sdO = smem + (size_t)n * 128;
  float* sL = reinterpret_cast<float*>(smem + (size_t)n * 256);
  float* sD = sL + n;
  const long long ld = 3LL * a.H;
  al_load_rows(sQ, qkv + (long long)tok0 * ld + head * AT_D, ld, n);
  al_load_rows(sdO, dctx + (long long)tok0 * a.H + head * AT_D, a.H, n);
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float dO[64], O[64];
    al_row_f32(sdO + i * 128, dO);
    al_global_row_f32(ctx + (long long)(tok0 + i) * a.H + head * AT_D, O);
    float Di = 0.f;
#pragma unroll
    for (int d = 0; d < 64; ++d) Di = fmaf(dO[d], O[d], Di);
    sD[i] = Di;
    sL[i] = lse[(long long)(tok0 + i) * a.heads + head];
  }
  __syncthreads();
  const int half = threadIdx.x & 1;
  for (int j0 = 0; j0 < n; j0 += AL_THREADS / 2) {
    const int j = j0 + (threadIdx.x >> 1);
    const bool ok = j < n;          // pairs stay together: the shuffle below needs both lanes
    float k[32], v[32], dk[32], dv[32];
#pragma unroll
    for (int d = 0; d < 32; ++d) k[d] = v[d] = dk[d] = dv[d] = 0.f;
    if (ok) {
      const __nv_bfloat16* kp = qkv + (long long)(tok0 + j) * ld + a.H + head * AT_D + half * 32;
      const __nv_bfloat16* vp = kp + a.H;
#pragma unroll
      for (int d = 0; d < 32; d += 2) {
        const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kp + d));
        const float2 y = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(vp + d));
        k[d] = x.x; k[d + 1] = x.y; v[d] = y.x; v[d + 1] = y.y;
      }
    }
    for (int i = 0; i < n; ++i) {
      const uint8_t* qrow = sQ + i * 128 + half * 64;
      const uint8_t* drow = sdO + i * 128 + half * 64;
      float q[32], dO[32];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint4 a4 = *reinterpret_cast<const uint4*>(qrow + u * 16);
        const uint4 b4 = *reinterpret_cast<const uint4*>(drow + u * 16);
        const uint32_t aw[4] = {a4.x, a4.y, a4.z, a4.w}, bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 x = unpack_bf16x2(aw[t]), y = unpack_bf16x2(bw[t]);
          q[u * 8 + 2 * t] = x.x; q[u * 8 + 2 * t + 1] = x.y;
          dO[u * 8 + 2 * t] = y.x; dO[u * 8 + 2 * t + 1] = y.y;
        }
      }
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        s = fmaf(q[d], k[d], s);
        dp = fmaf(dO[d], v[d], dp);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      dp += __shfl_xor_sync(0xffffffffu, dp, 1);
      const float p = ex2(fmaf(s, a.scale_log2, -sL[i]));
      const float keep = al_keep(a, tok0 + i, head, j);
      const float pd = p * keep;
      const float ds = p * (dp * keep - sD[i]) * a.scale;
#pragma unroll
      for (int d = 0; d < 32; ++d) {
        dv[d] = fmaf(pd, dO[d], dv[d]);
        dk[d] = fmaf(ds, q[d], dk[d]);
      }
    }
    if (ok) {
      __nv_bfloat16* dkp = dqkv + (long long)(tok0 + j) * ld + a.H + head * AT_D + half * 32;
      __nv_bfloat16* dvp = dkp + a.H;
#pragma unroll
      for (int d = 0; d < 32; d += 2) {
        *reinterpret_cast<uint32_t*>(dkp + d) = pack_bf16x2(dk[d], dk[d + 1]);
        *reinterpret_cast<uint32_t*>(dvp + d) = pack_bf16x2(dv[d], dv[d + 1]);
      }
      if (dbias != nullptr) {
        al_add_row(dbias + a.H + head * AT_D + half * 32, dk);
        al_add_row(dbias + 2 * a.H + head * AT_D + half * 32, dv);
      }
    }
  }
}

static int fill_args(AttnTcArgs* a, const int32_t* tile_tok0, const int32_t* tile_ntok,
                     const int32_t* seq_lo, const int32_t* seq_hi, int heads, int head_dim,
                     float scale, uint32_t thr, uint32_t key, float dscale) {
  HERO_REQUIRE(tile_tok0 && tile_ntok && seq_lo && seq_hi, "attn: null plan pointer");
  HERO_REQUIRE(head_dim == AT_D, "attn: head_dim must be 64 (got %d)", head_dim);
  HERO_REQUIRE(heads > 0, "attn: bad head count");
  a->tile_tok0 = tile_tok0;
  a->tile_ntok = tile_ntok;
  a->seq_lo = seq_lo;
  a->seq_hi = seq_hi;
  a->heads = heads;
  a->H = heads * head_dim;
  a->scale = scale;
  a->scale_log2 = scale * 1.4426950408889634f;
  a->drop_thr = thr;
  a->drop_key = key;
  a->drop_scale = dscale;
  return HERO_OK;
}

}  // namespace hero

using namespace hero;

static int long_smem_bytes(int max_long) { return max_long * 256 + max_long * 8 + 64; }

extern "C" int hero_attn_fwd(const void* qkv, const int32_t* tile_tok0, const int32_t* tile_ntok,
                                const int32_t* seq_lo, const int32_t* seq_hi, void* ctx, float* lse,
                                int32_t n_tok, int32_t n_tiles, int32_t n_long, int32_t max_long,
                                int32_t heads, int32_t head_dim,
                                float scale, uint32_t drop_threshold, uint32_t drop_key,
                                float drop_scale, void* stream) {
  HERO_REQUIRE(qkv && ctx, "attn_fwd: null pointer");
  HERO_REQUIRE(n_long >= 0 && n_long <= n_tiles && (n_long == 0 || (max_long > AT_ROWS && max_long <= AL_MAX)),
               "attn_fwd: bad long-sequence tiles (n_long %d, max_long %d; limit %d tokens)", n_long,
               max_long, AL_MAX);
  if (n_tiles <= 0 || n_tok <= 0) return HERO_OK;
  const int n_short = n_tiles - n_long;
  AttnTcArgs a;
  if (int rc = fill_args(&a, tile_tok0, tile_ntok, seq_lo, seq_hi, heads, head_dim, scale,
                         drop_threshold, drop_key, drop_scale))
    return rc;
  CUtensorMap tm;
  if (int rc = encode_tmap_2d_bf16(&tm, qkv, 3LL * a.H, n_tok, 3LL * a.H, AT_D, AT_ROWS)) return rc;
  const int smem = 3 * AT_TILE_BYTES + AT_P_BYTES + AT_MASK_BYTES + 64;
  static bool configured = false;
  if (!configured) {
    HERO_CUDA_CHECK(cudaFuncSetAttribute(attn_tc_fwd_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  if (n_short > 0) {
    dim3 grid(n_short, heads);
    HERO_CUDA_CHECK(launch_pdl(attn_tc_fwd_kernel, grid, dim3(128), smem,
                               reinterpret_cast<cudaStream_t>(stream), tm, a,
                               reinterpret_cast<__nv_bfloat16*>(ctx), lse));
  }
  if (n_long > 0) {
    const int lsm = long_smem_bytes(max_long);
    HERO_CUDA_CHECK(cudaFuncSetAttribute(attn_long_q_kernel<0>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, lsm));
    HERO_CUDA_CHECK(launch_pdl(attn_long_q_kernel<0>, dim3(n_long, heads), dim3(AL_THREADS), lsm,
                               reinterpret_cast<cudaStream_t>(stream), a, n_short,
                               reinterpret_cast<const __nv_bfloat16*>(qkv),
                               reinterpret_cast<__nv_bfloat16*>(ctx), lse,
                               static_cast<const __nv_bfloat16*>(nullptr),
                               static_cast<__nv_bfloat16*>(nullptr), static_cast<float*>(nullptr)));
  }
  return HERO_OK;
}

extern "C" int hero_attn_bwd(const void* qkv, const int32_t* tile_tok0, const int32_t* tile_ntok,
                                const int32_t* seq_lo, const int32_t* seq_hi, const void* ctx,
                                const void* dctx, const float* lse, void* dqkv, float* dbias,
                                int32_t n_tok,
                                int32_t n_tiles, int32_t n_long, int32_t max_long,
                                int32_t heads, int32_t head_dim, float scale,
                                uint32_t drop_threshold, uint32_t drop_key, float drop_scale,
                                void* stream) {
  HERO_REQUIRE(qkv && ctx && dctx && dqkv && lse, "attn_bwd: null pointer");
  HERO_REQUIRE(n_long >= 0 && n_long <= n_tiles && (n_long == 0 || (max_long > AT_ROWS && max_long <= AL_MAX)),
               "attn_bwd: bad long-sequence tiles (n_long %d, max_long %d; limit %d tokens)", n_long,
               max_long, AL_MAX);
  if (n_tiles <= 0 || n_tok <= 0) return HERO_OK;
  const int n_short = n_tiles - n_long;
  AttnTcArgs a;
  if (int rc = fill_args(&a, tile_tok0, tile_ntok, seq_lo, seq_hi, heads, head_dim, scale,
                         drop_threshold, drop_key, drop_scale))
    return rc;
  CUtensorMap tq, td, to;
  if (int rc = encode_tmap_2d_bf16(&tq, qkv, 3LL * a.H, n_tok, 3LL * a.H, AT_D, AT_ROWS)) return rc;
  if (int rc = encode_tmap_2d_bf16(&td, dctx, a.H, n_tok, a.H, AT_D, AT_ROWS)) return rc;
  if (int rc = encode_tmap_2d_bf16(&to, ctx, a.H, n_tok, a.H, AT_D, AT_ROWS)) return rc;
  const int smem = 5 * AT_TILE_BYTES + AT_P_BYTES + 64 + AT_ROWS * 4;
  static bool configured = false;
  if (!configured) {
    HERO_CUDA_CHECK(cudaFuncSetAttribute(attn_tc_bwd_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  if (n_short > 0) {
    dim3 grid(n_short, heads);
    HERO_CUDA_CHECK(launch_pdl(attn_tc_bwd_kernel, grid, dim3(AT_BWD_THREADS), smem,
                               reinterpret_cast<cudaStream_t>(stream), tq, td, to, a, lse,
                               reinterpret_cast<__nv_bfloat16*>(dqkv), dbias));
  }
  if (n_long > 0) {
    const int lsm = long_smem_bytes(max_long);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    HERO_CUDA_CHECK(cudaFuncSetAttribute(attn_long_q_kernel<1>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, lsm));
    HERO_CUDA_CHECK(cudaFuncSetAttribute(attn_long_kv_kernel,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, lsm));
    HERO_CUDA_CHECK(launch_pdl(attn_long_q_kernel<1>, dim3(n_long, heads), dim3(AL_THREADS), lsm, st,
                               a, n_short, reinterpret_cast<const __nv_bfloat16*>(qkv),
                               const_cast<__nv_bfloat16*>(reinterpret_cast<const __nv_bfloat16*>(ctx)),
                               const_cast<float*>(lse),
                               reinterpret_cast<const __nv_bfloat16*>(dctx),
                               reinterpret_cast<__nv_bfloat16*>(dqkv), dbias));
    HERO_CUDA_CHECK(launch_pdl(attn_long_kv_kernel, dim3(n_long, heads), dim3(AL_THREADS), lsm, st, a,
                               n_short, reinterpret_cast<const __nv_bfloat16*>(qkv),
                               reinterpret_cast<const __nv_bfloat16*>(ctx), lse,
                               reinterpret_cast<const __nv_bfloat16*>(dctx),
                               reinterpret_cast<__nv_bfloat16*>(dqkv), dbias));
  }
  return HERO_OK;
}

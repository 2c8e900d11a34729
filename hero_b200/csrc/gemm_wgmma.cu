// Persistent warp-specialised bf16 GEMM for sm_90a: TMA -> 128B-swizzled smem ring ->
// wgmma (fp32 accumulators in registers) -> fused epilogue.
//
// One CTA per SM, three warpgroups (384 threads), 128 x 128 tiles, ping-pong consumers:
//   WG0        TMA producer (one lane); the warpgroup gives its registers away (setmaxnreg 40).
//   WG1, WG2   consumers (setmaxnreg 232). Consumer WG w takes the CTA's local tiles j with
//              j = w (mod 2), each a whole 128 x 128 tile (128 fp32 accumulators per thread).
//              Main loop: per k16 step two wgmma.m64n128k16 (rows 0-63, rows 64-127) straight
//              from the smem ring, one MMA group in flight (the stage it read is released when
//              the next group has been issued). The two WGs take the tensor cores in turn: a
//              WG starts its main loop once the other has issued the previous tile's last MMAs
//              (a pair of named barriers), so one WG's epilogue runs under the other's MMAs.
//              Epilogue, per warp (16 rows in each 64-row half of the tile) and per slab (16 rows
//              x 64 bf16 columns, or 16 rows x 32 fp32 columns when the residual stream is
//              involved — always 16 x 128 B = one 2 KB swizzled smem slab), on the accumulator
//              fragment itself:
//                bias -> activation -> dropout -> residual -> pack -> smem -> TMA store
//              Everything that comes from or goes to HBM in tiles moves by TMA: the residual /
//              saved-derivative slab is prefetched one slab ahead into a warp-private smem slab
//              (its own mbarrier), outputs leave through double-buffered slabs so a store never
//              waits for the previous one to drain. No CTA-wide barrier in the epilogue.
// Pipeline: smem full/empty ring (TMA <-> MMA); each stage is consumed by the one WG that owns
// its tile. The producer runs ahead into the next tile while a consumer runs its epilogue.
// Work items (tile x k-split): a CTA's first item is blockIdx.x; the next is blockIdx.x +
// gridDim.x, ... (static), or, for grids that share the SMs with another stream's work
// (GemmShape::dynamic, the DYN instantiation), claimed by the producer lane from a per-stream device counter as the
// current item's loads start and passed to the eight consumer warps through a small smem ring
// (item index, or -1 = no more work). A CTA that reaches an SM late, because a grid on another stream still holds
// it, then takes fewer items instead of stretching the grid by its full static share.
//
// Wide form (BN = 256, the long-K GEMMs): 128 x 256 tiles, cooperative consumers. Both WGs take
// every tile; WG w issues one wgmma.m64n256k16 per k16 step into rows 64w..64w+63 (again 128
// accumulators per thread), so both read the same stage (empty barrier: 8 warp arrivals) and no
// turn-taking is needed. The epilogue is the same per-slab code over the warp's 16 rows x 256
// columns. Per 64-deep k-block the SM's shared memory then carries 48 KB of TMA writes and 80 KB
// of operand reads for 1 024 tensor-core cycles (128 B/clk), against 32 KB + 48 KB for 512 cycles
// (160 B/clk) with two m64n128k16 per step; but the tensor cores idle through the epilogue, which
// only pays where the main loop is long (DESIGN §4, "Two tilings").
//
// Replaces the cuBLAS calls behind nn.Linear in model/layers.py:125-127,176,237,251,
// model/embed.py:112 and model/layers.py:82-90 (reference), forward and backward.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <vector>

#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int BLOCK_M = 128;
// Tile width of the ping-pong form. A consumer thread holds the whole 128 x 128 tile's fragment
// (128 fp32 accumulators) beside the fused epilogue's working set within its 232 registers; in
// the wide form (BN = 256) the same 128 accumulators hold a 64 x 256 half tile.
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 bytes = one swizzle span
constexpr int WG_K = 16;      // K of one wgmma
constexpr int NUM_EPI_WARPS = 8;                       // = the consumer warps (WG1, WG2)
constexpr int NUM_THREADS = 3 * 128;                   // producer WG + two consumer WGs
constexpr int PRODUCER_REGS = 40;                      // 40 * 128 + 232 * 256 <= 64 K registers
constexpr int CONSUMER_REGS = 232;
constexpr int SLAB_ROWS = 16;                          // rows of a warp's accumulator fragment
constexpr int SLAB_BYTES = SLAB_ROWS * 128;            // 16 rows x 128 B, swizzle-128B
constexpr int SMEM_LIMIT = 232448;                     // 227 KB opt-in dynamic shared memory per CTA
constexpr int SCHED_SLOTS = 4;                         // work-item ring, producer -> consumer warps

// ACT_CE / ACT_CE_GRAD: the LM-head of the MLM task (model/layers.py:330-354 + the cross entropy of
// model/encoder.py:370-372) without materialising fp32 logits: the forward epilogue reduces every
// 64-column slab of a row to (max, sum exp) partials + the label's logit, the backward epilogue
// turns the recomputed logits into g * (softmax - onehot) in bf16.
enum { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2, ACT_GELU_GRAD = 3, ACT_CE = 4, ACT_CE_GRAD = 5 };
enum { OUT_BF16 = 0, OUT_F32_ATOMIC = 1, OUT_F32 = 2, OUT_NONE = 3 };
// RES_F32_LN: the fp32 residual is given in its pre-LayerNorm form — the epilogue applies
// (r - mean[row]) * rstd[row] * gamma[col] + beta[col] itself, so the LayerNorm kernel that feeds the
// next GEMM never has to write an fp32 copy of its output
enum { RES_NONE = 0, RES_BF16 = 1, RES_F32 = 2, RES_F32_LN = 3 };

struct GemmShape {
  int M, N, K;
  int num_m_blocks, num_n_blocks, k_splits, k_blocks;
  // 1, or 3 = split-bf16 operands: A = A_hi + A_lo, B = B_hi + B_lo, accumulate A_hi B_hi +
  // A_lo B_hi + A_hi B_lo into the same fp32 accumulator (~16 mantissa bits per operand): the
  // frame_transform pre-activation, whose ReLU gate flips on bf16 operand rounding
  int k_passes;
  // 1: CTAs claim items from the stream's counter (grids that share the SMs with another
  // stream's work); 0: CTA b takes items b, b + gridDim.x, ... Selects the kernel's DYN form.
  int dynamic;
};

struct GemmEpilogue {
  const float* bias;
  const float* ln_mean;    // RES_F32_LN: per-row statistics and per-column affine of the residual
  const float* ln_rstd;
  const float* ln_gamma;
  const float* ln_beta;
  // ACT_CE / ACT_CE_GRAD
  const int32_t* ce_label;   // [M] target column of each row
  float2* ce_partial;        // [ceil(N / 64)][ce_ld] (max, sum exp) per (slab, row)
  float* ce_lab;             // [M] logit of the label column
  const float* ce_lse;       // [M] log-sum-exp of the row (backward)
  const float* ce_g;         // [M] upstream gradient of the row's loss (backward)
  long long ce_ld;
  int ce_n_valid;            // columns >= this are vocabulary padding: excluded / zero gradient
  int has_aux;
  float* colsum;       // OUT_BF16: column sums of the stored rows accumulate here (may be NULL)
  void* out;           // OUT_F32_ATOMIC only
  long long ld_out;
  uint32_t drop_threshold;
  uint32_t drop_key;
  float drop_scale;
};

template <int ACT, int OUT, int RES, int BN>
struct GemmCfg {
  static_assert(BN == BLOCK_N || BN == 256, "tiles are 128 x 128 (ping-pong) or 128 x 256 (wide)");
  static constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
  static constexpr int B_BYTES = BN * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  // slab width in columns: 128-byte rows of the element type that travels
  static constexpr int W = (OUT == OUT_F32 || RES == RES_F32 || RES == RES_F32_LN) ? 32 : 64;
  // staging slabs per epilogue warp: output (double buffered; the GELU / ReLU kernels, which also
  // store a second tensor, use one slab per tensor), residual operand
  static constexpr int AUX = (ACT == ACT_GELU || ACT == ACT_RELU) ? 1 : 0;
  static constexpr int N_RES_BUF = RES ? 1 : 0;
  static constexpr int BAR_BYTES = 512;
  static constexpr int stages_with(int slabs_per_warp) {
    return (SMEM_LIMIT - NUM_EPI_WARPS * slabs_per_warp * SLAB_BYTES - BAR_BYTES) / STAGE_BYTES;
  }
  // a second output slab only where it leaves the operand pipeline at least 4 stages deep
  static constexpr int N_OUT_BUF =
      (OUT == OUT_F32_ATOMIC || OUT == OUT_NONE) ? 0
                                                 : ((!AUX && stages_with(2 + N_RES_BUF) >= 4) ? 2 : 1);
  static constexpr int SLABS_PER_WARP = N_OUT_BUF + AUX + N_RES_BUF;
  static constexpr int STAGING_BYTES = NUM_EPI_WARPS * SLABS_PER_WARP * SLAB_BYTES;
  static constexpr int MAX_STAGES = stages_with(SLABS_PER_WARP);
  static constexpr int STAGES = MAX_STAGES > 6 ? 6 : MAX_STAGES;
  static constexpr int STAGING_OFFSET = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFFSET = STAGING_OFFSET + STAGING_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFFSET + BAR_BYTES;
  static_assert(STAGES >= 3, "not enough shared memory for a 3-stage pipeline");
  static_assert(SMEM_BYTES <= SMEM_LIMIT, "shared memory budget exceeded");
  // stage full / empty, residual (one per epilogue warp), work-item full / empty, item indices
  static_assert((2 * STAGES + NUM_EPI_WARPS + 2 * SCHED_SLOTS) * 8 + SCHED_SLOTS * 4 <= BAR_BYTES,
                "barrier area too small");
};

// byte offset of byte `b` of row `r` in a 128-byte-swizzled slab (16-byte unit u stored at u ^ (r & 7))
__device__ __forceinline__ uint32_t slab_off(int r, int b) {
  return r * 128 + ((((b >> 4) ^ (r & 7))) << 4) + (b & 15);
}

template <int A_MN, int B_MN, int ACT, int OUT, int RES, int BN, bool DYN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                  const __grid_constant__ CUtensorMap tmap_b,
                  const __grid_constant__ CUtensorMap tmap_out,
                  const __grid_constant__ CUtensorMap tmap_aux,
                  const __grid_constant__ CUtensorMap tmap_res,
                  const __grid_constant__ CUtensorMap tmap_a_lo,
                  const __grid_constant__ CUtensorMap tmap_b_lo, const GemmShape s,
                  const GemmEpilogue e, uint32_t* __restrict__ sched) {
  using Cfg = GemmCfg<ACT, OUT, RES, BN>;
  constexpr bool WIDE = (BN == 256);
  constexpr int STAGES = Cfg::STAGES;
  constexpr int W = Cfg::W;
  constexpr int NSLAB = BN / W;
  constexpr int NV = W / 2;   // fragment values of one slab per thread
  // 64-row halves of a tile that one consumer WG holds: the whole tile (ping-pong), or its own
  // half (wide: WG w owns rows 64w..64w+63)
  constexpr int NHALF = WIDE ? 1 : 2;
  static_assert(!(ACT == ACT_GELU || ACT == ACT_RELU || ACT == ACT_GELU_GRAD) || W == 64,
                "activation epilogues use 64-column bf16 slabs");
  static_assert(ACT != ACT_GELU_GRAD || RES == RES_BF16, "GELU' multiplier arrives as a bf16 slab");
  static_assert(OUT != OUT_F32_ATOMIC || RES == RES_NONE, "split-K accumulation takes no residual");
  static_assert((ACT == ACT_CE) == (OUT == OUT_NONE), "the CE forward epilogue stores no tile");
  static_assert(RES == RES_NONE || OUT == OUT_BF16 || OUT == OUT_F32,
                "the residual slab is refilled after the staged store of the previous slab");

  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();  // swizzle-128B atoms need a 1024 B aligned base
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::BAR_OFFSET);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* res_bar = bars + 2 * STAGES;                     // one per epilogue warp
  uint64_t* item_full = res_bar + NUM_EPI_WARPS;             // work-item ring
  uint64_t* item_empty = item_full + SCHED_SLOTS;
  int* item_ring = reinterpret_cast<int*>(item_empty + SCHED_SLOTS);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (OUT != OUT_F32_ATOMIC && OUT != OUT_NONE) tma_prefetch_desc(&tmap_out);
    if (RES) tma_prefetch_desc(&tmap_res);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      // one arrive per warp of the consumer WG that owns the tile (wide: of both WGs)
      mbar_init(&empty_bar[i], WIDE ? 8 : 4);
    }
    for (int i = 0; i < NUM_EPI_WARPS; ++i) mbar_init(&res_bar[i], 1);
    for (int i = 0; i < SCHED_SLOTS; ++i) {
      mbar_init(&item_full[i], 1);
      mbar_init(&item_empty[i], NUM_EPI_WARPS);   // every consumer warp reads every item
    }
    fence_barrier_init();
  }
  __syncthreads();
  // everything above overlapped the tail of the previous kernel (PDL); from here on we touch its
  // outputs. Let the next kernel start its own prologue right away.
  pdl_wait();
  pdl_launch_dependents();

  const int total_tiles = s.num_m_blocks * s.num_n_blocks * s.k_splits;

  if (warp < 4) {
    // ------------------------------------------------------------- TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      // A CTA's first item is its blockIdx.x; claim c on sched[0] is item gridDim.x + c, and a
      // claim past the end stops the CTA, so every CTA overshoots exactly once. sched[1] counts
      // CTAs that have stopped. Both are zero when the grid starts: the previous launch on this
      // stream left them so, and pdl_wait() above has made its writes visible. The next item is
      // claimed as the current one starts, so the atomic's round trip hides behind its loads.
      uint32_t next = blockIdx.x;
      uint32_t it = 0;
      for (uint32_t j = 0;; ++j) {
        const int tile = next < (uint32_t)total_tiles ? (int)next : -1;
        if constexpr (DYN) {
          const uint32_t slot = j % SCHED_SLOTS;
          mbar_wait(&item_empty[slot], ((j / SCHED_SLOTS) & 1u) ^ 1u);
          item_ring[slot] = tile;
          mbar_arrive(&item_full[slot]);
        }
        if (tile < 0) break;
        next = DYN ? gridDim.x + atomicAdd(&sched[0], 1u) : next + gridDim.x;
        const int ks = tile % s.k_splits;
        const int t2 = tile / s.k_splits;
        const int n_blk = t2 % s.num_n_blocks;
        const int m_blk = t2 / s.num_n_blocks;
        const int kb0 = ks * s.k_blocks / s.k_splits;
        const int kb1 = (ks + 1) * s.k_blocks / s.k_splits;
        for (int pass = 0; pass < s.k_passes; ++pass) {
          // split-bf16 passes: (A_hi, B_hi), (A_lo, B_hi), (A_hi, B_lo)
          const CUtensorMap* ma = (pass == 1) ? &tmap_a_lo : &tmap_a;
          const CUtensorMap* mb = (pass == 2) ? &tmap_b_lo : &tmap_b;
          for (int kb = kb0; kb < kb1; ++kb, ++it) {
            const uint32_t stage = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1u;
            mbar_wait(&empty_bar[stage], ph ^ 1u);
            uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
            uint8_t* sb = sa + Cfg::A_BYTES;
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
            if (A_MN)
              tma_load_3d(sa, ma, &full_bar[stage], 0, kb * BLOCK_K, m_blk * (BLOCK_M / 64));
            else
              tma_load_2d(sa, ma, &full_bar[stage], kb * BLOCK_K, m_blk * BLOCK_M);
            if (B_MN)
              tma_load_3d(sb, mb, &full_bar[stage], 0, kb * BLOCK_K, n_blk * (BN / 64));
            else
              tma_load_2d(sb, mb, &full_bar[stage], kb * BLOCK_K, n_blk * BN);
          }
        }
      }
      // the last CTA to stop claiming returns the counter to zero for the next launch
      if (DYN) __threadfence();
      if (DYN && atomicAdd(&sched[1], 1u) == gridDim.x - 1) {
        __threadfence();
        sched[0] = 0u;
        sched[1] = 0u;
      }
    }
  } else {
    // ------------------------------------------------------------- consumer warpgroups
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = warp - 4;            // consumer warp 0..7: staging slabs, residual mbarrier
    const int wg = cw >> 2;             // 0 = WG1, 1 = WG2
    // this warp's 16 rows in each 64-row half the WG holds, from the tile's first row
    const int row_off = (WIDE ? wg * 64 : 0) + (cw & 3) * SLAB_ROWS;
    const int fr = lane >> 2;          // fragment rows fr, fr + 8 of the warp's 16
    const int fc = (lane & 3) * 2;     // fragment columns 8j + fc, 8j + fc + 1
    uint8_t* stage0 = smem + Cfg::STAGING_OFFSET + cw * Cfg::SLABS_PER_WARP * SLAB_BYTES;
    uint8_t* out_slab = stage0;                                            // N_OUT_BUF slabs
    uint8_t* aux_slab = stage0 + Cfg::N_OUT_BUF * SLAB_BYTES;             // AUX slab
    uint8_t* res_slab = stage0 + (Cfg::N_OUT_BUF + Cfg::AUX) * SLAB_BYTES;
    uint64_t* my_res_bar = &res_bar[cw];
    const bool has_aux = Cfg::AUX && e.has_aux;
    const bool has_bias = (e.bias != nullptr);
    // K-major: 8-row groups 1024 B apart (SBO), LBO unused (encoded 1).
    // MN-major: 64-element MN chunks BLOCK_K*128 B apart (LBO), 8-k groups 1024 B apart (SBO).
    // Rows 64..127 of A start 8 KB into the stage in both layouts; so do columns 64.. of B, and
    // an N = 256 wgmma reads all four 64-column chunks through the same descriptor.
    constexpr uint32_t A_LBO = A_MN ? BLOCK_K * 128 : 16;
    constexpr uint32_t B_LBO = B_MN ? BLOCK_K * 128 : 16;
    constexpr uint32_t A_KSTEP = A_MN ? WG_K * 128 : WG_K * 2;
    constexpr uint32_t B_KSTEP = B_MN ? WG_K * 128 : WG_K * 2;
    // main-loop turns: WG w waits on barrier 1 + w, the other WG arrives on it (2 x 128 threads)
    const int my_turn_bar = 1 + wg, other_turn_bar = 2 - wg;
    uint32_t res_phase = 0;
    uint32_t out_it = 0;
    uint32_t it = 0;   // ring position; advances over the other WG's k-blocks too
    float acc[NHALF][BN / 2];   // ping-pong: rows 0-63, rows 64-127 of the tile; wide: own half
    // the CTA's j-th work item: by stride, or as the producer claimed it
    auto next_item = [&](uint32_t j) -> int {
      if constexpr (!DYN) {
        const uint32_t t = blockIdx.x + j * gridDim.x;
        return t < (uint32_t)total_tiles ? (int)t : -1;
      }
      const uint32_t slot = j % SCHED_SLOTS;
      mbar_wait(&item_full[slot], (j / SCHED_SLOTS) & 1u);
      const int t = *reinterpret_cast<volatile int*>(&item_ring[slot]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&item_empty[slot]);
      return t;
    };

    uint32_t j = 0;   // local item index
    for (int tile = next_item(0); tile >= 0; ++j) {
      const int ks = tile % s.k_splits;
      const int t2 = tile / s.k_splits;
      const int n_blk = t2 % s.num_n_blocks;
      const int m_blk = t2 / s.num_n_blocks;
      const int kb0 = ks * s.k_blocks / s.k_splits;
      const int kb1 = (ks + 1) * s.k_blocks / s.k_splits;
      const int n_kb = (kb1 - kb0) * s.k_passes;
      if (!WIDE && (int)(j & 1u) != wg) {   // the other WG's tile
        it += n_kb;
        tile = next_item(j + 1);
        continue;
      }
      const int col_base = n_blk * BN;
      // the tile's first residual slab travels while the main loop runs
      if (RES && lane == 0) {
        mbar_arrive_expect_tx(my_res_bar, SLAB_BYTES);
        tma_load_2d(res_slab, &tmap_res, my_res_bar, col_base, m_blk * BLOCK_M + row_off);
      }

      // wait for the other WG to have issued the previous tile's main loop
      if (!WIDE && j > 0) named_bar_sync(my_turn_bar, 256);
      uint32_t prev_stage = 0;
      for (int kbi = 0; kbi < n_kb; ++kbi, ++it) {
        const uint32_t stage = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1u;
        mbar_wait(&full_bar[stage], ph);
        const uint32_t sa = smem_u32(smem + stage * Cfg::STAGE_BYTES);
        const uint32_t sb = sa + Cfg::A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k) {
          const uint64_t bdesc = make_sw128_desc(sb + k * B_KSTEP, B_LBO, 1024);
          const uint32_t scale_d = (kbi > 0 || k > 0) ? 1u : 0u;
          if constexpr (WIDE) {
            wgmma_m64n256k16<A_MN, B_MN>(
                acc[0], make_sw128_desc(sa + wg * 8192 + k * A_KSTEP, A_LBO, 1024), bdesc, scale_d);
          } else {
            wgmma_m64n128k16<A_MN, B_MN>(acc[0], make_sw128_desc(sa + k * A_KSTEP, A_LBO, 1024),
                                         bdesc, scale_d);
            wgmma_m64n128k16<A_MN, B_MN>(
                acc[1], make_sw128_desc(sa + 8192 + k * A_KSTEP, A_LBO, 1024), bdesc, scale_d);
          }
        }
        wgmma_commit();
        // the previous k-block's MMAs have retired once at most this group is pending
        wgmma_wait<1>();
        if (kbi > 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
      }
      // every MMA of this tile is issued: the other WG's next tile may take the tensor cores
      // (only if it has one, so that every arrive meets a sync). The producer has issued this
      // tile's last loads, so it is claiming or has claimed the next item.
      const int next_tile = next_item(j + 1);
      if (!WIDE && next_tile >= 0) named_bar_arrive(other_turn_bar, 256);
      wgmma_wait<0>();
#pragma unroll
      for (int half = 0; half < NHALF; ++half) wgmma_fence_acc(acc[half]);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      // ------------------------------------------------------------- epilogue
#pragma unroll
      for (int half = 0; half < NHALF; ++half) {
        const int row0 = m_blk * BLOCK_M + half * 64 + row_off;   // first row of this warp's slabs
        const int ra = row0 + fr, rb = ra + 8;
        const bool ra_ok = ra < s.M, rb_ok = rb < s.M;
        int lab_a = -1, lab_b = -1;
        float lse_a = 0.f, lse_b = 0.f, g_a = 0.f, g_b = 0.f;
        if (ACT == ACT_CE || ACT == ACT_CE_GRAD) {
          if (ra_ok) lab_a = __ldg(e.ce_label + ra);
          if (rb_ok) lab_b = __ldg(e.ce_label + rb);
          if (ACT == ACT_CE_GRAD) {
            if (ra_ok) { lse_a = __ldg(e.ce_lse + ra); g_a = __ldg(e.ce_g + ra); }
            if (rb_ok) { lse_b = __ldg(e.ce_lse + rb); g_b = __ldg(e.ce_g + rb); }
          }
        }
        float lsc_a = 0.f, lsh_a = 0.f, lsc_b = 0.f, lsh_b = 0.f;   // (r - mean) * rstd
        if (RES == RES_F32_LN) {
          if (ra_ok) { lsc_a = __ldg(e.ln_rstd + ra); lsh_a = -__ldg(e.ln_mean + ra) * lsc_a; }
          if (rb_ok) { lsc_b = __ldg(e.ln_rstd + rb); lsh_b = -__ldg(e.ln_mean + rb) * lsc_b; }
        }
#pragma unroll
        for (int c = 0; c < NSLAB; ++c) {
          const int col0 = col_base + c * W;
          if (col0 >= s.N) break;  // warp-uniform
          // v[4jj + 2h + x] = (row fr + 8h, column col0 + 8jj + fc + x). The accumulator is
          // cleared as it is read: the next tile's first MMA ignores it (scale-d 0), but to the
          // compiler it is an input, and 128 live accumulators beside the epilogue would spill.
          float v[NV];
#pragma unroll
          for (int q = 0; q < NV; ++q) {
            v[q] = acc[half][c * NV + q];
            acc[half][c * NV + q] = 0.f;
          }
          if (has_bias) {
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj) {
              const int col = col0 + 8 * jj + fc;
              if (col < s.N) {
                const float2 b = __ldg(reinterpret_cast<const float2*>(e.bias + col));
                v[4 * jj] += b.x; v[4 * jj + 1] += b.y; v[4 * jj + 2] += b.x; v[4 * jj + 3] += b.y;
              }
            }
          }
          // residual / saved-derivative slab (requested one slab ago) -> registers; the next one is
          // requested once these values have been used (below)
          uint32_t opnd[NV];   // bf16 pairs (W = 64: NV / 2 used) or fp32 bits (W = 32)
          if (RES) {
            mbar_wait(my_res_bar, res_phase);
            res_phase ^= 1u;
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = fr + 8 * h;
                if (W == 64) {
                  opnd[2 * jj + h] =
                      *reinterpret_cast<const uint32_t*>(res_slab + slab_off(r, (8 * jj + fc) * 2));
                } else {
                  const uint2 u =
                      *reinterpret_cast<const uint2*>(res_slab + slab_off(r, (8 * jj + fc) * 4));
                  opnd[4 * jj + 2 * h] = u.x;
                  opnd[4 * jj + 2 * h + 1] = u.y;
                }
              }
          }
          // activation (compile-time); the training FFN-up also emits gelu'(x) through its own slab
          if constexpr (ACT == ACT_GELU) {
            if (has_aux) {
              if (lane == 0) bulk_wait_read<1>();   // the aux slab's previous store (two groups back)
              __syncwarp();
#pragma unroll
              for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  float d0, d1;
                  v[4 * jj + 2 * h] = gelu_erf_with_grad(v[4 * jj + 2 * h], d0);
                  v[4 * jj + 2 * h + 1] = gelu_erf_with_grad(v[4 * jj + 2 * h + 1], d1);
                  *reinterpret_cast<uint32_t*>(aux_slab + slab_off(fr + 8 * h, (8 * jj + fc) * 2)) =
                      pack_bf16x2(d0, d1);
                }
              fence_proxy_async();
              __syncwarp();
              if (lane == 0) {
                tma_store_2d(&tmap_aux, aux_slab, col0, row0);
                bulk_commit();
              }
            } else {
#pragma unroll
              for (int q = 0; q < NV; ++q) v[q] = gelu_erf(v[q]);
            }
          } else if constexpr (ACT == ACT_RELU) {
            if (has_aux) {   // pre-activation copy (the ReLU backward needs its sign)
              if (lane == 0) bulk_wait_read<1>();
              __syncwarp();
#pragma unroll
              for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                  *reinterpret_cast<uint32_t*>(aux_slab + slab_off(fr + 8 * h, (8 * jj + fc) * 2)) =
                      pack_bf16x2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1]);
              fence_proxy_async();
              __syncwarp();
              if (lane == 0) {
                tma_store_2d(&tmap_aux, aux_slab, col0, row0);
                bulk_commit();
              }
            }
#pragma unroll
            for (int q = 0; q < NV; ++q) v[q] = fmaxf(v[q], 0.0f);
          } else if constexpr (ACT == ACT_CE) {
            // online-softmax partials of each row over the slab's valid columns: the four lanes of a
            // quad hold a row's columns
            float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int x = 0; x < 2; ++x)
                if (col0 + 8 * jj + fc + x < e.ce_n_valid) {
                  m[0] = fmaxf(m[0], v[4 * jj + x]);
                  m[1] = fmaxf(m[1], v[4 * jj + 2 + x]);
                }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
              m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
            }
            float ssum[2] = {0.f, 0.f};
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int x = 0; x < 2; ++x)
                if (col0 + 8 * jj + fc + x < e.ce_n_valid) {
                  ssum[0] += fast_ex2((v[4 * jj + x] - m[0]) * 1.4426950408889634f);
                  ssum[1] += fast_ex2((v[4 * jj + 2 + x] - m[1]) * 1.4426950408889634f);
                }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              ssum[h] += __shfl_xor_sync(0xffffffffu, ssum[h], 1);
              ssum[h] += __shfl_xor_sync(0xffffffffu, ssum[h], 2);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = h ? rb : ra;
              if (!(h ? rb_ok : ra_ok)) continue;
              if (fc == 0) e.ce_partial[(long long)(col0 / W) * e.ce_ld + row] = make_float2(m[h], ssum[h]);
              const int rel = (h ? lab_b : lab_a) - col0;
#pragma unroll
              for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
                for (int x = 0; x < 2; ++x)
                  if (rel == 8 * jj + fc + x) e.ce_lab[row] = v[4 * jj + 2 * h + x];
            }
          } else if constexpr (ACT == ACT_CE_GRAD) {
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int x = 0; x < 2; ++x) {
                  const int j = 8 * jj + fc + x;
                  const int q = 4 * jj + 2 * h + x;
                  float p = fast_ex2((v[q] - (h ? lse_b : lse_a)) * 1.4426950408889634f);
                  p = (j == (h ? lab_b : lab_a) - col0) ? p - 1.0f : p;
                  v[q] = (col0 + j < e.ce_n_valid) ? p * (h ? g_b : g_a) : 0.f;
                }
          } else if constexpr (ACT == ACT_GELU_GRAD) {   // multiply by the saved activation derivative
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float2 x = unpack_bf16x2(opnd[2 * jj + h]);
                v[4 * jj + 2 * h] *= x.x;
                v[4 * jj + 2 * h + 1] *= x.y;
              }
          }
          if (e.drop_threshold != 0u) {
            // one hash per even/odd column pair: low half -> even, high half -> odd (dropout_keep)
            const uint32_t t16 = e.drop_threshold >> 16;
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const uint32_t idx = (uint32_t)(h ? rb : ra) * (uint32_t)s.N + (uint32_t)(col0 + 8 * jj + fc);
                const uint32_t hh = hash_u32(e.drop_key, idx >> 1);
                const int q = 4 * jj + 2 * h;
                v[q] = ((hh & 0xFFFFu) >= t16) ? v[q] * e.drop_scale : 0.0f;
                v[q + 1] = ((hh >> 16) >= t16) ? v[q + 1] * e.drop_scale : 0.0f;
              }
          }
          if constexpr (RES == RES_F32) {
#pragma unroll
            for (int q = 0; q < NV; ++q) v[q] += __uint_as_float(opnd[q]);
          } else if constexpr (RES == RES_F32_LN) {
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj) {
              const int col = col0 + 8 * jj + fc;
              float2 ga = make_float2(0.f, 0.f), be = make_float2(0.f, 0.f);
              if (col < s.N) {
                ga = __ldg(reinterpret_cast<const float2*>(e.ln_gamma + col));
                be = __ldg(reinterpret_cast<const float2*>(e.ln_beta + col));
              }
              const int q = 4 * jj;
              v[q] += fmaf(fmaf(__uint_as_float(opnd[q]), lsc_a, lsh_a), ga.x, be.x);
              v[q + 1] += fmaf(fmaf(__uint_as_float(opnd[q + 1]), lsc_a, lsh_a), ga.y, be.y);
              v[q + 2] += fmaf(fmaf(__uint_as_float(opnd[q + 2]), lsc_b, lsh_b), ga.x, be.x);
              v[q + 3] += fmaf(fmaf(__uint_as_float(opnd[q + 3]), lsc_b, lsh_b), ga.y, be.y);
            }
          } else if constexpr (RES == RES_BF16 && ACT != ACT_GELU_GRAD) {
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float2 x = unpack_bf16x2(opnd[2 * jj + h]);
                v[4 * jj + 2 * h] += x.x;
                v[4 * jj + 2 * h + 1] += x.y;
              }
          }
          if constexpr (OUT == OUT_NONE) {
            // nothing to store
          } else if constexpr (OUT == OUT_F32_ATOMIC) {
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int col = col0 + 8 * jj + fc;
                if ((h ? rb_ok : ra_ok) && col < s.N) {
                  float* o = reinterpret_cast<float*>(e.out) + (long long)(h ? rb : ra) * e.ld_out + col;
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(o),
                               "f"(v[4 * jj + 2 * h]), "f"(v[4 * jj + 2 * h + 1])
                               : "memory");
                }
              }
          } else {
            // stage the slab in swizzled smem and let TMA write full 128 B rows. Output slabs are
            // double buffered: only the store issued two slabs ago must have finished READING smem
            // (bulk groups complete in order; with an aux store per slab the distance is the same).
            // (a GELU / ReLU kernel that stores no second tensor uses that tensor's slab as its
            // second output buffer: the slabs are adjacent)
            const bool two_bufs = (Cfg::N_OUT_BUF == 2) || (Cfg::AUX && !has_aux);
            uint8_t* slab = out_slab + (two_bufs ? (out_it & 1u) * SLAB_BYTES : 0);
            if (lane == 0) {
              // one group may stay in flight when it reads another slab (the other output buffer,
              // or this slab's derivative store); a lone slab must have drained
              if (two_bufs || has_aux) bulk_wait_read<1>(); else bulk_wait_read<0>();
            }
            __syncwarp();
#pragma unroll
            for (int jj = 0; jj < W / 8; ++jj)
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int r = fr + 8 * h, q = 4 * jj + 2 * h;
                if (OUT == OUT_F32)
                  *reinterpret_cast<float2*>(slab + slab_off(r, (8 * jj + fc) * 4)) =
                      make_float2(v[q], v[q + 1]);
                else
                  *reinterpret_cast<uint32_t*>(slab + slab_off(r, (8 * jj + fc) * 2)) =
                      pack_bf16x2(v[q], v[q + 1]);
              }
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
              tma_store_2d(&tmap_out, slab, col0, row0);
              bulk_commit();
            }
            // Every lane's residual values have now reached the slab just staged, so its reads of
            // the residual slab are complete and TMA may refill it with the next slab: this
            // half's next one, else the second half's first. (Issued right after the reads, the
            // refill could overtake shared-memory loads held back behind the other warpgroup's
            // MMA operand traffic.)
            if (RES && lane == 0) {
              if (c + 1 < NSLAB && col0 + W < s.N) {
                mbar_arrive_expect_tx(my_res_bar, SLAB_BYTES);
                tma_load_2d(res_slab, &tmap_res, my_res_bar, col0 + W, row0);
              } else if (half + 1 < NHALF) {
                mbar_arrive_expect_tx(my_res_bar, SLAB_BYTES);
                tma_load_2d(res_slab, &tmap_res, my_res_bar, col_base, row0 + 64);
              }
            }
            if constexpr (OUT == OUT_BF16 && W == 64) {
              // column sums of the slab just staged (bf16, as stored): lane l owns columns
              // 2l, 2l + 1 = word l of every 128-byte row (conflict-free), rows past M excluded
              if (e.colsum != nullptr) {
                const int rmax = min(SLAB_ROWS, s.M - row0);       // warp-uniform
                float sx = 0.f, sy = 0.f;
                const int u = lane >> 2, w4 = (lane & 3) * 4;
#pragma unroll 8
                for (int r = 0; r < rmax; ++r) {
                  const float2 x = unpack_bf16x2(
                      *reinterpret_cast<const uint32_t*>(slab + r * 128 + ((u ^ (r & 7)) << 4) + w4));
                  sx += x.x;
                  sy += x.y;
                }
                const int col = col0 + 2 * lane;
                if (col < s.N && rmax > 0)
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(e.colsum + col), "f"(sx),
                               "f"(sy)
                               : "memory");
              }
            }
            ++out_it;
          }
        }
      }
      tile = next_tile;
    }
    // the slabs must not go away under stores still reading them; their global writes are
    // complete when the grid is (a dependent kernel's griddepcontrol.wait covers them)
    if (OUT != OUT_F32_ATOMIC && OUT != OUT_NONE && lane == 0) bulk_wait_read<0>();
  }
}

// ------------------------------------------------------------------ host side: tensor maps
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) !=
          cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  return fn;
}

// Tensor maps are pure functions of (pointer, extents, leading dimension, box, kind), and the
// training loop presents the same few hundred combinations every step (weights never move;
// activation workspaces come back from the caching allocator at the same addresses): a small
// direct-mapped cache replaces ~400 cuTensorMapEncodeTiled calls per step with lookups.
enum { TM_KMAJOR = 0, TM_MNMAJOR = 1, TM_SLAB_BF16 = 2, TM_SLAB_F32 = 3 };
struct TmapKey {
  const void* ptr;
  long long ld;
  int d0, d1, box, kind;
  bool operator==(const TmapKey& o) const {
    return ptr == o.ptr && ld == o.ld && d0 == o.d0 && d1 == o.d1 && box == o.box && kind == o.kind;
  }
};
struct TmapEntry {
  TmapKey key;
  bool valid;
  CUtensorMap map;
};
constexpr int TMAP_CACHE_SIZE = 4096;   // entries (power of two)

static int encode_uncached(CUtensorMap* map, const TmapKey& k) {
  auto fn = get_encode_fn();
  if (!fn) return set_error(HERO_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  CUresult r;
  if (k.kind == TM_KMAJOR) {
    // global [rows = d0, k = d1] row-major (ld elements); box = 64 k x box rows
    cuuint64_t dims[2] = {(cuuint64_t)k.d1, (cuuint64_t)k.d0};
    cuuint64_t strides[1] = {(cuuint64_t)k.ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)k.box};
    cuuint32_t estr[2] = {1, 1};
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(k.ptr), dims, strides, box,
           estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else if (k.kind == TM_MNMAJOR) {
    // global [k = d0, mn = d1] row-major (ld elements), viewed as (64, k, mn/64) so one box
    // (64, BLOCK_K, box/64) lands in smem as consecutive [BLOCK_K x 128 B] swizzle-128B chunks
    cuuint64_t dims[3] = {64, (cuuint64_t)k.d0, (cuuint64_t)(k.d1 / 64)};
    cuuint64_t strides[2] = {(cuuint64_t)k.ld * 2, 128};
    cuuint32_t box[3] = {64, (cuuint32_t)BLOCK_K, (cuuint32_t)(k.box / 64)};
    cuuint32_t estr[3] = {1, 1, 1};
    r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(k.ptr), dims, strides, box,
           estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    // epilogue slab over a row-major [rows = d0, cols = d1] matrix: 16 rows x 128 bytes
    const bool f32 = (k.kind == TM_SLAB_F32);
    cuuint64_t dims[2] = {(cuuint64_t)k.d1, (cuuint64_t)k.d0};
    cuuint64_t strides[1] = {(cuuint64_t)k.ld * (f32 ? 4 : 2)};
    cuuint32_t box[2] = {(cuuint32_t)(f32 ? 32 : 64), (cuuint32_t)SLAB_ROWS};
    cuuint32_t estr[2] = {1, 1};
    r = fn(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
           const_cast<void*>(k.ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS)
    return set_error(HERO_ERR_CUDA, "cuTensorMapEncodeTiled(kind %d, %d x %d, ld %lld) failed: %d",
                     k.kind, k.d0, k.d1, k.ld, (int)r);
  return HERO_OK;
}

static int get_tmap(CUtensorMap* out, const void* ptr, int d0, int d1, long long ld, int box,
                    int kind) {
  static thread_local std::vector<TmapEntry> cache;
  if (cache.empty()) {
    cache.resize(TMAP_CACHE_SIZE);
    for (auto& en : cache) en.valid = false;
  }
  TmapKey k;
  memset(&k, 0, sizeof(k));
  k.ptr = ptr; k.ld = ld; k.d0 = d0; k.d1 = d1; k.box = box; k.kind = kind;
  uint64_t h = reinterpret_cast<uintptr_t>(ptr) >> 4;
  h ^= (uint64_t)d0 * 0x9E3779B97F4A7C15ull;
  h ^= ((uint64_t)d1 << 21) ^ ((uint64_t)box << 7) ^ (uint64_t)kind ^ ((uint64_t)ld << 40);
  h *= 0xD6E8FEB86659FD93ull;
  h ^= h >> 32;
  TmapEntry& en = cache[h & (TMAP_CACHE_SIZE - 1)];
  if (!(en.valid && en.key == k)) {
    if (int rc = encode_uncached(&en.map, k)) {
      en.valid = false;
      return rc;
    }
    en.key = k;
    en.valid = true;
  }
  *out = en.map;
  return HERO_OK;
}

struct GemmMaps {
  CUtensorMap a, b, out, aux, res, a_lo, b_lo;
};

// Work-item counters of the dynamic scheduler: two uint32 per (device, stream), claims and
// retired CTAs. A launch finds them at zero and leaves them at zero (its last CTA resets them), so
// launches need no memset and no host sync; launches on one stream are ordered by the stream and
// pdl_wait(), and streams never share a counter, so concurrent grids do not interfere. A pair is
// zeroed once, on its stream, when that stream first launches a GEMM.
struct SchedSlot {
  int device;
  cudaStream_t stream;
  uint32_t* counter;
};
constexpr int SCHED_CHUNK = 256;   // counter pairs per device allocation

static int sched_counter(cudaStream_t st, uint32_t** out) {
  static std::mutex mu;
  static std::vector<SchedSlot> slots;
  static std::vector<SchedSlot> chunks;   // (device, -, base of a SCHED_CHUNK-pair allocation)
  int dev = 0;
  HERO_CUDA_CHECK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  for (const SchedSlot& sl : slots)
    if (sl.device == dev && sl.stream == st) {
      *out = sl.counter;
      return HERO_OK;
    }
  int used = 0;
  for (const SchedSlot& sl : slots) used += (sl.device == dev);
  if (used % SCHED_CHUNK == 0) {
    void* p = nullptr;
    HERO_CUDA_CHECK(cudaMalloc(&p, SCHED_CHUNK * 2 * sizeof(uint32_t)));
    chunks.push_back(SchedSlot{dev, nullptr, static_cast<uint32_t*>(p)});
  }
  uint32_t* base = nullptr;
  for (const SchedSlot& c : chunks)
    if (c.device == dev) base = c.counter;   // the newest chunk of this device
  uint32_t* counter = base + 2 * (used % SCHED_CHUNK);
  HERO_CUDA_CHECK(cudaMemsetAsync(counter, 0, 2 * sizeof(uint32_t), st));
  slots.push_back(SchedSlot{dev, st, counter});
  *out = counter;
  return HERO_OK;
}

template <int A_MN, int B_MN, int ACT, int OUT, int RES, int BN = BLOCK_N>
static int launch(const GemmMaps& tm, const GemmShape& s, const GemmEpilogue& e,
                  cudaStream_t stream) {
  using Cfg = GemmCfg<ACT, OUT, RES, BN>;
  // the static schedule is a kernel of its own, so grids that have the SMs to themselves run
  // none of the ring's code
  auto kern = s.dynamic ? gemm_wgmma_kernel<A_MN, B_MN, ACT, OUT, RES, BN, true>
                        : gemm_wgmma_kernel<A_MN, B_MN, ACT, OUT, RES, BN, false>;
  static bool attr_set[2] = {false, false};
  if (!attr_set[s.dynamic]) {
    HERO_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::SMEM_BYTES));
    attr_set[s.dynamic] = true;
  }
  const int total = s.num_m_blocks * s.num_n_blocks * s.k_splits;
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");
  uint32_t* sched = nullptr;
  if (s.dynamic)
    if (int rc = sched_counter(stream, &sched)) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(total < sms ? total : sms);
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = serial_profiling() ? 0 : 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  HERO_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tm.a, tm.b, tm.out, tm.aux, tm.res, tm.a_lo, tm.b_lo, s, e,
                                     sched));
  return HERO_OK;
}

// The variants with a wide (128 x 256) form: the weight gradients, the forward FFN-down / out-
// projection into the fp32 residual stream, and the dgrads with a bf16 residual (FFN-up `da`, QKV
// `dx`). Must agree with the `wide ?` choices in dispatch().
static bool has_wide_form(const hero_gemm_args* g) {
  const int layout = g->a_mn_major * 2 + g->b_mn_major;
  if (g->out_f32_accumulate) return layout == 0 || layout == 3;
  if (g->out_f32_store) return layout == 0 && g->act == ACT_NONE && g->resid != nullptr;
  return layout == 1 && g->act == ACT_NONE && g->resid != nullptr;
}

static int dispatch(const hero_gemm_args* g, const GemmMaps& tm, const GemmShape& s,
                    const GemmEpilogue& e, bool wide, cudaStream_t st) {
  const int layout = g->a_mn_major * 2 + g->b_mn_major;
  const bool res = g->resid != nullptr;
  if (g->out_f32_accumulate) {
    if (layout == 3)
      return wide ? launch<1, 1, ACT_NONE, OUT_F32_ATOMIC, RES_NONE, 256>(tm, s, e, st)
                  : launch<1, 1, ACT_NONE, OUT_F32_ATOMIC, RES_NONE>(tm, s, e, st);
    if (layout == 0)
      return wide ? launch<0, 0, ACT_NONE, OUT_F32_ATOMIC, RES_NONE, 256>(tm, s, e, st)
                  : launch<0, 0, ACT_NONE, OUT_F32_ATOMIC, RES_NONE>(tm, s, e, st);
    return set_error(HERO_ERR_INVALID, "fp32-accumulate supports layouts (0,0) and (1,1)");
  }
  if (g->out_f32_store) {
    // the residual stream: fp32 pre-LayerNorm sums (forward out-projection / FFN-down)
    if (layout == 0 && g->act == ACT_NONE) {
      if (res && g->resid_ln_mean)
        return wide ? launch<0, 0, ACT_NONE, OUT_F32, RES_F32_LN, 256>(tm, s, e, st)
                    : launch<0, 0, ACT_NONE, OUT_F32, RES_F32_LN>(tm, s, e, st);
      if (res)
        return wide ? launch<0, 0, ACT_NONE, OUT_F32, RES_F32, 256>(tm, s, e, st)
                    : launch<0, 0, ACT_NONE, OUT_F32, RES_F32>(tm, s, e, st);
      return launch<0, 0, ACT_NONE, OUT_F32, RES_NONE>(tm, s, e, st);
    }
    return set_error(HERO_ERR_INVALID, "fp32-store output supports layout (0,0), act 0 only");
  }
  if (layout == 0) {
    switch (g->act) {
      case ACT_CE:
        if (!res) return launch<0, 0, ACT_CE, OUT_NONE, RES_NONE>(tm, s, e, st);
        break;
      case ACT_CE_GRAD:
        if (!res) return launch<0, 0, ACT_CE_GRAD, OUT_BF16, RES_NONE>(tm, s, e, st);
        break;
      case ACT_NONE:
        if (res) return launch<0, 0, ACT_NONE, OUT_BF16, RES_BF16>(tm, s, e, st);
        return launch<0, 0, ACT_NONE, OUT_BF16, RES_NONE>(tm, s, e, st);
      case ACT_GELU:
        if (!res) return launch<0, 0, ACT_GELU, OUT_BF16, RES_NONE>(tm, s, e, st);
        break;
      case ACT_RELU:
        if (res) return launch<0, 0, ACT_RELU, OUT_BF16, RES_BF16>(tm, s, e, st);
        return launch<0, 0, ACT_RELU, OUT_BF16, RES_NONE>(tm, s, e, st);
      default: break;
    }
  } else if (layout == 1) {
    switch (g->act) {
      case ACT_NONE:
        if (res)
          return wide ? launch<0, 1, ACT_NONE, OUT_BF16, RES_BF16, 256>(tm, s, e, st)
                      : launch<0, 1, ACT_NONE, OUT_BF16, RES_BF16>(tm, s, e, st);
        return launch<0, 1, ACT_NONE, OUT_BF16, RES_NONE>(tm, s, e, st);
      case ACT_GELU_GRAD:
        return launch<0, 1, ACT_GELU_GRAD, OUT_BF16, RES_BF16>(tm, s, e, st);
      default: break;
    }
  }
  return set_error(HERO_ERR_INVALID,
                   "unsupported gemm variant: a_mn=%d b_mn=%d act=%d f32acc=%d f32store=%d resid=%d",
                   g->a_mn_major, g->b_mn_major, g->act, g->out_f32_accumulate, g->out_f32_store,
                   (int)res);
}

// Optional per-launch timing (bench.py roofline): CUDA events on the launching stream around every
// GEMM launch between hero_gemm_profile_begin() and hero_gemm_profile_end().
struct GemmProfileRec {
  int m, n, k, a_mn, b_mn, act, f32, block_n;
};
struct GemmProfile {
  bool on = false;
  std::vector<cudaEvent_t> ev;   // pairs
  std::vector<cudaEvent_t> pool; // recycled events
  std::vector<GemmProfileRec> rec;
  double flops = 0.0;
};
static GemmProfile g_prof;

bool gemm_profile_active() { return g_prof.on; }

static thread_local bool g_shared_sms = false;
bool gemm_set_shared_sms(bool on) {
  const bool prev = g_shared_sms;
  g_shared_sms = on;
  return prev;
}

}  // namespace hero

extern "C" int hero_gemm_set_shared_sms(int32_t on) {
  hero::gemm_set_shared_sms(on != 0);
  return HERO_OK;
}

extern "C" int hero_gemm_profile_begin(void) {
  using namespace hero;
  for (cudaEvent_t e : g_prof.ev) g_prof.pool.push_back(e);
  g_prof.ev.clear();
  g_prof.rec.clear();
  g_prof.flops = 0.0;
  g_prof.on = true;
  return HERO_OK;
}

extern "C" int hero_gemm_profile_end(double* ms, double* flops, int64_t* launches) {
  using namespace hero;
  g_prof.on = false;
  double total = 0.0;
  // HERO_GEMM_PROFILE_DUMP=<path>: per-launch CSV (shape, variant, ms) for tuning
  const char* path = getenv("HERO_GEMM_PROFILE_DUMP");
  FILE* f = path ? fopen(path, "w") : nullptr;
  if (f) fprintf(f, "m,n,k,a_mn,b_mn,act,f32,block_n,ms\n");
  for (size_t i = 0; i + 1 < g_prof.ev.size(); i += 2) {
    HERO_CUDA_CHECK(cudaEventSynchronize(g_prof.ev[i + 1]));
    float t = 0.f;
    HERO_CUDA_CHECK(cudaEventElapsedTime(&t, g_prof.ev[i], g_prof.ev[i + 1]));
    total += t;
    if (f && i / 2 < g_prof.rec.size()) {
      const GemmProfileRec& r = g_prof.rec[i / 2];
      fprintf(f, "%d,%d,%d,%d,%d,%d,%d,%d,%.5f\n", r.m, r.n, r.k, r.a_mn, r.b_mn, r.act, r.f32,
              r.block_n, t);
    }
  }
  if (f) fclose(f);
  if (ms) *ms = total;
  if (flops) *flops = g_prof.flops;
  if (launches) *launches = (int64_t)(g_prof.ev.size() / 2);
  for (cudaEvent_t e : g_prof.ev) g_prof.pool.push_back(e);
  g_prof.ev.clear();
  return HERO_OK;
}

static int hero_gemm_bf16_impl(const hero_gemm_args* g, void* stream, int* bn_used);

extern "C" int hero_gemm_bf16(const hero_gemm_args* g, void* stream) {
  using namespace hero;
  if (!g_prof.on) return hero_gemm_bf16_impl(g, stream, nullptr);
  cudaEvent_t ev[2];
  for (int i = 0; i < 2; ++i) {
    if (!g_prof.pool.empty()) {
      ev[i] = g_prof.pool.back();
      g_prof.pool.pop_back();
    } else {
      HERO_CUDA_CHECK(cudaEventCreate(&ev[i]));
    }
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  HERO_CUDA_CHECK(cudaEventRecord(ev[0], st));
  int bn = 0;
  const int rc = hero_gemm_bf16_impl(g, stream, &bn);
  HERO_CUDA_CHECK(cudaEventRecord(ev[1], st));
  g_prof.ev.push_back(ev[0]);
  g_prof.ev.push_back(ev[1]);
  if (g)
    g_prof.rec.push_back(GemmProfileRec{g->m, g->n, g->k, g->a_mn_major, g->b_mn_major, g->act,
                                        g->out_f32_accumulate + 2 * g->out_f32_store, bn});
  // (a split-bf16 GEMM issues 3x the MMAs; the profile counts its algorithmic 2MNK once)
  if (rc == HERO_OK && g) g_prof.flops += 2.0 * (double)g->m * (double)g->n * (double)g->k;
  return rc;
}

static int hero_gemm_bf16_impl(const hero_gemm_args* g, void* stream, int* bn_used) {
  using namespace hero;
  HERO_REQUIRE(g != nullptr, "null args");
  HERO_REQUIRE(g->a && g->b && (g->out || g->act == ACT_CE), "null operand pointer");
  HERO_REQUIRE(g->m > 0 && g->n > 0 && g->k > 0, "empty gemm %dx%dx%d", g->m, g->n, g->k);
  HERO_REQUIRE(g->n % 8 == 0, "n must be a multiple of 8 (n=%d)", g->n);
  HERO_REQUIRE(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->ld_out % 4 == 0, "unaligned leading dim");
  HERO_REQUIRE(g->act != ACT_GELU_GRAD || g->aux_in != nullptr, "act=3 needs aux_in");
  HERO_REQUIRE(g->act != ACT_GELU_GRAD || g->resid == nullptr, "act=3 cannot take a residual");
  HERO_REQUIRE(!(g->out_f32_accumulate && g->out_f32_store), "fp32 store and accumulate exclude each other");
  HERO_REQUIRE(!g->out_f32_accumulate || (g->act == ACT_NONE && !g->resid && !g->aux_out),
               "fp32-accumulate output supports act=0 without residual only");
  HERO_REQUIRE(!g->resid || (g->resid_f32 != 0) == (g->out_f32_store != 0),
               "an fp32 residual goes with an fp32 stored output (and a bf16 one with bf16)");
  // (an MN-major A whose row count is not a multiple of 64 is accepted when its storage is: the
  // tail chunk then reads the zero padding, and rows >= m are never written)
  if (g->a_mn_major)
    HERO_REQUIRE(g->m % 64 == 0 || g->lda >= (g->m + 63) / 64 * 64,
                 "MN-major A needs m %% 64 == 0 or lda >= round_up(m, 64) (m=%d lda=%lld)", g->m,
                 (long long)g->lda);
  if (g->b_mn_major) HERO_REQUIRE(g->n % 64 == 0, "MN-major B needs n %% 64 == 0 (n=%d)", g->n);

  // block_n 128 runs the ping-pong 128 x 128 kernel, 256 the wide 128 x 256 one where the variant
  // has a wide form (else 128 x 128), 0 picks per shape. cta_pair (a Blackwell tiling) is accepted
  // and ignored.
  HERO_REQUIRE(g->block_n == 0 || g->block_n == 128 || g->block_n == 256,
               "block_n must be 0, 128 or 256");
  const int sms = sm_count();
  if (sms <= 0) return set_error(HERO_ERR_NO_DEVICE, "no CUDA device");

  GemmShape s;
  s.M = g->m; s.N = g->n; s.K = g->k;
  s.num_m_blocks = ceil_div(g->m, BLOCK_M);
  s.k_blocks = ceil_div(g->k, BLOCK_K);
  // Tiling and split-K count minimise a cost in units of one 64-deep k-block of a 128 x 128
  // ping-pong tile:  waves * (k-blocks per work item * kb_cost + epi),  waves = the persistent
  // grid's passes over (tiles x splits) work items. kb_cost is 1, or WIDE_KB for the twice-as-wide
  // tile; epi is what a work item's epilogue adds to its main loop. The ping-pong kernel hides a
  // stored epilogue under the other warpgroup's MMAs (epi 0), the wide one does not (WIDE_EPI).
  // A split-K item's fp32 atomics into L2 and pipeline fill cost SPLIT_EPI (x 2 for the wide
  // tile's twice as many atomics); an fp32 stored tile has twice the slabs of a bf16 one and
  // counts WIDE_EPI twice. Fitted to CUDA-event timings of both tilings (tools/gemm_probe.py) at
  // the training step's shapes, 16 512 and 3 200 tokens, on an H100 80GB HBM3 at 700 W:
  //   SPLIT_EPI = 64: any value from 43 to 128 picks the fastest 128 x 128 split, or one within
  //   3 % of it, at the four 16 512-token weight gradients (768 x 3072, 3072 x 768, 2304 x 768,
  //   768 x 768), where the earlier 10 picked splits up to 50 % slower.
  //   WIDE_KB = 1.7, WIDE_EPI = 12 from the bf16-residual dgrads (K = 3072 and 2304: wide 3 %
  //   faster and 1 % slower at 16 512 tokens). The wide split-K cost 2 x SPLIT_EPI (any value from
  //   96 to 128) then picks, over all 17 probed GEMMs, a (tiling, split) within 5 % of the fastest,
  //   and 128 x 256 for dW2 / dW1 (0.195 / 0.169 -> 0.157 / 0.137 ms) but not for dWqkv / dWo;
  //   the fp32 LayerNorm-form FFN-down stays 128 x 128 (wide: 2 % slower at 16 512 tokens).
  // Ties go to the 128 x 128 tiling and to the smaller split count; a split keeps >= 4 k-blocks so
  // the TMA pipeline has something to overlap.
  constexpr double WIDE_KB = 1.7, WIDE_EPI = 12.0, SPLIT_EPI = 64.0;
  const bool wide_ok = has_wide_form(g);
  double best_cost = -1.0;
  int bn = BLOCK_N, k_splits = 1;
  for (int cand = BLOCK_N; cand <= 256; cand *= 2) {
    if (cand == 256 ? (!wide_ok || g->block_n == 128) : (wide_ok && g->block_n == 256)) continue;
    const bool wide = (cand == 256);
    const int tiles = s.num_m_blocks * ceil_div(g->n, cand);
    int sp_lo = 1, sp_hi = 1;
    if (g->out_f32_accumulate) {
      if (g->k_splits > 0) {
        sp_lo = sp_hi = g->k_splits < s.k_blocks ? g->k_splits : s.k_blocks;
      } else {
        sp_hi = s.k_blocks / 4 > 1 ? s.k_blocks / 4 : 1;
        if (sp_hi > 64) sp_hi = 64;
      }
    }
    const double epi = g->out_f32_accumulate ? SPLIT_EPI * (wide ? 2.0 : 1.0)
                                             : (wide ? WIDE_EPI * (g->out_f32_store ? 2.0 : 1.0) : 0.0);
    for (int sp = sp_lo; sp <= sp_hi; ++sp) {
      const double waves = ceil_div(tiles * sp, sms);
      const double cost = waves * (ceil_div(s.k_blocks, sp) * (wide ? WIDE_KB : 1.0) + epi);
      if (best_cost < 0.0 || cost < best_cost) {
        best_cost = cost;
        bn = cand;
        k_splits = sp;
      }
    }
  }
  s.num_n_blocks = ceil_div(g->n, bn);
  // the kernels split the k-blocks in 32-bit arithmetic (a 64-bit division is a subroutine call,
  // and the registers live across it spill)
  HERO_REQUIRE((long long)k_splits * s.k_blocks < (1ll << 31), "k_splits x k-blocks overflows");
  s.k_splits = k_splits;
  HERO_REQUIRE((g->a_lo == nullptr) == (g->b_lo == nullptr), "a_lo and b_lo go together");
  s.k_passes = g->a_lo ? 3 : 1;
  s.dynamic = g_shared_sms ? 1 : 0;

  GemmEpilogue e;
  e.bias = g->bias;
  e.ln_mean = g->resid_ln_mean;
  e.ln_rstd = g->resid_ln_rstd;
  e.ln_gamma = g->resid_ln_gamma;
  e.ln_beta = g->resid_ln_beta;
  e.ce_label = g->ce_label;
  e.ce_partial = reinterpret_cast<float2*>(g->ce_partial);
  e.ce_lab = g->ce_label_logit;
  e.ce_lse = g->ce_lse;
  e.ce_g = g->ce_grad;
  e.colsum = g->out_colsum;
  if (g->out_colsum != nullptr)
    HERO_REQUIRE(!g->out_f32_accumulate && !g->out_f32_store && !g->resid_f32 && g->out != nullptr &&
                     g->n % 2 == 0 && g->act != ACT_CE,
                 "out_colsum goes with a stored bf16 output of even width");
  e.ce_ld = g->ce_ld_partial;
  e.ce_n_valid = g->ce_n_valid > 0 ? g->ce_n_valid : g->n;
  if (g->act == ACT_CE)
    HERO_REQUIRE(g->ce_label && g->ce_partial && g->ce_label_logit && g->ce_ld_partial >= g->m &&
                     !g->out_f32_accumulate && !g->out_f32_store,
                 "act 4 (cross-entropy partials) needs ce_label, ce_partial, ce_label_logit");
  if (g->act == ACT_CE_GRAD)
    HERO_REQUIRE(g->ce_label && g->ce_lse && g->ce_grad && !g->out_f32_accumulate && !g->out_f32_store,
                 "act 5 (cross-entropy gradient) needs ce_label, ce_lse, ce_grad");
  if (g->resid_ln_mean || g->resid_ln_rstd || g->resid_ln_gamma || g->resid_ln_beta)
    HERO_REQUIRE(g->resid && g->resid_f32 && g->resid_ln_mean && g->resid_ln_rstd &&
                     g->resid_ln_gamma && g->resid_ln_beta,
                 "a LayerNorm-form residual needs an fp32 resid and all four of mean/rstd/gamma/beta");
  e.has_aux = g->aux_out != nullptr;
  e.out = g->out;
  e.ld_out = g->ld_out;
  e.drop_threshold = g->drop_threshold;
  e.drop_key = g->drop_key;
  e.drop_scale = g->drop_scale;

  GemmMaps tm;
  int rc;
  if (g->a_mn_major)
    rc = get_tmap(&tm.a, g->a, g->k, (g->m + 63) / 64 * 64, g->lda, BLOCK_M, TM_MNMAJOR);
  else
    rc = get_tmap(&tm.a, g->a, g->m, g->k, g->lda, BLOCK_M, TM_KMAJOR);
  if (rc) return rc;
  if (g->b_mn_major)
    rc = get_tmap(&tm.b, g->b, g->k, g->n, g->ldb, bn, TM_MNMAJOR);
  else
    rc = get_tmap(&tm.b, g->b, g->n, g->k, g->ldb, bn, TM_KMAJOR);
  if (rc) return rc;
  tm.a_lo = tm.a;
  tm.b_lo = tm.b;
  if (g->a_lo) {     // same shapes / leading dimensions as the hi parts
    if (g->a_mn_major)
      rc = get_tmap(&tm.a_lo, g->a_lo, g->k, g->m, g->lda, BLOCK_M, TM_MNMAJOR);
    else
      rc = get_tmap(&tm.a_lo, g->a_lo, g->m, g->k, g->lda, BLOCK_M, TM_KMAJOR);
    if (rc) return rc;
    if (g->b_mn_major)
      rc = get_tmap(&tm.b_lo, g->b_lo, g->k, g->n, g->ldb, bn, TM_MNMAJOR);
    else
      rc = get_tmap(&tm.b_lo, g->b_lo, g->n, g->k, g->ldb, bn, TM_KMAJOR);
    if (rc) return rc;
  }
  tm.out = tm.a;
  tm.aux = tm.a;
  tm.res = tm.a;
  if (!g->out_f32_accumulate && g->act != ACT_CE) {
    if (g->out_f32_store) {
      if ((rc = get_tmap(&tm.out, g->out, g->m, g->n, g->ld_out, 32, TM_SLAB_F32))) return rc;
    } else {
      HERO_REQUIRE(g->ld_out % 8 == 0, "bf16 output needs ld_out %% 8 == 0");
      if ((rc = get_tmap(&tm.out, g->out, g->m, g->n, g->ld_out, 64, TM_SLAB_BF16))) return rc;
    }
    if (g->aux_out) {
      HERO_REQUIRE(g->ld_aux_out % 8 == 0, "aux_out needs ld %% 8 == 0");
      HERO_REQUIRE(g->act == ACT_GELU || g->act == ACT_RELU, "aux_out needs act 1 or 2");
      if ((rc = get_tmap(&tm.aux, g->aux_out, g->m, g->n, g->ld_aux_out, 64, TM_SLAB_BF16)))
        return rc;
    }
    if (g->act == ACT_GELU_GRAD) {
      HERO_REQUIRE(g->ld_aux_in % 8 == 0, "aux_in needs ld %% 8 == 0");
      if ((rc = get_tmap(&tm.res, g->aux_in, g->m, g->n, g->ld_aux_in, 64, TM_SLAB_BF16)))
        return rc;
    } else if (g->resid) {
      if (g->resid_f32) {
        HERO_REQUIRE(g->ld_resid % 4 == 0, "fp32 residual needs ld %% 4 == 0");
        if ((rc = get_tmap(&tm.res, g->resid, g->m, g->n, g->ld_resid, 32, TM_SLAB_F32))) return rc;
      } else {
        HERO_REQUIRE(g->ld_resid % 8 == 0, "bf16 residual needs ld %% 8 == 0");
        if ((rc = get_tmap(&tm.res, g->resid, g->m, g->n, g->ld_resid, 64, TM_SLAB_BF16)))
          return rc;
      }
    }
  }

  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (bn_used) *bn_used = bn;
  return dispatch(g, tm, s, e, bn == 256, st);
}

// Block-wide 8-bit radix select on the order-preserving uint32 image of a float, shared by the
// retrieval ranking (rank.cu: block_select_sorted) and the TVC sampler (decode_ctl.cu).
//
// Four passes of 8 bits, most significant first. Each pass histograms the items whose key matches
// the prefix found so far, scans the 256 bins in descending order and extends the prefix by the bin
// where the running weight reaches `need`; after the last pass the prefix is the full key of the
// threshold. The weight of an item is 1 (a count: the threshold is the need-th largest key) or, for
// a weighted source, Src::weight(t) (a mass: the threshold is the largest key whose items at or
// above it weigh at least `need`). Items of one warp that fall into the same bin are grouped with
// __match_any_sync and the group's lowest lane adds the group's count or mass with one shared-memory
// atomic (a row's keys crowd into a few bins in the first pass, where one atomic per item would
// serialise). Masses are 64-bit integers, so every bin's sum is exact and the result does not
// depend on the order of the additions.
#pragma once
#include <stdint.h>

namespace hero {

// float -> uint32 with the same order (negative floats reversed, positive above them)
__device__ __forceinline__ uint32_t ord_key(float x) {
  const uint32_t b = __float_as_uint(x);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <typename W>
struct RadixSmem {
  W hist[256];
  W need;
  uint32_t prefix, take_all;
};

// Every thread of the CTA (THREADS of them) must call it. src.get(t, key) says whether item t
// exists and gives its key. A weighted selection needs `scratch`, THREADS entries of W in shared
// memory, where each warp gathers its items' weights for the group sums. Returns the threshold
// key in `prefix_out` and the weight still needed at it in `need_out` (the weight above the
// threshold is need - need_out). A count selection whose items number no more than `need` sets
// take_all_out instead (every existing item is selected); a weighted one never does.
template <int THREADS, bool WEIGHTED, typename W, class Src>
__device__ void block_radix_select(const Src& src, int n_items, W need, RadixSmem<W>& sm,
                                   uint32_t& prefix_out, W& need_out, bool& take_all_out,
                                   W* scratch = nullptr) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr unsigned kFull = 0xffffffffu;
  uint32_t prefix = 0;
  bool take_all = false;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    const uint32_t hmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
    for (int i = tid; i < 256; i += THREADS) sm.hist[i] = 0;
    __syncthreads();
    for (int base = 0; base < n_items; base += THREADS) {   // warp-uniform trip count
      const int t = base + tid;
      uint32_t k = 0;
      int bin = -1;
      if (t < n_items && src.get(t, k) && (k & hmask) == prefix) bin = (int)((k >> shift) & 255u);
      const unsigned peers = __match_any_sync(kFull, bin);
      if constexpr (WEIGHTED) {
        W* ws = scratch + (tid & ~31);
        ws[lane] = bin >= 0 ? src.weight(t) : (W)0;
        __syncwarp();
        if (bin >= 0 && lane == __ffs(peers) - 1) {
          W sum = 0;
          for (unsigned m = peers; m != 0u; m &= m - 1u) sum += ws[__ffs(m) - 1];
          if (sum != 0) atomicAdd(&sm.hist[bin], sum);
        }
        __syncwarp();
      } else {
        if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(&sm.hist[bin], (W)__popc(peers));
      }
    }
    __syncthreads();
    if (warp == 0) {
      // lane l owns bins 255 - 8l .. 248 - 8l (descending)
      W c[8], s = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        c[i] = sm.hist[255 - 8 * lane - i];
        s += c[i];
      }
      W inc = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const W v = __shfl_up_sync(kFull, inc, o);
        if (lane >= o) inc += v;
      }
      const W total = __shfl_sync(kFull, inc, 31);
      if (!WEIGHTED && pass == 0 && total <= need) {   // no more items than asked for: keep all
        if (lane == 0) sm.take_all = 1u;
      } else {
        const unsigned hit = __ballot_sync(kFull, inc >= need);
        if (lane == __ffs(hit) - 1) {
          W acc = inc - s;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (acc + c[i] >= need) {
              sm.prefix = prefix | ((uint32_t)(255 - 8 * lane - i) << shift);
              sm.need = need - acc;
              break;
            }
            acc += c[i];
          }
        }
        if (lane == 0) sm.take_all = 0u;
      }
    }
    __syncthreads();
    take_all = sm.take_all != 0u;
    if (take_all) break;
    prefix = sm.prefix;
    need = sm.need;
  }
  prefix_out = prefix;
  need_out = need;
  take_all_out = take_all;
}

}  // namespace hero

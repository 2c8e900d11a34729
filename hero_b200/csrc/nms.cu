// Greedy temporal non-maximum suppression of ranked moment lists: the post-processing of the
// reference's full VCMR evaluation (utils/tvr_eval_utils.py:35-92 temporal_non_maximum_suppression,
// :132-175 filter_vcmr_by_nms, :193-234 post_processing_{vcmr,svmr}_nms), which the reference runs
// in Python on the host, one IoU call per pair.
//
// One CTA per query. The candidates (sorted by descending score, as hero_vcmr_moment_topn writes
// them) are staged in shared memory with the time values the evaluation reads; a greedy sweep in
// input order keeps an entry when it is still alive and suppresses the later entries of its group
// whose IoU with it exceeds the threshold, with one barrier per kept entry. The kept entries are then
// placed by counting on the reference's merge key.
#include "common.h"
#include "ptx.cuh"

namespace hero {

constexpr int NMS_THREADS = 256;
constexpr int NMS_MAX_N = 1024;       // n_in and n_out
// temporal_non_maximum_suppression(max_after_nms=100): filter_vcmr_by_nms and
// post_processing_svmr_nms call it with this default whatever their own max_after_nms is
constexpr int NMS_GROUP_CAP = 100;

struct NmsSmem {
  double st[NMS_MAX_N];
  double ed[NMS_MAX_N];
  float score[NMS_MAX_N];
  int32_t clip[NMS_MAX_N];
  int32_t grp[NMS_MAX_N];     // index of the first entry of the same clip (VCMR); 0 (SVMR)
  int32_t state[NMS_MAX_N];   // -1 suppressed, else the number of kept entries before it in its group
  int32_t n_valid, n_kept;
};
static_assert(sizeof(NmsSmem) <= 48 * 1024, "NMS state must fit the default shared memory limit");

// compute_temporal_iou (utils/tvr_eval_utils.py:14-32): the "union" is the hull of both spans
__device__ __forceinline__ double temporal_iou(double s0, double e0, double s1, double e1) {
  const double inter = fmax(0.0, __dsub_rn(fmin(e0, e1), fmax(s0, s1)));
  const double uni = __dsub_rn(fmax(e0, e1), fmin(s0, s1));
  return uni == 0.0 ? 0.0 : __ddiv_rn(inter, uni);
}

__global__ void __launch_bounds__(NMS_THREADS)
temporal_nms_kernel(const float* __restrict__ score, const int32_t* __restrict__ mom, int ld_in,
                    int n_in, double thd, double interval, int by_clip, int n_out,
                    float* __restrict__ out_score, int32_t* __restrict__ out_mom) {
  pdl_wait();
  pdl_launch_dependents();
  __shared__ NmsSmem sm;
  const int tid = threadIdx.x;
  const long long q = blockIdx.x;
  const float* sc = score + q * ld_in;
  const int32_t* mm = mom + q * ld_in * 3;
  if (tid == 0) {
    sm.n_valid = n_in;
    sm.n_kept = 0;
  }
  __syncthreads();
  for (int i = tid; i < n_in; i += NMS_THREADS)        // the list ends at its first padded entry
    if (mm[3 * i] < 0) atomicMin(&sm.n_valid, i);
  __syncthreads();
  const int n = sm.n_valid;
  // Time values exactly as the host records them (evalpass._moment_records): VCMR in fp32 with
  // every operation rounded (no FMA contraction), SVMR in fp64.
  const float ivf = (float)interval;
  for (int i = tid; i < n; i += NMS_THREADS) {
    const int s = mm[3 * i + 1], e = mm[3 * i + 2];
    if (by_clip) {
      sm.st[i] = (double)__fmul_rn((float)s, ivf);
      sm.ed[i] = (double)__fadd_rn(__fmul_rn((float)e, ivf), ivf);
    } else {
      sm.st[i] = __dmul_rn((double)s, interval);
      sm.ed[i] = __dmul_rn(__dadd_rn((double)e, 1.0), interval);
    }
    sm.score[i] = sc[i];
    sm.clip[i] = mm[3 * i];
    sm.state[i] = 0;
  }
  __syncthreads();
  for (int i = tid; i < n; i += NMS_THREADS) {
    int g = 0;
    if (by_clip) {
      const int c = sm.clip[i];
      while (sm.clip[g] != c) ++g;                     // stops at i at the latest
    }
    sm.grp[i] = g;
  }
  __syncthreads();
  // Greedy sweep. state[i] is final once every earlier entry has been visited, and it is only
  // written in iterations that keep an entry, each of which ends with a barrier, so the branch
  // below is uniform across the CTA.
  for (int i = 0; i < n; ++i) {
    const int si = sm.state[i];
    if (si < 0) continue;
    const int g = sm.grp[i];
    const bool full = si + 1 >= NMS_GROUP_CAP;        // the group's last kept entry
    const double s0 = sm.st[i], e0 = sm.ed[i];
    for (int j = i + 1 + tid; j < n; j += NMS_THREADS) {
      if (sm.grp[j] != g) continue;
      const int sj = sm.state[j];
      if (sj < 0) continue;
      sm.state[j] = (full || temporal_iou(s0, e0, sm.st[j], sm.ed[j]) > thd) ? -1 : sj + 1;
    }
    __syncthreads();
  }
  // Output rank of a kept entry: the reference concatenates the groups in order of first appearance
  // and stable-sorts by descending score, so ties go to the earlier group, then the earlier entry.
  float* os = out_score + q * n_out;
  int32_t* om = out_mom + q * n_out * 3;
  int local_kept = 0;
  for (int i = tid; i < n; i += NMS_THREADS) {
    if (sm.state[i] < 0) continue;
    ++local_kept;
    const float si = sm.score[i];
    const int gi = sm.grp[i];
    int pos = 0;
    for (int j = 0; j < n; ++j) {
      if (sm.state[j] < 0) continue;
      const float sj = sm.score[j];
      const int gj = sm.grp[j];
      pos += (sj > si) || (sj == si && (gj < gi || (gj == gi && j < i)));
    }
    if (pos < n_out) {
      os[pos] = si;
      om[3 * pos + 0] = sm.clip[i];
      om[3 * pos + 1] = mm[3 * i + 1];
      om[3 * pos + 2] = mm[3 * i + 2];
    }
  }
  if (local_kept) atomicAdd(&sm.n_kept, local_kept);
  __syncthreads();
  for (int p = sm.n_kept + tid; p < n_out; p += NMS_THREADS) {
    os[p] = 0.f;
    om[3 * p + 0] = om[3 * p + 1] = om[3 * p + 2] = -1;
  }
}

}  // namespace hero

using namespace hero;

extern "C" int hero_temporal_nms(const float* score, const int32_t* mom, int32_t nq, int32_t ld_in,
                                 int32_t n_in, double thd, double interval, int32_t by_clip,
                                 int32_t n_out, float* out_score, int32_t* out_mom, void* stream) {
  HERO_REQUIRE(score && mom && out_score && out_mom, "temporal_nms: null pointer");
  HERO_REQUIRE(nq >= 0, "temporal_nms: nq = %d < 0", nq);
  HERO_REQUIRE(n_in >= 0 && n_in <= NMS_MAX_N && n_in <= ld_in,
               "temporal_nms: n_in = %d outside [0, min(%d, ld_in %d)]", n_in, NMS_MAX_N, ld_in);
  HERO_REQUIRE(n_out >= 1 && n_out <= NMS_MAX_N, "temporal_nms: n_out = %d outside [1, %d]", n_out,
               NMS_MAX_N);
  HERO_REQUIRE(by_clip == 0 || by_clip == 1, "temporal_nms: by_clip = %d", by_clip);
  HERO_REQUIRE(isfinite(thd) && isfinite(interval) && interval > 0.0,
               "temporal_nms: threshold %g / interval %g", thd, interval);
  if (nq == 0) return HERO_OK;
  HERO_CUDA_CHECK(launch_pdl(temporal_nms_kernel, dim3(nq), dim3(NMS_THREADS), 0,
                             reinterpret_cast<cudaStream_t>(stream), score, mom, (int)ld_in,
                             (int)n_in, thd, interval, (int)by_clip, (int)n_out, out_score, out_mom));
  return HERO_OK;
}

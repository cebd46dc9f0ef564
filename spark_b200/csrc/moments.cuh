// moments.cuh -- VAR_POP / VAR_SAMP / STDDEV_POP / STDDEV_SAMP inside the hash aggregate (CentralMomentAgg.scala:49-290), csrc/moments.cu
#pragma once
#include <vector>
#include "agg_kernels.cuh"

namespace sb {

constexpr int MOM_MAX_INPUTS = AGG_MAX_SLOTS / 3;   // a distinct moment input has its own SUM, MIN and MAX slots

static inline bool is_moment_func(int32_t f) {
  return f == SB_AGG_VAR_POP || f == SB_AGG_VAR_SAMP || f == SB_AGG_STDDEV_POP || f == SB_AGG_STDDEV_SAMP;
}
// columns one aggregate occupies in a Partial / PartialMerge table (its buffer) -- the positional layout Final reads
static inline int agg_buffer_width(int32_t f) { return f == SB_AGG_AVG ? 2 : (is_moment_func(f) ? 3 : 1); }

// One distinct input of the plan's moment aggregates.  Pass 1 (the unchanged aggregate) accumulated four slots for it:
//   update modes: COUNT(x), SUM(x), MIN(x), MAX(x);  merge modes: SUM(n), SUM(n * avg), MIN(avg), MAX(avg) over non-empty partials.
struct MomentInput {
  const void *x;            // update: the value, any numeric type read as double; merge: avg, NULL where the partial is empty
  const uint8_t *xv;        // validity of x or nullptr
  int32_t xtype;
  const double *n, *m2;     // merge: n (0.0 for an empty partial) and m2 of the partial buffers
  int32_t slot_cnt, slot_sum, slot_min, slot_max;
};
// One moment aggregate's output columns: buffers (n, avg, m2) or its result
struct MomentOut {
  int32_t input, func, flags;
  void *out[3];
  uint32_t *out_valid;      // result validity (results only)
};

// Pass 2 and the finish step, after pass 1 has filled the table of `a`: streams the input once more (same fused filter, key
// packing and table probe as pass 1) and accumulates the deviations from each group's pass-1 mean, then writes the outputs of
// every moment aggregate for the `ngroups` occupied table slots listed in slot_ids.
void moments_run(const AggArgs &a, const std::vector<MomentInput> &ins, const std::vector<MomentOut> &outs, bool merge, bool emit_buffers,
                 const int64_t *slot_ids, int64_t ngroups, cudaStream_t st);
// merge modes: the (n, avg) buffer columns -> n with empty / NULL partials as 0.0, and avg valid only where n > 0
void moments_mask_buffers(const Column &n, const Column &avg, const Column &m2, Column &n_out, Column &avg_out, cudaStream_t st);

}  // namespace sb

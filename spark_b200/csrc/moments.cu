// moments.cu -- VAR_POP, VAR_SAMP, STDDEV_POP and STDDEV_SAMP in the hash aggregate.
//
// Reference semantics (sql/catalyst/.../expressions/aggregate/CentralMomentAgg.scala): buffer (n, avg, m2), all doubles, initial
// (0.0, 0.0, 0.0) (:78-80); update :122-160 (Welford: delta = x - avg, avg += delta / n, m2 += delta * (delta - delta / n));
// merge :83-120 (Chan et al., with an empty side taken as is); results :172-290 (NULL for n == 0; the _samp forms give NULL, or
// NaN when nullOnDivideByZero is off, for n == 1).
//
// Spark's update is sequential; here the same buffer comes from a corrected two-pass computation around the unchanged
// fixed-width aggregate:
//   pass 1  the aggregate's own kernels, with four extra slots per moment input in the same plan: COUNT, SUM, MIN and MAX of x
//           (update modes), or SUM(n), SUM(n * avg), MIN(avg) and MAX(avg) over non-empty partials (merge modes).  They give each
//           group its mean m^ = SUM / COUNT.
//   pass 2  one more stream over the input with the same fused filter, key packing (tile_keys / tile_keys_wide) and table probe
//           (table_slot / table_slot_wide) as pass 1 -- every key layout the aggregate takes works unchanged -- accumulating
//           S1 = sum d and S2 = sum d^2 per group, d = x - m^ (merge: n_i (avg_i - m^), n_i (avg_i - m^)^2 and sum m2_i).
//   finish  n = COUNT, avg = m^ + S1 / n, m2 = S2 - S1^2 / n (+ sum m2_i), clamped at +0.0.  The correction term makes m2 as
//           accurate as if the exact mean had been subtracted: values near 1e9 with unit spread keep every digit, where the naive
//           sum x^2 - (sum x)^2 / n keeps none.
// Two cases are exact in Spark and made exact here: a group whose MIN equals its MAX (constant, or one row) has m2 = +0.0 and
// avg = that value (+ 0.0, as Welford's first step from avg = +0.0 gives); a group with a NaN or infinite term has m2 = NaN.
#include <vector>
#include "moments.cuh"

namespace sb {

constexpr int MOM_ITEMS = 4;                 // rows per thread per tile (tiles of AGG_THREADS * MOM_ITEMS rows, as pass 1)
constexpr int MOM_MAX_OUTS = AGG_MAX_SLOTS;
#define kNaN __longlong_as_double(0x7FF8000000000000ll)   // Double.NaN
constexpr int MOM_SHARED_VALUES = 2048;      // per-block shared accumulators when groups x accumulators fit (16 KB)

struct MomentArgs {
  int32_t ninputs, nacc, nouts, merge, emit_buffers, shared;
  MomentInput in[MOM_MAX_INPUTS];
  MomentOut out[MOM_MAX_OUTS];
  int32_t *group_of_slot;         // [cap + 2]: dense group of an occupied table slot
  const int64_t *slot_ids;        // [ngroups]: table slot of a dense group
  double *mean;                   // [ninputs][ngroups]: pass-1 mean m^
  double *acc;                    // [ninputs][nacc][ngroups]: S1, S2 (, sum m2_i)
  int64_t ngroups;
};

__device__ __forceinline__ double ordered_to_double(uint64_t m) {   // inverse of the X_DOUBLE min / max transform
  return __longlong_as_double((int64_t)((m >> 63) ? (m ^ 0x8000000000000000ull) : ~m));
}

__global__ void moment_prep_kernel(const __grid_constant__ AggArgs a, const __grid_constant__ MomentArgs ma) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ma.ngroups) return;
  const int64_t slot = ma.slot_ids[g], stride = a.cap + 2;
  ma.group_of_slot[slot] = (int32_t)g;
  for (int i = 0; i < ma.ninputs; i++) {
    const MomentInput &in = ma.in[i];
    const uint64_t c = a.tacc[(int64_t)in.slot_cnt * stride + slot];
    const double n = ma.merge ? __longlong_as_double((int64_t)c) : (double)(int64_t)c;
    const double s = __longlong_as_double((int64_t)a.tacc[(int64_t)in.slot_sum * stride + slot]);
    ma.mean[i * ma.ngroups + g] = n > 0.0 ? __ddiv_rn(s, n) : 0.0;
  }
}

// pass 2: NW = key words of the plan (1: tile_keys, which also handles single 64-bit and NULL / sentinel keys); MERGE: the input
// is (n, avg, m2) buffers
template <int NW, bool MERGE>
__global__ void __launch_bounds__(AGG_THREADS) moment_pass2_kernel(const __grid_constant__ AggArgs a, const __grid_constant__ MomentArgs ma) {
  extern __shared__ double sacc[];
  constexpr int64_t TILE = (int64_t)AGG_THREADS * MOM_ITEMS;
  const int tid = threadIdx.x;
  const int64_t G = ma.ngroups;
  constexpr int NACC = MERGE ? 3 : 2;
  const int nvals = ma.ninputs * NACC;
  if (ma.shared) {
    for (int i = tid; i < nvals * G; i += AGG_THREADS) sacc[i] = 0.0;
    __syncthreads();
  }
  for (int64_t base = (int64_t)blockIdx.x * TILE; base < a.n; base += (int64_t)gridDim.x * TILE) {
    TileCtx t{base + tid, a.n - 1};
    bool keep[MOM_ITEMS];
    int64_t slot[MOM_ITEMS];
    if constexpr (NW == 1) {
      uint64_t key[MOM_ITEMS];
      int special[MOM_ITEMS];
      tile_keys<DynPlan, MOM_ITEMS, false>(a, t, keep, key, special);
#pragma unroll
      for (int k = 0; k < MOM_ITEMS; k++) slot[k] = keep[k] ? table_slot(a, key[k], special[k]) : -1;
    } else {
      uint64_t key[MOM_ITEMS][NW];
      tile_keys_wide<NW, MOM_ITEMS>(a, t, keep, key);
#pragma unroll
      for (int k = 0; k < MOM_ITEMS; k++) slot[k] = keep[k] ? table_slot_wide<NW>(a, key[k]) : -1;
    }
    int64_t g[MOM_ITEMS];
#pragma unroll
    for (int k = 0; k < MOM_ITEMS; k++) g[k] = slot[k] >= 0 ? ma.group_of_slot[slot[k]] : -1;
    for (int i = 0; i < ma.ninputs; i++) {
      const MomentInput &in = ma.in[i];
      double x[MOM_ITEMS];
      bool ok[MOM_ITEMS];
      load_f64_batch<MOM_ITEMS, false>(in.x, in.xtype, t, x);
#pragma unroll
      for (int k = 0; k < MOM_ITEMS; k++) ok[k] = g[k] >= 0;
      if (in.xv) {
        bool v[MOM_ITEMS];
        load_valid_batch<MOM_ITEMS, false>(in.xv, t, v);
#pragma unroll
        for (int k = 0; k < MOM_ITEMS; k++) ok[k] = ok[k] && v[k];
      }
      double w[MOM_ITEMS], m2[MOM_ITEMS];
      if constexpr (MERGE) {
        load_f64_batch<MOM_ITEMS, false>(in.n, SB_FLOAT64, t, w);
        load_f64_batch<MOM_ITEMS, false>(in.m2, SB_FLOAT64, t, m2);
      }
#pragma unroll
      for (int k = 0; k < MOM_ITEMS; k++) {
        if (!ok[k]) continue;
        const double d = __dsub_rn(x[k], ma.mean[i * G + g[k]]);
        double v[NACC];
        if constexpr (MERGE) {
          v[0] = __dmul_rn(w[k], d);
          v[1] = __dmul_rn(v[0], d);
          v[2] = m2[k];
        } else {
          v[0] = d;
          v[1] = __dmul_rn(d, d);
        }
#pragma unroll
        for (int j = 0; j < NACC; j++) {
          const int64_t at = (int64_t)(i * NACC + j) * G + g[k];
          atomicAdd(ma.shared ? &sacc[at] : &ma.acc[at], v[j]);
        }
      }
    }
  }
  if (ma.shared) {
    __syncthreads();
    for (int i = tid; i < nvals * G; i += AGG_THREADS)
      if (sacc[i] != 0.0) atomicAdd(&ma.acc[i], sacc[i]);   // -0.0 adds nothing to the +0.0 start
  }
}

// (n, avg, m2) of every group, then buffers or results (CentralMomentAgg.scala:179-290)
__global__ void moment_finish_kernel(const __grid_constant__ AggArgs a, const __grid_constant__ MomentArgs ma) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in_range = g < ma.ngroups;
  const int64_t G = ma.ngroups, stride = a.cap + 2;
  const int64_t slot = in_range ? ma.slot_ids[g] : 0;
  for (int o = 0; o < ma.nouts; o++) {
    const MomentOut &mo = ma.out[o];
    const MomentInput &in = ma.in[mo.input];
    double n = 0.0, avg = 0.0, m2 = 0.0;
    if (in_range) {
      const uint64_t c = a.tacc[(int64_t)in.slot_cnt * stride + slot];
      n = ma.merge ? __longlong_as_double((int64_t)c) : (double)(int64_t)c;
      if (n > 0.0) {
        const uint64_t lo = a.tacc[(int64_t)in.slot_min * stride + slot], hi = a.tacc[(int64_t)in.slot_max * stride + slot];
        const double mn = ordered_to_double(lo), mx = ordered_to_double(hi);
        const double mean = ma.mean[mo.input * G + g];
        const double *acc = ma.acc + (int64_t)mo.input * ma.nacc * G;
        const double s1 = acc[g], s2 = acc[G + g], sm2 = ma.merge ? acc[2 * G + g] : 0.0;
        if (!isfinite(mn) || !isfinite(mx)) {
          avg = __dadd_rn(mean, __ddiv_rn(s1, n));
          m2 = kNaN;
        } else if (lo == hi) {
          avg = __dadd_rn(mn, 0.0);
          m2 = sm2;
        } else {
          avg = __dadd_rn(mean, __ddiv_rn(s1, n));
          m2 = __dadd_rn(__dsub_rn(s2, __ddiv_rn(__dmul_rn(s1, s1), n)), sm2);
        }
        m2 = m2 <= 0.0 ? 0.0 : m2;   // rounding can leave a tiny negative; NaN stays
      }
    }
    if (ma.emit_buffers) {
      if (in_range) {
        ((double *)mo.out[0])[g] = n;
        ((double *)mo.out[1])[g] = avg;
        ((double *)mo.out[2])[g] = m2;
      }
      continue;
    }
    const bool samp = mo.func == SB_AGG_VAR_SAMP || mo.func == SB_AGG_STDDEV_SAMP;
    const bool sqrt_ = mo.func == SB_AGG_STDDEV_POP || mo.func == SB_AGG_STDDEV_SAMP;
    bool valid = in_range && n != 0.0;
    double r = 0.0;
    if (valid) {
      if (samp && n == 1.0) {
        valid = (mo.flags & SB_AGG_FLAG_NAN_ON_DIVIDE_BY_ZERO) != 0;
        r = kNaN;
      } else {
        r = __ddiv_rn(m2, samp ? __dsub_rn(n, 1.0) : n);
        if (sqrt_) r = __dsqrt_rn(r);
      }
    }
    if (in_range) ((double *)mo.out[0])[g] = valid ? r : 0.0;
    const uint32_t w = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0 && (g - (g & 31)) < G) mo.out_valid[g >> 5] = w;
  }
}

__global__ void moment_mask_kernel(const double *__restrict__ n, const uint8_t *__restrict__ nv, const double *__restrict__ avg,
                                   const uint8_t *__restrict__ av, const uint8_t *__restrict__ mv, int64_t rows, double *__restrict__ n_out,
                                   double *__restrict__ avg_out, uint32_t *__restrict__ avg_valid) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = r < rows;
  const bool ok = in && bit_valid(nv, r) && bit_valid(av, r) && bit_valid(mv, r) && n[r] > 0.0;
  if (in) {
    n_out[r] = ok ? n[r] : 0.0;
    avg_out[r] = ok ? avg[r] : 0.0;
  }
  const uint32_t w = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && (r - (r & 31)) < rows) avg_valid[r >> 5] = w;
}

void moments_mask_buffers(const Column &n, const Column &avg, const Column &m2, Column &n_out, Column &avg_out, cudaStream_t st) {
  const int64_t rows = n.length;
  n_out = column_alloc(SB_FLOAT64, 0, rows, false, st);
  avg_out = column_alloc(SB_FLOAT64, 0, rows, true, st);
  avg_out.null_count = -1;
  if (rows == 0) return;
  moment_mask_kernel<<<(unsigned)((rows + 255) / 256), 256, 0, st>>>((const double *)n.d(), n.v(), (const double *)avg.d(), avg.v(), m2.v(), rows,
                                                                    (double *)n_out.data->ptr, (double *)avg_out.data->ptr,
                                                                    (uint32_t *)avg_out.validity->ptr);
  SB_LAUNCH_CHECK();
}

void moments_run(const AggArgs &a, const std::vector<MomentInput> &ins, const std::vector<MomentOut> &outs, bool merge, bool emit_buffers,
                 const int64_t *slot_ids, int64_t ngroups, cudaStream_t st) {
  if (outs.empty() || ngroups == 0) return;
  SB_REQUIRE((int)ins.size() <= MOM_MAX_INPUTS, "internal: %zu moment inputs", ins.size());
  if ((int)outs.size() > MOM_MAX_OUTS) fail(SB_ERR_UNSUPPORTED, "at most %d variance / stddev aggregates per plan", MOM_MAX_OUTS);
  static thread_local MomentArgs ma;
  memset(&ma, 0, sizeof(ma));
  ma.ninputs = (int32_t)ins.size();
  ma.nacc = merge ? 3 : 2;
  ma.nouts = (int32_t)outs.size();
  ma.merge = merge;
  ma.emit_buffers = emit_buffers;
  for (size_t i = 0; i < ins.size(); i++) ma.in[i] = ins[i];
  for (size_t i = 0; i < outs.size(); i++) ma.out[i] = outs[i];
  const int64_t nvals = (int64_t)ma.ninputs * ma.nacc;
  ma.shared = nvals * ngroups <= MOM_SHARED_VALUES;
  Scratch gos((a.cap + 2) * 4, st), mean((int64_t)ma.ninputs * ngroups * 8, st), acc(nvals * ngroups * 8, st);
  SB_CUDA(cudaMemsetAsync(acc.ptr, 0, (size_t)(nvals * ngroups * 8), st));
  ma.group_of_slot = gos.as<int32_t>();
  ma.slot_ids = slot_ids;
  ma.mean = mean.as<double>();
  ma.acc = acc.as<double>();
  ma.ngroups = ngroups;
  const unsigned gblocks = (unsigned)((ngroups + 255) / 256);
  moment_prep_kernel<<<gblocks, 256, 0, st>>>(a, ma);
  SB_LAUNCH_CHECK();
  if (a.n > 0) {
    KernelTimer kt("moment_pass2", st);
    const size_t smem = ma.shared ? (size_t)(nvals * ngroups * 8) : 0;
    const int grid = grid_for(a.n, AGG_THREADS * MOM_ITEMS, rt().num_sms * 8);
    auto launch = [&](auto kernel) { kernel<<<grid, AGG_THREADS, smem, st>>>(a, ma); };
    switch (a.nwords * 2 + (merge ? 1 : 0)) {
      case 2: launch(moment_pass2_kernel<1, false>); break;
      case 3: launch(moment_pass2_kernel<1, true>); break;
      case 4: launch(moment_pass2_kernel<2, false>); break;
      case 5: launch(moment_pass2_kernel<2, true>); break;
      case 6: launch(moment_pass2_kernel<3, false>); break;
      case 7: launch(moment_pass2_kernel<3, true>); break;
      case 8: launch(moment_pass2_kernel<4, false>); break;
      default: launch(moment_pass2_kernel<4, true>); break;
    }
    SB_LAUNCH_CHECK();
  }
  KernelTimer kt("moment_finish", st);
  moment_finish_kernel<<<gblocks, 256, 0, st>>>(a, ma);
  SB_LAUNCH_CHECK();
}

}  // namespace sb

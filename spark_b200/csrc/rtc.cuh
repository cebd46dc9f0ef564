// rtc.cuh -- run-time specialisation of kernels with NVRTC: the GPU analogue of the reference's whole-stage code
// generation (WholeStageCodegenExec.scala: Janino compiles the fused Java of a stage when the plan is first executed).
#pragma once
#include <string>
#include <vector>
#include "common.cuh"

namespace sb {

struct RtcProgram {
  bool ok = false;
  std::string log;                       // compiler log or the reason the program is unavailable
  cudaLibrary_t library = nullptr;
  std::vector<const void *> kernels;     // cudaKernel_t handles (usable wherever a __global__ symbol is), order of `names`
  double compile_ms = 0;
  bool from_disk_cache = false;
};

// Compiles `source` (which may #include the embedded headers: agg_kernels.cuh, device_helpers.cuh, spark_b200.h) for
// sm_90a, instantiating the kernel name expressions in `names`.  Results are cached by `cache_key` in the process and
// as cubin files under $SB_RTC_CACHE_DIR (default ~/.cache/spark_b200/rtc).  Never throws: failure is reported in
// RtcProgram::ok / log and callers fall back to their precompiled generic kernels.
// load = false: compile only (no device needed; used by the CPU build check), nothing is cached on disk.
const RtcProgram *rtc_compile(const std::string &cache_key, const std::string &source, const std::vector<std::string> &names, bool load = true);

// library-wide settings (sb_config_set): "agg_rtc" = off | sync (default), "agg_rtc_min_rows" = n
struct Config {
  int agg_rtc = 1;                  // 0 off, 1 compile on first use
  int64_t agg_rtc_min_rows = 1 << 20;   // inputs smaller than this run the generic kernels (latency, not bandwidth)
  int agg_tier = 0;                 // 0 auto, 1 dictionary only, 2 shared-memory table only (tests)
  int agg_verbose = 0;
  int expr_interpret_only = 0;
  int regroup_ldst = 0;             // load/store multisplit instead of the copy-engine one
  int exchange_nccl = 0;            // NCCL send/recv data path instead of peer windows
  int join_cand = 2;                // join candidate pass: 0 = 16 consecutive rows per thread (16-byte loads); lane-strided with batched loads:
                                    // 1 = 8 rows per lane and step, 2 = 4 rows at 4 blocks / SM (default), 3 = 8 rows at 3 blocks / SM
  int sort_variant = 4;             // onesweep tile geometry: 4 = 384 threads x 12 keys (default)
};
Config &config();

}  // namespace sb

// Library-level entry points: version, thread-local error string, launch counter, and the
// developer tuning hook used by tools/sweep_embed.py (not part of the reference-facing ABI).
#include "common.cuh"
#include <atomic>
#include <string.h>

namespace dr {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int num_sms() {
  static const int n = [] {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v < 1)
      v = 132;   // no device visible (host-only callers): the H100 SXM count, never used for a launch
    return v;
  }();
  return n;
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

extern int g_tune_embed_fwd_unroll, g_tune_embed_bwd_unroll, g_tune_embed_block, g_tune_embed_ctas_per_sm,
    g_tune_embed_bwd_agg, g_tune_embed_bwd_mode, g_tune_embed_fwd_minblocks, g_tune_embed_fwd_linx, g_tune_embed_fwd_linx_shard, g_tune_embed_bwd_linx, g_tune_embed_l2_hints, g_tune_embed_bwd_carveout;
extern int g_tune_topk_variant;
extern int g_tune_tc_stages, g_tune_tc_l2_promo, g_tune_tc_dw_stages, g_tune_tc_dw_share, g_tune_tc_pair;
extern int g_tune_gemm_variant, g_tune_gemm_splitk, g_tune_gemm_bn, g_tune_tc_min_n;

}  // namespace dr

extern "C" int dr_version(void) { return 100; /* 0.1.0 */ }
extern "C" const char* dr_last_error(void) { return dr::g_err; }
extern "C" uint64_t dr_launch_count(void) { return dr::g_launches.load(std::memory_order_relaxed); }

// Developer hook: read back a knob (the few that tests save / restore around a case).
extern "C" int dr_tune_get(const char* key, int* value) {
  using namespace dr;
  if (!key || !value) return DR_EINVAL;
  if (!strcmp(key, "tc_pair")) *value = g_tune_tc_pair;
  else if (!strcmp(key, "tc_dw_share")) *value = g_tune_tc_dw_share;
  else if (!strcmp(key, "gemm_variant")) *value = g_tune_gemm_variant;
  else if (!strcmp(key, "gemm_bn")) *value = g_tune_gemm_bn;
  else if (!strcmp(key, "tc_min_n")) *value = g_tune_tc_min_n;
  else {
    set_error("dr_tune_get: unknown or write-only key '%s'", key);
    return DR_EINVAL;
  }
  return DR_OK;
}

// Developer hook: set a tuning knob by name.  Returns 0, or DR_EINVAL for an unknown key.
extern "C" int dr_tune_set(const char* key, int value) {
  using namespace dr;
  if (!key) return DR_EINVAL;
  if (!strcmp(key, "embed_fwd_unroll")) g_tune_embed_fwd_unroll = value;
  else if (!strcmp(key, "embed_bwd_unroll")) g_tune_embed_bwd_unroll = value;
  else if (!strcmp(key, "embed_block")) g_tune_embed_block = value;
  else if (!strcmp(key, "embed_ctas_per_sm")) g_tune_embed_ctas_per_sm = value;
  else if (!strcmp(key, "embed_bwd_agg")) g_tune_embed_bwd_agg = value;
  else if (!strcmp(key, "embed_bwd_mode")) g_tune_embed_bwd_mode = value;
  else if (!strcmp(key, "embed_fwd_minblocks")) g_tune_embed_fwd_minblocks = value;
  else if (!strcmp(key, "embed_fwd_linx")) g_tune_embed_fwd_linx = value;
  else if (!strcmp(key, "embed_fwd_linx_shard")) g_tune_embed_fwd_linx_shard = value;
  else if (!strcmp(key, "embed_bwd_linx")) g_tune_embed_bwd_linx = value;
  else if (!strcmp(key, "embed_l2_hints")) g_tune_embed_l2_hints = value;
  else if (!strcmp(key, "embed_bwd_carveout")) g_tune_embed_bwd_carveout = value;
  else if (!strcmp(key, "gemm_variant")) g_tune_gemm_variant = value;
  else if (!strcmp(key, "gemm_splitk")) g_tune_gemm_splitk = value;
  else if (!strcmp(key, "gemm_bn")) g_tune_gemm_bn = value;
  else if (!strcmp(key, "tc_min_n")) g_tune_tc_min_n = value;
  else if (!strcmp(key, "topk_variant")) g_tune_topk_variant = value;
  else if (!strcmp(key, "tc_stages")) g_tune_tc_stages = value;
  else if (!strcmp(key, "tc_l2_promo")) g_tune_tc_l2_promo = value;
  else if (!strcmp(key, "tc_dw_stages")) g_tune_tc_dw_stages = value;
  else if (!strcmp(key, "tc_dw_share")) g_tune_tc_dw_share = value;
  else if (!strcmp(key, "tc_pair")) g_tune_tc_pair = value;
  else if (!strcmp(key, "l2_fetch_granularity")) {
    // device-wide hint: how many bytes L2 fetches from HBM around a missing 32-B sector (32/64/128)
    cudaError_t e = cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)value);
    if (e != cudaSuccess) {
      set_error("dr_tune_set: cudaDeviceSetLimit(MaxL2FetchGranularity, %d): %s", value, cudaGetErrorString(e));
      return (int)e;
    }
  }
  else {
    set_error("dr_tune_set: unknown key '%s'", key);
    return DR_EINVAL;
  }
  return DR_OK;
}

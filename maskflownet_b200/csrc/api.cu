// api.cu -- bookkeeping half of the C ABI (include/maskflow_b200.h): version, thread-local error slot, launch counter.
// The operator entry points live next to their kernels (corr_fwd.cu, corr_bwd.cu, warp_fwd.cu, warp_bwd.cu).
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"

namespace mfn {

static thread_local char g_err[512] = "";
static thread_local const char* g_kernel = "";
static std::atomic<unsigned long long> g_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

void note_kernel(const char* name) { g_kernel = name; }

Tuning& tuning() {
  static Tuning t;
  return t;
}

int check_launch(const char* kernel_name) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail((int)e, "%s: launch failed: %s", kernel_name, cudaGetErrorString(e));
  g_kernel = kernel_name;
  g_launches.fetch_add(1, std::memory_order_relaxed);
  g_err[0] = '\0';
  return MFN_OK;
}

}  // namespace mfn

extern "C" int mfn_version(void) { return MFN_VERSION; }
extern "C" const char* mfn_last_error(void) { return mfn::g_err; }
extern "C" const char* mfn_last_kernel(void) { return mfn::g_kernel; }
extern "C" unsigned long long mfn_launch_count(void) { return mfn::g_launches.load(std::memory_order_relaxed); }

extern "C" int mfn_set_tuning(const char* key, int value) {
  if (!key) return mfn::fail(MFN_ERR_INVALID_ARG, "mfn_set_tuning: null key");
  if (!strcmp(key, "corr_grid_cap")) mfn::tuning().corr_grid_cap = value;
  else if (!strcmp(key, "corr_tma")) mfn::tuning().corr_tma = value;
  else if (!strcmp(key, "corr_rb")) mfn::tuning().corr_rb = value;
  else if (!strcmp(key, "warp_lin")) mfn::tuning().warp_lin = value;
  else if (!strcmp(key, "conv_wgmma")) mfn::tuning().conv_wgmma = value;
  else if (!strcmp(key, "conv_grid_cap")) mfn::tuning().conv_grid_cap = value;
  else if (!strcmp(key, "conv_splitk")) mfn::tuning().conv_splitk = value;
  else if (!strcmp(key, "conv_narrow")) mfn::tuning().conv_narrow = value;
  else if (!strcmp(key, "conv_tma_in")) mfn::tuning().conv_tma_in = value;
  else if (!strcmp(key, "conv_dbg")) mfn::tuning().conv_dbg = value;
  else return mfn::fail(MFN_ERR_INVALID_ARG, "mfn_set_tuning: unknown key '%s'", key);
  return MFN_OK;
}

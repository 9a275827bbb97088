// extern "C" surface of libmdm_b200.so (declared in include/mdm_b200.h).
#include <stdarg.h>
#include <stdio.h>

#include <string>

#include "engine.cuh"
#include "gemm_tc.cuh"
#include "mdm_b200.h"

namespace mdm {
static thread_local std::string g_err;
void set_error(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
}
}  // namespace mdm

extern "C" {

const char* mdm_last_error(void) { return mdm::g_err.c_str(); }
int mdm_version(void) { return 100; }
unsigned long long mdm_launch_count(void) { return mdm::g_launch_count; }

int mdm_profile_gemm(int enable) {
  mdm::g_profile = enable != 0;
  return 0;
}

int mdm_profile_dump(const char* path) {
  FILE* f = fopen(path, "w");
  if (f == nullptr) return -1;
  fprintf(f, "kind,majors,M,N,K,block_n,nz,nsplit,kblocks,H,W,nimg,ms,planes\n");
  for (size_t i = 0; i < mdm::g_profile_events.size(); ++i) {
    auto& ev = mdm::g_profile_events[i];
    cudaEventSynchronize(ev.second);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev.first, ev.second);
    const mdm_gemm_params& p = mdm::g_profile_params[i];
    fprintf(f, "%d,%d,%d,%d,%d,%d,%d,%d,%d,%d,%d,%d,%.5f,%d\n", p.kind, mdm::g_profile_majors[i], p.M, p.N, p.K,
            p.block_n, p.nz1 * p.nz2, p.nsplit, p.num_kblocks, p.H, p.W, p.nimg, ms, mdm::g_profile_planes[i]);
  }
  fclose(f);
  return 0;
}

int mdm_profile_read(double* total_ms, long long* launches) {
  double tot = 0.0;
  long long n = 0;
  mdm::g_profile_params.clear();
  mdm::g_profile_majors.clear();
  mdm::g_profile_planes.clear();
  for (auto& ev : mdm::g_profile_events) {
    cudaEventSynchronize(ev.second);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) {
      tot += ms;
      ++n;
    }
    cudaEventDestroy(ev.first);
    cudaEventDestroy(ev.second);
  }
  mdm::g_profile_events.clear();
  *total_ms = tot;
  *launches = n;
  return 0;
}

long long mdm_abi_sizeof(int which) {
  switch (which) {
    case 0: return static_cast<long long>(sizeof(mdm_tmap_spec));
    case 1: return static_cast<long long>(sizeof(mdm_gemm_params));
    case 2: return static_cast<long long>(sizeof(mdm_level_cfg));
    case 3: return static_cast<long long>(sizeof(mdm_net_cfg));
    case 4: return static_cast<long long>(sizeof(mdm_net_io));
    case 5: return static_cast<long long>(sizeof(mdm_net_grad_io));
    case 6: return static_cast<long long>(sizeof(mdm_opt_chunk));
    case 7: return static_cast<long long>(sizeof(mdm_adam_cfg));
    default: return -1;
  }
}

int mdm_gemm_raw_split(const mdm_tmap_spec* A, const mdm_tmap_spec* B, int a_mn, int b_mn, const mdm_gemm_params* p,
                       const void* b_lo, const void* a_lo, mdm_stream_t stream) {
  int rc = mdm::launch_gemm(*A, *B, a_mn, b_mn, *p, static_cast<cudaStream_t>(stream), b_lo, a_lo);
  if (rc != 0) {
    mdm::set_error("mdm_gemm_raw: launch failed (%d: %s)", rc,
                   rc > 0 ? cudaGetErrorString(static_cast<cudaError_t>(rc)) : "invalid arguments");
    return rc > 0 ? -rc : rc;
  }
  return 0;
}

int mdm_op_dropout_mask(uint64_t seed, uint32_t stream_id, int64_t n, float p, float* out_f32, mdm_stream_t stream) {
  if (!(p >= 0.f && p <= 1.f) || n < 0 || (n > 0 && out_f32 == nullptr)) {
    mdm::set_error("mdm_op_dropout_mask: p must lie in [0, 1], n >= 0 and out_f32 non-null");
    return -1;
  }
  if (n == 0) return 0;
  mdm::dropout_mask(seed, stream_id, n, p, out_f32, static_cast<cudaStream_t>(stream));
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    mdm::set_error("mdm_op_dropout_mask: %s", cudaGetErrorString(e));
    return -1;
  }
  return 0;
}

int mdm_gemm_raw(const mdm_tmap_spec* A, const mdm_tmap_spec* B, int a_mn, int b_mn,
                 const mdm_gemm_params* p, mdm_stream_t stream) {
  return mdm_gemm_raw_split(A, B, a_mn, b_mn, p, nullptr, nullptr, stream);
}
}

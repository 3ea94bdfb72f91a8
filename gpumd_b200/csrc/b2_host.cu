// b2_host.cu -- error string, launch counter, stage profiler.
#include "../../include/b200md.h"
#include "b2_host.h"
#include <cstdio>

namespace b2 {

static thread_local std::string g_error;
long long g_launch_count = 0;

void set_error(const std::string& msg) { g_error = msg; }

bool cuda_ok(cudaError_t e, const char* what, const char* file, int line)
{
  if (e == cudaSuccess)
    return true;
  char buf[512];
  snprintf(buf, sizeof buf, "CUDA error %s at %s:%d (%s)", cudaGetErrorString(e), file, line, what);
  g_error = buf;
  return false;
}

int load_error(const std::string& err)
{
  g_error = err;
  return err.rfind("Failed to open", 0) == 0 ? B200MD_ERR_IO : B200MD_ERR_ARG;
}

StageProfiler::~StageProfiler()
{
  if (created)
    for (int a = 0; a < MAX_SAMPLES; ++a)
      for (int b = 0; b < MAX_STAGES; ++b) {
        cudaEventDestroy(ev[a][b][0]);
        cudaEventDestroy(ev[a][b][1]);
      }
}

void StageProfiler::enable(bool on)
{
  if (on && !created) {
    for (int a = 0; a < MAX_SAMPLES; ++a)
      for (int b = 0; b < MAX_STAGES; ++b) {
        cudaEventCreate(&ev[a][b][0]);
        cudaEventCreate(&ev[a][b][1]);
      }
    created = true;
  }
  enabled = on;
  steps = 0;
  for (int a = 0; a < MAX_SAMPLES; ++a)
    for (int b = 0; b < MAX_STAGES; ++b)
      used[a][b] = false;
}

void StageProfiler::read(float* ms_sum, int* counts)
{
  cudaDeviceSynchronize();
  for (int b = 0; b < MAX_STAGES; ++b) {
    ms_sum[b] = 0.0f;
    counts[b] = 0;
  }
  const int ns = steps < MAX_SAMPLES ? steps : MAX_SAMPLES;
  for (int a = 0; a < ns; ++a)
    for (int b = 0; b < MAX_STAGES; ++b)
      if (used[a][b]) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, ev[a][b][0], ev[a][b][1]) == cudaSuccess) {
          ms_sum[b] += ms;
          counts[b] += 1;
        }
      }
}

} // namespace b2

extern "C" const char* b200md_last_error(void) { return b2::g_error.c_str(); }
extern "C" long long b200md_launch_count(void) { return b2::g_launch_count; }

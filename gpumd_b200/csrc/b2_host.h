// b2_host.h -- host-side helpers shared by the .cu translation units of libb200md.
#pragma once
#include "b2_common.cuh"
#include <cuda_runtime.h>
#include <string>

namespace b2 {

void set_error(const std::string& msg);
extern long long g_launch_count;

// returns false and records the message when a CUDA call failed
bool cuda_ok(cudaError_t e, const char* what, const char* file, int line);

#define B2_CUDA(call)                                    \
  do {                                                   \
    if (!b2::cuda_ok((call), #call, __FILE__, __LINE__)) \
      return B200MD_ERR_CUDA;                            \
  } while (0)

// count + launch-error check after every <<<>>> (the reference's GPU_CHECK_KERNEL,
// src/utilities/error.cuh:64-76)
#define B2_LAUNCHED()                   \
  do {                                  \
    ++b2::g_launch_count;               \
    B2_CUDA(cudaPeekAtLastError());     \
  } while (0)

// records the message of a failed load (b2_setup.h, NepModel::load) and returns its code: B200MD_ERR_IO when
// the file could not be opened, else B200MD_ERR_ARG
int load_error(const std::string& err);

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  ~DevBuf() { release(); }
  void release()
  {
    if (p)
      cudaFree(p);
    p = nullptr;
    n = 0;
  }
  // grows only; contents are NOT preserved
  cudaError_t reserve(size_t count)
  {
    if (count <= n)
      return cudaSuccess;
    release();
    cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
    if (e == cudaSuccess)
      n = count;
    return e;
  }
};

inline int grid_for(long long n, int block) { return (int)((n + block - 1) / block); }

// Optional per-stage device timing (CUDA events on the launching stream) for bench.py's roofline
// block.  Disabled by default: then begin()/end() are no-ops.
struct StageProfiler {
  static constexpr int MAX_STAGES = 16;
  static constexpr int MAX_SAMPLES = 256; // steps recorded before recording stops
  bool enabled = false;
  int steps = 0;
  cudaEvent_t ev[MAX_SAMPLES][MAX_STAGES][2];
  bool used[MAX_SAMPLES][MAX_STAGES];
  bool created = false;
  ~StageProfiler();
  void enable(bool on);
  void next_step()
  {
    if (enabled && steps < MAX_SAMPLES)
      ++steps;
  }
  void begin(cudaStream_t st, int stage)
  {
    if (enabled && steps > 0 && steps <= MAX_SAMPLES) {
      cudaEventRecord(ev[steps - 1][stage][0], st);
      used[steps - 1][stage] = true;
    }
  }
  void end(cudaStream_t st, int stage)
  {
    if (enabled && steps > 0 && steps <= MAX_SAMPLES)
      cudaEventRecord(ev[steps - 1][stage][1], st);
  }
  // synchronises; ms_sum[stage] = total milliseconds, counts[stage] = number of samples
  void read(float* ms_sum, int* counts);
};

} // namespace b2

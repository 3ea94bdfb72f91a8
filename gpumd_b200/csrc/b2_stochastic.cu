// b2_stochastic.cu -- the thermostats / barostat SURVEY.md 8f ranks third: Langevin (nvt_lan), BAOAB
// Langevin (nvt_bao) and the Berendsen barostat (npt_ber).
//
//   b200md_langevin_*          <- initialize_curand_states + gpu_langevin + gpu_find_momentum +
//                                 gpu_correct_momentum, src/integrate/langevin_utilities.cuh:26-127
//                                 (Ensemble_LAN::integrate_nvt_lan_half ensemble_lan.cu:92-124,
//                                 Ensemble_BAO::integrate_nvt_lan ensemble_bao.cu:91-120)
//   b200md_baoab_operator      <- gpu_operator_A / gpu_operator_B, ensemble_bao.cu:190-300
//   b200md_berendsen_pressure  <- cpu_pressure_{isotropic,orthogonal,triclinic} +
//                                 gpu_pressure_*, ensemble_ber.cu:88-172,237-285, npt_utilities.cuh:23-76
//
// The per-atom generator is cuRAND's XORWOW exactly as the reference uses it -- curand_init(seed, n, 0)
// and three curand_normal_double draws per atom per call -- so a run seeded like the reference
// (its -DDEBUG build passes glibc's first rand() = 1804289383) follows the reference's noise stream
// draw for draw.  That stream is pinned: tests/curand_oracle.py restates XORWOW (equal bit for bit to
// cuRAND built for the host), and tests/test_gpu_langevin_steps.py holds these kernels, heat_lan's and
// the driver's seeding to it, x, y, z per atom, the second Box-Muller value carried across calls, 64-bit
// seeds and padded layouts included (within a few ulp: the device's sincospi is not the host's sin).
// The momentum sums are one fused deterministic reduction (the block stage and ticket of b2_reduce.cuh)
// instead of the reference's <<<4,1024>>> strided loops.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_reduce.cuh"
#include <cmath>
#include <curand_kernel.h>
#include <new>

namespace b2 {
namespace {

constexpr int BLK = 256;

__global__ void __launch_bounds__(BLK) k_init_states(curandState* state, int n, unsigned long long seed)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    curand_init(seed, i, 0, &state[i]);
}

// v <- c1 v + c2 / sqrt(m) xi, and per-block partial sums of m v (x, y, z) and m
__global__ void __launch_bounds__(BLK) k_langevin(
  curandState* g_state, int n, int stride, double c1, double c2, const double* __restrict__ mass,
  double* vel, double* partial, unsigned int* ticket, double* mom4)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double t[4] = {0.0, 0.0, 0.0, 0.0};
  if (i < n) {
    curandState state = g_state[i];
    const double m = mass[i];
    const double c2m = c2 * sqrt(1.0 / m);
    const size_t N = (size_t)stride;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const double v = c1 * vel[d * N + i] + c2m * curand_normal_double(&state);
      vel[d * N + i] = v;
      t[d] = m * v;
    }
    t[3] = m;
    g_state[i] = state;
  }
  b2_block_totals<4, BLK>(t, partial + blockIdx.x, gridDim.x);
  // the blocks in index order by one thread per row (the order of b2_grid_totals differs)
  if (b2_last_block(ticket) && threadIdx.x < 4) {
    double v = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b)
      v += partial[(size_t)threadIdx.x * gridDim.x + b];
    mom4[threadIdx.x] = v;
  }
}

__global__ void __launch_bounds__(BLK) k_correct_momentum(int n, int stride, const double* mom4, double* vel)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double inv = 1.0 / mom4[3];
    const size_t N = (size_t)stride;
    vel[i] -= mom4[0] * inv;
    vel[N + i] -= mom4[1] * inv;
    vel[2 * N + i] -= mom4[2] * inv;
  }
}

// BAOAB half operators: A: x += v dt/2 (fixed atoms: v = 0), B: v += f/m dt/2 (fixed atoms: v = 0)
__global__ void __launch_bounds__(BLK) k_baoab(
  int which, int n, int stride, double dt, const double* __restrict__ mass, double* pos, double* vel,
  const double* __restrict__ f, const int* __restrict__ label, int fixed_group)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const size_t N = (size_t)stride;
  const double half = dt * 0.5;
  const bool fixed = label && label[i] == fixed_group;
  if (which == 0) {
#pragma unroll
    for (int d = 0; d < 3; ++d)
      pos[d * N + i] += (fixed ? 0.0 : vel[d * N + i]) * half;
  } else {
    const double minv = 1.0 / mass[i];
#pragma unroll
    for (int d = 0; d < 3; ++d)
      vel[d * N + i] = fixed ? 0.0 : vel[d * N + i] + f[d * N + i] * minv * half;
  }
}

__global__ void __launch_bounds__(BLK) k_scale_positions(
  int n, int stride, double m0, double m1, double m2, double m3, double m4, double m5, double m6,
  double m7, double m8, int diagonal, double* pos)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const size_t N = (size_t)stride;
  const double x = pos[i], y = pos[N + i], z = pos[2 * N + i];
  if (diagonal) {
    pos[i] = x * m0;
    pos[N + i] = y * m4;
    pos[2 * N + i] = z * m8;
  } else {
    pos[i] = m0 * x + m1 * y + m2 * z;
    pos[N + i] = m3 * x + m4 * y + m5 * z;
    pos[2 * N + i] = m6 * x + m7 * y + m8 * z;
  }
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_langevin {
  DevBuf<curandState> state;
  DevBuf<double> partial, mom4;
  DevBuf<unsigned int> ticket;
  int n = 0;
};

extern "C" {

int b200md_langevin_create(int n, unsigned long long seed, b200md_langevin** out)
{
  if (n <= 0 || !out) {
    set_error("b200md_langevin_create: bad argument");
    return B200MD_ERR_ARG;
  }
  b200md_langevin* p = new (std::nothrow) b200md_langevin;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->n = n;
  const int g = grid_for(n, BLK);
  if (p->state.reserve(n) != cudaSuccess || p->partial.reserve((size_t)g * 4) != cudaSuccess ||
      p->mom4.reserve(4) != cudaSuccess || p->ticket.reserve(1) != cudaSuccess) {
    set_error("out of device memory (Langevin generator states)");
    delete p;
    return B200MD_ERR_CUDA;
  }
  cudaMemset(p->ticket.p, 0, sizeof(unsigned int));
  k_init_states<<<g, BLK>>>(p->state.p, n, seed);
  ++g_launch_count;
  if (cudaDeviceSynchronize() != cudaSuccess) {
    set_error("curand_init failed");
    delete p;
    return B200MD_ERR_CUDA;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_langevin_destroy(b200md_langevin* p) { delete p; }

int b200md_langevin_apply(
  b200md_langevin* p, int n, int stride, double c1, double c2, const double* d_mass,
  double* d_velocity, void* stream)
{
  if (n != p->n) {
    set_error("b200md_langevin_apply: atom count differs from the one given at creation");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(n, BLK);
  k_langevin<<<g, BLK, 0, st>>>(
    p->state.p, n, stride, c1, c2, d_mass, d_velocity, p->partial.p, p->ticket.p, p->mom4.p);
  B2_LAUNCHED();
  k_correct_momentum<<<g, BLK, 0, st>>>(n, stride, p->mom4.p, d_velocity);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_baoab_operator(
  int which, int n, int stride, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, const int* d_group_label, int fixed_group, void* stream)
{
  if (which != 0 && which != 1) {
    set_error("b200md_baoab_operator: which must be 0 (A) or 1 (B)");
    return B200MD_ERR_ARG;
  }
  k_baoab<<<grid_for(n, BLK), BLK, 0, (cudaStream_t)stream>>>(
    which, n, stride, time_step, d_mass, d_position, d_velocity, d_force,
    fixed_group >= 0 ? d_group_label : nullptr, fixed_group);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_berendsen_pressure(
  int n, int stride, int num_components, const double target_pressure[6],
  const double pressure_coupling[6], const int deform[3], const double deform_rate[3],
  const int pbc[3], double h[9], const double* d_thermo, double* d_position, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  double p[6];
  // the box lives on the host and is passed by value to every kernel: like the reference
  // (ensemble_ber.cu:100,140,153) this is a blocking read of the six stress components
  B2_CUDA(cudaMemcpyAsync(p, d_thermo + 2, sizeof(double) * 6, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  double mu[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  int diagonal = 1;
  const double* p0 = target_pressure;
  const double* pc = pressure_coupling;
  if (num_components == 1) {
    const double s = 1.0 - pc[0] * (p0[0] - (p[0] + p[1] + p[2]) * 0.3333333333333333);
    mu[0] = mu[4] = mu[8] = s;
    h[0] *= s;
    h[4] *= s;
    h[8] *= s;
  } else if (num_components == 3) {
    for (int d = 0; d < 3; ++d) {
      double s = 1.0;
      if (deform && deform[d])
        s = (h[4 * d] + deform_rate[d]) / h[4 * d];
      else if (pbc[d])
        s = 1.0 - pc[d] * (p0[d] - p[d]);
      mu[4 * d] = s;
      h[4 * d] *= s;
    }
  } else if (num_components == 6) {
    // p0 / pc in Voigt order xx yy zz yz xz xy; thermo order is xx yy zz xy xz yz
    diagonal = 0;
    mu[0] = 1.0 - pc[0] * (p0[0] - p[0]);
    mu[4] = 1.0 - pc[1] * (p0[1] - p[1]);
    mu[8] = 1.0 - pc[2] * (p0[2] - p[2]);
    mu[3] = mu[1] = -pc[5] * (p0[5] - p[3]);
    mu[6] = mu[2] = -pc[4] * (p0[4] - p[4]);
    mu[7] = mu[5] = -pc[3] * (p0[3] - p[5]);
    double old[9];
    for (int k = 0; k < 9; ++k)
      old[k] = h[k];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) {
        double t = 0.0;
        for (int k = 0; k < 3; ++k)
          t += mu[r * 3 + k] * old[k * 3 + c];
        h[r * 3 + c] = t;
      }
  } else {
    set_error("b200md_berendsen_pressure: num_components must be 1, 3 or 6");
    return B200MD_ERR_ARG;
  }
  k_scale_positions<<<grid_for(n, BLK), BLK, 0, st>>>(
    n, stride, mu[0], mu[1], mu[2], mu[3], mu[4], mu[5], mu[6], mu[7], mu[8], diagonal, d_position);
  B2_LAUNCHED();
  return B200MD_OK;
}

} // extern "C"

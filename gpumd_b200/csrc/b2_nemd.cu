// b2_nemd.cu -- direct NEMD: the heat baths of heat_lan / heat_nhc / heat_bdp and the group-averaged
// `compute` output.
//
//   b200md_heat_bath_*     <- Ensemble_LAN::integrate_heat_lan_half (ensemble_lan.cu:43-85,128-195),
//                             Ensemble_NHC::integrate_heat_nhc_1/_2 (ensemble_nhc.cu:52-91,239-326),
//                             Ensemble_BDP::integrate_heat_bdp_2 (ensemble_bdp.cu:50-62,103-149) with
//                             find_vc_and_ke / scale_velocity_local (ensemble.cu:700-879)
//   b200md_group_compute_* <- Compute::preprocess / process / output_results (compute.cu:31-660)
//
// The reference copies the group kinetic energies to the host twice per half step, allocates device
// vectors on every call and reduces with one block per group.  Here the source and sink atoms are one
// index list; a single kernel reduces it with per-block partials, and the last block to finish sums
// them in a fixed order and, in the same launch, runs the chains / the stochastic rescaling and
// accumulates the energy transferred.  Nothing is copied to the host inside a step, nothing is
// allocated after creation, and every sum has a fixed order (run-to-run identical).
#include "../../include/b200md.h"
#include "b2_bdp.cuh"
#include "b2_host.h"
#include "b2_integrate.cuh"
#include "b2_reduce.cuh"
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <curand_kernel.h>
#include <new>
#include <vector>

namespace b2 {
namespace {

constexpr int BLK = 256;
constexpr double K_B = 8.617343e-5; // src/utilities/common.cuh:21

// device-resident record of one heat bath (kind 0 lan, 1 nhc, 2 bdp)
struct HeatState {
  double chain[2][12]; // heat_nhc: eta[4], v_eta[4], Q[4] of the source / sink chains
  double stat[2][5];   // last reduction: sum m, sum m v (3), sum m v^2 per group
  double vc[2][3];     // centre-of-mass velocities
  double factor[2];    // scale factors of the last rescaling
  double energy[2];    // energy transferred from the system to the source / sink baths (eV)
};

__global__ void __launch_bounds__(BLK) k_heat_init_states(
  curandState* state, int n_source, int n_total, unsigned long long seed_source,
  unsigned long long seed_sink)
{
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m < n_source)
    curand_init(seed_source, m, 0, &state[m]);
  else if (m < n_total)
    curand_init(seed_sink, m - n_source, 0, &state[m]);
}

// heat_lan: local Langevin half kick v <- c1 v + c2[g] / sqrt(m) xi on the source (g = 0) and sink
// (g = 1) atoms, generator state indexed by the position within the group (gpu_langevin with groups,
// langevin_utilities.cuh:127-149).  energy[g] += 1/2 sum m (v_before^2 - v_after^2).
__global__ void __launch_bounds__(BLK) k_heat_lan(
  curandState* g_state, const int* __restrict__ atoms, int n_source, int n_total, int stride,
  double c1, double c2_source, double c2_sink, const double* __restrict__ mass, double* vel,
  double* partial, unsigned int* ticket, HeatState* hs)
{
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  double t[2] = {0.0, 0.0};
  if (m < n_total) {
    const int g = m < n_source ? 0 : 1;
    const int i = atoms[m];
    curandState state = g_state[m];
    const double ms = mass[i];
    const double c2m = (g == 0 ? c2_source : c2_sink) * sqrt(1.0 / ms);
    const size_t N = (size_t)stride;
    double de = 0.0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const double v0 = vel[d * N + i];
      const double v1 = c1 * v0 + c2m * curand_normal_double(&state);
      vel[d * N + i] = v1;
      de += __dmul_rn(v0, v0) - __dmul_rn(v1, v1); // no FMA: an unchanged velocity adds exactly 0
    }
    g_state[m] = state;
    t[g] = 0.5 * ms * de;
  }
  b2_block_totals<2, BLK>(t, partial + blockIdx.x, gridDim.x);
  if (b2_last_block(ticket))
    b2_grid_totals<2, BLK>(partial, [&](int g, double v) { hs->energy[g] += v; });
}

// the serial bodies of the reduction tail, kept out of line so that they do not set the register
// allocation of the reduction itself
__device__ __noinline__ double heat_chain(double* state, double ek2, double dof, double kT, double dt_half)
{
  return b2_nhc_chain(state, ek2, dof, kT, dt_half);
}

__device__ __noinline__ double heat_resamplekin(B2BdpState* mt, double kk, double sigma, int ndeg, double taut)
{
  return b2_resamplekin(*mt, kk, sigma, ndeg, taut);
}

// heat_nhc / heat_bdp: per group sum m, m v, m v^2 (gpu_find_vc_and_ke, ensemble.cu:700-782); the last
// block turns them into the centre-of-mass velocity and relative kinetic energy and runs the two
// chains (kind 1) or the two resamplekin draws, source first (kind 2), leaving the factors in hs.
__global__ void __launch_bounds__(BLK) k_heat_reduce(
  int kind, const int* __restrict__ atoms, int n_source, int n_total, int stride,
  const double* __restrict__ mass, const double* __restrict__ vel, double* partial,
  unsigned int* ticket, HeatState* hs, B2BdpState* mt, double kT_source, double kT_sink,
  double dt_half, double coupling)
{
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  double t[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (m < n_total) {
    const int i = atoms[m];
    const size_t N = (size_t)stride;
    const double ms = mass[i], vx = vel[i], vy = vel[N + i], vz = vel[2 * N + i];
    const int o = m < n_source ? 0 : 5;
#pragma unroll
    for (int k = 0; k < 10; k += 5)
      if (k == o) {
        t[k] = ms;
        t[k + 1] = ms * vx;
        t[k + 2] = ms * vy;
        t[k + 3] = ms * vz;
        t[k + 4] = (vx * vx + vy * vy + vz * vz) * ms;
      }
  }
  b2_block_totals<10, BLK>(t, partial + blockIdx.x, gridDim.x);
  if (!b2_last_block(ticket))
    return;
  __shared__ double tot[10];
  b2_grid_totals<10, BLK>(partial, [&](int k, double v) { tot[k] = v; });
  if (threadIdx.x >= 2)
    return;
  double ek2[2];
  const int size[2] = {n_source, n_total - n_source};
  for (int g = 0; g < 2; ++g) {
    const double* s = tot + 5 * g;
    const double mc = s[0];
    const double vx = s[1] / mc, vy = s[2] / mc, vz = s[3] / mc;
    ek2[g] = s[4] - mc * (vx * vx + vy * vy + vz * vz); // relative kinetic energy times 2
    if (g == (int)threadIdx.x) {
      for (int k = 0; k < 5; ++k)
        hs->stat[g][k] = s[k];
      hs->vc[g][0] = vx;
      hs->vc[g][1] = vy;
      hs->vc[g][2] = vz;
    }
  }
  if (kind == 1) { // integrate_heat_nhc_1/_2, ensemble_nhc.cu:264-276: the two chains side by side
    const int g = threadIdx.x;
    const double e2 = g == 0 ? ek2[0] : ek2[1];
    const double f = heat_chain(hs->chain[g], e2, 3.0 * (g == 0 ? size[0] : size[1]),
                                g == 0 ? kT_source : kT_sink, dt_half);
    hs->energy[g] += e2 * 0.5 * (1.0 - f * f);
    hs->factor[g] = f;
  } else if (threadIdx.x == 0) { // integrate_heat_bdp_2, ensemble_bdp.cu:116-145: one stream, source first
    for (int g = 0; g < 2; ++g) {
      const double kT = g == 0 ? kT_source : kT_sink;
      const int dN = 3 * (size[g] - 1);
      const double ek = ek2[g] * 0.5;
      const double f = sqrt(heat_resamplekin(mt, ek, dN * kT * 0.5, dN, coupling) / ek);
      hs->energy[g] += ek * (1.0 - f * f);
      hs->factor[g] = f;
    }
  }
}

// v <- vc + f (v - vc) on the source and sink atoms (gpu_scale_velocity, ensemble.cu:805-879)
__global__ void __launch_bounds__(BLK) k_heat_scale(
  const int* __restrict__ atoms, int n_source, int n_total, int stride, const HeatState* hs, double* vel)
{
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_total)
    return;
  const int g = m < n_source ? 0 : 1;
  const int i = atoms[m];
  const size_t N = (size_t)stride;
  const double f = hs->factor[g];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double vc = hs->vc[g][d];
    vel[d * N + i] = vc + f * (vel[d * N + i] - vc);
  }
}

// ---- compute: group sums ----------------------------------------------------------------------
// Columns of one sample in the reference's fixed order: temperature, potential, force x3, virial x9
// (xx xy xz yx yy yz zx zy zz), jp x3, jk x3, momentum x3 (compute.cu:365-518).
constexpr int NQ = 23;
__constant__ int c_virial_row[9] = {0, 3, 4, 6, 1, 5, 7, 8, 2};

// Segmented reduction: the group contents are cut into chunks of at most CHUNK entries, and each
// (chunk, group) overlap is one segment that one block reduces into partial[q][segment].  Many
// small groups give many short segments, one large group many full ones: all SMs stay busy either
// way, and empty groups have no segment.
constexpr int CHUNK = 4 * BLK;

__global__ void __launch_bounds__(BLK) k_group_partial(
  unsigned mask, const int* __restrict__ seg_begin, const int* __restrict__ contents, int stride,
  const double* __restrict__ mass, const double* __restrict__ pe, const double* __restrict__ f,
  const double* __restrict__ W, const double* __restrict__ vel, double* partial)
{
  const int s = blockIdx.x;
  const int begin = seg_begin[s], end = seg_begin[s + 1];
  const size_t N = (size_t)stride;
  double t[NQ];
#pragma unroll
  for (int q = 0; q < NQ; ++q)
    t[q] = 0.0;
  for (int k = begin + threadIdx.x; k < end; k += BLK) {
    const int i = contents[k];
    double m = 0.0, vx = 0.0, vy = 0.0, vz = 0.0, p = 0.0;
    if (mask & (B200MD_COMPUTE_TEMPERATURE | B200MD_COMPUTE_JK | B200MD_COMPUTE_MOMENTUM))
      m = mass[i];
    if (mask & (B200MD_COMPUTE_TEMPERATURE | B200MD_COMPUTE_JP | B200MD_COMPUTE_JK |
                B200MD_COMPUTE_MOMENTUM)) {
      vx = vel[i];
      vy = vel[N + i];
      vz = vel[2 * N + i];
    }
    if (mask & (B200MD_COMPUTE_POTENTIAL | B200MD_COMPUTE_JK))
      p = pe[i];
    const double v2 = vx * vx + vy * vy + vz * vz;
    if (mask & B200MD_COMPUTE_TEMPERATURE)
      t[0] += m * v2 / (3.0 * K_B); // find_per_atom_temperature, compute.cu:85-100
    if (mask & B200MD_COMPUTE_POTENTIAL)
      t[1] += p;
    if (mask & B200MD_COMPUTE_FORCE) {
      t[2] += f[i];
      t[3] += f[N + i];
      t[4] += f[2 * N + i];
    }
    if (mask & (B200MD_COMPUTE_VIRIAL | B200MD_COMPUTE_JP)) {
      double w[9];
#pragma unroll
      for (int c = 0; c < 9; ++c)
        w[c] = W[c_virial_row[c] * N + i];
      if (mask & B200MD_COMPUTE_VIRIAL) {
#pragma unroll
        for (int c = 0; c < 9; ++c)
          t[5 + c] += w[c];
      }
      if (mask & B200MD_COMPUTE_JP) { // find_per_atom_jp, compute.cu:102-125
        t[14] += w[0] * vx + w[1] * vy + w[2] * vz;
        t[15] += w[3] * vx + w[4] * vy + w[5] * vz;
        t[16] += w[6] * vx + w[7] * vy + w[8] * vz;
      }
    }
    if (mask & B200MD_COMPUTE_JK) { // find_per_atom_jk, compute.cu:127-149
      const double e = m * v2 * 0.5 + p;
      t[17] += vx * e;
      t[18] += vy * e;
      t[19] += vz * e;
    }
    if (mask & B200MD_COMPUTE_MOMENTUM) {
      t[20] += vx * m;
      t[21] += vy * m;
      t[22] += vz * m;
    }
  }
  b2_block_totals<NQ, BLK>(t, partial + s, gridDim.x);
}

// one warp per (column, group): the group's segments in order, added to the running sum
__global__ void __launch_bounds__(BLK) k_group_finish(
  int num_groups, int num_cols, int num_segments, const int* __restrict__ col_q,
  const int* __restrict__ group_seg, const double* __restrict__ partial, double* sum)
{
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= num_groups * num_cols)
    return;
  const int c = warp / num_groups, g = warp - c * num_groups;
  const double v = b2_warp_ordered(
    partial + (size_t)col_q[c] * num_segments + group_seg[g], group_seg[g + 1] - group_seg[g]);
  if ((threadIdx.x & 31) == 0)
    sum[warp] += v; // column-major blocks of num_groups, as gpu_group_sum
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_heat_bath {
  int kind = 0, n_source = 0, n_total = 0, n = 0;
  double c1 = 0.0, c2_source = 0.0, c2_sink = 0.0, kT_source = 0.0, kT_sink = 0.0, time_step = 0.0,
         coupling = 0.0;
  DevBuf<int> atoms;
  DevBuf<curandState> state;
  DevBuf<double> partial;
  DevBuf<unsigned int> ticket;
  DevBuf<HeatState> hs;
  DevBuf<B2BdpState> mt;
};

struct b200md_group_compute {
  int num_groups = 0, num_segments = 0, num_cols = 0, n = 0;
  unsigned mask = 0;
  std::vector<int> sizes;
  DevBuf<int> contents, seg_begin, group_seg, col_q;
  DevBuf<double> partial, sum;
};

namespace b2 {
namespace {

__global__ void k_heat_seed_mt(B2BdpState* s, unsigned seed)
{
  if (threadIdx.x == 0 && blockIdx.x == 0)
    b2_mt_seed(*s, seed);
}

// the group with id `id` of a Group::find_contents list, or false if out of range
bool group_range(int num_groups, const int* sizes, int id, int* offset)
{
  if (id < 0 || id >= num_groups)
    return false;
  int o = 0;
  for (int k = 0; k < id; ++k)
    o += sizes[k];
  *offset = o;
  return true;
}

} // namespace
} // namespace b2

extern "C" {

int b200md_heat_bath_create(
  int kind, int n, int num_groups, const int* group_sizes, const int* contents, int source, int sink,
  double T, double Tc, double dT, double time_step, unsigned long long seed_source,
  unsigned long long seed_sink, b200md_heat_bath** out)
{
  int off_source = 0, off_sink = 0;
  if (kind < 0 || kind > 2 || n <= 0 || !group_sizes || !contents || !out ||
      !group_range(num_groups, group_sizes, source, &off_source) ||
      !group_range(num_groups, group_sizes, sink, &off_sink) || source == sink) {
    set_error("b200md_heat_bath_create: bad kind, atom count or source / sink group");
    return B200MD_ERR_ARG;
  }
  long long total = 0;
  for (int g = 0; g < num_groups; ++g) {
    if (group_sizes[g] < 0) {
      set_error("b200md_heat_bath_create: negative group size");
      return B200MD_ERR_ARG;
    }
    total += group_sizes[g];
  }
  const int ns = group_sizes[source], nk = group_sizes[sink];
  if (total > n || ns < 1 || nk < 1 || (kind == 2 && (ns < 2 || nk < 2)) ||
      (kind == 2 && 3LL * (ns > nk ? ns : nk) > 2147483647LL) || !(T > 0.0) || !(Tc >= 1.0) ||
      !(dT < T && dT > -T)) {
    set_error("b200md_heat_bath_create: empty source / sink (heat_bdp: fewer than two atoms), "
              "T <= 0, Tc < 1 or |dT| >= T");
    return B200MD_ERR_ARG;
  }
  std::vector<int> atoms((size_t)ns + nk);
  for (int m = 0; m < ns; ++m)
    atoms[m] = contents[off_source + m];
  for (int m = 0; m < nk; ++m)
    atoms[ns + m] = contents[off_sink + m];
  for (int i : atoms)
    if (i < 0 || i >= n) {
      set_error("b200md_heat_bath_create: atom index out of range in contents");
      return B200MD_ERR_ARG;
    }
  b200md_heat_bath* p = new (std::nothrow) b200md_heat_bath;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->kind = kind;
  p->n = n;
  p->n_source = ns;
  p->n_total = ns + nk;
  p->time_step = time_step;
  p->coupling = Tc;
  p->kT_source = K_B * (T + dT);
  p->kT_sink = K_B * (T - dT);
  p->c1 = exp(-0.5 / Tc); // ensemble_lan.cu:71-73
  p->c2_source = sqrt((1 - p->c1 * p->c1) * p->kT_source);
  p->c2_sink = sqrt((1 - p->c1 * p->c1) * p->kT_sink);
  const int g = grid_for(p->n_total, BLK);
  HeatState h = {};
  // Ensemble_NHC::Ensemble_NHC (heat), ensemble_nhc.cu:70-86: Q[0] scaled by 3 |group|
  const double tau = time_step * Tc;
  for (int c = 0; c < 2; ++c) {
    const double kT = c == 0 ? p->kT_source : p->kT_sink;
    double* s = h.chain[c];
    s[4] = s[6] = 1.0;
    s[5] = s[7] = -1.0;
    for (int k = 0; k < 4; ++k)
      s[8 + k] = kT * tau * tau;
    s[8] *= 3.0 * (c == 0 ? ns : nk);
  }
  h.factor[0] = h.factor[1] = 1.0;
  if (p->atoms.reserve(atoms.size()) != cudaSuccess || p->partial.reserve((size_t)g * 10) != cudaSuccess ||
      p->ticket.reserve(1) != cudaSuccess || p->hs.reserve(1) != cudaSuccess ||
      (kind == 0 && p->state.reserve(p->n_total) != cudaSuccess) ||
      (kind == 2 && p->mt.reserve(1) != cudaSuccess)) {
    set_error("out of device memory (heat bath)");
    delete p;
    return B200MD_ERR_CUDA;
  }
  cudaMemcpy(p->atoms.p, atoms.data(), atoms.size() * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(p->hs.p, &h, sizeof h, cudaMemcpyHostToDevice);
  cudaMemset(p->ticket.p, 0, sizeof(unsigned int));
  if (kind == 0) {
    k_heat_init_states<<<g, BLK>>>(p->state.p, ns, p->n_total, seed_source, seed_sink);
    ++g_launch_count;
  } else if (kind == 2) {
    k_heat_seed_mt<<<1, 32>>>(p->mt.p, (unsigned)seed_source);
    ++g_launch_count;
  }
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error(std::string("b200md_heat_bath_create: ") + cudaGetErrorString(e));
    delete p;
    return B200MD_ERR_CUDA;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_heat_bath_destroy(b200md_heat_bath* p) { delete p; }

int b200md_heat_bath_half(
  b200md_heat_bath* p, int after_vv2, int n, int stride, const double* d_mass, double* d_velocity,
  void* stream)
{
  if (!p || n != p->n || stride < n) {
    set_error("b200md_heat_bath_half: atom count differs from the one given at creation");
    return B200MD_ERR_ARG;
  }
  if (p->kind == 2 && !after_vv2) // heat_bdp rescales after the second half step only
    return B200MD_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(p->n_total, BLK);
  if (p->kind == 0) {
    k_heat_lan<<<g, BLK, 0, st>>>(
      p->state.p, p->atoms.p, p->n_source, p->n_total, stride, p->c1, p->c2_source, p->c2_sink, d_mass,
      d_velocity, p->partial.p, p->ticket.p, p->hs.p);
    B2_LAUNCHED();
    return B200MD_OK;
  }
  k_heat_reduce<<<g, BLK, 0, st>>>(
    p->kind, p->atoms.p, p->n_source, p->n_total, stride, d_mass, d_velocity, p->partial.p, p->ticket.p,
    p->hs.p, p->mt.p, p->kT_source, p->kT_sink, 0.5 * p->time_step, p->coupling);
  B2_LAUNCHED();
  k_heat_scale<<<g, BLK, 0, st>>>(p->atoms.p, p->n_source, p->n_total, stride, p->hs.p, d_velocity);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_heat_bath_energy(b200md_heat_bath* p, double out2[2], void* stream)
{
  if (!p || !out2) {
    set_error("b200md_heat_bath_energy: null handle or output");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(cudaMemcpyAsync(out2, reinterpret_cast<const char*>(p->hs.p) + offsetof(HeatState, energy),
                          2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200MD_OK;
}

int b200md_heat_bath_state(b200md_heat_bath* p, double* out, void* stream)
{
  if (!p || !out) {
    set_error("b200md_heat_bath_state: null handle or output");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  HeatState h;
  B2_CUDA(cudaMemcpyAsync(&h, p->hs.p, sizeof h, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const double* src[5] = {&h.chain[0][0], &h.stat[0][0], &h.vc[0][0], h.factor, h.energy};
  const int len[5] = {24, 10, 6, 2, 2};
  for (int k = 0, o = 0; k < 5; o += len[k], ++k)
    for (int j = 0; j < len[k]; ++j)
      out[o + j] = src[k][j];
  return B200MD_OK;
}

int b200md_group_compute_create(
  int n, int num_groups, const int* group_sizes, const int* contents, unsigned what_mask,
  b200md_group_compute** out)
{
  if (n <= 0 || num_groups <= 0 || !group_sizes || !contents || !out || what_mask == 0 ||
      (what_mask & ~(unsigned)B200MD_COMPUTE_ALL)) {
    set_error("b200md_group_compute_create: bad atom count, groups or quantity mask");
    return B200MD_ERR_ARG;
  }
  long long total = 0;
  for (int g = 0; g < num_groups; ++g) {
    if (group_sizes[g] < 0) {
      set_error("b200md_group_compute_create: negative group size");
      return B200MD_ERR_ARG;
    }
    total += group_sizes[g];
  }
  if (total > n) {
    set_error("b200md_group_compute_create: the groups hold more atoms than the system");
    return B200MD_ERR_ARG;
  }
  for (long long k = 0; k < total; ++k)
    if (contents[k] < 0 || contents[k] >= n) {
      set_error("b200md_group_compute_create: atom index out of range in contents");
      return B200MD_ERR_ARG;
    }
  // segments: every overlap of a chunk of CHUNK entries with a group; a group's segments are
  // consecutive, group_seg[g] .. group_seg[g+1]
  std::vector<int> seg_begin, group_seg(num_groups + 1, 0);
  int pos = 0;
  for (int g = 0; g < num_groups; ++g) {
    group_seg[g] = (int)seg_begin.size();
    const int end = pos + group_sizes[g];
    while (pos < end) {
      seg_begin.push_back(pos);
      pos = std::min(end, (pos / CHUNK + 1) * CHUNK);
    }
  }
  group_seg[num_groups] = (int)seg_begin.size();
  const int num_segments = (int)seg_begin.size();
  seg_begin.push_back(pos);
  // which of the NQ quantities each selected column is, in the reference's order
  const int width[7] = {1, 1, 3, 9, 3, 3, 3};
  std::vector<int> col_q;
  for (int k = 0, q = 0; k < 7; q += width[k], ++k)
    if (what_mask & (1u << k))
      for (int j = 0; j < width[k]; ++j)
        col_q.push_back(q + j);
  b200md_group_compute* p = new (std::nothrow) b200md_group_compute;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->n = n;
  p->num_groups = num_groups;
  p->num_segments = num_segments;
  p->num_cols = (int)col_q.size();
  p->mask = what_mask;
  p->sizes.assign(group_sizes, group_sizes + num_groups);
  const size_t sums = (size_t)p->num_cols * num_groups;
  if (p->contents.reserve(total > 0 ? total : 1) != cudaSuccess ||
      p->seg_begin.reserve(seg_begin.size()) != cudaSuccess ||
      p->group_seg.reserve(group_seg.size()) != cudaSuccess || p->col_q.reserve(col_q.size()) != cudaSuccess ||
      p->partial.reserve((size_t)(num_segments > 0 ? num_segments : 1) * NQ) != cudaSuccess ||
      p->sum.reserve(sums) != cudaSuccess) {
    set_error("out of device memory (compute)");
    delete p;
    return B200MD_ERR_CUDA;
  }
  cudaMemcpy(p->contents.p, contents, total * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(p->seg_begin.p, seg_begin.data(), seg_begin.size() * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(p->group_seg.p, group_seg.data(), group_seg.size() * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(p->col_q.p, col_q.data(), col_q.size() * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemset(p->sum.p, 0, sums * sizeof(double));
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error(std::string("b200md_group_compute_create: ") + cudaGetErrorString(e));
    delete p;
    return B200MD_ERR_CUDA;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_group_compute_destroy(b200md_group_compute* p) { delete p; }

int b200md_group_compute_columns(const b200md_group_compute* p) { return p ? p->num_cols : -1; }

int b200md_group_compute_sample(
  b200md_group_compute* p, int n, int stride, const double* d_mass, const double* d_potential,
  const double* d_force, const double* d_virial, const double* d_velocity, void* stream)
{
  if (!p || n != p->n || stride < n) {
    set_error("b200md_group_compute_sample: atom count differs from the one given at creation");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (p->num_segments > 0) {
    k_group_partial<<<p->num_segments, BLK, 0, st>>>(
      p->mask, p->seg_begin.p, p->contents.p, stride, d_mass, d_potential, d_force, d_virial, d_velocity,
      p->partial.p);
    B2_LAUNCHED();
  }
  const long long threads = 32LL * p->num_cols * p->num_groups;
  k_group_finish<<<grid_for(threads, BLK), BLK, 0, st>>>(
    p->num_groups, p->num_cols, p->num_segments, p->col_q.p, p->group_seg.p, p->partial.p, p->sum.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_group_compute_take(b200md_group_compute* p, int num_samples, double* out, void* stream)
{
  if (!p || !out || num_samples <= 0) {
    set_error("b200md_group_compute_take: null handle or output, or num_samples not positive");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t sums = (size_t)p->num_cols * p->num_groups;
  B2_CUDA(cudaMemcpyAsync(out, p->sum.p, sums * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemsetAsync(p->sum.p, 0, sums * sizeof(double), st));
  B2_CUDA(cudaStreamSynchronize(st));
  // Compute::output_results, compute.cu:540-561: average over the samples, temperature per atom
  const bool temperature = p->mask & B200MD_COMPUTE_TEMPERATURE;
  for (size_t k = 0; k < sums; ++k) {
    out[k] /= num_samples;
    if (temperature && k < (size_t)p->num_groups)
      out[k] /= p->sizes[k];
  }
  return B200MD_OK;
}

} // extern "C"

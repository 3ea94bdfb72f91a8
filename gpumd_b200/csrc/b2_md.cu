// b2_md.cu -- LJ potential, Force::compute pre-steps, velocity-Verlet and the fused thermo
// reduction of libb200md; C-ABI entry points b200md_lj_*, b200md_apply_pbc,
// b200md_zero_properties, b200md_velocity_verlet, b200md_find_thermo, b200md_scale_velocity.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_bdp.cuh"
#include "b2_integrate.cuh"
#include "b2_lj.cuh"
#include "b2_neighbor_host.h"
#include "b2_nep.cuh" // b2_body_unpack
#include "b2_reduce.cuh"
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

namespace b2 {
namespace {

constexpr int BLK = 256;
constexpr int THERMO_BLK = 256;
constexpr int THERMO_MAX_BLOCKS = 132 * 8; // H100 SXM: 132 SMs, a few resident blocks each

__global__ void __launch_bounds__(128) k_lj(B2LjView P, B2Box box)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_lj(i, P, box);
}

__global__ void __launch_bounds__(BLK) k_unpack_lj(
  int n, const int* __restrict__ perm, const double* __restrict__ acc, double* pe, double* force,
  double* virial)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    b2_body_unpack(i, n, perm, acc, pe, force, virial);
}

__global__ void __launch_bounds__(BLK) k_apply_pbc(int n, B2Box box, double* x, double* y, double* z)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    b2_body_apply_pbc(i, n, box, x, y, z);
}

// 13 contiguous double arrays per atom: grid-stride over the flat range with 16-byte stores
__global__ void __launch_bounds__(BLK) k_zero(size_t count, double* p)
{
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
    p[i] = 0.0;
}

__global__ void __launch_bounds__(BLK) k_vv(
  int n, int stride, int step1, double dt, const double* __restrict__ mass, double* pos,
  double* vel, const double* __restrict__ f)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    b2_body_vv(i, stride, step1 != 0, dt, mass, pos, vel, f);
}

__global__ void __launch_bounds__(BLK) k_vv_groups(
  int n, int stride, int step1, double dt, const double* __restrict__ mass, double* pos,
  double* vel, const double* __restrict__ f, const int* __restrict__ label, int fixed_group,
  int move_group, double mvx, double mvy, double mvz)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const double mv[3] = {mvx, mvy, mvz};
  if (i < n)
    b2_body_vv_groups(i, stride, step1 != 0, dt, mass, pos, vel, f, label, fixed_group, move_group, mv);
}

// out[k*n + i] = in[i*mn + k]
__global__ void __launch_bounds__(BLK) k_transpose_int(int n, int mn, const int* __restrict__ in, int* out)
{
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < (size_t)n * mn) {
    const int k = (int)(e / n), i = (int)(e - (size_t)k * n);
    out[e] = in[(size_t)i * mn + k];
  }
}

// halo pack: out[d*m + k] = pos[d*stride + idx[k]] + shift[d]  (ghost positions for a neighbour
// domain; the shift carries the periodic image / local-frame offset)
__global__ void __launch_bounds__(BLK) k_halo_pack(
  int m, const int* __restrict__ idx, int stride, const double* __restrict__ pos, double sx,
  double sy, double sz, double* out)
{
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) {
    const int a = idx[k];
    out[k] = pos[a] + sx;
    out[(size_t)m + k] = pos[(size_t)stride + a] + sy;
    out[2 * (size_t)m + k] = pos[2 * (size_t)stride + a] + sz;
  }
}

__global__ void __launch_bounds__(BLK) k_scale(size_t count, double factor, double* v)
{
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count)
    v[i] *= factor;
}

// ---- thermostats: the scale factor is produced ON THE DEVICE from thermo[0], so no half step
// needs a device->host copy (the reference copies T to the host and integrates the chain there,
// ensemble_nhc.cu:173-237) ----------------------------------------------------------------------

// Berendsen: factor = sqrt(1 + coupling*(T0/T - 1)), ensemble_ber.cu:70-86
__global__ void __launch_bounds__(BLK) k_berendsen(
  int n, int stride, double t_target, double coupling, const double* __restrict__ thermo, double* v)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double factor = sqrt(1.0 + coupling * (t_target / thermo[0] - 1.0));
    v[i] *= factor;
    v[(size_t)stride + i] *= factor;
    v[2 * (size_t)stride + i] *= factor;
  }
}

// Nose-Hoover chain (b2_nhc_chain); state = {eta[4], v_eta[4], Q[4], factor}.
__global__ void k_nhc_chain(
  double* state, const double* __restrict__ thermo, double dof, double kT, double dt_half)
{
  if (threadIdx.x != 0 || blockIdx.x != 0)
    return;
  const double ek2 = thermo[0] * dof * 8.617343e-5; // 2 x kinetic energy from the instantaneous T
  state[12] = b2_nhc_chain(state, ek2, dof, kT, dt_half);
}

__global__ void k_bdp_seed(B2BdpState* state, unsigned seed)
{
  if (threadIdx.x == 0 && blockIdx.x == 0)
    b2_mt_seed(*state, seed);
}

// BDP: one thread advances the generator and leaves the factor in the state record
__global__ void k_bdp_factor(
  B2BdpState* state, const double* __restrict__ thermo, int ndeg, double temperature,
  double temperature_coupling)
{
  if (threadIdx.x != 0 || blockIdx.x != 0)
    return;
  state->factor = b2_bdp_factor(*state, thermo[0], ndeg, temperature, temperature_coupling);
}

__global__ void __launch_bounds__(BLK) k_scale_by(
  int n, int stride, const double* __restrict__ factor, double* v)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const double f = factor[0];
    v[i] *= f;
    v[(size_t)stride + i] *= f;
    v[2 * (size_t)stride + i] *= f;
  }
}

// One pass over mass / velocity / potential / 6 virial rows for all 8 outputs (the reference
// launches <<<8,1024>>>, one block per output, each striding over all atoms:
// ensemble.cu:434-633,655), reduced in the fixed order of b2_reduce.cuh: deterministic.
__global__ void __launch_bounds__(THERMO_BLK) k_thermo(
  int n, int stride, int n_temperature, double volume, const double* __restrict__ mass,
  const double* __restrict__ pe, const double* __restrict__ vel, const double* __restrict__ virial,
  double* thermo, double* partial, unsigned int* ticket)
{
  double s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double t[8];
    b2_thermo_terms(i, stride, mass, pe, vel, virial, t);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      s[k] += t[k];
  }
  b2_block_totals<8, THERMO_BLK>(s, partial + blockIdx.x, gridDim.x);
  if (!b2_last_block(ticket))
    return;
  b2_grid_totals<8, THERMO_BLK>(partial, [&](int k, double v) {
    const double K_B = 8.617343e-5; // src/utilities/common.cuh:21
    thermo[k] = k == 0 ? v / (3.0 * n_temperature * K_B) : (k == 1 ? v : v / volume);
  });
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_lj {
  int nt = 0;
  int n = 0;
  double rc = 0.0;
  std::vector<std::string> symbols;
  Neighbor nb;
  DevBuf<float> s6e4, s12e4, rc2;
  DevBuf<double> acc;
  B2LjView view;
};

#define B2_TRY(expr)        \
  do {                      \
    const int rc_ = (expr); \
    if (rc_ != B200MD_OK)   \
      return rc_;           \
  } while (0)

extern "C" {

int b200md_lj_create(const char* path, int num_atoms, b200md_lj** out)
{
  if (!path || !out || num_atoms <= 0) {
    set_error("b200md_lj_create: bad argument");
    return B200MD_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("b200md_lj_create: no CUDA device (libb200md has no CPU fallback)");
    return B200MD_ERR_CUDA;
  }
  LjFile file;
  const std::string err = load_lj(path, file);
  if (!err.empty())
    return load_error(err);
  b200md_lj* p = new (std::nothrow) b200md_lj;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->nt = file.nt;
  p->symbols = file.symbols;
  p->rc = file.rc;
  p->n = num_atoms;
  const size_t N = (size_t)num_atoms;
  int rc = B200MD_OK;
  auto up = [&](DevBuf<float>& d, const std::vector<float>& h) -> int {
    B2_CUDA(d.reserve(h.size()));
    B2_CUDA(cudaMemcpy(d.p, h.data(), sizeof(float) * h.size(), cudaMemcpyHostToDevice));
    return B200MD_OK;
  };
  if ((rc = up(p->s6e4, file.s6e4)) || (rc = up(p->s12e4, file.s12e4)) || (rc = up(p->rc2, file.rc2))) {
    delete p;
    return rc;
  }
  if ((rc = p->nb.init(num_atoms, p->rc, file.mn_skin)) != B200MD_OK) {
    delete p;
    return rc;
  }
  if (p->acc.reserve(13 * N) != cudaSuccess) {
    delete p;
    set_error("out of device memory");
    return B200MD_ERR_CUDA;
  }
  B2LjView& P = p->view;
  P.nt = p->nt;
  P.s6e4 = p->s6e4.p;
  P.s12e4 = p->s12e4.p;
  P.rc2 = p->rc2.p;
  P.n = num_atoms;
  P.atoms = p->nb.atoms.p;
  P.nn_skin = p->nb.nn_skin.p;
  P.nl_skin = p->nb.nl_skin.p;
  P.acc = p->acc.p;
  cudaDeviceSynchronize();
  *out = p;
  return B200MD_OK;
}

void b200md_lj_destroy(b200md_lj* p) { delete p; }
double b200md_lj_rc(const b200md_lj* p) { return p->rc; }
const char* b200md_lj_symbol(const b200md_lj* p, int t)
{
  return (t >= 0 && t < p->nt) ? p->symbols[t].c_str() : "";
}
int b200md_lj_info(const b200md_lj* p, int what)
{
  if (what == 0)
    return p->nt;
  if (what == 6) {
    int bits = 0, rebuilds = 0;
    const_cast<b200md_lj*>(p)->nb.check(0, &bits, &rebuilds);
    return rebuilds;
  }
  return -1;
}

int b200md_lj_compute(
  b200md_lj* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  const B2Box box = make_box(h, pbc);
  B2_TRY(p->nb.update(box, d_type, d_position, n, st));
  p->n = n;
  p->view.n = n;
  k_lj<<<grid_for(n, 128), 128, 0, st>>>(p->view, box);
  B2_LAUNCHED();
  k_unpack_lj<<<grid_for(n, BLK), BLK, 0, st>>>(
    n, p->nb.perm.p, p->acc.p, d_potential, d_force, d_virial);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_lj_invalidate(b200md_lj* p, int n_new, void* stream)
{
  B2_TRY(p->nb.invalidate(n_new, (cudaStream_t)stream));
  p->n = n_new;
  p->view.n = n_new;
  return B200MD_OK;
}

int b200md_lj_check(b200md_lj* p, void* stream)
{
  int bits = 0, rebuilds = 0;
  B2_TRY(p->nb.check((cudaStream_t)stream, &bits, &rebuilds));
  if (bits) {
    set_error("LJ neighbour-list capacity exceeded on the device");
    return B200MD_ERR_OVERFLOW;
  }
  return B200MD_OK;
}

int b200md_apply_pbc_strided(
  int n, int stride, const double h[9], const int pbc[3], double* d_position, void* stream)
{
  const B2Box box = make_box(h, pbc);
  k_apply_pbc<<<grid_for(n, BLK), BLK, 0, (cudaStream_t)stream>>>(
    n, box, d_position, d_position + stride, d_position + 2 * (size_t)stride);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_apply_pbc(int n, const double h[9], const int pbc[3], double* d_position, void* stream)
{
  return b200md_apply_pbc_strided(n, n, h, pbc, d_position, stream);
}

int b200md_zero_properties(
  int n, double* d_potential, double* d_force, double* d_virial, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = (size_t)n;
  k_zero<<<grid_for(N, BLK * 4), BLK, 0, st>>>(N, d_potential);
  B2_LAUNCHED();
  k_zero<<<grid_for(3 * N, BLK * 4), BLK, 0, st>>>(3 * N, d_force);
  B2_LAUNCHED();
  k_zero<<<grid_for(9 * N, BLK * 4), BLK, 0, st>>>(9 * N, d_virial);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_velocity_verlet_strided(
  int is_step1, int n, int stride, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, void* stream)
{
  k_vv<<<grid_for(n, BLK), BLK, 0, (cudaStream_t)stream>>>(
    n, stride, is_step1, time_step, d_mass, d_position, d_velocity, d_force);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_velocity_verlet(
  int is_step1, int n, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, void* stream)
{
  return b200md_velocity_verlet_strided(
    is_step1, n, n, time_step, d_mass, d_position, d_velocity, d_force, stream);
}

int b200md_transpose_int(int n, int mn, const int* d_row_major, int* d_column_major, void* stream)
{
  if (n <= 0 || mn <= 0)
    return B200MD_OK;
  k_transpose_int<<<grid_for((long long)n * mn, BLK), BLK, 0, (cudaStream_t)stream>>>(
    n, mn, d_row_major, d_column_major);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_velocity_verlet_groups(
  int is_step1, int n, int stride, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, const int* d_group_label, int fixed_group,
  int move_group, const double move_velocity[3], void* stream)
{
  if (!d_group_label || (fixed_group < 0 && move_group < 0))
    return b200md_velocity_verlet_strided(
      is_step1, n, stride, time_step, d_mass, d_position, d_velocity, d_force, stream);
  const double z[3] = {0.0, 0.0, 0.0};
  const double* mv = move_velocity ? move_velocity : z;
  k_vv_groups<<<grid_for(n, BLK), BLK, 0, (cudaStream_t)stream>>>(
    n, stride, is_step1, time_step, d_mass, d_position, d_velocity, d_force, d_group_label,
    fixed_group, move_group, mv[0], mv[1], mv[2]);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_halo_pack(
  int m, const int* d_index, int stride, const double* d_position, const double shift[3],
  double* d_out, void* stream)
{
  if (m <= 0)
    return B200MD_OK;
  k_halo_pack<<<grid_for(m, BLK), BLK, 0, (cudaStream_t)stream>>>(
    m, d_index, stride, d_position, shift[0], shift[1], shift[2], d_out);
  B2_LAUNCHED();
  return B200MD_OK;
}

long long b200md_thermo_scratch_bytes(int n)
{
  return (long long)b2_scratch_bytes(8, b2_reduce_blocks(n, THERMO_BLK, THERMO_MAX_BLOCKS));
}

int b200md_find_thermo(
  int n, int n_temperature, double volume, const double* d_mass, const double* d_potential,
  const double* d_velocity, const double* d_virial, double* d_thermo8, void* d_scratch,
  void* stream)
{
  return b200md_find_thermo_strided(
    n, n, n_temperature, volume, d_mass, d_potential, d_velocity, d_virial, d_thermo8, d_scratch,
    stream);
}

int b200md_find_thermo_strided(
  int n, int stride, int n_temperature, double volume, const double* d_mass,
  const double* d_potential, const double* d_velocity, const double* d_virial, double* d_thermo8,
  void* d_scratch, void* stream)
{
  k_thermo<<<b2_reduce_blocks(n, THERMO_BLK, THERMO_MAX_BLOCKS), THERMO_BLK, 0, (cudaStream_t)stream>>>(
    n, stride, n_temperature, volume, d_mass, d_potential, d_velocity, d_virial, d_thermo8,
    b2_scratch_partials(d_scratch), b2_scratch_ticket(d_scratch));
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_berendsen_temperature(
  int n, int stride, double temperature, double temperature_coupling, const double* d_thermo,
  double* d_velocity, void* stream)
{
  // temperature_coupling is tau_T / time_step as in run.in; the kernel uses its inverse
  // (Ensemble_BER::Ensemble_BER, ensemble_ber.cu:26-35)
  if (temperature_coupling <= 0.0) {
    set_error("temperature coupling must be positive");
    return B200MD_ERR_ARG;
  }
  k_berendsen<<<grid_for(n, BLK), BLK, 0, (cudaStream_t)stream>>>(
    n, stride, temperature, 1.0 / temperature_coupling, d_thermo, d_velocity);
  B2_LAUNCHED();
  return B200MD_OK;
}

struct b200md_nhc {
  DevBuf<double> state; // eta[4], v_eta[4], Q[4], factor
  double dof = 0.0, kT = 0.0;
};

int b200md_nhc_create(
  long long n_global, double temperature, double temperature_coupling, double time_step,
  b200md_nhc** out)
{
  // Ensemble_NHC::Ensemble_NHC, ensemble_nhc.cu:31-50
  b200md_nhc* p = new (std::nothrow) b200md_nhc;
  if (!p || p->state.reserve(16) != cudaSuccess) {
    delete p;
    set_error("b200md_nhc_create: allocation failed");
    return B200MD_ERR_CUDA;
  }
  const double kT = 8.617343e-5 * temperature;
  const double tau = time_step * temperature_coupling;
  const double dof = 3.0 * (double)n_global;
  double h[16] = {0, 0, 0, 0, 1.0, -1.0, 1.0, -1.0, 0, 0, 0, 0, 1.0, 0, 0, 0};
  for (int i = 0; i < 4; ++i)
    h[8 + i] = kT * tau * tau;
  h[8] *= dof;
  B2_CUDA(cudaMemcpy(p->state.p, h, sizeof h, cudaMemcpyHostToDevice));
  p->dof = dof;
  p->kT = kT;
  *out = p;
  return B200MD_OK;
}

void b200md_nhc_destroy(b200md_nhc* p) { delete p; }

int b200md_nhc_half_step(
  b200md_nhc* p, int n, int stride, double time_step, const double* d_thermo, double* d_velocity,
  void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  k_nhc_chain<<<1, 32, 0, st>>>(p->state.p, d_thermo, p->dof, p->kT, 0.5 * time_step);
  B2_LAUNCHED();
  // n = 0: a domain block that owns no atoms still advances its copy of the chain
  if (n > 0) {
    k_scale_by<<<grid_for(n, BLK), BLK, 0, st>>>(n, stride, p->state.p + 12, d_velocity);
    B2_LAUNCHED();
  }
  return B200MD_OK;
}

struct b200md_bdp {
  DevBuf<B2BdpState> state;
  int ndeg = 0;
  double temperature = 0.0, coupling = 0.0;
};

int b200md_bdp_create(
  long long n_global, double temperature, double temperature_coupling, unsigned seed,
  b200md_bdp** out)
{
  if (n_global < 1 || 3 * n_global > 2147483647LL || temperature <= 0.0) {
    set_error("b200md_bdp_create: bad atom count or temperature");
    return B200MD_ERR_ARG;
  }
  b200md_bdp* p = new (std::nothrow) b200md_bdp;
  if (!p || p->state.reserve(1) != cudaSuccess) {
    delete p;
    set_error("b200md_bdp_create: allocation failed");
    return B200MD_ERR_CUDA;
  }
  k_bdp_seed<<<1, 32>>>(p->state.p, seed);
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    delete p;
    set_error(cudaGetErrorString(e));
    return B200MD_ERR_CUDA;
  }
  p->ndeg = (int)(3 * n_global);
  p->temperature = temperature;
  p->coupling = temperature_coupling;
  *out = p;
  return B200MD_OK;
}

void b200md_bdp_destroy(b200md_bdp* p) { delete p; }

int b200md_bdp_step(
  b200md_bdp* p, int n, int stride, const double* d_thermo, double* d_velocity, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  k_bdp_factor<<<1, 32, 0, st>>>(p->state.p, d_thermo, p->ndeg, p->temperature, p->coupling);
  B2_LAUNCHED();
  const double* factor = reinterpret_cast<const double*>(
    reinterpret_cast<const char*>(p->state.p) + offsetof(B2BdpState, factor));
  // n = 0: a domain block that owns no atoms still draws its copy of the random numbers
  if (n > 0) {
    k_scale_by<<<grid_for(n, BLK), BLK, 0, st>>>(n, stride, factor, d_velocity);
    B2_LAUNCHED();
  }
  return B200MD_OK;
}

int b200md_scale_velocity(int n, double factor, double* d_velocity, void* stream)
{
  const size_t count = 3 * (size_t)n;
  k_scale<<<grid_for(count, BLK), BLK, 0, (cudaStream_t)stream>>>(count, factor, d_velocity);
  B2_LAUNCHED();
  return B200MD_OK;
}

} // extern "C"

// b2_measure.cu -- heat-current autocorrelation (Green-Kubo) on top of the per-atom virial the force
// kernels produce: the consumer SURVEY.md 8f ranks fourth.
//
//   b200md_hac_create / _sample / _finish  <- HAC::preprocess / process / postprocess,
//       src/measure/hac.cu:32-280 (gpu_sum_heat :50-78, gpu_find_hac :111-170, find_rtc :173-181)
//
// sample(): every sample_interval steps the per-atom heat current (compute_heat.cu:32-90, our
// b200md_compute_heat) is summed into heat_all[nd + Nd*k], k = jx_in jx_out jy_in jy_out jz.
// finish(): hac[nc + Nc*k] = < J_k(0) (J_k(t) + J_partner(t)) > for the in/out pairs, < Jz(0) Jz(t) >
// for z (hac.cu:132-142), averaged over the Nd - nc available origins, and the running thermal
// conductivity by the trapezoidal rule with factor dt/2 / (k_B T^2 V) * KAPPA_UNIT_CONVERSION.
// The reductions are one block per component with a fixed summation order (deterministic).
//
// HNEMD (Fan et al., PRB 99, 064308 (2019)) and the spectral heat current:
//   b200md_hnemd_drive            <- gpu_add_driving_force + gpu_sum_force + gpu_correct_force,
//                                    src/force/force.cu:228-312, 857-897
//   b200md_hnemd_create/_sample/_take <- HNEMD::preprocess / process, src/measure/hnemd_kappa.cu:37-132
// The spectral heat current (b200md_shc_*) runs on the correlation engine of b2_correlate.cu.
// Every reduction has a fixed order: the results do not depend on scheduling.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_reduce.cuh"
#include "b2_tersoff.cuh" // b2_heat5
#include <cmath>
#include <new>
#include <vector>

namespace b2 {
namespace {

constexpr int RED_BLK = 256;        // atoms-per-block of the ticketed reductions
constexpr int RED_MAX_BLOCKS = 264; // two per SM of an H100 SXM
constexpr int FTOT_SLOT = 8;        // doubles of the drive's scratch between the ticket and the partials

// f_i += W_i^T fe, with the virial index map xx xy xz / yx yy yz / zx zy zz = 0 3 4 / 6 1 5 / 7 8 2
// (force.cu:857-878), and the total of the new forces.  nvcc -O3 compiles force.cu:248-250 to
//   t = fe_y * W_y.;  t = fma(fe_x, W_x., t);  t = fma(fe_z, W_z., t);  f = f + t
// (mul.f64, fma.rn.f64, fma.rn.f64, add.f64 in its PTX); spelt out here so that the per-atom force
// is the reference's bit for bit.  Only the order of the total-force sum differs.
__global__ void __launch_bounds__(RED_BLK) k_hnemd_drive(
  int n, int stride, double fe_x, double fe_y, double fe_z, const double* __restrict__ w, double* f,
  double* partial, unsigned int* ticket, double* ftot)
{
  const size_t s = (size_t)stride;
  double t[3] = {0.0, 0.0, 0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double gx = __fma_rn(fe_z, w[7 * s + i], __fma_rn(fe_x, w[i], __dmul_rn(fe_y, w[6 * s + i])));
    const double gy = __fma_rn(fe_z, w[8 * s + i], __fma_rn(fe_x, w[3 * s + i], __dmul_rn(fe_y, w[s + i])));
    const double gz = __fma_rn(fe_z, w[2 * s + i], __fma_rn(fe_x, w[4 * s + i], __dmul_rn(fe_y, w[5 * s + i])));
    const double fx = __dadd_rn(f[i], gx), fy = __dadd_rn(f[s + i], gy), fz = __dadd_rn(f[2 * s + i], gz);
    f[i] = fx;
    f[s + i] = fy;
    f[2 * s + i] = fz;
    t[0] += fx;
    t[1] += fy;
    t[2] += fz;
  }
  b2_block_totals<3, RED_BLK>(t, partial + blockIdx.x, gridDim.x);
  if (b2_last_block(ticket))
    b2_grid_totals<3, RED_BLK>(partial, [&](int k, double v) { ftot[k] = v; });
}

// f_i -= ftot / N as gpu_correct_force (force.cu:303-312): a product with the host's 1.0 / N, then
// a subtraction (not contracted into an fma by nvcc there, nor here)
__global__ void __launch_bounds__(256) k_hnemd_correct(
  int n, int stride, double one_over_n, const double* __restrict__ ftot, double* f)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const size_t s = (size_t)stride;
    f[i] = __dsub_rn(f[i], __dmul_rn(ftot[0], one_over_n));
    f[s + i] = __dsub_rn(f[s + i], __dmul_rn(ftot[1], one_over_n));
    f[2 * s + i] = __dsub_rn(f[2 * s + i], __dmul_rn(ftot[2], one_over_n));
  }
}

// compute_heat + gpu_sum_heat of hnemd_kappa.cu:52-106 in one pass: the per-atom heat current is
// summed straight into a row of five; the 5N per-atom array is never written.  row_at == nullptr: the
// row is rows[0..4]; otherwise it is row *row_at of rows[n_rows][5], and the last block advances
// *row_at (mod n_rows), so that one captured launch serves every step
__global__ void __launch_bounds__(RED_BLK) k_hnemd_heat(
  int n, int stride, const double* __restrict__ w, const double* __restrict__ v, double* rows,
  unsigned int* row_at, unsigned int n_rows, double* partial, unsigned int* ticket)
{
  double t[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double h[5];
    b2_heat5(i, stride, w, v, h);
#pragma unroll
    for (int k = 0; k < 5; ++k)
      t[k] += h[k];
  }
  b2_block_totals<5, RED_BLK>(t, partial + blockIdx.x, gridDim.x);
  if (b2_last_block(ticket)) {
    double* row5 = row_at ? rows + (size_t)5 * *row_at : rows;
    b2_grid_totals<5, RED_BLK>(partial, [&](int k, double v) { row5[k] = v; });
    if (row_at && threadIdx.x == 0) // after the barrier that ends b2_grid_totals: every put has read it
      *row_at = (*row_at + 1u) % n_rows;
  }
}

// one block per heat component: strided partial sums, then a tree -- the order of hac.cu:50-78
__global__ void __launch_bounds__(1024) k_sum_heat(int n, int heat_stride, int Nd, int nd, const double* g_heat, double* g_heat_all)
{
  __shared__ double s[1024];
  const int tid = threadIdx.x;
  double v = 0.0;
  for (int i = tid; i < n; i += 1024)
    v += g_heat[i + (size_t)heat_stride * blockIdx.x];
  s[tid] = v;
  __syncthreads();
  for (int o = 512; o > 0; o >>= 1) {
    if (tid < o)
      s[tid] += s[tid + o];
    __syncthreads();
  }
  if (tid == 0)
    g_heat_all[nd + (size_t)Nd * blockIdx.x] = s[0];
}

// block = correlation time nc; hac.cu:111-170
__global__ void __launch_bounds__(128) k_find_hac(int Nc, int Nd, const double* __restrict__ h, double* g_hac)
{
  __shared__ double s[5][128];
  const int tid = threadIdx.x, bid = blockIdx.x;
  double a[5] = {0, 0, 0, 0, 0};
  for (int i = tid; i + bid < Nd; i += 128) {
    const int j = i + bid;
    a[0] += h[i] * h[j] + h[i] * h[j + Nd];
    a[1] += h[i + Nd] * h[j + Nd] + h[i + Nd] * h[j];
    a[2] += h[i + 2 * Nd] * h[j + 2 * Nd] + h[i + 2 * Nd] * h[j + 3 * Nd];
    a[3] += h[i + 3 * Nd] * h[j + 3 * Nd] + h[i + 3 * Nd] * h[j + 2 * Nd];
    a[4] += h[i + 4 * Nd] * h[j + 4 * Nd];
  }
  for (int k = 0; k < 5; ++k)
    s[k][tid] = a[k];
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) {
    if (tid < o)
      for (int k = 0; k < 5; ++k)
        s[k][tid] += s[k][tid + o];
    __syncthreads();
  }
  if (tid == 0)
    for (int k = 0; k < 5; ++k)
      g_hac[bid + (size_t)Nc * k] = s[k][0] / (Nd - bid);
}

// |fe| as HNEMD::parse forms it, hnemd_kappa.cu:180-183
double fe_norm(const double fe[3])
{
  double norm = 0.0;
  for (int d = 0; d < 3; ++d)
    norm += fe[d] * fe[d];
  return std::sqrt(norm);
}

// the output branch of HNEMD::process, hnemd_kappa.cu:108-122: rows[m * 5 + k], m < oi, summed in
// order and scaled to W/mK
void hnemd_kappa(int oi, double volume, double temperature, double fe_norm, const double* rows, double* kappa5)
{
  const double KAPPA_UNIT_CONVERSION = 1.573769e+5; // common.cuh:27
  double factor = KAPPA_UNIT_CONVERSION / oi;
  factor /= (volume * temperature * fe_norm);
  for (int k = 0; k < 5; ++k) {
    double s = 0.0;
    for (int m = 0; m < oi; ++m)
      s += rows[(size_t)m * 5 + k];
    kappa5[k] = s * factor;
  }
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_hac {
  int number_of_steps = 0, sample_interval = 1, Nc = 0, Nd = 0;
  DevBuf<double> heat_all, heat, hac;
};

struct b200md_hnemd {
  int output_interval = 1;
  double fe[3] = {0, 0, 0}, fe_norm = 0.0;
  DevBuf<double> heat_all; // [output_interval][5], row = step % output_interval
  DevBuf<char> scratch;    // b2_scratch_bytes(5, blocks of k_hnemd_heat)
};

extern "C" {

int b200md_hac_create(int number_of_steps, int sample_interval, int Nc, b200md_hac** out)
{
  if (!out || number_of_steps <= 0 || sample_interval <= 0 || Nc <= 0 ||
      Nc > number_of_steps / sample_interval) {
    set_error("b200md_hac_create: need number_of_steps / sample_interval >= Nc > 0");
    return B200MD_ERR_ARG;
  }
  b200md_hac* p = new (std::nothrow) b200md_hac;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->number_of_steps = number_of_steps;
  p->sample_interval = sample_interval;
  p->Nc = Nc;
  p->Nd = number_of_steps / sample_interval;
  if (p->heat_all.reserve((size_t)5 * p->Nd) != cudaSuccess || p->hac.reserve((size_t)5 * Nc) != cudaSuccess) {
    delete p;
    set_error("out of device memory (HAC)");
    return B200MD_ERR_CUDA;
  }
  cudaMemset(p->heat_all.p, 0, sizeof(double) * 5 * p->Nd);
  *out = p;
  return B200MD_OK;
}

void b200md_hac_destroy(b200md_hac* p) { delete p; }

int b200md_hac_sample(
  b200md_hac* p, int step, int n, int stride, const double* d_virial, const double* d_velocity,
  void* stream)
{
  if ((step + 1) % p->sample_interval != 0)
    return B200MD_OK;
  const int nd = (step + 1) / p->sample_interval - 1;
  if (nd < 0 || nd >= p->Nd)
    return B200MD_OK; // beyond the run length given at creation
  B2_CUDA(p->heat.reserve((size_t)5 * n));
  const int rc = b200md_compute_heat(n, stride, d_virial, d_velocity, p->heat.p, n, stream);
  if (rc != B200MD_OK)
    return rc;
  k_sum_heat<<<5, 1024, 0, (cudaStream_t)stream>>>(n, n, p->Nd, nd, p->heat.p, p->heat_all.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_hac_finish(
  b200md_hac* p, double time_step, double temperature, double volume, double* hac_out,
  double* rtc_out, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  const int Nc = p->Nc;
  k_find_hac<<<Nc, 128, 0, st>>>(Nc, p->Nd, p->heat_all.p, p->hac.p);
  B2_LAUNCHED();
  std::vector<double> hac((size_t)5 * Nc);
  B2_CUDA(cudaMemcpyAsync(hac.data(), p->hac.p, sizeof(double) * 5 * Nc, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  const double K_B = 8.617343e-5, KAPPA_UNIT_CONVERSION = 1.573769e+5; // common.cuh:21,27
  const double dt = time_step * p->sample_interval;
  const double factor = dt * 0.5 / (K_B * temperature * temperature * volume) * KAPPA_UNIT_CONVERSION;
  for (int k = 0; k < 5; ++k) {
    double run = 0.0;
    for (int nc = 0; nc < Nc; ++nc) {
      const size_t idx = (size_t)Nc * k + nc;
      if (nc > 0)
        run += (hac[idx - 1] + hac[idx]) * factor; // find_rtc, hac.cu:173-181
      if (rtc_out)
        rtc_out[idx] = run;
      if (hac_out)
        hac_out[idx] = hac[idx];
    }
  }
  return B200MD_OK;
}

/* the recorded heat-current series heat_all[nd + Nd*k] (host copy; parity hook) */
int b200md_hac_series(b200md_hac* p, double* out, void* stream)
{
  B2_CUDA(cudaMemcpyAsync(out, p->heat_all.p, sizeof(double) * 5 * p->Nd, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  B2_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return B200MD_OK;
}

long long b200md_hnemd_drive_scratch_bytes(int n)
{
  return (long long)(b2_scratch_bytes(3, b2_reduce_blocks(n, RED_BLK, RED_MAX_BLOCKS)) + sizeof(double) * FTOT_SLOT);
}

int b200md_hnemd_drive_add(
  int n, int stride, const double fe[3], const double* d_virial, double* d_force, void* d_scratch,
  double* d_ftot, void* stream)
{
  if (n < 0 || stride < n || !fe || (n > 0 && (!d_virial || !d_force)) || !d_scratch || !d_ftot) {
    set_error("b200md_hnemd_drive_add: bad argument");
    return B200MD_ERR_ARG;
  }
  // the partials sit behind the FTOT_SLOT of b200md_hnemd_drive's layout; n = 0 is one block that
  // writes a zero total
  k_hnemd_drive<<<b2_reduce_blocks(n, RED_BLK, RED_MAX_BLOCKS), RED_BLK, 0, (cudaStream_t)stream>>>(
    n, stride, fe[0], fe[1], fe[2], d_virial, d_force, b2_scratch_partials(d_scratch) + FTOT_SLOT,
    b2_scratch_ticket(d_scratch), d_ftot);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_hnemd_drive_correct(
  int n, int stride, double one_over_n, const double* d_ftot, double* d_force, void* stream)
{
  if (n < 0 || stride < n || !d_ftot || (n > 0 && !d_force)) {
    set_error("b200md_hnemd_drive_correct: bad argument");
    return B200MD_ERR_ARG;
  }
  if (n == 0) // a zero-block grid is a launch error
    return B200MD_OK;
  k_hnemd_correct<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(n, stride, one_over_n, d_ftot, d_force);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_hnemd_drive(
  int n, int stride, const double fe[3], const double* d_virial, double* d_force, void* d_scratch,
  void* stream)
{
  if (n <= 0 || stride < n || !fe || !d_virial || !d_force || !d_scratch) {
    set_error("b200md_hnemd_drive: bad argument");
    return B200MD_ERR_ARG;
  }
  // the b2_scratch_* layout with ftot[3] in front of the partials
  double* ftot = b2_scratch_partials(d_scratch);
  const int rc = b200md_hnemd_drive_add(n, stride, fe, d_virial, d_force, d_scratch, ftot, stream);
  if (rc != B200MD_OK)
    return rc;
  return b200md_hnemd_drive_correct(n, stride, 1.0 / n, ftot, d_force, stream);
}

long long b200md_hnemd_heat_row_scratch_bytes(int n)
{
  return (long long)b2_scratch_bytes(5, b2_reduce_blocks(n, RED_BLK, RED_MAX_BLOCKS));
}

int b200md_hnemd_heat_row(
  int n, int stride, const double* d_virial, const double* d_velocity, double* d_rows, int n_rows,
  unsigned int* d_row, void* d_scratch, void* stream)
{
  if (n < 0 || stride < n || n_rows < 1 || (n > 0 && (!d_virial || !d_velocity)) || !d_rows || !d_row ||
      !d_scratch) {
    set_error("b200md_hnemd_heat_row: bad argument");
    return B200MD_ERR_ARG;
  }
  k_hnemd_heat<<<b2_reduce_blocks(n, RED_BLK, RED_MAX_BLOCKS), RED_BLK, 0, (cudaStream_t)stream>>>(
    n, stride, d_virial, d_velocity, d_rows, d_row, (unsigned int)n_rows, b2_scratch_partials(d_scratch),
    b2_scratch_ticket(d_scratch));
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_hnemd_create(int output_interval, const double fe[3], b200md_hnemd** out)
{
  if (!out || !fe || output_interval < 1) {
    set_error("b200md_hnemd_create: need output_interval >= 1 and fe[3]");
    return B200MD_ERR_ARG;
  }
  b200md_hnemd* p = new (std::nothrow) b200md_hnemd;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->output_interval = output_interval;
  for (int d = 0; d < 3; ++d)
    p->fe[d] = fe[d];
  p->fe_norm = fe_norm(fe);
  if (p->heat_all.reserve((size_t)5 * output_interval) != cudaSuccess) {
    delete p;
    set_error("out of device memory (HNEMD)");
    return B200MD_ERR_CUDA;
  }
  cudaMemset(p->heat_all.p, 0, sizeof(double) * 5 * output_interval);
  *out = p;
  return B200MD_OK;
}

void b200md_hnemd_destroy(b200md_hnemd* p) { delete p; }

int b200md_hnemd_sample(
  b200md_hnemd* p, int step, int n, int stride, const double* d_virial, const double* d_velocity,
  void* stream)
{
  if (!p || step < 0 || n <= 0 || stride < n) {
    set_error("b200md_hnemd_sample: bad argument");
    return B200MD_ERR_ARG;
  }
  const int g = b2_reduce_blocks(n, RED_BLK, RED_MAX_BLOCKS);
  const size_t need = b2_scratch_bytes(5, g);
  if (p->scratch.n < need) { // first call, or more atoms than before: the ticket starts at zero
    B2_CUDA(p->scratch.reserve(need));
    B2_CUDA(cudaMemsetAsync(p->scratch.p, 0, B2_TICKET_BYTES, (cudaStream_t)stream));
  }
  const int row = step % p->output_interval;
  k_hnemd_heat<<<g, RED_BLK, 0, (cudaStream_t)stream>>>(
    n, stride, d_virial, d_velocity, p->heat_all.p + (size_t)5 * row, nullptr, 0u,
    b2_scratch_partials(p->scratch.p), b2_scratch_ticket(p->scratch.p));
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_hnemd_take(
  b200md_hnemd* p, double volume, double temperature, double* kappa5, double* rows, void* stream)
{
  if (!p || !kappa5 || !(volume > 0.0) || !(temperature > 0.0) || !(p->fe_norm > 0.0)) {
    set_error("b200md_hnemd_take: need volume > 0, temperature > 0 and |fe| > 0");
    return B200MD_ERR_ARG;
  }
  const int oi = p->output_interval;
  std::vector<double> h((size_t)5 * oi);
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(cudaMemcpyAsync(h.data(), p->heat_all.p, sizeof(double) * 5 * oi, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  hnemd_kappa(oi, volume, temperature, p->fe_norm, h.data(), kappa5);
  if (rows)
    for (size_t k = 0; k < h.size(); ++k)
      rows[k] = h[k];
  return B200MD_OK;
}

int b200md_hnemd_kappa(
  int output_interval, double volume, double temperature, const double fe[3], const double* rows,
  double* kappa5)
{
  if (output_interval < 1 || !fe || !rows || !kappa5 || !(volume > 0.0) || !(temperature > 0.0) ||
      !(fe_norm(fe) > 0.0)) {
    set_error("b200md_hnemd_kappa: need output_interval >= 1, volume > 0, temperature > 0 and |fe| > 0");
    return B200MD_ERR_ARG;
  }
  hnemd_kappa(output_interval, volume, temperature, fe_norm(fe), rows, kappa5);
  return B200MD_OK;
}

} // extern "C"

// b2_minimize.cu -- energy minimization: steepest descent and FIRE with a fixed or a relaxing box.
//
//   b200md_minimizer_sd_*     <- Minimizer_SD::compute (src/minimize/minimizer_sd.cu:70-169)
//   b200md_minimizer_fire_step <- one iteration of Minimizer_FIRE::compute (minimizer_fire.cu:108-180) or of
//                                Minimizer_FIRE_Box_Change::compute (minimizer_fire_box_change.cu:239-406)
//
// The reference runs about ten streaming kernels and five single-block reductions per FIRE iteration, each
// reduction followed by a blocking copy, and allocates device vectors inside the loop.  Here one FIRE
// iteration is two kernels: a grid-stride reduction of max F^2, sum U, v.F, |F|^2, |v|^2 (and the nine
// summed virial components for box change) whose last block sums the per-block partials in block order and
// runs the FIRE control step on the device, and one update pass that applies move-back, kick, mixing and
// the position (and strain) update per atom.  SD is three kernels per iteration (trial energy + decision,
// accept + next f_max, trial positions).  The host reads one small record per iteration; nothing is
// allocated after creation.  The grid of every reduction is a function of n only, so the sums are
// run-to-run identical on any device.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_reduce.cuh"
#include <cmath>
#include <new>

namespace b2 {
namespace {

constexpr int BLK = 256;
constexpr int RED_GRID = 1024; // most blocks of a reduction (fixed: the block order of the sums)
constexpr int RED_K = 14;      // partials per block: max F^2, U, v.F, F^2, v^2, 9 virial sums

// FIRE constants, minimizer_fire.cuh:24-36 (dt in natural units: 1 fs / TIME_UNIT_CONVERSION)
constexpr double F_INC = 1.1, F_DEC = 0.5, ALPHA_START = 0.25, F_ALPHA = 0.99, MASS = 5.0;
constexpr double DT_0 = 1.0 / 1.018051e+1;
constexpr double DT_MAX = 10.0 * DT_0, DT_MIN = 0.02 * DT_0;
constexpr int N_MIN = 20;
constexpr double STRESS_TOLERANCE_GPA = 1e-4;    // minimizer_fire_box_change.cu:254
constexpr double SD_DECREASE = 0.2, SD_INCREASE = 1.2; // minimizer_sd.cu:27-28

struct FireParams {
  double tol, volume, L;
  int box_change, hydrostatic;
};

// The FIRE control step of one iteration on the sums s[] (minimizer_fire.cu:119-167 and
// minimizer_fire_box_change.cu:280-383), written to the record.  Serial, thread 0 of the last block; kept
// out of line so that it does not set the register allocation of the reduction.
__device__ __noinline__ void fire_control(const double* s, double* r, const FireParams prm)
{
  const double f_max = sqrt(s[0]);
  double P = s[2], F2 = s[3], v2 = s[4];
  bool converged = f_max < prm.tol;
  r[B200MD_MIN_FMAX] = f_max;
  r[B200MD_MIN_U] = s[1];
  if (prm.box_change) {
    // virial sums in the order xx xy xz yx yy yz zx zy zz (minimizer_fire_box_change.cu:262-274)
    double vir[9], stress_max = 0.0;
    for (int i = 0; i < 9; ++i)
      vir[i] = s[5 + i];
    double st[9];
    for (int i = 0; i < 9; ++i)
      st[i] = vir[i] / prm.volume * 160.2176621;
    const double pressure = (st[0] + st[4] + st[8]) / 3.0;
    if (prm.hydrostatic) {
      stress_max = fabs(pressure);
      const double tr = vir[0] + vir[4] + vir[8];
      for (int i = 0; i < 9; ++i)
        vir[i] = 0.0;
      vir[0] = vir[4] = vir[8] = tr / 3.0;
    } else {
      for (int i = 0; i < 9; ++i)
        stress_max = fmax(stress_max, fabs(st[i]));
    }
    for (int i = 0; i < 9; ++i) {
      const double fb = vir[i] / prm.L, vb = r[B200MD_MIN_VBOX + i];
      r[B200MD_MIN_FBOX + i] = fb;
      P += vb * fb;
      F2 += fb * fb;
      v2 += vb * vb;
    }
    r[B200MD_MIN_PRESSURE] = pressure;
    r[B200MD_MIN_STRESS] = stress_max;
    converged = converged && stress_max < STRESS_TOLERANCE_GPA;
  }
  r[B200MD_MIN_CONVERGED] = converged ? 1.0 : 0.0;
  r[B200MD_MIN_P] = P;
  if (converged)
    return;
  double dt = r[B200MD_MIN_DT], alpha = r[B200MD_MIN_ALPHA], n_neg = r[B200MD_MIN_NNEG];
  const bool uphill = !(P > 0);
  if (!uphill) {
    if (n_neg > N_MIN) {
      const double next_dt = dt * F_INC;
      if (prm.box_change)
        dt = next_dt > DT_MAX ? DT_MAX : next_dt; // clamped
      else if (next_dt < DT_MAX)
        dt = next_dt; // left unchanged otherwise
      alpha *= F_ALPHA;
    }
    n_neg += 1.0;
  } else {
    const double next_dt = dt * F_DEC;
    if (prm.box_change)
      dt = next_dt < DT_MIN ? DT_MIN : next_dt;
    else if (next_dt > DT_MIN)
      dt = next_dt;
    alpha = ALPHA_START;
    n_neg = 0.0;
    v2 = 0.0; // |v| after the zeroing
  }
  const double F_mod = sqrt(F2), v_mod = sqrt(v2);
  // box change: no mixing when |F| <= 1e-12 (minimizer_fire_box_change.cu:362-366)
  const double scale = (prm.box_change && !(F_mod > 1e-12)) ? 0.0 : alpha * v_mod / F_mod;
  r[B200MD_MIN_DT] = dt;
  r[B200MD_MIN_ALPHA] = alpha;
  r[B200MD_MIN_NNEG] = n_neg;
  r[B200MD_MIN_UPHILL] = uphill ? 1.0 : 0.0;
  r[B200MD_MIN_FMOD] = F_mod;
  r[B200MD_MIN_VMOD] = v_mod;
  r[B200MD_MIN_SCALE] = scale;
  if (prm.box_change) {
    const double dtm = dt / MASS, oma = 1 - alpha;
    for (int i = 0; i < 9; ++i) {
      const double fb = r[B200MD_MIN_FBOX + i];
      double vb = uphill ? 0.0 : r[B200MD_MIN_VBOX + i];
      vb = __dadd_rn(vb, __dmul_rn(fb, dtm));
      vb = __dadd_rn(__dmul_rn(vb, oma), __dmul_rn(fb, scale));
      r[B200MD_MIN_VBOX + i] = vb;
      r[B200MD_MIN_DEPS + i] = vb * dt / prm.L;
    }
  }
}

// FIRE reduction + control.  GPUMD's virial blocks are xx yy zz xy xz yz yx zx zy; vmap gathers them in
// the row-major order xx xy xz yx yy yz zx zy zz.
template <bool BOX>
__global__ void __launch_bounds__(BLK) k_fire_reduce(
  int n, const double* __restrict__ f, const double* __restrict__ v, const double* __restrict__ u,
  const double* __restrict__ w, double* partial, unsigned int* ticket, double* rec, FireParams prm)
{
  constexpr int K = BOX ? RED_K : 5;
  const size_t N = (size_t)n;
  double t[K];
#pragma unroll
  for (int k = 0; k < K; ++k)
    t[k] = 0.0;
  for (int i = blockIdx.x * BLK + threadIdx.x; i < n; i += gridDim.x * BLK) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const double fd = f[d * N + i], vd = v[d * N + i];
      t[0] = fmax(t[0], fd * fd);
      t[2] += vd * fd;
      t[3] += fd * fd;
      t[4] += vd * vd;
    }
    t[1] += u[i];
    if constexpr (BOX) {
      constexpr int vmap[9] = {0, 3, 4, 6, 1, 5, 7, 8, 2};
#pragma unroll
      for (int k = 0; k < 9; ++k)
        t[5 + k] += w[vmap[k] * N + i];
    }
  }
  b2_block_totals<K, BLK, 1u>(t, partial + blockIdx.x, gridDim.x); // row 0: max F^2
  if (!b2_last_block(ticket))
    return;
  __shared__ double s[RED_K];
  b2_grid_totals<K, BLK, 1u>(partial, [&](int k, double v) { s[k] = v; });
  if (threadIdx.x == 0)
    fire_control(s, rec, prm);
}

// FIRE update per atom (minimizer_fire.cu:148-176, minimizer_fire_box_change.cu:339-403) in the reference's
// order of operations, without contraction: move back by -0.5 dt v with the new dt and zero v (uphill,
// fixed box), v += dt/m F, v = (1 - alpha) v + alpha |v|/|F| F, x += dt v (+ dEps x_old for box change).
// The reference contracts its strain update (x + v dt + dEps x) into FMAs; here each step is rounded.
template <bool BOX>
__global__ void __launch_bounds__(BLK) k_fire_update(
  int n, double* __restrict__ x, double* __restrict__ v, const double* __restrict__ f,
  const double* __restrict__ rec)
{
  const int i = blockIdx.x * BLK + threadIdx.x;
  if (i >= n || rec[B200MD_MIN_CONVERGED] != 0.0)
    return;
  const size_t N = (size_t)n;
  const double dt = rec[B200MD_MIN_DT], alpha = rec[B200MD_MIN_ALPHA], scale = rec[B200MD_MIN_SCALE];
  const bool uphill = rec[B200MD_MIN_UPHILL] != 0.0;
  const double back = -0.5 * dt, dtm = dt / MASS, oma = 1 - alpha;
  double r[3], vn[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    double xd = x[d * N + i], vd = v[d * N + i];
    const double fd = f[d * N + i];
    if (uphill) {
      if (!BOX)
        xd = __dadd_rn(xd, __dmul_rn(vd, back));
      vd = 0.0;
    }
    vd = __dadd_rn(vd, __dmul_rn(fd, dtm));
    vd = __dadd_rn(__dmul_rn(vd, oma), __dmul_rn(fd, scale));
    r[d] = xd;
    vn[d] = vd;
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    double xd = __dadd_rn(r[d], __dmul_rn(vn[d], dt));
    if (BOX) {
      const double* e = rec + B200MD_MIN_DEPS + 3 * d;
      xd = __dadd_rn(xd, __dadd_rn(__dadd_rn(__dmul_rn(e[0], r[0]), __dmul_rn(e[1], r[1])), __dmul_rn(e[2], r[2])));
    }
    x[d * N + i] = xd;
    v[d * N + i] = vn[d];
  }
}

// SD: sum U_trial and decide (minimizer_sd.cu:126-137): uphill -> step *= 0.2, else accept and step *= 1.2
__global__ void __launch_bounds__(BLK) k_sd_energy(
  int n, const double* __restrict__ u_trial, double* partial, unsigned int* ticket, double* rec)
{
  double t[1] = {0.0};
  for (int i = blockIdx.x * BLK + threadIdx.x; i < n; i += gridDim.x * BLK)
    t[0] += u_trial[i];
  b2_block_totals<1, BLK>(t, partial + blockIdx.x, gridDim.x);
  if (!b2_last_block(ticket))
    return;
  __shared__ double Ut;
  b2_grid_totals<1, BLK>(partial, [&](int, double v) { Ut = v; });
  if (threadIdx.x == 0) {
    const double U = rec[B200MD_MIN_U];
    const bool uphill = Ut > U;
    rec[B200MD_MIN_UTRIAL] = Ut;
    rec[B200MD_MIN_USMALLER] = uphill ? U : Ut;
    rec[B200MD_MIN_UPHILL] = uphill ? 1.0 : 0.0;
    rec[B200MD_MIN_STEP] *= uphill ? SD_DECREASE : SD_INCREASE;
  }
}

// SD: copy the trial x, F, U over the current ones when the last decision accepted them, and reduce max F^2
// and sum U of the resulting state; the last block derives f_max, convergence and step / f_max
__global__ void __launch_bounds__(BLK) k_sd_accept(
  int n, int begin, double* __restrict__ x, double* __restrict__ f, double* __restrict__ u,
  const double* __restrict__ xt, const double* __restrict__ ft, const double* __restrict__ ut,
  double* partial, unsigned int* ticket, double* rec, double tol)
{
  const bool accept = !begin && rec[B200MD_MIN_UPHILL] == 0.0;
  const size_t N = (size_t)n;
  double t[2] = {0.0, 0.0};
  for (int i = blockIdx.x * BLK + threadIdx.x; i < n; i += gridDim.x * BLK) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      double fd;
      if (accept) {
        fd = ft[d * N + i];
        f[d * N + i] = fd;
        x[d * N + i] = xt[d * N + i];
      } else {
        fd = f[d * N + i];
      }
      t[0] = fmax(t[0], fd * fd);
    }
    double ui;
    if (accept) {
      ui = ut[i];
      u[i] = ui;
    } else {
      ui = u[i];
    }
    t[1] += ui;
  }
  b2_block_totals<2, BLK, 1u>(t, partial + blockIdx.x, gridDim.x); // row 0: max F^2
  if (!b2_last_block(ticket))
    return;
  __shared__ double s[2];
  b2_grid_totals<2, BLK, 1u>(partial, [&](int k, double v) { s[k] = v; });
  if (threadIdx.x == 0) {
    const double f_max = sqrt(s[0]);
    rec[B200MD_MIN_FMAX] = f_max;
    rec[B200MD_MIN_U] = s[1];
    rec[B200MD_MIN_CONVERGED] = f_max < tol ? 1.0 : 0.0;
    rec[B200MD_MIN_SCALE] = rec[B200MD_MIN_STEP] / f_max;
  }
}

// SD trial positions x + F step / f_max; atoms of the fixed group stay put (minimizer_sd.cu:32-66)
__global__ void __launch_bounds__(BLK) k_sd_trial(
  int n3, int n, const double* __restrict__ x, const double* __restrict__ f, const int* __restrict__ label,
  int fixed_group, double* __restrict__ xt, const double* __restrict__ rec)
{
  const int k = blockIdx.x * BLK + threadIdx.x;
  if (k >= n3 || rec[B200MD_MIN_CONVERGED] != 0.0)
    return;
  double change = 0.0;
  if (fixed_group < 0 || label[k % n] != fixed_group)
    change = __dmul_rn(f[k], rec[B200MD_MIN_SCALE]);
  xt[k] = __dadd_rn(x[k], change);
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_minimizer {
  int method = 0, n = 0, steps = 0, box_change = 0, hydrostatic = 0;
  double tol = 0.0, L = 0.0;
  DevBuf<double> v, partial, rec;
  DevBuf<unsigned int> ticket;
};

namespace {

int fetch(b200md_minimizer* p, double* record, cudaStream_t st)
{
  if (record) {
    B2_CUDA(cudaMemcpyAsync(record, p->rec.p, B200MD_MIN_RECORD * sizeof(double), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
  }
  return B200MD_OK;
}

bool bad_call(b200md_minimizer* p, int method, int n, const char* what)
{
  if (!p || p->method != method || n != p->n) {
    set_error(std::string(what) + ": null handle, other method, or atom count differs from the one given at "
                                  "creation");
    return true;
  }
  return false;
}

} // namespace

extern "C" {

int b200md_minimizer_create(
  int method, int n, double force_tolerance, int number_of_steps, int box_change, int hydrostatic,
  b200md_minimizer** out)
{
  if (!out || (method != 0 && method != 1) || n <= 0 || 3LL * n > 2147483647LL || number_of_steps <= 0 ||
      (box_change != 0 && box_change != 1) || (hydrostatic != 0 && hydrostatic != 1) ||
      (method == 0 && box_change)) {
    set_error("b200md_minimizer_create: method 0 (sd) or 1 (fire), n > 0, steps > 0, box_change and "
              "hydrostatic 0 or 1 (fire only)");
    return B200MD_ERR_ARG;
  }
  b200md_minimizer* p = new (std::nothrow) b200md_minimizer;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->method = method;
  p->n = n;
  p->steps = number_of_steps;
  p->tol = force_tolerance;
  p->box_change = box_change;
  p->hydrostatic = hydrostatic;
  const size_t n3 = (size_t)3 * n;
  cudaError_t e = cudaSuccess;
  if (method == 1)
    e = p->v.reserve(n3);
  if (e == cudaSuccess && (e = p->partial.reserve((size_t)RED_GRID * RED_K)) == cudaSuccess &&
      (e = p->rec.reserve(B200MD_MIN_RECORD)) == cudaSuccess)
    e = p->ticket.reserve(1);
  if (e != cudaSuccess) {
    set_error("out of device memory (minimizer)");
    delete p;
    return B200MD_ERR_CUDA;
  }
  double r[B200MD_MIN_RECORD] = {0};
  r[B200MD_MIN_DT] = DT_0;
  r[B200MD_MIN_ALPHA] = ALPHA_START;
  r[B200MD_MIN_STEP] = 0.1; // minimizer_sd.cu:78
  e = cudaMemcpy(p->rec.p, r, sizeof r, cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaMemset(p->ticket.p, 0, sizeof(unsigned int));
  if (e == cudaSuccess && method == 1)
    e = cudaMemset(p->v.p, 0, n3 * sizeof(double)); // the FIRE velocity starts at zero
  if (e == cudaSuccess)
    e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    set_error(std::string("b200md_minimizer_create: ") + cudaGetErrorString(e));
    delete p;
    return B200MD_ERR_CUDA;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_minimizer_destroy(b200md_minimizer* p) { delete p; }

double* b200md_minimizer_velocity(b200md_minimizer* p) { return p ? p->v.p : nullptr; }

int b200md_minimizer_set_record(b200md_minimizer* p, const double* record, void* stream)
{
  if (!p || !record) {
    set_error("b200md_minimizer_set_record: null handle or record");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (record[B200MD_MIN_LSCALE] > 0.0)
    p->L = record[B200MD_MIN_LSCALE];
  B2_CUDA(cudaMemcpyAsync(p->rec.p, record, B200MD_MIN_RECORD * sizeof(double), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200MD_OK;
}

// trial positions from the state the last reduction left in the record, then the record to the host
static int sd_trial(
  b200md_minimizer* p, int n, const double* d_position, const double* d_force, double* d_position_trial,
  const int* d_group_label, int fixed_group, double* record, cudaStream_t st)
{
  k_sd_trial<<<grid_for(3LL * n, BLK), BLK, 0, st>>>(
    3 * n, n, d_position, d_force, d_group_label, fixed_group, d_position_trial, p->rec.p);
  B2_LAUNCHED();
  return fetch(p, record, st);
}

static bool bad_sd(
  const double* d_position_trial, const double* d_force_trial, const double* d_potential_trial,
  int fixed_group, const int* d_group_label)
{
  if (!d_position_trial || !d_force_trial || !d_potential_trial || (fixed_group >= 0 && !d_group_label)) {
    set_error("b200md_minimizer_sd: the trial arrays are missing, or a fixed group without the group labels");
    return true;
  }
  return false;
}

int b200md_minimizer_sd_begin(
  b200md_minimizer* p, int n, double* d_position, double* d_force, double* d_potential,
  double* d_position_trial, const double* d_force_trial, const double* d_potential_trial,
  const int* d_group_label, int fixed_group, double* record, void* stream)
{
  if (bad_call(p, 0, n, "b200md_minimizer_sd_begin") ||
      bad_sd(d_position_trial, d_force_trial, d_potential_trial, fixed_group, d_group_label))
    return B200MD_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  k_sd_accept<<<b2_reduce_blocks(n, BLK, RED_GRID), BLK, 0, st>>>(
    n, 1, d_position, d_force, d_potential, d_position_trial, d_force_trial, d_potential_trial, p->partial.p, p->ticket.p, p->rec.p,
    p->tol);
  B2_LAUNCHED();
  return sd_trial(p, n, d_position, d_force, d_position_trial, d_group_label, fixed_group, record, st);
}

int b200md_minimizer_sd_step(
  b200md_minimizer* p, int n, double* d_position, double* d_force, double* d_potential,
  double* d_position_trial, const double* d_force_trial, const double* d_potential_trial,
  const int* d_group_label, int fixed_group, double* record, void* stream)
{
  if (bad_call(p, 0, n, "b200md_minimizer_sd_step") ||
      bad_sd(d_position_trial, d_force_trial, d_potential_trial, fixed_group, d_group_label))
    return B200MD_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int g = b2_reduce_blocks(n, BLK, RED_GRID);
  k_sd_energy<<<g, BLK, 0, st>>>(n, d_potential_trial, p->partial.p, p->ticket.p, p->rec.p);
  B2_LAUNCHED();
  k_sd_accept<<<g, BLK, 0, st>>>(
    n, 0, d_position, d_force, d_potential, d_position_trial, d_force_trial, d_potential_trial, p->partial.p, p->ticket.p, p->rec.p,
    p->tol);
  B2_LAUNCHED();
  return sd_trial(p, n, d_position, d_force, d_position_trial, d_group_label, fixed_group, record, st);
}

int b200md_minimizer_fire_step(
  b200md_minimizer* p, int n, double h[9], double* d_position, const double* d_force,
  const double* d_potential, const double* d_virial, double* record, void* stream)
{
  if (bad_call(p, 1, n, "b200md_minimizer_fire_step"))
    return B200MD_ERR_ARG;
  if (p->box_change && (!h || !d_virial)) {
    set_error("b200md_minimizer_fire_step: box change needs h and the virial");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  FireParams prm = {p->tol, 0.0, 1.0, p->box_change, p->hydrostatic};
  if (p->box_change) {
    const int pbc[3] = {1, 1, 1};
    prm.volume = make_box(h, pbc).volume;
    if (!(p->L > 0.0)) // L = cbrt(V) of the box the minimization starts from
      p->L = std::cbrt(prm.volume);
    prm.L = p->L;
    k_fire_reduce<true><<<b2_reduce_blocks(n, BLK, RED_GRID), BLK, 0, st>>>(
      n, d_force, p->v.p, d_potential, d_virial, p->partial.p, p->ticket.p, p->rec.p, prm);
    B2_LAUNCHED();
    k_fire_update<true><<<grid_for(n, BLK), BLK, 0, st>>>(n, d_position, p->v.p, d_force, p->rec.p);
  } else {
    k_fire_reduce<false><<<b2_reduce_blocks(n, BLK, RED_GRID), BLK, 0, st>>>(
      n, d_force, p->v.p, d_potential, nullptr, p->partial.p, p->ticket.p, p->rec.p, prm);
    B2_LAUNCHED();
    k_fire_update<false><<<grid_for(n, BLK), BLK, 0, st>>>(n, d_position, p->v.p, d_force, p->rec.p);
  }
  B2_LAUNCHED();
  double r[B200MD_MIN_RECORD];
  double* out = record ? record : r;
  if (fetch(p, out, st) != B200MD_OK)
    return B200MD_ERR_CUDA;
  out[B200MD_MIN_LSCALE] = p->L;
  if (p->box_change && out[B200MD_MIN_CONVERGED] == 0.0) {
    // h <- h + dEps h (minimizer_fire_box_change.cu:385-390), on the host copy the caller owns
    const double* e = out + B200MD_MIN_DEPS;
    double dh[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        dh[i * 3 + j] = 0.0;
        for (int k = 0; k < 3; ++k)
          dh[i * 3 + j] += e[i * 3 + k] * h[k * 3 + j];
      }
    for (int i = 0; i < 9; ++i)
      h[i] += dh[i];
  }
  return B200MD_OK;
}

} // extern "C"

// b2_integrate.cuh -- bodies of the streaming kernels around the force call:
//   position wrap        gpu_apply_pbc, src/force/force.cu:424-459
//   velocity-Verlet      gpu_velocity_verlet, src/integrate/ensemble.cu:176-214
//   thermo partial sums  gpu_find_thermo_instant_temperature, src/integrate/ensemble.cu:434-633
#pragma once
#include "b2_common.cuh"

B2_HD void b2_body_apply_pbc(int i, int n, const B2Box& b, double* x, double* y, double* z)
{
  const double px = x[i], py = y[i], pz = z[i];
  double sx = b.h[9] * px + b.h[10] * py + b.h[11] * pz;
  double sy = b.h[12] * px + b.h[13] * py + b.h[14] * pz;
  double sz = b.h[15] * px + b.h[16] * py + b.h[17] * pz;
  if (b.pbc[0]) {
    if (sx < 0.0)
      sx += 1.0;
    else if (sx > 1.0)
      sx -= 1.0;
  }
  if (b.pbc[1]) {
    if (sy < 0.0)
      sy += 1.0;
    else if (sy > 1.0)
      sy -= 1.0;
  }
  if (b.pbc[2]) {
    if (sz < 0.0)
      sz += 1.0;
    else if (sz > 1.0)
      sz -= 1.0;
  }
  x[i] = b.h[0] * sx + b.h[1] * sy + b.h[2] * sz;
  y[i] = b.h[3] * sx + b.h[4] * sy + b.h[5] * sz;
  z[i] = b.h[6] * sx + b.h[7] * sy + b.h[8] * sz;
}

// `stride` = distance between the x, y, z blocks of the SoA arrays (= n for GPUMD's own arrays;
// larger when only the first n atoms of a longer local array are owned, domain decomposition)
B2_HD void b2_body_vv(
  int i, int stride, bool step1, double dt, const double* mass, double* pos, double* vel,
  const double* f)
{
  const size_t N = (size_t)stride;
  const double minv = 1.0 / mass[i];
  const double half = dt * 0.5;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    double v = vel[d * N + i];
    v += f[d * N + i] * minv * half;
    vel[d * N + i] = v;
    if (step1)
      pos[d * N + i] += v * dt;
  }
}

// The same half step with the reference's group rules (gpu_velocity_verlet with groups,
// src/integrate/ensemble.cu:111-174): atoms of `fixed_group` do not move and have zero velocity,
// atoms of `move_group` are translated with the constant velocity mv[] (stored velocity zero, so
// that they do not enter the temperature); everything else is integrated normally.  label[] is
// Group::label of the grouping method the fix / move keywords named.
B2_HD void b2_body_vv_groups(
  int i, int stride, bool step1, double dt, const double* mass, double* pos, double* vel,
  const double* f, const int* label, int fixed_group, int move_group, const double* mv)
{
  const size_t N = (size_t)stride;
  const int g = label[i];
  if (g == fixed_group) {
#pragma unroll
    for (int d = 0; d < 3; ++d)
      vel[d * N + i] = 0.0; // pos += 0 * dt
    return;
  }
  if (g == move_group) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      vel[d * N + i] = 0.0;
      if (step1)
        pos[d * N + i] += mv[d] * dt;
    }
    return;
  }
  b2_body_vv(i, stride, step1, dt, mass, pos, vel, f);
}

// Nose-Hoover chain of length 4, Suzuki-Yoshida order 7 x 4 RESPA sub-steps (the `nhc` function of
// src/integrate/ensemble_nhc.cu:101-171, after Tuckerman) over half a time step.  state = {eta[4],
// v_eta[4], Q[4]}; ek2 = twice the kinetic energy the chain couples to, dof its degrees of freedom.
// Returns the velocity scale factor.  Shared by nvt_nhc and the two chains of heat_nhc.
B2_HD double b2_nhc_chain(double* state, double ek2, double dof, double kT, double dt_half)
{
  constexpr int M = 4;
  const double w[7] = {0.784513610477560, 0.235573213359357, -1.17767998417887, 1.31518632068391,
                       -1.17767998417887, 0.235573213359357, 0.784513610477560};
  double* eta = state;
  double* ve = state + M;
  const double* Q = state + 2 * M;
  double factor = 1.0;
  for (int a = 0; a < 7; ++a) {
    const double dt2 = dt_half * w[a] / 4.0, dt4 = 0.5 * dt2, dt8 = 0.5 * dt4;
    for (int b = 0; b < 4; ++b) {
      ve[M - 1] += dt4 * (ve[M - 2] * ve[M - 2] / Q[M - 2] - kT);
      for (int m = M - 2; m >= 0; --m) {
        const double damp = exp(-dt8 * ve[m + 1] / Q[m + 1]);
        const double G = (m == 0) ? ek2 - dof * kT : ve[m - 1] * ve[m - 1] / Q[m - 1] - kT;
        ve[m] = damp * (damp * ve[m] + dt4 * G);
      }
      for (int m = M - 1; m >= 0; --m)
        eta[m] += dt2 * ve[m] / Q[m];
      const double f = exp(-dt2 * ve[0] / Q[0]);
      ek2 *= f * f;
      factor *= f;
      for (int m = 0; m < M - 1; ++m) {
        const double damp = exp(-dt8 * ve[m + 1] / Q[m + 1]);
        const double G = (m == 0) ? ek2 - dof * kT : ve[m - 1] * ve[m - 1] / Q[m - 1] - kT;
        ve[m] = damp * (damp * ve[m] + dt4 * G);
      }
      ve[M - 1] += dt4 * (ve[M - 2] * ve[M - 2] / Q[M - 2] - kT);
    }
  }
  return factor;
}

// per-atom contributions to the 8 sums: m v^2, U, W_ab + m v_a v_b (ab = xx,yy,zz,xy,xz,yz)
B2_HD void b2_thermo_terms(
  int i, int stride, const double* mass, const double* pe, const double* vel, const double* virial,
  double* t)
{
  const size_t N = (size_t)stride;
  const double m = mass[i];
  const double vx = vel[i], vy = vel[N + i], vz = vel[2 * N + i];
  t[0] = (vx * vx + vy * vy + vz * vz) * m;
  t[1] = pe[i];
  t[2] = virial[i] + vx * vx * m;
  t[3] = virial[N + i] + vy * vy * m;
  t[4] = virial[2 * N + i] + vz * vz * m;
  t[5] = virial[3 * N + i] + vx * vy * m;
  t[6] = virial[4 * N + i] + vx * vz * m;
  t[7] = virial[5 * N + i] + vy * vz * m;
}

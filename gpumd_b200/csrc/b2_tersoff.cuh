// b2_tersoff.cuh -- Tersoff-1989 bodies (FP64 like the reference, src/force/tersoff1989.cu).
//
// The reference runs three passes over global arrays: step1 (b, b' per pair, O(NN^2) with an
// exp/cos per inner iteration, tersoff1989.cu:337-405), step2 (partial forces, again O(NN^2) with
// exp/cos inside, :408-505) and the pair reduction (potential.cu:35-134), after a separate local
// list filter (neighbor.cu:699-737).  Here one kernel does filter + step1 + step2 per atom: the
// per-neighbour radial functions (fc, fc', fa, fa', fr, fr') and unit data are evaluated ONCE into
// a small per-thread table, so the O(NN^2) loops are pure arithmetic; b/b' never touch global
// memory.  The second kernel is the gather-only pair reduction (binary search of the reverse slot
// in the ascending list).
#pragma once
#include "b2_common.cuh"

struct B2TersoffPara {
  double a, b, lambda, mu, beta, n, c2, d2, h, r1, r2, one_plus, pi_factor, mhn;
};

constexpr int B2_TERSOFF_MAXL = 32; // local neighbours per atom (covalent: 3-8)

struct B2TersoffView {
  B2TersoffPara p[3]; // [0] type 0-0, [1] type 1-1, [2] mixed (tersoff1989.cu:107-124)
  float rc2;          // FP32 membership test of the local list (neighbor.cu:720-735)
  int n;
  const B2Atom* atoms;
  const int* nn_skin;
  const int* nl_skin;
  int* nn;     // [n]
  int* nl;     // [MAXL * n]
  double* f12; // [3][MAXL * n]
  double* acc; // [13 * n]
  int* flags;
};

B2_HD void b2_tersoff_fc(const B2TersoffPara& t, double d, double& fc, double& fcp)
{
  if (d < t.r1) {
    fc = 1.0;
    fcp = 0.0;
  } else if (d < t.r2) {
    const double arg = t.pi_factor * (d - t.r1);
    fc = cos(arg) * 0.5 + 0.5;
    fcp = -sin(arg) * t.pi_factor * 0.5;
  } else {
    fc = 0.0;
    fcp = 0.0;
  }
}

B2_HD void b2_body_tersoff_partial(int i, const B2TersoffView& P, const B2Box& box)
{
  const size_t N = (size_t)P.n;
  const B2Geo geo = b2_geo(box);
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  const B2TersoffPara& ti = P.p[t1];
  int jl[B2_TERSOFF_MAXL];
  double rx[B2_TERSOFF_MAXL], ry[B2_TERSOFF_MAXL], rz[B2_TERSOFF_MAXL], dd[B2_TERSOFF_MAXL];
  double fcv[B2_TERSOFF_MAXL], fcpv[B2_TERSOFF_MAXL], fav[B2_TERSOFF_MAXL], bpv[B2_TERSOFF_MAXL];
  // ---- local list + per-neighbour radial functions ----
  int m = 0, overflow = 0;
  const int ns = P.nn_skin[i];
  for (int k = 0; k < ns; ++k) {
    const int j = P.nl_skin[(size_t)k * N + i];
    const B2Atom a2 = b2_load_atom(&P.atoms[j]);
    float xf, yf, zf;
    b2_r12(geo, box, a1, a2, xf, yf, zf);
    if (b2_d2(xf, yf, zf) >= P.rc2)
      continue;
    if (m >= B2_TERSOFF_MAXL) {
      overflow = 1;
      break;
    }
    double x12 = a2.x - a1.x, y12 = a2.y - a1.y, z12 = a2.z - a1.z;
    b2_mic(box, x12, y12, z12);
    const double d = sqrt(x12 * x12 + y12 * y12 + z12 * z12);
    const B2TersoffPara& tp = P.p[(t1 == a2.type) ? t1 : 2];
    jl[m] = j;
    rx[m] = x12;
    ry[m] = y12;
    rz[m] = z12;
    dd[m] = d;
    b2_tersoff_fc(tp, d, fcv[m], fcpv[m]);
    fav[m] = tp.b * exp(-tp.mu * d);
    ++m;
  }
  if (overflow)
    B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_ANGULAR_OVERFLOW);
  P.nn[i] = m;
  // ---- bond order: zeta_ij, b_ij, b'_ij (step 1) ----
  double bv[B2_TERSOFF_MAXL];
  for (int a = 0; a < m; ++a) {
    double zeta = 0.0;
    for (int c = 0; c < m; ++c) {
      if (c == a)
        continue;
      const double cs = (rx[a] * rx[c] + ry[a] * ry[c] + rz[a] * rz[c]) / (dd[a] * dd[c]);
      const double tmp = ti.d2 + (cs - ti.h) * (cs - ti.h);
      zeta += fcv[c] * (ti.one_plus - ti.c2 / tmp);
    }
    const double bzn = pow(ti.beta * zeta, ti.n);
    const double b12 = pow(1.0 + bzn, ti.mhn);
    if (zeta < 1.0e-16) { // avoid division by 0 (tersoff1989.cu:395-399)
      bv[a] = 1.0;
      bpv[a] = 0.0;
    } else {
      bv[a] = b12;
      bpv[a] = -b12 * bzn * 0.5 / ((1.0 + bzn) * zeta);
    }
  }
  // ---- partial forces (step 2) ----
  const size_t plane = (size_t)B2_TERSOFF_MAXL * N;
  double pe = 0.0;
  for (int a = 0; a < m; ++a) {
    const B2TersoffPara& tp = P.p[(t1 == P.atoms[jl[a]].type) ? t1 : 2];
    const double d12 = dd[a], d12inv = 1.0 / d12;
    const double fc12 = fcv[a], fcp12 = fcpv[a], fa12 = fav[a];
    const double fap12 = -tp.mu * fa12;
    const double fr12 = tp.a * exp(-tp.lambda * d12), frp12 = -tp.lambda * fr12;
    const double b12 = bv[a], bp12 = bpv[a];
    const double f3 = (fcp12 * (fr12 - b12 * fa12) + fc12 * (frp12 - b12 * fap12)) * d12inv;
    double fx = rx[a] * f3 * 0.5, fy = ry[a] * f3 * 0.5, fz = rz[a] * f3 * 0.5;
    pe += fc12 * (fr12 - b12 * fa12) * 0.5;
    for (int c = 0; c < m; ++c) {
      if (c == a)
        continue;
      const double inv = 1.0 / (d12 * dd[c]);
      const double cs = (rx[a] * rx[c] + ry[a] * ry[c] + rz[a] * rz[c]) * inv;
      const double cs_dd = cs * d12inv * d12inv;
      const double tmp = ti.d2 + (cs - ti.h) * (cs - ti.h);
      const double g = ti.one_plus - ti.c2 / tmp;
      const double gp = 2.0 * ti.c2 * (cs - ti.h) / (tmp * tmp);
      const double ta = (-bp12 * fc12 * fa12 * fcv[c] - bpv[c] * fcv[c] * fav[c] * fc12) * gp;
      const double tb = -bpv[c] * fcv[c] * fav[c] * fcp12 * g * d12inv;
      fx += (rx[a] * tb + ta * (rx[c] * inv - rx[a] * cs_dd)) * 0.5;
      fy += (ry[a] * tb + ta * (ry[c] * inv - ry[a] * cs_dd)) * 0.5;
      fz += (rz[a] * tb + ta * (rz[c] * inv - rz[a] * cs_dd)) * 0.5;
    }
    const size_t slot = (size_t)a * N + i;
    P.nl[slot] = jl[a];
    P.f12[slot] = fx;
    P.f12[plane + slot] = fy;
    P.f12[2 * plane + slot] = fz;
  }
  P.acc[i] = pe;
}

// F_i = sum_j (f12 - f21), W_i = sum_j r12 (x) f21 in FP64 (potential.cu:35-134)
B2_HD void b2_body_tersoff_reduce(int i, const B2TersoffView& P, const B2Box& box)
{
  const size_t N = (size_t)P.n;
  const size_t plane = (size_t)B2_TERSOFF_MAXL * N;
  const B2Atom a1 = P.atoms[i];
  const int m = P.nn[i];
  double f[3] = {0.0, 0.0, 0.0};
  double v[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int a = 0; a < m; ++a) {
    const size_t slot = (size_t)a * N + i;
    const int j = P.nl[slot];
    const B2Atom a2 = b2_load_atom(&P.atoms[j]);
    double r[3] = {a2.x - a1.x, a2.y - a1.y, a2.z - a1.z};
    b2_mic(box, r[0], r[1], r[2]);
    int lo = 0, hi = P.nn[j] - 1, rev = 0;
    while (lo <= hi) {
      const int mid = (lo + hi) >> 1;
      const int v2 = P.nl[(size_t)mid * N + j];
      if (v2 < i)
        lo = mid + 1;
      else if (v2 > i)
        hi = mid - 1;
      else {
        rev = mid;
        break;
      }
    }
    const size_t rslot = (size_t)rev * N + j;
    const double f12[3] = {P.f12[slot], P.f12[plane + slot], P.f12[2 * plane + slot]};
    const double f21[3] = {P.f12[rslot], P.f12[plane + rslot], P.f12[2 * plane + rslot]};
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      f[d] += f12[d] - f21[d];
#pragma unroll
      for (int e = 0; e < 3; ++e)
        v[d * 3 + e] += r[d] * f21[e];
    }
  }
  double* acc = P.acc + i;
  acc[1 * N] = f[0];
  acc[2 * N] = f[1];
  acc[3 * N] = f[2];
  acc[4 * N] = v[0];
  acc[5 * N] = v[4];
  acc[6 * N] = v[8];
  acc[7 * N] = v[1];
  acc[8 * N] = v[2];
  acc[9 * N] = v[5];
  acc[10 * N] = v[3];
  acc[11 * N] = v[6];
  acc[12 * N] = v[7];
}

// per-atom heat current jx_in jx_out jy_in jy_out jz (gpu_compute_heat,
// src/measure/compute_heat.cu:32-63).  The one definition of these expressions: compute_heat / HAC
// (b2_body_heat) and the fused HNEMD heat sum (b2_measure.cu) both call it.
B2_HD void b2_heat5(int i, int stride, const double* w, const double* vel, double h[5])
{
  const size_t n = (size_t)stride;
  const double vx = vel[i], vy = vel[n + i], vz = vel[2 * n + i];
  h[0] = w[i] * vx + w[3 * n + i] * vy;
  h[1] = w[4 * n + i] * vz;
  h[2] = w[6 * n + i] * vx + w[n + i] * vy;
  h[3] = w[5 * n + i] * vz;
  h[4] = w[7 * n + i] * vx + w[8 * n + i] * vy + w[2 * n + i] * vz;
}

B2_HD void b2_body_heat(
  int i, int stride, const double* w, const double* vel, double* heat, int hstride)
{
  double h[5];
  b2_heat5(i, stride, w, vel, h);
  for (int k = 0; k < 5; ++k)
    heat[(size_t)hstride * k + i] = h[k];
}

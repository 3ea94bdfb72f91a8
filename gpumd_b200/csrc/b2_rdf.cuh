// b2_rdf.cuh -- kernel bodies of the radial distribution function (compute_rdf).
//
// Replaces gpu_find_rdf_ON1 (src/measure/rdf.cu:37-125) with a different design:
//   * each UNORDERED pair is evaluated once: atom i of the cell-sorted order (b2_neighbor.cuh) walks the
//     +-2 cells around its own and takes the atoms j > i only.  The reference's d2 is bit-symmetric
//     under i <-> j (negation passes exactly through the orthogonal compares, nearbyint and the fma
//     nesting below), so the ordered counts follow in integers: partial(a,a) = 2 u(a,a),
//     partial(a<b) = u(a,b), total = 2 sum u;
//   * pairs are COUNTED into 64-bit integer bins, one counter per pair, and every sample is folded into
//     the FP64 accumulator as count x norm(V) in a fixed order.  The reference adds 1 / (N rho dV) with
//     one double atomicAdd per matching column, so its result depends on the order the atomics land;
//   * the bin is found in O(1) from sqrt(d2) / dr and settled with the reference's own two squared-bound
//     comparisons (rdf.cu:102-106), instead of a loop over every bin.
// Semantics kept from the reference: FP64 x[j] - x[i], the FP64 minimum image (box.cuh:37-82), the drop
// d2 > rc^2, bin w for (w dr)^2 < d2 <= ((w+1) dr)^2 (so d2 = 0 and d2 in ((num_bins dr)^2, rc^2] land in
// no bin), and dV = r_mid^2 4 pi dr evaluated left to right.
#pragma once
#include "b2_neighbor.cuh"

constexpr double B2_RDF_PI = 3.14159265358979323846; // rdf.cu:55

struct B2RdfPara {
  int num_bins;
  int num_types; // species present, in type-id order
  int num_pairs; // num_types (num_types + 1) / 2: the counter table is [num_pairs][num_bins]
  double dr;     // rc / num_bins
  double rc2;    // rc * rc
};

// FP64 minimum image with the fma nesting nvcc emits for the reference's apply_mic (read from the PTX of
// rdf.cu): a*x + b*y + c*z = fma(c,z, fma(a,x, b*y)).  Written out so that the host build (tests/emu) and
// the device compute the same bits.
B2_HD void b2_rdf_mic(const B2Box& b, double& x, double& y, double& z)
{
  if (b.ortho) {
    if (b.pbc[0]) {
      const double L = b.h[0];
      if (x < -L * 0.5)
        x += L;
      else if (x > L * 0.5)
        x -= L;
    }
    if (b.pbc[1]) {
      const double L = b.h[4];
      if (y < -L * 0.5)
        y += L;
      else if (y > L * 0.5)
        y -= L;
    }
    if (b.pbc[2]) {
      const double L = b.h[8];
      if (z < -L * 0.5)
        z += L;
      else if (z > L * 0.5)
        z -= L;
    }
  } else {
    double sx = fma(b.h[11], z, fma(b.h[9], x, b.h[10] * y));
    double sy = fma(b.h[14], z, fma(b.h[12], x, b.h[13] * y));
    double sz = fma(b.h[17], z, fma(b.h[15], x, b.h[16] * y));
    if (b.pbc[0])
      sx -= nearbyint(sx);
    if (b.pbc[1])
      sy -= nearbyint(sy);
    if (b.pbc[2])
      sz -= nearbyint(sz);
    x = fma(b.h[2], sz, fma(b.h[0], sx, b.h[1] * sy));
    y = fma(b.h[5], sz, fma(b.h[3], sx, b.h[4] * sy));
    z = fma(b.h[8], sz, fma(b.h[6], sx, b.h[7] * sy));
  }
}

// x12*x12 + y12*y12 + z12*z12 as nvcc contracts it in rdf.cu:97
B2_HD double b2_rdf_d2(double x, double y, double z) { return fma(z, z, fma(x, x, y * y)); }

// (w dr)^2, the reference's r_low of bin w and r_up of bin w - 1 (rdf.cu:102-103)
B2_HD double b2_rdf_edge(int w, double dr)
{
  const double r = w * dr;
  return r * r;
}

// the bin of a pair, or -1: a candidate from sqrt(d2) / dr, settled by the reference's comparisons
// d2 > r_low && d2 <= r_up.  The edges ascend with w, so at most one bin matches
B2_HD int b2_rdf_bin(double d2, const B2RdfPara& p)
{
  if (d2 > p.rc2)
    return -1;
  int w = (int)(sqrt(d2) / p.dr);
  if (w > p.num_bins - 1)
    w = p.num_bins - 1;
  while (w > 0 && !(d2 > b2_rdf_edge(w, p.dr)))
    --w;
  while (w < p.num_bins - 1 && d2 > b2_rdf_edge(w + 1, p.dr))
    ++w;
  return (d2 > b2_rdf_edge(w, p.dr) && d2 <= b2_rdf_edge(w + 1, p.dr)) ? w : -1;
}

// column of the species pair (a, b), a <= b, in the reference's order (0,0), (0,1), .. (0,T-1), (1,1), ..
B2_HD int b2_rdf_pair(int a, int b, int T) { return a * (2 * T - a + 1) / 2 + (b - a); }

// coordinate c + o of a +-2 walk along one direction (b2_axis_walk's cells): wrapped when periodic
// (nb >= 5, so the five are distinct), -1 past an open edge
B2_HD int b2_rdf_walk(int c, int o, int nb, int pbc)
{
  int k = c + o;
  if (k < 0)
    k = pbc ? k + nb : -1;
  else if (k >= nb)
    k = pbc ? k - nb : -1;
  return k;
}

// The unordered pairs (i, j > i) of sorted atom i over the +-2 cells of b2_body_skin_list.  The atoms are
// sorted by cell id, x fastest, so the x-cells of one (y, z) row are at most two runs of consecutive
// cells (two when the walk wraps), each one contiguous range of atoms; j > i keeps the part of a range
// after i (the cells below i's own hold only j < i).  The walk keeps no arrays, so nothing goes to local
// memory.  species[t] = the species of type t, or -1.  emit(k) is called with the counter
// k = pair * num_bins + bin of every binned pair.
template <class Emit>
B2_HD void b2_body_rdf_atom(
  int i, const B2Atom* atoms, const int* cell_start, const B2Box& box, const B2Grid& g, const B2RdfPara& p,
  const int* species, Emit emit)
{
  const B2Atom a1 = b2_load_atom(atoms + i);
  const int s1 = (unsigned)a1.type < (unsigned)B2_MAX_TYPES ? species[a1.type] : -1;
  if (s1 < 0)
    return;
  int cx, cy, cz;
  b2_cell_of(box, g, a1, &cx, &cy, &cz);
  // the x runs [x0, x1] and [x2, x3] (the second empty unless the walk wraps)
  int x0 = cx - 2, x1 = cx + 2, x2 = 0, x3 = -1;
  if (!box.pbc[0]) {
    x0 = x0 < 0 ? 0 : x0;
    x1 = x1 >= g.nb[0] ? g.nb[0] - 1 : x1;
  } else if (x0 < 0) {
    x2 = x0 + g.nb[0];
    x3 = g.nb[0] - 1;
    x0 = 0;
  } else if (x1 >= g.nb[0]) {
    x2 = 0;
    x3 = x1 - g.nb[0];
    x1 = g.nb[0] - 1;
  }
  for (int oz = -2; oz <= 2; ++oz) {
    const int kz = b2_rdf_walk(cz, oz, g.nb[2], box.pbc[2]);
    if (kz < 0)
      continue;
    for (int oy = -2; oy <= 2; ++oy) {
      const int ky = b2_rdf_walk(cy, oy, g.nb[1], box.pbc[1]);
      if (ky < 0)
        continue;
      const int row = g.nb[0] * (ky + g.nb[1] * kz);
      for (int run = 0; run < 2; ++run) {
        const int lo = run ? x2 : x0, hi = run ? x3 : x1;
        if (hi < lo)
          continue;
        const int s_end = cell_start[row + hi + 1];
        int j = cell_start[row + lo];
        if (j <= i)
          j = i + 1;
        for (; j < s_end; ++j) {
          const B2Atom a2 = b2_load_atom(atoms + j);
          const int s2 = (unsigned)a2.type < (unsigned)B2_MAX_TYPES ? species[a2.type] : -1;
          if (s2 < 0)
            continue;
          double x12 = a2.x - a1.x, y12 = a2.y - a1.y, z12 = a2.z - a1.z;
          b2_rdf_mic(box, x12, y12, z12);
          const int w = b2_rdf_bin(b2_rdf_d2(x12, y12, z12), p);
          if (w >= 0) {
            const int pair = s1 <= s2 ? b2_rdf_pair(s1, s2, p.num_types) : b2_rdf_pair(s2, s1, p.num_types);
            emit(pair * p.num_bins + w);
          }
        }
      }
    }
  }
}

// count x factor, never contracted into the accumulation that follows
B2_HD double b2_rdf_term(unsigned long long count, double factor)
{
#if defined(__CUDA_ARCH__)
  return __dmul_rn((double)count, factor);
#else
  return (double)count * factor;
#endif
}

// Fold bin w of one sample into acc[w][1 + num_pairs] (rdf.cu's rdf_g_ layout: total, then (a,b) for
// a <= b) and zero its counters.  volume = Box::get_volume at the sample; num_atoms[a] = atoms of species
// a, n = all atoms.  The factors are rdf.cu:102-112 in its order of operations: 1 / (N (N / V) dV) for
// the total, 1 / (N_a (N_b / V) dV) for (a, b), with dV = r_mid^2 * 4 * pi * dr
B2_HD void b2_body_rdf_fold(
  int w, const B2RdfPara& p, double volume, int n, const int* num_atoms, unsigned long long* counts, double* acc)
{
  const double r_mid = (w + 0.5) * p.dr;
  const double dV = r_mid * r_mid * 4 * B2_RDF_PI * p.dr;
  const int R = 1 + p.num_pairs;
  unsigned long long total = 0;
  int k = 0;
  for (int a = 0; a < p.num_types; ++a) {
    for (int b = a; b < p.num_types; ++b, ++k) {
      const unsigned long long u = counts[(size_t)k * p.num_bins + w];
      counts[(size_t)k * p.num_bins + w] = 0;
      total += u;
      const unsigned long long c = a == b ? 2 * u : u; // the ordered pairs i in a, j in b
      const double density_b = num_atoms[b] / volume;
      acc[(size_t)w * R + 1 + k] += b2_rdf_term(c, 1 / (num_atoms[a] * density_b * dV));
    }
  }
  const double density = n / volume;
  acc[(size_t)w * R] += b2_rdf_term(2 * total, 1 / (n * density * dV));
}

// tests/emu/rdf_emu.cpp -- TEST INFRASTRUCTURE ONLY: the RDF kernel bodies (gpumd_b200/csrc/b2_rdf.cuh)
// compiled for the host.  The cell sort is a serial restatement of the neighbour module's counting sort
// (ascending cell, then ascending atom index), the pair walk and the bin rule are the device's own
// b2_body_rdf_atom, and the fold is b2_body_rdf_fold.  The block-private tables, the warp-aggregated
// atomics and the flush are covered by the `-m gpu` tests only.
#include "../../gpumd_b200/csrc/b2_rdf.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace {

// Box::get_inverse / get_volume / thickness / set_is_orthogonal (b2_host.cu's make_box)
B2Box make_box(const double h[9], const int pbc[3])
{
  B2Box b;
  double* c = b.h;
  for (int d = 0; d < 9; ++d)
    c[d] = h[d];
  for (int d = 0; d < 3; ++d)
    b.pbc[d] = pbc[d] ? 1 : 0;
  c[9] = c[4] * c[8] - c[5] * c[7];
  c[10] = c[2] * c[7] - c[1] * c[8];
  c[11] = c[1] * c[5] - c[2] * c[4];
  c[12] = c[5] * c[6] - c[3] * c[8];
  c[13] = c[0] * c[8] - c[2] * c[6];
  c[14] = c[2] * c[3] - c[0] * c[5];
  c[15] = c[3] * c[7] - c[4] * c[6];
  c[16] = c[1] * c[6] - c[0] * c[7];
  c[17] = c[0] * c[4] - c[1] * c[3];
  const double det = c[0] * c[9] + c[1] * c[12] + c[2] * c[15];
  for (int d = 9; d < 18; ++d)
    c[d] /= det;
  b.volume = std::fabs(det);
  for (int d = 0; d < 3; ++d) {
    const int p = (d + 1) % 3, q = (d + 2) % 3;
    const double u[3] = {c[p], c[p + 3], c[p + 6]}, w[3] = {c[q], c[q + 3], c[q + 6]};
    const double s0 = u[1] * w[2] - u[2] * w[1], s1 = u[2] * w[0] - u[0] * w[2], s2 = u[0] * w[1] - u[1] * w[0];
    b.thickness[d] = b.volume / std::sqrt(s0 * s0 + s1 * s1 + s2 * s2);
  }
  b.ortho = c[1] == 0 && c[2] == 0 && c[3] == 0 && c[5] == 0 && c[6] == 0 && c[7] == 0;
  for (int d = 0; d < 18; ++d)
    b.hf[d] = (float)c[d];
  return b;
}

B2RdfPara make_para(double rc, int num_bins, int num_types)
{
  B2RdfPara p;
  p.num_bins = num_bins;
  p.num_types = num_types;
  p.num_pairs = num_types * (num_types + 1) / 2;
  p.dr = rc / num_bins;
  p.rc2 = rc * rc;
  return p;
}

} // namespace

extern "C" {

int rdf_emu_bin(double d2, double rc, int num_bins)
{
  return b2_rdf_bin(d2, make_para(rc, num_bins, 1));
}

// u[num_pairs][num_bins] of one sample; returns the number of cells, or -1 for a periodic direction
// with fewer than 5 of them
int rdf_emu_count(int n, const double* h9, const int* pbc, const int* type, const double* pos, double rc,
                  int num_bins, int num_types, const int* type_index, unsigned long long* u)
{
  const B2Box box = make_box(h9, pbc);
  const B2RdfPara p = make_para(rc, num_bins, num_types);
  B2Grid g; // make_grid, b2_neighbor.cu
  for (int d = 0; d < 3; ++d) {
    int nb = (int)floor(box.thickness[d] / (0.5 * rc));
    g.nb[d] = nb < 1 ? 1 : nb;
    g.scale[d] = (double)g.nb[d];
    if (box.pbc[d] && g.nb[d] < 5)
      return -1;
  }
  g.ncell = g.nb[0] * g.nb[1] * g.nb[2];
  std::vector<B2Atom> in(n);
  std::vector<int> cell(n), order(n);
  for (int i = 0; i < n; ++i) {
    in[i] = B2Atom{pos[i], pos[n + i], pos[2 * n + i], type[i], 0};
    int cx, cy, cz;
    cell[i] = b2_cell_of(box, g, in[i], &cx, &cy, &cz);
    order[i] = i;
  }
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return cell[a] < cell[b]; });
  std::vector<B2Atom> atoms(n);
  std::vector<int> cell_start(g.ncell + 1, 0);
  for (int i = 0; i < n; ++i) {
    atoms[i] = in[order[i]];
    ++cell_start[cell[order[i]] + 1];
  }
  for (int c = 0; c < g.ncell; ++c)
    cell_start[c + 1] += cell_start[c];
  int species[B2_MAX_TYPES];
  for (int t = 0; t < B2_MAX_TYPES; ++t)
    species[t] = -1;
  for (int a = 0; a < num_types; ++a)
    species[type_index[a]] = a;
  std::fill(u, u + (size_t)p.num_pairs * num_bins, 0ull);
  for (int i = 0; i < n; ++i)
    b2_body_rdf_atom(i, atoms.data(), cell_start.data(), box, g, p, species, [&](int k) { ++u[k]; });
  return g.ncell;
}

// one sample folded into acc[num_bins][1 + num_pairs] (u is zeroed, as on the device)
void rdf_emu_fold(double rc, int num_bins, int num_types, double volume, int n, const int* num_atoms,
                  unsigned long long* u, double* acc)
{
  const B2RdfPara p = make_para(rc, num_bins, num_types);
  for (int w = 0; w < num_bins; ++w)
    b2_body_rdf_fold(w, p, volume, n, num_atoms, u, acc);
}

double rdf_emu_volume(const double* h9)
{
  const int pbc[3] = {1, 1, 1};
  return make_box(h9, pbc).volume;
}

} // extern "C"

// tests/emu/rdf_emu.cpp -- TEST INFRASTRUCTURE ONLY: the RDF kernel bodies (gpumd_b200/csrc/b2_rdf.cuh)
// compiled for the host.  The cell sort is a serial restatement of the neighbour module's counting sort
// (ascending cell, then ascending atom index), the pair walk and the bin rule are the device's own
// b2_body_rdf_atom, and the fold is b2_body_rdf_fold.  The block-private tables, the warp-aggregated
// atomics and the flush are covered by the `-m gpu` tests only.
#include "../../gpumd_b200/csrc/b2_setup.h" // make_box, make_grid, rdf_para
#include <algorithm>
#include <cmath>
#include <vector>

using namespace b2;

extern "C" {

int rdf_emu_bin(double d2, double rc, int num_bins)
{
  return b2_rdf_bin(d2, rdf_para(rc, num_bins, 1));
}

// u[num_pairs][num_bins] of one sample; returns the number of cells, or -1 for a periodic direction
// with fewer than 5 of them
int rdf_emu_count(int n, const double* h9, const int* pbc, const int* type, const double* pos, double rc,
                  int num_bins, int num_types, const int* type_index, unsigned long long* u)
{
  const B2Box box = make_box(h9, pbc);
  const B2RdfPara p = rdf_para(rc, num_bins, num_types);
  const B2Grid g = make_grid(box, 0.5 * rc); // Neighbor::sort_cells
  if (grid_too_coarse(box, g))
    return -1;
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
  const B2RdfPara p = rdf_para(rc, num_bins, num_types);
  for (int w = 0; w < num_bins; ++w)
    b2_body_rdf_fold(w, p, volume, n, num_atoms, u, acc);
}

double rdf_emu_volume(const double* h9)
{
  const int pbc[3] = {1, 1, 1};
  return make_box(h9, pbc).volume;
}

} // extern "C"

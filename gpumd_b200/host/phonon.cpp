#include "phonon.h"
#include <algorithm>
#include <array>
#include <cmath>
#include <fstream>
#include <sstream>

namespace {

const double PI = 3.14159265358979; // src/utilities/common.cuh:20

std::vector<std::string> tokens_of(const std::string& line)
{
  std::istringstream ss(line);
  std::vector<std::string> t;
  std::string w;
  while (ss >> w)
    t.push_back(w);
  return t;
}

// get_double_from_token (src/utilities/error.cu:168-190): std::stod, which reads a leading number
double token_double(const std::string& s)
{
  double v = 0.0;
  try {
    v = std::stod(s);
  } catch (const std::exception& e) {
    printf("Standard exception:\n    Error message: %s\n", e.what());
    exit(1);
  }
  if (std::isinf(v) || std::isnan(v)) {
    printf("This number is %s.\n", std::isinf(v) ? "inf" : "nan");
    exit(1);
  }
  return v;
}

struct KPath {
  std::vector<double> kpoints, kpath, kpath_sym;
  std::vector<std::string> names; // one per segment, the point names joined by ' '
};

// Hessian::create_kpoints (hessian.cu:110-198)
KPath create_kpoints(const Box& box, const int cxyz[3])
{
  std::ifstream in("kpoints.in");
  if (!in.is_open())
    input_error("Cannot open kpoints.in file.");
  std::vector<std::vector<std::array<double, 3>>> hsps;
  std::vector<std::array<double, 3>> hsp;
  KPath kp;
  std::string line, k_names;
  while (std::getline(in, line)) {
    const auto t = tokens_of(line);
    if (t.empty()) { // a blank line closes a segment
      if (!hsp.empty()) {
        hsps.push_back(hsp);
        hsp.clear();
        kp.names.push_back(k_names);
        k_names.clear();
      }
      continue;
    }
    if (t[0][0] == '#')
      continue;
    if (t.size() < 4)
      input_error("kpoints.in file at least 4 parameters for each line.");
    hsp.push_back({token_double(t[0]), token_double(t[1]), token_double(t[2])});
    if (!k_names.empty())
      k_names += " ";
    k_names += t[3];
  }
  if (!hsp.empty()) {
    hsps.push_back(hsp);
    kp.names.push_back(k_names);
  }
  if (hsps.empty())
    input_error("kpoints.in has no k-point.");
  int nk = 1 - (int)hsps.size();
  for (const auto& s : hsps)
    nk += (int)s.size();
  nk = (nk - 1) * 100 + 1;
  double rec[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      rec[j][i] = 2.0 * PI * cxyz[i] * box.cpu_h[9 + i * 3 + j];
  auto mv = [&](const std::array<double, 3>& k) {
    return std::array<double, 3>{rec[0][0] * k[0] + rec[0][1] * k[1] + rec[0][2] * k[2],
                                 rec[1][0] * k[0] + rec[1][1] * k[1] + rec[1][2] * k[2],
                                 rec[2][0] * k[0] + rec[2][1] * k[1] + rec[2][2] * k[2]};
  };
  kp.kpoints.resize((size_t)3 * nk);
  kp.kpath.resize(nk);
  const auto k0 = mv(hsps[0][0]);
  for (int c = 0; c < 3; ++c)
    kp.kpoints[c] = k0[c];
  double len = 0.0;
  kp.kpath[0] = len;
  kp.kpath_sym.push_back(len);
  int idx = 1;
  for (const auto& s : hsps)
    for (size_t i = 1; i < s.size(); ++i) {
      const auto start = mv(s[i - 1]), end = mv(s[i]);
      auto last = start;
      for (int j = 1; j <= 100; ++j, ++idx) {
        std::array<double, 3> k;
        for (int c = 0; c < 3; ++c)
          k[c] = start[c] + j * 0.01 * (end[c] - start[c]);
        for (int c = 0; c < 3; ++c)
          kp.kpoints[(size_t)idx * 3 + c] = k[c];
        const double d0 = k[0] - last[0], d1 = k[1] - last[1], d2 = k[2] - last[2];
        len += std::sqrt(d0 * d0 + d1 * d1 + d2 * d2);
        kp.kpath[idx] = len;
        last = k;
        if (j == 100)
          kp.kpath_sym.push_back(len);
      }
    }
  return kp;
}

std::vector<double> read(b200md_phonon* p, int what, size_t count)
{
  std::vector<double> h(count);
  if (b200md_phonon_read(p, what, h.data(), nullptr) != B200MD_OK)
    b2h_fail("compute_phonon (copy to host)");
  return h;
}

} // namespace

void Hessian_B200::parse(const std::vector<std::string>& t)
{
  if (t.size() != 2)
    input_error("compute_phonon should have 2 parameters.");
  if (!valid_real(t[1], &displacement_))
    input_error("displacement for compute_phonon should be a number.");
  if (displacement_ <= 0)
    input_error("displacement for compute_phonon should be positive.");
  printf("displacement for compute_phonon = %g A.\n", displacement_);
}

void Hessian_B200::compute(Force& force, Box& box, Atom& atom, const int cxyz[3])
{
  // Hessian::initialize (hessian.cu:200-253)
  box.get_inverse(); // cpu_h[9..17], which the k-points are made from
  double cutoff = 0.0;
  for (const auto& p : force.potentials)
    cutoff = std::max(cutoff, p->rc);
  const double phonon_cutoff = cutoff * 2.0;
  printf("Using cutoff for phonon calculations: %g A.\n", phonon_cutoff);
  const int N = atom.number_of_atoms;
  int s_c[3] = {1, 1, 1}, pbc[3];
  b2h_pbc(box, pbc);
  const double volume = box.get_volume();
  for (int i = 0; i < 3; ++i) {
    // Box::get_area (src/model/box.cu:34-48): the face spanned by the other two lattice vectors
    const int p = (i + 1) % 3, q = (i + 2) % 3;
    const double* h = box.cpu_h;
    const double a[3] = {h[p], h[p + 3], h[p + 6]}, b[3] = {h[q], h[q + 3], h[q + 6]};
    const double s1 = a[1] * b[2] - a[2] * b[1], s2 = a[2] * b[0] - a[0] * b[2], s3 = a[0] * b[1] - a[1] * b[0];
    const double ori_thick = volume / std::sqrt(s1 * s1 + s2 * s2 + s3 * s3) / cxyz[i];
    if (pbc[i])
      for (int j = 1; j < 100; ++j)
        if (ori_thick * j >= cutoff * 4) {
          s_c[i] = j;
          break;
        }
  }
  printf("Suggested replicate size for phonon calculations:\n");
  printf("Replicate in x >= %d.\n", s_c[0]);
  printf("Replicate in y >= %d.\n", s_c[1]);
  printf("Replicate in z >= %d.\n", s_c[2]);
  const int num_basis = N / (cxyz[0] * cxyz[1] * cxyz[2]);
  if (num_basis > B200MD_PHONON_MAX_BASIS)
    input_error("compute_phonon supports at most 32 basis atoms (N / (cx * cy * cz) = " +
                std::to_string(num_basis) + ").");
  const KPath kp = create_kpoints(box, cxyz);
  const int nk = (int)kp.kpath.size(), dim = 3 * num_basis;

  b200md_phonon* ph = nullptr;
  if (b200md_phonon_create(N, num_basis, nk, kp.kpoints.data(), displacement_, &ph) != B200MD_OK)
    b2h_fail("compute_phonon (create)");
  if (b200md_phonon_begin(ph, N, box.cpu_h, pbc, phonon_cutoff, atom.position_per_atom.data(),
                          atom.mass.data(), nullptr) != B200MD_OK)
    b2h_fail("compute_phonon (begin)");
  for (int call = 0; call < 6 * num_basis; ++call) {
    force.compute(box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
                  atom.virial_per_atom);
    if (b200md_phonon_step(ph, call, atom.position_per_atom.data(), atom.force_per_atom.data(), nullptr) !=
        B200MD_OK)
      b2h_fail("compute_phonon (step)");
  }
  if (b200md_phonon_dynamical(ph, nullptr) != B200MD_OK || b200md_phonon_eig(ph, nullptr) != B200MD_OK)
    b2h_fail("compute_phonon (dynamical matrices / eigenvalues)");
  force.potentials[0]->check();
  const double natural_to_THz = 1.0e6 / (TIME_UNIT_CONVERSION * TIME_UNIT_CONVERSION);
  const size_t dd = (size_t)dim * dim;
  const std::vector<double> W = read(ph, B200MD_PHONON_W, (size_t)nk * dim);
  const std::vector<double> DR = read(ph, B200MD_PHONON_D_REAL, dd * nk);

  if (nk == 1) { // Hessian::find_eigenvectors (hessian.cu:460-492)
    const std::vector<double> V = read(ph, B200MD_PHONON_V, dd);
    b200md_phonon_destroy(ph);
    FILE* fid = fopen("eigenvector.out", "wb");
    for (int n = 0; n < dim; ++n) {
      const float om2 = (float)(W[n] * natural_to_THz);
      fwrite(&om2, sizeof(float), 1, fid);
    }
    for (int col = 0; col < dim; ++col)
      for (int a = 0; a < 3; ++a)
        for (int b = 0; b < num_basis; ++b) {
          const float e = (float)V[a + b * 3 + (size_t)col * dim];
          fwrite(&e, sizeof(float), 1, fid);
        }
    fclose(fid);
    return;
  }
  const std::vector<double> DI = read(ph, B200MD_PHONON_D_IMAG, dd * nk);
  b200md_phonon_destroy(ph);
  // Hessian::find_dispersion / output_D / find_omega(_batch) (hessian.cu:325-429)
  FILE* fid = fopen("omega2.out", "w");
  fprintf(fid, "#");
  for (double s : kp.kpath_sym)
    fprintf(fid, " %.6f", s);
  fprintf(fid, " ");
  for (size_t i = 0; i < kp.names.size(); ++i) {
    if (i > 0)
      fprintf(fid, "|");
    fprintf(fid, "%s", kp.names[i].c_str());
  }
  fprintf(fid, "\n");
  for (int k = 0; k < nk; ++k) {
    fprintf(fid, "%.6f ", kp.kpath[k]);
    for (int n = 0; n < dim; ++n)
      fprintf(fid, "%g ", W[(size_t)k * dim + n] * natural_to_THz);
    fprintf(fid, "\n");
  }
  fclose(fid);
  fid = fopen("D.out", "w");
  for (int k = 0; k < nk; ++k) {
    const size_t off = (size_t)k * dd;
    for (int r = 0; r < dim; ++r) {
      for (int c = 0; c < dim; ++c)
        fprintf(fid, "%g ", DR[off + r + (size_t)c * dim]);
      for (int c = 0; c < dim; ++c)
        fprintf(fid, "%g ", DI[off + r + (size_t)c * dim]);
      fprintf(fid, "\n");
    }
  }
  fclose(fid);
}

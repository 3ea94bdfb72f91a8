// b2_setup.h -- every decision libb200md makes on the host before its first launch: the box, the cell grid and
// the small-box rules, the potential files of LJ / Tersoff / EAM with their skin-list capacities, the RDF
// parameters, and the NEP kernel-path plan.  Header-only and free of the CUDA runtime, so that the CPU test
// build of the kernel bodies (tests/emu) runs this very code: it compiles under nvcc and g++ -std=c++17.
#pragma once
#include "b2_common.cuh"
#include "b2_eam.cuh"
#include "b2_nep.cuh"
#include "b2_nep_model.h"
#include "b2_rdf.cuh"
#include "b2_tersoff.cuh"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace b2 {

// Box::get_inverse / get_volume / thickness / set_is_orthogonal (src/model/box.cu:26-117)
inline B2Box make_box(const double h[9], const int pbc[3])
{
  B2Box b;
  double* c = b.h;
  for (int d = 0; d < 9; ++d)
    c[d] = h[d];
  for (int d = 0; d < 3; ++d)
    b.pbc[d] = pbc[d] ? 1 : 0;
  // adjugate / determinant
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
    // area of the face spanned by the other two lattice vectors (columns of h)
    const int p = (d + 1) % 3, q = (d + 2) % 3;
    const double u[3] = {c[p], c[p + 3], c[p + 6]}, w[3] = {c[q], c[q + 3], c[q + 6]};
    const double s0 = u[1] * w[2] - u[2] * w[1], s1 = u[2] * w[0] - u[0] * w[2],
                 s2 = u[0] * w[1] - u[1] * w[0];
    b.thickness[d] = b.volume / std::sqrt(s0 * s0 + s1 * s1 + s2 * s2);
  }
  b.ortho = c[1] == 0 && c[2] == 0 && c[3] == 0 && c[5] == 0 && c[6] == 0 && c[7] == 0;
  for (int d = 0; d < 18; ++d)
    b.hf[d] = (float)c[d];
  return b;
}

inline B2Grid make_grid(const B2Box& box, double cell_size)
{
  B2Grid g;
  for (int d = 0; d < 3; ++d) {
    int nb = (int)std::floor(box.thickness[d] / cell_size);
    if (nb < 1)
      nb = 1;
    g.nb[d] = nb;
    g.scale[d] = (double)nb;
  }
  g.ncell = g.nb[0] * g.nb[1] * g.nb[2];
  return g;
}

// the cell scans need at least 5 cells in every periodic direction
inline bool grid_too_coarse(const B2Box& box, const B2Grid& g)
{
  for (int d = 0; d < 3; ++d)
    if (box.pbc[d] && g.nb[d] < 5)
      return true;
  return false;
}

// Replica counts of the smallest supercell whose periodic thicknesses all exceed 2.5 (rc + skin), the
// thinnest box the skin list accepts (five cells of (rc + skin) / 2); returns their product (1: the box itself)
inline long long supercell_reps(const B2Box& box, double rc, double skin, int reps[3])
{
  const double need = 2.5 * (rc + skin);
  for (int d = 0; d < 3; ++d)
    reps[d] = box.pbc[d] && box.thickness[d] <= need ? (int)std::floor(need / box.thickness[d]) + 1 : 1;
  return (long long)reps[0] * reps[1] * reps[2];
}

// B200MD_TIGHT_LISTS=1: size the LJ / EAM skin lists by density instead of the reference's 700 / 400
inline bool tight_lists()
{
  const char* e = std::getenv("B200MD_TIGHT_LISTS");
  return e && e[0] == '1';
}

// neighbor.initialize(rc, N, k): k ((rc + skin) / rc)^3 skin entries per atom (neighbor.cu:824-829).  With
// tight_density > 0 and B200MD_TIGHT_LISTS=1, at most what a sphere of rc + skin holds at that many atoms per
// A^3, plus 32 (a memory knob for very large systems; an overflow is still latched and reported).
inline int skin_capacity(double rc, int k, double tight_density)
{
  const double rs = rc + 1.0;
  const int mn = (int)(k * rs * rs * rs / (rc * rc * rc));
  const int mn_dense = (int)(4.19 * rs * rs * rs * tight_density) + 32;
  return tight_density > 0 && tight_lists() && mn > mn_dense ? mn_dense : mn;
}

using File = std::unique_ptr<FILE, int (*)(FILE*)>;

inline File open_file(const char* path) { return File(std::fopen(path, "r"), std::fclose); }

// "<keyword> <count>" and then <count> symbols; false on a read error
inline bool read_header(FILE* f, char (&name)[64], int& nt)
{
  return std::fscanf(f, "%63s%d", name, &nt) == 2;
}

inline bool read_symbols(FILE* f, int nt, std::vector<std::string>& symbols)
{
  char name[64];
  for (int k = 0; k < nt; ++k) {
    if (std::fscanf(f, "%63s", name) != 1)
      return false;
    symbols.push_back(name);
  }
  return true;
}

// ---- LJ: "lj Nt sym..." then Nt*Nt lines "epsilon sigma cutoff" (force.cu:93-100, lj.cu:28-56) ----
struct LjFile {
  int nt = 0;
  std::vector<std::string> symbols;
  std::vector<float> s6e4, s12e4, rc2; // [nt*nt]
  double rc = 0.0;
  int mn_skin = 0;
};

// returns an empty string on success, else the error message
inline std::string load_lj(const char* path, LjFile& out)
{
  File f = open_file(path);
  if (!f)
    return std::string("Failed to open ") + path;
  char name[64];
  int& nt = out.nt;
  if (!read_header(f.get(), name, nt) || std::strcmp(name, "lj") != 0 || nt < 1 || nt > 10)
    return "Incorrect number of LJ parameters.";
  if (!read_symbols(f.get(), nt, out.symbols))
    return "Reading error for LJ potential.";
  for (int a = 0; a < nt * nt; ++a) {
    double eps, sig, cut;
    if (std::fscanf(f.get(), "%lf%lf%lf", &eps, &sig, &cut) != 3)
      return "Reading error for LJ potential.";
    out.s6e4.push_back((float)(std::pow(sig, 6.0) * eps * 4.0));
    out.s12e4.push_back((float)(std::pow(sig, 12.0) * eps * 4.0));
    out.rc2.push_back((float)(cut * cut));
    if (out.rc < cut)
      out.rc = cut;
  }
  out.mn_skin = skin_capacity(out.rc, 700, 0.06); // lj.cu:58; twice liquid-argon density
  return "";
}

// ---- Tersoff-1989: "tersoff_1989 <1|2> sym..." then 11 parameters per type (+ chi for two types) ----
struct TersoffFile {
  int nt = 0;
  std::vector<std::string> symbols;
  B2TersoffView view; // p[3] and rc2; the pointers are the caller's
  double rc = 0.0;
  int mn_skin = 0;
};

inline void tersoff_fill(B2TersoffPara& t, const double* p)
{
  t.a = p[0];
  t.b = p[1];
  t.lambda = p[2];
  t.mu = p[3];
  t.beta = p[4];
  t.n = p[5];
  t.c2 = p[6] * p[6];
  t.d2 = p[7] * p[7];
  t.h = p[8];
  t.r1 = p[9];
  t.r2 = p[10];
  t.one_plus = 1.0 + t.c2 / t.d2;
  t.pi_factor = 3.14159265358979 / (t.r2 - t.r1); // PI, src/utilities/common.cuh:19
  t.mhn = -0.5 / p[5];
}

inline std::string load_tersoff(const char* path, TersoffFile& out)
{
  File f = open_file(path);
  if (!f)
    return std::string("Failed to open ") + path;
  char name[64];
  int& nt = out.nt;
  if (!read_header(f.get(), name, nt) || std::strcmp(name, "tersoff_1989") != 0 || nt < 1 || nt > 2)
    return "tersoff_1989 potential file: first line must be 'tersoff_1989 <1|2> <symbols>'";
  if (!read_symbols(f.get(), nt, out.symbols))
    return "Reading error for Tersoff-1989 potential.";
  double para[23] = {0};
  for (int k = 0; k < (nt == 1 ? 11 : 23); ++k)
    if (std::fscanf(f.get(), "%lf", &para[k]) != 1)
      return "Reading error for Tersoff-1989 potential.";
  B2TersoffView& P = out.view;
  std::memset(&P, 0, sizeof P);
  tersoff_fill(P.p[0], para);
  out.rc = P.p[0].r2;
  if (nt == 2) { // mixing rules, tersoff1989.cu:100-130
    tersoff_fill(P.p[1], para + 11);
    const double chi = para[22];
    B2TersoffPara& m = P.p[2];
    m.a = std::sqrt(P.p[0].a * P.p[1].a);
    m.b = std::sqrt(P.p[0].b * P.p[1].b) * chi;
    m.lambda = 0.5 * (P.p[0].lambda + P.p[1].lambda);
    m.mu = 0.5 * (P.p[0].mu + P.p[1].mu);
    m.r1 = std::sqrt(P.p[0].r1 * P.p[1].r1);
    m.r2 = std::sqrt(P.p[0].r2 * P.p[1].r2);
    m.pi_factor = 3.14159265358979 / (m.r2 - m.r1);
    out.rc = P.p[0].r2 > P.p[1].r2 ? P.p[0].r2 : P.p[1].r2;
  } else {
    P.p[1] = P.p[0];
    P.p[2] = P.p[0];
  }
  P.rc2 = (float)(out.rc * out.rc);
  out.mn_skin = skin_capacity(out.rc, 50, 0.0); // tersoff1989.cu:149
  return "";
}

// ---- EAM: "eam_zhou_2004 <1..18> sym..." + 21 parameters per type, or "eam_dai_2006 1 sym" + 9 ----
struct EamFile {
  int nt = 0;
  std::vector<std::string> symbols;
  B2EamView view;        // model, nt, rc and the Dai-2006 scalars; the pointers are the caller's
  std::vector<float> zp; // Zhou-2004: [nt][EZ_COUNT]
  float rc = 0.0f;
  int mn_skin = 0;
};

inline std::string load_eam(const char* path, EamFile& out)
{
  File f = open_file(path);
  if (!f)
    return std::string("Failed to open ") + path;
  char name[64];
  int& nt = out.nt;
  if (!read_header(f.get(), name, nt))
    return "Reading error for EAM potential.";
  const int model = std::strcmp(name, "eam_zhou_2004") == 0 ? 0 : std::strcmp(name, "eam_dai_2006") == 0 ? 1 : -1;
  if (model < 0 || nt < 1 || nt > 18 || (model == 1 && nt != 1))
    return "EAM potential file: expected 'eam_zhou_2004 <1..18> ...' or 'eam_dai_2006 1 ...'";
  if (!read_symbols(f.get(), nt, out.symbols))
    return "Reading error for EAM potential.";
  B2EamView& P = out.view;
  std::memset(&P, 0, sizeof P);
  out.zp.assign((size_t)nt * EZ_COUNT, 0.0f);
  float& rc = out.rc;
  float x[21];
  auto read = [&](int count) {
    for (int k = 0; k < count; ++k)
      if (std::fscanf(f.get(), "%f", &x[k]) != 1)
        return false;
    return true;
  };
  if (model == 1) { // eam.cu:94-122
    if (!read(9))
      return "Reading error for EAM potential.";
    P.dA = x[0];
    P.dd = x[1];
    P.dc = x[2];
    P.dc0 = x[3];
    P.dc1 = x[4];
    P.dc2 = x[5];
    P.dc3 = x[6];
    P.dc4 = x[7];
    P.dB = x[8];
    rc = P.dc > P.dd ? P.dc : P.dd;
  }
  for (int t = 0; model == 0 && t < nt; ++t) { // eam.cu:46-92
    if (!read(21))
      return "Reading error for EAM potential.";
    float* e = &out.zp[(size_t)t * EZ_COUNT];
    e[EZ_RE_INV] = 1.0f / x[0];
    e[EZ_FE] = x[1];
    e[EZ_RHO_E_INV] = 1.0f / x[2];
    e[EZ_RHO_S_INV] = 1.0f / x[3];
    e[EZ_ALPHA] = x[4];
    e[EZ_BETA] = x[5];
    e[EZ_A] = x[6];
    e[EZ_B] = x[7];
    e[EZ_KAPPA] = x[8];
    e[EZ_LAMBDA] = x[9];
    e[EZ_FN0] = x[10];
    e[EZ_FN1] = x[11];
    e[EZ_FN2] = x[12];
    e[EZ_FN3] = x[13];
    e[EZ_F0] = x[14];
    e[EZ_F1] = x[15];
    e[EZ_F2] = x[16];
    e[EZ_F3] = x[17];
    e[EZ_ETA] = x[18];
    e[EZ_FE_EMBED] = x[19];
    e[EZ_RC] = x[20];
    e[EZ_RHO_N] = x[2] * 0.85;
    e[EZ_RHO_0] = x[2] * 1.15;
    e[EZ_RHO_N_INV] = 1.0f / e[EZ_RHO_N];
    if (rc < x[20])
      rc = x[20];
  }
  P.model = model;
  P.nt = nt;
  P.rc = rc;
  // eam.cu:43 ("very safe for EAM"); twice fcc-metal density
  out.mn_skin = skin_capacity(rc, 400, 0.2);
  return "";
}

// ---- RDF (rdf.cu:325-326) ----
inline B2RdfPara rdf_para(double rc, int num_bins, int num_types)
{
  B2RdfPara p;
  p.num_bins = num_bins;
  p.num_types = num_types;
  p.num_pairs = num_types * (num_types + 1) / 2;
  p.dr = rc / num_bins;
  p.rc2 = rc * rc;
  return p;
}

// ---- NEP ----
constexpr int NEP_BLK = 128; // threads per block of the thread-per-atom NEP kernels
// k_angular_fused runs for models with a zero-padded descriptor of 32 (the width whose instances ptxas
// compiles without spills at three blocks per SM; at 48 every instance spills) and where two of its
// blocks fit an SM's 228 KB of shared memory (1 KB reserved per block)
constexpr int FUSED_DIMP = 32;
constexpr size_t FUSED_MAX_SMEM = 113 * 1024;
// Angular shapes k_angular_fused is compiled for (B2AngShape): NEP4's default n_max = 4 4 with l_max = 4 2 0
// (dim 30) and 4 0 0 (dim 25).  Each shape adds 12 instances (NT x K1 x ORTHO, about 15 s of build time);
// every other shape within the budget runs the run-time-shape instance.
enum { FUSED_SHAPE_NONE, FUSED_SHAPE_RT, FUSED_SHAPE_4B, FUSED_SHAPE_3B };

inline int fused_shape_of(const NepModel& m)
{
  if (m.nr1 == 5 && m.na1 == 5 && !m.has1111)
    return m.has222 ? FUSED_SHAPE_4B : FUSED_SHAPE_3B;
  return FUSED_SHAPE_RT;
}

// The kernel paths, switches and budgets of one NEP model at one atom count (nep_plan)
struct NepPlan {
  int mn_skin = 0;          // skin-list capacity per atom
  int pitch_r = 0;          // row pitch of the radial list (lane teams)
  bool team = false;        // lane-team radial kernels (<= 2 types, B200MD_NEP_TEAM=1)
  bool fuse_split = false;  // many-type path: neighbour split inside the radial descriptor pass
  bool radial_v2 = false;   // few-type radial passes of b2_nep_radial.cuh (planes, branch-free loop)
  bool sched = false;       // their warps follow Neighbor::seg_order (B200MD_NEP_SCHED=0: identity, A/B runs)
  bool ang_fused = false;   // k_angular_fused instead of k_desc_angular2 + hidden layer + k_force_angular2
  int fused_shape = FUSED_SHAPE_NONE; // its instance (b200md_nep_info 10)
  size_t fused_smem = 0;    // its dynamic shared memory per block
  bool use_tc = false;      // hidden layer on the tensor cores (k_mlp_tc) instead of k_mlp
  bool utable_tc = false;   // the U table as k_mlp_tc's third GEMM (else k_utable)
  bool rev_slot = false;    // direct reverse slots for the angular pair reduction (B200MD_NEP_REVSLOT=1)
  bool slot_map = false;    // k_force_final2: thread per tile slot (type-pure warps); measured slower
                            // (H100, 1 M-atom PbTe: 1.26 vs 1.02 ms), B200MD_NEP_SLOTMAP=1 for A/B runs
  bool rad_reg = false;     // 3..16 types: radial accumulators in registers (k_desc_radial<4|8|16,...>); slower
                            // than the shared-memory accumulators on UNEP-v1, B200MD_NEP_RADREG=1
  bool rad_direct = false;  // many types: contract every pair on the spot (k_desc_radial<-1,...>)
  int rad_nt = 0;           // 3+ types: NT of the k_desc_radial instance (-1, 0, 4, 8, 16)
  bool c_r4 = true;         // padded radial coefficient rows (B2NepView::c_r4)
  bool ang_cstage = true;   // k_desc_angular: coefficient table staged in shared memory
  int variant = 0;          // B200MD_NEP_VARIANT: kernel tuning variants for A/B measurements
  int tc_ctas_cap = 0;      // B200MD_NEP_TC_CTAS: at most this many CTAs of k_mlp_tc (0: as many as fit)
  int debug_skip = 0;       // B200MD_DEBUG_SKIP (B2NepView::debug_skip)
  int ang_block = NEP_BLK;  // threads per block of the angular force kernel
  size_t ang_smem = 0, rad_smem = 0; // dynamic shared memory of the angular force / radial descriptor kernels
};

// The one place the B200MD_NEP_* and B200MD_DEBUG_SKIP switches are read.  Returns an empty string on
// success, else the error message.
inline std::string nep_plan(const NepModel& m, int num_atoms, NepPlan& p)
{
  p = NepPlan();
  const char* e;
  const double rc = m.rc_radial_max, rs = rc + 1.0;
  p.mn_skin = skin_capacity(rc, m.MN_radial, 0.0);
  p.pitch_r = (m.MN_radial + 7) / 8 * 8;
  // radial passes: thread per atom by default.  B200MD_NEP_TEAM=1 selects the lane-team kernels for one- and
  // two-type models: they cut the L1 gather wavefronts ~3x but cost ~30% more instructions and are slower.
  e = std::getenv("B200MD_NEP_TEAM");
  p.team = m.nt <= 2 && e && std::strcmp(e, "1") == 0;
  if ((e = std::getenv("B200MD_NEP_VARIANT")))
    p.variant = std::atoi(e);
  // fused split pays when few skin candidates fail the radial test: (rc+skin)^3 / rc^3 small
  p.fuse_split = rs * rs * rs / (rc * rc * rc) < 1.45;
  // one- and two-type models: the plane-based radial kernels (B200MD_NEP_RADIAL=v1 keeps the round-1 kernels
  // for A/B runs)
  e = std::getenv("B200MD_NEP_RADIAL");
  p.radial_v2 = m.nt <= 2 && !p.team && !(e && std::strcmp(e, "v1") == 0) &&
                (double)num_atoms * (p.mn_skin + 2) < 4.0e9; // 32-bit list offsets in those kernels
  if ((e = std::getenv("B200MD_NEP_SLOTMAP")))
    p.slot_map = std::atoi(e) != 0;
  if ((e = std::getenv("B200MD_NEP_RADREG")))
    p.rad_reg = std::atoi(e) != 0;
  if ((e = std::getenv("B200MD_NEP_CSTAGE")))
    p.ang_cstage = std::atoi(e) != 0;
  // Hidden layer and angular stages.  B200MD_NEP_MLP unset: k_angular_fused where the model fits its budget
  // (FUSED_DIMP, FUSED_MAX_SMEM; DESIGN.md 3.2); then the SIMT layer is also the hidden layer of the generic
  // kernels (B200MD_NEP_RADIAL=v1), which keeps the two paths bit-identical.  Otherwise the tensor cores
  // unless the shapes do not fit them.  B200MD_NEP_MLP=simt / =tc select the SIMT / the tensor-core layer
  // between separate angular kernels.
  const char* mlp = std::getenv("B200MD_NEP_MLP");
  p.fused_smem = b2_fused_smem_bytes(m.nt, m.na1, m.K1A, m.nneu, m.DIMP);
  const bool fused_fits = m.nt <= 2 && !mlp && m.DIMP == FUSED_DIMP && p.fused_smem <= FUSED_MAX_SMEM;
  p.ang_fused = fused_fits && p.radial_v2;
  p.fused_shape = p.ang_fused ? fused_shape_of(m) : FUSED_SHAPE_NONE;
  p.use_tc = m.tc_ok && !(mlp && std::strcmp(mlp, "simt") == 0) && !fused_fits;
  e = std::getenv("B200MD_NEP_UTABLE");
  p.utable_tc = p.use_tc && m.tc3_ok && !(e && std::strcmp(e, "simt") == 0);
  if ((e = std::getenv("B200MD_NEP_TC_CTAS"))) // tests: persistent CTAs that each walk many tiles
    p.tc_ctas_cap = std::atoi(e) > 0 ? std::atoi(e) : 0;
  e = std::getenv("B200MD_NEP_SCHED");
  p.sched = p.radial_v2 && !(e && e[0] == '0');
  // B200MD_NEP_REVSLOT=1 (many types with the neighbour split as its own kernel): direct reverse slots for the
  // angular pair reduction instead of a binary search per pair: k_force_final gets faster on UNEP-v1, but the
  // extra stores slow k_split down by more, so it stays an opt-in.
  e = std::getenv("B200MD_NEP_REVSLOT");
  p.rev_slot = m.nt > 2 && !p.team && !p.fuse_split && e && e[0] == '1';
  // B200MD_NEP_CVEC=0: scalar coefficient loads in the radial contraction (A/B switch; results are
  // bit-identical).  The angular kernels always use the padded rows.
  e = std::getenv("B200MD_NEP_CVEC");
  p.c_r4 = !(e && e[0] == '0');
  if ((e = std::getenv("B200MD_DEBUG_SKIP")))
    p.debug_skip = std::atoi(e);

  // shared-memory budgets (k_force_angular2: one padded row of b2_ang_ws4(na1) float4s per thread)
  const size_t ang_row = p.radial_v2 ? b2_ang_ws4(m.na1) * sizeof(float4) : m.na1 * B2_NABC * sizeof(float);
  p.ang_smem = ang_row * p.ang_block;
  while (p.ang_smem > 200 * 1024 && p.ang_block > 32) {
    p.ang_block /= 2;
    p.ang_smem = ang_row * p.ang_block;
  }
  // Radial descriptor of a many-type model: per-type accumulators in shared memory while two blocks of them
  // fit an SM, else (NEP89: 89 species) the per-pair contraction, which needs no such storage.
  // B200MD_NEP_RADDIRECT=1 forces the latter for any model with more than two types (tests, A/B).
  p.rad_smem = (size_t)m.nt * m.K1R * NEP_BLK * sizeof(float);
  if (m.nt > 2) {
    e = std::getenv("B200MD_NEP_RADDIRECT");
    if ((e && e[0] == '1') || p.rad_smem > 96 * 1024) {
      if (m.nqr > B2_NQMAX)
        return "n_max_radial above 19 is not supported for models with this many atom types";
      p.rad_direct = true;
      p.rad_smem = 0;
      p.c_r4 = true; // regardless of B200MD_NEP_CVEC
    }
  }
  // 3..16 types: register accumulators (B200MD_NEP_RADREG=1) when NT*K1 fits the register file; the default
  // keeps the accumulators in shared memory
  const int nt = m.nt;
  const int ntb = !p.rad_reg ? 0 : nt <= 4 ? 4 : nt <= 8 ? 8 : nt <= 16 ? 16 : 0;
  p.rad_nt = p.rad_direct ? -1 : ntb * m.K1R <= 160 ? ntb : 0;
  return "";
}

// A view holding the model's scalars and the plan's, every pointer null (the caller points them at its tables
// and buffers)
inline B2NepView nep_view(const NepModel& m, const NepPlan& plan, int num_atoms)
{
  B2NepView P;
  std::memset(&P, 0, sizeof P);
  P.nt = m.nt;
  P.nr1 = m.nr1;
  P.na1 = m.na1;
  P.kr1 = m.kr1;
  P.ka1 = m.ka1;
  P.K1R = m.K1R;
  P.K1A = m.K1A;
  P.KP = m.KP;
  P.UST = m.UST;
  P.has222 = m.has222;
  P.has1111 = m.has1111;
  P.num_L = m.num_L;
  P.dim = m.dim;
  P.dim_ang = m.dim_angular;
  P.nneu = m.nneu;
  P.DIMP = m.DIMP;
  P.zbl_enabled = m.zbl_enabled;
  P.zbl_flexible = m.zbl_flexible;
  P.zbl_typewise = m.zbl_typewise;
  P.zbl_rc_inner = m.zbl_rc_inner;
  P.zbl_rc_outer = m.zbl_rc_outer;
  P.zbl_typewise_factor = m.zbl_typewise_factor;
  P.nqr = m.nqr;
  P.debug_skip = plan.debug_skip;
  P.n = num_atoms;
  P.mn_r = m.MN_radial;
  P.mn_a = m.MN_angular;
  P.team = plan.team ? 1 : 0;
  P.pitch_r = plan.pitch_r;
  return P;
}

} // namespace b2

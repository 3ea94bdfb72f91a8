// tests/emu/emu.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Compiles the kernel BODIES of libb200md (gpumd_b200/csrc/*.cuh) for the host and drives them
// with plain loops, so the arithmetic and the list logic can be checked against the oracle in
// the GPU-less build container (`pytest -m "not gpu"`).  Nothing here is part of the product:
// libb200md.so never links or loads this file, and this library is never used by bench.py,
// __graft_entry__.py or the gpumd_b200 package.  The block-cooperative pieces of the real kernels
// (scan, shared-memory tile sort, atomics, warp reductions) are replaced by serial loops here
// and are therefore covered only by the `-m gpu` tests.
#include "../../gpumd_b200/csrc/b2_bdp.cuh"
#include "../../gpumd_b200/csrc/b2_integrate.cuh"
#include "../../gpumd_b200/csrc/b2_lj.cuh"
#include "../../gpumd_b200/csrc/b2_neighbor.cuh"
#include "../../gpumd_b200/csrc/b2_setup.h" // the library's own host setup
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

using namespace b2;

namespace {

struct EmuNeighbor {
  int n = 0, mn_skin = 0;
  double rc = 0, skin = 1.0;
  std::vector<B2Atom> atoms, atoms_tmp;
  std::vector<double> snap;
  std::vector<int> snap_type, perm, perm_tmp, cell_of, order_tmp, cell_count, cell_fill, cell_start, nn_skin,
    nl_skin, flags, rskin;
  bool reverse = false; // mirrors Neighbor::enable_reverse
  B2NeighborView v;
  int rebuilds = 0;
  bool row_major = false; // mirrors Neighbor::skin_row_major
  int pitch() const { return (mn_skin + 7) / 8 * 8; }

  void init(int n_, double rc_, int mn)
  {
    n = n_;
    rc = rc_;
    mn_skin = mn;
    atoms.resize(n);
    atoms_tmp.resize(n);
    snap.assign((size_t)3 * n, 0.0);
    snap_type.assign(n, 0);
    perm.resize(n);
    for (int i = 0; i < n; ++i)
      perm[i] = i;
    perm_tmp.resize(n);
    cell_of.resize(n);
    order_tmp.resize(n);
    nn_skin.resize(n);
    nl_skin.resize((size_t)pitch() * n);
    if (reverse)
      rskin.assign((size_t)pitch() * n, 0);
    flags.assign(4, 0);
    flags[0] = 1;
  }
  int update(const B2Box& box, const int* type, const double* pos)
  {
    int reps[3];
    const B2Grid g = make_grid(box, 0.5 * (rc + skin));
    if (supercell_reps(box, rc, skin, reps) > 1 || grid_too_coarse(box, g))
      return 4; // B200MD_ERR_SMALL_BOX, Neighbor::update
    cell_count.assign(g.ncell, 0);
    cell_fill.assign(g.ncell, 0);
    cell_start.assign(g.ncell + 1, 0);
    v.n = n;
    v.mn_skin = mn_skin;
    v.atoms = atoms.data();
    v.atoms_tmp = atoms_tmp.data();
    v.snap = snap.data();
    v.snap_type = snap_type.data();
    v.perm = perm.data();
    v.perm_tmp = perm_tmp.data();
    v.cell_of = cell_of.data();
    v.order_tmp = order_tmp.data();
    v.cell_count = cell_count.data();
    v.cell_fill = cell_fill.data();
    v.cell_start = cell_start.data();
    v.nn_skin = nn_skin.data();
    v.nl_skin = nl_skin.data();
    v.rskin = reverse ? rskin.data() : nullptr;
    v.skin_si = row_major ? (size_t)pitch() : 1;
    v.skin_sk = row_major ? 1 : (size_t)n;
    v.flags = flags.data();
    const float trigger = (float)(skin * skin * 0.25);
    const float cutoff = (float)((rc + skin) * (rc + skin));
    for (int i = 0; i < n; ++i)
      b2_body_pack_check(i, v, box, type, pos, pos + n, pos + 2 * (size_t)n, trigger);
    if (flags[0]) {
      for (int i = 0; i < n; ++i) {
        int cx, cy, cz;
        const int c = b2_cell_of(box, g, atoms[i], &cx, &cy, &cz);
        cell_of[i] = c;
        cell_count[c]++;
      }
      int run = 0;
      for (int c = 0; c < g.ncell; ++c) {
        cell_start[c] = run;
        run += cell_count[c];
      }
      cell_start[g.ncell] = run;
      for (int i = n - 1; i >= 0; --i) { // deliberately NOT ascending: mimics unordered atomics
        const int c = cell_of[i];
        order_tmp[cell_start[c] + cell_fill[c]++] = i;
      }
      for (int c = 0; c < g.ncell; ++c)
        b2_body_sort_cell(c, v);
      for (int i = 0; i < n; ++i)
        b2_body_commit(i, v);
      for (int i = 0; i < n; ++i)
        b2_body_skin_list(i, v, box, g, cutoff);
      if (reverse)
        for (int i = 0; i < n; ++i)
          b2_body_skin_reverse(i, v);
      flags[0] = 0;
      flags[2]++;
    }
    return 0;
  }
};

std::string g_err;

} // namespace

struct emu_nep {
  NepModel m;
  EmuNeighbor nb;
  int n = 0;
  std::vector<int> nn_r, nl_r, nn_a, nl_a;
  std::vector<float> q, sfx, FpR, FpA, U, f12;
  std::vector<double> acc;
  std::vector<int> zbl_z;
  std::vector<float> cov;
  B2NepView P;
  NepPlan plan;
  std::vector<int> aslot, nla_rs;
  int n_cell = 0;                        // atoms of the caller's cell (n > n_cell: supercell)
  int overwrite = 0, n_own = 0;          // b200md_nep_set_accumulate(p, 0) / set_owned requests
};

template <int K1>
static void run_desc_radial(emu_nep* p, const B2Box& box)
{
  std::vector<float> scratch((size_t)p->m.nt * K1 + 1);
  if (!p->plan.team && p->m.nt > 2 && !p->plan.fuse_split)
    for (int i = 0; i < p->n; ++i)
      b2_body_split(i, p->P, box);
  for (int i = 0; i < p->n; ++i) {
    if (p->plan.team && p->m.nt == 1)
      b2_team_desc_radial<1, K1>(i, 0, p->P, box);
    else if (p->plan.team)
      b2_team_desc_radial<2, K1>(i, 0, p->P, box);
    else if (p->m.nt == 1)
      b2_body_desc_radial<1, K1, true>(i, p->P, box, scratch.data(), 1, 0);
    else if (p->m.nt == 2)
      b2_body_desc_radial<2, K1, true>(i, p->P, box, scratch.data(), 1, 0);
    else {
      const int ntb = p->plan.rad_nt; // the k_desc_radial instance of dispatch_desc_radial
#define EMU_DR(NT_)                                                                         \
  do {                                                                                      \
    if (p->plan.fuse_split)                                                                 \
      b2_body_desc_radial<NT_, K1, true>(i, p->P, box, scratch.data(), 1, 0);               \
    else                                                                                    \
      b2_body_desc_radial<NT_, K1, false>(i, p->P, box, scratch.data(), 1, 0);              \
  } while (0)
      if (ntb == -1)
        EMU_DR(-1);
      else if (ntb == 4)
        EMU_DR(4);
      else if (ntb == 8)
        EMU_DR(8);
      else if (ntb == 16)
        EMU_DR(16);
      else
        EMU_DR(0);
#undef EMU_DR
    }
  }
}
template <int K1>
static void run_force_final(emu_nep* p, const B2Box& box, double* pe, double* f, double* v)
{
  for (int i = 0; i < p->n; ++i) {
    if (p->plan.team && p->m.nt == 1)
      b2_team_force_final<1, K1>(i, 0, p->P, box, pe, f, v);
    else if (p->plan.team)
      b2_team_force_final<2, K1>(i, 0, p->P, box, pe, f, v);
    else if (p->m.nt == 1)
      b2_body_force_final<1, K1>(i, p->P, box, pe, f, v);
    else if (p->m.nt == 2)
      b2_body_force_final<2, K1>(i, p->P, box, pe, f, v);
    else
      b2_body_force_final<0, K1>(i, p->P, box, pe, f, v);
  }
}
template <int K1>
static void run_angular(emu_nep* p, const B2Box& box, bool force)
{
  std::vector<float> w((size_t)p->m.na1 * B2_NABC + 1);
  for (int i = 0; i < p->n; ++i) {
    if (force)
      b2_body_force_angular<K1, 1>(i, p->P, box, w.data(), 0, p->P.c_a4, p->P.na1 * ((K1 + 3) / 4));
    else
      b2_body_desc_angular<K1, 5>(i, p->P, box, p->P.c_a4, p->P.na1 * ((K1 + 3) / 4));
  }
}
template <int DIMP>
static void run_mlp(emu_nep* p)
{
  for (int i = 0; i < p->n; ++i)
    b2_body_mlp<DIMP, true>(i, p->P, p->P.w0p, p->P.b0, p->P.w1);
}

extern "C" {

const char* emu_last_error(void) { return g_err.c_str(); }

// plan, (re)size every per-atom buffer for n atoms and point the view at them (nep_setup's host twin);
// returns the plan's error
static std::string emu_nep_alloc(emu_nep* p, int n)
{
  NepModel& m = p->m;
  const std::string err = nep_plan(m, n, p->plan);
  if (!err.empty())
    return err;
  const NepPlan& plan = p->plan;
  p->n = n;
  const size_t N = n;
  p->nb.row_major = plan.team;
  p->nb.reverse = plan.rev_slot;
  p->nb.init(n, m.rc_radial_max, plan.mn_skin);
  if (plan.rev_slot) {
    p->aslot.assign((size_t)p->nb.pitch() * n, -1);
    p->nla_rs.assign(N * m.MN_angular, 0);
  }
  p->nn_r.resize(N);
  p->nl_r.resize(N * plan.pitch_r);
  p->nn_a.resize(N);
  p->nl_a.resize(N * m.MN_angular);
  p->q.resize(N * m.dim);
  p->sfx.resize(N * m.na1 * B2_NABC);
  p->FpR.resize(N * m.nr1 + 1);
  p->FpA.resize(N * m.dim_angular + 1);
  p->U.resize(N * m.UST);
  p->f12.resize(N * 3 * m.MN_angular + 1);
  p->acc.resize(N * 13);
  p->zbl_z = m.atomic_numbers;
  p->cov.assign(COVALENT_RADIUS, COVALENT_RADIUS + 94);
  if (m.zbl_para.empty())
    m.zbl_para.push_back(0.0f);
  B2NepView& P = p->P;
  P = nep_view(m, plan, n);
  P.rc_r = m.rc_r.data(); P.rcinv_r = m.rcinv_r.data(); P.rc2_r = m.rc2_r.data();
  P.rc_a = m.rc_a.data(); P.rcinv_a = m.rcinv_a.data(); P.rc2_a = m.rc2_a.data();
  P.c_a4 = reinterpret_cast<const float4*>(m.c_a4.data());
  P.c_r4 = plan.c_r4 ? reinterpret_cast<const float4*>(m.c_r4.data()) : nullptr;
  P.c_r = m.c_r.data(); P.c_a = m.c_a.data(); P.w0p = m.w0p.data(); P.b0 = m.b0.data();
  P.w1 = m.w1.data(); P.bias = m.bias.data(); P.q_scaler = m.q_scaler.data();
  P.zbl_z = p->zbl_z.data(); P.zbl_para = m.zbl_para.data(); P.cov_radius = p->cov.data();
  P.nn_r = p->nn_r.data(); P.nl_r = p->nl_r.data(); P.nn_a = p->nn_a.data(); P.nl_a = p->nl_a.data();
  P.aslot = plan.rev_slot ? p->aslot.data() : nullptr;
  P.nla_rs = plan.rev_slot ? p->nla_rs.data() : nullptr;
  P.q = p->q.data(); P.sfx = p->sfx.data(); P.FpR = p->FpR.data(); P.FpA = p->FpA.data(); P.U = p->U.data();
  P.f12 = p->f12.data(); P.acc = p->acc.data();
  return "";
}

emu_nep* emu_nep_create(const char* path, int n)
{
  emu_nep* p = new emu_nep;
  g_err = p->m.load(path);
  if (g_err.empty())
    g_err = emu_nep_alloc(p, n);
  if (!g_err.empty()) {
    delete p;
    return nullptr;
  }
  p->n_cell = n;
  return p;
}

// the plan of the handle's last setup, in the order of emu_py.NEP_PLAN
void emu_nep_plan(const emu_nep* p, long long* out)
{
  const NepPlan& q = p->plan;
  const long long v[] = {q.mn_skin, q.pitch_r, q.team, q.fuse_split, q.radial_v2, q.sched, q.ang_fused,
                         q.fused_shape, (long long)q.fused_smem, q.use_tc, q.utable_tc, q.rev_slot, q.slot_map,
                         q.rad_reg, q.rad_direct, q.rad_nt, q.c_r4, q.ang_cstage, q.variant, q.tc_ctas_cap,
                         q.debug_skip, q.ang_block, (long long)q.ang_smem, (long long)q.rad_smem};
  std::copy(std::begin(v), std::end(v), out);
}

void emu_nep_destroy(emu_nep* p) { delete p; }
int emu_nep_rebuilds(emu_nep* p) { return p->nb.flags[2]; }
int emu_nep_error_bits(emu_nep* p) { return p->nb.flags[1]; }

// the pipeline proper on p->n atoms (declared below)
static int emu_nep_pipeline(
  emu_nep* p, const B2Box& box, const int* type, const double* pos, double* pe, double* force,
  double* virial);

int emu_nep_compute(
  emu_nep* p, int n, const double h[9], const int pbc[3], const int* type, const double* pos,
  double* pe, double* force, double* virial)
{
  if (n != p->n_cell)
    return 1;
  B2Box box = make_box(h, pbc);
  // small periodic boxes: supercell replication, the host twin of b200md_nep_compute
  int reps[3];
  const int R = (int)supercell_reps(box, p->nb.rc, p->nb.skin, reps);
  if (R == 1) {
    if (p->n != n && !(g_err = emu_nep_alloc(p, n)).empty())
      return 1;
    p->P.overwrite = p->overwrite;
    p->P.n_own = p->n_own;
    return emu_nep_pipeline(p, box, type, pos, pe, force, virial);
  }
  const int nR = n * R;
  if (p->n != nR && !(g_err = emu_nep_alloc(p, nR)).empty())
    return 1;
  p->P.overwrite = p->overwrite;
  p->P.n_own = p->n_own;
  std::vector<int> t2(nR);
  std::vector<double> x2((size_t)3 * nR), out((size_t)13 * nR, 0.0);
  for (int r = 0; r < R; ++r) {
    const int c = r % reps[2], b = (r / reps[2]) % reps[1], a = r / (reps[2] * reps[1]);
    for (int i = 0; i < n; ++i) {
      const size_t e = (size_t)r * n + i;
      t2[e] = type[i];
      x2[e] = pos[i] + a * box.h[0] + b * box.h[1] + c * box.h[2];
      x2[nR + e] = pos[(size_t)n + i] + a * box.h[3] + b * box.h[4] + c * box.h[5];
      x2[2 * (size_t)nR + e] = pos[2 * (size_t)n + i] + a * box.h[6] + b * box.h[7] + c * box.h[8];
    }
  }
  double hs[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      hs[3 * r + c] = h[3 * r + c] * reps[c];
  box = make_box(hs, pbc);
  const int rc = emu_nep_pipeline(
    p, box, t2.data(), x2.data(), out.data(), out.data() + nR, out.data() + 4 * (size_t)nR);
  // k_fold_replica
  const int w = p->overwrite;
  const int n_fold = p->n_own > 0 && p->n_own < n ? p->n_own : n;
  for (int i = 0; i < n_fold; ++i) {
    pe[i] = (w ? 0.0 : pe[i]) + out[i];
    for (int k = 0; k < 3; ++k)
      force[(size_t)k * n + i] = (w ? 0.0 : force[(size_t)k * n + i]) + out[nR + (size_t)k * nR + i];
    for (int k = 0; k < 9; ++k)
      virial[(size_t)k * n + i] =
        (w ? 0.0 : virial[(size_t)k * n + i]) + out[4 * (size_t)nR + (size_t)k * nR + i];
  }
  return rc;
}

// b200md_nep_set_accumulate(p, !overwrite) and b200md_nep_set_owned(p, n_own)
void emu_nep_set_mode(emu_nep* p, int overwrite, int n_own)
{
  p->overwrite = overwrite;
  p->n_own = n_own;
}
}

static int emu_nep_pipeline(
  emu_nep* p, const B2Box& box, const int* type, const double* pos, double* pe, double* force,
  double* virial)
{
  const int n = p->n;
  const int rc = p->nb.update(box, type, pos);
  if (rc)
    return rc;
  B2NepView& P = p->P;
  P.atoms = p->nb.atoms.data();
  P.perm = p->nb.perm.data();
  P.nn_skin = p->nb.nn_skin.data();
  P.nl_skin = p->nb.nl_skin.data();
  P.rskin = p->plan.rev_slot ? p->nb.rskin.data() : nullptr;
  P.skin_si = p->nb.v.skin_si;
  P.skin_sk = p->nb.v.skin_sk;
  P.flags = p->nb.flags.data();
  switch (p->m.K1R) {
    case 9: run_desc_radial<9>(p, box); break;
    case 13: run_desc_radial<13>(p, box); break;
    default: run_desc_radial<17>(p, box); break;
  }
  switch (p->m.K1A) {
    case 9: run_angular<9>(p, box, false); break;
    case 13: run_angular<13>(p, box, false); break;
    default: run_angular<17>(p, box, false); break;
  }
  switch (p->m.DIMP) {
    case 16: run_mlp<16>(p); break;
    case 32: run_mlp<32>(p); break;
    case 48: run_mlp<48>(p); break;
    case 64: run_mlp<64>(p); break;
    case 80: run_mlp<80>(p); break;
    case 96: run_mlp<96>(p); break;
    case 112: run_mlp<112>(p); break;
    default: run_mlp<128>(p); break;
  }
  for (int i = 0; i < n; ++i) {
    if (p->m.K1R == 9)
      p->plan.team ? b2_body_utable_planes<9>(i, P) : b2_body_utable<9>(i, P);
    else if (p->m.K1R == 13)
      p->plan.team ? b2_body_utable_planes<13>(i, P) : b2_body_utable<13>(i, P);
    else
      p->plan.team ? b2_body_utable_planes<17>(i, P) : b2_body_utable<17>(i, P);
  }
  switch (p->m.K1A) {
    case 9: run_angular<9>(p, box, true); break;
    case 13: run_angular<13>(p, box, true); break;
    default: run_angular<17>(p, box, true); break;
  }
  switch (p->m.K1R) {
    case 9: run_force_final<9>(p, box, pe, force, virial); break;
    case 13: run_force_final<13>(p, box, pe, force, virial); break;
    default: run_force_final<17>(p, box, pe, force, virial); break;
  }
  return p->nb.flags[1] ? 5 : 0;
}

extern "C" {

static void export_list(
  int n, int n_cell, const int* perm, const int* nn, const int* nl, size_t si, size_t sk, int mn,
  int* NN, int* NL)
{
  for (int i = 0; i < n; ++i) {
    const int a = perm[i];
    if (a >= n_cell)
      continue; // supercell: report the first replica only
    const int cnt = nn[i] < mn ? nn[i] : mn;
    int* row = NL + (size_t)a * mn;
    for (int k = 0; k < cnt; ++k) {
      const int v = perm[nl[(size_t)i * si + (size_t)k * sk]] % n_cell;
      int q = k - 1;
      while (q >= 0 && row[q] > v) {
        row[q + 1] = row[q];
        --q;
      }
      row[q + 1] = v;
    }
    NN[a] = cnt;
  }
}

void emu_nep_export_neighbors(
  emu_nep* p, int mn_r, int* NN_r, int* NL_r, int mn_a, int* NN_a, int* NL_a)
{
  export_list(
    p->n, p->n_cell, p->P.perm, p->nn_r.data(), p->nl_r.data(),
    p->plan.team ? (size_t)p->P.pitch_r : 1, p->plan.team ? 1 : (size_t)p->n, mn_r, NN_r, NL_r);
  export_list(
    p->n, p->n_cell, p->P.perm, p->nn_a.data(), p->nl_a.data(), 1, (size_t)p->n, mn_a, NN_a, NL_a);
}

void emu_nep_export_descriptors(emu_nep* p, float* q)
{
  for (int i = 0; i < p->n; ++i)
    for (int d = 0; d < p->m.dim; ++d)
      if (p->P.perm[i] < p->n_cell)
        q[(size_t)d * p->n_cell + p->P.perm[i]] = p->q[(size_t)d * p->n + i] * p->m.q_scaler[d];
}

// skin list of the last rebuild, in caller indices (row-major, ascending) -- neighbour tests
void emu_nep_export_skin(emu_nep* p, int mn, int* NN, int* NL)
{
  export_list(
    p->n, p->n_cell, p->P.perm, p->nb.nn_skin.data(), p->nb.nl_skin.data(), p->nb.v.skin_si,
    p->nb.v.skin_sk, mn, NN, NL);
}

// ---- LJ -------------------------------------------------------------------------------------
struct emu_lj {
  LjFile file;
  EmuNeighbor nb;
  std::vector<double> acc;
};

emu_lj* emu_lj_create(const char* path, int n)
{
  emu_lj* p = new emu_lj;
  g_err = load_lj(path, p->file);
  if (!g_err.empty()) {
    delete p;
    return nullptr;
  }
  p->nb.init(n, p->file.rc, p->file.mn_skin);
  p->acc.resize((size_t)13 * n);
  return p;
}
void emu_lj_destroy(emu_lj* p) { delete p; }
int emu_lj_error_bits(emu_lj* p) { return p->nb.flags[1]; }
int emu_lj_compute(
  emu_lj* p, int n, const double h[9], const int pbc[3], const int* type, const double* pos,
  double* pe, double* force, double* virial)
{
  const B2Box box = make_box(h, pbc);
  const int rc = p->nb.update(box, type, pos);
  if (rc)
    return rc;
  B2LjView P;
  P.nt = p->file.nt;
  P.s6e4 = p->file.s6e4.data();
  P.s12e4 = p->file.s12e4.data();
  P.rc2 = p->file.rc2.data();
  P.n = n;
  P.atoms = p->nb.atoms.data();
  P.nn_skin = p->nb.nn_skin.data();
  P.nl_skin = p->nb.nl_skin.data();
  P.acc = p->acc.data();
  for (int i = 0; i < n; ++i)
    b2_body_lj(i, P, box);
  for (int i = 0; i < n; ++i)
    b2_body_unpack(i, n, p->nb.perm.data(), p->acc.data(), pe, force, virial);
  return p->nb.flags[1] ? 5 : 0;
}

// ---- Tersoff --------------------------------------------------------------------------------
struct emu_tersoff {
  B2TersoffView P;
  EmuNeighbor nb;
  std::vector<int> nn, nl;
  std::vector<double> f12, acc;
};

emu_tersoff* emu_tersoff_create(const char* path, int n)
{
  emu_tersoff* p = new emu_tersoff;
  TersoffFile file;
  g_err = load_tersoff(path, file);
  if (!g_err.empty()) {
    delete p;
    return nullptr;
  }
  p->P = file.view;
  p->nb.init(n, file.rc, file.mn_skin);
  p->nn.resize(n);
  p->nl.resize((size_t)n * B2_TERSOFF_MAXL);
  p->f12.resize((size_t)3 * n * B2_TERSOFF_MAXL);
  p->acc.resize((size_t)13 * n);
  return p;
}
void emu_tersoff_destroy(emu_tersoff* p) { delete p; }
int emu_tersoff_error_bits(emu_tersoff* p) { return p->nb.flags[1]; }
int emu_tersoff_compute(
  emu_tersoff* p, int n, const double h[9], const int pbc[3], const int* type, const double* pos,
  double* pe, double* force, double* virial)
{
  const B2Box box = make_box(h, pbc);
  const int rc = p->nb.update(box, type, pos);
  if (rc)
    return rc;
  B2TersoffView& P = p->P;
  P.n = n;
  P.atoms = p->nb.atoms.data();
  P.nn_skin = p->nb.nn_skin.data();
  P.nl_skin = p->nb.nl_skin.data();
  P.nn = p->nn.data();
  P.nl = p->nl.data();
  P.f12 = p->f12.data();
  P.acc = p->acc.data();
  P.flags = p->nb.flags.data();
  for (int i = 0; i < n; ++i)
    b2_body_tersoff_partial(i, P, box);
  for (int i = 0; i < n; ++i)
    b2_body_tersoff_reduce(i, P, box);
  for (int i = 0; i < n; ++i)
    b2_body_unpack(i, n, p->nb.perm.data(), p->acc.data(), pe, force, virial);
  return p->nb.flags[1] ? 5 : 0;
}
void emu_compute_heat(int n, const double* w, const double* v, double* heat)
{
  for (int i = 0; i < n; ++i)
    b2_body_heat(i, n, w, v, heat, n);
}

// ---- EAM ------------------------------------------------------------------------------------
struct emu_eam {
  EamFile file;
  std::vector<float> Fp;
  std::vector<double> acc;
  EmuNeighbor nb;
};

emu_eam* emu_eam_create(const char* path, int n)
{
  emu_eam* p = new emu_eam;
  g_err = load_eam(path, p->file);
  if (!g_err.empty()) {
    delete p;
    return nullptr;
  }
  p->nb.init(n, p->file.rc, p->file.mn_skin);
  p->Fp.resize(n);
  p->acc.resize((size_t)13 * n);
  return p;
}
void emu_eam_destroy(emu_eam* p) { delete p; }
int emu_eam_error_bits(emu_eam* p) { return p->nb.flags[1]; }
int emu_eam_compute(
  emu_eam* p, int n, const double h[9], const int pbc[3], const int* type, const double* pos,
  double* pe, double* force, double* virial)
{
  const B2Box box = make_box(h, pbc);
  const int rc = p->nb.update(box, type, pos);
  if (rc)
    return rc;
  B2EamView& P = p->file.view;
  P.zp = p->file.zp.data();
  P.n = n;
  P.atoms = p->nb.atoms.data();
  P.nn_skin = p->nb.nn_skin.data();
  P.nl_skin = p->nb.nl_skin.data();
  P.Fp = p->Fp.data();
  P.acc = p->acc.data();
  for (int i = 0; i < n; ++i)
    b2_body_eam_density(i, P, box);
  for (int i = 0; i < n; ++i)
    b2_body_eam_force(i, P, box);
  for (int i = 0; i < n; ++i)
    b2_body_unpack(i, n, p->nb.perm.data(), p->acc.data(), pe, force, virial);
  return p->nb.flags[1] ? 5 : 0;
}

// ---- integrate ------------------------------------------------------------------------------
void emu_apply_pbc(int n, const double h[9], const int pbc[3], double* pos)
{
  const B2Box box = make_box(h, pbc);
  for (int i = 0; i < n; ++i)
    b2_body_apply_pbc(i, n, box, pos, pos + n, pos + 2 * (size_t)n);
}
void emu_velocity_verlet(
  int step1, int n, double dt, const double* mass, double* pos, double* vel, const double* f)
{
  for (int i = 0; i < n; ++i)
    b2_body_vv(i, n, step1 != 0, dt, mass, pos, vel, f); // stride = n
}
void emu_velocity_verlet_groups(
  int step1, int n, double dt, const double* mass, double* pos, double* vel, const double* f,
  const int* label, int fixed_group, int move_group, const double* mv)
{
  for (int i = 0; i < n; ++i)
    b2_body_vv_groups(i, n, step1 != 0, dt, mass, pos, vel, f, label, fixed_group, move_group, mv);
}
void emu_find_thermo(
  int n, int n_temp, double volume, const double* mass, const double* pe, const double* vel,
  const double* virial, double* thermo)
{
  double s[8] = {0};
  for (int i = 0; i < n; ++i) {
    double t[8];
    b2_thermo_terms(i, n, mass, pe, vel, virial, t);
    for (int k = 0; k < 8; ++k)
      s[k] += t[k];
  }
  thermo[0] = s[0] / (3.0 * n_temp * 8.617343e-5);
  thermo[1] = s[1];
  for (int k = 2; k < 8; ++k)
    thermo[k] = s[k] / volume;
}

// ---- BDP thermostat body (b2_bdp.cuh) ----
void* emu_bdp_create(unsigned seed)
{
  B2BdpState* st = new B2BdpState;
  b2_mt_seed(*st, seed);
  return st;
}
void emu_bdp_destroy(void* st) { delete static_cast<B2BdpState*>(st); }
double emu_bdp_rand01(void* st) { return b2_rand01(*static_cast<B2BdpState*>(st)); }
double emu_bdp_factor(void* st, double t_instant, int ndeg, double temperature, double coupling)
{
  return b2_bdp_factor(*static_cast<B2BdpState*>(st), t_instant, ndeg, temperature, coupling);
}
}

// ensemble.cpp -- see ensemble.h.  Every kernel runs on the legacy default stream, like the
// reference's integrators (SURVEY.md 8b).
#include "ensemble.h"
#include "potential.h"
#include <cmath>
#include <cstdio>
#include <cstdlib>

static void set_move(Ensemble& e, int mg, const double mv[3])
{
  e.move_group = mg;
  for (int d = 0; d < 3; ++d)
    e.move_velocity[d] = mv ? mv[d] : 0.0;
}

void B200_Integrator::b2_velocity_verlet(
  const Ensemble& e, const bool is_step1, const double time_step, const std::vector<Group>& group,
  Atom& atom)
{
  const int n = atom.number_of_atoms;
  const int* label = nullptr;
  if (e.fixed_group >= 0 || e.move_group >= 0) {
    if ((int)group.size() <= e.fixed_grouping_method) {
      fprintf(stderr, "Input Error:\n    fix / move need a grouping method in model.xyz.\n");
      exit(1);
    }
    label = group[e.fixed_grouping_method].label.data();
  }
  if (b200md_velocity_verlet_groups(
        is_step1 ? 1 : 0, n, n, time_step, atom.mass.data(), atom.position_per_atom.data(),
        atom.velocity_per_atom.data(), atom.force_per_atom.data(), label, e.fixed_group,
        e.move_group, e.move_velocity, nullptr) != B200MD_OK)
    b2h_fail("Ensemble::velocity_verlet");
}

int B200_Integrator::b2_num_integrated(const Ensemble& e, const std::vector<Group>& group, int n)
{
  if (e.fixed_group >= 0)
    n -= group[e.fixed_grouping_method].cpu_size[e.fixed_group];
  if (e.move_group >= 0)
    n -= group[e.move_grouping_method].cpu_size[e.move_group];
  return n;
}

void B200_Integrator::b2_find_thermo(
  const Ensemble& e, const double volume, const std::vector<Group>& group, Atom& atom,
  GPU_Vector<double>& thermo)
{
  const int n = atom.number_of_atoms;
  const int n_temperature = b2_num_integrated(e, group, n); // ensemble.cu:645-651
  const size_t need = (size_t)b200md_thermo_scratch_bytes(n);
  if (scratch_.size() != need)
    scratch_.resize(need, 0);
  if (b200md_find_thermo(
        n, n_temperature, volume, atom.mass.data(), atom.potential_per_atom.data(),
        atom.velocity_per_atom.data(), atom.virial_per_atom.data(), thermo.data(),
        scratch_.data(), nullptr) != B200MD_OK)
    b2h_fail("Ensemble::find_thermo");
}

void Ensemble_NVE_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  b2_velocity_verlet(*this, true, time_step, group, atom);
}

void Ensemble_NVE_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  b2_velocity_verlet(*this, false, time_step, group, atom);
  b2_find_thermo(*this, box.get_volume(), group, atom, thermo);
}

Ensemble_BER_B200::Ensemble_BER_B200(int t, int mg, const double mv[3], double T, double Tc)
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, mg, mv);
}

Ensemble_BER_B200::Ensemble_BER_B200(
  int t, double T, double Tc, const double target_p[6], int num_target_p, const double pc[6], int dx,
  int dy, int dz, const double rate[3])
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, -1, nullptr);
  for (int k = 0; k < 6; ++k) {
    b2_target_p_[k] = target_p[k];
    b2_pc_[k] = pc[k];
  }
  b2_num_p_ = num_target_p;
  b2_deform_[0] = dx;
  b2_deform_[1] = dy;
  b2_deform_[2] = dz;
  for (int d = 0; d < 3; ++d)
    b2_rate_[d] = rate ? rate[d] : 0.0;
}

void Ensemble_BER_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  b2_velocity_verlet(*this, true, time_step, group, atom);
}

void Ensemble_BER_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  b2_velocity_verlet(*this, false, time_step, group, atom);
  b2_find_thermo(*this, box.get_volume(), group, atom, thermo);
  const int n = atom.number_of_atoms;
  if (b200md_berendsen_temperature(
        n, n, temperature, temperature_coupling, thermo.data(), atom.velocity_per_atom.data(),
        nullptr) != B200MD_OK)
    b2h_fail("Ensemble_BER_B200::compute2");
  if (type == 11) { // npt_ber: rescale the box (host) and the positions (device)
    int pbc[3];
    b2h_pbc(box, pbc);
    if (b200md_berendsen_pressure(
          n, n, b2_num_p_, b2_target_p_, b2_pc_, b2_deform_, b2_rate_, pbc, box.cpu_h, thermo.data(),
          atom.position_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("Ensemble_BER_B200::compute2 (pressure)");
    box.get_inverse();
  }
}

Ensemble_BDP_B200::Ensemble_BDP_B200(int t, int mg, const double mv[3], double T, double Tc, unsigned seed)
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, mg, mv);
  seed_ = seed;
}

Ensemble_BDP_B200::~Ensemble_BDP_B200() { b200md_bdp_destroy(bdp_); }

void Ensemble_BDP_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  b2_velocity_verlet(*this, true, time_step, group, atom);
}

void Ensemble_BDP_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  b2_velocity_verlet(*this, false, time_step, group, atom);
  b2_find_thermo(*this, box.get_volume(), group, atom, thermo);
  const int n = atom.number_of_atoms;
  // the first step: `fix` / `move` are set by now (integrate.cu:279-281), so the generator gets
  // ndeg = 3 (N - N_fixed - N_move) (ensemble_bdp.cu:87-95); the seed is fixed, so creating it
  // here rather than in the constructor leaves the stream unchanged
  if (!bdp_ && b200md_bdp_create(b2_num_integrated(*this, group, n), temperature, temperature_coupling,
                                 seed_, &bdp_) != B200MD_OK)
    b2h_fail("Ensemble_BDP_B200");
  if (b200md_bdp_step(bdp_, n, n, thermo.data(), atom.velocity_per_atom.data(), nullptr) != B200MD_OK)
    b2h_fail("Ensemble_BDP_B200::compute2");
}

Ensemble_NHC_B200::Ensemble_NHC_B200(
  int t, int mg, const double mv[3], int N, double T, double Tc, double time_step_in)
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, mg, mv);
  if (b200md_nhc_create(N, T, Tc, time_step_in, &nhc_) != B200MD_OK)
    b2h_fail("Ensemble_NHC_B200");
}

Ensemble_NHC_B200::~Ensemble_NHC_B200() { b200md_nhc_destroy(nhc_); }

void Ensemble_NHC_B200::thermostat(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  b2_find_thermo(*this, box.get_volume(), group, atom, thermo);
  const int n = atom.number_of_atoms;
  if (b200md_nhc_half_step(
        nhc_, n, n, time_step, thermo.data(), atom.velocity_per_atom.data(), nullptr) != B200MD_OK)
    b2h_fail("Ensemble_NHC_B200::thermostat");
}

void Ensemble_NHC_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  thermostat(time_step, group, box, atom, thermo);
  b2_velocity_verlet(*this, true, time_step, group, atom);
}

void Ensemble_NHC_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  b2_velocity_verlet(*this, false, time_step, group, atom);
  thermostat(time_step, group, box, atom, thermo);
}

// ---- nvt_lan: half Langevin kick, velocity-Verlet, half Langevin kick -------------------------
static const double B2H_K_B = 8.617343e-5; // common.cuh:21

Ensemble_LAN_B200::Ensemble_LAN_B200(int t, int N, double T, double Tc, unsigned long long seed)
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, -1, nullptr);
  c1_ = exp(-0.5 / temperature_coupling);
  if (b200md_langevin_create(N, seed, &lan_) != B200MD_OK)
    b2h_fail("Ensemble_LAN_B200");
}

Ensemble_LAN_B200::~Ensemble_LAN_B200() { b200md_langevin_destroy(lan_); }

void Ensemble_LAN_B200::half(Atom& atom)
{
  const int n = atom.number_of_atoms;
  const double c2 = sqrt((1 - c1_ * c1_) * B2H_K_B * temperature); // the target may ramp (ensemble_lan.cu:98)
  if (b200md_langevin_apply(lan_, n, n, c1_, c2, atom.mass.data(), atom.velocity_per_atom.data(), nullptr) !=
      B200MD_OK)
    b2h_fail("Ensemble_LAN_B200");
}

void Ensemble_LAN_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  half(atom);
  b2_velocity_verlet(*this, true, time_step, group, atom);
}

void Ensemble_LAN_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  b2_velocity_verlet(*this, false, time_step, group, atom);
  half(atom);
  b2_find_thermo(*this, box.get_volume(), group, atom, thermo);
}

// ---- nvt_bao: B A O A | force | B -----------------------------------------------------------------
Ensemble_BAO_B200::Ensemble_BAO_B200(int t, int N, double T, double Tc, unsigned long long seed)
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, -1, nullptr);
  c1_ = exp(-1.0 / temperature_coupling);
  if (b200md_langevin_create(N, seed, &lan_) != B200MD_OK)
    b2h_fail("Ensemble_BAO_B200");
}

Ensemble_BAO_B200::~Ensemble_BAO_B200() { b200md_langevin_destroy(lan_); }

void Ensemble_BAO_B200::op(
  int which, const double time_step, const std::vector<Group>& group, Atom& atom)
{
  const int n = atom.number_of_atoms;
  const int* label = fixed_group >= 0 ? group[fixed_grouping_method].label.data() : nullptr;
  if (b200md_baoab_operator(
        which, n, n, time_step, atom.mass.data(), atom.position_per_atom.data(),
        atom.velocity_per_atom.data(), atom.force_per_atom.data(), label, fixed_group, nullptr) !=
      B200MD_OK)
    b2h_fail("Ensemble_BAO_B200");
}

void Ensemble_BAO_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  op(1, time_step, group, atom);
  op(0, time_step, group, atom);
  const int n = atom.number_of_atoms;
  const double c2 = sqrt((1 - c1_ * c1_) * B2H_K_B * temperature);
  if (b200md_langevin_apply(lan_, n, n, c1_, c2, atom.mass.data(), atom.velocity_per_atom.data(), nullptr) !=
      B200MD_OK)
    b2h_fail("Ensemble_BAO_B200");
  op(0, time_step, group, atom);
}

void Ensemble_BAO_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
  GPU_Vector<double>& thermo)
{
  op(1, time_step, group, atom);
  b2_find_thermo(*this, box.get_volume(), group, atom, thermo);
}

// ---- heat_lan / heat_nhc / heat_bdp: bath half, velocity-Verlet, bath half --------------------------
Ensemble_HEAT_B200::Ensemble_HEAT_B200(
  int t, int kind, int N, const std::vector<int>& group_sizes, const int* contents, int source, int sink,
  double T, double Tc, double dT, double time_step, unsigned long long seed_source,
  unsigned long long seed_sink)
{
  type = t;
  temperature = T;
  temperature_coupling = Tc;
  set_move(*this, -1, nullptr);
  if (b200md_heat_bath_create(
        kind, N, (int)group_sizes.size(), group_sizes.data(), contents, source, sink, T, Tc, dT,
        time_step, seed_source, seed_sink, &bath_) != B200MD_OK)
    b2h_fail("Ensemble_HEAT_B200");
}

Ensemble_HEAT_B200::~Ensemble_HEAT_B200() { b200md_heat_bath_destroy(bath_); }

void Ensemble_HEAT_B200::compute1(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  const int n = atom.number_of_atoms;
  if (b200md_heat_bath_half(bath_, 0, n, n, atom.mass.data(), atom.velocity_per_atom.data(), nullptr) !=
      B200MD_OK)
    b2h_fail("Ensemble_HEAT_B200::compute1");
  b2_velocity_verlet(*this, true, time_step, group, atom);
}

void Ensemble_HEAT_B200::compute2(
  const double time_step, const std::vector<Group>& group, Box&, Atom& atom, GPU_Vector<double>&)
{
  b2_velocity_verlet(*this, false, time_step, group, atom);
  const int n = atom.number_of_atoms;
  if (b200md_heat_bath_half(bath_, 1, n, n, atom.mass.data(), atom.velocity_per_atom.data(), nullptr) !=
      B200MD_OK)
    b2h_fail("Ensemble_HEAT_B200::compute2");
}

void Ensemble_HEAT_B200::read_energy_transferred()
{
  if (b200md_heat_bath_energy(bath_, b2_energy_transferred, nullptr) != B200MD_OK)
    b2h_fail("Ensemble_HEAT_B200::read_energy_transferred");
}

Ensemble_HEAT_LAN_B200::Ensemble_HEAT_LAN_B200(
  int t, int mg, const double mv[3], int N, const std::vector<int>& group_sizes, const int* contents,
  int source, int sink, double T, double Tc, double dT, unsigned long long seed_source,
  unsigned long long seed_sink)
    : Ensemble_HEAT_B200(t, 0, N, group_sizes, contents, source, sink, T, Tc, dT, 0.0, seed_source, seed_sink)
{
  set_move(*this, mg, mv);
}

Ensemble_HEAT_NHC_B200::Ensemble_HEAT_NHC_B200(
  int t, int N, const std::vector<int>& group_sizes, const int* contents, int source, int sink, double T,
  double Tc, double dT, double time_step)
    : Ensemble_HEAT_B200(t, 1, N, group_sizes, contents, source, sink, T, Tc, dT, time_step, 0, 0)
{
}

Ensemble_HEAT_BDP_B200::Ensemble_HEAT_BDP_B200(
  int t, int N, const std::vector<int>& group_sizes, const int* contents, int source, int sink, double T,
  double Tc, double dT, unsigned seed)
    : Ensemble_HEAT_B200(t, 2, N, group_sizes, contents, source, sink, T, Tc, dT, 0.0, seed, 0)
{
}

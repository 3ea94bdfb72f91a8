// ensemble.h -- adapters that put libb200md's integrator kernels behind GPUMD's Ensemble plugin
// interface (src/integrate/ensemble.cuh:26-157): compute1 / compute2 with the reference's
// signatures, `fix` / `move` groups honoured, thermo[0..7] left on the device after compute2.
//   Ensemble_NVE_B200  replaces Ensemble_NVE, src/integrate/ensemble_nve.cu:31-95
//   Ensemble_BER_B200  replaces Ensemble_BER (type 1, nvt_ber), ensemble_ber.cu:178-233
//   Ensemble_NHC_B200  replaces Ensemble_NHC (type 2, nvt_nhc), ensemble_nhc.cu:173-237
//   Ensemble_BDP_B200  replaces Ensemble_BDP (type 4, nvt_bdp), ensemble_bdp.cu:69-101,151-196
//   Ensemble_LAN_B200  replaces Ensemble_LAN (type 3, nvt_lan), ensemble_lan.cu:29-41,92-124,190-269
//   Ensemble_BAO_B200  replaces Ensemble_BAO (type 5, nvt_bao), ensemble_bao.cu:29-41,91-120,419-470
//   Ensemble_BER_B200 with a target pressure = npt_ber (type 11), ensemble_ber.cu:38-64,88-172,237-285
// Inside the reference tree (B200MD_IN_GPUMD, oracle/Makefile.gpumd_b200) they derive from the
// reference's own class Ensemble; the standalone driver uses a same-shaped base.
#pragma once
#include "../../include/b200md.h"
#include <vector>

#if defined(B200MD_IN_GPUMD)
#include "integrate/ensemble.cuh"
#include "model/atom.cuh"
#include "model/box.cuh"
#include "model/group.cuh"
#else
#include "model.h"

class Ensemble
{
public:
  virtual ~Ensemble() = default;
  virtual void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) = 0;
  virtual void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) = 0;
  int type = 0;
  int fixed_group = -1; // ID of the group whose atoms are frozen (`fix`, integrate.cu:1362-1403)
  int move_group = -1;  // ID of the group that moves with a constant velocity (`move`, :1405-1470)
  int fixed_grouping_method = 0;
  int move_grouping_method = 0;
  double move_velocity[3] = {0.0, 0.0, 0.0};
  double temperature = 0.0;
  double temperature_coupling = 100.0;
};
#endif

// the part every adapter shares: the two half steps and the thermo reduction
class B200_Integrator
{
protected:
  // Ensemble::velocity_verlet (ensemble.cu:348-397) with or without groups
  void b2_velocity_verlet(
    const Ensemble& e, const bool is_step1, const double time_step, const std::vector<Group>& group,
    Atom& atom);
  // the atoms outside the fixed and moving groups, ensemble.cu:645-651 and ensemble_bdp.cu:87-88
  static int b2_num_integrated(const Ensemble& e, const std::vector<Group>& group, int n);
  // Ensemble::find_thermo (ensemble.cu:636-673): fixed / moving atoms do not count for T
  void b2_find_thermo(
    const Ensemble& e, const double volume, const std::vector<Group>& group, Atom& atom,
    GPU_Vector<double>& thermo);
  GPU_Vector<char> scratch_;
};

class Ensemble_NVE_B200 : public Ensemble, protected B200_Integrator
{
public:
  explicit Ensemble_NVE_B200(int t = 0) { type = t; }
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
};

class Ensemble_BER_B200 : public Ensemble, protected B200_Integrator
{
public:
  Ensemble_BER_B200(int t, int mg, const double mv[3], double T, double Tc);
  // npt_ber: target pressure / coupling in natural units (integrate.cu:1150-1153), 1, 3 or 6 components
  Ensemble_BER_B200(
    int t, double T, double Tc, const double target_p[6], int num_target_p, const double pc[6], int dx,
    int dy, int dz, const double rate[3]);
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;

private:
  double b2_target_p_[6] = {0, 0, 0, 0, 0, 0}, b2_pc_[6] = {0, 0, 0, 0, 0, 0}, b2_rate_[3] = {0, 0, 0};
  int b2_num_p_ = 0, b2_deform_[3] = {0, 0, 0};
};

// cuRAND XORWOW state per atom on the device, seeded like the reference (rand())
class Ensemble_LAN_B200 : public Ensemble, protected B200_Integrator
{
public:
  Ensemble_LAN_B200(int t, int N, double T, double Tc, unsigned long long seed);
  ~Ensemble_LAN_B200() override;
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;

private:
  void half(Atom& atom);
  b200md_langevin* lan_ = nullptr;
  double c1_ = 0.0;
};

class Ensemble_BAO_B200 : public Ensemble, protected B200_Integrator
{
public:
  Ensemble_BAO_B200(int t, int N, double T, double Tc, unsigned long long seed);
  ~Ensemble_BAO_B200() override;
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;

private:
  void op(int which, const double time_step, const std::vector<Group>& group, Atom& atom);
  b200md_langevin* lan_ = nullptr;
  double c1_ = 0.0;
};

// the generator lives on the device; seed 12345678 follows the reference's -DDEBUG stream.  It is
// created at the first compute2, when `fix` / `move` are known: its degrees of freedom are
// ndeg = 3 (N - N_fixed - N_move) (ensemble_bdp.cu:87-95)
class Ensemble_BDP_B200 : public Ensemble, protected B200_Integrator
{
public:
  Ensemble_BDP_B200(int t, int mg, const double mv[3], double T, double Tc, unsigned seed = 12345678u);
  ~Ensemble_BDP_B200() override;
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;

private:
  b200md_bdp* bdp_ = nullptr;
  unsigned seed_ = 0;
};

class Ensemble_NHC_B200 : public Ensemble, protected B200_Integrator
{
public:
  Ensemble_NHC_B200(int t, int mg, const double mv[3], int N, double T, double Tc, double time_step);
  ~Ensemble_NHC_B200() override;
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;

private:
  void thermostat(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo);
  b200md_nhc* nhc_ = nullptr;
};

// Direct NEMD (heat_lan / heat_nhc / heat_bdp, types 22 / 21 / 23): a heat source at T + dT and a heat
// sink at T - dT, groups `source` and `sink` of grouping method 0, whose sizes and Group::find_contents
// list the caller passes (the reference reads them from group[0], integrate.cu:158-199).  The bath acts
// before velocity-Verlet step 1 and after step 2 (heat_bdp: after step 2 only); like the reference,
// compute2 does NOT call find_thermo, so thermo keeps its last value.  The energy transferred stays on
// the device; read_energy_transferred() synchronises and fills energy_transferred[2].
//   Ensemble_HEAT_LAN_B200 replaces Ensemble_LAN (heat), ensemble_lan.cu:43-85,128-269 (`move` allowed)
//   Ensemble_HEAT_NHC_B200 replaces Ensemble_NHC (heat), ensemble_nhc.cu:52-91,239-326
//   Ensemble_HEAT_BDP_B200 replaces Ensemble_BDP (heat), ensemble_bdp.cu:50-62,103-149
class Ensemble_HEAT_B200 : public Ensemble, protected B200_Integrator
{
public:
  ~Ensemble_HEAT_B200() override;
  void compute1(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void compute2(
    const double time_step, const std::vector<Group>& group, Box& box, Atom& atom,
    GPU_Vector<double>& thermo) override;
  void read_energy_transferred();
  double b2_energy_transferred[2] = {0.0, 0.0};

protected:
  Ensemble_HEAT_B200(
    int t, int kind, int N, const std::vector<int>& group_sizes, const int* contents, int source,
    int sink, double T, double Tc, double dT, double time_step, unsigned long long seed_source,
    unsigned long long seed_sink);
  b200md_heat_bath* bath_ = nullptr;
};

class Ensemble_HEAT_LAN_B200 : public Ensemble_HEAT_B200
{
public:
  // seeds: the reference's next two rand() values (ensemble_lan.cu:78-81)
  Ensemble_HEAT_LAN_B200(
    int t, int mg, const double mv[3], int N, const std::vector<int>& group_sizes, const int* contents,
    int source, int sink, double T, double Tc, double dT, unsigned long long seed_source,
    unsigned long long seed_sink);
};

class Ensemble_HEAT_NHC_B200 : public Ensemble_HEAT_B200
{
public:
  Ensemble_HEAT_NHC_B200(
    int t, int N, const std::vector<int>& group_sizes, const int* contents, int source, int sink,
    double T, double Tc, double dT, double time_step);
};

class Ensemble_HEAT_BDP_B200 : public Ensemble_HEAT_B200
{
public:
  Ensemble_HEAT_BDP_B200(
    int t, int N, const std::vector<int>& group_sizes, const int* contents, int source, int sink,
    double T, double Tc, double dT, unsigned seed = 12345678u);
};

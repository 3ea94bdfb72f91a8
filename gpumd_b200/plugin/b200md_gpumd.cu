// b200md_gpumd.cu -- see b200md_gpumd.cuh.  One translation unit inside the GPUMD build: the adapter
// sources of gpumd_b200/host compiled against the reference's headers.
#define B200MD_IN_GPUMD 1
#include "b200md_gpumd.cuh"
#include "../host/ensemble.cpp"
#include "../host/potential.cpp"
#include <chrono>
#include <cstdlib>
#include <cstring>

static bool b200md_enabled()
{
  const char* v = std::getenv("GPUMD_B200");
  return v && std::strcmp(v, "0") != 0;
}

bool b200md_make_potential(
  const char* name, const char* file, const int number_of_atoms,
  std::unique_ptr<Potential>& potential)
{
  if (!b200md_enabled())
    return false;
  if (std::strcmp(name, "nep3") == 0 || std::strcmp(name, "nep3_zbl") == 0 ||
      std::strcmp(name, "nep4") == 0 || std::strcmp(name, "nep4_zbl") == 0 ||
      std::strcmp(name, "nep5") == 0 || std::strcmp(name, "nep5_zbl") == 0) {
    // a model option libb200md rejects (b200md_nep_create fails) ends the run with its message,
    // like any other input error
    potential.reset(new NEP_B200(file, number_of_atoms));
  } else if (std::strcmp(name, "lj") == 0) {
    potential.reset(new LJ_B200(file, number_of_atoms));
  } else if (std::strcmp(name, "tersoff_1989") == 0) {
    potential.reset(new Tersoff1989_B200(file, number_of_atoms));
  } else if (std::strcmp(name, "eam_zhou_2004") == 0 || std::strcmp(name, "eam_dai_2006") == 0) {
    potential.reset(new EAM_B200(file, number_of_atoms));
  } else {
    return false;
  }
  return true;
}

bool b200md_make_ensemble(
  const int type, const int move_group, const double* move_velocity, const int number_of_atoms,
  const double temperature, const double temperature_coupling, const double time_step,
  const double* target_pressure, const int num_target_pressure_components,
  const double* pressure_coupling, const int deform_x, const int deform_y, const int deform_z,
  const double* deform_rate, std::unique_ptr<Ensemble>& ensemble)
{
  if (!b200md_enabled())
    return false;
  switch (type) {
    case 0: ensemble.reset(new Ensemble_NVE_B200(type)); break;
    case 1:
      ensemble.reset(
        new Ensemble_BER_B200(type, move_group, move_velocity, temperature, temperature_coupling));
      break;
    case 2:
      ensemble.reset(new Ensemble_NHC_B200(
        type, move_group, move_velocity, number_of_atoms, temperature, temperature_coupling, time_step));
      break;
    case 4: {
#ifdef DEBUG
      const unsigned seed = 12345678u; // ensemble_bdp.cu:31-32
#else
      const unsigned seed = (unsigned)std::chrono::system_clock::now().time_since_epoch().count();
#endif
      ensemble.reset(new Ensemble_BDP_B200(
        type, move_group, move_velocity, temperature, temperature_coupling, seed));
      break;
    }
    case 3: // the reference seeds cuRAND with rand() (ensemble_lan.cu:39): same call, same stream
      ensemble.reset(new Ensemble_LAN_B200(
        type, number_of_atoms, temperature, temperature_coupling, (unsigned long long)rand()));
      break;
    case 5:
      ensemble.reset(new Ensemble_BAO_B200(
        type, number_of_atoms, temperature, temperature_coupling, (unsigned long long)rand()));
      break;
    case 11:
      ensemble.reset(new Ensemble_BER_B200(
        type, temperature, temperature_coupling, target_pressure, num_target_pressure_components,
        pressure_coupling, deform_x, deform_y, deform_z, deform_rate));
      break;
    default: return false; // every other ensemble stays with the reference's own class
  }
  printf("Use the b200md integrator for ensemble type %d.\n", type);
  return true;
}

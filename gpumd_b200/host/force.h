// force.h -- the Force driver (src/force/force.cuh:27-85): parse_potential + compute.
#pragma once
#include "potential.h"
#include <memory>
#include <vector>

class Force
{
public:
  // factory keyed on the first token of the potential file (force.cu:75-218); only the potentials
  // libb200md implements are accepted
  void parse_potential(const char* file_potential, const int num_atoms);
  // Force::compute, force.cu:771-985: wrap positions, zero the outputs, run the potential
  void compute(
    Box& box, GPU_Vector<double>& position_per_atom, GPU_Vector<int>& type,
    GPU_Vector<double>& potential_per_atom, GPU_Vector<double>& force_per_atom,
    GPU_Vector<double>& virial_per_atom);
  // compute_hnemd (Force::set_hnemd_parameters, force.cu:341-360): every following compute adds the
  // driving force W_i^T fe and removes the net force; finalize() switches it off again after a run
  // (Force::finalize, force.cu:335-339)
  void set_hnemd(const double fe[3]);
  void finalize() { hnemd_ = false; }
  bool hnemd_on() const { return hnemd_; }
  std::vector<std::unique_ptr<Potential>> potentials;

private:
  bool zero_first_ = true; // false when the single potential overwrites its outputs (NEP_B200)
  bool hnemd_ = false;
  double fe_[3] = {0.0, 0.0, 0.0};
  GPU_Vector<char> drive_scratch_; // b200md_hnemd_drive_scratch_bytes, allocated once
};

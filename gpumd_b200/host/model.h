// model.h -- Box / Atom / Group with the members the hot path touches
// (src/model/box.cuh:18-35, src/model/atom.cuh:21-52, src/model/group.cuh:20-37).
#pragma once
#include "gpu_vector.h"
#include <string>
#include <vector>

class Box
{
public:
  int pbc_x = 1, pbc_y = 1, pbc_z = 1;
  double cpu_h[18] = {0}; // [0..8] row-major (lattice vectors are columns), [9..17] inverse
  double get_volume() const
  {
    const double* h = cpu_h;
    const double v = h[0] * (h[4] * h[8] - h[5] * h[7]) + h[1] * (h[5] * h[6] - h[3] * h[8]) +
                     h[2] * (h[3] * h[7] - h[4] * h[6]);
    return v < 0 ? -v : v;
  }
  // Box::get_inverse, src/model/box.cu:26-60: cpu_h[9..17] = inverse of cpu_h[0..8]
  void get_inverse()
  {
    double* h = cpu_h;
    h[9] = h[4] * h[8] - h[5] * h[7];
    h[10] = h[2] * h[7] - h[1] * h[8];
    h[11] = h[1] * h[5] - h[2] * h[4];
    h[12] = h[5] * h[6] - h[3] * h[8];
    h[13] = h[0] * h[8] - h[2] * h[6];
    h[14] = h[2] * h[3] - h[0] * h[5];
    h[15] = h[3] * h[7] - h[4] * h[6];
    h[16] = h[1] * h[6] - h[0] * h[7];
    h[17] = h[0] * h[4] - h[1] * h[3];
    const double det = h[0] * h[9] + h[1] * h[12] + h[2] * h[15];
    for (int k = 9; k < 18; ++k)
      h[k] /= det;
  }
  void pbc(int out[3]) const
  {
    out[0] = pbc_x;
    out[1] = pbc_y;
    out[2] = pbc_z;
  }
};

class Group
{
public:
  int number = 0;             // number of groups of this grouping method
  std::vector<int> cpu_label; // group label of every atom (group.cuh:25)
  std::vector<int> cpu_size;  // atoms per group
  std::vector<int> cpu_size_sum; // atoms in the groups before each group (group.cu:50-56)
  std::vector<int> contents;  // atom indices sorted by group, then by index (Group::find_contents,
                              // group.cu:58-70)
  GPU_Vector<int> label;      // device copy of cpu_label
};

class Atom
{
public:
  int number_of_atoms = 0;
  std::vector<int> cpu_type;
  std::vector<double> cpu_mass, cpu_position_per_atom, cpu_velocity_per_atom;
  std::vector<std::string> cpu_atom_symbol;
  GPU_Vector<int> type;
  GPU_Vector<double> mass, position_per_atom, velocity_per_atom, force_per_atom, virial_per_atom,
    potential_per_atom;
};

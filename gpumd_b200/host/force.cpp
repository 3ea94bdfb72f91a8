#include "force.h"
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <string>

void Force::parse_potential(const char* file_potential, const int num_atoms)
{
  std::ifstream in(file_potential);
  if (!in.is_open()) {
    fprintf(stderr, "Input Error:\n    Failed to open %s.\n", file_potential);
    exit(1);
  }
  std::string name;
  in >> name;
  in.close();
  potentials.clear();
  zero_first_ = true;
  if (name.rfind("nep", 0) == 0) {
    NEP_B200* nep = new NEP_B200(file_potential, num_atoms);
    nep->set_accumulate(false); // the only potential: store instead of += and skip the zeroing pass
    zero_first_ = false;
    potentials.emplace_back(nep);
  } else if (name == "lj") {
    potentials.emplace_back(new LJ_B200(file_potential, num_atoms));
  } else if (name == "tersoff_1989") {
    potentials.emplace_back(new Tersoff1989_B200(file_potential, num_atoms));
  } else if (name == "eam_zhou_2004" || name == "eam_dai_2006") {
    potentials.emplace_back(new EAM_B200(file_potential, num_atoms));
  } else {
    fprintf(stderr, "Input Error:\n    illegal potential model '%s' for the b200md backend.\n",
            name.c_str());
    exit(1);
  }
  potentials[0]->N1 = 0;
  potentials[0]->N2 = num_atoms;
}

void Force::compute(
  Box& box, GPU_Vector<double>& position_per_atom, GPU_Vector<int>& type,
  GPU_Vector<double>& potential_per_atom, GPU_Vector<double>& force_per_atom,
  GPU_Vector<double>& virial_per_atom)
{
  const int n = (int)type.size();
  int pbc[3];
  b2h_pbc(box, pbc);
  if (b200md_apply_pbc(n, box.cpu_h, pbc, position_per_atom.data(), nullptr) != B200MD_OK)
    b2h_fail("Force::compute (apply_pbc)");
  if (zero_first_ &&
      b200md_zero_properties(
        n, potential_per_atom.data(), force_per_atom.data(), virial_per_atom.data(), nullptr) !=
        B200MD_OK)
    b2h_fail("Force::compute (zero)");
  potentials[0]->compute(
    box, type, position_per_atom, potential_per_atom, force_per_atom, virial_per_atom);
  if (hnemd_) { // force.cu:857-897, after the potential has stored or accumulated its outputs
    const size_t need = (size_t)b200md_hnemd_drive_scratch_bytes(n);
    if (drive_scratch_.size() < need)
      drive_scratch_.resize(need, 0); // the ticket starts at zero
    if (b200md_hnemd_drive(n, n, fe_, virial_per_atom.data(), force_per_atom.data(),
                           drive_scratch_.data(), nullptr) != B200MD_OK)
      b2h_fail("Force::compute (HNEMD driving force)");
  }
}

void Force::set_hnemd(const double fe[3])
{
  hnemd_ = true;
  for (int d = 0; d < 3; ++d)
    fe_[d] = fe[d];
}

#include "minimize.h"
#include <cstdio>

Minimizer_B200::Minimizer_B200(
  int method, int number_of_atoms, int number_of_steps, double force_tolerance, int box_change,
  int hydrostatic)
  : method_(method), n_(number_of_atoms), steps_(number_of_steps), box_change_(box_change),
    tol_(force_tolerance)
{
  if (method == 0) {
    position_trial_.resize((size_t)3 * number_of_atoms);
    force_trial_.resize((size_t)3 * number_of_atoms);
    potential_trial_.resize((size_t)number_of_atoms);
  }
  if (b200md_minimizer_create(
        method, number_of_atoms, force_tolerance, number_of_steps, box_change, hydrostatic, &p_) !=
      B200MD_OK)
    b2h_fail("Minimizer (create)");
}

Minimizer_B200::~Minimizer_B200() { b200md_minimizer_destroy(p_); }

void Minimizer_B200::compute(Force& force, Box& box, Atom& atom, const int* d_label, int fixed_group)
{
  if (method_ == 0)
    compute_sd(force, box, atom, d_label, fixed_group);
  else
    compute_fire(force, box, atom);
}

// minimizer_sd.cu:70-169
void Minimizer_B200::compute_sd(Force& force, Box& box, Atom& atom, const int* d_label, int fixed_group)
{
  force.compute(box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
                atom.virial_per_atom);
  const int base = steps_ >= 10 ? steps_ / 10 : 1;
  double rec[B200MD_MIN_RECORD];
  printf("\nEnergy minimization started.\n");
  if (b200md_minimizer_sd_begin(p_, n_, atom.position_per_atom.data(), atom.force_per_atom.data(),
                                atom.potential_per_atom.data(), position_trial_.data(), force_trial_.data(),
                                potential_trial_.data(), d_label, fixed_group, rec, nullptr) != B200MD_OK)
    b2h_fail("Minimizer_SD (begin)");
  for (int step = 0; step < steps_; ++step) {
    if (rec[B200MD_MIN_CONVERGED] != 0.0) {
      printf("    step %d: f_max = %g eV/A.\n", step, rec[B200MD_MIN_FMAX]);
      break;
    }
    const double force_max = rec[B200MD_MIN_FMAX];
    // the virial of the trial evaluation overwrites the atoms', as in the reference
    force.compute(box, position_trial_, atom.type, potential_trial_, force_trial_, atom.virial_per_atom);
    if (b200md_minimizer_sd_step(p_, n_, atom.position_per_atom.data(), atom.force_per_atom.data(),
                                 atom.potential_per_atom.data(), position_trial_.data(), force_trial_.data(),
                                potential_trial_.data(), d_label, fixed_group, rec, nullptr) != B200MD_OK)
      b2h_fail("Minimizer_SD (step)");
    const double u = rec[B200MD_MIN_USMALLER];
    if (rec[B200MD_MIN_STEP] < 1e-8) { // MIN_POSITION_STEP, minimizer_sd.cu:25
      printf("    step %d: total_potential = %.10f eV, f_max = %.10f eV/A.\n", step + 1, u, force_max);
      printf("    Position step is 0, SD minimizer can't find a better solution\n");
      break;
    }
    if (step == 0)
      printf("    step 0: total_potential = %.10f eV, f_max = %.10f eV/A.\n", u, force_max);
    if ((step + 1) % base == 0)
      printf("    step %d: total_potential = %.10f eV, f_max = %.10f eV/A.\n", step + 1, u, force_max);
  }
  printf("Energy minimization finished.\n");
}

// minimizer_fire.cu:108-180 and minimizer_fire_box_change.cu:239-406
void Minimizer_B200::compute_fire(Force& force, Box& box, Atom& atom)
{
  const int base = steps_ >= 10 ? steps_ / 10 : 1;
  double rec[B200MD_MIN_RECORD];
  printf(box_change_ ? "\nEnergy minimization with changed box started.\n" : "\nEnergy minimization started.\n");
  for (int step = 0; step < steps_; ++step) {
    force.compute(box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
                  atom.virial_per_atom);
    if (b200md_minimizer_fire_step(p_, n_, box.cpu_h, atom.position_per_atom.data(), atom.force_per_atom.data(),
                                   atom.potential_per_atom.data(), atom.virial_per_atom.data(), rec,
                                   nullptr) != B200MD_OK)
      b2h_fail("Minimizer_FIRE (step)");
    if (box_change_)
      box.get_inverse();
    const bool converged = rec[B200MD_MIN_CONVERGED] != 0.0;
    if (step == 0 || (step + 1) % base == 0 || converged) {
      if (box_change_)
        printf("    step %d: total_potential = %.10f eV, f_max_atom = %.10f eV/A, pressure = %.6f GPa.\n",
               step == 0 ? 0 : step + 1, rec[B200MD_MIN_U], rec[B200MD_MIN_FMAX], rec[B200MD_MIN_PRESSURE]);
      else
        printf("    step %d: total_potential = %.10f eV, f_max = %.10f eV/A.\n", step == 0 ? 0 : step + 1,
               rec[B200MD_MIN_U], rec[B200MD_MIN_FMAX]);
      if (converged) {
        if (box_change_)
          printf("  Converged! f_max_atom = %.2e < %.2e AND max_stress = %.2e GPa < %.2e GPa\n",
                 rec[B200MD_MIN_FMAX], tol_, rec[B200MD_MIN_STRESS], 1e-4);
        break;
      }
    }
  }
  printf(box_change_ ? "Energy minimization finished.\n\n" : "Energy minimization finished.\n");
}

// minimize.h -- the minimizers behind the `minimize` keyword (src/minimize/minimize.cu:32-156) on
// libb200md's b200md_minimizer: the reference's Minimizer_SD, Minimizer_FIRE and Minimizer_FIRE_Box_Change
// loops with the force evaluation through Force::compute, every other step on the device and one record
// read per iteration.  The progress lines are the reference's, character for character.
#pragma once
#include "force.h"

class Minimizer_B200
{
public:
  // method 0 sd, 1 fire; box_change / hydrostatic for fire only
  Minimizer_B200(
    int method, int number_of_atoms, int number_of_steps, double force_tolerance, int box_change,
    int hydrostatic);
  ~Minimizer_B200();
  // Minimizer::compute (minimizer.cuh:52-57).  SD keeps the atoms of label fixed_group in place (d_label:
  // the device labels of the fixed grouping method, NULL with fixed_group -1); FIRE ignores them, as the
  // reference builds it with fixed group -1 (minimize.cu:126,142).  Box change updates box.cpu_h.
  void compute(Force& force, Box& box, Atom& atom, const int* d_label, int fixed_group);

private:
  void compute_sd(Force& force, Box& box, Atom& atom, const int* d_label, int fixed_group);
  void compute_fire(Force& force, Box& box, Atom& atom);
  b200md_minimizer* p_ = nullptr;
  GPU_Vector<double> position_trial_, force_trial_, potential_trial_; // SD's _temp vectors, minimizer.cuh:38-40
  int method_, n_, steps_, box_change_;
  double tol_;
};

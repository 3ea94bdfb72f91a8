// phonon.h -- the `compute_phonon` keyword (src/phonon/hessian.cu) on libb200md's b200md_phonon: the force
// constants from 6 * num_basis force calls through Force::compute, D(k) and the eigensolver on the device, and
// the reference's kpoints.in parsing, prints and output files (omega2.out and D.out, or eigenvector.out for a
// single k-point).
#pragma once
#include "driver.h"
#include "force.h"

class Hessian_B200
{
public:
  // Hessian::parse (hessian.cu:494-507)
  void parse(const std::vector<std::string>& t);
  // Hessian::compute (hessian.cu:65-81) at the current positions and box; cxyz: the replicate factors
  void compute(Force& force, Box& box, Atom& atom, const int cxyz[3]);

private:
  double displacement_ = 0.0;
};

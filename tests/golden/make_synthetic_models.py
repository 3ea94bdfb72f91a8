#!/usr/bin/env python
"""Synthetic NEP model files for code paths no shipped fixture reaches (random but fixed parameters;
physics-free, only the arithmetic matters):

  nep_synth_50types.txt          50 species -- more than the shared-memory radial accumulators can hold, the
                                 situation of the reference's NEP89 model (potentials/nep/nep89_20250409, 89
                                 species, 8 MB).  Global cutoffs, so the reference's own NEP_CPU reads it.
  nep_synth_pertype_cutoff.txt   3 species with the `cutoff` line in its 2*Nt+2 form (nep.cu:197-237).

One- and two-species models, for the few-species kernels (b2_nep_radial.cuh, b2_nep_angular.cuh):

  nep_synth_2sp_nep5_flexzbl.txt   nep5_zbl: per-species bias, flexible ZBL table; K1 = 13/13, l_max 4 2 1
  nep_synth_2sp_typewise_zbl.txt   nep4_zbl: universal ZBL with the typewise cutoff (`zbl 1.0 2.2 0.7`); Li/Si,
                                   whose covalent radii give the three pairs outer cutoffs of 2.2 (capped),
                                   2.09 and 1.94 A
  nep_synth_2sp_pertype_cut.txt    nep4, `cutoff 5.0 4.0 4.2 3.4`: three distinct radial and angular pair
                                   cutoffs (5.0 / 4.6 / 4.2 and 4.0 / 3.7 / 3.4)
  nep_synth_1sp_zbl_k17.txt        nep4_zbl universal (`zbl 1.0 2.25`: cutoffs exact in float), K1 = 17/17
  nep_synth_1sp_nep5.txt           nep5, K1 = 9/13, 4- and 5-body terms
  nep_synth_2sp_namax17.txt        n_max 5 17, K1A = 17, l_max 4 2 0, 8 neurons: the angular force kernel's
                                   per-thread weight rows exceed 200 KB per 128 threads (n_max_angular >= 16),
                                   so it runs in 64-thread blocks; with the tensor-core hidden layer the
                                   angular descriptor kernel stages 90 descriptors per thread plus the
                                   coefficient table, 51 840 B > 48 KB.  Among the models whose hidden layer
                                   fits the tensor cores (D = 96 at most here), that staging exceeds 48 KB only
                                   for n_max_angular >= 17 with l_max 4 2 0 and K1A = 17.

All global-cutoff models above are read by the reference's NEP_CPU as they are: its syntax differs from the
GPU code's only in the typewise ZBL factor (on the `cutoff` line there), and typewise ZBL is pinned to the
reference GPU code instead (NEP_CPU uses rc_inner = rc_outer / 2 for it, nep.cu uses 0).

File layout as NEP::NEP reads it (nep.cu:88-420): header line, optional `zbl` line, `cutoff` ... `ANN` lines,
ANN parameters per type (w0[nneu][dim], b0[nneu], w1[nneu], and for NEP5 the per-type bias), the common bias,
c_radial then c_angular in the order [(n*(K+1)+k)*Nt^2 + t1*Nt + t2], q_scaler[dim], and for flexible ZBL
10 numbers per unordered type pair t1 <= t2 (rc_inner, rc_outer, then four (a, b) of phi = sum a exp(-b x)).

usage: python tests/golden/make_synthetic_models.py   (writes next to itself)
"""
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ELEMENTS = ("H He Li Be B C N O F Ne Na Mg Al Si P S Cl Ar K Ca Sc Ti V Cr Mn Fe Co Ni Cu Zn Ga Ge As Se Br Kr Rb "
            "Sr Y Zr Nb Mo Tc Ru Rh Pd Ag Cd In Sn").split()


# the universal ZBL screening function's (a, b) pairs, which the flexible tables perturb
ZBL_PHI = (0.18175, 3.1998, 0.50986, 0.94229, 0.28022, 0.4029, 0.02817, 0.20162)
# the one- and two-species models are exercised on fcc a = 3.1 A: up to ~45 neighbours within 4 A
FEW = "100 60"


def write(path, symbols, cutoff_line, n_max, basis, l_max, nneu, seed, head="nep4", zbl_line=None, f32=False):
    """f32: write every parameter as the exact decimal value of its float32 rounding, so that a reader that
    parses it in double (the reference's NEP_CPU) and one that parses it in float (the GPU code) hold the same
    number.  The ZBL exponents b * r / a reach ~50 at the shortest pairs, which turns the 3e-8 relative
    rounding of a parameter into 1e-6 of a pair force."""
    rng = np.random.default_rng(seed)
    version = 5 if head.startswith("nep5") else 4
    nt = len(symbols)
    nr1, na1 = n_max[0] + 1, n_max[1] + 1
    kr1, ka1 = basis[0] + 1, basis[1] + 1
    num_l = l_max[0] + (1 if l_max[1] else 0) + (1 if l_max[2] else 0)
    dim = nr1 + na1 * num_l
    vals = []
    for _ in range(nt):
        vals += list(rng.normal(0.0, 0.4, nneu * dim))   # w0
        vals += list(rng.normal(0.0, 0.3, nneu))         # b0
        vals += list(rng.normal(0.0, 0.5, nneu))         # w1
        if version == 5:
            vals.append(rng.normal(0.0, 1.0))            # per-type bias
    vals.append(rng.normal(0.0, 1.0))                    # b1
    vals += list(rng.normal(0.0, 0.3, nt * nt * nr1 * kr1))
    vals += list(rng.normal(0.0, 0.3, nt * nt * na1 * ka1))
    vals += list(rng.uniform(0.05, 0.6, dim))            # q_scaler
    if zbl_line == "zbl 0 0":                            # flexible ZBL table
        for _ in range(nt * (nt + 1) // 2):
            vals += [rng.uniform(0.8, 1.2), rng.uniform(1.9, 2.4)]
            vals += list(np.array(ZBL_PHI) * rng.uniform(0.8, 1.2, 8))
    with open(path, "w") as f:
        f.write("%s %d %s\n" % (head, nt, " ".join(symbols)))
        if zbl_line:
            f.write(zbl_line + "\n")
        f.write(cutoff_line + "\n")
        f.write("n_max %d %d\nbasis_size %d %d\nl_max %d %d %d\nANN %d 0\n" % (*n_max, *basis, *l_max, nneu))
        for v in vals:
            f.write(("%r\n" % float(np.float32(v))) if f32 else ("%.7e\n" % v))
    print(path.name, nt, "types, dim", dim, len(vals), "parameters,", path.stat().st_size // 1024, "KB")


write(HERE / "nep_synth_50types.txt", ELEMENTS[:50], "cutoff 5 4 80 40", (1, 1), (3, 3), (4, 2, 1), 4, seed=11)
write(HERE / "nep_synth_pertype_cutoff.txt", ["Cu", "O", "H"], "cutoff 5.0 4.0 4.4 3.6 3.8 3.2 80 40",
      (3, 2), (6, 5), (4, 2, 0), 10, seed=12)
write(HERE / "nep_synth_2sp_nep5_flexzbl.txt", ["Mo", "Ta"], f"cutoff 5 4 {FEW}", (5, 4), (12, 12), (4, 2, 1), 8,
      seed=13, head="nep5_zbl", zbl_line="zbl 0 0", f32=True)
write(HERE / "nep_synth_2sp_typewise_zbl.txt", ["Li", "Si"], f"cutoff 5 4 {FEW}", (4, 3), (6, 5), (4, 2, 0), 8,
      seed=14, head="nep4_zbl", zbl_line="zbl 1.0 2.2 0.7", f32=True)
write(HERE / "nep_synth_2sp_pertype_cut.txt", ["Cu", "O"], f"cutoff 5.0 4.0 4.2 3.4 {FEW}", (4, 4), (8, 6),
      (4, 2, 1), 8, seed=15, f32=True)
write(HERE / "nep_synth_1sp_zbl_k17.txt", ["Si"], f"cutoff 5 4 {FEW}", (4, 4), (16, 16), (4, 2, 0), 8, seed=16,
      head="nep4_zbl", zbl_line="zbl 1.0 2.25", f32=True)
write(HERE / "nep_synth_1sp_nep5.txt", ["W"], f"cutoff 5 4 {FEW}", (6, 5), (7, 12), (4, 2, 1), 8, seed=17,
      head="nep5", f32=True)
write(HERE / "nep_synth_2sp_namax17.txt", ["Al", "Ni"], f"cutoff 5 4 {FEW}", (5, 17), (6, 16), (4, 2, 0), 8,
      seed=18, f32=True)

#!/usr/bin/env python
"""Run the UNMODIFIED reference gpumd (oracle/_ref/gpumd_ref, built by oracle/Makefile.gpumd_ref)
on the GPU box, on inputs written by our own generators, and collect
  (1) single-point E / per-atom force / virial dumps  -> tests/golden/refgpu_*.npz candidates
  (2) short NVE thermo trajectories from given velocities
  (3) its "Speed of this run" line at the BASELINE sizes (the reference-GPU bar, BASELINE.md 3.2).
Outputs go to refgpu_out/.  Baseline/oracle infrastructure only -- never on the product path.

    python scripts/run_reference_gpumd.py [--skip-speed]
"""
import argparse
import json
import re
import shutil
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from gpumd_b200.structures import (fcc, init_velocities, nep_type_order, read_xyz,  # noqa: E402
                                   rocksalt_pbte, write_xyz)

GOLDEN = ROOT / "tests" / "golden"
BIN = ROOT / "oracle" / "_ref" / "gpumd_ref"
OUT = ROOT / "refgpu_out"


# the direct-NEMD cases; tests/test_gpu_nemd.py runs the same inputs through the b200md driver
NEMD_GRAPHENE_RUN = ("ensemble nvt_ber 300 300 100\nfix 0\ntime_step 1\ndump_thermo 10\nrun 200\n"
                     "ensemble heat_{kind} 300 100 10 1 8\nfix 0\ndump_thermo 100\n"
                     "compute 0 10 10 temperature potential force virial jp jk momentum\n"
                     "compute_shc 2 100 1 200 400.0 group 0 4\nrun 600\n")
NEMD_PBTE_RUN = ("ensemble nvt_ber 300 300 100\ntime_step 1\ndump_thermo 10\nrun 100\n"
                 "ensemble heat_lan 300 100 20 2 5\nfix 0\nmove 1 0 0.001 0\n"
                 "compute 0 10 20 temperature jp jk\nrun 600\n")

# time correlations: the graphene sheet (FP64 Tersoff) after a short nvt_ber run, and NEP Si (FP32 force
# path) from the reference's silicon_liquid/restart1.xyz; tests/test_gpu_correlation.py runs the same inputs
# through the b200md driver
CORR_GRAPHENE_PRE = "ensemble nvt_ber 300 300 100\ntime_step 1\nrun 200\nensemble nve\n"
CORR_GRAPHENE_RUNS = {
    "dos": "compute_dos 5 100 400.0\nrun 1000\n",
    "dos_groups": "compute_dos 5 100 400.0 group 0 -1 num_dos_points 150\nrun 1000\n",
    "sdc_msd": "compute_sdc 2 100 group 0 3\ncompute_msd 2 100 all_groups 0 save_every 500\nrun 1000\n",
}
CORR_SI_RUN = "time_step 2\nensemble nve\ncompute_sdc 2 100\ncompute_msd 2 100 save_every 300\nrun 400\n"


# energy minimization: `minimize ...` followed by the single-point tail; tests/test_gpu_minimize.py runs the
# same inputs through the b200md driver.  case: (structure, symbols (None: the NEP file's order), potential
# file, lines before `minimize` and the `minimize` line, head before `potential`, model.xyz to copy)
MIN_TAIL = "velocity 1\nensemble nve\ntime_step 0\ndump_xyz 1 dump.xyz precision double force\nrun 1\n"


def _min_si(group=False):
    from gpumd_b200.structures import diamond
    s = diamond(4, a=5.431, rattle=0.05, seed=31)  # 512 atoms
    if group:  # group 0: every fourth atom
        s["group"] = (np.arange(s["type"].shape[0]) % 4 != 0).astype(np.int32)
    return s


def _min_pbte():
    s = rocksalt_pbte(4, rattle=0.03, seed=32)  # 512 atoms, strained by -2 %
    return dict(s, h=s["h"] * 0.98, pos=s["pos"] * 0.98)


MIN_CASES = {
    "min_si_sd": (_min_si, ["Si"], "tersoff_Si_1989.txt", "minimize sd 1.0e-4 1000\n", "", None),
    "min_si_sd_fix": (lambda: _min_si(True), ["Si"], "tersoff_Si_1989.txt", "fix 0\nminimize sd 1.0e-4 1000\n",
                      "", None),
    "min_si_fire": (_min_si, ["Si"], "tersoff_Si_1989.txt", "minimize fire 1.0e-4 1000\n", "", None),
    "min_si_fire_fix": (lambda: _min_si(True), ["Si"], "tersoff_Si_1989.txt",
                        "fix 0\nminimize fire 1.0e-4 1000\n", "", None),
    # 50 iterations: further on this rattled, compressed cell rearranges into a much denser structure (about
    # 0.8 eV/atom lower after 1000 iterations, in the reference too), where FP32 rounding decides the path
    "min_pbte_fire_box": (_min_pbte, None, "nep_PbTe.txt", "minimize fire 1.0e-4 50 1\n", "", None),
    "min_pbte_fire_box_hydro": (_min_pbte, None, "nep_PbTe.txt", "minimize fire 1.0e-4 50 1 1\n", "", None),
    "min_lj_fire": (lambda: fcc(6, 5.26, rattle=0.1, seed=33), ["Ar"], "lj_Ar_10A.txt",
                    "minimize fire 1.0e-4 1000\n", "", None),
    "min_eam_sd": (lambda: fcc(7, 3.615, rattle=0.05, seed=34, symbols=("Cu",)), ["Cu"], "eam_Cu_Zhou_2004.txt",
                   "minimize sd 1.0e-4 1000\n", "", None),
    # the reference's tests/gpumd/silicon_dispersion recipe (its two-atom cell, replicated 6 x 6 x 6)
    "min_si_dispersion": (None, ["Si"], "tersoff_Si_1989.txt", "minimize sd 1.0e-6 10000\n", "replicate 6 6 6\n",
                          GOLDEN / "silicon_dispersion_model.xyz"),
}


# phonons: `compute_phonon` at parse time (after `minimize` for silicon_dispersion); tests/test_gpu_phonon.py runs
# the same inputs through the b200md driver.  case: (structure of the replicated cell, or None with model_file;
# symbols (None: the NEP file's order); potential file; `replicate` line; lines after `potential`; model.xyz to
# copy; kpoints.in; whether D.out is kept (the cells of at most two atoms: larger ones exceed 1 MB))
FCC_PATH = "0 0 0 G\n0.5 0 0.5 X\n0.375 0.375 0.75 K\n0 0 0 G\n0.5 0.5 0.5 L\n"


def fcc_primitive(a, symbols, basis=((0.0, 0.0, 0.0),)):
    """The primitive fcc cell (lattice vectors a/2 (0,1,1), (1,0,1), (1,1,0)) with atoms at the given
    fractions of the cubic edge a."""
    h = 0.5 * a * np.array([[0, 1, 1], [1, 0, 1], [1, 1, 0]], dtype=float)  # columns
    pos = a * np.array(basis, dtype=float).T
    from gpumd_b200.structures import MASS
    return dict(h=h.reshape(9), pbc=np.array([1, 1, 1]), pos=pos, type=np.arange(len(basis), dtype=np.int32),
                mass=np.array([MASS[symbols[t]] for t in range(len(basis))]))


def fcc_two_atom(a, symbol):
    """fcc in its two-atom tetragonal cell: lattice vectors (a/2)(1,1,0), (a/2)(-1,1,0), (0,0,a), atoms at 0 and
    (a/2)(1,0,1) (the reference reads no model of fewer than two atoms)."""
    from gpumd_b200.structures import MASS
    h = np.array([[0.5 * a, -0.5 * a, 0.0], [0.5 * a, 0.5 * a, 0.0], [0.0, 0.0, a]])  # columns
    pos = np.array([[0.0, 0.5 * a], [0.0, 0.0], [0.0, 0.5 * a]])
    return dict(h=h.reshape(9), pbc=np.array([1, 1, 1]), pos=pos, type=np.zeros(2, np.int32),
                mass=np.full(2, MASS[symbol]))


def _zincblende_sic():
    from gpumd_b200.structures import diamond
    s = diamond(1, a=4.36)
    s["type"] = np.array([0, 0, 0, 0, 1, 1, 1, 1], np.int32)
    return s


def _diamond(reps):
    from gpumd_b200.structures import diamond
    return lambda: diamond(reps)


PHONON_CASES = {
    # the reference's tests/gpumd/silicon_dispersion input, exactly
    "phonon_si_dispersion": (None, ["Si"], "tersoff_Si_1989.txt", "replicate 6 6 6\n",
                             "minimize sd 1.0e-6 10000\ncompute_phonon 0.005\n", GOLDEN / "silicon_dispersion_model.xyz",
                             (GOLDEN / "ref_silicon_dispersion_kpoints.in").read_text(), True),
    # two masses, two k-path segments (the '|' header)
    "phonon_sic": (_zincblende_sic, ["Si", "C"], "tersoff_SiC_1989.txt", "replicate 3 3 3\n", "compute_phonon 0.005\n",
                   None, "0 0 0 G\n0.5 0 0.5 X\n\n0.5 0.5 0.5 L\n0 0 0 G\n", False),
    "phonon_pbte": (lambda: fcc_primitive(6.57, ["Te", "Pb"], ((0, 0, 0), (0.5, 0.5, 0.5))), None, "nep_PbTe.txt",
                    "replicate 6 6 6\n", "compute_phonon 0.005\n", None, FCC_PATH, True),
    "phonon_lj": (lambda: fcc_two_atom(5.26, "Ar"), ["Ar"], "lj_Ar_10A.txt", "replicate 8 8 6\n",
                  "compute_phonon 0.005\n", None, "0 0 0 G\n0.5 0 0 X\n0.5 0.5 0.5 R\n", True),
    "phonon_eam": (lambda: fcc_two_atom(3.615, "Cu"), ["Cu"], "eam_Cu_Zhou_2004.txt", "replicate 8 8 6\n",
                   "compute_phonon 0.005\n", None, "0 0 0 G\n0.5 0 0 X\n0.5 0.5 0.5 R\n", True),
    # 16 basis atoms: the reference's per-k-point zheevd branch (more than 10)
    "phonon_si16": (_diamond((2, 1, 1)), ["Si"], "tersoff_Si_1989.txt", "replicate 2 3 3\n", "compute_phonon 0.005\n",
                    None, "0 0 0 G\n0.5 0 0 X\n", False),
    # one k-point: eigenvector.out
    "phonon_gamma": (_diamond(1), ["Si"], "tersoff_Si_1989.txt", "replicate 2 2 2\n", "compute_phonon 0.005\n",
                     None, "0 0 0 G\n", False),
}


def collect_phonon(d, name, keep_d):
    """-> refgpu_out/refgpu_<name>_omega2.out, _D.out.gz, _eigenvector.out (those the run wrote)"""
    if d is None:
        return
    import gzip
    if (d / "omega2.out").exists():
        shutil.copyfile(d / "omega2.out", OUT / f"refgpu_{name}_omega2.out")
    if keep_d and (d / "D.out").exists():
        (OUT / f"refgpu_{name}_D.out.gz").write_bytes(gzip.compress((d / "D.out").read_bytes(), mtime=0))
    if (d / "eigenvector.out").exists():
        shutil.copyfile(d / "eigenvector.out", OUT / f"refgpu_{name}_eigenvector.out")
    (OUT / f"refgpu_{name}_stdout.txt").write_text((d / "stdout.txt").read_text())


def min_progress(stdout):
    """The minimizer's progress lines of a gpumd / b200md stdout."""
    return [ln for ln in stdout.splitlines() if ln.startswith(("    step ", "    Position step", "  Converged!"))]


def write_model(path, s, symbols, vel=None):
    write_xyz(path, s, symbols, vel)


ONLY = None  # --only REGEX: run just the matching cases


def run_case(name, s, symbols, potential, run_in, vel=None, timeout=900, gpus=1, model_file=None, head="",
             files=None):
    """gpus > 1: that many visible devices -> the reference takes its NEP_MULTIGPU path
    (src/force/force.cu:139-160); skipped when the box has fewer.  model_file: copy this model.xyz
    instead of writing one from s.  head: keywords before the `potential` line (replicate).  files: name ->
    text of further input files (kpoints.in)."""
    if ONLY and not re.search(ONLY, name):
        return None, None
    import os
    env = dict(os.environ)
    if gpus > 1:
        try:
            import torch
            have = torch.cuda.device_count()
        except Exception:
            have = 1
        if have < gpus:
            print(f"skip {name}: needs {gpus} GPUs, box has {have}")
            return None, None
    env["CUDA_VISIBLE_DEVICES"] = ",".join(str(k) for k in range(gpus))
    d = OUT / name
    shutil.rmtree(d, ignore_errors=True)
    d.mkdir(parents=True)
    shutil.copyfile(potential, d / "potential.txt")
    if model_file is None:
        write_model(d / "model.xyz", s, symbols, vel)
    else:
        shutil.copyfile(model_file, d / "model.xyz")
    (d / "run.in").write_text(head + "potential potential.txt\n" + run_in)
    for fname, text in (files or {}).items():
        (d / fname).write_text(text)
    t0 = time.time()
    r = subprocess.run([str(BIN)], cwd=d, capture_output=True, text=True, timeout=timeout, env=env)
    wall = time.time() - t0
    (d / "stdout.txt").write_text(r.stdout[-20000:] + "\n--- stderr ---\n" + r.stderr[-5000:])
    speed = re.findall(r"Speed of this run = ([0-9.eE+-]+) atom\*step/second", r.stdout)
    info = {"case": name, "returncode": r.returncode, "wall_s": wall,
            "speed_atom_step_per_s": [float(x) for x in speed],
            "n_atoms": int(s["type"].shape[0]) if s is not None else None}
    (d / "model.xyz").unlink()  # large; regenerated from the seeded generators
    return d, info


def collect_single_point(d, s, symbols):
    if d is None:
        return
    out = read_xyz(d / "dump.xyz", symbols)
    np.savez_compressed(
        d / "single_point.npz", type=s["type"], h=s["h"], pbc=s["pbc"], pos=s["pos"],
        energy=out["energy"], virial=out.get("virial"), force=out["forces"],
        wrapped_pos=out["pos"])
    (d / "dump.xyz").unlink()


def collect_minimize(d, name):
    """-> refgpu_out/refgpu_<name>_progress.txt (the progress lines) and refgpu_<name>_dump.xyz.gz"""
    if d is None:
        return
    import gzip
    text = (d / "stdout.txt").read_text()
    (OUT / f"refgpu_{name}_progress.txt").write_text("\n".join(min_progress(text)) + "\n")
    (OUT / f"refgpu_{name}_dump.xyz.gz").write_bytes(gzip.compress((d / "dump.xyz").read_bytes(), mtime=0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-speed", action="store_true")
    ap.add_argument("--only", default=None, help="regex: run only the matching cases")
    args = ap.parse_args()
    global ONLY
    ONLY = args.only
    if not BIN.exists():
        raise SystemExit(f"{BIN} missing: build it with make -C oracle -f Makefile.gpumd_ref")
    OUT.mkdir(parents=True, exist_ok=True)
    infos = []
    sp = "velocity 1\nensemble nve\ntime_step 0\ndump_xyz 1 dump.xyz precision double force\nrun 1\n"

    # ---- (0) energy minimization ----
    for name, (make, symbols, pot, lines, head, model_file) in MIN_CASES.items():
        sym = symbols or nep_type_order(GOLDEN / pot)
        s = make() if make else None
        d, i = run_case(name, s, sym, GOLDEN / pot, lines + MIN_TAIL, model_file=model_file, head=head)
        collect_minimize(d, name); infos.append(i)

    # ---- (0b) phonons ----
    for name, (make, symbols, pot, head, lines, model_file, kpoints, keep_d) in PHONON_CASES.items():
        sym = symbols or nep_type_order(GOLDEN / pot)
        s = make() if make else None
        d, i = run_case(name, s, sym, GOLDEN / pot, lines, model_file=model_file, head=head,
                        files={"kpoints.in": kpoints})
        collect_phonon(d, name, keep_d); infos.append(i)

    # ---- (1) single points on the large-box path ----
    pbte_sym = nep_type_order(GOLDEN / "nep_PbTe.txt")
    s = rocksalt_pbte(12, rattle=0.05, seed=21)  # 13 824 atoms, 78.8 A box
    d, i = run_case("sp_pbte", s, pbte_sym, GOLDEN / "nep_PbTe.txt", sp)
    collect_single_point(d, s, pbte_sym); infos.append(i)

    unep_sym = nep_type_order(GOLDEN / "nep_UNEP_v1.txt")
    s = fcc(12, 3.9, rattle=0.08, seed=22, num_types=16, symbols=unep_sym)  # 6912 atoms, 46.8 A
    d, i = run_case("sp_unep", s, unep_sym, GOLDEN / "nep_UNEP_v1.txt", sp)
    collect_single_point(d, s, unep_sym); infos.append(i)

    s = fcc(14, 5.30, rattle=0.1, seed=23)  # 10 976 Ar atoms, 74.2 A
    d, i = run_case("sp_lj", s, ["Ar"], GOLDEN / "lj_Ar_10A.txt", sp)
    collect_single_point(d, s, ["Ar"]); infos.append(i)

    from gpumd_b200.structures import diamond
    s = diamond(10, a=5.431, rattle=0.08, seed=24)  # 8000 Si atoms, 54.3 A
    d, i = run_case("sp_si", s, ["Si"], GOLDEN / "tersoff_Si_1989.txt", sp)
    collect_single_point(d, s, ["Si"]); infos.append(i)

    s = fcc(10, 3.615, rattle=0.08, seed=25, num_types=3, symbols=["Cu", "Fe", "Ni"])  # 4000 atoms
    d, i = run_case("sp_eam", s, ["Cu", "Fe", "Ni"], GOLDEN / "eam_zhou_2004_CuFeNi.txt", sp)
    collect_single_point(d, s, ["Cu", "Fe", "Ni"]); infos.append(i)

    # one- and two-species synthetic models (tests/golden/make_synthetic_models.py) on the features NEP_CPU
    # cannot pin: typewise ZBL, per-species cutoffs, and NEP5 with flexible ZBL.  fcc a = 3.1 A with the two
    # species drawn i.i.d., 2048 atoms, 24.8 A box
    for name, model in (("sp_typewise_zbl", "nep_synth_2sp_typewise_zbl.txt"),
                        ("sp_pertype_cut", "nep_synth_2sp_pertype_cut.txt"),
                        ("sp_nep5_flexzbl", "nep_synth_2sp_nep5_flexzbl.txt")):
        sym = nep_type_order(GOLDEN / model)
        s = fcc(8, 3.1, rattle=0.15, seed=61, num_types=2, symbols=("Ar", "Ar"))
        d, i = run_case(name, s, sym, GOLDEN / model, sp)
        collect_single_point(d, s, sym); infos.append(i)
    # the same for three and four species: typewise ZBL over Li / Mg / Al / Si, and NEP5 with the six rows of a
    # flexible ZBL table (tests/test_many_species_cpu.py)
    for name, model in (("sp_4sp_typewise_zbl", "nep_synth_4sp_typewise_zbl.txt"),
                        ("sp_3sp_nep5_flexzbl", "nep_synth_3sp_nep5_flexzbl.txt")):
        sym = nep_type_order(GOLDEN / model)
        s = fcc(8, 3.1, rattle=0.15, seed=62, num_types=len(sym), symbols=("Ar",) * len(sym))
        d, i = run_case(name, s, sym, GOLDEN / model, sp)
        collect_single_point(d, s, sym); infos.append(i)

    # LJ / Tersoff / EAM beyond one orthogonal, periodic, few-species crystal (tests/cases_classical.py):
    # per-pair LJ tables in a triclinic box, the Tersoff SiC mixing rules (also with an open direction),
    # Dai-2006, and the power/log embedding branch of Zhou-2004 Cu (a = 3.3 A)
    sys.path.insert(0, str(ROOT / "tests"))
    from cases import shear, slab
    from cases_classical import _sic
    lj3 = ["Ar", "Ne", "Kr"]
    s = shear(fcc(8, 5.30, rattle=0.1, seed=62, num_types=3, symbols=("Ar", "Ar", "Ar")))  # 2048 atoms
    d, i = run_case("sp_lj3_tric", s, lj3, GOLDEN / "lj_synth_3types.txt", sp)
    collect_single_point(d, s, lj3); infos.append(i)
    for name, s in (("sp_sic", _sic(6, 63)), ("sp_sic_slab", slab(_sic(6, 64)))):  # 1728 atoms, 26.2 A
        d, i = run_case(name, s, ["Si", "C"], GOLDEN / "tersoff_SiC_1989.txt", sp)
        collect_single_point(d, s, ["Si", "C"]); infos.append(i)
    s = fcc(8, 3.615, rattle=0.08, seed=65, symbols=("Cu",))  # 2048 atoms
    d, i = run_case("sp_eam_dai", s, ["Cu"], GOLDEN / "eam_Cu_Dai_2006.txt", sp)
    collect_single_point(d, s, ["Cu"]); infos.append(i)
    s = fcc(8, 3.3, rattle=0.08, seed=66, symbols=("Cu",))
    d, i = run_case("sp_eam_cu_compressed", s, ["Cu"], GOLDEN / "eam_Cu_Zhou_2004.txt", sp)
    collect_single_point(d, s, ["Cu"]); infos.append(i)
    s = shear(fcc(8, 3.615, rattle=0.08, seed=67, num_types=3, symbols=["Cu", "Fe", "Ni"]))
    d, i = run_case("sp_eam_alloy_tric", s, ["Cu", "Fe", "Ni"], GOLDEN / "eam_zhou_2004_CuFeNi.txt", sp)
    collect_single_point(d, s, ["Cu", "Fe", "Ni"]); infos.append(i)

    # ---- (2) NVE trajectories from given velocities: thermo.out every 10 steps ----
    md = "ensemble nve\ntime_step {dt}\ndump_thermo 10\nrun {steps}\n"
    s = fcc(10, 3.615, rattle=0.0, seed=1, num_types=3, symbols=["Cu", "Fe", "Ni"])  # 4000 atoms
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("md_eam", s, ["Cu", "Fe", "Ni"], GOLDEN / "eam_zhou_2004_CuFeNi.txt",
                    md.format(dt=1, steps=200), vel)
    infos.append(i)
    s = rocksalt_pbte(20, rattle=0.02, seed=1)  # 64 000 atoms
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("md_pbte", s, pbte_sym, GOLDEN / "nep_PbTe.txt", md.format(dt=1, steps=200), vel)
    infos.append(i)
    # the same start through the reference's multi-GPU path (2 visible devices)
    d, i = run_case("md_pbte_2gpu", s, pbte_sym, GOLDEN / "nep_PbTe.txt", md.format(dt=1, steps=200), vel, gpus=2)
    infos.append(i)
    s = fcc(25, 5.30, rattle=0.0, seed=1)  # 62 500 atoms
    vel = init_velocities(s["mass"], 80.0, seed=42)
    d, i = run_case("md_lj", s, ["Ar"], GOLDEN / "lj_Ar_10A.txt", md.format(dt=5, steps=200), vel)
    infos.append(i)

    s = diamond(20, a=5.431, rattle=0.0, seed=1)  # 64 000 Si atoms
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("md_si", s, ["Si"], GOLDEN / "tersoff_Si_1989.txt", md.format(dt=1, steps=200), vel)
    infos.append(i)

    # NVT from the same start: Nose-Hoover chain and Berendsen (deterministic thermostats)
    s = rocksalt_pbte(20, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    # ... and Bussi-Donadio-Parrinello: the reference binary is built -DDEBUG, i.e. std::mt19937(12345678)
    # Langevin / BAOAB: cuRAND seeded with rand(), which is glibc's first value (1804289383) in a -DDEBUG
    # build when model.xyz carries the velocities; npt_ber: isotropic, 0 GPa, 50 GPa modulus, tau_p 1000
    for name, ens in (("md_pbte_nhc", "nvt_nhc 300 300 100"), ("md_pbte_ber", "nvt_ber 300 300 100"),
                      ("md_pbte_bdp", "nvt_bdp 300 300 100"), ("md_pbte_lan", "nvt_lan 300 300 100"),
                      ("md_pbte_bao", "nvt_bao 300 300 100"), ("md_pbte_npt", "npt_ber 300 300 100 0 50 1000")):
        d, i = run_case(name, s, pbte_sym, GOLDEN / "nep_PbTe.txt",
                        f"ensemble {ens}\ntime_step 1\ndump_thermo 10\nrun 200\n", vel)
        infos.append(i)

    # heat-current autocorrelation: FP64 Tersoff, short run
    s = diamond(10, a=5.431, rattle=0.08, seed=24)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("hac_si", s, ["Si"], GOLDEN / "tersoff_Si_1989.txt",
                    "ensemble nvt_ber 300 300 100\ntime_step 1\nrun 100\nensemble nve\ncompute_hac 2 50 1\nrun 400\n",
                    vel)
    infos.append(i)

    # HNEMD + SHC: the sheet of the reference's own graphene_kappa_hnemd case (FP64 Tersoff), shortened,
    # and PbTe NEP (FP32 force path) with SHC over every group but 0 of four slabs along x
    from gpumd_b200.structures import graphene_sheet
    s = graphene_sheet()  # 40 400 atoms, 9 groups along y
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("hnemd_graphene", s, ["C"], GOLDEN / "Graphene_Lindsay_2010_modified.txt",
                    "ensemble nvt_nhc 300 300 100\ntime_step 1\ndump_thermo 10\ncompute_hnemd 20 0 0.00001 0\n"
                    "compute_shc 1 100 1 200 400.0 group 0 4\nrun 400\n", vel)
    infos.append(i)
    s = rocksalt_pbte(12, rattle=0.02, seed=31)  # 13 824 atoms
    s["group"] = np.minimum((s["pos"][0] / s["h"][0] * 4).astype(np.int32), 3)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("hnemd_pbte", s, pbte_sym, GOLDEN / "nep_PbTe.txt",
                    "ensemble nvt_ber 300 300 100\ntime_step 1\ndump_thermo 10\ncompute_hnemd 10 0.00002 0 0\n"
                    "compute_shc 2 100 0 100 200 group 0 -1\nrun 250\n", vel)
    infos.append(i)

    # direct NEMD: the graphene sheet (FP64 Tersoff) with each heat bath after an nvt_ber run, and PbTe NEP
    # with `fix`, `move` and heat_lan over six slabs along x.  Outputs: thermo.out, compute.out, shc.out
    s = graphene_sheet()
    vel = init_velocities(s["mass"], 300.0, seed=42)
    for kind in ("lan", "nhc", "bdp"):
        d, i = run_case(f"nemd_graphene_{kind}", s, ["C"], GOLDEN / "Graphene_Lindsay_2010_modified.txt",
                        NEMD_GRAPHENE_RUN.format(kind=kind), vel)
        infos.append(i)
    s = rocksalt_pbte(12, rattle=0.02, seed=32)  # 13 824 atoms
    s["group"] = np.minimum((s["pos"][0] / s["h"][0] * 6).astype(np.int32), 5)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    d, i = run_case("nemd_pbte_lan", s, pbte_sym, GOLDEN / "nep_PbTe.txt", NEMD_PBTE_RUN, vel)
    infos.append(i)

    # time correlations (outputs: mvac.out, dos.out, sdc.out, msd.out, msd_step*.out)
    s = graphene_sheet()
    vel = init_velocities(s["mass"], 300.0, seed=42)
    for name, run in CORR_GRAPHENE_RUNS.items():
        d, i = run_case(f"corr_graphene_{name}", s, ["C"], GOLDEN / "Graphene_Lindsay_2010_modified.txt",
                        CORR_GRAPHENE_PRE + run, vel)
        infos.append(i)
    d, i = run_case("corr_si_sdc_msd", None, ["Si"], GOLDEN / "nep_Si_2022_NEP4_3body.txt", CORR_SI_RUN,
                    model_file=GOLDEN / "ref_silicon_liquid_restart1.xyz")
    infos.append(i)

    # radial distribution functions (rdf.out): one static sample of each case of tests/test_gpu_rdf.py at 21
    # and 500 bins, and a 200-step PbTe NVE run sampled every 20 steps -> refgpu_rdf_<case>_<bins>.out.gz,
    # refgpu_rdf_pbte_nve.out.gz
    import gzip
    import rdf_support
    for case, (s, rc, sym, pot) in rdf_support.rdf_cases().items():
        for nb in rdf_support.RDF_BINS:
            d, i = run_case(f"rdf_{case}_{nb}", s, sym, pot, rdf_support.RDF_STATIC.format(rc=rc, nb=nb))
            if d is not None:
                (OUT / f"refgpu_rdf_{case}_{nb}.out.gz").write_bytes(gzip.compress((d / "rdf.out").read_bytes(),
                                                                                   mtime=0))
            infos.append(i)
    s, vel, sym, pot = rdf_support.rdf_nve_case()
    d, i = run_case("rdf_pbte_nve", s, sym, pot, rdf_support.RDF_NVE_RUN, vel)
    if d is not None:
        (OUT / "refgpu_rdf_pbte_nve.out.gz").write_bytes(gzip.compress((d / "rdf.out").read_bytes(), mtime=0))
    infos.append(i)

    # ---- (3) throughput at the BASELINE sizes ----
    if not args.skip_speed:
        s = rocksalt_pbte(50, rattle=0.02, seed=1)  # C3: 1 000 000 atoms
        vel = init_velocities(s["mass"], 300.0, seed=42)
        d, i = run_case("speed_pbte_1m", s, pbte_sym, GOLDEN / "nep_PbTe.txt",
                        "ensemble nve\ntime_step 1\ndump_thermo 100\nrun 200\n", vel, timeout=1500)
        infos.append(i)
        s = fcc(63, 5.30, rattle=0.0, seed=1)  # C2: 1 000 188 atoms
        vel = init_velocities(s["mass"], 80.0, seed=42)
        d, i = run_case("speed_lj_1m", s, ["Ar"], GOLDEN / "lj_Ar_10A.txt",
                        "ensemble nve\ntime_step 5\ndump_thermo 100\nrun 200\n", vel, timeout=1500)
        infos.append(i)
        s = diamond(63, a=5.431, rattle=0.0, seed=1)  # C5: 2 000 376 Si atoms
        vel = init_velocities(s["mass"], 300.0, seed=42)
        d, i = run_case("speed_si_2m", s, ["Si"], GOLDEN / "tersoff_Si_1989.txt",
                        "ensemble nve\ntime_step 1\ndump_thermo 100\nrun 200\n", vel, timeout=1500)
        infos.append(i)
        s = fcc(63, 3.9, rattle=0.0, seed=7, num_types=16, symbols=unep_sym)  # C4 per-GPU share: 1 000 188 atoms
        vel = init_velocities(s["mass"], 300.0, seed=42)
        d, i = run_case("speed_unep_1m", s, unep_sym, GOLDEN / "nep_UNEP_v1.txt",
                        "ensemble nvt_ber 300 300 100\ntime_step 1\ndump_thermo 100\nrun 100\n", vel,
                        timeout=1500)
        infos.append(i)
    infos = [i for i in infos if i is not None]
    (OUT / "summary.json").write_text(json.dumps(infos, indent=1))
    print(json.dumps(infos, indent=1))


if __name__ == "__main__":
    main()

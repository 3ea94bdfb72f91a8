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


def write_model(path, s, symbols, vel=None):
    write_xyz(path, s, symbols, vel)


ONLY = None  # --only REGEX: run just the matching cases


def run_case(name, s, symbols, potential, run_in, vel=None, timeout=900, gpus=1):
    """gpus > 1: that many visible devices -> the reference takes its NEP_MULTIGPU path
    (src/force/force.cu:139-160); skipped when the box has fewer."""
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
    write_model(d / "model.xyz", s, symbols, vel)
    (d / "run.in").write_text("potential potential.txt\n" + run_in)
    t0 = time.time()
    r = subprocess.run([str(BIN)], cwd=d, capture_output=True, text=True, timeout=timeout, env=env)
    wall = time.time() - t0
    (d / "stdout.txt").write_text(r.stdout[-20000:] + "\n--- stderr ---\n" + r.stderr[-5000:])
    speed = re.findall(r"Speed of this run = ([0-9.eE+-]+) atom\*step/second", r.stdout)
    info = {"case": name, "returncode": r.returncode, "wall_s": wall,
            "speed_atom_step_per_s": [float(x) for x in speed], "n_atoms": int(s["type"].shape[0])}
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

    # ---- (2) NVE trajectories from given velocities: thermo.out every 10 steps ----
    md = "ensemble nve\ntime_step {dt}\ndump_thermo 10\nrun {steps}\n"
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

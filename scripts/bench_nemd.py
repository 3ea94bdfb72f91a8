#!/usr/bin/env python
"""Cost of direct NEMD (heat baths + `compute`) on the GPU.

  (1) CUDA-event times at 1 M atoms in 9 slabs of one heat-bath half step of each kind (source and sink
      are two of the slabs) and of one `compute` sample with all seven quantities, with the bytes each
      moves and the achieved bytes/s;
  (2) a 1 M-atom PbTe NEP run through the `b200md` driver with 9 x-slabs three ways: nvt_ber only,
      heat_lan + `compute 0 10 100 temperature`, and the same input through the reference gpumd
      (oracle/_ref/gpumd_ref, when built).
The card's name and power limit are printed with the numbers.  Output: one JSON line; the run directories
live under a temporary directory.

    python scripts/bench_nemd.py [--atoms-per-side 50] [--steps 1000] [--skip-runs]
"""
import argparse
import json
import re
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
GOLDEN = ROOT / "tests" / "golden"
SLABS = 9


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def time_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernels(n, reps):
    import torch
    from gpumd_b200 import engine
    rng = np.random.default_rng(1)
    atom = engine.Atom(np.zeros(n, np.int32), np.zeros((3, n)), rng.uniform(20, 200, n),
                       rng.normal(size=(3, n)) * 0.05)
    atom.virial_per_atom.copy_(torch.as_tensor(rng.normal(size=9 * n), device="cuda"))
    atom.force_per_atom.copy_(torch.as_tensor(rng.normal(size=3 * n), device="cuda"))
    label = (np.arange(n) * SLABS // n).astype(np.int32)
    m_bath = int(((label == 1) | (label == 8)).sum())
    dt = 1.0 / engine.TIME_UNIT_CONVERSION
    out = {}
    baths = [("heat_lan", engine.Ensemble_HEAT_LAN(label, 1, 8, 300.0, 100.0, 10.0), 1,
              m_bath * (4 + 8 + 6 * 8 + 48 * 2)),  # index, mass, v in / out, XORWOW state in / out
             ("heat_nhc", engine.Ensemble_HEAT_NHC(label, 1, 8, 300.0, 100.0, 10.0, dt), 0,
              m_bath * (2 * 4 + 8 + 3 * 8 + 6 * 8)),  # reduce: index, m, v; scale: index, v in / out
             ("heat_bdp", engine.Ensemble_HEAT_BDP(label, 1, 8, 300.0, 100.0, 10.0), 1,
              m_bath * (2 * 4 + 8 + 3 * 8 + 6 * 8))]
    for name, ens, after, nbytes in baths:
        ms = time_ms(lambda: ens.half(after, atom), reps)
        out[name] = dict(ms=ms, bytes=nbytes, GBps=nbytes / ms / 1e6, bath_atoms=m_bath)
    comp = engine.Compute(label, 1, 1, engine.COMPUTE_QUANTITIES)
    ms = time_ms(lambda: comp.sample(atom), reps)
    comp.take(reps + 1)
    nbytes = n * (4 + 8 * (1 + 3 + 1 + 3 + 9))  # contents, m, v, U, f, W
    out["compute_sample"] = dict(ms=ms, bytes=nbytes, GBps=nbytes / ms / 1e6, groups=SLABS)
    return out


def driver_runs(reps_side, steps):
    from gpumd_b200 import build
    from gpumd_b200.structures import init_velocities, nep_type_order, rocksalt_pbte, write_xyz
    exe = build.build_host()
    ref = ROOT / "oracle" / "_ref" / "gpumd_ref"
    s = rocksalt_pbte(reps_side, rattle=0.02, seed=1)
    s["group"] = np.minimum((s["pos"][0] / s["h"][0] * SLABS).astype(np.int32), SLABS - 1)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    tmp = Path(tempfile.mkdtemp(prefix="bench_nemd_"))
    base = "potential potential.txt\ntime_step 1\nfix 0\n"
    plain = base + "ensemble nvt_ber 300 300 100\n"
    nemd = base + "ensemble heat_lan 300 100 10 1 8\ncompute 0 10 100 temperature\n"
    legs = [("b200md_nvt_ber", exe, plain), ("b200md_heat_lan_compute", exe, nemd)]
    if ref.exists():
        legs.append(("reference_heat_lan_compute", ref, nemd))
    out = {}
    model = tmp / "model.xyz"
    write_xyz(model, s, nep_type_order(GOLDEN / "nep_PbTe.txt"), vel)
    for name, binary, run_in in legs:
        d = tmp / name
        d.mkdir()
        shutil.copyfile(model, d / "model.xyz")
        shutil.copyfile(GOLDEN / "nep_PbTe.txt", d / "potential.txt")
        (d / "run.in").write_text(run_in + f"run {steps}\n")
        r = subprocess.run([str(binary)], cwd=d, capture_output=True, text=True, timeout=3000)
        t = re.findall(r"Time used for this run = ([0-9.eE+-]+) second", r.stdout)
        out[name] = dict(returncode=r.returncode, seconds=float(t[-1]) if t else None,
                         ms_per_step=1e3 * float(t[-1]) / steps if t else None)
        if r.returncode != 0:
            out[name]["stderr"] = r.stderr[-500:]
    shutil.rmtree(tmp, ignore_errors=True)
    return dict(atoms=int(s["type"].shape[0]), steps=steps, runs=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--atoms-per-side", type=int, default=50)  # rocksalt PbTe: 8 x 50^3 = 1 000 000 atoms
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--skip-runs", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the measurement needs the GPU")
    res = dict(card=card(), kernels=kernels(8 * args.atoms_per_side ** 3, args.reps))
    if not args.skip_runs:
        res["driver"] = driver_runs(args.atoms_per_side, args.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Cost of compute_hnemd + compute_shc on the GPU.

  (1) CUDA-event times of the HNEMD drive (b200md_hnemd_drive), the fused heat-current sum
      (b200md_hnemd_sample) and the SHC sample / blocked flush at 1 M atoms, with the bytes each moves
      and the achieved bytes/s;
  (2) a 1 M-atom PbTe nvt_nhc run through the `b200md` driver with `compute_hnemd 1000 ...` and
      `compute_shc 2 250 0 1000 400` over the whole system, the same run without them, and the
      reference gpumd (oracle/_ref/gpumd_ref, when built) on the same inputs.
The card's name and power limit are printed with the numbers.  Outputs: one JSON line, and the run
directories under a temporary directory.

    python scripts/bench_heat_transport.py [--atoms-per-side 50] [--steps 1000] [--skip-runs]
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


def kernels(n, Nc, reps):
    import torch
    from gpumd_b200 import engine
    rng = np.random.default_rng(1)
    atom = engine.Atom(np.zeros(n, np.int32), np.zeros((3, n)), np.ones(n), rng.normal(size=(3, n)))
    atom.virial_per_atom.copy_(torch.as_tensor(rng.normal(size=9 * n), device="cuda"))
    atom.force_per_atom.copy_(torch.as_tensor(rng.normal(size=3 * n), device="cuda"))
    out = {}
    ms = time_ms(lambda: engine.hnemd_drive(n, (0.0, 1e-5, 0.0), atom.virial_per_atom, atom.force_per_atom), reps)
    nbytes = n * (9 * 8 + 3 * 8 * 2 + 3 * 8 * 2)  # drive: W, f in / out; correction: f in / out
    out["drive"] = dict(ms=ms, bytes=nbytes, GBps=nbytes / ms / 1e6)
    h = engine.HNEMD(1000, (0.0, 1e-5, 0.0))
    step = [0]

    def heat():
        h.process(step[0], atom)
        step[0] += 1
    ms = time_ms(heat, reps)
    nbytes = n * (9 + 3) * 8
    out["heat_sum"] = dict(ms=ms, bytes=nbytes, GBps=nbytes / ms / 1e6)
    # SHC: whole system, sample_interval 1; the steady-state cost per sample (gather every sample, one
    # blocked flush every B samples) from the time of 4 flush periods after the first origin
    steps = Nc + 64 * 4
    shc = engine.SHC(1, Nc, 0, 10 ** 7, num_atoms=n)
    for s in range(Nc - 1):
        shc.process(s, atom)
    torch.cuda.synchronize()
    k = [Nc - 1]

    def sample():
        shc.process(k[0], atom)
        k[0] += 1
    ms = time_ms(sample, steps - Nc)
    # per sample: the gather (6 reads + 6 writes) and, amortised, one flush's ring reads: the "now"
    # frames of B origins and the Nc + B - 1 past frames, 3 arrays each, for each of the two halves
    B = 16
    per_flush = 2 * 3 * 8 * n * (B + Nc + B - 1)
    nbytes = 12 * 8 * n + per_flush / B
    out["shc_per_sample"] = dict(ms=ms, bytes=nbytes, GBps=nbytes / ms / 1e6, Nc=Nc,
                                 reference_bytes_per_sample=48 * n * Nc)
    return out


def driver_runs(reps_side, steps):
    from gpumd_b200 import build
    from gpumd_b200.structures import init_velocities, nep_type_order, rocksalt_pbte, write_xyz
    exe = build.build_host()
    ref = ROOT / "oracle" / "_ref" / "gpumd_ref"
    s = rocksalt_pbte(reps_side, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    tmp = Path(tempfile.mkdtemp(prefix="bench_heat_"))
    base = "potential potential.txt\nensemble nvt_nhc 300 300 100\ntime_step 1\n"
    heat = f"compute_hnemd 1000 0.00001 0 0\ncompute_shc 2 250 0 1000 400\n"
    legs = [("b200md_plain", exe, base), ("b200md_hnemd_shc", exe, base + heat)]
    if ref.exists():
        legs.append(("reference_hnemd_shc", ref, base + heat))
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
    res = dict(card=card(), kernels=kernels(8 * args.atoms_per_side ** 3, 250, args.reps))
    if not args.skip_runs:
        res["driver"] = driver_runs(args.atoms_per_side, args.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

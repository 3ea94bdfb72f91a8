#!/usr/bin/env python
"""Cost of the time correlations (compute_dos, compute_sdc, compute_msd) on the GPU.

  (1) CUDA-event times at 1 M atoms (whole system) of one gather and of the blocked correlation per
      sample, amortised over whole flushes, for DOS, SDC and MSD at Nc = 200 and Nc = 1000, with the bytes
      the algorithm moves and the achieved bytes/s.  A flush of P origins reads the Nc + B - 1 ring frames
      once (24 bytes per atom each) plus the P "now" frames; per sample that is (Nc + B - 1 + B) / B
      frames.  --blocks measures other origin-block sizes B with diagnostic builds of the library
      (gpumd_b200.build.build_lib(variant=...)), each in its own process;
  (2) the per-step cost of the unwrapped-position update (copy before compute1, add after it);
  (3) a 1 M-atom PbTe NEP NVE run through the `b200md` driver with and without `compute_dos 5 200 400.0`,
      and the same two inputs through the reference gpumd (oracle/_ref/gpumd_ref, when built).
The card's name and power limit are printed with the numbers.  Output: one JSON line; run directories
live under a temporary directory.

    python scripts/bench_correlation.py [--atoms 1000000] [--blocks 8,16,32] [--steps 3000] [--skip-runs]
"""
import argparse
import json
import os
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
DEFAULT_B = 16  # B200MD_CORR_BLOCK of the default build (csrc/b2_correlate.cu)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def kernels(n, B, flushes):
    """(1) and (2) with the library the process loaded (B200MD_LIB)."""
    import torch
    from gpumd_b200 import engine
    rng = np.random.default_rng(1)
    atom = engine.Atom(np.zeros(n, np.int32), rng.uniform(0, 100, (3, n)), rng.uniform(20, 200, n),
                       rng.normal(size=(3, n)) * 0.05)
    dt = 1.0 / engine.TIME_UNIT_CONVERSION
    frame = 24 * n
    out = {}
    for Nc in (200, 1000):
        steps = Nc + B * (flushes + 1)
        for kind in ("dos", "sdc", "msd"):
            if kind == "dos":
                obj = engine.DOS(1, Nc, 400.0, steps, dt, atom)
            elif kind == "sdc":
                obj = engine.SDC(1, Nc, steps, dt, n)
            else:
                obj = engine.MSD(1, Nc, steps, dt, n)
            x = atom.velocity_per_atom if kind != "msd" else atom.position_per_atom

            def sample(step):
                if kind == "msd":
                    obj.process(step, x)
                else:
                    obj.process(step, atom)

            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for step in range(Nc - 1 - 2):  # fill the ring; no time origin yet: gathers only
                sample(step)
            torch.cuda.synchronize()
            a.record()
            for step in range(Nc - 3, Nc - 1):
                sample(step)
            b.record()
            torch.cuda.synchronize()
            gather_ms = a.elapsed_time(b) / 2
            first = Nc - 1 + B - 1  # completes the first block (warm-up of the correlation kernels)
            for step in range(Nc - 1, first + 1):
                sample(step)
            torch.cuda.synchronize()
            a.record()
            for step in range(first + 1, first + 1 + B * flushes):
                sample(step)
            b.record()
            torch.cuda.synchronize()
            per_sample = a.elapsed_time(b) / (B * flushes)
            corr_ms = per_sample - gather_ms
            corr_bytes = (Nc + B - 1 + B) * frame / B + (8 * n / B if kind == "dos" else 0)
            out[f"{kind}_Nc{Nc}"] = dict(
                gather_ms=gather_ms, gather_GBps=2 * frame / gather_ms / 1e6,
                sample_ms=per_sample, correlation_ms=corr_ms, correlation_bytes_per_sample=corr_bytes,
                correlation_GBps=corr_bytes / corr_ms / 1e6)
            del obj
            torch.cuda.empty_cache()
    unwrapped = engine.UnwrappedPosition(atom)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    unwrapped.begin(atom)
    unwrapped.end(atom)
    reps = 100
    a.record()
    for _ in range(reps):
        unwrapped.begin(atom)
        unwrapped.end(atom)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / reps
    out["unwrap_step"] = dict(ms=ms, bytes=5 * frame, GBps=5 * frame / ms / 1e6)
    return out


def driver_runs(reps_side, steps):
    from gpumd_b200 import build
    from gpumd_b200.structures import init_velocities, nep_type_order, rocksalt_pbte, write_xyz
    exe = build.build_host()
    ref = ROOT / "oracle" / "_ref" / "gpumd_ref"
    s = rocksalt_pbte(reps_side, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 300.0, seed=42)
    tmp = Path(tempfile.mkdtemp(prefix="bench_corr_"))
    plain = "potential potential.txt\ntime_step 1\nensemble nve\n"
    dos = plain + "compute_dos 5 200 400.0\n"
    legs = [("b200md_nve", exe, plain), ("b200md_nve_dos", exe, dos)]
    if ref.exists():
        legs += [("reference_nve", ref, plain), ("reference_nve_dos", ref, dos)]
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
    ap.add_argument("--atoms", type=int, default=1_000_000)
    ap.add_argument("--atoms-per-side", type=int, default=50)  # rocksalt PbTe: 8 x 50^3 = 1 000 000 atoms
    ap.add_argument("--blocks", default=str(DEFAULT_B))
    ap.add_argument("--flushes", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3000)  # 401 time origins at Nc = 200
    ap.add_argument("--skip-runs", action="store_true")
    ap.add_argument("--kernels-only", type=int, default=0, help=argparse.SUPPRESS)  # child: its B
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the measurement needs the GPU")
    if args.kernels_only:
        print(json.dumps(kernels(args.atoms, args.kernels_only, args.flushes)))
        return
    from gpumd_b200 import build
    res = dict(card=card(), atoms=args.atoms, kernels={})
    for B in [int(b) for b in args.blocks.split(",")]:
        env = dict(os.environ)
        if B != DEFAULT_B:
            env["B200MD_LIB"] = str(build.build_lib(variant=f"corr_b{B}", defs=[f"B200MD_CORR_BLOCK={B}"]))
        r = subprocess.run([sys.executable, __file__, "--kernels-only", str(B), "--atoms", str(args.atoms),
                            "--flushes", str(args.flushes)], capture_output=True, text=True, env=env)
        res["kernels"][f"B{B}"] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else \
            dict(error=r.stderr[-1000:])
    if not args.skip_runs:
        res["driver"] = driver_runs(args.atoms_per_side, args.steps)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

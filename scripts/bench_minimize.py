#!/usr/bin/env python
"""Cost of a FIRE minimization iteration on the GPU, fixed box and with box change.

A rattled 1 M-atom PbTe NEP crystal runs a fixed number of FIRE iterations through the Python mirror
(engine.Minimizer, the same library calls the b200md driver makes).  Reported per iteration: wall ms (host
clock, the loop ends in the record copy, which synchronises), the force ms (CUDA events around Force.compute),
the minimizer call ms (CUDA events around the library call: its two kernels, the record copy and the host's
wake-up from the synchronisation), the minimizer kernel ms (device time of k_fire_reduce and k_fire_update from
torch.profiler, in a run of its own), and the algorithmic bytes of the two kernels (reduction: F, v, U =
56 B/atom, plus the virial, 72 B/atom, with box change; update: read x, v, F and write x, v = 120 B/atom) over
the kernel ms.  When oracle/_ref/gpumd_ref was built, the unmodified reference runs the same
`minimize fire 0 K [1]` input and its wall time is reported beside.  The card's name and power limit are printed with the numbers; one JSON line.

    python scripts/bench_minimize.py [--atoms-per-side 50] [--iters 200] [--skip-reference]
"""
import argparse
import json
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
GOLDEN = ROOT / "tests" / "golden"
REF = ROOT / "oracle" / "_ref" / "gpumd_ref"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run_fire(s, iters, box_change):
    import torch
    from gpumd_b200 import engine as E
    n = s["type"].shape[0]
    atom = E.Atom(s["type"], s["pos"], s["mass"])
    box = E.Box(s["h"].copy(), s["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / "nep_PbTe.txt", n)
    a = atom
    args = (a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
    warm = E.Minimizer("fire", n, 0.0, 5, box_change)  # tolerance 0: never converges
    for _ in range(5):
        force.compute(box, *args)
        warm.fire_step(box, a)
    mz = E.Minimizer("fire", n, 0.0, iters, box_change)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(iters)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(iters):
        ev[k][0].record()
        force.compute(box, *args)
        ev[k][1].record()
        mz.fire_step(box, a)
        ev[k][2].record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / iters
    force_ms = sum(e[0].elapsed_time(e[1]) for e in ev) / iters
    call_ms = sum(e[1].elapsed_time(e[2]) for e in ev) / iters
    kernel_ms = minimizer_kernel_ms(force, box, a, args, n, box_change)
    nbytes = n * (56 + 120 + (72 if box_change else 0))
    force.potentials[0].check()
    return dict(ms_per_iter=round(wall, 4), force_ms=round(force_ms, 4), minimizer_call_ms=round(call_ms, 4),
                minimizer_kernel_ms=round(kernel_ms, 4), minimizer_bytes=nbytes,
                minimizer_GBps=round(nbytes / (kernel_ms * 1e-3) / 1e9, 1))


def minimizer_kernel_ms(force, box, a, args, n, box_change, iters=50):
    """Device time per iteration of the minimizer's two kernels, from torch.profiler's CUDA activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from gpumd_b200 import engine as E
    mz = E.Minimizer("fire", n, 0.0, iters, box_change)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            force.compute(box, *args)
            mz.fire_step(box, a)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "k_fire_" in e.key)
    if us <= 0:
        raise RuntimeError("the profiler recorded no k_fire_* kernel")
    return us / 1e3 / iters


def run_reference(s, iters, box_change):
    from gpumd_b200.structures import nep_type_order, write_xyz
    d = Path(tempfile.mkdtemp(prefix="bench_minimize_"))
    try:
        write_xyz(d / "model.xyz", s, nep_type_order(GOLDEN / "nep_PbTe.txt"))
        shutil.copyfile(GOLDEN / "nep_PbTe.txt", d / "nep.txt")
        (d / "run.in").write_text(f"potential nep.txt\nminimize fire 0 {iters}{' 1' if box_change else ''}\n")
        t0 = time.perf_counter()
        r = subprocess.run([str(REF)], cwd=d, capture_output=True, text=True, timeout=3600)
        wall = time.perf_counter() - t0
        if r.returncode != 0:
            return dict(error=(r.stdout + r.stderr)[-500:])
        return dict(wall_s=round(wall, 3), ms_per_iter_incl_setup=round(wall * 1e3 / iters, 3))
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--atoms-per-side", type=int, default=50)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--skip-reference", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_minimize.py measures on a GPU; none found")
    from gpumd_b200.structures import rocksalt_pbte
    s = rocksalt_pbte(a.atoms_per_side, rattle=0.05, seed=1)
    out = dict(card=card(), atoms=int(s["type"].shape[0]), iters=a.iters)
    for bc in (0, 1):
        key = "fire_box_change" if bc else "fire"
        out[key] = run_fire(s, a.iters, bc)
        if REF.exists() and not a.skip_reference:
            out[key]["reference"] = run_reference(s, a.iters, bc)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

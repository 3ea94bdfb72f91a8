#!/usr/bin/env python
"""Cost of one compute_rdf sample on the 1 M-atom PbTe crystal of bench.py.

    python scripts/bench_rdf.py [--samples 100] [--reference]

Times b200md_rdf_sample (cell sort + counting + fold) with CUDA events over --samples samples after a
warm-up, at rc 6 and 10 A with 100 and 500 bins, and prints one JSON line per setting with the card's name
and power limit.  --reference also times the unmodified reference gpumd (oracle/_ref/gpumd_ref) per sample:
NVE runs of the same crystal with and without `compute_rdf rc bins 1`, from its "Time used for this run"
lines, (with - without) / steps.
"""
import argparse
import json
import re
import shutil
import subprocess
import sys
import tempfile
import types
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def time_ours(s, rc, num_bins, samples, warmup=5):
    import torch
    from gpumd_b200 import engine
    rdf = engine.RDF(rc, num_bins, s["type"])
    atom = types.SimpleNamespace(type=torch.as_tensor(s["type"], device="cuda"),
                                 position_per_atom=torch.as_tensor(np.ascontiguousarray(s["pos"]).reshape(-1),
                                                                   device="cuda"))
    box = engine.Box(s["h"], s["pbc"])
    for _ in range(warmup):
        rdf.process(box, atom)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(samples):
        rdf.process(box, atom)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / samples


def time_reference(s, rc, num_bins, steps):
    from gpumd_b200.structures import init_velocities, write_xyz
    exe = ROOT / "oracle" / "_ref" / "gpumd_ref"
    if not exe.exists():
        return None
    d = Path(tempfile.mkdtemp(prefix="bench_rdf_ref_"))
    try:
        write_xyz(d / "model.xyz", s, ["Te", "Pb"], init_velocities(s["mass"], 300.0, seed=1))
        shutil.copyfile(ROOT / "tests" / "golden" / "nep_PbTe.txt", d / "nep.txt")
        sec = {}
        for tag, extra in (("without", ""), ("with", f"compute_rdf {rc} {num_bins} 1\n")):
            (d / "run.in").write_text(f"potential nep.txt\ntime_step 1\nensemble nve\n{extra}run {steps}\n")
            r = subprocess.run([str(exe)], cwd=d, capture_output=True, text=True, timeout=1800)
            m = re.findall(r"Time used for this run = ([0-9.eE+-]+) second", r.stdout)
            if r.returncode != 0 or not m:
                return None
            sec[tag] = float(m[-1])
        return (sec["with"] - sec["without"]) / steps * 1e3, sec
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--ref-steps", type=int, default=100)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_rdf.py needs a GPU")
    from gpumd_b200.structures import rocksalt_pbte
    s = rocksalt_pbte(50, rattle=0.02, seed=1)
    gpu = card()
    for rc in (6.0, 10.0):
        for nb in (100, 500):
            row = {"atoms": int(s["type"].size), "rc": rc, "num_bins": nb, "samples": a.samples,
                   "ms_per_sample": round(time_ours(s, rc, nb, a.samples), 4), "gpu": gpu}
            if a.reference:
                ref = time_reference(s, rc, nb, a.ref_steps)
                row["reference_ms_per_sample"] = None if ref is None else round(ref[0], 4)
                row["reference_run_seconds"] = None if ref is None else ref[1]
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()

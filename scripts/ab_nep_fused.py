"""A/B of builds of libb200md on the NEP force call of bench.py's flagship workload (1 M-atom PbTe), in
one process.

Every library (--lib name=path; gpumd_b200.build.build_lib(variant=...) makes diagnostic ones) is
loaded side by side and owns one NEP potential and one copy of the atoms.  Rounds of --steps force calls
alternate between the libraries, so a drift of the clocks or of other work on the host spreads over all
of them.  Then --prof-steps further calls per library with the NEP stage profiler on give the per-stage
times (k_angular_fused among them).  --model runs another model of the crystal's two species (a model of
another angular shape reaches another k_angular_fused instance).  Outputs of the first call (pe, force, virial) are compared bit for
bit with those of the first library; --no-compare skips that for builds that compute something else
(the B2_FUSED_STOP variants).  Prints one JSON line.

    python scripts/ab_nep_fused.py --lib parent=gpumd_b200/libb200md_parent.so \\
        --lib new=gpumd_b200/libb200md.so --steps 200 --rounds 3
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def card():
    """Name, power limit and max SM clock of GPU 0, read where the numbers are measured."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def make(engine, lib, torch, s, path, model):
    """A NEP potential bound to the library at `path` and its own copy of the atoms."""
    lib._LIB = None
    lib.LIB_PATH = Path(path)
    pot = engine.NEP(model, s["type"].shape[0])
    pot.set_accumulate(False)
    atom = engine.Atom(s["type"], s["pos"], s["mass"], s["vel"])
    box = engine.Box(s["h"], s["pbc"])
    args = (box, atom.type, atom.position_per_atom, atom.potential_per_atom, atom.force_per_atom,
            atom.virial_per_atom)
    pot.compute(*args)
    pot.check()
    torch.cuda.synchronize()
    out = [t.cpu().numpy().copy() for t in args[3:]]
    return dict(pot=pot, call=lambda: pot.compute(*args), out=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="name=path of a libb200md build")
    ap.add_argument("--cells", type=int, default=50, help="conventional cells per edge (50 -> 1M atoms)")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prof-steps", type=int, default=50)
    ap.add_argument("--no-compare", action="store_true")
    ap.add_argument("--model", default="", help="NEP model file for the crystal's two species (default: bench's)")
    args = ap.parse_args()
    import torch
    from bench import MODEL, crystal
    from gpumd_b200 import engine
    from gpumd_b200 import lib as L
    if not torch.cuda.is_available():
        raise SystemExit("ab_nep_fused.py: no CUDA device")
    libs = dict(item.split("=", 1) for item in args.lib)
    for p in libs.values():
        if not Path(p).exists():
            raise SystemExit(f"ab_nep_fused.py: {p} is missing")
    s = crystal(args.cells)
    model = Path(args.model) if args.model else MODEL
    runs = {k: make(engine, L, torch, s, p, model) for k, p in libs.items()}
    for r in runs.values():
        for _ in range(args.warmup):
            r["call"]()
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k, r in runs.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                r["call"]()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / args.steps)
    stages = {}
    for k, r in runs.items():
        r["pot"].profile(True)
        for _ in range(args.prof_steps):
            r["call"]()
        stages[k] = {name: round(v[0] / max(v[1], 1), 4) for name, v in r["pot"].profile_read().items()}
        r["pot"].profile(False)
        r["pot"].check()
    first = next(iter(runs))
    out = {"card": card(), "model": str(model), "atoms": int(s["type"].shape[0]), "calls_per_round": args.steps,
           "rounds": args.rounds, "libs": {}}
    for k in runs:
        v = np.array(ms[k])
        # fused_shape: the k_angular_fused instance (b200md_nep_info 10; -1 from a library without it)
        rec = {"path": libs[k], "fused_shape": runs[k]["pot"].fused_shape, "ms_per_call": [round(x, 4) for x in v],
               "median": round(float(np.median(v)), 4),
               "spread_pct": round(float((v.max() - v.min()) / np.median(v) * 100), 2), "stage_ms": stages[k]}
        if not args.no_compare:
            rec["bitwise_equal_to_" + first] = all(
                np.array_equal(a, b) for a, b in zip(runs[k]["out"], runs[first]["out"]))
        out["libs"][k] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()

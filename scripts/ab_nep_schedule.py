"""A/B of the NEP warp schedule on bench.py's flagship workload (1 M-atom PbTe, NVE), in one process:

  identity  B200MD_NEP_SCHED=0: warp w evaluates the sorted atoms [32 w, 32 w + 32)
  bricks    default: warp w evaluates segment seg_order[w] (b2_neighbor.cuh), so the warps of a block and
            the blocks resident on an SM gather from one brick of cells

Each setting owns its own atoms and potential (the switch is read when the potential is created) and runs
bench.py's step (VV1, force, VV2).  Rounds of --steps timed steps alternate between the settings, so a drift
of the clocks or of other work on the host spreads over both.  Both settings carry the packed f12 layout; its
share shows in k_force_final of `identity` against an earlier commit.  Prints one JSON line: the card, per
setting the ms/step of every round, their median and spread, the per-stage times of the NEP profiler
(pot.profile_read()) over --prof-steps further steps, and whether the two trajectories ended bit-identical.

    python scripts/ab_nep_schedule.py --steps 200 --rounds 3
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

SETTINGS = {"identity": "0", "bricks": None}


def card():
    """Name and power limit of GPU 0, read where the numbers are measured."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def make(engine, torch, s, sched, model):
    if sched is None:
        os.environ.pop("B200MD_NEP_SCHED", None)
    else:
        os.environ["B200MD_NEP_SCHED"] = sched
    from gpumd_b200.structures import TIME_UNIT_CONVERSION
    n = s["type"].shape[0]
    atom = engine.Atom(s["type"], s["pos"], s["mass"], s["vel"])
    box = engine.Box(s["h"], s["pbc"])
    force = engine.Force()
    pot = force.parse_potential(model, n)
    ens = engine.Ensemble_NVE(n)
    thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
    dt = 1.0 / TIME_UNIT_CONVERSION
    fargs = (box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
             atom.virial_per_atom)

    def step():
        ens.compute1(dt, box, atom, thermo)
        force.compute(*fargs)
        ens.compute2(dt, box, atom, thermo)

    force.compute(*fargs)
    pot.check()
    return dict(step=step, pot=pot, atom=atom, force=force)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=50, help="conventional cells per edge (50 -> 1M atoms)")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prof-steps", type=int, default=20)
    args = ap.parse_args()
    import torch
    from bench import MODEL, crystal
    from gpumd_b200 import build, engine
    if not torch.cuda.is_available():
        raise SystemExit("ab_nep_schedule.py: no CUDA device")
    build.build_lib()
    s = crystal(args.cells)
    n = s["type"].shape[0]
    runs = {k: make(engine, torch, s, v, MODEL) for k, v in SETTINGS.items()}
    os.environ.pop("B200MD_NEP_SCHED", None)
    for r in runs.values():
        for _ in range(args.warmup):
            r["step"]()
    torch.cuda.synchronize()
    ms = {k: [] for k in runs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for k, r in runs.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.steps):
                r["step"]()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / args.steps)
    stages = {}
    for k, r in runs.items():
        r["pot"].profile(True)
        for _ in range(args.prof_steps):
            r["step"]()
        stages[k] = {name: round(v[0] / max(v[1], 1), 4) for name, v in r["pot"].profile_read().items()}
        r["pot"].profile(False)
        r["pot"].check()
    a, b = (runs[k]["atom"] for k in SETTINGS)
    identical = all(bool(torch.equal(getattr(a, f), getattr(b, f)))
                    for f in ("position_per_atom", "force_per_atom", "virial_per_atom", "potential_per_atom"))
    out = {"card": card(), "atoms": n, "steps_per_round": args.steps, "rounds": args.rounds,
           "rebuilds": {k: r["pot"].num_rebuilds for k, r in runs.items()},
           "trajectories_bit_identical": identical, "settings": {}}
    for k in runs:
        v = np.array(ms[k])
        out["settings"][k] = {"ms_per_step": [round(x, 4) for x in v], "median": round(float(np.median(v)), 4),
                              "spread_pct": round(float((v.max() - v.min()) / np.median(v) * 100), 2),
                              "stage_ms": stages[k]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

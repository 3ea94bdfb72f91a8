#!/usr/bin/env python
"""Cost of HNEMD inside the block-domain step (b200md_mgpu_hnemd_set / _take).

1 M-atom PbTe (rocksalt_pbte(50)), NEP, nvt_nhc, CUDA graph on.  One group per grid; on that group the
drive is switched on and off in turn (b200md_mgpu_hnemd_set re-evaluates the forces and discards the
captured step, so every timed window starts with a warm-up that re-captures it), and each window is
timed with CUDA events around b200md_mgpu_run.  Grids 1x1x1 and 2x1x1 in local mode (all blocks on
GPU 0), and Nx1x1 over NCCL with torch.distributed.run when N > 1 GPUs are visible.  Printed with the
times: kernel launches per step, the HBM bytes per atom the HNEMD kernels move (from the arrays they
touch), and the card's name and power limit.  Output: one JSON line.

    python scripts/bench_mgpu_hnemd.py [--cells 50] [--steps 200] [--warmup 20] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
NEP = ROOT / "tests" / "golden" / "nep_PbTe.txt"
FE = (2e-5, 0.0, 0.0)
OUTPUT_INTERVAL = 100

# FP64 words per atom each HNEMD kernel reads + writes (b2_measure.cu): the drive reads W (9) and f (3)
# and writes f (3); the correction reads and writes f (3 + 3); the heat row reads W (9) and v (3).  The
# reductions' partials and the 5-double rows are per block, not per atom.
WORDS_PER_ATOM = {"k_hnemd_drive": 9 + 3 + 3, "k_hnemd_correct": 3 + 3, "k_hnemd_heat": 9 + 3}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def make_group(grid, cells, distributed=False):
    from gpumd_b200 import mgpu
    from gpumd_b200.structures import TIME_UNIT_CONVERSION, init_velocities, rocksalt_pbte
    s = rocksalt_pbte(cells, rattle=0.02, seed=1)
    g = mgpu.DomainGroup(s["h"], s["pbc"], grid, NEP, ensemble="nvt_nhc", temperature=300.0,
                         temperature_coupling=100.0, time_step=1.0 / TIME_UNIT_CONVERSION, skin=1.0,
                         cuda_graph=True, distributed=distributed)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=42))
    return g, s["type"].shape[0]


def alternate(g, steps, warmup, reps):
    """ms/step with HNEMD off and on, alternated reps times, and the launches per step of each."""
    out = {"off": [], "on": []}
    launches = {}
    max_intervals = (warmup + steps) // OUTPUT_INTERVAL + 1
    for _ in range(reps):
        for mode in ("off", "on"):
            g.set_hnemd(OUTPUT_INTERVAL, FE if mode == "on" else (0.0, 0.0, 0.0), max_intervals=max_intervals)
            g.run(warmup)  # eager step + capture + replays
            launches[mode] = g.launches_per_step
            out[mode].append(g.run_timed(steps) / steps)
            if mode == "on":
                kappa, _ = g.hnemd_take(300.0)
                assert kappa.shape[0] == (warmup + steps) // OUTPUT_INTERVAL
    return dict(ms_per_step=out, launches_per_step=launches,
                overhead_ms=min(out["on"]) - min(out["off"]))


def worker(args):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl")
    world = dist.get_world_size()
    g, n = make_group((world, 1, 1), args.cells, distributed=True)
    r = alternate(g, args.steps, args.warmup, args.reps)
    if dist.get_rank() == 0:
        Path(args.worker).write_text(json.dumps(dict(r, atoms=n)))
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=50)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)  # result file of a distributed rank
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    import torch
    from gpumd_b200 import build
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    build.build_lib()
    build.build_mgpu()
    res = dict(card=card(), cells=args.cells, steps=args.steps, warmup=args.warmup, reps=args.reps,
               hbm_bytes_per_atom={k: 8 * w for k, w in WORDS_PER_ATOM.items()},
               hbm_bytes_per_atom_total=8 * sum(WORDS_PER_ATOM.values()), runs={})
    for grid in ((1, 1, 1), (2, 1, 1)):
        g, n = make_group(grid, args.cells)
        res["atoms"] = n
        res["runs"]["local_%dx%dx%d" % grid] = alternate(g, args.steps, args.warmup, args.reps)
        del g
        torch.cuda.synchronize()
    ngpu = torch.cuda.device_count()
    if ngpu > 1:
        with tempfile.TemporaryDirectory() as tmp:
            out = Path(tmp) / "rank0.json"
            cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ngpu}",
                   "--master-addr", "127.0.0.1", "--master-port", "29541", str(Path(__file__).resolve()),
                   "--cells", str(args.cells), "--steps", str(args.steps), "--warmup", str(args.warmup),
                   "--reps", str(args.reps), "--worker", str(out)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(r.stdout[-2000:] + r.stderr[-3000:])
            res["runs"][f"nccl_{ngpu}x1x1"] = json.loads(out.read_text())
    print(json.dumps(res))


if __name__ == "__main__":
    main()

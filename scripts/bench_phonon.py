#!/usr/bin/env python
"""Cost of `compute_phonon` on the GPU, phase by phase.

Each workload runs the calculation through the library calls the b200md driver makes (b200md_phonon_*), with
CUDA events around every phase: the 6 * num_basis force calls, the sweep kernel between them (which builds H),
D(k) for all k-points, the eigensolver, and (host clock) the copy to the host and the writing of omega2.out and
D.out.  Workloads: the reference's silicon_dispersion input (2-atom Tersoff Si cell x 6^3, 401 k-points), an
8-atom NEP PbTe cell x 6^3 (1728 atoms), and a 32-atom Tersoff Si basis x 3 x 3 x 6 (the largest basis the
eigensolver takes).  When oracle/_ref/gpumd_ref was built, the unmodified reference runs each workload and its
wall time is reported beside.  The card's name and power limit are printed with the numbers;
one JSON line.

    python scripts/bench_phonon.py [--skip-reference]
"""
import argparse
import ctypes as C
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
SI_KPOINTS = [[[0, 0, 0], [0.5, 0, 0.5], [0.375, 0.375, 0.75], [0, 0, 0], [0.5, 0.5, 0.5]]]


def replicate(s, r):
    """Positions, types and masses in the order of the driver's `replicate` (copies outer, atoms inner)."""
    h = np.asarray(s["h"]).reshape(3, 3)
    pos = [s["pos"] + (h @ np.array([i, j, k], float))[:, None]
           for i in range(r[0]) for j in range(r[1]) for k in range(r[2])]
    c = r[0] * r[1] * r[2]
    return dict(pos=np.concatenate(pos, axis=1), type=np.tile(s["type"], c), mass=np.tile(s["mass"], c),
                h=(h * np.array(r)[None, :]).reshape(9), pbc=s["pbc"])


def run_case(name, s, r, pot):
    import torch
    from gpumd_b200 import engine as E
    from gpumd_b200 import lib as L
    big = replicate(s, r)
    n = big["type"].shape[0]
    atom = E.Atom(big["type"], big["pos"], big["mass"])
    box = E.Box(big["h"], big["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / pot, n)
    lib = L.load()
    nb = n // (r[0] * r[1] * r[2])
    kpts, kpath, _ = E.kpoint_path(SI_KPOINTS, box, r)
    nk = kpts.shape[0]
    cutoff = 2.0 * force.potentials[0].rc
    a = atom
    force.compute(box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
    torch.cuda.synchronize()
    h = C.c_void_p()
    kp = np.ascontiguousarray(kpts.reshape(-1))
    L.check(lib.b200md_phonon_create(n, nb, nk, kp.ctypes.data_as(C.POINTER(C.c_double)), 0.005, C.byref(h)))
    st = E._stream()
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    t_wall = time.perf_counter()
    e0 = ev()
    e0.record()
    L.check(lib.b200md_phonon_begin(h, n, box._h, box._p, cutoff, E._ptr(a.position_per_atom), E._ptr(a.mass), st))
    marks = []
    for call in range(6 * nb):
        f0, f1, f2 = ev(), ev(), ev()
        f0.record()
        force.compute(box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
        f1.record()
        L.check(lib.b200md_phonon_step(h, call, E._ptr(a.position_per_atom), E._ptr(a.force_per_atom), st))
        f2.record()
        marks.append((f0, f1, f2))
    d0, d1, d2 = ev(), ev(), ev()
    d0.record()
    L.check(lib.b200md_phonon_dynamical(h, st))
    d1.record()
    L.check(lib.b200md_phonon_eig(h, st))
    d2.record()
    torch.cuda.synchronize()
    t_dev = time.perf_counter()
    dim = 3 * nb
    W = E.phonon_read(h, E.PHONON_W, nk * dim) * E.NATURAL_TO_THZ2
    DR = E.phonon_read(h, E.PHONON_D_REAL, nk * dim * dim)
    DI = E.phonon_read(h, E.PHONON_D_IMAG, nk * dim * dim)
    with tempfile.TemporaryDirectory() as tmp:
        with open(Path(tmp) / "omega2.out", "w") as f:
            for k in range(nk):
                f.write("%.6f " % kpath[k] + "".join("%g " % w for w in W[k * dim:(k + 1) * dim]) + "\n")
        with open(Path(tmp) / "D.out", "w") as f:
            for k in range(nk):
                R = DR[k * dim * dim:(k + 1) * dim * dim].reshape(dim, dim)
                I = DI[k * dim * dim:(k + 1) * dim * dim].reshape(dim, dim)
                for row in range(dim):
                    f.write("".join("%g " % v for v in R[:, row]) + "".join("%g " % v for v in I[:, row]) + "\n")
    t_end = time.perf_counter()
    lib.b200md_phonon_destroy(h)
    return dict(case=name, atoms=n, num_basis=nb, kpoints=nk, force_calls=6 * nb,
                force_ms=sum(f0.elapsed_time(f1) for f0, f1, _ in marks),
                sweep_kernel_ms=sum(f1.elapsed_time(f2) for _, f1, f2 in marks),
                dynamical_ms=d0.elapsed_time(d1), eig_ms=d1.elapsed_time(d2),
                device_total_ms=e0.elapsed_time(d2), output_ms=(t_end - t_dev) * 1e3,
                wall_ms=(t_end - t_wall) * 1e3)


def reference_wall(name, s, symbols, r, pot):
    """The unmodified reference on the same workload: `replicate r`, `potential`, `compute_phonon 0.005` with the
    same kpoints.in; wall time of the whole process (start-up, model read and output files included)."""
    from gpumd_b200.structures import write_xyz
    with tempfile.TemporaryDirectory() as tmp:
        t = Path(tmp)
        write_xyz(t / "model.xyz", s, symbols)
        shutil.copyfile(GOLDEN / pot, t / "potential.txt")
        (t / "kpoints.in").write_text("\n".join(" ".join(str(x) for x in k) + f" P{i}"
                                                for i, k in enumerate(SI_KPOINTS[0])) + "\n")
        (t / "run.in").write_text(f"replicate {r[0]} {r[1]} {r[2]}\npotential potential.txt\ncompute_phonon 0.005\n")
        t0 = time.perf_counter()
        p = subprocess.run([str(REF)], cwd=t, capture_output=True, text=True, timeout=3600)
        return dict(case=name, reference_wall_s=time.perf_counter() - t0, returncode=p.returncode)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-reference", action="store_true")
    args = ap.parse_args()
    import torch
    from gpumd_b200.structures import diamond, nep_type_order, read_xyz, rocksalt_pbte
    torch.cuda.set_device(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    si = read_xyz(GOLDEN / "silicon_dispersion_model.xyz", ["Si"])
    si["mass"] = np.full(2, 28.085)
    pbte = rocksalt_pbte(1, rattle=0.0)
    si32 = diamond((2, 2, 1))
    cases = [("silicon_dispersion", si, (6, 6, 6), "tersoff_Si_1989.txt", ["Si"]),
             ("pbte_nep_8x216", pbte, (6, 6, 6), "nep_PbTe.txt", nep_type_order(GOLDEN / "nep_PbTe.txt")),
             ("si_tersoff_32x54", si32, (3, 3, 6), "tersoff_Si_1989.txt", ["Si"])]
    out = []
    for name, s, r, pot, _ in cases:
        run_case(name, s, r, pot)  # warm-up: module load, allocations
        res = run_case(name, s, r, pot)
        print(name, {k: round(v, 3) if isinstance(v, float) else v for k, v in res.items()}, file=sys.stderr)
        out.append(res)
    ref = None
    if not args.skip_reference and REF.exists():
        ref = [reference_wall(name, s, sym, r, pot) for name, s, r, pot, sym in cases]
    print(json.dumps(dict(gpu=q, cases=out, reference=ref)))


if __name__ == "__main__":
    main()

"""Host-side helpers: extended-XYZ reader (GPUMD's model.xyz dialect) and the seeded synthetic
bulk crystals BASELINE.md's configs use.  Pure numpy; no device code.

model.xyz format follows /root/reference src/model/read_xyz.cu:145-425: line 2 holds
``lattice="ax ay az bx by bz cx cy cz"`` (case-insensitive), optional ``pbc="T T F"`` and
``properties=species:S:1:pos:R:3[...]``.  The box is stored the way GPUMD's Box::cpu_h is
(read_xyz.cu:203-219): row-major 3x3 with the lattice vectors as COLUMNS.
"""
import re

import numpy as np

K_B = 8.617343e-5           # eV/K, src/utilities/common.cuh:21
TIME_UNIT_CONVERSION = 1.018051e+1  # fs per natural time unit, common.cuh:26

MASS = {  # subset of MASS_TABLE, src/model/read_xyz.cu:36-142 (amu)
    "H": 1.008, "C": 12.011, "Fe": 55.845, "Co": 58.933, "Ge": 72.63, "O": 15.999, "Al": 26.9815385, "Si": 28.085, "Ar": 39.948,
    "Ti": 47.867, "V": 50.9415, "Cr": 51.9961, "Ni": 58.6934, "Cu": 63.546, "Zr": 91.224,
    "Mo": 95.95, "Pd": 106.42, "Ag": 107.8682, "Te": 127.6, "Ba": 137.327, "Ta": 180.94788,
    "W": 183.84, "Pt": 195.084, "Au": 196.966569, "Pb": 207.2, "Mg": 24.305,
}


def lattice_to_h(lat9):
    """lattice="ax ay az bx by bz cx cy cz" -> GPUMD cpu_h[0..8] (a,b,c as columns)."""
    a = np.asarray(lat9, dtype=np.float64).reshape(3, 3)
    return np.ascontiguousarray(a.T).reshape(9)


def read_xyz(path, type_order=None):
    """Returns dict(symbols, pos[3,N], h[9], pbc[3], type[N] (if type_order given), extra cols)."""
    with open(path) as f:
        lines = f.read().splitlines()
    n = int(lines[0].split()[0])
    hdr = lines[1]
    m = re.search(r'lattice\s*=\s*"([^"]+)"', hdr, re.I)
    if not m:
        raise ValueError("model.xyz: no lattice on line 2")
    h = lattice_to_h([float(v) for v in m.group(1).split()])
    pbc = np.array([1, 1, 1], np.int32)
    m = re.search(r'pbc\s*=\s*"([^"]+)"', hdr, re.I)
    if m:
        pbc = np.array([1 if t.upper().startswith("T") else 0 for t in m.group(1).split()],
                       np.int32)
    cols = [("species", "S", 1), ("pos", "R", 3)]
    m = re.search(r'properties\s*=\s*(\S+)', hdr, re.I)
    if m:
        toks = m.group(1).split(":")
        cols = [(toks[i].lower(), toks[i + 1], int(toks[i + 2])) for i in range(0, len(toks), 3)]
    out = {"h": h, "pbc": pbc}
    rows = [ln.split() for ln in lines[2:2 + n]]
    c = 0
    for name, kind, width in cols:
        if kind == "S":
            out["symbols" if name == "species" else name] = [r[c] for r in rows]
        else:
            arr = np.array([[float(v) for v in r[c:c + width]] for r in rows])
            out[name] = np.ascontiguousarray(arr.T)
        c += width
    if type_order is not None:
        idx = {s: i for i, s in enumerate(type_order)}
        out["type"] = np.array([idx[s] for s in out["symbols"]], np.int32)
    out["energy"] = None
    m = re.search(r'energy\s*=\s*([-+0-9.eE]+)', hdr, re.I)
    if m:
        out["energy"] = float(m.group(1))
    m = re.search(r'virial\s*=\s*"([^"]+)"', hdr, re.I)
    if m:
        out["virial"] = np.array([float(v) for v in m.group(1).split()])
    return out


def write_xyz(path, s, symbols, vel=None):
    """model.xyz in GPUMD's dialect; vel (natural units) is written in A/fs (read_xyz.cu:380-387).
    s["group"] (optional, int [N]): one grouping method, written as group:I:1 (read_xyz.cu:271-287)."""
    n = s["type"].shape[0]
    h = np.asarray(s["h"], dtype=np.float64).reshape(3, 3)
    lat = " ".join(f"{v:.17g}" for v in h.T.reshape(-1))  # lattice= lists a, b, c
    props = "species:S:1:pos:R:3" + (":vel:R:3" if vel is not None else "")
    pbc = " ".join("T" if p else "F" for p in s["pbc"])
    pos = s["pos"]
    cols = [pos[0], pos[1], pos[2]]
    if vel is not None:
        v = np.asarray(vel) / TIME_UNIT_CONVERSION
        cols += [v[0], v[1], v[2]]
    if s.get("group") is not None:
        props += ":group:I:1"
        cols.append(np.asarray(s["group"], dtype=np.int64))
    sym = np.asarray(symbols)[s["type"]]
    with open(path, "w") as f:
        f.write(f"{n}\n")
        f.write(f'pbc="{pbc}" lattice="{lat}" properties={props}\n')
        if n >= 100000:  # C-speed writer for the million-atom benchmark inputs (shortest round-trip repr)
            try:
                import pyarrow as pa
                import pyarrow.csv as pc
                f.flush()
                tbl = pa.table({"s": pa.array(sym), **{f"c{k}": pa.array(np.ascontiguousarray(c))
                                                       for k, c in enumerate(cols)}})
                with open(path, "ab") as fb:
                    pc.write_csv(tbl, fb, pc.WriteOptions(include_header=False, delimiter=" ",
                                                          quoting_style="none"))
                return
            except ImportError:
                pass
        for i in range(n):
            f.write(sym[i] + " " + " ".join(f"{c[i]:.17g}" for c in cols) + "\n")


def nep_type_order(nep_txt):
    with open(nep_txt) as f:
        toks = f.readline().split()
    return toks[2:2 + int(toks[1])]


def _lattice(basis_frac, a, reps):
    nx, ny, nz = reps
    g = np.stack(np.meshgrid(np.arange(nx), np.arange(ny), np.arange(nz), indexing="ij"), -1)
    g = g.reshape(-1, 3).astype(np.float64)
    pos = (g[:, None, :] + np.asarray(basis_frac)[None, :, :]).reshape(-1, 3) * a
    return pos


_FCC = [(0, 0, 0), (0.5, 0.5, 0), (0.5, 0, 0.5), (0, 0.5, 0.5)]


def _finish(pos, types, box, rattle, seed):
    rng = np.random.default_rng(seed)
    if rattle > 0:
        pos = pos + rng.normal(0.0, rattle, pos.shape)
    pos = np.mod(pos, np.asarray(box)[None, :])
    h = np.diag(box).astype(np.float64).reshape(9)
    return dict(pos=np.ascontiguousarray(pos.T), type=np.asarray(types, np.int32), h=h,
                pbc=np.array([1, 1, 1], np.int32))


def rocksalt_pbte(reps, a=6.570, rattle=0.02, seed=1):
    """Rocksalt PbTe (config C1/C3): type 0 = Te, 1 = Pb, the order in tests/golden/nep_PbTe.txt."""
    if isinstance(reps, int):
        reps = (reps,) * 3
    basis = _FCC + [(0.5, 0.5, 0.5), (0, 0, 0.5), (0, 0.5, 0), (0.5, 0, 0)]
    pos = _lattice(basis, a, reps)
    types = np.tile(np.array([0, 0, 0, 0, 1, 1, 1, 1], np.int32), reps[0] * reps[1] * reps[2])
    s = _finish(pos, types, [a * reps[0], a * reps[1], a * reps[2]], rattle, seed)
    s["symbols"] = ["Te", "Pb"]
    s["mass"] = np.where(s["type"] == 0, MASS["Te"], MASS["Pb"]).astype(np.float64)
    return s


def fcc(reps, a, rattle=0.0, seed=1, num_types=1, symbols=("Ar",)):
    """fcc crystal (C2 argon a=5.30; C4 alloy a=3.9 with species drawn i.i.d.)."""
    if isinstance(reps, int):
        reps = (reps,) * 3
    pos = _lattice(_FCC, a, reps)
    rng = np.random.default_rng(seed + 1000)
    types = rng.integers(0, num_types, pos.shape[0]).astype(np.int32) if num_types > 1 else \
        np.zeros(pos.shape[0], np.int32)
    s = _finish(pos, types, [a * reps[0], a * reps[1], a * reps[2]], rattle, seed)
    s["symbols"] = list(symbols)
    s["mass"] = np.array([MASS[symbols[t]] for t in s["type"]], np.float64)
    return s


def diamond(reps, a=5.431, rattle=0.0, seed=1, symbol="Si"):
    if isinstance(reps, int):
        reps = (reps,) * 3
    basis = _FCC + [(x + 0.25, y + 0.25, z + 0.25) for x, y, z in _FCC]
    pos = _lattice(basis, a, reps)
    s = _finish(pos, np.zeros(pos.shape[0], np.int32), [a * r for r in reps], rattle, seed)
    s["symbols"] = [symbol]
    s["mass"] = np.full(pos.shape[0], MASS[symbol])
    return s



def graphene_sheet(nx=100, ny=101):
    """The sheet of the reference's graphene HNEMD case (tests/gpumd/graphene_kappa_hnemd/create_xyz.m):
    4-atom rectangular cell (a = 1.42 sqrt 3, b = 4.26, c = 3.35 A), nx x ny x 1 cells, pbc T T F, and
    one grouping method of 9 slabs along y (cell rows 0 | 1-20 | 21-30 | ... | 71-80 | 81-)."""
    r0 = np.array([[0.5, 0, 0], [0, 1 / 6, 0], [0, 0.5, 0], [0.5, 2 / 3, 0]])
    a = np.array([1.42 * np.sqrt(3), 1.42 * 3, 3.35])
    pos, label = [], []
    for j in range(ny):
        for i in range(nx):
            for m in range(4):
                pos.append(a * (np.array([i, j, 0]) + r0[m]))
                label.append(0 if j == 0 else 1 if j <= 20 else min(2 + (j - 21) // 10, 8))
    pos = np.array(pos)
    n = pos.shape[0]
    return dict(pos=np.ascontiguousarray(pos.T), type=np.zeros(n, np.int32),
                h=np.diag(a * np.array([nx, ny, 1])).reshape(9), pbc=np.array([1, 1, 0], np.int32),
                group=np.array(label, np.int32), mass=np.full(n, MASS["C"]), symbols=["C"])


def init_velocities(mass, temperature, seed=42):
    """Maxwell-like initial velocities with zero total momentum, scaled to exactly T
    (same invariants as src/main_gpumd/velocity.cu:55-75,312-347; different PRNG).
    Returns v[3,N] in GPUMD natural units (A / natural-time)."""
    rng = np.random.default_rng(seed)
    n = mass.shape[0]
    v = rng.normal(0.0, 1.0, (3, n)) / np.sqrt(mass)[None, :]
    p = (v * mass[None, :]).sum(axis=1) / mass.sum()
    v -= p[:, None]
    ke2 = (mass[None, :] * v * v).sum()
    t_now = ke2 / (3.0 * n * K_B)
    v *= np.sqrt(temperature / t_now)
    return np.ascontiguousarray(v)

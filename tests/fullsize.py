"""A tiled oracle for the benchmark-size systems (test infrastructure).

The whole-system oracle (oracle/oracle_py.py) runs on one core: 0.5-2 M atoms take minutes to an hour.
This module cuts an orthogonal periodic box into tiles and evaluates the tiles in parallel on a process
pool.  A tile's sub-system is its own atoms plus a halo: every atom that has a periodic image within `halo`
of the tile.  Only the owned atoms' outputs are kept, so a halo of the potential's reach (2 rc for NEP,
Tersoff and EAM, whose forces need the neighbours' descriptors, bond orders or densities; rc for LJ) plus
a margin reproduces the periodic evaluation.

The sub-system keeps the periodic box and every atom's own coordinates, in ascending global id, instead of
an open box of shifted images.  The oracle then forms every displacement exactly as it does for the whole
system: x_j - x_i in FP64, rounded to FP32, then the minimum-image shift by L in FP32.  An open box would
carry x_j + L in FP64 instead, and that rounds differently by up to half an FP32 ulp of L (1.5e-5 A at
L = 330 A), which moves FP32 forces near the faces by up to ~1e-4 eV/A, ten times the force tolerance.
With the same displacements and the same neighbour order, the tiles reproduce the whole-system oracle
bit for bit, in FP32 and FP64 (tests/test_full_size_cpu.py).

The pool uses the spawn context: the GPU tests call it after CUDA is initialised, and a fork of such a
process is unsafe.  Arrays go in and out as numpy arrays."""
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor
from pathlib import Path
import multiprocessing as mp

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

MARGIN = 0.5  # A beyond the potential's reach
_POOL = None
_POOL_SIZE = 0
_HANDLES = {}  # per worker process: potential file -> NepOracle


def num_workers():
    return max(1, min(os.cpu_count() or 1, 16))


def _pool():
    global _POOL, _POOL_SIZE
    if _POOL is None:
        _POOL_SIZE = num_workers()
        _POOL = ProcessPoolExecutor(max_workers=_POOL_SIZE, mp_context=mp.get_context("spawn"))
    return _POOL


def shutdown():
    global _POOL
    if _POOL is not None:
        _POOL.shutdown(wait=True)
        _POOL = None


# ---------------------------------------------------------------- potentials

def nep(path, precision=32):
    """NEP through oracle_py.NepOracle (FP32 or FP64 arithmetic)."""
    from oracle import oracle_py
    orc = oracle_py.NepOracle(path)
    rc = max(orc.rc_radial, orc.rc_angular)
    return dict(kind="nep", path=str(path), precision=int(precision), rc=rc, reach=2.0 * rc)


def lj(path):
    import cases_classical as cc
    table = cc.lj_table(path)
    rc = float(table[..., 2].max())
    return dict(kind="lj", para=table, rc=rc, reach=rc)


def tersoff(path):
    from oracle import oracle_py
    import cases_classical as cc
    nt, para = oracle_py.tersoff_parameters(path)
    rc = float(cc.cutoff("tersoff", path))
    return dict(kind="tersoff", nt=nt, para=para, rc=rc, reach=2.0 * rc)


def eam(path):
    from oracle import oracle_py
    import cases_classical as cc
    model, nt, para = oracle_py.eam_parameters(path)
    rc = float(cc.cutoff("eam", path))
    return dict(kind="eam", model=model, nt=nt, para=para, rc=rc, reach=2.0 * rc)


def default_halo(pot):
    return pot["reach"] + MARGIN


# ---------------------------------------------------------------- one tile (runs in a worker)

def _tile(pot, type_, h, pos, own, gid, lists):
    """Evaluate one sub-system (periodic box h, own: indices of the owned atoms in it)."""
    from oracle import oracle_py
    pbc = np.ones(3, np.int32)
    kind = pot["kind"]
    if kind == "nep":
        orc = _HANDLES.get(pot["path"])
        if orc is None:
            orc = _HANDLES[pot["path"]] = oracle_py.NepOracle(pot["path"])
        r = orc.compute(type_, h, pbc, pos, precision=pot["precision"], lists=lists)
    elif kind == "lj":
        r = oracle_py.lj_compute(pot["para"], type_, h, pbc, pos)
    elif kind == "tersoff":
        r = oracle_py.tersoff_compute(pot["nt"], pot["para"], type_, h, pbc, pos)
    else:
        r = oracle_py.eam_compute(pot["model"], pot["nt"], pot["para"], type_, h, pbc, pos)
    out = dict(pe=r["pe"][own], force=np.ascontiguousarray(r["force"][:, own]),
               virial=np.ascontiguousarray(r["virial"][:, own]))
    if lists and kind == "nep":
        for which in ("radial", "angular"):
            NN = r[f"NN_{which}"][own]
            NL = r[f"NL_{which}"][own, :max(int(NN.max()) if NN.size else 0, 1)]
            # gid ascends, so the rows stay ascending in global ids
            out[f"NN_{which}"] = NN
            out[f"NL_{which}"] = np.where(NL >= 0, gid[np.maximum(NL, 0)], -1).astype(np.int32)
    return out


# ---------------------------------------------------------------- the tiling

def tile_counts(L, halo, workers):
    """Tiles per direction: edges of at least 3 halos (the halo work stays below ~8x the owned work) and
    about two tiles per worker where the box allows it."""
    edge = max(3.0 * halo, (np.prod(L) / (2.0 * workers)) ** (1.0 / 3.0))
    return [max(1, int(L[d] // edge)) for d in range(3)]


def subsystems(h, pos, halo, tiles, offset=0.0):
    """Yield (owned global ids, sub-system global ids, index of the owned atoms in the sub-system) for every
    tile.  Tile (i, j, k) owns the atoms whose wrapped coordinates u = x - n L (u in [offset, offset + L))
    lie in [offset + i w, offset + (i + 1) w); its sub-system is every atom that has an image within `halo`
    of the tile, once, in ascending global id, at its own position."""
    h = np.asarray(h, dtype=np.float64).reshape(3, 3)
    assert np.count_nonzero(h - np.diag(np.diag(h))) == 0, "the tiled oracle takes orthogonal boxes only"
    L = np.diag(h).copy()
    off = np.broadcast_to(np.asarray(offset, dtype=np.float64), (3,))
    u = pos - np.floor((pos - off[:, None]) / L[:, None]) * L[:, None]
    w = L / np.asarray(tiles)
    cell = np.clip(np.floor((u - off[:, None]) / w[:, None]).astype(np.int64), 0, np.asarray(tiles)[:, None] - 1)
    reps = [int(np.ceil(halo / L[d])) + 1 for d in range(3)]
    for i in range(tiles[0]):
        for j in range(tiles[1]):
            for k in range(tiles[2]):
                t = (i, j, k)
                lo = off + np.array(t) * w
                hi = lo + w
                own = np.nonzero((cell[0] == i) & (cell[1] == j) & (cell[2] == k))[0]
                near = np.ones(pos.shape[1], bool)
                for d in range(3):  # some image of the atom lies in the window along every direction
                    in_d = np.zeros(pos.shape[1], bool)
                    for m in range(-reps[d], reps[d] + 1):
                        c = u[d] + m * L[d]
                        in_d |= (c >= lo[d] - halo) & (c < hi[d] + halo)
                    near &= in_d
                near[own] = True
                gid = np.nonzero(near)[0]
                yield own, gid, np.searchsorted(gid, own)


def evaluate(pot, type_, h, pbc, pos, lists=False, halo=None, tiles=None, offset=0.0):
    """pe[N], force[3, N], virial[9, N] (and with lists=True for NEP: NN_/NL_radial, NN_/NL_angular in
    global ids, ascending, -1 padded) of the periodic system, assembled from the tiles.  Also returns
    `seconds` (wall time) and `tiles`."""
    t0 = time.perf_counter()
    assert np.all(np.asarray(pbc) == 1), "the tiled oracle takes fully periodic boxes only"
    type_ = np.ascontiguousarray(type_, dtype=np.int32)
    pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3, -1)
    n = pos.shape[1]
    halo = default_halo(pot) if halo is None else float(halo)
    pool = _pool()
    L = np.diag(np.asarray(h, dtype=np.float64).reshape(3, 3))
    tiles = tile_counts(L, halo, _POOL_SIZE) if tiles is None else list(tiles)
    jobs = []
    hbox = np.asarray(h, dtype=np.float64).reshape(9)
    for own, gid, where in subsystems(h, pos, halo, tiles, offset):
        sub = np.ascontiguousarray(pos[:, gid])
        jobs.append((own, pool.submit(_tile, pot, type_[gid], hbox, sub, where, gid, lists)))
    out = dict(pe=np.zeros(n), force=np.zeros((3, n)), virial=np.zeros((9, n)))
    parts = []
    seen = np.zeros(n, np.int32)
    for own, fut in jobs:
        r = fut.result()
        seen[own] += 1
        out["pe"][own] = r["pe"]
        out["force"][:, own] = r["force"]
        out["virial"][:, own] = r["virial"]
        if lists:
            parts.append((own, r))
    assert np.all(seen == 1), "every atom is owned by exactly one tile"
    if lists and pot["kind"] == "nep":
        for which in ("radial", "angular"):
            w = max(p[f"NL_{which}"].shape[1] for _, p in parts)
            NN = np.zeros(n, np.int32)
            NL = np.full((n, w), -1, np.int32)
            for own, p in parts:
                NN[own] = p[f"NN_{which}"]
                NL[own, :p[f"NL_{which}"].shape[1]] = p[f"NL_{which}"]
            out[f"NN_{which}"], out[f"NL_{which}"] = NN, NL
    out["seconds"] = time.perf_counter() - t0
    out["tiles"] = tiles
    return out


# ---------------------------------------------------------------- comparing neighbour lists

def list_difference(NN_a, NL_a, NN_b, NL_b):
    """The pairs (i, j) in exactly one of two neighbour relations (rows ascending, -1 padded)."""
    def pairs(NN, NL):
        w = NL.shape[1]
        mask = np.arange(w)[None, :] < NN[:, None]
        i = np.broadcast_to(np.arange(NN.shape[0])[:, None], NL.shape)[mask]
        return i.astype(np.int64) * (1 << 32) + NL[mask].astype(np.int64)
    a, b = pairs(NN_a, NL_a), pairs(NN_b, NL_b)
    diff = np.setxor1d(a, b, assume_unique=True)
    return np.stack([diff >> 32, diff & 0xFFFFFFFF], axis=1)


def pair_distance(h, pos, pairs):
    """Minimum-image FP64 distances of (i, j) pairs in an orthogonal periodic box."""
    L = np.diag(np.asarray(h, dtype=np.float64).reshape(3, 3))
    d = pos[:, pairs[:, 1]] - pos[:, pairs[:, 0]]
    d -= np.round(d / L[:, None]) * L[:, None]
    return np.sqrt((d * d).sum(axis=0))


def assert_same_lists(NN_a, NL_a, NN_b, NL_b, h, pos, what=""):
    """Identical neighbour relations and rows; a failure names the differing pairs and their distances."""
    pairs = list_difference(NN_a, NL_a, NN_b, NL_b)
    if pairs.size:
        r = pair_distance(h, pos, pairs[:10])
        raise AssertionError(f"{what}: {len(pairs)} pairs differ, e.g. (i, j, r) = "
                             f"{[(int(p[0]), int(p[1]), float(x)) for p, x in zip(pairs[:10], r)]}")
    w = min(NL_a.shape[1], NL_b.shape[1])
    assert np.array_equal(NN_a, NN_b), what
    assert np.array_equal(NL_a[:, :w], NL_b[:, :w]), what
    assert np.all(NL_a[:, w:] == -1) and np.all(NL_b[:, w:] == -1), what

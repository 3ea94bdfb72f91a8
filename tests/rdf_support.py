"""Test helpers for compute_rdf: the brute-force C oracle (oracle/rdf_oracle.c) and the host build of the
RDF kernel bodies (tests/emu/rdf_emu.cpp), compiled once per session into a temporary directory, plus the
systems the CPU and GPU tests share."""
import ctypes as C
import subprocess
import tempfile
from functools import lru_cache
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
_ll = C.POINTER(C.c_longlong)
_ull = C.POINTER(C.c_ulonglong)
_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


@lru_cache(maxsize=None)
def _build():
    d = Path(tempfile.mkdtemp(prefix="rdf_oracle_"))
    subprocess.run(["gcc", "-O2", "-std=c11", "-D_GNU_SOURCE", "-ffp-contract=off", "-fPIC", "-shared", "-o",
                    str(d / "librdf_oracle.so"), str(ROOT / "oracle" / "rdf_oracle.c"), "-lm"], check=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                    "-o", str(d / "librdf_emu.so"), str(ROOT / "tests" / "emu" / "rdf_emu.cpp")], check=True)
    O = C.CDLL(str(d / "librdf_oracle.so"))
    O.rdf_oracle_volume.restype = C.c_double
    O.rdf_oracle_volume.argtypes = [_dp]
    O.rdf_oracle_counts.restype = None
    O.rdf_oracle_counts.argtypes = [C.c_int, _dp, _ip, _ip, _dp, C.c_double, C.c_int, C.c_int, _ip, _ll]
    O.rdf_oracle_unordered.restype = C.c_longlong
    O.rdf_oracle_unordered.argtypes = [C.c_int, _dp, _ip, _ip, _dp, C.c_double, C.c_int, C.c_int, _ip, _ll]
    O.rdf_oracle_factors.restype = None
    O.rdf_oracle_factors.argtypes = [C.c_double, C.c_int, C.c_double, C.c_int, C.c_int, _ip, _dp]
    E = C.CDLL(str(d / "librdf_emu.so"))
    E.rdf_emu_bin.restype = C.c_int
    E.rdf_emu_bin.argtypes = [C.c_double, C.c_double, C.c_int]
    E.rdf_emu_count.restype = C.c_int
    E.rdf_emu_count.argtypes = [C.c_int, _dp, _ip, _ip, _dp, C.c_double, C.c_int, C.c_int, _ip, _ull]
    E.rdf_emu_fold.restype = None
    E.rdf_emu_fold.argtypes = [C.c_double, C.c_int, C.c_int, C.c_double, C.c_int, _ip, _ull, _dp]
    E.rdf_emu_volume.restype = C.c_double
    E.rdf_emu_volume.argtypes = [_dp]
    return O, E


def _arr(s):
    h = np.ascontiguousarray(s["h"], np.float64).reshape(9)
    pbc = np.ascontiguousarray(s["pbc"], np.int32)
    ty = np.ascontiguousarray(s["type"], np.int32)
    pos = np.ascontiguousarray(s["pos"], np.float64).reshape(-1)
    return h, pbc, ty, pos


def species(type_):
    """the types with at least one atom, in type-id order, and their atom counts"""
    c = np.bincount(np.asarray(type_, np.int64))
    ti = np.nonzero(c)[0].astype(np.int32)
    return ti, c[ti].astype(np.int32)


def num_rdfs(T):
    return 1 + T * (T + 1) // 2


def volume(h):
    return _build()[0].rdf_oracle_volume(np.ascontiguousarray(h, np.float64).reshape(9).ctypes.data_as(_dp))


def oracle_counts(s, rc, num_bins):
    """[num_bins, R] ordered-pair counts: total, then (a, b) for a <= b with i in a, j in b"""
    O, _ = _build()
    h, pbc, ty, pos = _arr(s)
    ti, _n = species(ty)
    out = np.zeros((num_bins, num_rdfs(len(ti))), np.int64)
    O.rdf_oracle_counts(ty.size, h.ctypes.data_as(_dp), pbc.ctypes.data_as(_ip), ty.ctypes.data_as(_ip),
                        pos.ctypes.data_as(_dp), rc, num_bins, len(ti), ti.ctypes.data_as(_ip),
                        out.ctypes.data_as(_ll))
    return out


def oracle_unordered(s, rc, num_bins):
    """([P, num_bins] unordered counts u(a <= b), number of pairs whose d2 is not bit-symmetric)"""
    O, _ = _build()
    h, pbc, ty, pos = _arr(s)
    ti, _n = species(ty)
    T = len(ti)
    u = np.zeros((T * (T + 1) // 2, num_bins), np.int64)
    asym = O.rdf_oracle_unordered(ty.size, h.ctypes.data_as(_dp), pbc.ctypes.data_as(_ip), ty.ctypes.data_as(_ip),
                                  pos.ctypes.data_as(_dp), rc, num_bins, T, ti.ctypes.data_as(_ip),
                                  u.ctypes.data_as(_ll))
    return u, asym


def ordered_from_unordered(u, T):
    """the ordered counts [num_bins, R] from u: total 2 sum u, (a, a) 2 u, (a < b) u"""
    num_bins = u.shape[1]
    out = np.zeros((num_bins, num_rdfs(T)), np.int64)
    out[:, 0] = 2 * u.sum(axis=0)
    k = 0
    for a in range(T):
        for b in range(a, T):
            out[:, 1 + k] = 2 * u[k] if a == b else u[k]
            k += 1
    return out


def factors(vol, n, rc, num_bins, num_atoms):
    O, _ = _build()
    na = np.ascontiguousarray(num_atoms, np.int32)
    f = np.zeros((num_bins, num_rdfs(na.size)))
    O.rdf_oracle_factors(vol, n, rc, num_bins, na.size, na.ctypes.data_as(_ip), f.ctypes.data_as(_dp))
    return f


def emu_counts(s, rc, num_bins):
    """the device walk and bin rule on the host: u [P, num_bins] (None for a box with < 5 cells)"""
    _, E = _build()
    h, pbc, ty, pos = _arr(s)
    ti, _n = species(ty)
    T = len(ti)
    u = np.zeros((T * (T + 1) // 2, num_bins), np.uint64)
    rc_ = E.rdf_emu_count(ty.size, h.ctypes.data_as(_dp), pbc.ctypes.data_as(_ip), ty.ctypes.data_as(_ip),
                          pos.ctypes.data_as(_dp), rc, num_bins, T, ti.ctypes.data_as(_ip), u.ctypes.data_as(_ull))
    return None if rc_ < 0 else u.astype(np.int64)


def emu_fold(u, rc, num_bins, vol, n, num_atoms, acc=None):
    _, E = _build()
    na = np.ascontiguousarray(num_atoms, np.int32)
    uu = np.ascontiguousarray(u, np.uint64).copy()
    acc = np.zeros((num_bins, num_rdfs(na.size))) if acc is None else np.ascontiguousarray(acc).copy()
    E.rdf_emu_fold(rc, num_bins, na.size, vol, n, na.ctypes.data_as(_ip), uu.ctypes.data_as(_ull),
                   acc.ctypes.data_as(_dp))
    assert not uu.any()
    return acc


def emu_bin(d2, rc, num_bins):
    return _build()[1].rdf_emu_bin(d2, rc, num_bins)


def ref_bin(d2, rc, num_bins):
    """rdf.cu:98-106 literally"""
    dr = rc / num_bins
    if d2 > rc * rc:
        return -1
    for w in range(num_bins):
        if d2 > (w * dr) * (w * dr) and d2 <= ((w + 1) * dr) * ((w + 1) * dr):
            return w
    return -1


# ---- systems ------------------------------------------------------------------------------------------
def triclinic(s, tilt=(0.13, -0.07, 0.09)):
    """the same atoms in a sheared cell (fractional coordinates kept)"""
    h = np.asarray(s["h"], np.float64).reshape(3, 3).copy()
    frac = np.linalg.solve(h, np.asarray(s["pos"]))
    L = np.diag(h).copy()
    h[0, 1], h[0, 2], h[1, 2] = tilt[0] * L[1], tilt[1] * L[2], tilt[2] * L[2]
    return dict(s, h=h.reshape(9), pos=h @ frac)


def open_slab(s, gap=12.0, outside=0.8):
    """pbc T T F: the cell grown by gap along z, and the atoms of the top layer moved past the box's upper
    face (open directions allow atoms outside the box)"""
    h = np.asarray(s["h"], np.float64).reshape(3, 3).copy()
    pos = np.asarray(s["pos"], np.float64).copy()
    Lz = h[2, 2]
    top = pos[2] > Lz - 2.0
    pos[2, top] += gap + outside + 2.0
    h[2, 2] = Lz + gap
    return dict(s, h=h.reshape(9), pos=pos, pbc=np.array([1, 1, 0], np.int32))


def random_types(s, T, seed, absent=()):
    rng = np.random.default_rng(seed)
    keep = [t for t in range(T) if t not in absent]
    return dict(s, type=rng.choice(keep, s["type"].shape[0]).astype(np.int32))


# ---- the cases compared with the oracle and with the reference binary (scripts/run_reference_gpumd.py) ----
GOLDEN = ROOT / "tests" / "golden"
RDF_STATIC = "velocity 1\nensemble nve\ntime_step 0\ncompute_rdf {rc} {nb} 1\nrun 1\n"
RDF_NVE_RUN = "ensemble nve\ntime_step 1\ncompute_rdf 6 100 20\nrun 200\n"
RDF_BINS = (21, 500)


def rdf_cases():
    """name -> (structure, rc, symbols in the potential's order, potential file)"""
    from gpumd_b200.structures import fcc, nep_type_order, rocksalt_pbte
    pbte = rocksalt_pbte(12, rattle=0.1, seed=11)  # 13 824 atoms, 78.8 A
    small = rocksalt_pbte(8, rattle=0.1, seed=12)  # 4096 atoms
    alloy = fcc(10, 3.6, rattle=0.1, seed=13)      # 4000 atoms, 36 A
    pbte_pot, pbte_sym = GOLDEN / "nep_PbTe.txt", ["Te", "Pb"]
    nep50 = GOLDEN / "nep_synth_50types.txt"
    return {
        "pbte_ortho": (pbte, 6.0, pbte_sym, pbte_pot),
        "pbte_tric": (triclinic(small), 6.0, pbte_sym, pbte_pot),
        "pbte_open_z_outside": (open_slab(small), 6.0, pbte_sym, pbte_pot),
        "lj_3types": (random_types(fcc(10, 3.9, rattle=0.12, seed=14), 3, seed=15), 7.0, ["Ar", "Ne", "Kr"],
                      GOLDEN / "lj_synth_3types.txt"),
        "cufeni_without_fe": (random_types(alloy, 3, seed=16, absent=(1,)), 5.5, ["Cu", "Fe", "Ni"],
                              GOLDEN / "eam_zhou_2004_CuFeNi.txt"),
        "one_species": (fcc(10, 5.3, rattle=0.15, seed=17), 10.0, ["Ar"], GOLDEN / "lj_Ar_10A.txt"),
        "fifty_species": (random_types(fcc(12, 3.6, rattle=0.1, seed=18), 50, seed=19), 5.0,
                          nep_type_order(nep50), nep50),
    }


def rdf_nve_case():
    """the 200-step PbTe NVE run sampled every 20 steps: (structure, velocities, symbols, potential)"""
    from gpumd_b200.structures import init_velocities, rocksalt_pbte
    s = rocksalt_pbte(6, rattle=0.05, seed=21)  # 1728 atoms, 39.4 A
    return s, init_velocities(s["mass"], 300.0, seed=21), ["Te", "Pb"], GOLDEN / "nep_PbTe.txt"

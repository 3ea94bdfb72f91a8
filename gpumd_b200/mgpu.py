"""ctypes binding of libb200md_mgpu.so (include/b200md_mgpu.h): block / slab domain decomposition of
the MD hot path in C++ / CUDA / NCCL.  Python only hands over the global arrays and, in distributed
mode, carries the ncclUniqueId from rank 0 to the other ranks through torch.distributed."""
import ctypes as C
from pathlib import Path

import numpy as np

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libb200md_mgpu.so"


class Config(C.Structure):
    _fields_ = [("h", C.c_double * 9), ("pbc", C.c_int * 3), ("grid", C.c_int * 3), ("rank", C.c_int),
                ("potential_file", C.c_char_p), ("skin", C.c_double), ("ensemble", C.c_int),
                ("temperature", C.c_double), ("temperature_coupling", C.c_double),
                ("time_step", C.c_double), ("bdp_seed", C.c_uint), ("capacity_factor", C.c_double),
                ("use_cuda_graph", C.c_int)]


_LIB = None
ENSEMBLES = {"nve": 0, "nvt_ber": 1, "nvt_nhc": 2, "nvt_bdp": 4}


class MgpuError(RuntimeError):
    pass


def load():
    global _LIB
    if _LIB is None:
        if not LIB_PATH.exists():
            raise MgpuError(f"{LIB_PATH} is missing: build it with gpumd_b200.build.build_mgpu()")
        from . import lib as _base
        _base.load()  # libb200md.so first (same directory, $ORIGIN rpath)
        L = C.CDLL(str(LIB_PATH))
        vp, dp = C.c_void_p, C.POINTER(C.c_double)
        L.b200md_mgpu_last_error.restype = C.c_char_p
        L.b200md_mgpu_unique_id.argtypes = [C.c_char_p]
        L.b200md_mgpu_create.argtypes = [C.POINTER(Config), C.c_char_p, C.POINTER(vp)]
        L.b200md_mgpu_destroy.argtypes = [vp]
        L.b200md_mgpu_destroy.restype = None
        L.b200md_mgpu_distribute.argtypes = [vp, C.c_int, vp, vp, vp, vp]
        L.b200md_mgpu_run.argtypes = [vp, C.c_int, C.c_int]
        L.b200md_mgpu_run_timed.argtypes = [vp, C.c_int, C.c_int, dp]
        L.b200md_mgpu_thermo.argtypes = [vp, dp]
        L.b200md_mgpu_heat_current.argtypes = [vp, dp]
        L.b200md_mgpu_info.argtypes = [vp, C.c_int, C.c_int]
        L.b200md_mgpu_info.restype = C.c_longlong
        L.b200md_mgpu_get_owned.argtypes = [vp, C.c_int, vp, vp, vp, vp, vp, vp]
        L.b200md_mgpu_get_local.argtypes = [vp, C.c_int, vp, vp, dp, C.POINTER(C.c_int)]
        L.b200md_mgpu_profile.argtypes = [vp, C.c_int, dp, C.c_int]
        L.b200md_mgpu_check.argtypes = [vp]
        L.b200md_mgpu_hnemd_set.argtypes = [vp, C.c_int, dp, C.c_int]
        L.b200md_mgpu_hnemd_take.argtypes = [vp, C.c_double, C.POINTER(C.c_int), dp, dp]
        _LIB = L
    return _LIB


def _check(rc):
    if rc != 0:
        raise MgpuError(f"libb200md_mgpu error {rc}: {load().b200md_mgpu_last_error().decode()}")


class DomainGroup:
    """grid = (Px, Py, Pz).  distributed=False: all Px*Py*Pz domains on the current device, in lock
    step (tests, single GPU); distributed=True: this process is rank `rank` of a torch.distributed
    job with world size Px*Py*Pz, one GPU each, NCCL between them."""

    def __init__(self, h, pbc, grid, potential_file, ensemble="nve", temperature=300.0,
                 temperature_coupling=100.0, time_step=0.0, skin=1.0, distributed=False, rank=0,
                 bdp_seed=12345678, capacity_factor=1.35, cuda_graph=False):
        L = load()
        cfg = Config()
        cfg.h[:] = list(np.asarray(h, dtype=np.float64).reshape(9))
        cfg.pbc[:] = [int(p) for p in pbc]
        cfg.grid[:] = [int(g) for g in grid]
        cfg.rank = int(rank)
        self._file = str(potential_file).encode()
        cfg.potential_file = self._file
        cfg.skin = float(skin)
        cfg.ensemble = ENSEMBLES[ensemble] if isinstance(ensemble, str) else int(ensemble)  # name or C-ABI code
        cfg.temperature, cfg.temperature_coupling = float(temperature), float(temperature_coupling)
        cfg.time_step = float(time_step)
        cfg.bdp_seed = int(bdp_seed)
        cfg.capacity_factor = float(capacity_factor)
        cfg.use_cuda_graph = 1 if cuda_graph else 0
        nccl_id = None
        if distributed:
            import torch
            import torch.distributed as dist
            buf = C.create_string_buffer(128)
            if dist.get_rank() == 0:
                _check(L.b200md_mgpu_unique_id(buf))
            t = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).cuda()
            dist.broadcast(t, 0)
            nccl_id = bytes(t.cpu().numpy().tobytes())
            cfg.rank = dist.get_rank()
        self._h = C.c_void_p()
        self._L = L
        _check(L.b200md_mgpu_create(C.byref(cfg), nccl_id, C.byref(self._h)))
        self.grid = tuple(int(g) for g in grid)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_mgpu_destroy(self._h)
            self._h = None

    def distribute(self, type_, pos, mass, vel=None):
        n = int(np.asarray(type_).shape[0])
        t = np.ascontiguousarray(type_, dtype=np.int32)
        p = np.ascontiguousarray(pos, dtype=np.float64).reshape(-1)
        m = np.ascontiguousarray(mass, dtype=np.float64)
        v = None if vel is None else np.ascontiguousarray(vel, dtype=np.float64).reshape(-1)
        _check(self._L.b200md_mgpu_distribute(
            self._h, n, t.ctypes.data, p.ctypes.data, m.ctypes.data, None if v is None else v.ctypes.data))
        self.n_global = n

    def run(self, nsteps, check_every=5):
        _check(self._L.b200md_mgpu_run(self._h, int(nsteps), int(check_every)))

    def run_timed(self, nsteps, check_every=5):
        """run() bracketed by CUDA events on the module's stream; returns milliseconds."""
        ms = C.c_double(0.0)
        _check(self._L.b200md_mgpu_run_timed(self._h, int(nsteps), int(check_every), C.byref(ms)))
        return ms.value

    @property
    def launches_per_step(self):
        return self.info(6)

    def thermo(self):
        out = (C.c_double * 8)()
        _check(self._L.b200md_mgpu_thermo(self._h, out))
        return np.array(out[:])

    def heat_current(self):
        out = (C.c_double * 5)()
        _check(self._L.b200md_mgpu_heat_current(self._h, out))
        return np.array(out[:])

    _hnemd = (1, 1)  # (output_interval, max_intervals) of the last set_hnemd: the sizes of a take

    def set_hnemd(self, output_interval, fe, max_intervals=100):
        """compute_hnemd inside the step (after distribute): fe (3 floats, 1/A) drives every step, a heat
        row is summed every step and hnemd_take() returns the finished intervals.  fe = 0 switches it
        off.  A run that would leave more than max_intervals intervals untaken is refused."""
        fe3 = (C.c_double * 3)(*[float(x) for x in fe])
        _check(self._L.b200md_mgpu_hnemd_set(self._h, int(output_interval), fe3, int(max_intervals)))
        self._hnemd = (int(output_interval), int(max_intervals))

    def hnemd_take(self, temperature):
        """(kappa[n, 5] in W/mK, rows[n, output_interval, 5]) of the n intervals finished since the last
        take; an unfinished interval carries over."""
        oi, mx = self._hnemd
        kappa, rows, n = np.zeros(5 * mx), np.zeros(5 * oi * mx), C.c_int(0)
        dp = C.POINTER(C.c_double)
        _check(self._L.b200md_mgpu_hnemd_take(self._h, float(temperature), C.byref(n), kappa.ctypes.data_as(dp),
                                              rows.ctypes.data_as(dp)))
        m = n.value
        return kappa[:5 * m].reshape(m, 5), rows[:5 * oi * m].reshape(m, oi, 5)

    def info(self, what, k=0):
        return int(self._L.b200md_mgpu_info(self._h, int(what), int(k)))

    @property
    def num_local_domains(self):
        return self.info(0)

    @property
    def migrations(self):
        return self.info(3)

    def check(self):
        _check(self._L.b200md_mgpu_check(self._h))

    def owned(self, k):
        """Owned atoms of local domain k: dict(id, pos[3,n] (global coordinates), vel, force, pe, virial)."""
        n = self.info(1, k)
        ids = np.zeros(n, np.int64)
        pos, vel, frc = np.zeros((3, n)), np.zeros((3, n)), np.zeros((3, n))
        pe, vir = np.zeros(n), np.zeros((9, n))
        _check(self._L.b200md_mgpu_get_owned(self._h, k, ids.ctypes.data, pos.ctypes.data, vel.ctypes.data,
                                             frc.ctypes.data, pe.ctypes.data, vir.ctypes.data))
        return dict(id=ids, pos=pos, vel=vel, force=frc, pe=pe, virial=vir)

    def local_system(self, k=0):
        """The local (owned + ghost) system of domain k as the potential sees it."""
        n = self.info(2, k)
        ty, pos = np.zeros(n, np.int32), np.zeros(3 * n)
        h, pbc = (C.c_double * 9)(), (C.c_int * 3)()
        _check(self._L.b200md_mgpu_get_local(self._h, k, ty.ctypes.data, pos.ctypes.data, h, pbc))
        return dict(type=ty, pos=pos, h=np.array(h[:]), pbc=np.array(pbc[:], dtype=np.int32),
                    n_own=self.info(1, k))

    def gather_local(self):
        """All owned atoms of the local domains merged and ordered by global id (local mode: the
        whole system)."""
        parts = [self.owned(k) for k in range(self.num_local_domains)]
        ids = np.concatenate([p["id"] for p in parts])
        order = np.argsort(ids)
        out = {k: np.concatenate([p[k] for p in parts], axis=-1)[..., order] for k in ("pos", "vel", "force", "pe", "virial")}
        out["id"] = ids[order]
        return out

    def profile(self, enable=True):
        out = (C.c_double * 4)()
        n = self._L.b200md_mgpu_profile(self._h, 1 if enable else 0, out, 4)
        names = ["vv1+wrap", "halo", "force", "vv2+thermo"]
        return {names[k]: out[k] for k in range(n)}

"""ctypes wrapper for tests/emu/libb2emu.so (host build of the kernel bodies; tests only)."""
import ctypes as C

import numpy as np

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_fp = C.POINTER(C.c_float)


def _d(a):
    return a.ctypes.data_as(_dp)


def _i(a):
    return a.ctypes.data_as(_ip)


# NepPlan's fields in the order emu_nep_plan writes them
NEP_PLAN = ("mn_skin", "pitch_r", "team", "fuse_split", "radial_v2", "sched", "ang_fused", "fused_shape", "fused_smem",
            "use_tc", "utable_tc", "rev_slot", "slot_map", "rad_reg", "rad_direct", "rad_nt", "c_r4", "ang_cstage",
            "variant", "tc_ctas_cap", "debug_skip", "ang_block", "ang_smem", "rad_smem")


class EmuNep:
    def __init__(self, E, path, n):
        self.E = E
        self.n = n
        self.h = E.emu_nep_create(str(path).encode(), n)
        if not self.h:
            raise RuntimeError(E.emu_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.E.emu_nep_destroy(self.h)
            self.h = None

    def compute(self, type_, h, pbc, pos, prefill=(0.0, 0.0, 0.0)):
        """prefill: the values pe / force / virial hold before the call (accumulate mode adds to them)."""
        n = self.n
        pe, f, v = np.full(n, prefill[0]), np.full(3 * n, prefill[1]), np.full(9 * n, prefill[2])
        ty = np.ascontiguousarray(type_, np.int32)
        p = np.ascontiguousarray(pos, np.float64).reshape(-1)
        hh = np.ascontiguousarray(h, np.float64).reshape(9)
        pb = np.ascontiguousarray(pbc, np.int32)
        rc = self.E.emu_nep_compute(self.h, n, _d(hh), _i(pb), _i(ty), _d(p), _d(pe), _d(f), _d(v))
        return rc, dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))

    def set_mode(self, accumulate=True, n_owned=0):
        """b200md_nep_set_accumulate / b200md_nep_set_owned"""
        self.E.emu_nep_set_mode(self.h, 0 if accumulate else 1, int(n_owned))

    def neighbors(self, mn_r, mn_a):
        n = self.n
        NNr = np.zeros(n, np.int32)
        NLr = np.full((n, mn_r), -1, np.int32)
        NNa = np.zeros(n, np.int32)
        NLa = np.full((n, mn_a), -1, np.int32)
        self.E.emu_nep_export_neighbors(self.h, mn_r, _i(NNr), _i(NLr), mn_a, _i(NNa), _i(NLa))
        return NNr, NLr, NNa, NLa

    def skin(self, mn):
        NN = np.zeros(self.n, np.int32)
        NL = np.full((self.n, mn), -1, np.int32)
        self.E.emu_nep_export_skin(self.h, mn, _i(NN), _i(NL))
        return NN, NL

    def descriptors(self, dim):
        q = np.zeros((dim, self.n), np.float32)
        self.E.emu_nep_export_descriptors(self.h, q.ctypes.data_as(_fp))
        return q

    @property
    def rebuilds(self):
        return self.E.emu_nep_rebuilds(self.h)

    @property
    def plan(self):
        """the library's NepPlan for this model and atom count (b2_setup.h nep_plan)"""
        v = (C.c_longlong * len(NEP_PLAN))()
        self.E.emu_nep_plan(self.h, v)
        return dict(zip(NEP_PLAN, v))


class EmuClassical:
    """emu_{lj,tersoff,eam}_*: a potential file on n atoms"""

    def __init__(self, E, kind, path, n):
        self.E = E
        self.kind = kind
        self.n = n
        self.h = getattr(E, f"emu_{kind}_create")(str(path).encode(), n)
        if not self.h:
            raise RuntimeError(E.emu_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            getattr(self.E, f"emu_{self.kind}_destroy")(self.h)
            self.h = None

    def compute(self, type_, h, pbc, pos):
        n = self.n
        pe, f, v = np.zeros(n), np.zeros(3 * n), np.zeros(9 * n)
        ty = np.ascontiguousarray(type_, np.int32)
        p = np.ascontiguousarray(pos, np.float64).reshape(-1)
        hh = np.ascontiguousarray(h, np.float64).reshape(9)
        pb = np.ascontiguousarray(pbc, np.int32)
        rc = getattr(self.E, f"emu_{self.kind}_compute")(self.h, n, _d(hh), _i(pb), _i(ty), _d(p), _d(pe), _d(f),
                                                          _d(v))
        return rc, dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))


class Emu:
    def __init__(self, path):
        E = C.CDLL(path)
        E.emu_last_error.restype = C.c_char_p
        E.emu_nep_create.restype = C.c_void_p
        E.emu_nep_create.argtypes = [C.c_char_p, C.c_int]
        E.emu_nep_destroy.argtypes = [C.c_void_p]
        E.emu_nep_rebuilds.argtypes = [C.c_void_p]
        for k in ("nep", "lj", "tersoff", "eam"):
            getattr(E, f"emu_{k}_error_bits").argtypes = [C.c_void_p]
        E.emu_nep_compute.argtypes = [C.c_void_p, C.c_int, _dp, _ip, _ip, _dp, _dp, _dp, _dp]
        E.emu_nep_export_neighbors.argtypes = [C.c_void_p, C.c_int, _ip, _ip, C.c_int, _ip, _ip]
        E.emu_nep_export_skin.argtypes = [C.c_void_p, C.c_int, _ip, _ip]
        E.emu_nep_export_descriptors.argtypes = [C.c_void_p, _fp]
        E.emu_nep_set_mode.argtypes = [C.c_void_p, C.c_int, C.c_int]
        E.emu_nep_plan.argtypes = [C.c_void_p, C.POINTER(C.c_longlong)]
        for k in ("lj", "tersoff", "eam"):
            getattr(E, f"emu_{k}_create").restype = C.c_void_p
            getattr(E, f"emu_{k}_create").argtypes = [C.c_char_p, C.c_int]
            getattr(E, f"emu_{k}_destroy").argtypes = [C.c_void_p]
            getattr(E, f"emu_{k}_compute").argtypes = [C.c_void_p, C.c_int, _dp, _ip, _ip, _dp, _dp, _dp, _dp]
        E.emu_compute_heat.argtypes = [C.c_int, _dp, _dp, _dp]
        E.emu_apply_pbc.argtypes = [C.c_int, _dp, _ip, _dp]
        E.emu_velocity_verlet.argtypes = [C.c_int, C.c_int, C.c_double, _dp, _dp, _dp, _dp]
        E.emu_velocity_verlet_groups.argtypes = [C.c_int, C.c_int, C.c_double, _dp, _dp, _dp, _dp, _ip,
                                                 C.c_int, C.c_int, _dp]
        E.emu_find_thermo.argtypes = [C.c_int, C.c_int, C.c_double, _dp, _dp, _dp, _dp, _dp]
        E.emu_bdp_create.restype = C.c_void_p
        E.emu_bdp_create.argtypes = [C.c_uint]
        E.emu_bdp_destroy.argtypes = [C.c_void_p]
        E.emu_bdp_rand01.restype = C.c_double
        E.emu_bdp_rand01.argtypes = [C.c_void_p]
        E.emu_bdp_factor.restype = C.c_double
        E.emu_bdp_factor.argtypes = [C.c_void_p, C.c_double, C.c_int, C.c_double, C.c_double]
        self.E = E

    def nep(self, path, n):
        return EmuNep(self.E, path, n)

    def lj(self, path, n):
        return EmuClassical(self.E, "lj", path, n)

    def tersoff(self, path, n):
        return EmuClassical(self.E, "tersoff", path, n)

    def eam(self, path, n):
        return EmuClassical(self.E, "eam", path, n)

    def compute_heat(self, virial, vel):
        n = vel.shape[1]
        heat = np.zeros(5 * n)
        self.E.emu_compute_heat(n, _d(np.ascontiguousarray(virial, np.float64).reshape(-1)),
                                _d(np.ascontiguousarray(vel, np.float64).reshape(-1)), _d(heat))
        return heat.reshape(5, n)

    def apply_pbc(self, h, pbc, pos):
        n = pos.shape[1]
        p = np.ascontiguousarray(pos, np.float64).reshape(-1).copy()
        self.E.emu_apply_pbc(n, _d(np.ascontiguousarray(h, np.float64).reshape(9)),
                             _i(np.ascontiguousarray(pbc, np.int32)), _d(p))
        return p.reshape(3, n)

    def velocity_verlet(self, step1, dt, mass, pos, vel, force):
        n = mass.shape[0]
        p = np.ascontiguousarray(pos, np.float64).reshape(-1).copy()
        v = np.ascontiguousarray(vel, np.float64).reshape(-1).copy()
        f = np.ascontiguousarray(force, np.float64).reshape(-1)
        self.E.emu_velocity_verlet(int(step1), n, float(dt), _d(np.ascontiguousarray(mass)), _d(p),
                                   _d(v), _d(f))
        return p.reshape(3, n), v.reshape(3, n)

    def velocity_verlet_groups(self, step1, dt, mass, pos, vel, force, label, fixed_group, move_group, mv):
        n = mass.shape[0]
        p = np.ascontiguousarray(pos, np.float64).reshape(-1).copy()
        v = np.ascontiguousarray(vel, np.float64).reshape(-1).copy()
        f = np.ascontiguousarray(force, np.float64).reshape(-1)
        self.E.emu_velocity_verlet_groups(
            int(step1), n, float(dt), _d(np.ascontiguousarray(mass)), _d(p), _d(v), _d(f),
            _i(np.ascontiguousarray(label, np.int32)), int(fixed_group), int(move_group),
            _d(np.ascontiguousarray(mv, np.float64)))
        return p.reshape(3, n), v.reshape(3, n)

    def find_thermo(self, n_temp, volume, mass, pe, vel, virial):
        n = mass.shape[0]
        t = np.zeros(8)
        self.E.emu_find_thermo(
            n, n_temp, float(volume), _d(np.ascontiguousarray(mass)), _d(np.ascontiguousarray(pe)),
            _d(np.ascontiguousarray(vel, np.float64).reshape(-1)),
            _d(np.ascontiguousarray(virial, np.float64).reshape(-1)), _d(t))
        return t

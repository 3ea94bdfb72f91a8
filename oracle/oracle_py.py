"""ctypes bindings for the TEST-ONLY CPU oracle (oracle/liboracle.so, oracle/_ref/libnep_cpu_ref.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  The product path (gpumd_b200/) never does.
"""
import ctypes as C
import os
import subprocess
from pathlib import Path

import math

import numpy as np

HERE = Path(__file__).resolve().parent
_LIB = None
_REF = None

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


def build():
    """(Re)build liboracle.so and, when /root/reference is present, _ref/libnep_cpu_ref.so."""
    subprocess.run(["make", "-C", str(HERE), "all"], check=True, capture_output=True)


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _i(a):
    return None if a is None else a.ctypes.data_as(_ip)


def lib():
    global _LIB
    if _LIB is None:
        path = HERE / "liboracle.so"
        if not path.exists():
            build()
        L = C.CDLL(str(path))
        L.oracle_nep_load.restype = C.c_void_p
        L.oracle_nep_load.argtypes = [C.c_char_p]
        L.oracle_nep_free.argtypes = [C.c_void_p]
        L.oracle_nep_info.argtypes = [C.c_void_p, C.c_int]
        L.oracle_nep_rc_radial_max.restype = C.c_double
        L.oracle_nep_rc_radial_max.argtypes = [C.c_void_p]
        L.oracle_nep_rc_angular_max.restype = C.c_double
        L.oracle_nep_rc_angular_max.argtypes = [C.c_void_p]
        L.oracle_nep_compute.argtypes = [
            C.c_void_p, C.c_int, C.c_int, _ip, _dp, _ip, _dp, _dp, _dp, _dp, _dp,
            _ip, _ip, C.c_int, _ip, _ip, C.c_int]
        L.oracle_neighbor_list.argtypes = [C.c_int, _dp, _ip, _dp, C.c_double, _ip, _ip, C.c_int]
        L.oracle_lj_compute.argtypes = [C.c_int, _dp, C.c_int, _ip, _dp, _ip, _dp, _dp, _dp, _dp]
        L.oracle_tersoff_compute.argtypes = [C.c_int, _dp, C.c_int, _ip, _dp, _ip, _dp, _dp, _dp, _dp]
        L.oracle_eam_compute.argtypes = [C.c_int, C.c_int, _dp, C.c_int, _ip, _dp, _ip, _dp, _dp, _dp, _dp]
        L.oracle_compute_heat.argtypes = [C.c_int, _dp, _dp, _dp]
        L.oracle_apply_pbc.argtypes = [C.c_int, _dp, _ip, _dp]
        L.oracle_velocity_verlet.argtypes = [C.c_int, C.c_int, C.c_double, _dp, _dp, _dp, _dp]
        L.oracle_velocity_verlet_groups.argtypes = [C.c_int, C.c_int, C.c_double, _dp, _dp, _dp, _dp, _ip,
                                                    C.c_int, C.c_int, _dp]
        L.oracle_find_thermo.argtypes = [C.c_int, C.c_int, C.c_double, _dp, _dp, _dp, _dp, _dp]
        _LIB = L
    return _LIB


def _box(h, pbc):
    h = np.ascontiguousarray(np.asarray(h, dtype=np.float64).reshape(9))
    pbc = np.ascontiguousarray(np.asarray(pbc, dtype=np.int32).reshape(3))
    return h, pbc


class NepOracle:
    """oracle_nep_* (plain-C restatement of src/force/nep.cu)."""

    INFO = dict(num_types=0, dim=1, num_neurons=2, n_max_radial=3, n_max_angular=4,
                basis_size_radial=5, basis_size_angular=6, L_max=7, num_L=8, MN_radial=9,
                MN_angular=10, zbl=11, version=12)

    def __init__(self, path):
        self.L = lib()
        self.h = self.L.oracle_nep_load(str(path).encode())
        if not self.h:
            raise RuntimeError(f"oracle: cannot load {path}")
        self.info = {k: self.L.oracle_nep_info(self.h, v) for k, v in self.INFO.items()}
        self.rc_radial = self.L.oracle_nep_rc_radial_max(self.h)
        self.rc_angular = self.L.oracle_nep_rc_angular_max(self.h)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.oracle_nep_free(self.h)
            self.h = None

    def compute(self, type_, h, pbc, pos, precision=32, lists=False, descriptors=False):
        """pos: (3,N) float64 SoA. Returns dict(pe[N], force[3,N], virial[9,N], ...)."""
        n = int(np.asarray(type_).shape[0])
        type_ = np.ascontiguousarray(type_, dtype=np.int32)
        pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n)
        h, pbc = _box(h, pbc)
        pe = np.zeros(n)
        f = np.zeros(3 * n)
        v = np.zeros(9 * n)
        q = np.zeros(self.info["dim"] * n) if descriptors else None
        mn_r = mn_a = 0
        NNr = NLr = NNa = NLa = None
        if lists:
            mn_r, mn_a = max(self.info["MN_radial"], 1) * 4, max(self.info["MN_angular"], 1) * 4
            NNr = np.zeros(n, np.int32)
            NLr = np.full(n * mn_r, -1, np.int32)
            NNa = np.zeros(n, np.int32)
            NLa = np.full(n * mn_a, -1, np.int32)
        rc = self.L.oracle_nep_compute(
            self.h, precision, n, _i(type_), _d(h), _i(pbc), _d(pos), _d(pe), _d(f), _d(v), _d(q),
            _i(NNr), _i(NLr), mn_r, _i(NNa), _i(NLa), mn_a)
        if rc != 0:
            raise RuntimeError(f"oracle_nep_compute failed: {rc}")
        out = dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))
        if descriptors:
            out["q"] = q.reshape(self.info["dim"], n)
        if lists:
            out.update(NN_radial=NNr, NL_radial=NLr.reshape(n, mn_r), NN_angular=NNa,
                       NL_angular=NLa.reshape(n, mn_a))
        return out


def neighbor_list(h, pbc, pos, rc, mn=512):
    L = lib()
    n = pos.shape[1]
    pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n)
    h, pbc = _box(h, pbc)
    NN = np.zeros(n, np.int32)
    NL = np.full(n * mn, -1, np.int32)
    r = L.oracle_neighbor_list(n, _d(h), _i(pbc), _d(pos), float(rc), _i(NN), _i(NL), mn)
    if r != 0:
        raise RuntimeError(f"oracle_neighbor_list failed: {r}")
    return NN, NL.reshape(n, mn)


def lj_compute(para, type_, h, pbc, pos):
    """para: (nt,nt,3) eps, sigma, cutoff."""
    L = lib()
    para = np.ascontiguousarray(para, dtype=np.float64)
    nt = para.shape[0]
    n = pos.shape[1]
    type_ = np.ascontiguousarray(type_, dtype=np.int32)
    pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n)
    h, pbc = _box(h, pbc)
    pe, f, v = np.zeros(n), np.zeros(3 * n), np.zeros(9 * n)
    r = L.oracle_lj_compute(nt, _d(para.reshape(-1)), n, _i(type_), _d(h), _i(pbc), _d(pos),
                            _d(pe), _d(f), _d(v))
    if r != 0:
        raise RuntimeError(f"oracle_lj_compute failed: {r}")
    return dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))


def tersoff_parameters(path):
    """(nt, flat parameter array) from a tersoff_1989 potential file."""
    toks = open(path).read().split()
    nt = int(toks[1])
    vals = [float(v) for v in toks[2 + nt:]]
    return nt, np.array(vals[:11 if nt == 1 else 23], dtype=np.float64)


def tersoff_compute(nt, para, type_, h, pbc, pos):
    L = lib()
    n = pos.shape[1]
    type_ = np.ascontiguousarray(type_, dtype=np.int32)
    pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n)
    para = np.ascontiguousarray(para, dtype=np.float64)
    h, pbc = _box(h, pbc)
    pe, f, v = np.zeros(n), np.zeros(3 * n), np.zeros(9 * n)
    r = L.oracle_tersoff_compute(nt, _d(para), n, _i(type_), _d(h), _i(pbc), _d(pos), _d(pe), _d(f), _d(v))
    if r != 0:
        raise RuntimeError(f"oracle_tersoff_compute failed: {r}")
    return dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))


def eam_parameters(path):
    """(model, nt, flat parameter array) from an eam_zhou_2004 / eam_dai_2006 potential file."""
    toks = open(path).read().split()
    model = {"eam_zhou_2004": 0, "eam_dai_2006": 1}[toks[0]]
    nt = int(toks[1])
    vals = [float(v) for v in toks[2 + nt:]]
    return model, nt, np.array(vals[:21 * nt if model == 0 else 9], dtype=np.float64)


def eam_compute(model, nt, para, type_, h, pbc, pos):
    L = lib()
    n = pos.shape[1]
    type_ = np.ascontiguousarray(type_, dtype=np.int32)
    pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n)
    para = np.ascontiguousarray(para, dtype=np.float64)
    h, pbc = _box(h, pbc)
    pe, f, v = np.zeros(n), np.zeros(3 * n), np.zeros(9 * n)
    r = L.oracle_eam_compute(model, nt, _d(para), n, _i(type_), _d(h), _i(pbc), _d(pos), _d(pe), _d(f), _d(v))
    if r != 0:
        raise RuntimeError(f"oracle_eam_compute failed: {r}")
    return dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))


def compute_heat(virial, vel):
    L = lib()
    n = vel.shape[-1] if vel.ndim == 2 else vel.shape[0] // 3
    heat = np.zeros(5 * n)
    L.oracle_compute_heat(n, _d(np.ascontiguousarray(virial, np.float64).reshape(-1)),
                          _d(np.ascontiguousarray(vel, np.float64).reshape(-1)), _d(heat))
    return heat.reshape(5, n)


def apply_pbc(h, pbc, pos):
    L = lib()
    n = pos.shape[1]
    out = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n).copy()
    h, pbc = _box(h, pbc)
    L.oracle_apply_pbc(n, _d(h), _i(pbc), _d(out))
    return out.reshape(3, n)


def velocity_verlet(step1, dt, mass, pos, vel, force):
    L = lib()
    n = mass.shape[0]
    p = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n).copy()
    v = np.ascontiguousarray(vel, dtype=np.float64).reshape(3 * n).copy()
    f = np.ascontiguousarray(force, dtype=np.float64).reshape(3 * n)
    m = np.ascontiguousarray(mass, dtype=np.float64)
    L.oracle_velocity_verlet(int(step1), n, float(dt), _d(m), _d(p), _d(v), _d(f))
    return p.reshape(3, n), v.reshape(3, n)


def velocity_verlet_groups(step1, dt, mass, pos, vel, force, label, fixed_group, move_group, move_velocity):
    L = lib()
    n = mass.shape[0]
    p = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n).copy()
    v = np.ascontiguousarray(vel, dtype=np.float64).reshape(3 * n).copy()
    f = np.ascontiguousarray(force, dtype=np.float64).reshape(3 * n)
    m = np.ascontiguousarray(mass, dtype=np.float64)
    lab = np.ascontiguousarray(label, dtype=np.int32)
    mv = np.ascontiguousarray(move_velocity, dtype=np.float64)
    L.oracle_velocity_verlet_groups(int(step1), n, float(dt), _d(m), _d(p), _d(v), _d(f), _i(lab),
                                    int(fixed_group), int(move_group), _d(mv))
    return p.reshape(3, n), v.reshape(3, n)


def find_thermo(n_temp, volume, mass, pe, vel, virial):
    L = lib()
    n = mass.shape[0]
    t = np.zeros(8)
    L.oracle_find_thermo(
        n, int(n_temp), float(volume), _d(np.ascontiguousarray(mass, dtype=np.float64)),
        _d(np.ascontiguousarray(pe, dtype=np.float64)),
        _d(np.ascontiguousarray(vel, dtype=np.float64).reshape(3 * n)),
        _d(np.ascontiguousarray(virial, dtype=np.float64).reshape(9 * n)), _d(t))
    return t


# ---------------------------------------------------------------- thermostats (host-side maths)

def nhc_chain(state, ek2, kT, dN, dt2_particle):
    """Nose-Hoover chain update -- restates `nhc()`, src/integrate/ensemble_nhc.cu:101-171 (run on the
    host by the reference).  state = dict(pos[4], vel[4], mas[4]) is updated in place; returns the
    velocity scale factor.  ek2 = 2 x kinetic energy."""
    M, n_sy, n_respa = 4, 7, 4
    w = [0.784513610477560, 0.235573213359357, -1.17767998417887, 1.31518632068391,
         -1.17767998417887, 0.235573213359357, 0.784513610477560]
    pos, vel, mas = state["pos"], state["vel"], state["mas"]
    factor = 1.0
    for n1 in range(n_sy):
        dt2 = dt2_particle * w[n1] / n_respa
        dt4 = dt2 * 0.5
        dt8 = dt4 * 0.5
        for _ in range(n_respa):
            G = vel[M - 2] * vel[M - 2] / mas[M - 2] - kT
            vel[M - 1] += dt4 * G
            for m in range(M - 2, -1, -1):
                tmp = np.exp(-dt8 * vel[m + 1] / mas[m + 1])
                G = ek2 - dN * kT if m == 0 else vel[m - 1] * vel[m - 1] / mas[m - 1] - kT
                vel[m] = tmp * (tmp * vel[m] + dt4 * G)
            for m in range(M - 1, -1, -1):
                pos[m] += dt2 * vel[m] / mas[m]
            fl = np.exp(-dt2 * vel[0] / mas[0])
            ek2 *= fl * fl
            factor *= fl
            for m in range(M - 1):
                tmp = np.exp(-dt8 * vel[m + 1] / mas[m + 1])
                G = ek2 - dN * kT if m == 0 else vel[m - 1] * vel[m - 1] / mas[m - 1] - kT
                vel[m] = tmp * (tmp * vel[m] + dt4 * G)
            G = vel[M - 2] * vel[M - 2] / mas[M - 2] - kT
            vel[M - 1] += dt4 * G
    return factor


def nhc_state(n_atoms, temperature, temperature_coupling, time_step):
    """Initial chain state, Ensemble_NHC::Ensemble_NHC, src/integrate/ensemble_nhc.cu:31-50."""
    kT = 8.617343e-5 * temperature
    tau = time_step * temperature_coupling
    mas = [kT * tau * tau] * 4
    mas[0] *= 3.0 * n_atoms
    return dict(pos=[0.0] * 4, vel=[1.0, -1.0, 1.0, -1.0], mas=mas)


def berendsen_factor(temperature, temperature_coupling, t_now):
    """gpu_berendsen_temperature, src/integrate/ensemble_ber.cu:70-86 (coupling = 1/tau, :34)."""
    return np.sqrt(1.0 + (1.0 / temperature_coupling) * (temperature / t_now - 1.0))


class BdpOracle:
    """Bussi-Donadio-Parrinello rescaling factor with the reference's random stream: restates
    resamplekin / resamplekin_sumnoises / gamdev / gasdev (src/integrate/svr_utilities.cuh:27-135, the
    published routines of G. Bussi) on std::mt19937 + uniform_real_distribution<double>(0,1) semantics
    (libstdc++: two 32-bit draws, low word first, / 2^64), and Ensemble_BDP::integrate_nvt_bdp_2
    (src/integrate/ensemble_bdp.cu:91-100).  Pure Python: a few hundred draws per step."""

    def __init__(self, seed=12345678):  # the -DDEBUG seed, ensemble_bdp.cu:31-32
        mt = [seed & 0xFFFFFFFF]
        for i in range(1, 624):
            mt.append((1812433253 * (mt[-1] ^ (mt[-1] >> 30)) + i) & 0xFFFFFFFF)
        self.mt, self.idx = mt, 624
        self.iset, self.gset = 0, 0.0

    def raw(self):
        mt = self.mt
        if self.idx >= 624:
            for k in range(624):
                y = (mt[k] & 0x80000000) | (mt[(k + 1) % 624] & 0x7FFFFFFF)
                mt[k] = mt[(k + 397) % 624] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
            self.idx = 0
        y = mt[self.idx]
        self.idx += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return y & 0xFFFFFFFF

    def rand01(self):
        lo = float(self.raw())
        hi = float(self.raw())
        r = (lo + hi * 4294967296.0) / 18446744073709551616.0
        return r if r < 1.0 else float(np.nextafter(1.0, 0.0))

    def gasdev(self):
        if self.iset == 0:
            while True:
                v1 = 2.0 * self.rand01() - 1.0
                v2 = 2.0 * self.rand01() - 1.0
                rsq = v1 * v1 + v2 * v2
                if 0.0 < rsq < 1.0:
                    break
            fac = math.sqrt(-2.0 * math.log(rsq) / rsq)
            self.gset, self.iset = v1 * fac, 1
            return v2 * fac
        self.iset = 0
        return self.gset

    def gamdev(self, ia):
        if ia < 6:
            x = 1.0
            for _ in range(ia):
                x *= self.rand01()
            return -math.log(x)
        while True:
            while True:
                while True:
                    v1 = self.rand01()
                    v2 = 2.0 * self.rand01() - 1.0
                    if v1 * v1 + v2 * v2 <= 1.0:
                        break
                y = v2 / v1
                am = ia - 1
                s = math.sqrt(2.0 * am + 1.0)
                x = s * y + am
                if x > 0.0:
                    break
            e = (1.0 + y * y) * math.exp(am * math.log(x / am) - s * y)
            if self.rand01() <= e:
                return x

    def sumnoises(self, nn):
        if nn == 0:
            return 0.0
        if nn == 1:
            rr = self.gasdev()
            return rr * rr
        if nn % 2 == 0:
            return 2.0 * self.gamdev(nn // 2)
        rr = self.gasdev()
        return 2.0 * self.gamdev((nn - 1) // 2) + rr * rr

    def resamplekin(self, kk, sigma, ndeg, taut):
        factor = math.exp(-1.0 / taut) if taut > 0.1 else 0.0
        rr = self.gasdev()
        noise = self.sumnoises(ndeg - 1)
        return (kk + (1.0 - factor) * (sigma * (noise + rr * rr) / ndeg - kk)
                + 2.0 * rr * math.sqrt(kk * sigma / ndeg * (1.0 - factor) * factor))

    def factor(self, t_instant, n_atoms, temperature, temperature_coupling):
        """n_atoms counts the atoms that are integrated, N - N_fixed - N_move: ndeg = 3 n_atoms
        (ensemble_bdp.cu:87-95)."""
        ndeg = 3 * n_atoms
        ek = t_instant * ndeg * 8.617343e-5 * 0.5
        sigma = ndeg * 8.617343e-5 * temperature * 0.5
        return math.sqrt(self.resamplekin(ek, sigma, ndeg, temperature_coupling) / ek)


def stdrng():
    """ctypes handle on oracle/libstdrng.so (the C++ standard library's own generator objects)."""
    R = C.CDLL(str(HERE / "libstdrng.so"))
    R.stdrng_uniform01.argtypes = [C.c_uint, C.c_int, C.c_void_p]
    R.stdrng_raw.argtypes = [C.c_uint, C.c_int, C.c_void_p]
    return R


# ---------------------------------------------------------------- the reference's own NEP_CPU

def ref_available():
    return (HERE / "_ref" / "libnep_cpu_ref.so").exists()


def ref():
    global _REF
    if _REF is None:
        R = C.CDLL(str(HERE / "_ref" / "libnep_cpu_ref.so"))
        R.refnep_load.restype = C.c_void_p
        R.refnep_load.argtypes = [C.c_char_p]
        R.refnep_free.argtypes = [C.c_void_p]
        R.refnep_compute.argtypes = [C.c_void_p, C.c_int, _ip, _dp, _dp, _dp, _dp, _dp]
        _REF = R
    return _REF


class RefNepCpu:
    """The reference's vendored NEP_CPU (tools/.../nep.cpp NEP3::compute), FP64, PBC in all
    three directions (it has no pbc argument)."""

    def __init__(self, path):
        self.R = ref()
        # NEP_CPU prints the model summary to stdout in its constructor; silence it
        fd = os.dup(1)
        devnull = os.open(os.devnull, os.O_WRONLY)
        os.dup2(devnull, 1)
        try:
            self.h = self.R.refnep_load(str(path).encode())
        finally:
            os.dup2(fd, 1)
            os.close(fd)
            os.close(devnull)

    def __del__(self):
        if getattr(self, "h", None):
            self.R.refnep_free(self.h)
            self.h = None

    def compute(self, type_, h, pos):
        n = int(np.asarray(type_).shape[0])
        type_ = np.ascontiguousarray(type_, dtype=np.int32)
        pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(3 * n)
        h = np.ascontiguousarray(np.asarray(h, dtype=np.float64).reshape(9))
        pe, f, v = np.zeros(n), np.zeros(3 * n), np.zeros(9 * n)
        self.R.refnep_compute(self.h, n, _i(type_), _d(h), _d(pos), _d(pe), _d(f), _d(v))
        return dict(pe=pe, force=f.reshape(3, n), virial=v.reshape(9, n))


# ---- SURVEY 8f rank 3: BAOAB operators and the Berendsen barostat (test infrastructure) ----------
def baoab_operator(which, dt, mass, pos, vel, force, label=None, fixed_group=-1):
    """gpu_operator_A (which = 0: x += v dt/2) / gpu_operator_B (which = 1: v += f/m dt/2) with the fixed
    group frozen, src/integrate/ensemble_bao.cu:190-300."""
    p, v = np.array(pos, dtype=np.float64), np.array(vel, dtype=np.float64)
    fixed = np.zeros(p.shape[1], bool) if label is None or fixed_group < 0 else (np.asarray(label) == fixed_group)
    if which == 0:
        p += np.where(fixed, 0.0, v) * (dt * 0.5)
    else:
        v = np.where(fixed, 0.0, v + np.asarray(force) / np.asarray(mass)[None, :] * (dt * 0.5))
    return p, v


def berendsen_pressure(h, pbc, thermo, target_p, p_coupling, num_components, deform=None, deform_rate=None):
    """cpu_pressure_isotropic / _orthogonal / _triclinic, src/integrate/ensemble_ber.cu:88-172: returns
    (new h[9], mu[9]); positions transform as r <- mu r.  thermo[2..7] = sxx syy szz sxy sxz syz; target_p /
    p_coupling in natural units, Voigt order xx yy zz yz xz xy for 6 components.  deform[3] / deform_rate[3]
    (3 components only, `deform`): a deformed direction grows by its rate (A per step) whether it is
    periodic or open, s = (h + rate) / h; that test comes before the pbc test."""
    h = np.array(h, dtype=np.float64).reshape(9)
    p = np.asarray(thermo, dtype=np.float64)[2:8]
    p0, pc = np.asarray(target_p, dtype=np.float64), np.asarray(p_coupling, dtype=np.float64)
    mu = np.eye(3).reshape(9)
    if num_components == 1:
        sfac = 1.0 - pc[0] * (p0[0] - (p[0] + p[1] + p[2]) * 0.3333333333333333)
        mu[[0, 4, 8]] = sfac
        h[[0, 4, 8]] *= sfac
    elif num_components == 3:
        for d in range(3):
            if deform is not None and deform[d]:
                sfac = (h[4 * d] + deform_rate[d]) / h[4 * d]
            else:
                sfac = 1.0 - pc[d] * (p0[d] - p[d]) if pbc[d] else 1.0
            mu[4 * d] = sfac
            h[4 * d] *= sfac
    else:
        mu[0] = 1.0 - pc[0] * (p0[0] - p[0])
        mu[4] = 1.0 - pc[1] * (p0[1] - p[1])
        mu[8] = 1.0 - pc[2] * (p0[2] - p[2])
        mu[3] = mu[1] = -pc[5] * (p0[5] - p[3])
        mu[6] = mu[2] = -pc[4] * (p0[4] - p[4])
        mu[7] = mu[5] = -pc[3] * (p0[3] - p[5])
        h = (mu.reshape(3, 3) @ h.reshape(3, 3)).reshape(9)
    return h, mu


# ---- SURVEY 8f rank 4: heat-current autocorrelation (test infrastructure) -------------------------
def find_hac(heat_all, Nc, dt_sample, temperature, volume):
    """gpu_find_hac + find_rtc, src/measure/hac.cu:111-181.  heat_all[5, Nd] = jx_in jx_out jy_in jy_out jz;
    returns hac[5, Nc], rtc[5, Nc] (W/mK).  dt_sample = time_step * sample_interval, natural units."""
    K_B, KAPPA = 8.617343e-5, 1.573769e+5
    h = np.asarray(heat_all, dtype=np.float64)
    Nd = h.shape[1]
    hac = np.zeros((5, Nc))
    for nc in range(Nc):
        a, b = slice(0, Nd - nc), slice(nc, Nd)
        hac[0, nc] = np.sum(h[0, a] * h[0, b] + h[0, a] * h[1, b])
        hac[1, nc] = np.sum(h[1, a] * h[1, b] + h[1, a] * h[0, b])
        hac[2, nc] = np.sum(h[2, a] * h[2, b] + h[2, a] * h[3, b])
        hac[3, nc] = np.sum(h[3, a] * h[3, b] + h[3, a] * h[2, b])
        hac[4, nc] = np.sum(h[4, a] * h[4, b])
        hac[:, nc] /= Nd - nc
    factor = dt_sample * 0.5 / (K_B * temperature * temperature * volume) * KAPPA
    rtc = np.zeros((5, Nc))
    for nc in range(1, Nc):
        rtc[:, nc] = rtc[:, nc - 1] + (hac[:, nc - 1] + hac[:, nc]) * factor
    return hac, rtc

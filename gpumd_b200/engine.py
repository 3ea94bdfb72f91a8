"""Python mirror of GPUMD's plugin surface for the hot path, over the libb200md C-ABI.

Class and method names follow the reference (paths relative to the GPUMD tree):
  Box            src/model/box.cuh:18-35
  Atom           src/model/atom.cuh:21-52        (SoA float64 device arrays)
  Potential      src/force/potential.cuh:20-113  (compute(box, type, position, potential, force, virial))
  NEP, LJ        src/force/nep.cuh:27-184, src/force/lj.cuh:31-49
  Force          src/force/force.cuh:27-85       (parse_potential, compute)
  Ensemble_NVE   src/integrate/ensemble_nve.cuh  (compute1, compute2)
The C++ adapters a GPUMD maintainer would compile into the reference live in gpumd_b200/host/.

Device arrays are torch CUDA tensors (torch = allocator + stream provider only); all arithmetic
happens in libb200md.so.  Without the library or without a GPU these classes raise.
"""
import ctypes as C

import numpy as np
import torch

from . import lib as _lib

K_B = 8.617343e-5                    # src/utilities/common.cuh:21
TIME_UNIT_CONVERSION = 1.018051e+1   # src/utilities/common.cuh:26


def _require_cuda():
    if not torch.cuda.is_available():
        raise _lib.B200mdError("no CUDA device: gpumd_b200 has no CPU fallback")


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class Box:
    """cpu_h[0..8] (row-major, lattice vectors as columns) + pbc flags."""

    def __init__(self, h, pbc=(1, 1, 1)):
        self.cpu_h = np.ascontiguousarray(np.asarray(h, dtype=np.float64).reshape(9))
        self.pbc = np.ascontiguousarray(np.asarray(pbc, dtype=np.int32).reshape(3))

    def get_volume(self):
        return abs(float(np.linalg.det(self.cpu_h.reshape(3, 3))))

    @property
    def _h(self):
        return self.cpu_h.ctypes.data_as(C.POINTER(C.c_double))

    @property
    def _p(self):
        return self.pbc.ctypes.data_as(C.POINTER(C.c_int))


class Atom:
    """Per-atom device state, same arrays and layouts as GPUMD's Atom."""

    def __init__(self, type_, position, mass, velocity=None, device="cuda"):
        _require_cuda()
        n = int(np.asarray(type_).shape[0])
        self.number_of_atoms = n
        dev = torch.device(device)
        self.type = torch.as_tensor(np.ascontiguousarray(type_, dtype=np.int32), device=dev)
        self.position_per_atom = torch.as_tensor(
            np.ascontiguousarray(position, dtype=np.float64).reshape(3 * n), device=dev)
        self.mass = torch.as_tensor(np.ascontiguousarray(mass, dtype=np.float64), device=dev)
        v = np.zeros(3 * n) if velocity is None else np.ascontiguousarray(
            velocity, dtype=np.float64).reshape(3 * n)
        self.velocity_per_atom = torch.as_tensor(v, device=dev)
        self.force_per_atom = torch.zeros(3 * n, dtype=torch.float64, device=dev)
        self.virial_per_atom = torch.zeros(9 * n, dtype=torch.float64, device=dev)
        self.potential_per_atom = torch.zeros(n, dtype=torch.float64, device=dev)


class Potential:
    """Abstract base, src/force/potential.cuh:20-113."""

    N1 = 0
    N2 = 0
    rc = 0.0

    def compute(self, box, type_, position, potential, force, virial):
        raise NotImplementedError


class NEP(Potential):
    """NEP(file_potential, num_atoms), src/force/nep.cu:100-395; compute = nep.cu:1356-1389."""

    def __init__(self, file_potential, num_atoms):
        _require_cuda()
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.b200md_nep_create(str(file_potential).encode(), int(num_atoms), C.byref(h)))
        self._h = h
        self._path = str(file_potential)
        self.N1, self.N2 = 0, int(num_atoms)
        self.rc = self._L.b200md_nep_rc(h)
        self.num_types = self._L.b200md_nep_info(h, 0)
        self.dim = self._L.b200md_nep_info(h, 1)
        self.MN_radial = self._L.b200md_nep_info(h, 3)
        self.MN_angular = self._L.b200md_nep_info(h, 4)
        self.symbols = [self._L.b200md_nep_symbol(h, t).decode() for t in range(self.num_types)]

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_nep_destroy(self._h)
            self._h = None

    def compute(self, box, type_, position, potential, force, virial):
        n = type_.shape[0]
        _lib.check(self._L.b200md_nep_compute(
            self._h, n, box._h, box._p, _ptr(type_), _ptr(position), _ptr(potential), _ptr(force),
            _ptr(virial), _stream()))

    def compute_host(self, box, type_, position, potential, force, virial):
        """Host (numpy or pinned torch CPU) buffers in and out; outputs are overwritten."""
        n = int(type_.shape[0])

        def p(a):
            return C.c_void_p(a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data)

        _lib.check(self._L.b200md_nep_compute_host(
            self._h, n, box._h, box._p, p(type_), p(position), p(potential), p(force), p(virial)))

    def check(self):
        _lib.check(self._L.b200md_nep_check(self._h, _stream()))

    def invalidate(self, n_new):
        _lib.check(self._L.b200md_nep_invalidate(self._h, int(n_new), _stream()))

    def set_accumulate(self, accumulate):
        """False: outputs are overwritten instead of added to (the caller may skip its zeroing pass)."""
        _lib.check(self._L.b200md_nep_set_accumulate(self._h, 1 if accumulate else 0))

    def set_owned(self, n_owned):
        """Spatial domains: only caller indices < n_owned get outputs (0 = all)."""
        _lib.check(self._L.b200md_nep_set_owned(self._h, int(n_owned)))

    def set_active_region(self, lo=None, hi=None):
        """Spatial domains: atoms outside [lo, hi) only serve as neighbours (None = no region)."""
        if lo is None or hi is None:
            _lib.check(self._L.b200md_nep_set_active_region(self._h, None, None))
            return
        lo, hi = ((C.c_double * 3)(*[float(x) for x in v]) for v in (lo, hi))
        _lib.check(self._L.b200md_nep_set_active_region(self._h, lo, hi))

    @property
    def num_rebuilds(self):
        return self._L.b200md_nep_info(self._h, 6)

    def profile(self, enable=True):
        _lib.check(self._L.b200md_nep_profile(self._h, 1 if enable else 0))

    def profile_read(self):
        """{stage name: (total ms, samples)} recorded since profile(True)."""
        ms = (C.c_float * 16)()
        cnt = (C.c_int * 16)()
        m = self._L.b200md_nep_profile_read(self._h, 16, ms, cnt)
        return {self._L.b200md_nep_stage_name(k).decode(): (float(ms[k]), int(cnt[k]))
                for k in range(m) if cnt[k] > 0}

    def mean_neighbors(self):
        out = (C.c_double * 3)()
        _lib.check(self._L.b200md_nep_mean_neighbors(self._h, out))
        return dict(skin=out[0], radial=out[1], angular=out[2])

    def export_neighbors(self, mn_r=None, mn_a=None):
        """(NN_radial, NL_radial[n,mn_r], NN_angular, NL_angular[n,mn_a]) of the last compute, in the
        caller's atom indices, ascending; -1 padded."""
        n = self.N2
        mn_r = mn_r or self.MN_radial
        mn_a = mn_a or self.MN_angular
        dev = torch.device("cuda")
        NNr = torch.zeros(n, dtype=torch.int32, device=dev)
        NLr = torch.full((n, mn_r), -1, dtype=torch.int32, device=dev)
        NNa = torch.zeros(n, dtype=torch.int32, device=dev)
        NLa = torch.full((n, mn_a), -1, dtype=torch.int32, device=dev)
        _lib.check(self._L.b200md_nep_export_neighbors(
            self._h, mn_r, _ptr(NNr), _ptr(NLr), mn_a, _ptr(NNa), _ptr(NLa), _stream()))
        self.check()
        return NNr.cpu().numpy(), NLr.cpu().numpy(), NNa.cpu().numpy(), NLa.cpu().numpy()

    def export_schedule(self):
        """The warp schedule of the last list rebuild: dict(nb, brick, seg_order, cell_start), or None
        when the handle runs the identity schedule."""
        nseg = self._L.b200md_nep_info(self._h, 7)
        if nseg == 0:
            return None
        dims = (C.c_int * 6)()
        _lib.check(self._L.b200md_nep_export_schedule(self._h, dims, None, None, _stream()))
        nb = [int(x) for x in dims[:3]]
        order = torch.zeros(nseg, dtype=torch.int32, device="cuda")
        start = torch.zeros(nb[0] * nb[1] * nb[2] + 1, dtype=torch.int32, device="cuda")
        _lib.check(self._L.b200md_nep_export_schedule(self._h, dims, _ptr(order), _ptr(start), _stream()))
        self.check()
        return dict(nb=nb, brick=[int(x) for x in dims[3:]], seg_order=order.cpu().numpy(),
                    cell_start=start.cpu().numpy())

    def export_descriptors(self):
        q = torch.zeros(self.dim, self.N2, dtype=torch.float32, device="cuda")
        _lib.check(self._L.b200md_nep_export_descriptors(self._h, _ptr(q), _stream()))
        return q.cpu().numpy()

    @property
    def num_tiles(self):
        """Type tiles of the last list rebuild (0: the SIMT hidden layer has none)."""
        return self._L.b200md_nep_info(self._h, 8)

    @property
    def tc_ctas(self):
        """CTAs of the last tensor-core hidden-layer launch (0: the last compute did not run it)."""
        return self._L.b200md_nep_info(self._h, 9)

    def export_tiles(self, n=None):
        """(slot[n] of every caller-order atom, tile_type[num_tiles]) of the last list rebuild."""
        n = n or self.N2
        slot = torch.full((n,), -1, dtype=torch.int32, device="cuda")
        tile_type = torch.full((max(self.num_tiles, 1),), -1, dtype=torch.int32, device="cuda")
        _lib.check(self._L.b200md_nep_export_tiles(self._h, _ptr(slot), _ptr(tile_type), _stream()))
        self.check()
        return slot.cpu().numpy(), tile_type[:self.num_tiles].cpu().numpy()

    def export_mlp(self, n=None):
        """(dU/dq [dim, n] times q_scaler, U table [num_types, K, n]) of the last compute, caller order;
        K = the padded radial basis (9, 13 or 17)."""
        n = n or self.N2
        k1 = next(k for k in (9, 13, 17) if k >= self._basis_radial())
        fp = torch.full((self.dim, n), float("nan"), dtype=torch.float32, device="cuda")
        u = torch.full((self.num_types, k1, n), float("nan"), dtype=torch.float32, device="cuda")
        _lib.check(self._L.b200md_nep_export_mlp(self._h, _ptr(fp), _ptr(u), _stream()))
        self.check()
        return fp.cpu().numpy(), u.cpu().numpy()

    def _basis_radial(self):
        with open(self._path) as f:
            for line in f:
                tok = line.split()
                if tok and tok[0] == "basis_size":
                    return int(tok[1]) + 1
        raise _lib.B200mdError("no basis_size line in " + str(self._path))


class LJ(Potential):
    """LJ potential; the file is the whole potential file ("lj Nt sym..." + Nt^2 lines),
    src/force/lj.cu:28-59; compute = lj.cu:184-219."""

    def __init__(self, file_potential, num_atoms):
        _require_cuda()
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.b200md_lj_create(str(file_potential).encode(), int(num_atoms), C.byref(h)))
        self._h = h
        self.N1, self.N2 = 0, int(num_atoms)
        self.rc = self._L.b200md_lj_rc(h)
        self.num_types = self._L.b200md_lj_info(h, 0)
        self.symbols = [self._L.b200md_lj_symbol(h, t).decode() for t in range(self.num_types)]

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_lj_destroy(self._h)
            self._h = None

    def compute(self, box, type_, position, potential, force, virial):
        n = type_.shape[0]
        _lib.check(self._L.b200md_lj_compute(
            self._h, n, box._h, box._p, _ptr(type_), _ptr(position), _ptr(potential), _ptr(force),
            _ptr(virial), _stream()))

    def check(self):
        _lib.check(self._L.b200md_lj_check(self._h, _stream()))

    def invalidate(self, n_new):
        _lib.check(self._L.b200md_lj_invalidate(self._h, int(n_new), _stream()))

    @property
    def num_rebuilds(self):
        return self._L.b200md_lj_info(self._h, 6)


class Tersoff1989(Potential):
    """Tersoff-1989, FP64 (src/force/tersoff1989.cu:31-586); file = whole potential file."""

    def __init__(self, file_potential, num_atoms):
        _require_cuda()
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.b200md_tersoff_create(str(file_potential).encode(), int(num_atoms), C.byref(h)))
        self._h = h
        self.N1, self.N2 = 0, int(num_atoms)
        self.rc = self._L.b200md_tersoff_rc(h)
        self.num_types = self._L.b200md_tersoff_info(h, 0)
        self.symbols = [self._L.b200md_tersoff_symbol(h, t).decode() for t in range(self.num_types)]

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_tersoff_destroy(self._h)
            self._h = None

    def compute(self, box, type_, position, potential, force, virial):
        n = type_.shape[0]
        _lib.check(self._L.b200md_tersoff_compute(
            self._h, n, box._h, box._p, _ptr(type_), _ptr(position), _ptr(potential), _ptr(force),
            _ptr(virial), _stream()))

    def check(self):
        _lib.check(self._L.b200md_tersoff_check(self._h, _stream()))

    def invalidate(self, n_new):
        _lib.check(self._L.b200md_tersoff_invalidate(self._h, int(n_new), _stream()))

    @property
    def num_rebuilds(self):
        return self._L.b200md_tersoff_info(self._h, 6)


class EAM(Potential):
    """Analytic EAM (eam_zhou_2004 / eam_dai_2006), src/force/eam.cu:28-580."""

    def __init__(self, file_potential, num_atoms):
        _require_cuda()
        self._L = _lib.load()
        h = C.c_void_p()
        _lib.check(self._L.b200md_eam_create(str(file_potential).encode(), int(num_atoms), C.byref(h)))
        self._h = h
        self.N1, self.N2 = 0, int(num_atoms)
        self.rc = self._L.b200md_eam_rc(h)
        self.num_types = self._L.b200md_eam_info(h, 0)
        self.symbols = [self._L.b200md_eam_symbol(h, t).decode() for t in range(self.num_types)]

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_eam_destroy(self._h)
            self._h = None

    def compute(self, box, type_, position, potential, force, virial):
        n = type_.shape[0]
        _lib.check(self._L.b200md_eam_compute(
            self._h, n, box._h, box._p, _ptr(type_), _ptr(position), _ptr(potential), _ptr(force),
            _ptr(virial), _stream()))

    def check(self):
        _lib.check(self._L.b200md_eam_check(self._h, _stream()))

    def invalidate(self, n_new):
        _lib.check(self._L.b200md_eam_invalidate(self._h, int(n_new), _stream()))

    @property
    def num_rebuilds(self):
        return self._L.b200md_eam_info(self._h, 6)


def compute_heat(atom, heat=None):
    """Per-atom heat current (compute_heat, src/measure/compute_heat.cu:66-90): heat[5N]."""
    n = atom.number_of_atoms
    if heat is None:
        heat = torch.zeros(5 * n, dtype=torch.float64, device=atom.velocity_per_atom.device)
    _lib.check(_lib.load().b200md_compute_heat(
        n, n, _ptr(atom.virial_per_atom), _ptr(atom.velocity_per_atom), _ptr(heat), n, _stream()))
    return heat


class HAC:
    """compute_hac, src/measure/hac.cu:32-280: sample the total heat current every sample_interval steps,
    then the autocorrelation hac[5, Nc] and the running thermal conductivity rtc[5, Nc] (W/mK)."""

    def __init__(self, number_of_steps, sample_interval, Nc):
        _require_cuda()
        self._L = _lib.load()
        self.Nc, self.Nd = int(Nc), int(number_of_steps) // int(sample_interval)
        self.sample_interval = int(sample_interval)
        h = C.c_void_p()
        _lib.check(self._L.b200md_hac_create(int(number_of_steps), int(sample_interval), int(Nc), C.byref(h)))
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_hac_destroy(self._h)
            self._h = None

    def process(self, step, atom):
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_hac_sample(self._h, int(step), n, n, _ptr(atom.virial_per_atom),
                                             _ptr(atom.velocity_per_atom), _stream()))

    def series(self):
        out = np.zeros(5 * self.Nd)
        _lib.check(self._L.b200md_hac_series(self._h, out.ctypes.data_as(C.POINTER(C.c_double)), _stream()))
        return out.reshape(5, self.Nd)

    def postprocess(self, time_step, temperature, volume):
        hac, rtc = np.zeros(5 * self.Nc), np.zeros(5 * self.Nc)
        dp = C.POINTER(C.c_double)
        _lib.check(self._L.b200md_hac_finish(self._h, float(time_step), float(temperature), float(volume),
                                             hac.ctypes.data_as(dp), rtc.ctypes.data_as(dp), _stream()))
        return hac.reshape(5, self.Nc), rtc.reshape(5, self.Nc)


class Force:
    """Force driver, src/force/force.cu: parse_potential (75-218) and compute (771-985)."""

    def __init__(self):
        self.potentials = []
        self._L = _lib.load()

    def parse_potential(self, file_potential, num_atoms):
        with open(file_potential) as f:
            first = f.readline().split()[0]
        if first.startswith("nep"):
            pot = NEP(file_potential, num_atoms)
        elif first == "lj":
            pot = LJ(file_potential, num_atoms)
        elif first == "tersoff_1989":
            pot = Tersoff1989(file_potential, num_atoms)
        elif first in ("eam_zhou_2004", "eam_dai_2006"):
            pot = EAM(file_potential, num_atoms)
        else:
            raise _lib.B200mdError(f"illegal potential model '{first}' for gpumd_b200")
        self.potentials = [pot]
        # a single NEP potential: let its final kernel store the outputs and drop the zeroing pass
        # (Force::compute zeroes because its potentials accumulate, force.cu:794-801)
        self._zero = True
        if isinstance(pot, NEP):
            pot.set_accumulate(False)
            self._zero = False
        return pot

    _fe = None

    def set_hnemd(self, fe):
        """compute_hnemd's driving force (Force::set_hnemd_parameters, force.cu:341-360): every following
        compute() adds W_i^T fe to each force and removes the net force.  fe = None switches it off
        (Force::finalize, force.cu:335-339)."""
        self._fe = None if fe is None else (C.c_double * 3)(*[float(x) for x in fe])

    def compute(self, box, position, type_, potential, force, virial):
        n = type_.shape[0]
        st = _stream()
        _lib.check(self._L.b200md_apply_pbc(n, box._h, box._p, _ptr(position), st))
        if self._zero:
            _lib.check(self._L.b200md_zero_properties(n, _ptr(potential), _ptr(force), _ptr(virial), st))
        self.potentials[0].compute(box, type_, position, potential, force, virial)
        if self._fe is not None:
            hnemd_drive(n, self._fe, virial, force)


_drive_scratch = {}


def hnemd_drive(n, fe, virial, force):
    """b200md_hnemd_drive on device arrays: force += W^T fe per atom, then the net force is removed
    (force.cu:857-897).  fe: 3 floats (1/A)."""
    L = _lib.load()
    dev = force.device
    need = int(L.b200md_hnemd_drive_scratch_bytes(int(n)))
    s = _drive_scratch.get(dev)
    if s is None or s.numel() < need:
        s = torch.zeros(need, dtype=torch.uint8, device=dev)  # the ticket starts at zero
        _drive_scratch[dev] = s
    fe3 = fe if isinstance(fe, C.Array) else (C.c_double * 3)(*[float(x) for x in fe])
    _lib.check(L.b200md_hnemd_drive(int(n), int(n), fe3, _ptr(virial), _ptr(force), _ptr(s), _stream()))


class HNEMD:
    """compute_hnemd, src/measure/hnemd_kappa.cu: process(step, atom) every step; take() after every
    output_interval-th step returns kappa[5] (W/mK: xx_in xx_out yy_in yy_out zz) and the heat sums
    rows[output_interval, 5] of the finished interval."""

    def __init__(self, output_interval, fe):
        _require_cuda()
        self._L = _lib.load()
        self.output_interval = int(output_interval)
        h = C.c_void_p()
        _lib.check(self._L.b200md_hnemd_create(self.output_interval, (C.c_double * 3)(*[float(x) for x in fe]),
                                               C.byref(h)))
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_hnemd_destroy(self._h)
            self._h = None

    def process(self, step, atom):
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_hnemd_sample(self._h, int(step), n, n, _ptr(atom.virial_per_atom),
                                               _ptr(atom.velocity_per_atom), _stream()))

    def take(self, volume, temperature):
        kappa, rows = np.zeros(5), np.zeros(5 * self.output_interval)
        dp = C.POINTER(C.c_double)
        _lib.check(self._L.b200md_hnemd_take(self._h, float(volume), float(temperature), kappa.ctypes.data_as(dp),
                                             rows.ctypes.data_as(dp), _stream()))
        return kappa, rows.reshape(self.output_interval, 5)


def _groups_arg(num_atoms, groups):
    """(sizes, contents) of b200md_*_create: None -> the whole system in atom order."""
    if groups is None:
        return np.array([int(num_atoms)], np.int32), None
    sizes = np.array([len(g) for g in groups], np.int32)
    contents = np.ascontiguousarray(np.concatenate([np.asarray(g, np.int32) for g in groups]))
    return sizes, contents


class _Correlation:
    """The shared shape of DOS, SDC, MSD and SHC: process(step, atom) every step, postprocess() at the end
    (or, for MSD, at any time).  groups: None for the whole system of num_atoms atoms, or a list of int
    arrays, the atom indices of each output group (Group::find_contents order)."""
    _kind = ""

    def _create(self, head, num_atoms, groups, tail=()):
        _require_cuda()
        self._L = _lib.load()
        sizes, contents = _groups_arg(num_atoms, groups)
        self.num_groups = sizes.shape[0]
        ip = C.POINTER(C.c_int)
        h = C.c_void_p()
        _lib.check(getattr(self._L, f"b200md_{self._kind}_create")(
            *head, self.num_groups, sizes.ctypes.data_as(ip),
            None if contents is None else contents.ctypes.data_as(ip), *tail, C.byref(h)))
        self._h = h

    def __del__(self):
        if getattr(self, "_h", None):
            getattr(self._L, f"b200md_{self._kind}_destroy")(self._h)
            self._h = None

    def _sample(self, step, n, x):
        _lib.check(getattr(self._L, f"b200md_{self._kind}_sample")(self._h, int(step), n, n, _ptr(x), _stream()))

    def _finish(self, rows_a, rows_b):
        a, b = np.zeros(self.num_groups * 3 * rows_a), np.zeros(self.num_groups * 3 * rows_b)
        dp = C.POINTER(C.c_double)
        _lib.check(getattr(self._L, f"b200md_{self._kind}_finish")(
            self._h, a.ctypes.data_as(dp), b.ctypes.data_as(dp), _stream()))
        return a.reshape(self.num_groups, 3, rows_a), b.reshape(self.num_groups, 3, rows_b)


class SHC(_Correlation):
    """compute_shc, src/measure/shc.cu.  process(step, atom) every step; postprocess() returns ki, ko
    [num_groups, 2Nc-1] and shc_i, shc_o [num_groups, num_omega]."""
    _kind = "shc"

    def __init__(self, sample_interval, Nc, direction, number_of_steps, num_atoms=None, groups=None):
        self.Nc, self.sample_interval = int(Nc), int(sample_interval)
        self._create((self.Nc, self.sample_interval, int(direction), int(number_of_steps)), num_atoms, groups)

    def process(self, step, atom):
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_shc_sample(self._h, int(step), n, n, _ptr(atom.virial_per_atom),
                                             _ptr(atom.velocity_per_atom), _stream()))

    def postprocess(self, time_step, num_omega, max_omega):
        g, nk, nw = self.num_groups, 2 * self.Nc - 1, int(num_omega)
        ki, ko, si, so = np.zeros(g * nk), np.zeros(g * nk), np.zeros(max(g * nw, 1)), np.zeros(max(g * nw, 1))
        dp = C.POINTER(C.c_double)
        _lib.check(self._L.b200md_shc_finish(
            self._h, float(time_step), nw, float(max_omega), ki.ctypes.data_as(dp), ko.ctypes.data_as(dp),
            si.ctypes.data_as(dp), so.ctypes.data_as(dp), _stream()))
        return ki.reshape(g, nk), ko.reshape(g, nk), si[:g * nw].reshape(g, nw), so[:g * nw].reshape(g, nw)


class DOS(_Correlation):
    """compute_dos, src/measure/dos.cu.  The masses are gathered from atom.mass once, here.
    postprocess() returns mvac [num_groups, 3, Nc] (normalised) and dos [num_groups, 3, num_dos_points]."""
    _kind = "dos"

    def __init__(self, sample_interval, Nc, omega_max, number_of_steps, time_step, atom, groups=None,
                 num_dos_points=None):
        self.Nc, self.sample_interval = int(Nc), int(sample_interval)
        self.num_dos_points = self.Nc if num_dos_points is None else int(num_dos_points)
        n = atom.number_of_atoms
        self._create((self.Nc, self.sample_interval, int(number_of_steps), float(time_step), float(omega_max),
                      self.num_dos_points), n, groups, (n, _ptr(atom.mass)))

    def process(self, step, atom):
        self._sample(step, atom.number_of_atoms, atom.velocity_per_atom)

    def postprocess(self):
        return self._finish(self.Nc, self.num_dos_points)


class SDC(_Correlation):
    """compute_sdc, src/measure/sdc.cu.  postprocess() returns vac (A^2/ps^2) and sdc (A^2/ps), each
    [num_groups, 3, Nc]."""
    _kind = "sdc"

    def __init__(self, sample_interval, Nc, number_of_steps, time_step, num_atoms=None, groups=None):
        self.Nc, self.sample_interval = int(Nc), int(sample_interval)
        self._create((self.Nc, self.sample_interval, int(number_of_steps), float(time_step)), num_atoms, groups)

    def process(self, step, atom):
        self._sample(step, atom.number_of_atoms, atom.velocity_per_atom)

    def postprocess(self):
        return self._finish(self.Nc, self.Nc)


class MSD(_Correlation):
    """compute_msd, src/measure/msd.cu, on the unwrapped positions of an UnwrappedPosition.
    postprocess() returns msd (A^2) and sdc (A^2/ps), each [num_groups, 3, Nc]; it may be called during
    the run and then covers every time origin sampled so far."""
    _kind = "msd"

    def __init__(self, sample_interval, Nc, number_of_steps, time_step, num_atoms=None, groups=None):
        self.Nc, self.sample_interval = int(Nc), int(sample_interval)
        self._create((self.Nc, self.sample_interval, int(number_of_steps), float(time_step)), num_atoms, groups)

    def process(self, step, unwrapped):
        """unwrapped: an UnwrappedPosition (or a [3 * n] float64 device tensor)."""
        x = getattr(unwrapped, "unwrapped_position", unwrapped)
        self._sample(step, x.shape[0] // 3, x)

    def postprocess(self):
        return self._finish(self.Nc, self.Nc)


class UnwrappedPosition:
    """atom.unwrapped_position of the reference (msd.cu:471-477, integrate.cu:347-374): starts as a copy
    of the current positions; call begin(atom) before an ensemble's compute1 and end(atom) after it."""

    def __init__(self, atom):
        _require_cuda()
        self._L = _lib.load()
        self.unwrapped_position = atom.position_per_atom.clone()
        self.position_temp = torch.empty_like(atom.position_per_atom)

    def begin(self, atom):
        _lib.check(self._L.b200md_unwrap_begin(atom.number_of_atoms, _ptr(atom.position_per_atom),
                                               _ptr(self.position_temp), _stream()))

    def end(self, atom):
        _lib.check(self._L.b200md_unwrap_end(atom.number_of_atoms, _ptr(atom.position_per_atom),
                                             _ptr(self.position_temp), _ptr(self.unwrapped_position), _stream()))


class Ensemble_NVE:
    """NVE integrator, src/integrate/ensemble_nve.cu:31-95 (velocity-Verlet + thermo)."""

    def __init__(self, num_atoms):
        _require_cuda()
        self._L = _lib.load()
        nbytes = self._L.b200md_thermo_scratch_bytes(int(num_atoms))
        self._scratch = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")

    # `fix` / `move` keywords (integrate.cu:1362-1470): label = Group::label of the grouping method
    fixed_group = -1
    move_group = -1

    def set_groups(self, label, fixed_group=-1, move_group=-1, move_velocity=(0.0, 0.0, 0.0)):
        """label: int32 group label per atom (host array or device tensor).  Atoms of fixed_group stay
        put, atoms of move_group translate with move_velocity (natural units); neither enters the
        temperature (ensemble.cu:111-174, 645-651)."""
        lab = torch.as_tensor(np.ascontiguousarray(label, dtype=np.int32)) if not torch.is_tensor(label) else label
        self._label = lab.to(device="cuda", dtype=torch.int32).contiguous()
        self.fixed_group, self.move_group = int(fixed_group), int(move_group)
        self._move_velocity = (C.c_double * 3)(*[float(v) for v in move_velocity])
        excluded = 0
        for g in (self.fixed_group, self.move_group):
            if g >= 0:
                excluded += int((self._label == g).sum().item())
        self._n_excluded = excluded

    def _vv(self, step1, time_step, atom):
        n = atom.number_of_atoms
        if self.fixed_group < 0 and self.move_group < 0:
            _lib.check(self._L.b200md_velocity_verlet(
                step1, n, float(time_step), _ptr(atom.mass), _ptr(atom.position_per_atom),
                _ptr(atom.velocity_per_atom), _ptr(atom.force_per_atom), _stream()))
        else:
            _lib.check(self._L.b200md_velocity_verlet_groups(
                step1, n, n, float(time_step), _ptr(atom.mass), _ptr(atom.position_per_atom),
                _ptr(atom.velocity_per_atom), _ptr(atom.force_per_atom), _ptr(self._label),
                self.fixed_group, self.move_group, self._move_velocity, _stream()))

    def compute1(self, time_step, box, atom, thermo=None):
        self._vv(1, time_step, atom)

    def compute2(self, time_step, box, atom, thermo):
        self._vv(0, time_step, atom)
        self.find_thermo(box.get_volume(), atom, thermo)

    def find_thermo(self, volume, atom, thermo):
        n = atom.number_of_atoms
        n_t = n - getattr(self, "_n_excluded", 0)  # ensemble.cu:645-651
        _lib.check(self._L.b200md_find_thermo(
            n, n_t, float(volume), _ptr(atom.mass), _ptr(atom.potential_per_atom),
            _ptr(atom.velocity_per_atom), _ptr(atom.virial_per_atom), _ptr(thermo),
            _ptr(self._scratch), _stream()))


class Ensemble_BER(Ensemble_NVE):
    """nvt_ber, src/integrate/ensemble_ber.cu:178-233: velocity-Verlet, thermo, Berendsen scaling
    with the factor computed on the device from thermo[0]."""

    def __init__(self, num_atoms, temperature, temperature_coupling):
        super().__init__(num_atoms)
        self.temperature = float(temperature)
        self.temperature_coupling = float(temperature_coupling)

    def compute2(self, time_step, box, atom, thermo):
        super().compute2(time_step, box, atom, thermo)
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_berendsen_temperature(
            n, n, self.temperature, self.temperature_coupling, _ptr(thermo),
            _ptr(atom.velocity_per_atom), _stream()))


K_B = 8.617343e-5  # common.cuh:21
PRESSURE_UNIT_CONVERSION = 1.602177e+2  # common.cuh:25


class Ensemble_NPT_BER(Ensemble_BER):
    """npt_ber, src/integrate/ensemble_ber.cu:38-64,88-172,237-285: Berendsen thermostat + barostat.
    target_pressure / elastic_modulus in GPa (1, 3 or 6 values, Voigt order for 6), tau_p in steps, as
    on the `ensemble npt_ber` line; converted like integrate.cu:690-700,1150-1153.  The box is updated
    in place on the host (Box.h), positions are rescaled on the device."""

    def __init__(self, num_atoms, temperature, temperature_coupling, target_pressure, elastic_modulus, tau_p):
        super().__init__(num_atoms, temperature, temperature_coupling)
        p = np.atleast_1d(np.asarray(target_pressure, dtype=np.float64))
        c = np.atleast_1d(np.asarray(elastic_modulus, dtype=np.float64))
        if p.shape[0] not in (1, 3, 6) or c.shape != p.shape:
            raise ValueError("npt_ber takes 1, 3 or 6 pressure components and as many elastic moduli")
        self.num_p = int(p.shape[0])
        pc = np.ones(6)
        pc[:self.num_p] = c
        coupling = np.where(pc > 2.0e3, 0.0, 1.0 / (float(tau_p) * 3.0 * pc))
        p6 = np.zeros(6)
        p6[:self.num_p] = p
        self._p0 = (C.c_double * 6)(*(p6 / PRESSURE_UNIT_CONVERSION))
        self._pc = (C.c_double * 6)(*(coupling * PRESSURE_UNIT_CONVERSION))
        self._zero3i = (C.c_int * 3)(0, 0, 0)
        self._zero3d = (C.c_double * 3)(0.0, 0.0, 0.0)

    def compute2(self, time_step, box, atom, thermo):
        super().compute2(time_step, box, atom, thermo)
        n = atom.number_of_atoms
        # box.cpu_h is updated in place (the next force call sees the new box)
        _lib.check(self._L.b200md_berendsen_pressure(
            n, n, self.num_p, self._p0, self._pc, self._zero3i, self._zero3d, box._p, box._h, _ptr(thermo),
            _ptr(atom.position_per_atom), _stream()))


class Ensemble_LAN(Ensemble_NVE):
    """nvt_lan, src/integrate/ensemble_lan.cu:29-41,92-124,190-269: half Langevin kick (c1 =
    exp(-0.5/Tc)) + momentum correction, velocity-Verlet, half kick.  cuRAND XORWOW per atom, seeded
    like the reference (seed 1804289383 = glibc's first rand(), what its -DDEBUG build passes)."""
    C1_EXPONENT = -0.5

    def __init__(self, num_atoms, temperature, temperature_coupling, seed=1804289383):
        super().__init__(num_atoms)
        self.temperature = float(temperature)
        self.c1 = float(np.exp(self.C1_EXPONENT / float(temperature_coupling)))
        h = C.c_void_p()
        _lib.check(self._L.b200md_langevin_create(int(num_atoms), int(seed), C.byref(h)))
        self._lan = h

    def __del__(self):
        if getattr(self, "_lan", None):
            self._L.b200md_langevin_destroy(self._lan)
            self._lan = None

    def _kick(self, atom):
        n = atom.number_of_atoms
        c2 = float(np.sqrt((1.0 - self.c1 * self.c1) * K_B * self.temperature))
        _lib.check(self._L.b200md_langevin_apply(self._lan, n, n, self.c1, c2, _ptr(atom.mass),
                                                 _ptr(atom.velocity_per_atom), _stream()))

    def compute1(self, time_step, box, atom, thermo=None):
        self._kick(atom)
        self._vv(1, time_step, atom)

    def compute2(self, time_step, box, atom, thermo):
        self._vv(0, time_step, atom)
        self._kick(atom)
        self.find_thermo(box.get_volume(), atom, thermo)


class Ensemble_BAO(Ensemble_LAN):
    """nvt_bao, src/integrate/ensemble_bao.cu:29-41,91-120,190-470: B A O A | force | B with the full
    Ornstein-Uhlenbeck step O (c1 = exp(-1/Tc))."""
    C1_EXPONENT = -1.0

    def _op(self, which, time_step, atom):
        n = atom.number_of_atoms
        label = _ptr(self._label) if self.fixed_group >= 0 else None
        _lib.check(self._L.b200md_baoab_operator(
            which, n, n, float(time_step), _ptr(atom.mass), _ptr(atom.position_per_atom),
            _ptr(atom.velocity_per_atom), _ptr(atom.force_per_atom), label, self.fixed_group, _stream()))

    def compute1(self, time_step, box, atom, thermo=None):
        self._op(1, time_step, atom)
        self._op(0, time_step, atom)
        self._kick(atom)
        self._op(0, time_step, atom)

    def compute2(self, time_step, box, atom, thermo):
        self._op(1, time_step, atom)
        self.find_thermo(box.get_volume(), atom, thermo)


class Ensemble_BDP(Ensemble_NVE):
    """nvt_bdp, src/integrate/ensemble_bdp.cu:69-101: velocity-Verlet, thermo, then the stochastic
    rescaling of Bussi et al.; generator and factor live on the device (seed 12345678 = the
    reference's -DDEBUG stream)."""

    def __init__(self, num_atoms, temperature, temperature_coupling, seed=12345678):
        super().__init__(num_atoms)
        h = C.c_void_p()
        _lib.check(self._L.b200md_bdp_create(int(num_atoms), float(temperature),
                                             float(temperature_coupling), int(seed), C.byref(h)))
        self._bdp = h

    def __del__(self):
        if getattr(self, "_bdp", None):
            self._L.b200md_bdp_destroy(self._bdp)
            self._bdp = None

    def compute2(self, time_step, box, atom, thermo):
        super().compute2(time_step, box, atom, thermo)
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_bdp_step(
            self._bdp, n, n, _ptr(thermo), _ptr(atom.velocity_per_atom), _stream()))


class Ensemble_NHC(Ensemble_NVE):
    """nvt_nhc, src/integrate/ensemble_nhc.cu:173-237 (chain integrated on the device)."""

    def __init__(self, num_atoms, temperature, temperature_coupling, time_step):
        super().__init__(num_atoms)
        h = C.c_void_p()
        _lib.check(self._L.b200md_nhc_create(int(num_atoms), float(temperature),
                                             float(temperature_coupling), float(time_step), C.byref(h)))
        self._nhc = h

    def __del__(self):
        if getattr(self, "_nhc", None):
            self._L.b200md_nhc_destroy(self._nhc)
            self._nhc = None

    def _thermostat(self, time_step, box, atom, thermo):
        n = atom.number_of_atoms
        self.find_thermo(box.get_volume(), atom, thermo)
        _lib.check(self._L.b200md_nhc_half_step(
            self._nhc, n, n, float(time_step), _ptr(thermo), _ptr(atom.velocity_per_atom), _stream()))

    def compute1(self, time_step, box, atom, thermo):
        self._thermostat(time_step, box, atom, thermo)
        super().compute1(time_step, box, atom, thermo)

    def compute2(self, time_step, box, atom, thermo):
        self._vv(0, time_step, atom)
        self._thermostat(time_step, box, atom, thermo)


def _group_contents(label):
    """Group::find_contents (group.cu:50-70) of a label array: sizes[g], atom indices by group."""
    lab = np.asarray(label.cpu() if torch.is_tensor(label) else label, dtype=np.int64).reshape(-1)
    sizes = np.bincount(lab).astype(np.int32) if lab.size else np.zeros(1, np.int32)
    contents = np.ascontiguousarray(np.argsort(lab, kind="stable").astype(np.int32))
    return sizes, contents


class _Ensemble_HEAT(Ensemble_NVE):
    """Direct NEMD with a heat source and a heat sink (groups of grouping method 0, `label`):
    the bath acts before velocity-Verlet step 1 and after step 2; no thermo is computed, as in the
    reference.  energy_transferred() synchronises and returns the energy (eV) moved from the system
    into the source and sink baths so far."""
    KIND = -1

    def __init__(self, label, source, sink, temperature, temperature_coupling, delta_temperature,
                 time_step, seed_source=0, seed_sink=0):
        lab = np.asarray(label.cpu() if torch.is_tensor(label) else label, dtype=np.int32).reshape(-1)
        super().__init__(lab.shape[0])
        self._label = torch.as_tensor(lab, device="cuda")
        sizes, contents = _group_contents(lab)
        ip = C.POINTER(C.c_int)
        h = C.c_void_p()
        _lib.check(self._L.b200md_heat_bath_create(
            self.KIND, lab.shape[0], sizes.shape[0], sizes.ctypes.data_as(ip), contents.ctypes.data_as(ip),
            int(source), int(sink), float(temperature), float(temperature_coupling), float(delta_temperature),
            float(time_step), int(seed_source), int(seed_sink), C.byref(h)))
        self._bath = h

    def __del__(self):
        if getattr(self, "_bath", None):
            self._L.b200md_heat_bath_destroy(self._bath)
            self._bath = None

    def set_groups(self, label=None, fixed_group=-1, move_group=-1, move_velocity=(0.0, 0.0, 0.0)):
        """fix / move on grouping method 0 (the label given at construction when label is None).  Only
        heat_lan allows a moving group (integrate.cu:69)."""
        if int(move_group) >= 0 and self.KIND != 0:
            raise ValueError("It is only allowed to use nvt_ber, nvt_nhc, or nvt_bdp with a moving group.")
        super().set_groups(self._label if label is None else label, fixed_group, move_group, move_velocity)

    def half(self, after_vv2, atom):
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_heat_bath_half(self._bath, int(after_vv2), n, n, _ptr(atom.mass),
                                                 _ptr(atom.velocity_per_atom), _stream()))

    def compute1(self, time_step, box, atom, thermo=None):
        self.half(0, atom)
        self._vv(1, time_step, atom)

    def compute2(self, time_step, box, atom, thermo=None):
        self._vv(0, time_step, atom)
        self.half(1, atom)

    def energy_transferred(self):
        out = np.zeros(2)
        _lib.check(self._L.b200md_heat_bath_energy(self._bath, out.ctypes.data_as(C.POINTER(C.c_double)),
                                                   _stream()))
        return out

    def state(self):
        """dict of the device record: chain[2,12], stat[2,5], vc[2,3], factor[2], energy[2]."""
        out = np.zeros(44)
        _lib.check(self._L.b200md_heat_bath_state(self._bath, out.ctypes.data_as(C.POINTER(C.c_double)),
                                                  _stream()))
        return {"chain": out[:24].reshape(2, 12), "stat": out[24:34].reshape(2, 5),
                "vc": out[34:40].reshape(2, 3), "factor": out[40:42], "energy": out[42:44]}


class Ensemble_HEAT_LAN(_Ensemble_HEAT):
    """heat_lan (type 22), ensemble_lan.cu:43-85,128-269: local Langevin half kicks on source and sink.
    seed_source / seed_sink: the reference's first and second rand() (1804289383, 846930886 under its
    -DDEBUG build)."""
    KIND = 0

    def __init__(self, label, source, sink, temperature, temperature_coupling, delta_temperature,
                 time_step=1.0 / TIME_UNIT_CONVERSION, seed_source=1804289383, seed_sink=846930886):
        super().__init__(label, source, sink, temperature, temperature_coupling, delta_temperature,
                         time_step, seed_source, seed_sink)


class Ensemble_HEAT_NHC(_Ensemble_HEAT):
    """heat_nhc (type 21), ensemble_nhc.cu:52-91,239-326: two Nose-Hoover chains on the relative
    kinetic energies of source and sink, scaling about each group's centre of mass."""
    KIND = 1

    def __init__(self, label, source, sink, temperature, temperature_coupling, delta_temperature, time_step):
        super().__init__(label, source, sink, temperature, temperature_coupling, delta_temperature, time_step)


class Ensemble_HEAT_BDP(_Ensemble_HEAT):
    """heat_bdp (type 23), ensemble_bdp.cu:50-62,103-149: stochastic velocity rescaling of source then
    sink after step 2, one MT19937 stream (seed 12345678 = the reference's -DDEBUG seed)."""
    KIND = 2

    def __init__(self, label, source, sink, temperature, temperature_coupling, delta_temperature,
                 time_step=1.0 / TIME_UNIT_CONVERSION, seed=12345678):
        super().__init__(label, source, sink, temperature, temperature_coupling, delta_temperature,
                         time_step, seed, 0)


COMPUTE_QUANTITIES = ("temperature", "potential", "force", "virial", "jp", "jk", "momentum")
COMPUTE_WIDTH = (1, 1, 3, 9, 3, 3, 3)


class Compute:
    """`compute`, src/measure/compute.cu: group sums of the selected quantities over grouping method
    `label`, sampled every sample_interval steps and averaged over output_interval samples.
    process(step, atom) every step returns None, or on an output step the averages as an array
    [columns, num_groups] in the reference's column order (temperature per atom)."""

    def __init__(self, label, sample_interval, output_interval, quantities):
        _require_cuda()
        self._L = _lib.load()
        mask = 0
        for q in quantities:
            if q not in COMPUTE_QUANTITIES:
                raise ValueError(f"Invalid property for compute: {q}")
            mask |= 1 << COMPUTE_QUANTITIES.index(q)
        self.sizes, contents = _group_contents(label)
        self.num_atoms = int(np.asarray(label.cpu() if torch.is_tensor(label) else label).reshape(-1).shape[0])
        self.num_groups = int(self.sizes.shape[0])
        self.sample_interval, self.output_interval = int(sample_interval), int(output_interval)
        ip = C.POINTER(C.c_int)
        h = C.c_void_p()
        _lib.check(self._L.b200md_group_compute_create(self.num_atoms, self.num_groups,
                                                       self.sizes.ctypes.data_as(ip),
                                                       contents.ctypes.data_as(ip), mask, C.byref(h)))
        self._h = h
        self.num_columns = self._L.b200md_group_compute_columns(h)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.b200md_group_compute_destroy(self._h)
            self._h = None

    def sample(self, atom):
        n = atom.number_of_atoms
        _lib.check(self._L.b200md_group_compute_sample(
            self._h, n, n, _ptr(atom.mass), _ptr(atom.potential_per_atom), _ptr(atom.force_per_atom),
            _ptr(atom.virial_per_atom), _ptr(atom.velocity_per_atom), _stream()))

    def take(self, num_samples=None):
        out = np.zeros(self.num_columns * self.num_groups)
        _lib.check(self._L.b200md_group_compute_take(
            self._h, int(num_samples or self.output_interval), out.ctypes.data_as(C.POINTER(C.c_double)),
            _stream()))
        return out.reshape(self.num_columns, self.num_groups)

    def process(self, step, atom):
        """Compute::process, compute.cu:351-538."""
        if (step + 1) % self.sample_interval != 0:
            return None
        self.sample(atom)
        if ((step + 1) // self.sample_interval) % self.output_interval == 0:
            return self.take()
        return None


def launch_count():
    return _lib.load().b200md_launch_count()

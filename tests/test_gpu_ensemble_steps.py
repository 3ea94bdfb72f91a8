"""Every ensemble, step by step, against the float64 restatement of tests/ensemble_oracle.py: after each
piece of each step the device state is compared with the restatement applied to the device's own state
before that piece, so nothing diverges and no tolerance grows with time.

  - Engine level (gpumd_b200.engine): NEP PbTe and LJ Ar, {nve, nvt_ber, nvt_nhc, nvt_bdp} x {no groups,
    fix, fix + move on grouping method 0, fix + move on method 1 of a two-method label set}, and npt_ber
    in every form (isotropic, 3 components periodic / with an open direction / with a direction stiffer
    than 2000 GPa, 6 components on a triclinic box, isotropic with a fixed group).
  - Driver level (the b200md executable): the same restatement frame to frame of dump_xyz output.

Tolerances: velocity-Verlet and the group rules bit for bit; velocities a thermostat scaled rtol 1e-12
(device exp / sqrt / log may sit 1 ulp from the host's); box and positions after the barostat 1e-14;
the force driver's wrap into the box (x -> h (h^-1 x)) 1e-12 A."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN
from ensemble_oracle import EnsembleStep
from gpumd_b200.structures import TIME_UNIT_CONVERSION, fcc, init_velocities, nep_type_order, rocksalt_pbte

pytestmark = pytest.mark.gpu

STEPS = 20
MOVE_VELOCITY = (0.002 * TIME_UNIT_CONVERSION, -0.001 * TIME_UNIT_CONVERSION, 0.0015 * TIME_UNIT_CONVERSION)


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def tilt(s, xy, xz, yz):
    """The same crystal on a triclinic cell: fractional coordinates kept, lattice vectors b and c tilted."""
    H = s["h"].reshape(3, 3)
    frac = np.linalg.solve(H, s["pos"])
    H2 = H.copy()
    H2[0, 1], H2[0, 2], H2[1, 2] = xy, xz, yz
    return dict(s, h=H2.reshape(9).copy(), pos=np.ascontiguousarray(H2 @ frac))


def system(pot, triclinic=False, open_z=False):
    """(structure, potential file, initial temperature, time step in fs)."""
    if pot == "nep":
        s, f, T0, dt = rocksalt_pbte(6, rattle=0.02, seed=1), "nep_PbTe.txt", 300.0, 1.0  # 1728 atoms
    else:
        s, f, T0, dt = fcc(8, 5.60, rattle=0.02, seed=1), "lj_Ar_10A.txt", 40.0, 2.0  # 2048 atoms
    if triclinic:
        L = s["h"][0]
        s = tilt(s, 0.08 * L, -0.05 * L, 0.06 * L)
    if open_z:
        s = dict(s, pbc=np.array([1, 1, 0], np.int32))
    return s, f, T0, dt


def labels(s):
    """Two grouping methods: method 0 cuts the cell into four slabs along a, method 1 labels atoms by index
    modulo 3."""
    frac = np.linalg.solve(s["h"].reshape(3, 3), s["pos"])
    g0 = np.clip((np.mod(frac[0], 1.0) * 4).astype(np.int32), 0, 3)
    g1 = (np.arange(s["type"].shape[0]) % 3).astype(np.int32)
    return g0, g1


GROUPS = {
    "none": None,
    "fix": (0, 1, -1),            # (grouping method, fixed group, moving group)
    "fix_move_m0": (0, 0, 3),
    "fix_move_m1": (1, 2, 0),
}

NPT = {
    # name: (target pressures GPa, elastic moduli GPa, triclinic, open z, fixed group)
    "iso": ([0.0], [50.0], False, False, False),
    "xyz": ([0.0, 0.1, -0.1], [50.0, 40.0, 60.0], False, False, False),
    "xyz_open_z": ([0.0, 0.1, -0.1], [50.0, 40.0, 60.0], False, True, False),
    "xyz_stiff_y": ([0.0, 0.1, -0.1], [50.0, 2500.0, 60.0], False, False, False),
    "triclinic6": ([0.0, 0.1, -0.1, 0.05, -0.05, 0.02], [50.0, 40.0, 60.0, 30.0, 30.0, 30.0], True, False,
                   False),
    "iso_fix": ([0.0], [50.0], False, False, True),
}


def make_ensemble(eng, kind, n, T, dt, npt=None):
    if kind == "nve":
        return eng.Ensemble_NVE(n)
    if kind == "nvt_ber":
        return eng.Ensemble_BER(n, T, 50.0)
    if kind == "nvt_nhc":
        return eng.Ensemble_NHC(n, T, 50.0, dt)
    if kind == "nvt_bdp":
        return eng.Ensemble_BDP(n, T, 50.0)
    if kind == "nvt_lan":
        return eng.Ensemble_LAN(n, T, 50.0)
    if kind == "nvt_bao":
        return eng.Ensemble_BAO(n, T, 50.0)
    return eng.Ensemble_NPT_BER(n, T, 50.0, npt[0], npt[1], 200.0)


class Device:
    """An engine run whose state is read back after every piece of a step."""

    def __init__(self, eng, s, potfile, T0, kind, dt, npt=None):
        import torch
        self.torch = torch
        self.n = n = s["type"].shape[0]
        vel = init_velocities(s["mass"], T0, seed=42)
        self.atom = eng.Atom(s["type"], s["pos"], s["mass"], vel)
        self.box = eng.Box(s["h"], s["pbc"])
        self.force = eng.Force()
        self.pot = self.force.parse_potential(GOLDEN / potfile, n)
        self.ens = make_ensemble(eng, kind, n, T0, dt, npt)
        self.thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
        self.dt = dt

    def get(self, t, rows):
        return t.cpu().numpy().reshape(rows, self.n).copy()

    def state(self):
        a = self.atom
        return self.get(a.position_per_atom, 3), self.get(a.velocity_per_atom, 3), self.box.cpu_h.copy()

    def forces(self):
        a = self.atom
        self.force.compute(self.box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom,
                           a.virial_per_atom)
        return (self.get(a.position_per_atom, 3), self.get(a.force_per_atom, 3),
                a.potential_per_atom.cpu().numpy().copy(), self.get(a.virial_per_atom, 9))


def check(got, want, exact, rtol, what, scale=None):
    if exact:
        assert np.array_equal(got, want), (what, np.abs(got - want).max())
    else:
        atol = rtol * (np.abs(want).max() if scale is None else scale)
        assert np.allclose(got, want, rtol=rtol, atol=atol), (what, np.abs(got - want).max())


LANGEVIN = ("nvt_lan", "nvt_bao")


def run_locked(oracle, dev, ref, kind, steps=STEPS, fixed=None, moving=None):
    """Step the device and restate each piece from the device state before it.  The Langevin kinds draw
    their noise from the restated cuRAND stream, in step with the device's: their velocities agree to
    1e-13 of the largest, the device's sincospi and log sitting a few ulp from the host's libm."""
    scaled = kind != "nve"
    npt = kind == "npt_ber"
    noisy = kind in LANGEVIN
    tol = 1e-13 if noisy else 1e-12
    _, f0, _, _ = dev.forces()
    for step in range(steps):
        p0, v0, h0 = dev.state()
        dev.ens.compute1(dev.dt, dev.box, dev.atom, dev.thermo)
        p1, v1, _ = dev.state()
        rp1, rv1 = ref.compute1(h0, p0, v0, f0)
        # nvt_nhc scales and the Langevin kinds kick before the drift; everything else is bit for bit
        check(p1, rp1, kind != "nvt_nhc" and not noisy, tol, f"{step}: positions after compute1")
        check(v1, rv1, kind != "nvt_nhc" and not noisy, tol, f"{step}: velocities after compute1")
        pw, f1, pe1, vir1 = dev.forces()
        assert np.allclose(pw, oracle.apply_pbc(h0, ref.pbc, p1), rtol=0, atol=1e-12), step
        dev.ens.compute2(dev.dt, dev.box, dev.atom, dev.thermo)
        p2, v2, h2 = dev.state()
        th = dev.thermo.cpu().numpy()
        rp2, rv2, rh2, rth = ref.compute2(h0, pw, v1, f1, pe1, vir1)
        assert np.allclose(th[:2], rth[:2], rtol=1e-12, atol=0), (step, th[:2], rth[:2])
        check(th[2:], rth[2:], False, 1e-12, f"{step}: stress")
        check(v2, rv2, not scaled, tol, f"{step}: velocities after compute2")
        check(p2, rp2, not npt, 1e-14, f"{step}: positions after compute2")
        check(h2, rh2, not npt, 1e-14, f"{step}: box")
        # the group rules, on the device state itself
        # (nvt_lan's last kick and nvt_bao's O step draw noise for the fixed atoms too)
        if fixed is not None:
            assert np.array_equal(p1[:, fixed], p0[:, fixed]), step
            assert kind == "nvt_bao" or np.all(v1[:, fixed] == 0), step
            assert kind == "nvt_lan" or np.all(v2[:, fixed] == 0), step
        if moving is not None and moving.any():
            assert np.all(v1[:, moving] == 0) and np.all(v2[:, moving] == 0), step
        f0 = f1
    dev.pot.check()


# NEP runs every grouping; LJ the ungrouped case and fix + move on grouping method 1
THERMOSTAT_CASES = [(pot, kind, groups) for kind in ("nve", "nvt_ber", "nvt_nhc", "nvt_bdp")
                    for pot, gs in (("nep", list(GROUPS)), ("lj", ["none", "fix_move_m1"])) for groups in gs]


@pytest.mark.parametrize("pot,kind,groups", THERMOSTAT_CASES)
def test_thermostat_steps_match_restatement(oracle, eng, pot, kind, groups):
    s, potfile, T0, dt_fs = system(pot)
    dt = dt_fs / TIME_UNIT_CONVERSION
    dev = Device(eng, s, potfile, T0, kind, dt)
    grp = GROUPS[groups]
    fixed = moving = None
    label = None
    kw = {}
    if grp is not None:
        method, fg, mg = grp
        label = labels(s)[method]
        mv = MOVE_VELOCITY if mg >= 0 else (0.0, 0.0, 0.0)
        dev.ens.set_groups(label, fixed_group=fg, move_group=mg, move_velocity=mv)
        kw = dict(label=label, fixed_group=fg, move_group=mg, move_velocity=mv)
        fixed = label == fg
        moving = label == mg if mg >= 0 else None
    ref = EnsembleStep(kind, s["mass"], dt, pbc=s["pbc"], temperature=T0, temperature_coupling=50.0, **kw)
    run_locked(oracle, dev, ref, kind, fixed=fixed, moving=moving)


# NEP runs every form; LJ the isotropic, open and triclinic ones
NPT_CASES = [("nep", c) for c in NPT] + [("lj", c) for c in ("iso", "xyz_open_z", "triclinic6")]


@pytest.mark.parametrize("pot,case", NPT_CASES)
def test_npt_ber_steps_match_restatement(oracle, eng, pot, case):
    p, c, triclinic, open_z, with_fix = NPT[case]
    s, potfile, T0, dt_fs = system(pot, triclinic=triclinic, open_z=open_z)
    dt = dt_fs / TIME_UNIT_CONVERSION
    dev = Device(eng, s, potfile, T0, "npt_ber", dt, npt=(p, c))
    kw, fixed = {}, None
    if with_fix:
        label = labels(s)[0]
        dev.ens.set_groups(label, fixed_group=2)
        kw = dict(label=label, fixed_group=2)
        fixed = label == 2
    ref = EnsembleStep("npt_ber", s["mass"], dt, pbc=s["pbc"], temperature=T0, temperature_coupling=50.0,
                       target_pressure=p, elastic_modulus=c, tau_p=200.0, **kw)
    h_start = s["h"].copy()
    run_locked(oracle, dev, ref, "npt_ber", fixed=fixed)
    h_end = dev.box.cpu_h
    # directions the barostat leaves alone keep their box vectors bit for bit; the others moved
    untouched = {"xyz_open_z": [8], "xyz_stiff_y": [4]}.get(case, [])
    for k in untouched:
        assert h_end[k] == h_start[k]
    assert h_end[0] != h_start[0]
    if case == "triclinic6":
        assert h_end[1] != h_start[1]


@pytest.mark.parametrize("kind", ["nvt_lan", "nvt_bao"])
def test_langevin_ensembles_keep_the_group_rules(eng, kind):
    """The group rules of the Langevin ensembles on their own (test_gpu_langevin_steps.py restates the
    whole steps, noise included).  Fixed atoms never move: no
    half of a step changes their positions (the force driver's wrap rounds them by at most 1e-12 A).
    nvt_bao's B step leaves their velocities at zero.  The total momentum is zero after each Langevin kick: at the
    end of an nvt_lan step and after the O step of nvt_bao."""
    s, potfile, T0, dt_fs = system("nep")
    dt = dt_fs / TIME_UNIT_CONVERSION
    dev = Device(eng, s, potfile, T0, kind, dt)
    label = labels(s)[1]
    dev.ens.set_groups(label, fixed_group=1)
    fixed = label == 1
    mass = s["mass"]
    dev.forces()
    start, _, _ = dev.state()
    for step in range(STEPS):
        p0, _, _ = dev.state()
        dev.ens.compute1(dev.dt, dev.box, dev.atom, dev.thermo)
        p1, v1, _ = dev.state()
        assert np.array_equal(p1[:, fixed], p0[:, fixed]), step
        if kind == "nvt_bao":  # B A O A: the O step's kick removes the momentum of all atoms
            assert np.abs((v1 * mass).sum(axis=1)).max() < 1e-10, step
        pw, _, _, _ = dev.forces()
        dev.ens.compute2(dev.dt, dev.box, dev.atom, dev.thermo)
        p2, v2, _ = dev.state()
        assert np.array_equal(p2[:, fixed], pw[:, fixed]), step
        if kind == "nvt_bao":
            assert np.all(v2[:, fixed] == 0), step
        else:
            assert np.abs((v2 * mass).sum(axis=1)).max() < 1e-10, step
        assert np.abs(v2[:, ~fixed]).max() > 0
    end, _, _ = dev.state()
    assert np.allclose(end[:, fixed], start[:, fixed], rtol=0, atol=1e-12)
    dev.pot.check()


# ---------------------------------------------------------------- driver level: the b200md executable

def write_model(path, s, symbols, vel, groups):
    """model.xyz with velocities (A/fs; none if vel is None) and one group column per grouping method."""
    n = s["type"].shape[0]
    h = np.asarray(s["h"], dtype=np.float64).reshape(3, 3)
    lat = " ".join(f"{v:.17g}" for v in h.T.reshape(-1))
    pbc = " ".join("T" if p else "F" for p in s["pbc"])
    v = np.zeros((0, n)) if vel is None else np.asarray(vel) / TIME_UNIT_CONVERSION
    props = "species:S:1:pos:R:3" + ("" if vel is None else ":vel:R:3") + f":group:I:{len(groups)}"
    with open(path, "w") as f:
        f.write(f"{n}\npbc=\"{pbc}\" lattice=\"{lat}\" properties={props}\n")
        for i in range(n):
            f.write(f"{symbols[s['type'][i]]} " + " ".join(f"{x:.17g}" for x in
                                                          (*s["pos"][:, i], *v[:, i])) +
                    "".join(f" {g[i]}" for g in groups) + "\n")


VIRIAL_COLUMNS = [0, 3, 4, 6, 1, 5, 7, 8, 2]  # dump_xyz's row-major 3x3 columns -> GPUMD's component order


def read_frames(path):
    """dump_xyz frames (`precision double mass velocity force potential virial`): per frame h[9] and
    mass, pos, vel (natural units), force, pe, virial [9, N] in GPUMD's component order."""
    lines = open(path).read().splitlines()
    frames, i = [], 0
    while i < len(lines):
        n = int(lines[i])
        hdr = lines[i + 1]
        lat = np.array([float(x) for x in hdr.split('Lattice="')[1].split('"')[0].split()])
        rows = np.array([ln.split()[1:] for ln in lines[i + 2:i + 2 + n]], dtype=np.float64).T
        vir = np.empty((9, n))
        vir[VIRIAL_COLUMNS] = rows[11:20]
        frames.append(dict(h=lat.reshape(3, 3).T.reshape(9).copy(), pos=rows[0:3], mass=rows[3],
                           vel=rows[4:7] * TIME_UNIT_CONVERSION, force=rows[7:10], pe=rows[10],
                           virial=vir))
        i += n + 2
    return frames


def read_thermo(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#")], dtype=np.float64)


def single_point_force(eng, s, potfile, pos, h):
    """Forces at `pos` from the engine's force driver, which wraps positions into the box and calls the
    same kernels as the executable's: the forces the executable's own first evaluation finds."""
    import torch
    n = s["type"].shape[0]
    atom = eng.Atom(s["type"], pos, s["mass"])
    box = eng.Box(h, s["pbc"])
    force = eng.Force()
    force.parse_potential(GOLDEN / potfile, n)
    force.compute(box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
                  atom.virial_per_atom)
    force.potentials[0].check()
    torch.cuda.synchronize()
    return atom.force_per_atom.cpu().numpy().reshape(3, n).copy()


DUMP = "precision double mass velocity force potential virial"

DRIVER = {
    # case: (run.in body after `potential`, restatement kind, ensemble kw, grouping, triclinic, open z)
    "nvt_bdp_fix_move": ("ensemble nvt_bdp 300 300 50 seed 12345678\nfix 0 0\nmove 0 3 0.002 -0.001 0.0015\n",
                         "nvt_bdp", {}, (0, 0, 3), False, False),
    "nvt_nhc_fix_move": ("ensemble nvt_nhc 300 300 50\nfix 1 2\nmove 1 0 0.002 -0.001 0.0015\n",
                         "nvt_nhc", {}, (1, 2, 0), False, False),
    "nvt_ber_fix_method1": ("ensemble nvt_ber 300 300 50\nfix 1 1\n", "nvt_ber", {}, (1, 1, -1), False, False),
    "npt_ber_xyz_open_z": ("ensemble npt_ber 300 300 50 0 0.1 -0.1 50 40 60 200\n", "npt_ber",
                           dict(target_pressure=[0, 0.1, -0.1], elastic_modulus=[50, 40, 60], tau_p=200.0),
                           None, False, True),
    "npt_ber_triclinic6": ("ensemble npt_ber 300 300 50 0 0.1 -0.1 0.05 -0.05 0.02 50 40 60 30 30 30 200\n",
                           "npt_ber", dict(target_pressure=[0, 0.1, -0.1, 0.05, -0.05, 0.02],
                                           elastic_modulus=[50, 40, 60, 30, 30, 30], tau_p=200.0),
                           None, True, False),
}


def restate_run(frames, thermo, ref, f_start, h_start, pos_start, vel_start, first_step_fp32=False):
    """Restate frame k -> k+1 of one run and compare positions, velocities, box and T (thermo None: no
    T).  first_step_fp32:
    f_start reproduces the executable's first force evaluation only to FP32 rounding, so the first step
    is held to that (1e-7 of a force moves a position by ~1e-11 A in one step)."""
    prev = dict(h=h_start, pos=pos_start, vel=vel_start, force=f_start)
    for k, fr in enumerate(frames):
        p, v, h, th = ref.step(prev["h"], prev["pos"], prev["vel"], prev["force"], fr["force"], fr["pe"],
                               fr["virial"])
        loose = first_step_fp32 and k == 0
        assert np.allclose(fr["pos"], p, rtol=1e-14, atol=1e-9 if loose else 1e-12), \
            (k, np.abs(fr["pos"] - p).max())
        vs = np.abs(v).max()
        assert np.allclose(fr["vel"], v, rtol=1e-12, atol=(1e-7 if loose else 1e-12) * vs), \
            (k, np.abs(fr["vel"] - v).max() / vs)
        assert np.allclose(fr["h"], h, rtol=1e-14, atol=1e-14 * np.abs(h).max()), k
        if thermo is not None:
            assert thermo[k, 0] == pytest.approx(th[0], rel=1e-7 if loose else 1e-9), k
        prev = fr


def driver_setup(tmp_path, triclinic=False, open_z=False):
    s, potfile, T0, _ = system("nep", triclinic=triclinic, open_z=open_z)
    sym = nep_type_order(GOLDEN / potfile)
    vel = init_velocities(s["mass"], T0, seed=42)
    groups = labels(s)
    write_model(tmp_path / "model.xyz", s, sym, vel, groups)
    shutil.copyfile(GOLDEN / potfile, tmp_path / "potential.txt")
    # the state the executable starts from: model.xyz parsed the way it parses it
    vel_read = np.array([[float(f"{x:.17g}") for x in row] for row in vel / TIME_UNIT_CONVERSION]) \
        * TIME_UNIT_CONVERSION
    return s, potfile, groups, vel_read


def run_exe(tmp_path):
    from gpumd_b200 import build
    exe = build.build_host()
    r = subprocess.run([str(exe)], cwd=tmp_path, capture_output=True, text=True, timeout=600,
                       env=dict(os.environ))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r


@pytest.mark.parametrize("case", list(DRIVER))
def test_driver_steps_match_restatement(oracle, eng, tmp_path, case):
    """The executable's ensembles with `fix` / `move` on either grouping method and npt_ber with an open
    direction or six components, restated frame to frame from dump_xyz.  nvt_bdp with fix + move draws
    its noise for ndeg = 3 (N - N_fixed - N_move) degrees of freedom, as the reference does."""
    body, kind, kw, grp, triclinic, open_z = DRIVER[case]
    s, potfile, groups, vel0 = driver_setup(tmp_path, triclinic, open_z)
    (tmp_path / "run.in").write_text(
        f"potential potential.txt\n{body}time_step 1\ndump_thermo 1\ndump_xyz 1 dump.xyz {DUMP}\nrun {STEPS}\n")
    run_exe(tmp_path)
    frames = read_frames(tmp_path / "dump.xyz")
    thermo = read_thermo(tmp_path / "thermo.out")
    assert len(frames) == thermo.shape[0] == STEPS
    mass = frames[0]["mass"]
    if grp is not None:
        method, fg, mg = grp
        mv = MOVE_VELOCITY if mg >= 0 else (0.0, 0.0, 0.0)
        kw = dict(kw, label=groups[method], fixed_group=fg, move_group=mg, move_velocity=mv)
    ref = EnsembleStep(kind, mass, 1.0 / TIME_UNIT_CONVERSION, pbc=s["pbc"], temperature=300.0,
                       temperature_coupling=50.0, **kw)
    f_start = single_point_force(eng, s, potfile, s["pos"], s["h"])
    restate_run(frames, thermo, ref, f_start, s["h"], s["pos"], vel0)


def test_driver_second_run_resets_groups_and_chain(oracle, eng, tmp_path):
    """Two runs: nvt_nhc with fix + move, then the same ensemble without them and at half the time step.
    `run` ends the groups (run.cu's Integrate::finalize), so every atom integrates in the second run and
    counts for T, and the second run starts a fresh chain with masses from the new time step."""
    s, potfile, groups, vel0 = driver_setup(tmp_path)
    (tmp_path / "run.in").write_text(
        "potential potential.txt\nensemble nvt_nhc 300 300 50\nfix 0 0\nmove 0 3 0.002 -0.001 0.0015\n"
        f"time_step 1\ndump_thermo 1\ndump_xyz 1 a.xyz {DUMP}\nrun {STEPS}\n"
        f"time_step 0.5\ndump_thermo 1\ndump_xyz 1 b.xyz {DUMP}\nrun {STEPS}\n")
    run_exe(tmp_path)
    a, b = read_frames(tmp_path / "a.xyz"), read_frames(tmp_path / "b.xyz")
    thermo = read_thermo(tmp_path / "thermo.out")
    assert len(a) == len(b) == STEPS and thermo.shape[0] == 2 * STEPS
    mass = a[0]["mass"]
    ref = EnsembleStep("nvt_nhc", mass, 1.0 / TIME_UNIT_CONVERSION, pbc=s["pbc"], temperature=300.0,
                       temperature_coupling=50.0, label=groups[0], fixed_group=0, move_group=3,
                       move_velocity=MOVE_VELOCITY)
    f_start = single_point_force(eng, s, potfile, s["pos"], s["h"])
    restate_run(a, thermo[:STEPS], ref, f_start, s["h"], s["pos"], vel0)
    last = a[-1]
    ref2 = EnsembleStep("nvt_nhc", mass, 0.5 / TIME_UNIT_CONVERSION, pbc=s["pbc"], temperature=300.0,
                        temperature_coupling=50.0)
    # the second run starts with a force evaluation on the executable's own neighbour list, which a fresh
    # single-point evaluation sums in another order: its first step is compared at FP32 resolution
    f_start = single_point_force(eng, s, potfile, last["pos"], last["h"])
    restate_run(b, thermo[STEPS:], ref2, f_start, last["h"], last["pos"], last["vel"], first_step_fp32=True)
    # the atoms that were fixed or moving in the first run integrate in the second
    was_held = (groups[0] == 0) | (groups[0] == 3)
    assert np.all(a[-1]["vel"][:, was_held] == 0)
    assert np.abs(b[-1]["vel"][:, was_held]).min(axis=0).max() > 0
    assert not np.array_equal(b[-1]["pos"][:, groups[0] == 0], a[-1]["pos"][:, groups[0] == 0])

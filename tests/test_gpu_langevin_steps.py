"""nvt_lan, nvt_bao and heat_lan draw for draw: the device's cuRAND XORWOW noise against the numpy
restatement of tests/curand_oracle.py, at every level that seeds or consumes it.

  - Kernel level: b200md_langevin_create / _apply and heat_lan's b200md_heat_bath_half through the C-ABI,
    on atom counts around the block size, padded velocity layouts (stride > n), 64-bit seeds, several
    consecutive calls (the cached second Box-Muller value crosses calls) and group contents that are not
    contiguous.
  - Engine level: the run_locked restatement of test_gpu_ensemble_steps.py, each piece of each step
    restated from the device's own state before it.
  - Driver level: the b200md executable's dump_xyz frames restated frame to frame, each generator's
    seed predicted from glibc's rand() stream the way the driver consumes it.

Velocities agree within 1e-13 of the largest |v|: the device's sincospi and log sit a few ulp from the
host libm the restatement uses.  Each test prints the largest gap it met."""
import ctypes as C

import numpy as np
import pytest

import test_gpu_ensemble_steps as S
from curand_oracle import GlibcRand, XorwowStates
from conftest import GOLDEN
from ensemble_oracle import EnsembleStep
from nemd_oracle import HeatLan
from gpumd_b200.structures import TIME_UNIT_CONVERSION, nep_type_order

pytestmark = pytest.mark.gpu
K_B = 8.617343e-5
SEEDS = [0, 1804289383, 846930886, 2 ** 32 + 5, 2 ** 63 + 12345]
C1S = [0.0, 0.5, float(np.exp(-0.5 / 50.0)), 1.0]
VEL_RTOL = 1e-13


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


@pytest.fixture(scope="module")
def lib(eng):
    from gpumd_b200 import lib as L
    return L


def padded(vel, stride, rng):
    """[3 * stride] device layout of vel [3, n], the padding filled with noise that must survive."""
    n = vel.shape[1]
    buf = rng.normal(size=(3, stride)) * 7.0
    buf[:, :n] = vel
    return buf


def gap(got, want, scale):
    return float(np.abs(got - want).max() / scale) if got.size else 0.0


# ---------------------------------------------------------------- kernel level

@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("n", [1, 255, 256, 257, 4097, 100_003])
def test_langevin_kernel_draws_match_restatement(lib, n, seed):
    """Seven consecutive applies at c1 in {0, 1/2, exp(-1/2 / 50), 1}, masses 1 to 200, for stride = n and
    stride = n + 37: v <- c1 v + c2 / sqrt(m) xi with xi = normals 3c..3c+2 of curand_init(seed, i, 0),
    then the total momentum removed.  The padding of the larger stride stays bit for bit."""
    import torch
    L = lib.load()
    rng = np.random.default_rng(n + seed % 1000)
    mass = rng.uniform(1.0, 200.0, n)
    vel0 = rng.normal(size=(3, n)) * np.sqrt(K_B * 300.0 / mass)
    d_mass = torch.as_tensor(mass, device="cuda")
    stream0 = XorwowStates(seed, np.arange(n))
    worst = 0.0
    for stride in (n, n + 37):
        h = C.c_void_p()
        lib.check(L.b200md_langevin_create(n, seed, C.byref(h)))
        try:
            stream = stream0.copy()
            buf = padded(vel0, stride, rng)
            d_vel = torch.as_tensor(buf.reshape(-1).copy(), device="cuda")
            for k in range(7):
                c1 = C1S[k % 4]
                c2 = float(np.sqrt((1.0 - c1 * c1) * K_B * 300.0))
                before = d_vel.cpu().numpy().reshape(3, stride)
                lib.check(L.b200md_langevin_apply(h, n, stride, c1, c2, C.c_void_p(d_mass.data_ptr()),
                                                  C.c_void_p(d_vel.data_ptr()), None))
                after = d_vel.cpu().numpy().reshape(3, stride)
                v = c1 * before[:, :n] + (c2 * np.sqrt(1.0 / mass))[None, :] * stream.normal_double(3)
                want = v - (v * mass).sum(axis=1, keepdims=True) / mass.sum()
                scale = max(np.abs(want).max(), np.abs(before[:, :n]).max(), c2)
                got = after[:, :n]
                assert np.allclose(got, want, rtol=0, atol=VEL_RTOL * scale), (stride, k, gap(got, want, scale))
                assert np.array_equal(after[:, n:], buf[:, n:]), (stride, k)
                worst = max(worst, gap(got, want, scale))
        finally:
            L.b200md_langevin_destroy(h)
    print(f"langevin n={n} seed={seed}: largest |v_device - v_restated| / max|v| = {worst:.2e}")


def group_shape(shape, rng):
    """(label, source, sink) of one heat_lan layout."""
    if shape == "slabs":
        x = rng.uniform(0.0, 1.0, 20_011)
        return np.minimum((x * 8).astype(np.int32), 7), 1, 5
    if shape == "interleaved":
        return rng.integers(0, 5, 30_000).astype(np.int32), 3, 0
    label = np.zeros(1000, np.int32)  # a one-atom sink beside a 300-atom source
    label[rng.choice(1000, 301, replace=False)] = 1
    label[np.nonzero(label == 1)[0][137]] = 2
    return label, 1, 2


@pytest.mark.parametrize("pad", [0, 37])
@pytest.mark.parametrize("shape,seeds", [("slabs", (1804289383, 846930886)), ("interleaved", (2 ** 32 + 5, 0)),
                                         ("one_atom_sink", (2 ** 63 + 12345, 846930886))])
def test_heat_lan_kernel_draws_match_restatement(lib, shape, seeds, pad):
    """Six halves of b200md_heat_bath_half: source and sink kicked from their own streams, the
    subsequence being the atom's place in the group's contents; the energy moved into each bath within
    rtol 1e-12; every other atom, and the padding, bit for bit."""
    import torch
    from nemd_oracle import contents
    L = lib.load()
    rng = np.random.default_rng(17 + pad)
    label, source, sink = group_shape(shape, rng)
    n = label.shape[0]
    stride = n + pad
    mass = rng.uniform(1.0, 200.0, n)
    vel0 = rng.normal(size=(3, n)) * np.sqrt(K_B * 300.0 / mass)
    T, Tc, dT = 300.0, 10.0, 30.0
    sizes, order = contents(label)
    sizes, order = sizes.astype(np.int32), order.astype(np.int32)
    ip = C.POINTER(C.c_int)
    h = C.c_void_p()
    lib.check(L.b200md_heat_bath_create(0, n, sizes.shape[0], sizes.ctypes.data_as(ip), order.ctypes.data_as(ip),
                                        source, sink, T, Tc, dT, 1.0 / TIME_UNIT_CONVERSION, seeds[0], seeds[1],
                                        C.byref(h)))
    try:
        bath = HeatLan(mass, label, source, sink, T, Tc, dT, *seeds)
        d_mass = torch.as_tensor(mass, device="cuda")
        buf = padded(vel0, stride, rng)
        d_vel = torch.as_tensor(buf.reshape(-1).copy(), device="cuda")
        in_bath = (label == source) | (label == sink)
        worst = 0.0
        for k in range(6):
            before = d_vel.cpu().numpy().reshape(3, stride)
            lib.check(L.b200md_heat_bath_half(h, k % 2, n, stride, C.c_void_p(d_mass.data_ptr()),
                                              C.c_void_p(d_vel.data_ptr()), None))
            after = d_vel.cpu().numpy().reshape(3, stride)
            want = bath.half(before[:, :n])
            scale = max(np.abs(want).max(), np.abs(before[:, :n]).max())
            got = after[:, :n]
            assert np.allclose(got, want, rtol=0, atol=VEL_RTOL * scale), (k, gap(got, want, scale))
            worst = max(worst, gap(got, want, scale))
            assert np.array_equal(got[:, ~in_bath], before[:, :n][:, ~in_bath]), k
            assert np.array_equal(after[:, n:], buf[:, n:]), k
            energy = np.zeros(2)
            lib.check(L.b200md_heat_bath_energy(h, energy.ctypes.data_as(C.POINTER(C.c_double)), None))
            for g, grp in enumerate((source, sink)):
                ke = 0.5 * (mass[label == grp] * (got[:, label == grp] ** 2).sum(0)).sum()
                assert energy[g] == pytest.approx(bath.energy[g], rel=1e-12, abs=1e-12 * ke), (k, g)
    finally:
        L.b200md_heat_bath_destroy(h)
    print(f"heat_lan {shape} pad={pad}: largest |v_device - v_restated| / max|v| = {worst:.2e}")


# ---------------------------------------------------------------- engine level

LANGEVIN_GROUPS = {"none": None, "fix_m0": (0, 1), "fix_m1": (1, 2)}  # (grouping method, fixed group)


@pytest.mark.parametrize("groups", list(LANGEVIN_GROUPS))
@pytest.mark.parametrize("kind", ["nvt_lan", "nvt_bao"])
@pytest.mark.parametrize("pot", ["nep", "lj"])
def test_langevin_steps_match_restatement(oracle, eng, pot, kind, groups):
    """NEP PbTe (1728 atoms) and LJ Ar (2048 atoms), 20 steps, with and without a fixed group on either
    grouping method: the engine's seed 1804289383 restated draw for draw."""
    s, potfile, T0, dt_fs = S.system(pot)
    dt = dt_fs / TIME_UNIT_CONVERSION
    dev = S.Device(eng, s, potfile, T0, kind, dt)
    kw, fixed = {}, None
    if LANGEVIN_GROUPS[groups] is not None:
        method, fg = LANGEVIN_GROUPS[groups]
        label = S.labels(s)[method]
        dev.ens.set_groups(label, fixed_group=fg)
        kw, fixed = dict(label=label, fixed_group=fg), label == fg
    ref = EnsembleStep(kind, s["mass"], dt, pbc=s["pbc"], temperature=T0, temperature_coupling=50.0, **kw)
    S.run_locked(oracle, dev, ref, kind, fixed=fixed)


class HeatLanStep:
    """heat_lan's whole step: bath half, velocity-Verlet step 1 (with fix / move), the force driver's wrap,
    step 2, bath half (Ensemble_HEAT_B200::compute1 / compute2).  Computes no thermo."""

    def __init__(self, bath, nve):
        self.bath, self.nve = bath, nve

    def compute1(self, h, pos, vel, force):
        return self.nve.velocity_verlet(True, pos, self.bath.half(vel), force)

    def compute2(self, pos, vel, force):
        _, vel = self.nve.velocity_verlet(False, pos, vel, force)
        return self.bath.half(vel)

    def step(self, h, pos, vel, force_before, force_after, pe_after, virial_after):
        from oracle import oracle_py as O
        pos, vel = self.compute1(h, pos, vel, force_before)
        pos = O.apply_pbc(h, self.nve.pbc, pos)
        return pos, self.compute2(pos, vel, force_after), np.asarray(h, dtype=np.float64).reshape(9), None


HEAT_GROUPS = {"none": (-1, -1), "fix": (0, -1), "move": (-1, 2), "fix_move": (0, 2)}  # on the four slabs


@pytest.mark.parametrize("groups", list(HEAT_GROUPS))
def test_heat_lan_steps_match_restatement(oracle, eng, groups):
    """heat_lan on PbTe slabs (source slab 1, sink slab 3), 20 steps, with slab 0 fixed and / or slab 2
    moving: velocities, positions and the energy moved into each bath, restated piece by piece."""
    s, potfile, T0, dt_fs = S.system("nep")
    dt = dt_fs / TIME_UNIT_CONVERSION
    dev = S.Device(eng, s, potfile, T0, "nve", dt)
    label = S.labels(s)[0]
    dev.ens = eng.Ensemble_HEAT_LAN(label, 1, 3, 300.0, 10.0, 30.0)
    fg, mg = HEAT_GROUPS[groups]
    mv = S.MOVE_VELOCITY if mg >= 0 else (0.0, 0.0, 0.0)
    if fg >= 0 or mg >= 0:
        dev.ens.set_groups(None, fixed_group=fg, move_group=mg, move_velocity=mv)
    nve = EnsembleStep("nve", s["mass"], dt, pbc=s["pbc"], label=label, fixed_group=fg, move_group=mg,
                       move_velocity=mv)
    ref = HeatLanStep(HeatLan(s["mass"], label, 1, 3, 300.0, 10.0, 30.0, 1804289383, 846930886), nve)
    _, f0, _, _ = dev.forces()
    worst = 0.0
    for step in range(S.STEPS):
        p0, v0, h0 = dev.state()
        dev.ens.compute1(dev.dt, dev.box, dev.atom, dev.thermo)
        p1, v1, _ = dev.state()
        rp1, rv1 = ref.compute1(h0, p0, v0, f0)
        S.check(p1, rp1, False, VEL_RTOL, f"{step}: positions after compute1")
        S.check(v1, rv1, False, VEL_RTOL, f"{step}: velocities after compute1")
        pw, f1, _, _ = dev.forces()
        dev.ens.compute2(dev.dt, dev.box, dev.atom, dev.thermo)
        _, v2, _ = dev.state()
        rv2 = ref.compute2(pw, v1, f1)
        S.check(v2, rv2, False, VEL_RTOL, f"{step}: velocities after compute2")
        worst = max(worst, gap(v1, rv1, np.abs(rv1).max()), gap(v2, rv2, np.abs(rv2).max()))
        # atoms outside the baths integrate bit for bit like nve, the held groups stay held
        outside = (label != 1) & (label != 3)
        _, nv = nve.velocity_verlet(False, pw, v1, f1)
        assert np.array_equal(v2[:, outside], nv[:, outside]), step
        if fg >= 0:
            assert np.array_equal(p1[:, label == fg], p0[:, label == fg]) and np.all(v2[:, label == fg] == 0)
        if mg >= 0:
            assert np.all(v1[:, label == mg] == 0) and np.all(v2[:, label == mg] == 0)
        energy = dev.ens.energy_transferred()
        for g, grp in enumerate((1, 3)):
            ke = 0.5 * (s["mass"][label == grp] * (v2[:, label == grp] ** 2).sum(0)).sum()
            assert energy[g] == pytest.approx(ref.bath.energy[g], rel=1e-12, abs=1e-12 * ke), (step, g)
        f0 = f1
    dev.pot.check()
    print(f"heat_lan engine {groups}: largest |v_device - v_restated| / max|v| = {worst:.2e}")


# ---------------------------------------------------------------- driver level

def glibc_seeds(*ops):
    """Replay the driver's use of glibc's stream: ops are ("rand", k) for k values drawn and ("srand", s);
    returns the values of every ("seed",) op, in order.  The stream starts as after srand(1)."""
    r = GlibcRand()
    r.srand(1)
    out = []
    for op in ops:
        if op[0] == "srand":
            r.srand(op[1])
        elif op[0] == "rand":
            for _ in range(op[1]):
                r.rand()
        else:
            out.append(r.rand())
    return out


DRIVER = {
    # case: (run.in lines between `potential` and `time_step`, kind, grouping, glibc ops before the seed)
    "nvt_lan": ("ensemble nvt_lan 300 300 50\n", "nvt_lan", None, ()),
    "nvt_bao_fix": ("ensemble nvt_bao 300 300 50\nfix 1 1\n", "nvt_bao", (1, 1, -1), ()),
    "heat_lan_fix_move": ("ensemble heat_lan 300 10 30 1 3\nfix 0 0\nmove 0 2 0.002 -0.001 0.0015\n",
                          "heat_lan", (0, 0, 2), ()),
}


def driver_run(tmp_path, body, steps=S.STEPS, velocity="", extra=""):
    (tmp_path / "run.in").write_text(
        f"potential potential.txt\n{velocity}{body}time_step 1\ndump_thermo 1\n"
        f"dump_xyz 1 dump.xyz {S.DUMP}\nrun {steps}\n{extra}")
    S.run_exe(tmp_path)
    return S.read_frames(tmp_path / "dump.xyz"), S.read_thermo(tmp_path / "thermo.out")


def restatement(kind, s, mass, groups, grp, seeds):
    dt = 1.0 / TIME_UNIT_CONVERSION
    kw = {}
    if grp is not None:
        method, fg, mg = grp
        kw = dict(label=groups[method], fixed_group=fg, move_group=mg,
                  move_velocity=S.MOVE_VELOCITY if mg >= 0 else (0.0, 0.0, 0.0))
    if kind == "heat_lan":
        nve = EnsembleStep("nve", mass, dt, pbc=s["pbc"], **kw)
        return HeatLanStep(HeatLan(mass, groups[0], 1, 3, 300.0, 10.0, 30.0, seeds[0], seeds[1]), nve)
    return EnsembleStep(kind, mass, dt, pbc=s["pbc"], temperature=300.0, temperature_coupling=50.0,
                        seed=seeds[0], **kw)


@pytest.mark.parametrize("case", list(DRIVER))
def test_driver_langevin_steps_match_restatement(oracle, eng, tmp_path, case):
    """The executable's Langevin ensembles with velocities from model.xyz, seeded with glibc's first
    rand() (nvt_lan, nvt_bao) or its first two (heat_lan's source, then its sink), restated frame to
    frame from dump_xyz."""
    body, kind, grp, _ = DRIVER[case]
    s, potfile, groups, vel0 = S.driver_setup(tmp_path)
    frames, thermo = driver_run(tmp_path, body)
    assert len(frames) == S.STEPS
    seeds = glibc_seeds(("seed",), ("seed",))
    assert seeds == [1804289383, 846930886]
    ref = restatement(kind, s, frames[0]["mass"], groups, grp, seeds)
    f_start = S.single_point_force(eng, s, potfile, s["pos"], s["h"])
    S.restate_run(frames, None if kind == "heat_lan" else thermo, ref, f_start, s["h"], s["pos"], vel0)


def test_driver_second_run_takes_the_next_seed(oracle, eng, tmp_path):
    """Two runs: nvt_lan, then nvt_bao, which seeds its generators with the next rand() (846930886)."""
    s, potfile, groups, vel0 = S.driver_setup(tmp_path)
    (tmp_path / "run.in").write_text(
        f"potential potential.txt\nensemble nvt_lan 300 300 50\ntime_step 1\ndump_thermo 1\n"
        f"dump_xyz 1 a.xyz {S.DUMP}\nrun {S.STEPS}\nensemble nvt_bao 300 300 50\ndump_thermo 1\n"
        f"dump_xyz 1 b.xyz {S.DUMP}\nrun {S.STEPS}\n")
    S.run_exe(tmp_path)
    a, b = S.read_frames(tmp_path / "a.xyz"), S.read_frames(tmp_path / "b.xyz")
    thermo = S.read_thermo(tmp_path / "thermo.out")
    mass = a[0]["mass"]
    s1, s2 = glibc_seeds(("seed",), ("seed",))
    ref = restatement("nvt_lan", s, mass, groups, None, [s1])
    S.restate_run(a, thermo[:S.STEPS], ref, S.single_point_force(eng, s, potfile, s["pos"], s["h"]),
                  s["h"], s["pos"], vel0)
    last = a[-1]
    ref2 = restatement("nvt_bao", s, mass, groups, None, [s2])
    f_start = S.single_point_force(eng, s, potfile, last["pos"], last["h"])
    S.restate_run(b, thermo[S.STEPS:], ref2, f_start, last["h"], last["pos"], last["vel"], first_step_fp32=True)


@pytest.mark.parametrize("seeded", [False, True])
def test_driver_seed_after_velocity(oracle, eng, tmp_path, seeded):
    """On a model.xyz without velocities (with them, `velocity` is ignored and draws nothing), `velocity
    300` draws 3N rand() values and `velocity 300 seed S` reseeds before each of them, last with
    srand(S + 3N - 1).  The nvt_lan that follows takes the next rand().  The initial velocities are the
    driver's own, so the restatement starts from the first frame, its stream advanced past the first
    step's two kicks."""
    s, potfile, groups, _ = S.driver_setup(tmp_path)
    S.write_model(tmp_path / "model.xyz", s, nep_type_order(GOLDEN / potfile), None, groups)
    n = s["type"].shape[0]
    S_seed = 4321
    velocity = f"velocity 300 seed {S_seed}\n" if seeded else "velocity 300\n"
    frames, thermo = driver_run(tmp_path, "ensemble nvt_lan 300 300 50\n", velocity=velocity)
    ops = (("srand", S_seed + 3 * n - 1), ("rand", 1), ("seed",)) if seeded else (("rand", 3 * n), ("seed",))
    (seed,) = glibc_seeds(*ops)
    ref = restatement("nvt_lan", s, frames[0]["mass"], groups, None, [seed])
    ref.noise.normal_double(6)  # the first step's two kicks
    f0 = frames[0]
    S.restate_run(frames[1:], thermo[1:], ref, f0["force"], f0["h"], f0["pos"], f0["vel"])

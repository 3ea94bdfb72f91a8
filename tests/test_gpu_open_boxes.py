"""The structures of tests/test_open_boxes_cpu.py (clusters, wires and ribbons with open x or y directions,
atoms outside the box, small-box supercells with open directions, N = 1, 2, 3, list overflow at MN + 1 and
MN) on every device kernel path their model dispatches, each asserting the instance it is named for:

  - one and two species: the fused angular kernel (default), the tensor-core and SIMT hidden layers with the
    plane-based radial kernels, the lane teams (B200MD_NEP_TEAM=1), the generic kernels
    (B200MD_NEP_RADIAL=v1) and k_utable (B200MD_NEP_UTABLE=simt);
  - three and more species: the default radial instance, RADREG, RADDIRECT, REVSLOT=1, CSTAGE=0, the
    tensor-core and the SIMT hidden layer;
  - LJ, Tersoff and EAM through their kernels against the FP32 oracle and the FP64 references;
  - NVE and Berendsen runs of drifting clusters and a wire, restated step by step, and one run of the
    executable on an all-open model.xyz.

Every NEP case calls check_nep (neighbour lists bit for bit, descriptors, E/F/virial against FP32 and FP64);
the tensor-core and SIMT cases also check_mlp."""
import numpy as np
import pytest

import cases_classical as cc
from conftest import GOLDEN, assert_close
from ensemble_oracle import EnsembleStep
from gpumd_b200.structures import TIME_UNIT_CONVERSION, init_velocities, nep_type_order
from test_classical_cpu import check_vs_fp64, check_vs_oracle
from test_gpu_classical import compute as classical_compute
from test_gpu_ensemble_steps import (DUMP, Device, check, read_frames, read_thermo, restate_run, run_exe,
                                     single_point_force, write_model)
from test_gpu_many_species import EXPECT, RADREG_NT, expected
from test_gpu_nep_species import _env, check_mlp, load_ann
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)
from test_kernel_bodies_cpu import check_fv, check_nep
from test_open_boxes_cpu import (CLASSICAL_CASES, FEW_ATOM_MODELS, NEP_OPEN, NEP_OPEN_MANY, SKIN_POT, check_few_atoms,
                                 classical_case, few_atom_case, open_box, overflow_models, overflow_shell, pbte,
                                 skin_shell, tersoff_shell)

pytestmark = pytest.mark.gpu

# one- and two-species paths: environment, and the radial instance (b200md_nep_info 12) they select
FEW_PATHS = {
    "fused": ({}, 100),
    "tc": ({"B200MD_NEP_MLP": "tc"}, 100),
    "simt": ({"B200MD_NEP_MLP": "simt"}, 100),
    "team": ({"B200MD_NEP_TEAM": "1"}, 200),
    "v1": ({"B200MD_NEP_RADIAL": "v1"}, 0),
    "utable": ({"B200MD_NEP_MLP": "tc", "B200MD_NEP_UTABLE": "simt"}, 100),
}
# the models whose hidden layer fits k_angular_fused (test_gpu_angular_fused.py) and two that do not
FUSED = {"nep_PbTe.txt": True, "nep_synth_1sp_zbl_k17.txt": True, "nep_C_2022_NEP4.txt": False,
         "nep_synth_2sp_nep5_flexzbl.txt": False}


def set_env(monkeypatch, env):
    """_env, and the two switches it leaves alone."""
    for k in ("B200MD_NEP_UTABLE", "B200MD_NEP_CSTAGE"):
        monkeypatch.delenv(k, raising=False)
    _env(monkeypatch, env)


def run_few(oracle, eng, model, s, path, monkeypatch):  # noqa: F811
    env, base = FEW_PATHS[path]
    set_env(monkeypatch, env)
    n = s["type"].shape[0]
    nt = len(nep_type_order(GOLDEN / model))
    dev = GpuNep(eng, model, n)
    out = check_nep(oracle, dev, model, s, n)
    inst = dev.pot.instances
    assert inst["radial_nt"] == base + nt, (path, inst)
    if path == "fused" and model in FUSED:
        assert (inst["ang_block"] == 0) == FUSED[model], inst
    if path != "fused":
        assert inst["ang_block"] != 0, (path, inst)  # B200MD_NEP_MLP or a non-plane radial pass: not fused
    if path == "simt":
        assert inst["mlp_dimp"] > 0 and dev.pot.num_tiles == 0, inst
    if path == "utable":
        assert inst["utable"] == 2, inst
    if path in ("tc", "simt"):
        check_mlp(load_ann(GOLDEN / model), dev.pot, s["type"], out["pe"], what=f"{model}/{path}")
    return dev, out


@pytest.mark.parametrize("path", list(FEW_PATHS))
@pytest.mark.parametrize("case", list(NEP_OPEN))
def test_open_boxes_few_species_paths(oracle, eng, case, path, monkeypatch):  # noqa: F811
    model, make = NEP_OPEN[case]
    run_few(oracle, eng, model, make(), path, monkeypatch)


def many_paths(case):
    key = case.split("_ribbon")[0]
    out = ["tc", "simt", "RADDIRECT", "REVSLOT"]
    if key not in EXPECT:  # UNEP-v1, 50 species: the layers and the switches every model takes
        return out
    if key in RADREG_NT:
        out.append("RADREG")
    if EXPECT[key]["cstage"]:
        out.append("CSTAGE0")
    return out


MANY_CASES = [(c, p) for c in NEP_OPEN_MANY for p in many_paths(c)]


@pytest.mark.parametrize("case,path", MANY_CASES)
def test_open_boxes_many_species_paths(oracle, eng, case, path, monkeypatch):  # noqa: F811
    model, make = NEP_OPEN_MANY[case]
    key = case.split("_ribbon")[0]
    env = {"tc": {"B200MD_NEP_MLP": "tc"}, "simt": {"B200MD_NEP_MLP": "simt"},
           "RADDIRECT": {"B200MD_NEP_RADDIRECT": "1"}, "REVSLOT": {"B200MD_NEP_REVSLOT": "1"},
           "RADREG": {"B200MD_NEP_RADREG": "1"}, "CSTAGE0": {"B200MD_NEP_CSTAGE": "0"}}[path]
    set_env(monkeypatch, env)
    s = make()
    n = s["type"].shape[0]
    dev = GpuNep(eng, model, n)
    out = check_nep(oracle, dev, model, s, n)
    inst = dev.pot.instances
    if key in EXPECT:
        mlp = "simt" if path == "simt" else "tc"
        over = {"RADDIRECT": dict(radial_nt=-1), "RADREG": dict(radial_nt=RADREG_NT.get(key)),
                "REVSLOT": dict(revslot=1 - EXPECT[key]["split"]), "CSTAGE0": dict(cstage=0)}.get(path, {})
        assert inst == expected(key, mlp, **over), (case, path, inst)
    else:
        if path == "RADDIRECT":
            assert inst["radial_nt"] == -1, inst
        assert inst["revslot"] == int(path == "REVSLOT" and inst["split"] == 0), inst
        assert (inst["mlp_dimp"] > 0) == (path == "simt"), inst
    if path in ("tc", "simt"):
        check_mlp(load_ann(GOLDEN / model), dev.pot, s["type"], out["pe"], what=f"{case}/{path}")


FEW_ATOM_CASES = [(c, p) for c in FEW_ATOM_MODELS
                  for p in (("fused", "simt", "team", "v1") if c in ("1sp", "2sp") else ("tc", "simt"))]


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("case,path", FEW_ATOM_CASES)
def test_one_two_three_atoms(oracle, eng, case, path, n, monkeypatch):  # noqa: F811
    """A lone atom (site energy ann(q = 0), zero force and virial), a pair at 0.7 rc and a collinear triple:
    one type tile of padding, warps with 31 of 32 lanes idle, a brick schedule of mostly empty bricks."""
    model = FEW_ATOM_MODELS[case]
    env = {"fused": {}, "tc": {}, "simt": {"B200MD_NEP_MLP": "simt"}, "team": {"B200MD_NEP_TEAM": "1"},
           "v1": {"B200MD_NEP_RADIAL": "v1"}}[path]
    set_env(monkeypatch, env)
    for which in (0, 1):
        s = few_atom_case(model, n, which)
        check_few_atoms(oracle, GpuNep(eng, model, n), model, s)


@pytest.mark.parametrize("case", CLASSICAL_CASES)
def test_classical_open_boxes(oracle, eng, case):  # noqa: F811
    kind, path, s = classical_case(case)
    n = s["type"].shape[0]
    r32 = cc.oracle32(kind, path, s)
    r64 = cc.reference64(kind, path, s, f32_params=True)
    out, _ = classical_compute(eng, kind, path, s)
    check_vs_oracle(out, r32, n, kind, path)
    check_vs_fp64(out, r64, n, kind, path, gap=cc.gaps(r32, r64))


# ---------------------------------------------------------------- list overflow

# path -> environment: the plane-based radial kernel of one and two species (k_desc_radial2), the lane teams,
# the generic kernels; three species always run the generic many-species kernels
OVERFLOW_PATHS = {"plane": {}, "team": {"B200MD_NEP_TEAM": "1"}, "generic": {"B200MD_NEP_RADIAL": "v1"}}
OVERFLOW_CASES = [(m, p, b) for m in ("1sp", "2sp", "3sp") for p in OVERFLOW_PATHS for b in (1, 2, 4)
                  if m != "3sp" or p == "plane"]


@pytest.mark.parametrize("name,path,bit", OVERFLOW_CASES)
def test_list_overflow_bits(oracle, eng, tmp_path, name, path, bit, monkeypatch):  # noqa: F811
    """One atom at count = MN + 1 of the skin (bit 1), radial (2) or angular (4) list: check() raises with
    exactly that bit.  The same shell at count = MN: no bit, and the result equals the oracle's.  Every list
    writer stores only while count < MN (b2_body_skin_list, k_desc_radial2, the team and generic bodies), and
    tests/test_open_boxes_cpu.py runs the same shells through the host build first."""
    set_env(monkeypatch, OVERFLOW_PATHS[path])
    model = overflow_models(tmp_path)[name]
    base = model.name.split("_", 3)[3]
    s = overflow_shell(base, bit, 1)
    dev = GpuNep(eng, model, s["type"].shape[0])
    with pytest.raises(Exception, match=rf"bits={bit}\b"):
        dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    s = overflow_shell(base, bit, 0)
    n = s["type"].shape[0]
    dev = GpuNep(eng, model, n)
    check_nep(oracle, dev, model, s, n)
    nt = len(nep_type_order(GOLDEN / base))
    if nt <= 2:
        assert dev.pot.instances["radial_nt"] == {"plane": 100, "team": 200, "generic": 0}[path] + nt


def test_tersoff_angular_overflow(oracle, eng):  # noqa: F811
    """33 neighbours inside Tersoff's cutoff (its local list holds 32): check() raises; 32 match the oracle."""
    from gpumd_b200.lib import B200mdError
    s = tersoff_shell(1)
    with pytest.raises(B200mdError, match="Tersoff neighbour capacity"):
        classical_compute(eng, "tersoff", cc.SI, s)
    s = tersoff_shell(0)
    out, _ = classical_compute(eng, "tersoff", cc.SI, s)
    check_vs_oracle(out, cc.oracle32("tersoff", cc.SI, s), s["type"].shape[0], "tersoff", cc.SI)


@pytest.mark.parametrize("tight", [False, True])
@pytest.mark.parametrize("kind", list(SKIN_POT))
def test_classical_skin_overflow(oracle, eng, kind, tight, monkeypatch):  # noqa: F811
    """LJ / EAM skin list at capacity + 1 (check() raises) and at capacity (matches the oracle), with the
    default capacity and with B200MD_TIGHT_LISTS=1."""
    from gpumd_b200.lib import B200mdError
    if tight:
        monkeypatch.setenv("B200MD_TIGHT_LISTS", "1")
    else:
        monkeypatch.delenv("B200MD_TIGHT_LISTS", raising=False)
    path = SKIN_POT[kind][0]
    s = skin_shell(kind, 1, tight)
    with pytest.raises(B200mdError, match="capacity exceeded"):
        classical_compute(eng, kind, path, s)
    s = skin_shell(kind, 0, tight)
    out, _ = classical_compute(eng, kind, path, s)
    r = cc.oracle32(kind, path, s)
    if tight:
        check_vs_oracle(out, r, s["type"].shape[0], kind, path)
    else:  # ~1.2 A apart: site energies of 1e4 - 1e5 eV, so only the relative parts of the tolerances apply
        assert_close(out["pe"], r["pe"], rtol=1e-5, atol=1e-5, what="pe")
        check_fv(out, r)


# ---------------------------------------------------------------- trajectories

STEPS = 200
DRIFT = np.array([0.03, -0.02, 0.025]) * TIME_UNIT_CONVERSION  # A/fs: ~6 A over the run


def trajectory_system(name):
    """(structure, potential file, T0, dt in fs)."""
    if name == "nep_cluster":
        return open_box(pbte(4, 91), (0, 0, 0)), "nep_PbTe.txt", 300.0, 1.0
    if name == "nep_wire_001":
        return open_box(pbte((4, 4, 2), 92), (0, 0, 1)), "nep_PbTe.txt", 300.0, 1.0
    from gpumd_b200.structures import fcc
    return open_box(fcc(6, 5.30, rattle=0.02, seed=93), (0, 0, 0)), "lj_Ar_10A.txt", 40.0, 2.0


def force_reference(oracle, potfile, s, pos):
    t = dict(s, pos=pos)
    if potfile.startswith("nep"):
        r32 = oracle.NepOracle(GOLDEN / potfile).compute(t["type"], t["h"], t["pbc"], pos, precision=32)
        return r32, "nep"
    return cc.oracle32("lj", GOLDEN / potfile, t), "lj"


@pytest.mark.parametrize("kind", ["nve", "nvt_ber"])
@pytest.mark.parametrize("name", ["nep_cluster", "nep_wire_001", "lj_cluster"])
def test_drifting_open_system_steps(oracle, eng, name, kind):  # noqa: F811
    """200 steps with a centre-of-mass drift that carries atoms further out of the box and rebuilds the lists
    several times: the force driver's wrap never shifts an open coordinate (it round-trips every coordinate
    through fractional coordinates, as the reference's gpu_apply_pbc does, which may move the last bit of an
    open one, so those are held to 1e-12 A of the unwrapped value), velocity-Verlet matches the
    restatement bit for bit (Berendsen's scaled velocities to 1e-12), and after every rebuild the forces match
    the oracle at the device's own positions."""
    s, potfile, T0, dt_fs = trajectory_system(name)
    dt = dt_fs / TIME_UNIT_CONVERSION
    dev = Device(eng, s, potfile, T0, kind, dt)
    vel = init_velocities(s["mass"], T0, seed=42) + DRIFT[:, None]
    dev.atom.velocity_per_atom.copy_(dev.torch.as_tensor(vel.reshape(-1), device="cuda"))
    ref = EnsembleStep(kind, s["mass"], dt, pbc=s["pbc"], temperature=T0, temperature_coupling=50.0)
    per = np.asarray(s["pbc"]).astype(bool)
    scaled = kind != "nve"
    _, f0, _, _ = dev.forces()
    rebuilds = dev.pot.num_rebuilds
    checked = 0
    for step in range(STEPS):
        p0, v0, h0 = dev.state()
        dev.ens.compute1(dev.dt, dev.box, dev.atom, dev.thermo)
        p1, v1, _ = dev.state()
        rp1, rv1 = ref.compute1(h0, p0, v0, f0)
        check(p1, rp1, True, 0, f"{step}: positions after compute1")
        check(v1, rv1, True, 0, f"{step}: velocities after compute1")
        pw, f1, pe1, vir1 = dev.forces()
        assert np.abs(pw[~per] - p1[~per]).max() <= 1e-12, step
        assert np.allclose(pw, oracle.apply_pbc(h0, ref.pbc, p1), rtol=0, atol=1e-12), step
        if dev.pot.num_rebuilds != rebuilds:
            rebuilds = dev.pot.num_rebuilds
            r, _ = force_reference(oracle, potfile, s, pw)
            check_fv(dict(force=f1, virial=vir1), r)
            checked += 1
        dev.ens.compute2(dev.dt, dev.box, dev.atom, dev.thermo)
        p2, v2, _ = dev.state()
        _, rv2, _, _ = ref.compute2(h0, pw, v1, f1, pe1, vir1)
        check(v2, rv2, not scaled, 1e-12, f"{step}: velocities after compute2")
        assert np.array_equal(p2, pw), step
        f0 = f1
    dev.pot.check()
    frac = np.linalg.solve(s["h"].reshape(3, 3), p2)
    assert checked >= 3, checked
    assert ((frac[~per] < 0) | (frac[~per] > 1)).any(axis=0).mean() > 0.05  # atoms out of the box


def test_driver_all_open_nve(oracle, eng, tmp_path):  # noqa: F811
    """The executable on a model.xyz with pbc="F F F" (the PbTe cluster, atoms on both sides outside the box),
    `ensemble nve`, restated frame by frame from dump_xyz."""
    import shutil
    s, potfile, T0, _ = trajectory_system("nep_cluster")
    sym = nep_type_order(GOLDEN / potfile)
    vel = init_velocities(s["mass"], T0, seed=42)
    write_model(tmp_path / "model.xyz", s, sym, vel, [np.zeros(s["type"].shape[0], np.int32)])
    shutil.copyfile(GOLDEN / potfile, tmp_path / "potential.txt")
    vel0 = np.array([[float(f"{x:.17g}") for x in row] for row in vel / TIME_UNIT_CONVERSION]) * TIME_UNIT_CONVERSION
    steps = 40
    (tmp_path / "run.in").write_text(
        f"potential potential.txt\nensemble nve\ntime_step 1\ndump_thermo 1\ndump_xyz 1 dump.xyz {DUMP}\n"
        f"run {steps}\n")
    run_exe(tmp_path)
    frames = read_frames(tmp_path / "dump.xyz")
    thermo = read_thermo(tmp_path / "thermo.out")
    assert len(frames) == steps
    assert 'pbc="F F F"' in (tmp_path / "model.xyz").read_text().splitlines()[1]
    ref = EnsembleStep("nve", frames[0]["mass"], 1.0 / TIME_UNIT_CONVERSION, pbc=s["pbc"], temperature=T0,
                       temperature_coupling=50.0)
    f_start = single_point_force(eng, s, potfile, s["pos"], s["h"])
    restate_run(frames, thermo, ref, f_start, s["h"], s["pos"], vel0)
    last = frames[-1]
    r = oracle.NepOracle(GOLDEN / potfile).compute(s["type"], s["h"], s["pbc"], last["pos"], precision=32)
    check_fv(dict(force=last["force"], virial=last["virial"]), r)

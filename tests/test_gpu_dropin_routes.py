"""Every route of the GPUMD plugin (gpumd_b200/plugin/b200md_gpumd.cu) inside the patched reference binary
oracle/_ref/gpumd_b200: each case runs the same binary on the same inputs twice, with GPUMD_B200=1 (libb200md
behind the reference's Potential / Ensemble classes) and with it unset (the reference's own classes), and
asserts from the output which route served it.

- Forces: `run 1` under NVE dumps positions and, for them, forces, site energies and 9-component virials in
  double precision; those are checked against the oracle at the dumped positions (FP32 restatement plus its
  FP32-FP64 gap for NEP / LJ / EAM, the FP64 restatement for Tersoff) and against the plugin-off run.  Every
  potential runs on an orthogonal, a triclinic and an open-z box; multi-species inputs list their atoms in
  the reverse order of the potential file's species, and two leave out a species the file lists.
- Ensembles and `deform`: FP64 Tersoff on both sides, so the two trajectories differ only by the summation
  order of the forces and of the thermo reductions.  Positions, velocities, box and thermo.out are compared
  on every step (bound: see STEP_BOUND).
- Reference classes on plugin outputs: heat_lan / heat_nhc / heat_bdp (declined by the plugin, run by the
  reference on plugin forces), compute_hac, compute_shc and two NEP potentials in `average` and `observe`
  mode, whose per-atom arrays must be the mean of (or the first of) two oracle evaluations."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import cases_classical as cc
from cases import shear, slab
from conftest import GOLDEN, ROOT, TOL, assert_close
from gpumd_b200.structures import diamond, fcc, init_velocities, nep_type_order, \
    rocksalt_pbte, write_xyz
from test_classical_cpu import check_vs_fp64, check_vs_oracle
from test_few_species_cpu import alloy
from test_gpu_ensemble_steps import labels, read_frames, read_thermo, tilt, write_model
from test_kernel_bodies_cpu import check_fv

pytestmark = pytest.mark.gpu
EXE = ROOT / "oracle" / "_ref" / "gpumd_b200"
DUMP = "dump_xyz 1 dump.xyz precision double mass velocity force potential virial"
BACKEND = {"nep": "NEP", "lj": "LJ", "tersoff": "Tersoff-1989", "eam": "EAM"}


@pytest.fixture(scope="module")
def exe():
    if not EXE.exists():
        pytest.skip("oracle/_ref/gpumd_b200 not built (make -C oracle -f Makefile.gpumd_b200; needs the reference)")
    return EXE


def run_both(tmp, files, run_in, timeout=300):
    """The binary once with GPUMD_B200=1 (tmp/on) and once without (tmp/off) on the same inputs;
    files: name -> text or source path.  Returns {"on": (stdout, dir), "off": (stdout, dir)}."""
    out = {}
    for tag in ("on", "off"):
        d = tmp / tag
        d.mkdir()
        for name, src in files.items():
            if isinstance(src, str):
                (d / name).write_text(src)
            else:
                shutil.copyfile(src, d / name)
        (d / "run.in").write_text(run_in)
        env = dict(os.environ)
        env.pop("GPUMD_B200", None)
        if tag == "on":
            env["GPUMD_B200"] = "1"
        env["CUDA_VISIBLE_DEVICES"] = env.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]  # NEP, not NEP_MULTIGPU
        r = subprocess.run([str(EXE)], cwd=d, capture_output=True, text=True, timeout=timeout, env=env)
        assert r.returncode == 0, (tag, r.stdout[-3000:] + r.stderr[-2000:])
        out[tag] = (r.stdout, d)
    assert "b200md" not in out["off"][0]
    return out


def assert_routes(out, kind, ensemble_type):
    """The plugin served the potential, and the ensemble when ensemble_type is not None (else it declined)."""
    text = out["on"][0]
    assert f"Use the b200md {BACKEND[kind]} backend" in text, text[-2000:]
    if ensemble_type is None:
        assert "Use the b200md integrator" not in text
    else:
        assert f"Use the b200md integrator for ensemble type {ensemble_type}." in text, text[-2000:]


def reverse_species(s):
    """The atoms re-listed with the potential file's last species first."""
    order = np.argsort(-s["type"], kind="stable")
    s = dict(s, pos=np.ascontiguousarray(s["pos"][:, order]), type=s["type"][order].copy())
    if "mass" in s:
        s["mass"] = s["mass"][order]
    return s


def mic(h, pbc, d):
    """Displacements under the fractional minimum image along the periodic directions."""
    H = np.asarray(h, dtype=np.float64).reshape(3, 3)
    f = np.linalg.solve(H, d)
    p = np.asarray(pbc).astype(bool)
    f[p] -= np.round(f[p])
    return H @ f


# ---------------------------------------------------------------- 1. forces through the plugin

def _batio3():
    order = nep_type_order(GOLDEN / "nep_BaTiO3.txt")
    s = fcc(6, 4.0, rattle=0.08, seed=51, num_types=3, symbols=("Ar", "Ar", "Ar"))  # 864 atoms, 24 A
    s["symbols"] = order
    return s


def _lj3_without_ne():
    s = cc._lj3_alloy(42)
    s["type"] = np.where(s["type"] == 1, 2, s["type"]).astype(np.int32)
    return s


def _cufeni_without_fe():
    s = cc._eam("cufeni", 3.615, 46)
    s["type"] = np.where(s["type"] == 1, 2, s["type"]).astype(np.int32)
    return s


# name -> (kind, potential file, structure factory)
POTENTIALS = {
    "nep4_PbTe": ("nep", GOLDEN / "nep_PbTe.txt", lambda: rocksalt_pbte(4, rattle=0.05, seed=1)),
    "nep4_zbl_2sp": ("nep", GOLDEN / "nep_synth_2sp_typewise_zbl.txt",
                     lambda: alloy("nep_synth_2sp_typewise_zbl.txt", seed=32)),
    "nep4_zbl_BaTiO3": ("nep", GOLDEN / "nep_BaTiO3.txt", _batio3),
    "nep5_1sp": ("nep", GOLDEN / "nep_synth_1sp_nep5.txt", lambda: alloy("nep_synth_1sp_nep5.txt", seed=35)),
    "nep5_zbl_2sp": ("nep", GOLDEN / "nep_synth_2sp_nep5_flexzbl.txt",
                     lambda: alloy("nep_synth_2sp_nep5_flexzbl.txt", seed=31)),
    "lj_Ar": ("lj", cc.LJ1, cc.STRUCTURES["lj_ar"][2]),
    "lj_3sp": ("lj", cc.LJ3, cc.STRUCTURES["lj_3sp"][2]),
    "tersoff_Si": ("tersoff", cc.SI, cc.STRUCTURES["si"][2]),
    "tersoff_SiC": ("tersoff", cc.SIC, cc.STRUCTURES["sic"][2]),
    "eam_zhou_Cu": ("eam", GOLDEN / cc.EAM_FILES["cu_zhou"], cc.STRUCTURES["eam_cu_zhou_a0"][2]),
    "eam_zhou_CuFeNi": ("eam", GOLDEN / cc.EAM_FILES["cufeni"], cc.STRUCTURES["eam_cufeni_a0"][2]),
    "eam_dai_Cu": ("eam", GOLDEN / cc.EAM_FILES["cu_dai"], cc.STRUCTURES["eam_cu_dai_a0"][2]),
}
BOXES = {"ortho": lambda s: s, "tric": shear, "slab": slab}
FORCE_CASES = [f"{p}-{b}" for p in POTENTIALS for b in BOXES] + [
    "lj_3sp_without_Ne-ortho", "eam_zhou_CuFeNi_without_Fe-tric"]
MISSING = {"lj_3sp_without_Ne": ("lj", cc.LJ3, _lj3_without_ne),
           "eam_zhou_CuFeNi_without_Fe": ("eam", GOLDEN / cc.EAM_FILES["cufeni"], _cufeni_without_fe)}


def make_force_case(case):
    name, box = case.rsplit("-", 1)
    kind, path, factory = {**POTENTIALS, **MISSING}[name]
    s = BOXES[box](factory())
    if len(nep_type_order(path)) > 1:
        s = reverse_species(s)
    return kind, path, s


def check_nep_dump(path, s, fr):
    """check_nep's E/F/virial assertions (test_kernel_bodies_cpu.py) on a dumped frame."""
    from oracle import oracle_py
    orc = oracle_py.NepOracle(path)
    r32 = orc.compute(s["type"], fr["h"], s["pbc"], fr["pos"], precision=32)
    r64 = orc.compute(s["type"], fr["h"], s["pbc"], fr["pos"], precision=64)
    n = s["type"].shape[0]
    energy_tol = TOL["energy_per_atom"] * max(1.0, abs(r64["pe"].sum()) / n)
    gap = abs(r32["pe"].sum() - r64["pe"].sum()) / n
    assert abs(fr["pe"].sum() - r32["pe"].sum()) / n < energy_tol
    assert abs(fr["pe"].sum() - r64["pe"].sum()) / n < energy_tol + 2 * gap
    assert_close(fr["pe"], r32["pe"], rtol=TOL["energy"]["rtol"],
                 atol=TOL["energy"]["rtol"] * max(1.0, np.abs(r32["pe"]).max()), what="pe")
    gap_f = np.abs(r32["force"] - r64["force"]).max()
    gap_v = np.abs(r32["virial"] - r64["virial"]).max()
    check_fv(fr, r32, gap_f=gap_f, gap_v=gap_v)
    check_fv(fr, r64, gap_f=gap_f, gap_v=gap_v)
    return r32


def check_dump(kind, path, s, fr):
    if kind == "nep":
        return check_nep_dump(path, s, fr)
    st = dict(s, h=fr["h"], pos=fr["pos"])
    r32 = cc.oracle32(kind, path, st)
    check_vs_oracle(fr, r32, s["type"].shape[0], kind, path)
    if kind != "tersoff":
        r64 = cc.reference64(kind, path, st, f32_params=True)
        check_vs_fp64(fr, r64, s["type"].shape[0], kind, path, gap=cc.gaps(r32, r64))
    return r32


@pytest.mark.parametrize("case", FORCE_CASES)
def test_forces_through_the_plugin_match_the_oracle(oracle, exe, tmp_path, case):
    """One NVE step: the dumped forces, site energies and virials of both runs against the oracle at the
    dumped positions, and against each other (Tersoff: FP64 on both sides)."""
    kind, path, s = make_force_case(case)
    symbols = nep_type_order(path)
    mass = s.get("mass", np.ones(s["type"].shape[0]))
    vel = init_velocities(np.asarray(mass, dtype=np.float64), 100.0, seed=7)
    write_xyz(tmp_path / "model.xyz", s, symbols, vel)
    model = (tmp_path / "model.xyz").read_text()
    out = run_both(tmp_path, {"model.xyz": model, "potential.txt": path},
                   f"potential potential.txt\ntime_step 1\nensemble nve\ndump_thermo 1\n{DUMP}\nrun 1\n")
    assert_routes(out, kind, 0)
    frames = {tag: read_frames(d / "dump.xyz") for tag, (_, d) in out.items()}
    assert len(frames["on"]) == len(frames["off"]) == 1
    on, off = frames["on"][0], frames["off"][0]
    check_dump(kind, path, s, on)
    check_dump(kind, path, s, off)
    if kind == "tersoff":
        assert_close(on["force"], off["force"], rtol=1e-9, atol=1e-10, what="force on/off")
        assert_close(on["virial"], off["virial"], rtol=1e-9, atol=1e-10, what="virial on/off")
        assert_close(on["pe"], off["pe"], rtol=1e-10, atol=1e-11, what="pe on/off")
    else:
        check_fv(on, off)
        assert_close(on["pe"], off["pe"], rtol=TOL["energy"]["rtol"],
                     atol=TOL["energy"]["rtol"] * max(1.0, np.abs(off["pe"]).max()), what="pe on/off")


# ---------------------------------------------------------------- 2. + 3. ensembles and deform, FP64 Tersoff

STEPS = 30
# The two runs differ by the summation order of FP64 forces (|df|/|f| ~ 1e-15) and of the thermo
# reductions.  Over STEPS steps of 1 fs a force difference df moves a position by ~ STEPS^2 dt^2 df / m
# ~ 1e-17 A for Si, below the rounding of the positions themselves (|r| ~ 40 A: ~1e-14 A per step); a
# Lyapunov time of ~0.1 ps amplifies that by < 1.5 over 30 fs.  Velocities take dt df / m per step, ~1e-15 of
# their thermal magnitude, plus the rounding of the thermostat factors.  So the gap grows by at most ~1e-14
# per step (A for positions, relative to the largest velocity), and the bounds allow 1e3 times STEPS of that
# (measured on an H100: positions <= 7e-14 A, velocities <= 5e-13, box <= 1e-17 relative, thermo.out equal
# to ~1e-10 of its printed digits).  A wrong random stream, seed, group rule or barostat branch moves
# velocities by O(1) of their thermal magnitude and positions by >= 1e-4 A within a few steps.
STEP_BOUND = dict(pos=STEPS * 1e-14 * 1e3, vel=STEPS * 1e-14 * 1e3, h=STEPS * 1e-15 * 1e3, thermo=1e-8)
FIX = "fix 0\n"
FIX_MOVE = "fix 0\nmove 3 0.002 -0.001 0.0015\n"
NPT3 = "ensemble npt_ber 300 300 50 0 0.1 -0.1 100 90 110 200\n"

# name -> (run.in body before `run`, ensemble type, structure variant)
ENSEMBLES = {
    "nve": ("ensemble nve\n", 0, "si"),
    "nvt_ber": ("ensemble nvt_ber 300 300 50\n", 1, "si"),
    "nvt_ber_fix_move": ("ensemble nvt_ber 300 300 50\n" + FIX_MOVE, 1, "si"),
    "nvt_nhc": ("ensemble nvt_nhc 300 300 50\n", 2, "si"),
    "nvt_nhc_fix_move": ("ensemble nvt_nhc 300 300 50\n" + FIX_MOVE, 2, "sic"),
    "nvt_bdp": ("ensemble nvt_bdp 300 300 50\n", 4, "si"),
    "nvt_bdp_fix_move": ("ensemble nvt_bdp 300 300 50\n" + FIX_MOVE, 4, "si"),
    "nvt_lan": ("ensemble nvt_lan 300 300 50\n", 3, "si"),
    "nvt_lan_fix": ("ensemble nvt_lan 300 300 50\n" + FIX, 3, "si"),
    "nvt_bao": ("ensemble nvt_bao 300 300 50\n", 5, "si"),
    "nvt_bao_fix": ("ensemble nvt_bao 300 300 50\n" + FIX, 5, "si"),
    "npt_ber_iso": ("ensemble npt_ber 300 300 50 0.5 100 200\n", 11, "si"),
    "npt_ber_3": (NPT3, 11, "si"),
    "npt_ber_3_open_z": (NPT3, 11, "si_open_z"),
    "npt_ber_6_triclinic": ("ensemble npt_ber 300 300 50 0 0.1 -0.1 0.05 -0.05 0.02 100 90 110 60 60 60 200\n",
                            11, "si_tric"),
    "deform_x": (NPT3 + "deform 1e-4 1 0 0\n", 11, "si"),
    "deform_xyz_three_rates": (NPT3 + "deform 1e-4 2e-4 -1e-4 1 1 1\n", 11, "si"),
    "deform_open_z": (NPT3 + "deform 2e-4 0 1 1\n", 11, "si_open_z"),
}


def tersoff_system(variant):
    if variant == "sic":
        s = cc._sic(8, 45, rattle=0.05)  # 4096 atoms
        return s, cc.SIC
    s = diamond(8, a=5.431, rattle=0.05, seed=3)  # 4096 atoms, 43.4 A
    if variant == "si_open_z":
        s = dict(s, pbc=np.array([1, 1, 0], np.int32))
    if variant == "si_tric":
        L = s["h"][0]
        s = tilt(s, 0.08 * L, -0.05 * L, 0.06 * L)
    return s, cc.SI


def compare_runs(out, what):
    """Frame-by-frame gaps of the on run from the off run; returns the measured maxima."""
    fa = read_frames(out["on"][1] / "dump.xyz")
    fb = read_frames(out["off"][1] / "dump.xyz")
    ta = read_thermo(out["on"][1] / "thermo.out")
    tb = read_thermo(out["off"][1] / "thermo.out")
    assert len(fa) == len(fb) == ta.shape[0] == tb.shape[0] and len(fa) > 0
    gap = dict(pos=0.0, vel=0.0, h=0.0, thermo=0.0)
    for k, (a, b) in enumerate(zip(fa, fb)):
        hs = np.abs(b["h"]).max()
        gap["h"] = max(gap["h"], np.abs(a["h"] - b["h"]).max() / hs)
        gap["pos"] = max(gap["pos"], np.abs(mic(b["h"], [1, 1, 1], a["pos"] - b["pos"])).max())
        gap["vel"] = max(gap["vel"], np.abs(a["vel"] - b["vel"]).max() / np.abs(b["vel"]).max())
        scale = np.maximum(np.abs(tb[k]), 1e-3 * np.abs(tb).max(axis=0) + 1e-300)
        gap["thermo"] = max(gap["thermo"], (np.abs(ta[k] - tb[k]) / scale).max())
        for key in gap:
            assert gap[key] <= STEP_BOUND[key], (what, k, key, gap[key])
    print(f"\non/off gap {what}: " + " ".join(f"{k}={v:.2e}" for k, v in gap.items()))
    return gap, fa, fb


def run_tersoff(tmp_path, variant, body, vel=True):
    s, path = tersoff_system(variant)
    v = init_velocities(s["mass"], 300.0, seed=11) if vel else None
    write_model(tmp_path / "model.xyz", s, nep_type_order(path), v, [labels(s)[0]])
    model = (tmp_path / "model.xyz").read_text()
    out = run_both(tmp_path, {"model.xyz": model, "potential.txt": path},
                   f"potential potential.txt\ntime_step 1\n{body}")
    return s, out


@pytest.mark.parametrize("case", list(ENSEMBLES))
def test_plugin_ensembles_follow_the_reference_step_by_step(exe, tmp_path, case):
    """Every ensemble the plugin takes over, on FP64 Tersoff through the plugin and through the reference."""
    body, etype, variant = ENSEMBLES[case]
    s, out = run_tersoff(tmp_path, variant, f"{body}dump_thermo 1\n{DUMP}\nrun {STEPS}\n")
    assert_routes(out, "tersoff", etype)
    _, fa, fb = compare_runs(out, case)
    h0, h1 = s["h"], fb[-1]["h"]
    if case.startswith("deform"):
        rates = [float(x) for x in body.split("deform ")[1].split()[:-3]]
        rates = rates * 3 if len(rates) == 1 else rates
        flags = [int(x) for x in body.split("deform ")[1].split()[-3:]]
        for d in range(3):  # the deformed directions grow by the rate per step, open or not
            want = h0[4 * d] + STEPS * rates[d] if flags[d] else None
            if want is not None:
                assert abs(h1[4 * d] - want) < 1e-9, (d, h1[4 * d], want)
    if variant == "si_open_z" and "deform_open_z" not in case:
        assert fb[-1]["h"][8] == h0[8]
    if "fix" in case and not case.startswith("nvt_lan"):  # the fixed group at rest on both sides (nvt_lan's
        fixed = labels(s)[0] == 0  # last kick draws noise for the fixed atoms too)
        assert np.all(fa[-1]["vel"][:, fixed] == 0) and np.all(fb[-1]["vel"][:, fixed] == 0)


def test_velocity_then_two_runs_draw_the_same_rand_values(exe, tmp_path):
    """`velocity 300` draws rand() on both sides, then each ensemble seeds its generator with the next
    rand() value: the second run's nvt_bao must take the value after nvt_lan's."""
    body = (f"velocity 300\nensemble nvt_lan 300 300 50\ndump_thermo 1\n{DUMP}\nrun {STEPS // 2}\n"
            f"ensemble nvt_bao 300 300 50\ndump_thermo 1\n{DUMP}\nrun {STEPS // 2}\n")
    _, out = run_tersoff(tmp_path, "si", body, vel=False)
    assert_routes(out, "tersoff", 3)
    assert "Use the b200md integrator for ensemble type 5." in out["on"][0]
    compare_runs(out, "velocity+lan+bao")


# ---------------------------------------------------------------- 3. deform in the library's barostat

def berendsen_call(h, pbc, thermo, p0, pc, deform, rate, pos):
    import torch
    from gpumd_b200 import lib as L
    lib = L.load()
    n = pos.shape[1]
    d_pos = torch.as_tensor(pos.reshape(-1).copy(), device="cuda")
    d_th = torch.as_tensor(thermo, device="cuda")
    hh = (C.c_double * 9)(*h)
    L.check(lib.b200md_berendsen_pressure(
        n, n, 3, p0.ctypes.data_as(C.POINTER(C.c_double)), pc.ctypes.data_as(C.POINTER(C.c_double)),
        (C.c_int * 3)(*deform), (C.c_double * 3)(*rate), pbc.ctypes.data_as(C.POINTER(C.c_int)), hh,
        C.c_void_p(d_th.data_ptr()), C.c_void_p(d_pos.data_ptr()), None))
    return np.array(hh[:]), d_pos.cpu().numpy().reshape(3, n)


@pytest.mark.parametrize("case", ["x", "xyz_one_rate", "xyz_three_rates", "open_z"])
def test_deform_in_the_barostat_matches_restatement(oracle, case):
    """b200md_berendsen_pressure with `deform` (3 components): a deformed direction grows by its rate,
    even when it is open; the others follow the pressure (periodic) or stay (open)."""
    rng = np.random.default_rng(8)
    n = 20_011
    h = np.diag([40.0, 41.0, 42.0]).reshape(9)
    pbc = np.array([1, 1, 0 if case == "open_z" else 1], np.int32)
    pos = rng.uniform(0, 40, (3, n))
    thermo = np.array([300.0, -1.0, 0.010, 0.012, 0.008, 0.001, -0.002, 0.0005])
    p0 = np.array([0.003, 0.002, 0.001, 0.0, 0.0, 0.0])
    pc = np.array([0.5, 0.4, 0.3, 0.0, 0.0, 0.0])
    deform, rate = {"x": ((1, 0, 0), (1e-3, 1e-3, 1e-3)), "xyz_one_rate": ((1, 1, 1), (2e-3, 2e-3, 2e-3)),
                    "xyz_three_rates": ((1, 1, 1), (1e-3, -2e-3, 3e-3)),
                    "open_z": ((0, 1, 1), (1e-3, 2e-3, 3e-3))}[case]
    got_h, got_pos = berendsen_call(h, pbc, thermo, p0, pc, deform, rate, pos)
    h_ref, mu = oracle.berendsen_pressure(h, pbc, thermo, p0, pc, 3, deform=deform, deform_rate=rate)
    assert np.allclose(got_h, h_ref, rtol=1e-15, atol=1e-15)
    assert np.allclose(got_pos, mu.reshape(3, 3) @ pos, rtol=1e-14, atol=1e-14 * 40)
    for d in range(3):
        if deform[d]:
            assert abs(got_h[4 * d] - (h[4 * d] + rate[d])) < 1e-12


# ---------------------------------------------------------------- 4. reference classes on plugin outputs

HEAT = {"heat_lan": "ensemble heat_lan 300 50 20 1 3\n", "heat_nhc": "ensemble heat_nhc 300 50 20 1 3\n",
        "heat_bdp": "ensemble heat_bdp 300 50 20 1 3\n"}


@pytest.mark.parametrize("kind", list(HEAT))
def test_reference_heat_baths_run_on_plugin_tersoff(exe, tmp_path, kind):
    """The plugin declines heat_*: the reference's own baths integrate on libb200md's Tersoff forces and
    its `compute` averages them; FP64 on both sides, so compute.out agrees to its printed digits."""
    body = f"{HEAT[kind]}{FIX}compute 0 2 10 temperature potential force virial\ndump_thermo 1\n{DUMP}\nrun {STEPS}\n"
    _, out = run_tersoff(tmp_path, "si", body)
    assert_routes(out, "tersoff", None)
    compare_runs(out, kind)
    a = np.loadtxt(out["on"][1] / "compute.out")
    b = np.loadtxt(out["off"][1] / "compute.out")
    assert a.shape == b.shape and a.size > 0
    assert np.allclose(a, b, rtol=1e-8, atol=1e-8 * np.abs(b).max())


def read_table(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#") and ln.strip()], dtype=np.float64)


def _pbte_model(tmp_path, reps=6):
    s = rocksalt_pbte(reps, rattle=0.02, seed=1)
    write_model(tmp_path / "model.xyz", s, nep_type_order(GOLDEN / "nep_PbTe.txt"),
                init_velocities(s["mass"], 300.0, seed=42), [labels(s)[0]])
    return s, (tmp_path / "model.xyz").read_text()


@pytest.mark.parametrize("pot", ["tersoff", "nep"])
def test_reference_hac_and_shc_read_plugin_virials(exe, tmp_path, pot):
    """compute_hac and compute_shc of the reference on the per-atom virials the plugin writes (GPUMD's
    [9, N] layout): hac.out and shc.out as without the plugin -- to the printed digits on FP64 Tersoff,
    to the FP32 tolerance on NEP PbTe."""
    meas = "compute_hac 1 10 1\ncompute_shc 1 100 0 20 400.0 group 0 1\n"  # the reference wants Nc >= 100
    if pot == "tersoff":
        _, out = run_tersoff(tmp_path, "si", f"ensemble nve\n{meas}run 120\n")
        rtol = 1e-8
    else:
        _, model = _pbte_model(tmp_path)
        out = run_both(tmp_path, {"model.xyz": model, "potential.txt": GOLDEN / "nep_PbTe.txt"},
                       f"potential potential.txt\ntime_step 1\nensemble nve\n{meas}run 120\n")
        rtol = 1e-4
    assert_routes(out, "tersoff" if pot == "tersoff" else "nep", 0)
    for f in ("hac.out", "shc.out"):
        a = read_table(out["on"][1] / f)
        b = read_table(out["off"][1] / f)
        assert a.shape == b.shape and a.size > 0, f
        assert np.array_equal(np.isnan(a), np.isnan(b)), f  # columns the reference leaves undefined
        scale = np.nanmax(np.abs(b), axis=0)
        assert np.nanmax(scale) > 0, f
        assert np.allclose(a, b, rtol=rtol, atol=rtol * np.nan_to_num(scale), equal_nan=True), \
            (f, np.nanmax(np.abs(a - b)))


@pytest.mark.parametrize("mode", ["average", "observe"])
def test_two_nep_potentials_average_and_observe(oracle, exe, tmp_path, mode):
    """Two NEP models over the same species: the reference zeroes the per-atom arrays once and every
    potential adds into them; `average` divides by two, `observe` runs the first only.  The dumped arrays
    against the mean of (or the first of) two oracle evaluations at the dumped positions."""
    s, model = _pbte_model(tmp_path, reps=4)
    a, b = GOLDEN / "nep_PbTe.txt", GOLDEN / "nep_PbTe_static.txt"
    out = run_both(tmp_path, {"model.xyz": model, "a.txt": a, "b.txt": b},
                   f"potential a.txt\npotential b.txt\ntime_step 1\nensemble nve\n"
                   f"dump_observer {mode} 1 1 0 1\ndump_thermo 1\n{DUMP}\nrun 1\n")
    assert_routes(out, "nep", 0)
    assert out["on"][0].count("Use the b200md NEP backend") == 2
    from oracle import oracle_py
    for tag in ("on", "off"):
        fr = read_frames(out[tag][1] / "dump.xyz")[0]
        rs = [oracle_py.NepOracle(p).compute(s["type"], fr["h"], s["pbc"], fr["pos"], precision=32) for p in (a, b)]
        want = rs[0] if mode == "observe" else {k: 0.5 * (rs[0][k] + rs[1][k]) for k in ("pe", "force", "virial")}
        check_fv(fr, want)
        n = s["type"].shape[0]
        assert abs(fr["pe"].sum() - want["pe"].sum()) / n < TOL["energy_per_atom"], tag
    # the two models differ by ~40 times the force tolerance, so averaging and observing are told apart
    assert np.abs(rs[0]["force"] - rs[1]["force"]).max() > 5e-3

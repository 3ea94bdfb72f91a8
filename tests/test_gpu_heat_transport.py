"""HNEMD (driving force, heat-current sums, kappa) and SHC (blocked ring correlation) on the device,
against the numpy restatements of tests/heat_oracle.py, and through the `b200md` driver against the
unmodified reference gpumd (tests/golden/refgpu_hnemd_*, scripts/run_reference_gpumd.py)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import heat_oracle as ho
from conftest import GOLDEN
from gpumd_b200.structures import (TIME_UNIT_CONVERSION, graphene_sheet, init_velocities, nep_type_order,
                                   read_xyz, rocksalt_pbte, write_xyz)

pytestmark = pytest.mark.gpu
ROWS = [[0, 3, 4], [6, 1, 5], [7, 8, 2]]  # virial row of each transport direction, shc.cu:188


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def _dev(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64).reshape(-1), device="cuda")


@pytest.mark.parametrize("n", [1, 1001, 1_000_000])
def test_drive_matches_restatement(eng, n):
    rng = np.random.default_rng(n)
    w, f = rng.normal(size=(9, n)), rng.normal(size=(3, n))
    fe = (2e-3, -1e-3, 5e-4)
    d_w, d_f = _dev(w), _dev(f)
    eng.hnemd_drive(n, fe, d_w, d_f)
    got = d_f.cpu().numpy().reshape(3, n)
    want = ho.hnemd_drive(w, f, fe)
    assert np.allclose(got, want, rtol=1e-13, atol=1e-13 * np.abs(want).max())
    assert np.abs(got.sum(axis=1)).max() <= 1e-12 * np.abs(got).sum()
    # deterministic: the same call on the same input gives the same bits
    d_f2 = _dev(f)
    eng.hnemd_drive(n, fe, d_w, d_f2)
    assert np.array_equal(d_f2.cpu().numpy(), d_f.cpu().numpy())


def test_drive_per_atom_add_is_the_references_fma_nesting(eng):
    """32 atoms, atom 16 + i the negative of atom i: the first shuffle step of the block sum pairs
    exactly these, so ftot is exactly zero and the correction is a no-op.  The output is then the
    per-atom add alone, which must equal f + fma(fe_z, W_z, fma(fe_x, W_x, fe_y * W_y)) bit for bit
    (numpy has no fused multiply-add: the reference expression is rebuilt from exact rationals)."""
    from fractions import Fraction
    rng = np.random.default_rng(9)
    n = 32
    w = rng.normal(size=(9, n // 2))
    w = np.concatenate([w, -w], axis=1)
    f = rng.normal(size=(3, n // 2))
    f = np.concatenate([f, -f], axis=1)
    fe = (2e-3, -1e-3, 5e-4)
    d_f = _dev(f)
    eng.hnemd_drive(n, fe, _dev(w), d_f)
    got = d_f.cpu().numpy().reshape(3, n)

    def fma(a, b, c):
        return float(Fraction(a) * Fraction(b) + Fraction(c))

    maps = [(0, 6, 7), (3, 1, 8), (4, 5, 2)]  # (W_x., W_y., W_z.) of each force component
    for d, (ix, iy, iz) in enumerate(maps):
        for i in range(n):
            t = fe[1] * w[iy, i]
            t = fma(fe[0], w[ix, i], t)
            t = fma(fe[2], w[iz, i], t)
            assert got[d, i] == f[d, i] + t, (d, i)


def test_hnemd_heat_sums_and_kappa_match_restatement(eng):
    rng = np.random.default_rng(5)
    n, oi, fe = 20_011, 7, (0.0, 1e-5, 0.0)
    atom = eng.Atom(np.zeros(n, np.int32), np.zeros((3, n)), np.ones(n), np.zeros((3, n)))
    h = eng.HNEMD(oi, fe)
    V, T = 5.0e4, 300.0
    rows = []
    for step in range(2 * oi):
        v, w = rng.normal(size=(3, n)), rng.normal(size=(9, n))
        atom.velocity_per_atom.copy_(_dev(v))
        atom.virial_per_atom.copy_(_dev(w))
        rows.append(ho.hnemd_heat_row(w, v))
        h.process(step, atom)
        if (step + 1) % oi == 0:
            kappa, got_rows = h.take(V, T)
            want_rows = np.array(rows[-oi:])
            assert np.allclose(got_rows, want_rows, rtol=1e-12, atol=1e-12 * np.abs(want_rows).max())
            want = ho.hnemd_kappa(want_rows, V, T, fe)
            assert np.allclose(kappa, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


def _shc_run(eng, n, sample_interval, Nc, direction, steps, groups, seed=1):
    """Drive the device SHC and the brute-force restatement with the same random series."""
    import torch
    rng = np.random.default_rng(seed)
    atom = eng.Atom(np.zeros(n, np.int32), np.zeros((3, n)), np.ones(n), np.zeros((3, n)))
    shc = eng.SHC(sample_interval, Nc, direction, steps, num_atoms=n, groups=groups)
    s_hist, v_hist = [], []
    for step in range(steps):
        if (step + 1) % sample_interval == 0:
            w = rng.normal(size=(9, n))
            v = rng.normal(size=(3, n))
            atom.virial_per_atom.copy_(torch.as_tensor(w.reshape(-1), device="cuda"))
            atom.velocity_per_atom.copy_(torch.as_tensor(v.reshape(-1), device="cuda"))
            s_hist.append(w[ROWS[direction]])
            v_hist.append(v)
        shc.process(step, atom)
    return shc, np.array(s_hist), np.array(v_hist)


SHC_CASES = {
    # name: (n, sample_interval, Nc, direction, steps, groups builder)
    "single_group_Nc100_exact": (3000, 1, 100, 0, 100, lambda n, r: [r.permutation(n)[:1234]]),
    "uneven_groups_Nc100": (4000, 2, 100, 1, 2 * 171 + 1, lambda n, r: [np.arange(0, 1), r.permutation(n)[:257],
                                                                        np.arange(1000, 4000)]),
    "whole_system_Nc100_wraps": (2500, 3, 100, 2, 3 * 237, None),
    "uneven_groups_Nc1000": (700, 1, 1000, 1, 1037, lambda n, r: [np.arange(0, 300), np.arange(300, 333),
                                                                 np.arange(333, 700)]),
    "whole_system_Nc1000_exact": (500, 1, 1000, 0, 1000, None),
}


@pytest.mark.parametrize("case", list(SHC_CASES))
def test_shc_matches_brute_force(eng, case):
    n, si, Nc, direction, steps, build = SHC_CASES[case]
    groups = None if build is None else build(n, np.random.default_rng(7))
    shc, s_hist, v_hist = _shc_run(eng, n, si, Nc, direction, steps, groups)
    dt, num_omega, max_omega = 1.0 / TIME_UNIT_CONVERSION, 50, 400.0
    ki, ko, si_, so_ = shc.postprocess(dt, num_omega, max_omega)
    dt_in_ps = dt * si * TIME_UNIT_CONVERSION / 1000.0
    for g, idx in enumerate([np.arange(n)] if groups is None else groups):
        k, origins = ho.shc_brute_force(s_hist[:, :, idx], v_hist[:, :, idx], Nc)
        assert origins == steps // si - Nc + 1
        want_i, want_o = ho.shc_window(*ho.shc_average_k(k, Nc, origins), Nc)
        for got, want in ((ki[g], want_i), (ko[g], want_o)):
            assert np.allclose(got, want, rtol=1e-11, atol=1e-11 * np.abs(want).max())
        _, wsi, wso = ho.shc_transform(want_i, want_o, Nc, dt_in_ps, num_omega, max_omega)
        assert np.allclose(si_[g], wsi, rtol=1e-11, atol=1e-11 * np.abs(wsi).max())
        assert np.allclose(so_[g], wso, rtol=1e-11, atol=1e-11 * np.abs(wso).max())


def test_shc_is_deterministic(eng):
    n, si, Nc, direction, steps = 5000, 1, 100, 1, 160
    groups = [np.arange(0, 2500), np.arange(2500, 5000)]
    out = []
    for _ in range(2):
        shc, _, _ = _shc_run(eng, n, si, Nc, direction, steps, groups, seed=3)
        out.append(shc.postprocess(0.1, 20, 100.0))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_shc_rejects_bad_arguments(eng):
    from gpumd_b200 import lib
    for args in ((1, 99, 0, 1000), (1, 1001, 0, 2000), (0, 100, 0, 1000), (51, 100, 0, 10000),
                 (1, 100, 3, 1000), (2, 100, 0, 199)):  # the last: 99 samples, no time origin
        with pytest.raises(lib.B200mdError):
            eng.SHC(*args, num_atoms=100)
    eng.SHC(2, 100, 0, 200, num_atoms=100)  # exactly one time origin


# ---- the `b200md` driver -----------------------------------------------------------------------

def _run_exe(tmp_path, run_in, timeout=900):
    from gpumd_b200 import build
    exe = build.build_host()
    (tmp_path / "run.in").write_text(run_in)
    return subprocess.run([str(exe)], cwd=tmp_path, capture_output=True, text=True, timeout=timeout)


def read_thermo(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#")], dtype=np.float64)


def read_shc(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#") and ln.strip()], dtype=np.float64)


def _graphene_inputs(tmp_path):
    s = graphene_sheet()
    write_xyz(tmp_path / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    return s


GRAPHENE_RUN = ("potential potential.txt\nensemble nvt_nhc 300 300 100\ntime_step 1\ndump_thermo 10\n"
                "compute_hnemd 20 0 0.00001 0\ncompute_shc 1 100 1 200 400.0 group 0 4\nrun 400\n")


def test_driver_graphene_hnemd_matches_reference(tmp_path):
    """FP64 Tersoff, nvt_nhc, the reference's graphene HNEMD case shortened to 400 steps: kappa.out,
    shc.out and thermo.out against the unmodified reference gpumd."""
    if not (GOLDEN / "refgpu_hnemd_graphene_kappa.out").exists():
        pytest.skip("refgpu_hnemd_graphene_* not generated yet")
    _graphene_inputs(tmp_path)
    r = _run_exe(tmp_path, GRAPHENE_RUN)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    # trajectory tolerance of the HAC pin (test_gpu_host_exe.py): FP64 force field, same integrator
    mine, ref = read_thermo(tmp_path / "thermo.out"), read_thermo(GOLDEN / "refgpu_hnemd_graphene_thermo.out")
    assert mine.shape == ref.shape == (40, 18)
    assert np.allclose(mine[:, :3], ref[:, :3], rtol=1e-5, atol=1e-6 * np.abs(ref[:, :3]).max())
    k_mine, k_ref = np.loadtxt(tmp_path / "kappa.out"), np.loadtxt(GOLDEN / "refgpu_hnemd_graphene_kappa.out")
    assert k_mine.shape == k_ref.shape == (20, 5)
    assert np.allclose(k_mine, k_ref, rtol=1e-5, atol=1e-6 * np.abs(k_ref).max())
    s_mine, s_ref = read_shc(tmp_path / "shc.out"), read_shc(GOLDEN / "refgpu_hnemd_graphene_shc.out")
    assert s_mine.shape == s_ref.shape == (399, 3)
    assert np.array_equal(s_mine[:, 0], s_ref[:, 0])
    assert np.allclose(s_mine[:, 1:], s_ref[:, 1:], rtol=1e-4, atol=1e-5 * np.abs(s_ref[:, 1:]).max())
    head = [ln for ln in open(tmp_path / "shc.out") if ln.startswith("#")]
    assert head == [ln for ln in open(GOLDEN / "refgpu_hnemd_graphene_shc.out") if ln.startswith("#")]


def test_driver_pbte_nep_hnemd_matches_reference(tmp_path):
    """FP32 NEP (store mode: the drive runs after the overwriting final kernel), nvt_ber, SHC over all
    groups but 0 of four slabs along x."""
    if not (GOLDEN / "refgpu_hnemd_pbte_kappa.out").exists():
        pytest.skip("refgpu_hnemd_pbte_* not generated yet")
    s = rocksalt_pbte(12, rattle=0.02, seed=31)
    s["group"] = np.minimum((s["pos"][0] / s["h"][0] * 4).astype(np.int32), 3)
    write_xyz(tmp_path / "model.xyz", s, nep_type_order(GOLDEN / "nep_PbTe.txt"),
              init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "nep_PbTe.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\nensemble nvt_ber 300 300 100\ntime_step 1\ndump_thermo 10\n"
                           "compute_hnemd 10 0.00002 0 0\ncompute_shc 2 100 0 100 200 group 0 -1\nrun 250\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    mine, ref = read_thermo(tmp_path / "thermo.out"), read_thermo(GOLDEN / "refgpu_hnemd_pbte_thermo.out")
    assert mine.shape == ref.shape == (25, 18)
    for k in range(25):  # NEP trajectory tolerances of test_gpu_host_exe.py
        tol = 2e-5 * (1 + k)
        assert abs(mine[k, 0] - ref[k, 0]) < tol * 10 * 300.0
        assert abs(mine[k, 2] - ref[k, 2]) < tol * abs(ref[k, 2])
    k_mine, k_ref = np.loadtxt(tmp_path / "kappa.out"), np.loadtxt(GOLDEN / "refgpu_hnemd_pbte_kappa.out")
    assert k_mine.shape == k_ref.shape == (25, 5)
    # FP32 forces: the heat current of a 10-step interval follows the trajectory to ~1e-3 of its scale
    assert np.allclose(k_mine, k_ref, rtol=0, atol=2e-2 * np.abs(k_ref).max()), np.abs(k_mine - k_ref).max()
    s_mine, s_ref = read_shc(tmp_path / "shc.out"), read_shc(GOLDEN / "refgpu_hnemd_pbte_shc.out")
    assert s_mine.shape == s_ref.shape == (3 * 299, 3)
    assert np.array_equal(s_mine[:, 0], s_ref[:, 0])
    assert np.allclose(s_mine[:, 1:], s_ref[:, 1:], rtol=0, atol=2e-2 * np.abs(s_ref[:, 1:]).max())


def test_driver_resets_hnemd_and_shc_after_a_run(tmp_path, eng):
    """A second `run` without the keywords writes no kappa.out rows and no shc.out block, and its forces
    are the undriven forces of the potential (Force::finalize)."""
    s = graphene_sheet(20, 21)
    s["group"] = np.minimum((s["pos"][0] / s["h"][0] * 3).astype(np.int32), 2)  # three slabs along x
    write_xyz(tmp_path / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\nensemble nvt_ber 300 300 100\ntime_step 1\n"
                           "compute_hnemd 10 0 0.001 0\ncompute_shc 1 100 1 10 400.0 group 0 -1\nrun 120\n"
                           "ensemble nve\ntime_step 0\ndump_xyz 1 dump.xyz precision double force\nrun 3\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert np.loadtxt(tmp_path / "kappa.out").shape == (12, 5)
    text = open(tmp_path / "shc.out").read()
    assert text.count("# compute_shc") == 1 and "# num_output_groups 2" in text
    assert read_shc(tmp_path / "shc.out").shape == (2 * (199 + 10), 3)
    frames = open(tmp_path / "dump.xyz").read()
    n = s["type"].shape[0]
    last = "\n".join(frames.splitlines()[-(n + 2):]) + "\n"
    (tmp_path / "last.xyz").write_text(last)
    out = read_xyz(tmp_path / "last.xyz", ["C"])
    pot = eng.Tersoff1989(GOLDEN / "Graphene_Lindsay_2010_modified.txt", n)
    atom = eng.Atom(np.zeros(n, np.int32), out["pos"], s["mass"])
    box = eng.Box(s["h"], s["pbc"])
    pot.compute(box, atom.type, atom.position_per_atom, atom.potential_per_atom, atom.force_per_atom,
                atom.virial_per_atom)
    f = atom.force_per_atom.cpu().numpy().reshape(3, n)
    assert np.allclose(out["forces"], f, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("line,msg", [
    ("compute_hnemdec 0 1000 0 0.00001 0", "not a keyword"),
    ("compute_shc 1 100 1 200 400.0\nrun 50", "no time origin"),
    ("compute_shc 1 99 1 200 400.0", "Nc for SHC should >= 100"),
    ("compute_shc 51 100 1 200 400.0", "should <= 50"),
    ("compute_hnemd 0 0 0.00001 0", "larger than 0"),
    ("compute_hnemd 10 0 1e-5 0\ncompute_hnemd 10 0 1e-5 0", "more than one HNEMD"),
])
def test_driver_rejects_bad_heat_transport_input(tmp_path, line, msg):
    _ = tmp_path
    s = graphene_sheet(10, 11)
    write_xyz(tmp_path / "model.xyz", s, ["C"])
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, f"potential potential.txt\nvelocity 300\nensemble nve\n{line}\n", timeout=120)
    assert r.returncode == 1 and "Input Error" in r.stderr and msg in r.stderr, r.stderr


def test_patched_reference_binary_runs_hnemd_on_libb200md_virials(tmp_path):
    """The reference gpumd with libb200md behind its Potential interface (oracle/_ref/gpumd_b200,
    GPUMD_B200=1) keeps running compute_hnemd / compute_shc through its own Force and Measure code on
    top of libb200md's per-atom virial: kappa.out and shc.out as without GPUMD_B200."""
    from conftest import ROOT
    exe = ROOT / "oracle" / "_ref" / "gpumd_b200"
    if not exe.exists():
        pytest.skip("oracle/_ref/gpumd_b200 is built by build() only where the reference tree exists")
    out = {}
    for flag in ("0", "1"):
        d = tmp_path / flag
        d.mkdir()
        _graphene_inputs(d)
        (d / "run.in").write_text(GRAPHENE_RUN)
        env = dict(os.environ)
        env.pop("GPUMD_B200", None)
        if flag == "1":
            env["GPUMD_B200"] = "1"
        r = subprocess.run([str(exe)], cwd=d, capture_output=True, text=True, timeout=900, env=env)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        out[flag] = (np.loadtxt(d / "kappa.out"), read_shc(d / "shc.out"))
    (k0, s0), (k1, s1) = out["0"], out["1"]
    assert k0.shape == k1.shape == (20, 5) and s0.shape == s1.shape
    assert np.allclose(k1, k0, rtol=1e-5, atol=1e-6 * np.abs(k0).max())
    assert np.allclose(s1[:, 1:], s0[:, 1:], rtol=1e-4, atol=1e-5 * np.abs(s0[:, 1:]).max())

"""Energy minimization on the device (b2_minimize.cu) against the numpy restatement of the reference's
minimizers (tests/minimize_oracle.py): single iterations from random states, lock-step trajectories on
every potential, and the `minimize` keyword of the b200md driver."""
import shutil
import subprocess

import numpy as np
import pytest
import torch

import minimize_oracle as M
from conftest import GOLDEN
from gpumd_b200.structures import diamond, fcc, nep_type_order, read_xyz, rocksalt_pbte, write_xyz

pytestmark = pytest.mark.gpu


def _engine():
    from gpumd_b200 import engine
    return engine


def to_np(t, rows):
    return t.detach().cpu().numpy().reshape(rows, -1)


def random_atom(rng, n, scale=1.0):
    E = _engine()
    atom = E.Atom(np.zeros(n, np.int32), rng.uniform(0, 20, (3, n)), np.ones(n))
    atom.force_per_atom.copy_(torch.as_tensor(rng.normal(0, scale, 3 * n)))
    atom.potential_per_atom.copy_(torch.as_tensor(rng.normal(-3, 0.1, n)))
    atom.virial_per_atom.copy_(torch.as_tensor(rng.normal(0, 1.0, 9 * n)))
    return atom


def close(a, b, rtol=1e-12):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.allclose(a, b, rtol=rtol, atol=rtol * max(1.0, np.abs(b).max()))


def check_record(rec, ref, box_change):
    E = _engine()
    assert bool(rec[E.MIN_CONVERGED]) == ref["converged"]
    assert close(rec[E.MIN_FMAX], ref["f_max"]) and close(rec[E.MIN_U], ref["u"])
    assert close(rec[E.MIN_P], ref["P"], 1e-10)
    if box_change:
        assert close(rec[E.MIN_PRESSURE], ref["pressure"]) and close(rec[E.MIN_STRESS], ref["stress"])
    if not ref["converged"]:
        assert bool(rec[E.MIN_UPHILL]) == ref["uphill"]
        assert close(rec[E.MIN_FMOD], ref["F_mod"]) and close(rec[E.MIN_VMOD], ref["v_mod"])


@pytest.mark.parametrize("box_change,hydrostatic", [(0, 0), (1, 0), (1, 1)])
def test_fire_single_iterations_match_the_restatement(box_change, hydrostatic):
    """Random forces drive both P branches; one stretch starts at N_neg = N_min - 1 near dt_max with F
    along v (the N_neg > N_min crossing and the dt_max rule), one near dt_min with F against v."""
    E = _engine()
    rng = np.random.default_rng(7 + box_change + hydrostatic)
    n = 3000
    atom = random_atom(rng, n)
    h = np.array([20.0, 0.5, 0.2, 0.0, 21.0, 0.3, 0.0, 0.0, 19.0])
    box = E.Box(h.copy())
    mz = E.Minimizer("fire", n, 1e-30, 100, box_change, hydrostatic)
    x = to_np(atom.position_per_atom, 3)
    v = np.zeros((3, n))
    st = M.fire_state(L=np.cbrt(abs(np.linalg.det(h.reshape(3, 3)))))
    seen = dict(uphill=0, down=0, crossing=0, dtmax=0, dtmin=0)
    for it in range(40):
        if it == 12:  # just below the N_neg crossing, dt near dt_max
            st = dict(st, n_neg=M.N_MIN - 1, dt=0.97 * M.DT_MAX, alpha=0.2)
        if it == 28:  # near dt_min
            st = dict(st, dt=1.2 * M.DT_MIN)
        if it in (12, 28):
            rec = np.zeros(E.MIN_RECORD)
            rec[E.MIN_DT], rec[E.MIN_ALPHA], rec[E.MIN_NNEG] = st["dt"], st["alpha"], st["n_neg"]
            rec[E.MIN_VBOX:E.MIN_VBOX + 9] = st["v_box"]
            rec[E.MIN_LSCALE] = st["L"]
            mz.set_record(rec)
        F = rng.normal(0, 1.0, (3, n))
        if 12 <= it < 28:
            F = F * 0.1 + v / max(np.abs(v).max(), 1e-30)  # downhill
        elif it >= 28:
            F = F * 0.1 - v / max(np.abs(v).max(), 1e-30)  # uphill when v != 0
        W = rng.normal(0, 1.0, (9, n))
        U = rng.normal(-3, 0.1, n)
        atom.force_per_atom.copy_(torch.as_tensor(F.reshape(-1)))
        atom.virial_per_atom.copy_(torch.as_tensor(W.reshape(-1)))
        atom.potential_per_atom.copy_(torch.as_tensor(U))
        dt_before, alpha_before = st["dt"], st["alpha"]
        rec = mz.fire_step(box, atom)
        x, v, h, st, ref = M.fire_step(x, v, F, U, W, h, st, 1e-30, bool(box_change), bool(hydrostatic))
        check_record(rec, ref, box_change)
        assert rec[E.MIN_NNEG] == st["n_neg"] and close(rec[E.MIN_DT], st["dt"]) and close(
            rec[E.MIN_ALPHA], st["alpha"])
        assert close(to_np(atom.position_per_atom, 3), x)
        if box_change:
            assert close(box.cpu_h, h) and close(rec[E.MIN_VBOX:E.MIN_VBOX + 9], st["v_box"])
            if hydrostatic:
                assert np.count_nonzero(rec[E.MIN_FBOX:E.MIN_FBOX + 9][[1, 2, 3, 5, 6, 7]]) == 0
        crossing = not ref["uphill"] and st["alpha"] < alpha_before
        seen["uphill" if ref["uphill"] else "down"] += 1
        seen["crossing"] += crossing
        seen["dtmax"] += crossing and dt_before * M.F_INC >= M.DT_MAX
        seen["dtmin"] += ref["uphill"] and dt_before * M.F_DEC <= M.DT_MIN
    assert all(v > 0 for v in seen.values()), seen


def test_fire_box_change_force_guard_zeroes_the_mixing():
    E = _engine()
    n = 256
    rng = np.random.default_rng(3)
    atom = random_atom(rng, n)
    atom.force_per_atom.zero_()
    atom.virial_per_atom.zero_()
    box = E.Box(np.diag([10.0, 10.0, 10.0]).reshape(9))
    mz = E.Minimizer("fire", n, -1.0, 10, 1, 0)  # a negative tolerance never converges
    rec = mz.fire_step(box, atom)
    assert rec[E.MIN_FMOD] == 0.0 and rec[E.MIN_SCALE] == 0.0 and np.isfinite(to_np(atom.position_per_atom, 3)).all()


@pytest.mark.parametrize("fixed", [False, True])
def test_sd_single_iterations_match_the_restatement(fixed):
    E = _engine()
    rng = np.random.default_rng(11)
    n = 2000
    atom = random_atom(rng, n)
    label = rng.integers(0, 3, n).astype(np.int32)
    lab = torch.as_tensor(label, device="cuda") if fixed else None
    fg = 1 if fixed else -1
    mz = E.Minimizer("sd", n, 1e-30, 100)
    x, F = to_np(atom.position_per_atom, 3), to_np(atom.force_per_atom, 3)
    U = atom.potential_per_atom.cpu().numpy()
    rec = mz.sd_begin(atom, lab, fg)
    step = M.SD_STEP_0
    seen = set()
    for it in range(12):
        f_max = np.sqrt(np.max(F * F))
        assert close(rec[E.MIN_FMAX], f_max) and close(rec[E.MIN_U], U.sum())
        xt = M.sd_trial(x, F, f_max, step, label, fg)
        assert np.array_equal(to_np(mz.trial_position, 3), xt)  # the same two IEEE operations
        if fixed:
            assert np.array_equal(xt[:, label == fg], x[:, label == fg])
        Ft = rng.normal(0, 1.0, (3, n))
        Ut = U + rng.normal(0.0, 1e-3, n) + (1e-3 if it % 3 == 0 else -1e-3)
        mz.trial_force.copy_(torch.as_tensor(Ft.reshape(-1)))
        mz.trial_potential.copy_(torch.as_tensor(Ut))
        rec = mz.sd_step(atom, lab, fg)
        uphill, step, u_small = M.sd_decide(U, Ut, step)
        seen.add(uphill)
        assert bool(rec[E.MIN_UPHILL]) == uphill and close(rec[E.MIN_STEP], step)
        assert close(rec[E.MIN_USMALLER], u_small)
        if not uphill:
            x, F, U = xt, Ft, Ut
        assert np.array_equal(to_np(atom.position_per_atom, 3), x)
        assert np.array_equal(to_np(atom.force_per_atom, 3), F)
    assert seen == {True, False}


# lock-step systems: (structure, potential file, symbols)
def _triclinic(s):
    H = s["h"].reshape(3, 3).copy()
    H[0, 1] = 0.1 * H[1, 1]
    s = dict(s, h=H.reshape(9))
    s["pos"] = s["pos"] + np.outer(H[:, 1] - np.array([0, H[1, 1], 0]), s["pos"][1] / H[1, 1])
    return s


SYSTEMS = {
    "nep_pbte": (lambda: rocksalt_pbte(5, rattle=0.05, seed=2), "nep_PbTe.txt", None),
    "nep_pbte_triclinic": (lambda: _triclinic(rocksalt_pbte(5, rattle=0.05, seed=2)), "nep_PbTe.txt", None),
    "nep_pbte_small_box": (lambda: rocksalt_pbte(2, rattle=0.05, seed=2), "nep_PbTe.txt", None),
    "tersoff_si": (lambda: diamond(4, rattle=0.05, seed=4), "tersoff_Si_1989.txt", ["Si"]),
    "lj_ar": (lambda: fcc(6, 5.26, rattle=0.1, seed=3), "lj_Ar_10A.txt", ["Ar"]),
    "eam_cu": (lambda: fcc(7, 3.615, rattle=0.05, seed=5, symbols=("Cu",)), "eam_Cu_Zhou_2004.txt", ["Cu"]),
}


def _setup(case):
    E = _engine()
    make, pot, _ = SYSTEMS[case]
    s = make()
    n = s["type"].shape[0]
    atom = E.Atom(s["type"], s["pos"], s["mass"])
    box = E.Box(s["h"].copy(), s["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / pot, n)
    return atom, box, force, n


@pytest.mark.parametrize("method", ["fire", "fire_box", "sd"])
@pytest.mark.parametrize("case", list(SYSTEMS))
def test_lock_step_trajectory(case, method):
    """At every iteration the restatement gets the GPU's forces and must land on the GPU's state."""
    E = _engine()
    atom, box, force, n = _setup(case)
    a = atom
    iters = 40
    if method == "sd":
        mz = E.Minimizer("sd", n, 1e-12, iters)
        force.compute(box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
        x, F, U = to_np(a.position_per_atom, 3), to_np(a.force_per_atom, 3), a.potential_per_atom.cpu().numpy()
        rec = mz.sd_begin(a)
        step = M.SD_STEP_0
        for _ in range(iters):
            xt = M.sd_trial(x, F, np.sqrt(np.max(F * F)), step)
            assert close(to_np(mz.trial_position, 3), xt)
            force.compute(box, mz.trial_position, a.type, mz.trial_potential, mz.trial_force, a.virial_per_atom)
            xt, Ft, Ut = to_np(mz.trial_position, 3), to_np(mz.trial_force, 3), mz.trial_potential.cpu().numpy()
            rec = mz.sd_step(a)
            uphill, step, _ = M.sd_decide(U, Ut, step)
            assert bool(rec[E.MIN_UPHILL]) == uphill and close(rec[E.MIN_STEP], step)
            if not uphill:
                x, F, U = xt, Ft, Ut
            assert np.array_equal(to_np(a.position_per_atom, 3), x)
        return
    bc = method == "fire_box"
    mz = E.Minimizer("fire", n, 1e-12, iters, int(bc), 0)
    v = np.zeros((3, n))
    h = box.cpu_h.copy()
    st = M.fire_state(L=np.cbrt(box.get_volume()))
    for _ in range(iters):
        force.compute(box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
        x, F, W = to_np(a.position_per_atom, 3), to_np(a.force_per_atom, 3), to_np(a.virial_per_atom, 9)
        U = a.potential_per_atom.cpu().numpy()
        rec = mz.fire_step(box, a)
        x, v, h, st, ref = M.fire_step(x, v, F, U, W, h, st, 1e-12, bc)
        check_record(rec, ref, bc)
        assert close(to_np(a.position_per_atom, 3), x) and close(box.cpu_h, h)
    force.potentials[0].check()


def test_launch_count_per_iteration():
    """FIRE: one reduction + one update; SD: trial energy, accept + f_max, trial positions -- no helper
    kernels in between."""
    E = _engine()
    atom, box, force, n = _setup("lj_ar")
    a = atom
    for method, kernels in (("fire", 2), ("sd", 3)):
        mz = E.Minimizer(method, n, 1e-12, 10)
        force.compute(box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
        if method == "sd":
            mz.sd_begin(a)
            force.compute(box, mz.trial_position, a.type, mz.trial_potential, mz.trial_force, a.virial_per_atom)
            c0 = E.launch_count()
            mz.sd_step(a)
        else:
            c0 = E.launch_count()
            mz.fire_step(box, a)
        assert E.launch_count() - c0 == kernels


# ---- the `minimize` keyword of the driver ------------------------------------------------------------

def run_driver(tmp_path, s, symbols, potfile, run_in, timeout=600):
    from gpumd_b200 import build
    exe = build.build_host()
    write_xyz(tmp_path / "model.xyz", s, symbols)
    shutil.copyfile(GOLDEN / potfile, tmp_path / "potential.txt")
    (tmp_path / "run.in").write_text(run_in)
    return subprocess.run([str(exe)], cwd=tmp_path, capture_output=True, text=True, timeout=timeout)


def _progress(stdout):
    return [ln for ln in stdout.splitlines() if ln.startswith(("    step ", "    Position step", "  Converged!"))]


def test_driver_fire_box_change_then_nve(tmp_path):
    """minimize fire with box change, then NVE in the relaxed box: the neighbour lists follow the new box,
    energy is conserved, dump_restart and dump_xyz carry the relaxed box, and the progress lines are the
    ones the Python mirror prints for the same run."""
    s = fcc(6, 5.26 * 0.98, rattle=0.02, seed=3)  # LJ argon compressed by 2 %
    sym = ["Ar"]
    r = run_driver(tmp_path, s, sym, "lj_Ar_10A.txt",
                   "potential potential.txt\nminimize fire 1.0e-4 400 1\nvelocity 20 seed 3\nensemble nve\n"
                   "time_step 1\ndump_thermo 10\ndump_restart 200\ndump_xyz 200 dump.xyz precision double\n"
                   "run 200\n")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "Energy minimization with changed box started." in r.stdout
    # the Python mirror on the same library
    E = _engine()
    written = read_xyz(tmp_path / "model.xyz", sym)
    atom = E.Atom(written["type"], written["pos"], s["mass"])
    box = E.Box(written["h"].copy(), written["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / "lj_Ar_10A.txt", atom.number_of_atoms)
    lines, _ = E.Minimizer("fire", atom.number_of_atoms, 1e-4, 400, 1, 0).compute(force, box, atom)
    assert _progress(r.stdout) == lines
    thermo = np.loadtxt(tmp_path / "thermo.out")
    etot = thermo[:, 1] + thermo[:, 2]
    # The same NVE run from the ideal lattice in the relaxed box: plain-cutoff LJ at 1 fs does not hold the
    # total energy flat by itself (0.12 eV of swing in 200 fs, with or without a minimization before), so the
    # relaxed run must follow the control's energy history.  Measured: 5e-4 eV apart.
    a = np.diag(box.cpu_h.reshape(3, 3)) / 6
    ctl = tmp_path / "control"
    ctl.mkdir()
    r2 = run_driver(ctl, fcc(6, float(a.mean())), sym, "lj_Ar_10A.txt",
                    "potential potential.txt\nvelocity 20 seed 3\nensemble nve\ntime_step 1\ndump_thermo 10\n"
                    "run 200\n")
    assert r2.returncode == 0, r2.stderr[-2000:]
    control = np.loadtxt(ctl / "thermo.out")
    assert np.abs(etot - (control[:, 1] + control[:, 2])).max() < 5e-3
    rs = read_xyz(tmp_path / "restart.xyz", sym)
    dump = read_xyz(tmp_path / "dump.xyz", sym)
    assert np.allclose(rs["h"], box.cpu_h, rtol=1e-5) and np.allclose(dump["h"], box.cpu_h, rtol=1e-9)
    assert not np.allclose(box.cpu_h, s["h"], rtol=1e-3)  # the box did relax
    assert np.allclose(thermo[:, -9:].reshape(-1, 9)[0][[0, 4, 8]], np.diag(box.cpu_h.reshape(3, 3)), rtol=1e-5)


def test_driver_sd_with_fix_is_bit_identical_run_to_run(tmp_path):
    """SD with `fix 0` through the driver twice: identical dumps (fixed-order reductions), fixed atoms in
    place, and the progress lines of the Python mirror."""
    s = diamond(4, rattle=0.05, seed=4)
    n = s["type"].shape[0]
    s["group"] = (np.arange(n) % 4 == 0).astype(np.int32)
    out = []
    for k in range(2):
        d = tmp_path / str(k)
        d.mkdir()
        write = dict(s)
        r = run_driver(d, write, ["Si"], "tersoff_Si_1989.txt",
                       "potential potential.txt\nfix 1\nminimize sd 1.0e-5 500\nensemble nve\ntime_step 0\n"
                       "dump_xyz 1 dump.xyz precision double force\nrun 1\n")
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
        out.append(((d / "dump.xyz").read_bytes(), _progress(r.stdout)))
    assert out[0][0] == out[1][0]
    dump = read_xyz(tmp_path / "0" / "dump.xyz", ["Si"])
    model = read_xyz(tmp_path / "0" / "model.xyz", ["Si"])
    fixed = s["group"] == 1
    assert np.allclose(dump["pos"][:, fixed], model["pos"][:, fixed], rtol=0, atol=1e-12)
    assert not np.allclose(dump["pos"][:, ~fixed], model["pos"][:, ~fixed], rtol=0, atol=1e-6)
    E = _engine()
    atom = E.Atom(model["type"], model["pos"], np.full(n, 28.085))
    box = E.Box(model["h"].copy(), model["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / "tersoff_Si_1989.txt", n)
    label = torch.as_tensor(model["group"].astype(np.int32).reshape(-1), device="cuda")
    lines, _ = E.Minimizer("sd", n, 1e-5, 500).compute(force, box, atom, label, 1)
    assert out[0][1] == lines


def test_driver_fire_ignores_fix(tmp_path):
    """`fix 1` + `minimize fire`: the reference builds its FIRE minimizer with fixed group -1
    (minimize.cu:126), so the atoms of the fixed group relax with the others."""
    s = diamond(4, rattle=0.05, seed=4)
    n = s["type"].shape[0]
    s["group"] = (np.arange(n) % 4 == 0).astype(np.int32)
    r = run_driver(tmp_path, s, ["Si"], "tersoff_Si_1989.txt",
                   "potential potential.txt\nfix 1\nminimize fire 1.0e-4 300\nensemble nve\ntime_step 0\n"
                   "dump_xyz 1 dump.xyz precision double\nrun 1\n")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    dump = read_xyz(tmp_path / "dump.xyz", ["Si"])
    model = read_xyz(tmp_path / "model.xyz", ["Si"])
    fixed = s["group"] == 1
    moved = np.sqrt(((dump["pos"] - model["pos"]) ** 2).sum(axis=0))
    assert (moved[fixed] > 1e-3).mean() > 0.9  # the fixed group relaxes like the rest


MINIMIZE_ERRORS = [
    ("minimize sd 1e-5", "minimize sd should have 2 parameters."),
    ("minimize fire 1e-5", "minimize fire should have 2 to 4 parameters."),
    ("minimize fire 1e-5 10 1 0 0", "minimize fire should have 2 to 4 parameters."),
    ("minimize sd x 10", "Force tolerance should be a number."),
    ("minimize sd 1e-5 ten", "Number of steps should be an integer."),
    ("minimize sd 1e-5 0", "Number of steps should > 0."),
    ("minimize fire 1e-5 10 yes", "Box_change should be an integer."),
    ("minimize fire 1e-5 10 2", "Box_change should be 1 or 0."),
    ("minimize fire 1e-5 10 1 yes", "Hydrostatic_strain should be an integer."),
    ("minimize fire 1e-5 10 1 2", "Hydrostatic_strain should be 1 or 0."),
    ("minimize cg 1e-5 10", "Invalid minimizer."),
]


@pytest.mark.parametrize("line,message", MINIMIZE_ERRORS + [(None, "'potential' must precede 'minimize'.")])
def test_driver_minimize_input_errors(tmp_path, line, message):
    s = fcc(6, 5.26, rattle=0.0)
    run_in = "minimize sd 1e-5 10\n" if line is None else f"potential potential.txt\n{line}\n"
    r = run_driver(tmp_path, s, ["Ar"], "lj_Ar_10A.txt", run_in, timeout=120)
    assert r.returncode == 1 and "Input Error" in r.stderr and message in r.stderr, r.stderr


# ---- the driver against the unmodified reference gpumd (tests/golden/refgpu_min_*) -------------------

def _reference_runs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("run_reference_gpumd",
                                                  GOLDEN.parent.parent / "scripts" / "run_reference_gpumd.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


REF = _reference_runs()


def _numbers(line):
    import re
    return [float(v) for v in re.findall(r"-?\d+\.?\d*(?:e[-+]?\d+)?", line)]


def _lattice_gap(mine, ref, h):
    """Largest distance between the two position sets after wrapping into the box and removing the mean
    displacement."""
    H = np.asarray(h).reshape(3, 3)
    frac = np.linalg.solve(H, mine - ref)
    frac -= np.round(frac)
    d = H @ frac
    d -= d.mean(axis=1, keepdims=True)
    return np.sqrt((d * d).sum(axis=0)).max()


# case: (largest position gap in A, how the progress lines must agree).  Position gaps from tol over the
# softest stiffness, except where the paths are the same to rounding; measured gaps on an H100 in comments.
#   "all": FP64 Tersoff, every line equal to its printed digits up to the last one (rtol 1e-9);
#   "first": the step-0 line, its numbers within the FP32 energy tolerance of the suite (rtol 1e-5; measured
#            at most 6e-7, NEP f_max); the final energy within 1e-6 eV/atom in every case.
# SD with a fixed group ends in a stall (the trial energies differ from the current one at the rounding
# level), where the summation order of sum U decides accept / reject: same final energy, not the same lines.
MIN_REF_TOL = {
    "min_si_sd": (1e-6, "all"),          # measured gap 1.1e-11 A
    "min_si_sd_fix": (1e-6, "first"),    # 6.2e-8 A; lines: 92 vs 103 iterations in the final stall
    "min_si_fire": (1e-6, "all"),        # 1.6e-14 A
    "min_si_fire_fix": (1e-6, "all"),    # 1.6e-14 A; the fixed group relaxes in both
    "min_pbte_fire_box": (1e-4, "first"),        # 3.2e-7 A, box 1.7e-8
    "min_pbte_fire_box_hydro": (1e-4, "first"),  # 1.3e-7 A, box 2.6e-9
    "min_lj_fire": (5e-3, "first"),      # 6.6e-7 A (tol 1e-4 over ~0.02 eV/A^2)
    "min_eam_sd": (5e-3, "first"),       # 1.1e-3 A: both stall (step < 1e-8) at f_max ~ 1e-3 eV/A
    "min_si_dispersion": (1e-9, "first"),  # 1.5e-14 A; f_max is rounding noise (6.2e-10) at the ideal lattice
}


@pytest.mark.parametrize("case", list(REF.MIN_CASES))
def test_driver_matches_the_reference_minimizer(tmp_path, case):
    """`minimize ...` + the single-point tail through b200md and through the unmodified reference gpumd
    (scripts/run_reference_gpumd.py on an H100): final energy, relaxed positions, box and progress lines."""
    from gpumd_b200 import build
    make, symbols, pot, lines, head, model_file = REF.MIN_CASES[case]
    sym = symbols or nep_type_order(GOLDEN / pot)
    if model_file is None:
        write_xyz(tmp_path / "model.xyz", make(), sym)
    else:
        shutil.copyfile(model_file, tmp_path / "model.xyz")
    shutil.copyfile(GOLDEN / pot, tmp_path / "potential.txt")
    (tmp_path / "run.in").write_text(head + "potential potential.txt\n" + lines + REF.MIN_TAIL)
    r = subprocess.run([str(build.build_host())], cwd=tmp_path, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    mine_lines = REF.min_progress(r.stdout)
    ref_lines = (GOLDEN / f"refgpu_{case}_progress.txt").read_text().splitlines()
    mine, ref = read_xyz(tmp_path / "dump.xyz", sym), read_xyz(GOLDEN / f"refgpu_{case}_dump.xyz", sym)
    n = mine["pos"].shape[1]
    de = abs(mine["energy"] - ref["energy"]) / n
    dh = np.abs(mine["h"] - ref["h"]).max() / np.abs(ref["h"]).max()
    gap = _lattice_gap(mine["pos"], ref["pos"], ref["h"])
    print(f"\n{case}: dE/atom {de:.3e} dh {dh:.3e} gap {gap:.3e} lines {len(mine_lines)} / {len(ref_lines)}")
    print("\n".join(f"  mine {a}\n  ref  {b}" for a, b in zip(mine_lines, ref_lines)))
    gap_tol, lines_rule = MIN_REF_TOL[case]
    assert de < 1e-6       # measured: Tersoff 8e-15, LJ 2e-10, NEP 8e-8, EAM 1.3e-7 eV/atom
    assert dh < 1e-5       # measured: NEP box change 1.7e-8 (the other cases keep the box)
    assert gap < gap_tol
    a, b = _numbers(mine_lines[0]), _numbers(ref_lines[0])
    assert a[0] == b[0] and np.allclose(a, b, rtol=1e-5, atol=1e-8), (mine_lines[0], ref_lines[0])
    if lines_rule == "all":
        assert len(mine_lines) == len(ref_lines)
        for a, b in zip(mine_lines, ref_lines):
            assert np.allclose(_numbers(a), _numbers(b), rtol=1e-9, atol=1e-9), (a, b)

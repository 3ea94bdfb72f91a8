"""The numpy restatement of the minimizers (tests/minimize_oracle.py) on the oracle's LJ forces: SD and
FIRE relax a rattled fcc argon crystal back to its lattice, FIRE with box change finds the lattice constant
of the truncated lattice sum, and the reference's quirks are pinned one by one."""
import numpy as np
import pytest
from scipy.optimize import minimize_scalar

import minimize_oracle as M
from cases_classical import lj_table
from conftest import GOLDEN
from gpumd_b200.structures import fcc

LJ = GOLDEN / "lj_Ar_10A.txt"


def lattice_energy(a, eps, sig, rc):
    """Energy per atom of the fcc lattice a under the plain LJ potential cut at rc (no shift)."""
    k = int(np.ceil(2 * rc / a)) + 1
    g = np.stack(np.meshgrid(*[np.arange(-k, k + 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    g = g[(g.sum(axis=1) % 2 == 0) & (np.abs(g).sum(axis=1) > 0)]  # fcc sites (a/2)(i,j,k), i+j+k even
    r = np.sqrt((g * g).sum(axis=1)) * a / 2
    r = r[r < rc]
    return 0.5 * np.sum(4 * eps * ((sig / r) ** 12 - (sig / r) ** 6))


@pytest.fixture(scope="module")
def lj(oracle):
    para = lj_table(LJ)
    eps, sig, rc = para[0, 0]
    a0 = minimize_scalar(lambda a: lattice_energy(a, eps, sig, rc), bounds=(5.05, 5.34), method="bounded",
                         options=dict(xatol=1e-9)).x

    def forces(s):
        def compute(x, h=None):
            h = s["h"] if h is None else h
            xw = oracle.apply_pbc(h, s["pbc"], np.asarray(x).reshape(3, -1))
            r = oracle.lj_compute(para, s["type"], h, s["pbc"], xw)
            return xw, r["force"].astype(np.float64), r["pe"], r["virial"]
        return compute
    return dict(a0=a0, forces=forces)


def lattice_gap(x, s0, h):
    """Largest distance of an atom from its ideal site after removing the mean displacement."""
    H = np.asarray(h).reshape(3, 3)
    d = x - s0["ideal"]
    frac = np.linalg.solve(H, d)
    frac -= np.round(frac)
    d = H @ frac
    d -= d.mean(axis=1, keepdims=True)
    return np.sqrt((d * d).sum(axis=0)).max()


def rattled(a, rattle=0.1):
    s = fcc(4, a, rattle=rattle, seed=3)
    s["ideal"] = fcc(4, a)["pos"]
    return s


def test_sd_relaxes_rattled_fcc_to_its_lattice(lj):
    s = rattled(lj["a0"])
    compute = lj["forces"](s)
    x, lines = M.run_sd(lambda x: compute(x)[:3], s["pos"], 1e-4, 5000)
    assert lines[-1].startswith("    step ") and "f_max = " in lines[-1] and "total_potential" not in lines[-1]
    assert lattice_gap(x, s, s["h"]) < 50 * 1e-4  # tol over the softest stiffness of Ar (~0.02 eV/A^2); measured: 2.8e-3 A


def test_fire_relaxes_rattled_fcc_to_its_lattice(lj):
    s = rattled(lj["a0"])
    x, h, lines = M.run_fire(lj["forces"](s), s["pos"], s["h"], 1e-4, 3000)
    f_max = float(lines[-1].split("f_max = ")[1].split()[0])
    assert f_max < 1e-4
    assert lattice_gap(x, s, s["h"]) < 50 * 1e-4  # measured: 1.7e-3 A


@pytest.mark.parametrize("hydrostatic", [False, True])
def test_fire_box_change_finds_the_lattice_constant(lj, hydrostatic):
    a_start = lj["a0"] * 0.98  # stay between the shells at a/sqrt(2) * sqrt(8) and sqrt(7) = 10 A
    s = rattled(a_start, rattle=0.02)
    x, h, lines = M.run_fire(lj["forces"](s), s["pos"], s["h"], 1e-4, 5000, box_change=True,
                             hydrostatic=hydrostatic)
    assert lines[-1].startswith("  Converged!")
    H = h.reshape(3, 3)
    a = np.diag(H) / 4
    assert np.allclose(a, lj["a0"], rtol=1e-4), (a, lj["a0"])  # measured: 8e-7 relative
    if hydrostatic:  # only the diagonal moves, by one factor
        assert np.count_nonzero(H - np.diag(np.diag(H))) == 0
        assert np.ptp(np.diag(H)) < 1e-12 * H[0, 0]


def test_first_fire_iteration_halves_dt_and_the_move_back_uses_the_new_dt():
    rng = np.random.default_rng(0)
    n = 8
    x, F, U, W = rng.normal(size=(3, n)), rng.normal(size=(3, n)), rng.normal(size=n), np.zeros((9, n))
    st = M.fire_state()
    x1, v1, _, st1, rec = M.fire_step(x, np.zeros((3, n)), F, U, W, np.eye(3).reshape(9), st, 1e-6)
    assert rec["P"] == 0 and rec["uphill"] and st1["dt"] == M.DT_0 * 0.5 and st1["n_neg"] == 0
    # uphill with a moving state: x first moves back by -0.5 dt_new v, then the MD step from v = 0
    v = rng.normal(size=(3, n))
    F = -v
    st = dict(M.fire_state(), dt=4 * M.DT_0, n_neg=7)
    x2, v2, _, st2, rec = M.fire_step(x, v, F, U, W, np.eye(3).reshape(9), st, 1e-6)
    dt = 2 * M.DT_0
    assert st2["dt"] == dt and st2["alpha"] == M.ALPHA_START and st2["n_neg"] == 0 and rec["v_mod"] == 0
    vk = (np.zeros_like(v) + F * (dt / M.MASS)) * (1 - M.ALPHA_START)
    assert np.array_equal(v2, vk)
    assert np.array_equal(x2, (x + v * (-0.5 * dt)) + vk * dt)


@pytest.mark.parametrize("box_change", [False, True])
def test_dt_left_unchanged_fixed_box_clamped_box_change(box_change):
    rng = np.random.default_rng(1)
    n = 4
    x, U = rng.normal(size=(3, n)), np.zeros(n)
    W = np.zeros((9, n))
    h = (np.eye(3) * 10).reshape(9)
    v = rng.normal(size=(3, n))
    # downhill, N_neg > N_min, dt near dt_max: fixed box keeps dt, box change clamps it to dt_max
    st = dict(M.fire_state(L=10.0), dt=0.95 * M.DT_MAX, n_neg=M.N_MIN + 1)
    _, _, _, s1, rec = M.fire_step(x, v, v, U, W, h, st, 1e-9, box_change)
    assert not rec["uphill"] and s1["alpha"] == M.ALPHA_START * M.F_ALPHA
    assert s1["dt"] == (M.DT_MAX if box_change else 0.95 * M.DT_MAX)
    # at N_neg == N_min dt and alpha stay; N_neg still counts up
    st = dict(st, n_neg=M.N_MIN)
    _, _, _, s1, _ = M.fire_step(x, v, v, U, W, h, st, 1e-9, box_change)
    assert s1["dt"] == st["dt"] and s1["alpha"] == M.ALPHA_START and s1["n_neg"] == M.N_MIN + 1
    # uphill near dt_min: fixed box keeps dt, box change clamps it to dt_min
    st = dict(M.fire_state(L=10.0), dt=1.5 * M.DT_MIN)
    _, _, _, s1, rec = M.fire_step(x, v, -v, U, W, h, st, 1e-9, box_change)
    assert rec["uphill"] and s1["dt"] == (M.DT_MIN if box_change else 1.5 * M.DT_MIN)


def test_box_change_has_no_move_back_and_no_mixing_below_the_force_guard():
    n = 2
    x = np.ones((3, n))
    v = np.full((3, n), 0.3)
    F = np.full((3, n), -1e-14)  # uphill, |F| < 1e-12 with the zero virial
    h = (np.eye(3) * 10).reshape(9)
    st = dict(M.fire_state(L=10.0), alpha=0.1)
    x1, v1, h1, _, rec = M.fire_step(x, v, F, np.zeros(n), np.zeros((9, n)), h, st, 1e-20, True)
    dt = 0.5 * M.DT_0
    assert rec["uphill"] and rec["scale"] == 0.0
    assert np.array_equal(v1, (F * (dt / M.MASS)) * (1 - M.ALPHA_START))
    assert np.array_equal(x1, x + v1 * dt)  # no -0.5 dt v; zero strain
    assert np.array_equal(h1, h)


def test_sd_uphill_rejection_and_the_minimum_step_stop():
    uphill, step, u = M.sd_decide(np.array([1.0]), np.array([2.0]), 0.1)
    assert uphill and step == 0.1 * 0.2 and u == 1.0
    uphill, step, u = M.sd_decide(np.array([1.0]), np.array([0.5]), 0.1)
    assert not uphill and step == 0.1 * 1.2 and u == 0.5
    # a force that points uphill everywhere: every trial is rejected until the step falls below 1e-8
    calls = []

    def compute(x):
        calls.append(1)
        return x, np.ones_like(x), np.full(x.shape[1], np.sum(x))
    x0 = np.zeros((3, 4))
    x, lines = M.run_sd(compute, x0, 1e-12, 100)
    assert np.array_equal(x, x0)
    k = int(np.ceil(np.log(1e-8 / 0.1) / np.log(0.2)))  # rejections until 0.1 * 0.2^k < 1e-8
    assert len(calls) == 1 + k
    assert lines[-1] == "    Position step is 0, SD minimizer can't find a better solution"
    assert lines[-2].startswith("    step %d: total_potential" % k)


def test_sd_leaves_fixed_atoms_bit_for_bit(lj):
    s = rattled(lj["a0"])
    label = (np.arange(s["type"].shape[0]) % 3 == 0).astype(np.int32)
    compute = lj["forces"](s)
    x0 = compute(s["pos"])[0]
    # positions passed through unwrapped (the LJ oracle takes minimum images): the oracle's own wrap goes
    # through fractional coordinates and would touch the last bits
    x, _ = M.run_sd(lambda x: (x,) + compute(x)[1:3], x0, 1e-3, 200, label=label, fixed_group=1)
    assert np.array_equal(x[:, label == 1], x0[:, label == 1])
    assert not np.array_equal(x[:, label == 0], x0[:, label == 0])

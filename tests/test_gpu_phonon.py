"""Phonons on the device (b2_phonon.cu): the force constants against the same basis-displacement scheme
restated with the same device forces, D(k) against the numpy restatement (tests/phonon_oracle.py), the Jacobi
eigensolver on random matrices, and the `compute_phonon` keyword of the driver against the reference's own
silicon_dispersion output."""
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

import phonon_oracle as P
from conftest import GOLDEN
from gpumd_b200.structures import diamond, fcc, read_xyz, rocksalt_pbte, write_xyz

pytestmark = pytest.mark.gpu


def _engine():
    from gpumd_b200 import engine
    return engine


# (structure, replicate factors of its conventional cell, potential file)
CASES = {
    "nep": (lambda: rocksalt_pbte(3, rattle=0.0), (3, 3, 3), "nep_PbTe.txt"),
    "lj": (lambda: fcc(6, 5.26), (6, 6, 6), "lj_Ar_10A.txt"),
    "tersoff": (lambda: diamond(3), (3, 3, 3), "tersoff_Si_1989.txt"),
    "eam": (lambda: fcc(6, 3.615, symbols=("Cu",)), (6, 6, 6), "eam_Cu_Zhou_2004.txt"),
}
def _triclinic_si():
    """The reference's silicon_dispersion cell (triclinic, 2 atoms) x 4^3, in the driver's replicate order."""
    s = read_xyz(GOLDEN / "silicon_dispersion_model.xyz", ["Si"])
    h = np.asarray(s["h"]).reshape(3, 3)
    pos = [s["pos"] + (h @ np.array([i, j, k], float))[:, None] for i in range(4) for j in range(4) for k in range(4)]
    return dict(pos=np.concatenate(pos, axis=1), type=np.zeros(128, np.int32), mass=np.full(128, 28.085),
                h=(h * 4).reshape(9), pbc=np.array([1, 1, 1]))


CASES["tersoff_triclinic"] = (_triclinic_si, (4, 4, 4), "tersoff_Si_1989.txt")
SEGS = [[[0, 0, 0], [0.5, 0, 0.5]], [[0.5, 0.5, 0.5], [0, 0, 0]]]


def _setup(case):
    E = _engine()
    make, cxyz, pot = CASES[case]
    s = make()
    n = s["type"].shape[0]
    atom = E.Atom(s["type"], s["pos"], s["mass"])
    box = E.Box(s["h"], s["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / pot, n)
    return s, atom, box, force, cxyz


def _restated_H(case, d, nb, mask):
    """The sweep's force calls made one by one from Python on a fresh handle: same positions, same order."""
    s, atom, box, force, _ = _setup(case)
    n = s["type"].shape[0]
    x0 = atom.position_per_atom.clone()
    pos = atom.position_per_atom
    H = np.zeros((nb, n, 9))
    for n1 in range(nb):
        for a in range(3):
            f = []
            for sgn in (-d, d):
                k = a * n + n1
                for c in range(3):  # the wrap of the previous call may have moved any coordinate
                    pos[c * n + n1] = x0[c * n + n1]
                pos[k] = x0[k] + sgn
                force.compute(box, pos, atom.type, atom.potential_per_atom, atom.force_per_atom,
                              atom.virial_per_atom)
                f.append(atom.force_per_atom.cpu().numpy().reshape(3, n).copy())
            for c in range(3):
                pos[c * n + n1] = x0[c * n + n1]
            H[n1, :, 3 * a:3 * a + 3] = ((f[0] - f[1]) / (2 * d)).T
    return H * mask[:, :, None]


@pytest.mark.parametrize("case", list(CASES))
def test_force_constants_and_D_match_the_restatement(case):
    E = _engine()
    s, atom, box, force, cxyz = _setup(case)
    x_before = atom.position_per_atom.clone()
    d = 0.005
    out = E.Phonon(d).compute(force, box, atom, cxyz, SEGS)
    assert torch.equal(atom.position_per_atom, x_before)  # bit for bit
    nb = out["num_basis"]
    x = x_before.cpu().numpy().reshape(3, -1)
    r12, mask = P.geometry(x, s["h"], s["pbc"], nb, out["cutoff"])
    H = _restated_H(case, d, nb, mask)
    assert np.array_equal(out["H"], H), np.abs(out["H"] - H).max()
    mass = s["mass"][:nb]
    D = P.dynamical(out["H"], r12, mask, mass, out["kpoints"])
    err = np.abs(out["D"] - D).max() / np.abs(D).max()
    print(f"\n{case}: nb {nb} D rel err {err:.2e} max omega2 {out['omega2'].max():.4g}")
    assert err <= 1e-14
    w = np.linalg.eigvalsh(D) * P.NATURAL_TO_THZ2
    assert np.abs(out["omega2"] - w).max() <= 1e-11 * np.abs(w).max()
    # run to run: a second calculation from the same state gives the same bits
    _, atom2, box2, force2, _ = _setup(case)
    out2 = E.Phonon(d).compute(force2, box2, atom2, cxyz, SEGS)
    for key in ("H", "D", "omega2"):
        assert np.array_equal(out[key], out2[key]), key


def test_one_kernel_launch_between_force_calls():
    E = _engine()
    s, atom, box, force, cxyz = _setup("tersoff")
    before, after = [], []

    class Counting:
        potentials = force.potentials

        def compute(self, *args):
            before.append(E.launch_count())
            force.compute(*args)

    E.Phonon(0.005).compute(Counting(), box, atom, cxyz, SEGS, sweep_hook=lambda c: after.append(E.launch_count()))
    assert len(before) == 6 * 8
    assert all(b - a == 1 for a, b in zip(after[:-1], before[1:]))


def _random_hermitian(rng, dim, kind):
    if kind == "degenerate":
        Q, _ = np.linalg.qr(rng.normal(size=(dim, dim)) + 1j * rng.normal(size=(dim, dim)))
        lam = np.repeat(np.arange((dim + 2) // 3), 3)[:dim].astype(float) - 2.0
        return Q @ np.diag(lam) @ Q.conj().T
    X = rng.normal(size=(dim, dim)) + 1j * rng.normal(size=(dim, dim))
    return X + X.conj().T


@pytest.mark.parametrize("dim", [3, 4, 17, 48, 95, 96])
@pytest.mark.parametrize("kind", ["random", "degenerate"])
def test_jacobi_eigensolver(dim, kind):
    E = _engine()
    rng = np.random.default_rng(dim)
    A = np.stack([_random_hermitian(rng, dim, kind) for _ in range(3)])
    # only the lower triangle is read: garbage above it
    junk = np.triu(rng.normal(size=(dim, dim)), 1) * 1e3
    w = E.jacobi_eig(np.tril(A.real) + junk, np.tril(A.imag) + junk)
    for Ak, wk in zip(A, w):
        ref = np.linalg.eigvalsh(Ak, UPLO="L")
        assert np.abs(wk - ref).max() <= 1e-12 * np.linalg.norm(Ak)
    S = np.stack([(a.real + a.real.T) / 2 for a in A])
    w, V = E.jacobi_eig(np.tril(S) + junk, vectors=True)
    for Sk, wk, Vk in zip(S, w, V):
        nrm = np.linalg.norm(Sk)
        assert np.abs(wk - np.linalg.eigvalsh(Sk)).max() <= 1e-12 * nrm
        assert np.all(np.diff(wk) >= 0)
        assert np.abs(Sk @ Vk - Vk * wk).max() <= 1e-13 * nrm * dim
        assert np.abs(Vk.T @ Vk - np.eye(dim)).max() <= 1e-13 * dim


# ---- the `compute_phonon` keyword of the driver ---------------------------------------------------------

def _run(tmp_path, model, symbols, pot, run_in, kpoints, timeout=900):
    from gpumd_b200 import build
    if isinstance(model, dict):
        write_xyz(tmp_path / "model.xyz", model, symbols)
    else:
        shutil.copyfile(model, tmp_path / "model.xyz")
    shutil.copyfile(GOLDEN / pot, tmp_path / "potential.txt")
    (tmp_path / "run.in").write_text(run_in)
    if kpoints is not None:
        (tmp_path / "kpoints.in").write_text(kpoints)
    return subprocess.run([str(build.build_host())], cwd=tmp_path, capture_output=True, text=True,
                          timeout=timeout)


def _omega2(path):
    lines = path.read_text().splitlines()
    return lines[0], [ln.split()[0] for ln in lines[1:]], np.array([[float(v) for v in ln.split()[1:]]
                                                                    for ln in lines[1:]])


SI_RUN = "replicate 6 6 6\npotential potential.txt\nminimize sd 1.0e-6 10000\ncompute_phonon 0.005\n"
# |omega2 - reference| over the largest omega2 of the reference's silicon_dispersion output; measured 9.8e-6 on
# an H100 (the O(d^2) difference between the two finite-difference schemes)
SI_REF_TOL = 3e-5


def test_driver_silicon_dispersion_matches_the_reference_output(tmp_path):
    r = _run(tmp_path, GOLDEN / "silicon_dispersion_model.xyz", None, "tersoff_Si_1989.txt", SI_RUN,
             (GOLDEN / "ref_silicon_dispersion_kpoints.in").read_text())
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert "Using cutoff for phonon calculations: 6 A." in r.stdout
    assert "Replicate in x >= " in r.stdout
    head, col, w = _omega2(tmp_path / "omega2.out")
    rhead, rcol, rw = _omega2(GOLDEN / "ref_silicon_dispersion_omega21.out")
    assert head == rhead and col == rcol
    err = np.abs(w - rw).max() / np.abs(rw).max()
    print(f"\nsilicon_dispersion: max |omega2 - ref| / max omega2 = {err:.3e}")
    assert err < SI_REF_TOL
    D = (tmp_path / "D.out").read_text().splitlines()
    assert len(D) == 401 * 6 and all(len(ln.split()) == 12 for ln in D)


def _reference_runs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("run_reference_gpumd",
                                                  GOLDEN.parent.parent / "scripts" / "run_reference_gpumd.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


REF = _reference_runs()
# case: (largest |omega2 - reference| over the largest reference omega2, the same for D over the largest |D|).
# Fixed from the first H100 run; measured values in the comments.  The difference is the O(d^2) difference of
# the two finite-difference schemes (FP64 Tersoff, LJ and EAM) and FP32 force rounding (NEP).
PHONON_REF_TOL = {
    "phonon_si_dispersion": (3e-5, 6e-5),   # 9.8e-6, D 2.0e-5
    "phonon_sic": (5e-5, None),             # 1.5e-5
    "phonon_pbte": (1e-2, 1e-2),            # 2.8e-3, D 3.8e-3 (FP32 NEP forces over 2d = 0.01 A)
    "phonon_lj": (5e-4, 5e-4),              # 1.1e-4, D 1.6e-4 (FP32 pair math)
    "phonon_eam": (1e-3, 2e-3),             # 2.8e-4, D 7.2e-4 (FP32 pair math)
    "phonon_si16": (1e-11, None),           # 1.5e-13
    "phonon_gamma": (1e-6, None),           # 5.3e-13 (float32 output); projectors 2.7e-8
}

def _read_d(path, dim):
    """D.out -> complex [nk, dim, dim] (row, col): each line is one row, real parts then imaginary parts."""
    v = np.loadtxt(path).reshape(-1, dim, 2 * dim)
    return v[:, :, :dim] + 1j * v[:, :, dim:]


def _eigenvector_out(path, dim):
    """eigenvector.out -> (omega2 [dim], V [dim, dim] with the eigenvectors as columns, row = a + 3 b)."""
    vals = np.fromfile(path, dtype=np.float32).astype(np.float64)
    assert vals.shape == (dim + dim * dim,)
    nb = dim // 3
    vec = vals[dim:].reshape(dim, 3, nb)  # [col][a][b]
    return vals[:dim], vec.transpose(0, 2, 1).reshape(dim, dim).T


@pytest.mark.parametrize("case", list(REF.PHONON_CASES))
def test_driver_matches_the_reference_phonons(tmp_path, case):
    """The same input through b200md and through the unmodified reference gpumd
    (scripts/run_reference_gpumd.py on an H100, tests/golden/refgpu_phonon_*)."""
    make, symbols, pot, head, lines, model_file, kpoints, keep_d = REF.PHONON_CASES[case]
    from gpumd_b200.structures import nep_type_order
    sym = symbols or nep_type_order(GOLDEN / pot)
    r = _run(tmp_path, model_file if make is None else make(), sym, pot, head + "potential potential.txt\n" + lines,
             kpoints)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    w_tol, d_tol = PHONON_REF_TOL[case]
    if case == "phonon_gamma":
        dim = 24
        w, V = _eigenvector_out(tmp_path / "eigenvector.out", dim)
        rw, rV = _eigenvector_out(GOLDEN / f"refgpu_{case}_eigenvector.out", dim)
        err = np.abs(w - rw).max() / np.abs(rw).max()
        # projectors onto groups of equal eigenvalues (the acoustic triplet, the degenerate optical sets)
        groups = np.split(np.arange(dim), np.nonzero(np.diff(rw) > 1e-3 * np.abs(rw).max())[0] + 1)
        perr = max(np.abs(V[:, g] @ V[:, g].T - rV[:, g] @ rV[:, g].T).max() for g in groups)
        print(f"\n{case}: omega2 {err:.3e} projectors {perr:.3e} groups {[len(g) for g in groups]}")
        assert err < w_tol
        assert perr < 1e-6  # float32 output
        return
    head_m, col, w = _omega2(tmp_path / "omega2.out")
    rhead, rcol, rw = _omega2(GOLDEN / f"refgpu_{case}_omega2.out")
    assert head_m == rhead and col == rcol
    err = np.abs(w - rw).max() / np.abs(rw).max()
    msg = f"\n{case}: omega2 {err:.3e}"
    if keep_d:
        dim = w.shape[1]
        D, rD = _read_d(tmp_path / "D.out", dim), _read_d(GOLDEN / f"refgpu_{case}_D.out", dim)
        derr = np.abs(D - rD).max() / np.abs(rD).max()
        msg += f" D {derr:.3e}"
    print(msg)
    assert err < w_tol
    if keep_d:
        assert derr < d_tol


def test_driver_gamma_only_writes_eigenvectors(tmp_path):
    E = _engine()
    s = diamond(1)
    run_in = "replicate 2 2 2\npotential potential.txt\ncompute_phonon 0.005\n"
    r = _run(tmp_path, s, ["Si"], "tersoff_Si_1989.txt", run_in, "0 0 0 G\n")
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    assert not (tmp_path / "omega2.out").exists() and not (tmp_path / "D.out").exists()
    raw = (tmp_path / "eigenvector.out").read_bytes()
    dim = 24
    vals = np.array(struct.unpack(f"{dim + dim * dim}f", raw))
    w, vec = vals[:dim], vals[dim:].reshape(dim, 3, 8)          # [col][a][b]
    V = vec.transpose(0, 2, 1).reshape(dim, dim).T                # row = a + 3 b
    # the same calculation through the engine
    big = diamond(2)
    atom = E.Atom(big["type"], _replicate_order(s, (2, 2, 2)), big["mass"])
    box = E.Box(np.asarray(s["h"]) * 2, s["pbc"])
    force = E.Force()
    force.parse_potential(GOLDEN / "tersoff_Si_1989.txt", atom.number_of_atoms)
    out = E.Phonon(0.005).compute(force, box, atom, (2, 2, 2), [[[0, 0, 0]]])
    assert np.allclose(w, out["omega2"][0], rtol=1e-6, atol=1e-4 * np.abs(w).max())
    D = out["D"][0].real
    assert np.abs(D @ V - V * (w / P.NATURAL_TO_THZ2)).max() < 1e-5 * np.abs(D).max()
    # eigenvectors through the projectors onto groups of equal eigenvalues
    wr, Vr = np.linalg.eigh(D)
    groups = np.split(np.arange(dim), np.nonzero(np.diff(wr) > 1e-6 * np.abs(wr).max())[0] + 1)
    for g in groups:
        assert np.abs(V[:, g] @ V[:, g].T - Vr[:, g] @ Vr[:, g].T).max() < 1e-5


def _replicate_order(s, r):
    """Positions in the order of the driver's `replicate`: copies a-slowest, c-fastest, atoms innermost."""
    h = np.asarray(s["h"]).reshape(3, 3)
    out = []
    for i in range(r[0]):
        for j in range(r[1]):
            for k in range(r[2]):
                out.append(s["pos"] + (h @ np.array([i, j, k], dtype=float))[:, None])
    return np.concatenate(out, axis=1)


def test_driver_uses_the_relaxed_positions_and_box(tmp_path):
    """minimize with box change, then compute_phonon, gives what compute_phonon gives on the relaxed cell
    written back with full precision."""
    s = diamond(1, a=5.50)
    kp = "0 0 0 G\n0.5 0 0.5 X\n"
    head = "replicate 3 3 3\npotential potential.txt\nminimize fire 1e-6 3000 1\n"
    a = tmp_path / "a"
    a.mkdir()
    r = _run(a, s, ["Si"], "tersoff_Si_1989.txt", head + "compute_phonon 0.005\n", kp)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    b = tmp_path / "b"
    b.mkdir()
    tail = "velocity 1\nensemble nve\ntime_step 0\ndump_xyz 1 dump.xyz precision double\nrun 1\n"
    r = _run(b, s, ["Si"], "tersoff_Si_1989.txt", head + tail, None)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    relaxed = read_xyz(b / "dump.xyz", ["Si"])
    c = tmp_path / "c"
    c.mkdir()
    shutil.copyfile(b / "dump.xyz", c / "relaxed.xyz")
    # the relaxed supercell is the model; replicate 1 1 1 would make every atom a basis atom, so the
    # factors come from a replicate line of the same cell: the first 8 atoms and a third of the box
    prim = dict(type=np.zeros(8, np.int32), pos=relaxed["pos"][:, :8], h=np.asarray(relaxed["h"]) / 3,
                pbc=relaxed["pbc"])
    r = _run(c, prim, ["Si"], "tersoff_Si_1989.txt", "replicate 3 3 3\npotential potential.txt\n"
             "compute_phonon 0.005\n", kp)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    ha, ca, wa = _omega2(a / "omega2.out")
    hc, cc, wc = _omega2(c / "omega2.out")
    assert abs(np.asarray(relaxed["h"]).reshape(9)[0] - 3 * 5.50) > 0.1  # the box did relax
    assert ha == hc and ca == cc
    err = np.abs(wa - wc).max() / np.abs(wc).max()
    print(f"\nrelaxed vs written back: {err:.3e}")
    assert err < 1e-12


def test_driver_takes_the_product_of_every_replicate_line(tmp_path):
    """`replicate` wherever it stands, and two lines whose product sets num_basis, give the dispersion of one
    `replicate 2 2 2` on the first line (the same atoms in another order: equal within rounding)."""
    s = diamond(1)
    kp = "0 0 0 G\n0.5 0 0.5 X\n"
    out = {}
    for name, head in (("one", "replicate 2 2 2\n"), ("late", "time_step 1\nreplicate 2 2 2\n"),
                       ("two", "time_step 1\nreplicate 2 1 1\nreplicate 1 2 2\n")):
        d = tmp_path / name
        d.mkdir()
        r = _run(d, s, ["Si"], "tersoff_Si_1989.txt", head + "potential potential.txt\ncompute_phonon 0.005\n", kp)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
        out[name] = _omega2(d / "omega2.out")
    h, c, w = out["one"]
    assert w.shape == (101, 24)
    for name in ("late", "two"):
        assert out[name][0] == h and out[name][1] == c
        assert np.abs(out[name][2] - w).max() < 1e-9 * np.abs(w).max(), name


PHONON_ERRORS = [
    ("compute_phonon", "compute_phonon should have 2 parameters."),
    ("compute_phonon 0.01 2", "compute_phonon should have 2 parameters."),
    ("compute_phonon abc", "displacement for compute_phonon should be a number."),
    ("compute_phonon -0.01", "displacement for compute_phonon should be positive."),
]


@pytest.mark.parametrize("line,message", PHONON_ERRORS)
def test_driver_compute_phonon_parameter_errors(tmp_path, line, message):
    r = _run(tmp_path, diamond(1), ["Si"], "tersoff_Si_1989.txt",
             f"replicate 2 2 2\npotential potential.txt\n{line}\n", "0 0 0 G\n", timeout=120)
    assert r.returncode == 1 and message in r.stderr, r.stderr


@pytest.mark.parametrize("run_in,kpoints,message", [
    ("replicate 2 2 2\ncompute_phonon 0.005\n", "0 0 0 G\n", "'potential' must precede 'compute_phonon'."),
    ("potential potential.txt\ncompute_phonon 0.005\n", "0 0 0 G\n", "replicate keyword not found in run.in file."),
    ("replicate 2 2 2\npotential potential.txt\ncompute_phonon 0.005\n", None, "Cannot open kpoints.in file."),
    ("replicate 2 2 2\npotential potential.txt\ncompute_phonon 0.005\n", "0 0 0\n",
     "kpoints.in file at least 4 parameters for each line."),
])
def test_driver_compute_phonon_input_errors(tmp_path, run_in, kpoints, message):
    r = _run(tmp_path, diamond(1), ["Si"], "tersoff_Si_1989.txt", run_in, kpoints, timeout=120)
    assert r.returncode == 1 and message in r.stderr, r.stderr


def test_driver_refuses_more_than_32_basis_atoms(tmp_path):
    s = diamond((3, 2, 1))  # 48 atoms
    r = _run(tmp_path, s, ["Si"], "tersoff_Si_1989.txt",
             "replicate 1 1 2\npotential potential.txt\ncompute_phonon 0.005\n", "0 0 0 G\n", timeout=120)
    assert r.returncode == 1 and "at most 32 basis atoms" in r.stderr, r.stderr

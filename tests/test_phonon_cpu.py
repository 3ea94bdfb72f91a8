"""The numpy restatement of the phonon calculation (tests/phonon_oracle.py): the k-path and header of the
reference's silicon_dispersion output, kpoints.in parsing, the basis-displacement force constants of LJ argon
against an analytic lattice sum, and the two finite-difference schemes on Tersoff silicon."""
import numpy as np
import pytest

import phonon_oracle as P
from cases_classical import lj_table
from conftest import GOLDEN
from gpumd_b200.structures import diamond, read_xyz

SI_KPOINTS = (GOLDEN / "ref_silicon_dispersion_kpoints.in").read_text()


def test_silicon_dispersion_kpath_and_header_match_the_reference_output():
    s = read_xyz(GOLDEN / "silicon_dispersion_model.xyz")
    h = np.asarray(s["h"]) * 6  # replicate 6 6 6
    segs, names = P.parse_kpoints(SI_KPOINTS)
    assert names == ["G X K G L"] and len(segs[0]) == 5
    k, path, sym = P.kpath(segs, h, (6, 6, 6))
    ref = (GOLDEN / "ref_silicon_dispersion_omega21.out").read_text().splitlines()
    assert P.header(sym, names) == ref[0]
    col = [ln.split()[0] for ln in ref[1:]]
    assert len(col) == len(path) == 401
    assert ["%.6f" % p for p in path] == col


def test_two_segments_join_names_with_a_bar_and_skip_the_jump():
    text = "# comment\n0 0 0 G\n0.5 0 0.5 X\n\n  \n0.5 0.5 0.5 L\n0 0 0 G\n"
    segs, names = P.parse_kpoints(text)
    assert names == ["G X", "L G"]
    h = np.diag([5.0, 5.0, 5.0])
    k, path, sym = P.kpath(segs, h, (1, 1, 1))
    assert len(path) == 201 and len(sym) == 3
    # the second segment starts at L, without the X -> L jump
    leg1 = np.linalg.norm(k[100] - k[0])
    leg2 = np.linalg.norm(k[200] - P.kpath([[segs[1][0]]], h, (1, 1, 1))[0][0])
    assert np.isclose(sym[1], leg1) and np.isclose(sym[2], leg1 + leg2)
    assert P.header(sym, names).endswith(" G X|L G")


def test_single_point_gives_one_kpoint_and_short_lines_are_refused():
    segs, names = P.parse_kpoints("0 0 0 G\n")
    k, path, sym = P.kpath(segs, np.eye(3) * 4, (1, 1, 1))
    assert k.shape == (1, 3) and path.tolist() == [0.0]
    with pytest.raises(ValueError, match="at least 4 parameters"):
        P.parse_kpoints("0 0 0\n")


def _fcc_primitive(a, c):
    """The one-atom fcc cell replicated c x c x c (atom n = cell n, positions from the lattice vectors)."""
    A = 0.5 * a * np.array([[0, 1, 1], [1, 0, 1], [1, 1, 0]], dtype=float).T   # columns a1 a2 a3
    idx = np.stack(np.meshgrid(*[np.arange(c)] * 3, indexing="ij"), -1).reshape(-1, 3)
    return (A @ idx.T), (A * c).reshape(9), A


def _lj_analytic_D(k, A, eps, sig, rc, mass, c):
    """D(k) = (1/m) sum_{R != 0, |R| < rc} k_ab(R) (1 - cos k.R), k_ab the pair stiffness of the plain
    truncated LJ potential."""
    m = int(np.ceil(rc / 3.0)) + 2
    g = np.stack(np.meshgrid(*[np.arange(-m, m + 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    R = (A @ g.T).T
    r = np.linalg.norm(R, axis=1)
    keep = (r > 0) & (r < rc)
    R, r = R[keep], r[keep]
    d1 = 4 * eps * (-12 * sig**12 / r**13 + 6 * sig**6 / r**7)
    d2 = 4 * eps * (156 * sig**12 / r**14 - 42 * sig**6 / r**8)
    u = R / r[:, None]
    K = (d2 - d1 / r)[:, None, None] * u[:, :, None] * u[:, None, :] + (d1 / r)[:, None, None] * np.eye(3)
    return np.einsum("rab,r->ab", K, 1 - np.cos(R @ k)) / mass


def test_lj_basis_displacement_matches_the_analytic_lattice_sum(oracle):
    para = lj_table(GOLDEN / "lj_Ar_10A.txt")
    eps, sig, rc = para[0, 0]
    a, c, mass, d = 5.26, 7, 39.948, 0.005
    x, h, A = _fcc_primitive(a, c)
    n = x.shape[1]
    pbc = np.array([1, 1, 1])
    typ = np.zeros(n, np.int32)

    def forces(y):
        return oracle.lj_compute(para, typ, h, pbc, oracle.apply_pbc(h, pbc, y))["force"].astype(np.float64)

    r12, mask = P.geometry(x, h, pbc, 1, 2 * rc)
    H = P.h_basis(forces, x, 1, d, mask)
    segs = [[[0, 0, 0], [0.5, 0, 0.5], [0.375, 0.375, 0.75], [0, 0, 0], [0.5, 0.5, 0.5]]]
    kpts, _, _ = P.kpath(segs, h, (c, c, c))
    # commensurate with the 7 x 7 x 7 cell: the phases of the images agree
    G = 2 * np.pi * np.linalg.inv(A).T
    kc = [G @ (np.array(f) / c) for f in ([0, 0, 0], [1, 0, 0], [2, 1, 0], [3, 3, 3], [1, 2, 3])]
    Dm = P.dynamical(H, r12, mask, [mass], np.array(kc))
    Da = [_lj_analytic_D(k, A, eps, sig, rc, mass, c) for k in kc]
    scale = max(np.abs(D).max() for D in Da)
    for D, ref, k in zip(Dm, Da, kc):
        assert np.abs(D.imag).max() < 1e-4 * scale  # the oracle LJ forces are FP32 sums
        assert np.abs(D.real - ref).max() < 1e-4 * scale, (k, D.real, ref)
    # the acoustic omega^2 at Gamma vanish
    assert np.abs(np.linalg.eigvalsh(Dm[0])).max() < 1e-5 * scale
    assert kpts.shape == (401, 3)


def test_tersoff_basis_and_neighbour_displacement_agree_to_second_order(oracle):
    from oracle.oracle_py import tersoff_parameters
    nt, para = tersoff_parameters(GOLDEN / "tersoff_Si_1989.txt")
    s = diamond(2)
    x, h, pbc = s["pos"], s["h"], s["pbc"]
    typ = np.zeros(x.shape[1], np.int32)

    def forces(y):
        return oracle.tersoff_compute(nt, para, typ, h, pbc, oracle.apply_pbc(h, pbc, y))["force"]

    r12, mask = P.geometry(x, h, pbc, 1, 2 * 3.0)
    diffs = []
    for d in (0.01, 0.005):
        Hb = P.h_basis(forces, x, 1, d, mask)
        Hn = P.h_neighbour(forces, x, 1, d, mask)
        diffs.append(np.abs(Hb - Hn).max())
    scale = np.abs(Hb).max()
    assert diffs[1] < 1e-4 * scale
    # second order in d: halving d divides the difference by about 4
    assert diffs[1] < 0.35 * diffs[0], diffs

"""libb200md_mgpu (C++ / CUDA / NCCL block decomposition, include/b200md_mgpu.h).

Local mode runs ALL domains of a Px x Py x Pz grid on one GPU in lock step through exactly the entry
points, kernels, ghost lists and message layout of the distributed run (device copies stand in for
ncclSend/Recv), so the decomposition is checked against the ORACLE on the driver's single-GPU box;
the NCCL transport itself is covered by the 2-process test below (needs 2 GPUs)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import cases_classical as cc
from conftest import GOLDEN, ROOT, TOL
from gpumd_b200.structures import TIME_UNIT_CONVERSION, diamond, fcc, init_velocities, rocksalt_pbte
from test_kernel_bodies_cpu import check_fv

pytestmark = pytest.mark.gpu

NEP = GOLDEN / "nep_PbTe.txt"
NEP_HALO = 2 * 8.0  # 2 rc of nep_PbTe.txt (radial cutoff 8 A); the group adds its skin
DT = 1.0 / TIME_UNIT_CONVERSION
CUFENI = GOLDEN / cc.EAM_FILES["cufeni"]
ENSEMBLES = ["nve", "nvt_ber", "nvt_nhc", "nvt_bdp"]


@pytest.fixture(scope="module")
def mg():
    import torch
    from gpumd_b200 import build
    build.build_lib()
    build.build_mgpu()
    assert torch.cuda.is_available()
    from gpumd_b200 import mgpu
    return mgpu


def nep_check(oracle, s, out, pos=None):
    """Owned forces / virials against the FP32 oracle on the WHOLE system at `pos` (default: the start),
    with the FP32 restatement's distance from FP64 added as in check_nep; returns the FP32 result."""
    orc = oracle.NepOracle(NEP)
    p = s["pos"] if pos is None else pos
    r = orc.compute(s["type"], s["h"], s["pbc"], p, precision=32)
    r64 = orc.compute(s["type"], s["h"], s["pbc"], p, precision=64)
    gap_v = np.abs(r["virial"] - r64["virial"]).max()
    check_fv(out, r, gap_f=np.abs(r["force"] - r64["force"]).max(), gap_v=gap_v)
    r["gap_v"] = gap_v
    return r


def block_coords(grid, rank):
    return rank // (grid[1] * grid[2]), (rank // grid[2]) % grid[1], rank % grid[2]


def lengths(s):
    return np.asarray(s["h"], dtype=np.float64).reshape(9)[[0, 4, 8]]


@pytest.mark.parametrize("grid,cells,pbc", [
    ((2, 1, 1), 14, (1, 1, 1)), ((2, 2, 1), 14, (1, 1, 1)), ((2, 2, 2), 14, (1, 1, 1)), ((3, 1, 2), 14, (1, 1, 1)),
    ((2, 1, 1), 6, (1, 1, 1)),   # w = 19.7 A: halo <= w < 2 halo, one atom can go to both faces
    ((3, 1, 1), 9, (1, 1, 1)),   # w = 19.7 A, lower and upper neighbour differ
    ((2, 2, 1), 14, (1, 1, 0)),  # slab: z open and undecomposed
], ids=["grid0", "grid1", "grid2", "grid3", "narrow_211", "narrow_311", "slab_221"])
def test_blocks_match_the_oracle_single_point(oracle, mg, grid, cells, pbc):
    """Forces / energies / virials of every owned atom of every block against the FP32 oracle evaluated
    on the WHOLE system (same tolerances as the single-domain parity tests)."""
    s = rocksalt_pbte(cells, rattle=0.05, seed=3)  # 14 cells: 21 952 atoms, 92 A: three 30.7 A blocks > 17 A halo
    s["pbc"] = np.array(pbc, np.int32)
    n = s["type"].shape[0]
    g = mg.DomainGroup(s["h"], s["pbc"], grid, NEP)
    g.distribute(s["type"], s["pos"], s["mass"])
    assert g.num_local_domains == grid[0] * grid[1] * grid[2]
    out = g.gather_local()
    assert np.array_equal(out["id"], np.arange(n))
    r = nep_check(oracle, s, out)
    assert abs(out["pe"].sum() - r["pe"].sum()) / n < 1e-6
    # thermo of the decomposed system = sum over blocks
    th = g.thermo()
    assert abs(th[1] - r["pe"].sum()) < 1e-6 * n


@pytest.mark.parametrize("grid", [(2, 1, 1), (2, 2, 1)])
def test_blocks_match_the_oracle_many_types(oracle, mg, grid):
    """The many-type kernels (UNEP-v1: 16 species, ZBL, separate neighbour split, direct reverse slots in the
    angular reduction) inside block domains: ghosts outside the active region must not disturb them."""
    from gpumd_b200.structures import nep_type_order
    model = GOLDEN / "nep_UNEP_v1.txt"
    s = fcc((10, 10, 8), 3.9, rattle=0.08, seed=5, num_types=16, symbols=nep_type_order(model))  # 39 A: 19.5 A blocks > 13 A halo
    n = s["type"].shape[0]
    g = mg.DomainGroup(s["h"], s["pbc"], grid, model)
    g.distribute(s["type"], s["pos"], s["mass"])
    out = g.gather_local()
    assert np.array_equal(out["id"], np.arange(n))
    orc = oracle.NepOracle(model)
    r = orc.compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32)
    r64 = orc.compute(s["type"], s["h"], s["pbc"], s["pos"], precision=64)
    check_fv(out, r, gap_f=np.abs(r["force"] - r64["force"]).max(), gap_v=np.abs(r["virial"] - r64["virial"]).max())
    assert abs(out["pe"].sum() - r["pe"].sum()) / n < 1e-6


def assert_owned_near_their_block(g, L, lim):
    """Every owned atom sits in its block or at most `lim` outside it (owners change only at exchanges)."""
    grid = np.array(g.grid)
    w = L / grid
    for k in range(g.num_local_domains):
        c = np.array(block_coords(g.grid, g.info(5, k)))
        pos = g.owned(k)["pos"]
        for d in range(3):
            if grid[d] > 1:
                x = np.mod(pos[d] - c[d] * w[d] + lim, L[d])
                assert x.max() <= w[d] + 2 * lim, (k, d, x.max() - lim - w[d])


def face_crossings(start, end, L, P, d):
    """Per block b of direction d: atoms whose block went b -> b+1 (its upper face, the last block's
    through the periodic wrap to block 0) and b -> b-1 (its lower face), from positions at two times."""
    w = L[d] / P
    c0 = np.minimum(np.floor(np.mod(start[d], L[d]) / w).astype(int), P - 1)
    c1 = np.minimum(np.floor(np.mod(end[d], L[d]) / w).astype(int), P - 1)
    up = (c1 - c0) % P == 1
    down = (c0 - c1) % P == 1
    return np.bincount(c0[up], minlength=P), np.bincount(c0[down], minlength=P)


TRAJECTORY_CASES = [pytest.param(e, g, id=e if g == (2, 2, 2) else f"{e}-{g[0]}{g[1]}{g[2]}")
                    for g in [(2, 2, 2), (4, 1, 1), (1, 2, 3)] for e in ENSEMBLES]


@pytest.mark.parametrize("ensemble,grid", TRAJECTORY_CASES)
def test_blocks_follow_the_single_domain_trajectory(oracle, mg, ensemble, grid):
    """200 steps on blocks vs one domain (same library, no decomposition), then the state against
    the oracle.  Hot enough (900 K, skin 1 A) that atoms cross block faces: migrations must happen.
    At 12 cells every block face (x = 0 and the wrap included) lies on a lattice plane, so with three
    or more blocks in a direction atoms change owner through both faces of every block."""
    from gpumd_b200 import engine
    import test_gpu_md
    s = rocksalt_pbte(12, rattle=0.02, seed=1)  # 13 824 atoms, 78.8 A -> 19.7 to 39.4 A blocks
    n = s["type"].shape[0]
    L = lengths(s)
    vel = init_velocities(s["mass"], 900.0, seed=42)
    g = mg.DomainGroup(s["h"], s["pbc"], grid, NEP, ensemble=ensemble,
                       temperature=900.0, temperature_coupling=100.0, time_step=DT, skin=1.0)
    g.distribute(s["type"], s["pos"], s["mass"], vel)
    g.run(200, check_every=5)
    g.check()
    assert g.migrations >= 1
    assert_owned_near_their_block(g, L, 0.35 * 1.0 + 0.1)  # + up to check_every steps of motion
    th = g.thermo()
    out = g.gather_local()
    assert np.array_equal(out["id"], np.arange(n))
    for d in range(3):
        if grid[d] >= 3:
            up, down = face_crossings(s["pos"], out["pos"], L, grid[d], d)
            assert (up > 0).all() and (down > 0).all(), (d, up, down)
    # single domain, same start
    atom, pot, rows = test_gpu_md.run_nve(engine, s, NEP, 200, 1.0, 900.0, seed=42,
                                          ensemble=ensemble, T_target=900.0)
    ref = rows[-1]
    assert abs(th[0] - ref[0]) < 0.05 and abs(th[1] - ref[1]) < 2e-6 * n
    # and the decomposed state is self-consistent with the oracle at its own positions
    nep_check(oracle, s, out, out["pos"])


@pytest.mark.parametrize("ensemble", ["nve", "nvt_ber", "nvt_nhc", "nvt_bdp", "lj"])
def test_one_block_is_the_single_domain_library(mg, ensemble):
    """Grid 1x1x1 with a skin that rules out any exchange runs the same kernels in the same order on the
    same atom order as the single-domain engine: every output is bit-identical after 100 steps."""
    from gpumd_b200 import engine
    import test_gpu_md
    if ensemble == "lj":
        s, pot_file, T, ensemble = fcc(12, 5.30, rattle=0.1, seed=5), GOLDEN / "lj_Ar_10A.txt", 80.0, "nve"
    else:
        s, pot_file, T = rocksalt_pbte(12, rattle=0.02, seed=1), NEP, 300.0
    n = s["type"].shape[0]
    # the engine wraps positions through the device apply_pbc (a round trip through fractional
    # coordinates, which moves in-box coordinates by an ulp) before its first force call; distribute
    # wraps on the host.  Hand the module the engine's first wrapped positions.
    a0, box = engine.Atom(s["type"], s["pos"], s["mass"]), engine.Box(s["h"], s["pbc"])
    engine._lib.check(engine._lib.load().b200md_apply_pbc(n, box._h, box._p, engine._ptr(a0.position_per_atom),
                                                          engine._stream()))
    p0 = a0.position_per_atom.cpu().numpy().reshape(3, n)
    g = mg.DomainGroup(s["h"], s["pbc"], (1, 1, 1), pot_file, ensemble=ensemble, temperature=T,
                       temperature_coupling=100.0, time_step=DT, skin=5.0)
    g.distribute(s["type"], p0, s["mass"], init_velocities(s["mass"], T, seed=42))
    g.run(100, check_every=5)
    g.check()
    assert g.migrations == 0  # an exchange would re-sort the lists, and with them the FP32 sums
    out = g.gather_local()
    th = g.thermo()
    atom, pot, rows = test_gpu_md.run_nve(engine, s, pot_file, 100, 1.0, T, seed=42, ensemble=ensemble, T_target=T)
    mine = dict(pos=out["pos"], vel=out["vel"], force=out["force"], virial=out["virial"], pe=out["pe"])
    theirs = dict(pos=atom.position_per_atom, vel=atom.velocity_per_atom, force=atom.force_per_atom,
                  virial=atom.virial_per_atom, pe=atom.potential_per_atom)
    for k, v in theirs.items():
        assert np.array_equal(mine[k], v.cpu().numpy().reshape(mine[k].shape)), k
    # temperature and energy bit for bit; the stress divides by the volume, which the engine takes as
    # numpy's determinant of h and the module as Lx Ly Lz (1.1e-15 apart for these boxes)
    assert np.array_equal(th[:2], rows[-1][:2])
    H = np.asarray(s["h"], dtype=np.float64).reshape(3, 3)
    v_gap = abs(abs(np.linalg.det(H)) / (H[0, 0] * H[1, 1] * H[2, 2]) - 1.0)
    assert (np.abs(th[2:] - rows[-1][2:]) <= (v_gap + 4e-16) * np.abs(rows[-1][2:])).all(), (th, rows[-1])


def read_thermo(path):
    return np.array([ln.split()[:18] for ln in open(path) if not ln.startswith("#")], dtype=np.float64)


@pytest.mark.parametrize("fixture,grid", [("refgpu_md_pbte_2gpu_thermo.out", (2, 1, 1)),
                                          ("refgpu_md_pbte_thermo.out", (2, 2, 2)),
                                          ("refgpu_md_pbte_ber_thermo.out", (2, 2, 2)),
                                          ("refgpu_md_pbte_bdp_thermo.out", (2, 2, 2)),
                                          ("refgpu_md_pbte_nhc_thermo.out", (2, 2, 2))])
def test_blocks_track_the_reference_gpu_trajectory(mg, fixture, grid):
    """thermo.out of the UNMODIFIED reference for 64 000 PbTe atoms, 200 steps from given velocities:
    NVE written by its NEP_MULTIGPU path on 2 GPUs (refgpu_md_pbte_2gpu_thermo.out) and by its
    single-GPU path (refgpu_md_pbte_thermo.out), nvt_ber / nvt_bdp / nvt_nhc (300 K, coupling 100) by
    its single-GPU path, scripts/run_reference_gpumd.py.  Our decomposed run must track them like the
    single-domain run does (test_gpu_md.py); the default bdp_seed is the reference's -DDEBUG stream."""
    if not (GOLDEN / fixture).exists():
        pytest.skip(f"{fixture} not generated yet (needs a 2-GPU box)")
    tag = fixture.split("_")[3]
    ensemble = "nvt_" + tag if tag in ("ber", "bdp", "nhc") else "nve"
    s = rocksalt_pbte(20, rattle=0.02, seed=1)
    n = s["type"].shape[0]
    ref = read_thermo(GOLDEN / fixture)
    g = mg.DomainGroup(s["h"], s["pbc"], grid, NEP, ensemble=ensemble, temperature=300.0,
                       temperature_coupling=100.0, time_step=DT, skin=1.0)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=42))
    rows = []
    for _ in range(20):
        g.run(10, check_every=5)
        rows.append(g.thermo())
    g.check()
    mine = np.array(rows)
    for k in range(20):
        tol = 2e-5 * (1 + k)
        assert abs(mine[k, 0] - ref[k, 0]) < tol * 3000, (k, mine[k, 0], ref[k, 0])
        assert abs(mine[k, 1] - ref[k, 2]) < tol * abs(ref[k, 2]), (k, mine[k, 1], ref[k, 2])
        for c in range(3):
            assert abs(mine[k, 2 + c] * 1.602177e+2 - ref[k, 3 + c]) < 2e-3 + 1e-3 * abs(ref[k, 3 + c])
    # first output (step 10): round-off limited.  2e-7 eV/atom in the single-domain test; the 2x2x2 blocks
    # change the FP32 summation order of every atom near a face and landed at 2.4e-7
    assert abs(mine[0, 0] - ref[0, 0]) < 2e-3 and abs(mine[0, 1] - ref[0, 2]) / n < 4e-7


# ---------------------------------------------------------------- heat current

def check_heat(oracle, g, out, ref_virial, virial_tol):
    """g.heat_current() against (a) the oracle's per-atom heat current of the gathered owned atoms (only
    the summation order differs) and (b) the same sum from the whole-system oracle virial at the
    gathered positions, within |virial error| * |v| summed over atoms and terms.  virial_tol: per-atom
    bound on the virial error, same shape as ref_virial."""
    j = g.heat_current()
    vel = out["vel"]
    mine = oracle.compute_heat(out["virial"], vel).sum(axis=1)
    scale = oracle.compute_heat(np.abs(out["virial"]), np.abs(vel)).sum(axis=1)
    assert (np.abs(j - mine) <= 1e-12 * scale + 1e-300).all(), (j, mine, scale)
    truth = oracle.compute_heat(ref_virial, vel).sum(axis=1)
    bound = oracle.compute_heat(virial_tol, np.abs(vel)).sum(axis=1)
    assert (np.abs(j - truth) <= bound).all(), (j, truth, bound)
    assert np.abs(j).max() > 0.0
    return j


def fv_virial_tol(r, gap_v=0.0):
    """check_fv's per-atom virial tolerance (conftest rtol and atol scaled by the largest component)."""
    vs = max(1.0, np.abs(r["virial"]).max())
    return TOL["virial"]["rtol"] * np.abs(r["virial"]) + TOL["virial"]["atol"] * vs + gap_v


HEAT_CASES = {  # name -> (kind, file, structure, grid, temperature, time step in fs)
    "nep_pbte_222": ("nep", NEP, lambda: rocksalt_pbte(12, rattle=0.02, seed=11), (2, 2, 2), 900.0, 1.0),
    "tersoff_sic_221": ("tersoff", cc.SIC, lambda: cc._sic(6, 12), (2, 2, 1), 1500.0, 1.0),
    "eam_cufeni_222": ("eam", CUFENI, lambda: fcc(10, 3.615, rattle=0.05, seed=13, num_types=3,
                                                 symbols=["Cu", "Fe", "Ni"]), (2, 2, 2), 900.0, 1.0),
    "lj_ar_221": ("lj", GOLDEN / "lj_Ar_10A.txt", lambda: fcc(12, 5.30, rattle=0.1, seed=14), (2, 2, 1), 80.0, 5.0),
}


def whole_system_virial(oracle, kind, path, s, pos):
    """(virial, per-atom virial tolerance) of the whole-system oracle at `pos`."""
    if kind == "nep":
        orc = oracle.NepOracle(path)
        r = orc.compute(s["type"], s["h"], s["pbc"], pos, precision=32)
        r64 = orc.compute(s["type"], s["h"], s["pbc"], pos, precision=64)
        return r["virial"], fv_virial_tol(r, np.abs(r["virial"] - r64["virial"]).max())
    r = cc.oracle32(kind, path, dict(s, pos=pos))
    if kind == "tersoff":  # FP64 on both sides: check_vs_oracle's virial tolerance
        return r["virial"], 1e-9 * np.abs(r["virial"]) + 1e-10
    return r["virial"], fv_virial_tol(r)


@pytest.mark.parametrize("name", list(HEAT_CASES))
def test_heat_current_of_the_blocks(oracle, mg, name):
    """b200md_mgpu_heat_current right after distribute and after a 200-step run with migrations."""
    kind, path, make, grid, T, dt_fs = HEAT_CASES[name]
    s = make()
    n = s["type"].shape[0]
    g = mg.DomainGroup(s["h"], s["pbc"], grid, path, time_step=dt_fs / TIME_UNIT_CONVERSION, skin=1.0)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], T, seed=21))
    for steps in (0, 200):
        if steps:
            g.run(steps, check_every=5)
            g.check()
            assert g.migrations >= 1
        out = g.gather_local()
        assert np.array_equal(out["id"], np.arange(n))
        check_heat(oracle, g, out, *whole_system_virial(oracle, kind, path, s, out["pos"]))


@pytest.mark.parametrize("case", ["lj", "si"])
def test_blocks_other_potentials(oracle, mg, case):
    """Pair (halo rc + skin) and FP64 many-body (halo 2 rc + skin) potentials through the same blocks."""
    if case == "lj":
        s = fcc(12, 5.30, rattle=0.1, seed=5)  # 6912 atoms, 63.6 A
        g = mg.DomainGroup(s["h"], s["pbc"], (2, 2, 1), GOLDEN / "lj_Ar_10A.txt")
        g.distribute(s["type"], s["pos"], s["mass"])
        out = g.gather_local()
        r = oracle.lj_compute(np.array([[[1.032e-2, 3.405, 10.0]]]), s["type"], s["h"], s["pbc"], s["pos"])
        check_fv(out, r)
    else:
        s = diamond(8, a=5.431, rattle=0.08, seed=6)  # 4096 atoms, 43.4 A
        g = mg.DomainGroup(s["h"], s["pbc"], (2, 2, 2), GOLDEN / "tersoff_Si_1989.txt")
        g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=1))
        out = g.gather_local()
        nt, p0 = oracle.tersoff_parameters(GOLDEN / "tersoff_Si_1989.txt")
        r = oracle.tersoff_compute(nt, p0, s["type"], s["h"], s["pbc"], s["pos"])
        assert np.allclose(out["force"], r["force"], rtol=1e-9, atol=1e-10)
        assert np.allclose(out["pe"], r["pe"], rtol=1e-10, atol=1e-12)
        check_heat(oracle, g, out, r["virial"], 1e-9 * np.abs(r["virial"]) + 1e-10)


# ---------------------------------------------------------------- ghost set

def images_in_block(type_, pos, L, grid, c, halo, lo, hi):
    """(type, local position) of every periodic image of the atoms whose local coordinate
    x - (c_d w_d - halo) lies in [lo, hi) in every decomposed direction d; other directions keep x."""
    idx = np.arange(type_.shape[0])
    p = np.array(pos, dtype=np.float64)
    for d in range(3):
        if grid[d] == 1:
            continue
        w = L[d] / grid[d]
        x = p[d] - (c[d] * w - halo)
        keep_i, keep_p = [], []
        for m in range(-2, 3):
            xm = x + m * L[d]
            sel = (xm >= lo[d]) & (xm < hi[d])
            q = p[:, sel].copy()
            q[d] = xm[sel]
            keep_i.append(idx[sel])
            keep_p.append(q)
        idx, p = np.concatenate(keep_i), np.concatenate(keep_p, axis=1)
    return type_[idx], p


def points(type_, pos):
    return np.column_stack([1.0e3 * type_, pos.T])  # types 1000 A apart: never within the match radius


def assert_ghost_sets(g, s, pos, halo, margin):
    """Exact (margin None): owned + ghosts of every domain == images with local coordinates in
    [0, w + 2 halo), owned == those in [halo, halo + w), no duplicate and no missing image.
    margin m: every image in [m, w + 2 halo - m) is present exactly once."""
    from scipy.spatial import cKDTree
    L = lengths(s)
    grid = np.array(g.grid)
    w = L / grid
    for k in range(g.num_local_domains):
        c = block_coords(g.grid, g.info(5, k))
        loc = g.local_system(k)
        m_loc = loc["type"].shape[0]
        got = points(loc["type"], loc["pos"].reshape(3, m_loc))
        tree = cKDTree(got)
        if margin is None:
            t, p = images_in_block(s["type"], pos, L, grid, c, halo, [0.0] * 3, w + 2 * halo)
            want = points(t, p)
            assert got.shape == want.shape, (k, got.shape, want.shape)
            assert not tree.query_pairs(1e-9), k  # no image twice
            d_got, _ = cKDTree(want).query(got)
            d_want, _ = tree.query(want)
            assert d_got.max() < 1e-9 and d_want.max() < 1e-9, (k, d_got.max(), d_want.max())
            t, p = images_in_block(s["type"], pos, L, grid, c, halo, [halo] * 3, w + halo)
            own = points(t, p)
            assert own.shape[0] == loc["n_own"]
            d_own, _ = cKDTree(got[:loc["n_own"]]).query(own)
            assert d_own.max() < 1e-9, k
        else:
            t, p = images_in_block(s["type"], pos, L, grid, c, halo, [margin] * 3, w + 2 * halo - margin)
            count = tree.query_ball_point(points(t, p), 1e-9, return_length=True)
            assert (count == 1).all(), (k, np.bincount(count))


@pytest.mark.parametrize("grid,cells", [((2, 2, 2), 14), ((3, 1, 2), 14), ((2, 1, 1), 6)],
                         ids=["222", "312", "narrow_211"])
def test_ghost_set_is_every_image_in_the_halo(mg, grid, cells):
    """The atoms each domain holds, right after distribute and after 200 steps with an exchange check
    every step (900 K, skin 1 A): between exchanges atoms move at most 0.35 skin (+ one step)."""
    s = rocksalt_pbte(cells, rattle=0.05, seed=3)
    skin = 1.0
    halo = NEP_HALO + skin
    g = mg.DomainGroup(s["h"], s["pbc"], grid, NEP, time_step=DT, skin=skin)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 900.0, seed=42))
    assert_ghost_sets(g, s, s["pos"], halo, None)
    g.run(200, check_every=1)
    assert g.migrations >= 1
    assert_ghost_sets(g, s, g.gather_local()["pos"], halo, 0.35 * skin + 0.05)


# ---------------------------------------------------------------- CUDA graph

def test_cuda_graph_replay_is_bit_identical(mg):
    """The per-step CUDA graph (all launches + the staged halo copies of one step) replays to the same
    trajectory as eager launches."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    dt = 1.0 / TIME_UNIT_CONVERSION
    vel = init_velocities(s["mass"], 300.0, seed=42)
    res = []
    for graph in (False, True):
        g = mg.DomainGroup(s["h"], s["pbc"], (2, 1, 1), GOLDEN / "nep_PbTe.txt", time_step=dt, skin=3.0,
                           cuda_graph=graph)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        g.run(50, check_every=5)
        g.check()
        res.append(g.gather_local())
    assert np.array_equal(res[0]["pos"], res[1]["pos"]) and np.array_equal(res[0]["vel"], res[1]["vel"])


@pytest.mark.parametrize("ensemble", ENSEMBLES)
@pytest.mark.parametrize("grid", [(2, 2, 1), (4, 1, 1)])
def test_cuda_graph_replay_across_exchanges_is_bit_identical(mg, grid, ensemble):
    """As above, hot enough (900 K, skin 1 A, 200 steps) that both runs migrate: every exchange destroys
    and re-captures the graph, and the NHC chain / BDP random state advances on the device inside it.
    The whole final state and the thermo must agree bit for bit."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 900.0, seed=42)
    res = []
    for graph in (False, True):
        g = mg.DomainGroup(s["h"], s["pbc"], grid, NEP, ensemble=ensemble, temperature=900.0,
                           temperature_coupling=100.0, time_step=DT, skin=1.0, cuda_graph=graph)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        g.run(200, check_every=5)
        g.check()
        assert g.migrations >= 1
        res.append((g.migrations, g.thermo(), g.gather_local()))
    assert res[0][0] == res[1][0]
    assert np.array_equal(res[0][1], res[1][1])
    for k in ("pos", "vel", "force", "virial", "pe"):
        assert np.array_equal(res[0][2][k], res[1][2][k]), k


# ---------------------------------------------------------------- open direction

def test_slab_follows_the_single_domain_trajectory(oracle, mg):
    """PbTe slab (z open, undecomposed) on 2x2x1 blocks, 200 steps at 900 K against one domain: the
    open direction is never wrapped and never enters the displacement check's minimum image."""
    from gpumd_b200 import engine
    import test_gpu_md
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    s["pbc"] = np.array([1, 1, 0], np.int32)
    s["pos"][2] = s["pos"][2] + 1.0  # the z = 0 plane clear of the open face: both surfaces are whole planes
    n = s["type"].shape[0]
    g = mg.DomainGroup(s["h"], s["pbc"], (2, 2, 1), NEP, temperature=900.0, time_step=DT, skin=1.0)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 900.0, seed=42))
    g.run(200, check_every=5)
    g.check()
    assert g.migrations >= 1
    th = g.thermo()
    out = g.gather_local()
    dz = out["pos"][2] - s["pos"][2]
    assert np.abs(dz).max() < 2.0  # no atom wrapped in z
    atom, pot, rows = test_gpu_md.run_nve(engine, s, NEP, 200, 1.0, 900.0, seed=42)
    assert abs(th[0] - rows[-1][0]) < 0.05 and abs(th[1] - rows[-1][1]) < 2e-6 * n
    nep_check(oracle, s, out, out["pos"])


# ---------------------------------------------------------------- blocks that own no atoms

def vacuum_slab():
    """PbTe slab of 5 cells (32.9 A) along x in a 160 A box, periodic in x, y, z.  On 4x1x1 blocks
    (w = 40 A, halo 17 A) block 0 owns every atom, blocks 1 and 3 own none but hold ghosts across
    x = 40 and the periodic wrap, block 2 holds nothing."""
    s = rocksalt_pbte((5, 6, 6), rattle=0.02, seed=7)  # 1440 atoms
    s["pos"][0] = s["pos"][0] + 3.5
    s["h"] = s["h"].copy()
    s["h"][0] = 160.0
    return s


def empty_block_checks():
    """Body of test_blocks_that_own_no_atoms (run in a child process)."""
    from gpumd_b200 import engine, mgpu
    from oracle import oracle_py as oracle
    import test_gpu_md
    s = vacuum_slab()
    n = s["type"].shape[0]
    vel = init_velocities(s["mass"], 300.0, seed=42)
    for ensemble in ("nve", "nvt_bdp"):
        g = mgpu.DomainGroup(s["h"], s["pbc"], (4, 1, 1), NEP, ensemble=ensemble, temperature=300.0,
                             temperature_coupling=100.0, time_step=DT, skin=1.0)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        n_own = [g.info(1, k) for k in range(4)]
        n_loc = [g.info(2, k) for k in range(4)]
        assert n_own == [n, 0, 0, 0] and n_loc[1] > 0 and n_loc[2] == 0 and n_loc[3] > 0, (n_own, n_loc)
        out = g.gather_local()
        assert np.array_equal(out["id"], np.arange(n))
        r = nep_check(oracle, s, out)
        assert abs(out["pe"].sum() - r["pe"].sum()) / n < 1e-6
        th = g.thermo()
        assert abs(th[1] - r["pe"].sum()) < 1e-6 * n
        check_heat(oracle, g, out, r["virial"], fv_virial_tol(r, r["gap_v"]))
        g.run(100, check_every=5)
        g.check()
        th = g.thermo()
        out = g.gather_local()
        atom, pot, rows = test_gpu_md.run_nve(engine, s, NEP, 100, 1.0, 300.0, seed=42, ensemble=ensemble,
                                              T_target=300.0)
        assert abs(th[0] - rows[-1][0]) < 0.05 and abs(th[1] - rows[-1][1]) < 2e-6 * n, (th, rows[-1])
        assert np.abs(out["pos"] - atom.position_per_atom.cpu().numpy().reshape(3, n)).max() < 1e-5
        r = nep_check(oracle, s, out, out["pos"])
        check_heat(oracle, g, out, r["virial"], fv_virial_tol(r, r["gap_v"]))
    print("empty blocks: ok")


def test_blocks_that_own_no_atoms(oracle, mg):
    """A slab across vacuum: blocks with ghosts but no owned atoms, and a block with no atoms at all, in the
    single point, 100 NVE and BDP steps against one domain, thermo and heat current.  Runs in a child
    process: a failed launch leaves an error that every later launch check of the process would report."""
    code = "import sys; sys.path[:0] = sys.argv[1:]; import test_gpu_mgpu; test_gpu_mgpu.empty_block_checks()"
    r = subprocess.run([sys.executable, "-c", code, str(ROOT), str(ROOT / "tests")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "empty blocks: ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# ---------------------------------------------------------------- rejected configurations

def test_rejected_configurations(mg):
    """Refused with a message, never run."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    tric = s["h"].copy()
    tric[1] = 2.0
    with pytest.raises(mg.MgpuError, match="orthogonal box"):
        mg.DomainGroup(tric, s["pbc"], (2, 1, 1), NEP)
    with pytest.raises(mg.MgpuError, match="decomposed directions must be periodic"):
        mg.DomainGroup(s["h"], [1, 1, 0], (1, 1, 2), NEP)
    small = rocksalt_pbte(5, rattle=0.02, seed=1)  # 32.9 A: 16.4 A blocks < 17 A halo
    with pytest.raises(mg.MgpuError, match="narrower than the halo"):
        mg.DomainGroup(small["h"], small["pbc"], (2, 1, 1), NEP)
    g = mg.DomainGroup(s["h"], s["pbc"], (2, 1, 1), NEP, ensemble=3)
    with pytest.raises(mg.MgpuError, match="unsupported ensemble"):
        g.distribute(s["type"], s["pos"], s["mass"])


WORKER = r"""
import os, sys, json
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2_ROOT"]); sys.path.insert(0, os.path.join(os.environ["B2_ROOT"], "tests"))
from gpumd_b200 import mgpu
from gpumd_b200.structures import TIME_UNIT_CONVERSION, init_velocities, rocksalt_pbte
rank = int(os.environ["RANK"]); torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl")
s = rocksalt_pbte(12, rattle=0.02, seed=1)
vel = init_velocities(s["mass"], 300.0, seed=42)
g = mgpu.DomainGroup(s["h"], s["pbc"], (2, 1, 1), os.environ["B2_MODEL"], time_step=1.0 / TIME_UNIT_CONVERSION,
                     skin=1.0, distributed=True)
g.distribute(s["type"], s["pos"], s["mass"], vel)
g.run(100, check_every=5); g.check()
o = g.owned(0)
np.savez(os.path.join(os.environ["B2_OUT"], f"rank{rank}.npz"), thermo=g.thermo(), **o)
dist.barrier(); dist.destroy_process_group()
"""


def test_two_ranks_over_nccl_match_the_local_run(mg, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    (tmp_path / "worker.py").write_text(WORKER)
    env = dict(os.environ, B2_ROOT=str(ROOT), B2_MODEL=str(GOLDEN / "nep_PbTe.txt"), B2_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29533", str(tmp_path / "worker.py")],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    parts = [np.load(tmp_path / f"rank{k}.npz") for k in range(2)]
    ids = np.concatenate([p["id"] for p in parts])
    order = np.argsort(ids)
    pos = np.concatenate([p["pos"] for p in parts], axis=1)[:, order]
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    g = mg.DomainGroup(s["h"], s["pbc"], (2, 1, 1), GOLDEN / "nep_PbTe.txt", time_step=1.0 / TIME_UNIT_CONVERSION,
                       skin=1.0)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=42))
    g.run(100, check_every=5)
    loc = g.gather_local()
    assert np.array_equal(np.sort(ids), np.arange(s["type"].shape[0]))
    assert np.array_equal(pos, loc["pos"])  # same kernels, same message order: bit-identical
    assert np.allclose(parts[0]["thermo"], g.thermo(), rtol=1e-13)

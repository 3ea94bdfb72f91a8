"""LJ, Tersoff-1989 and EAM kernels on the device: triclinic, open and multi-species boxes against the FP32
oracle and the FP64 references (tests/cases_classical.py), known-answer clusters, per-pair LJ cutoffs,
skin-list reuse / rebuild / invalidation, NVE runs and block domains (the benchmark sizes: test_gpu_full_size.py)."""
import numpy as np
import pytest

import cases_classical as cc
from conftest import GOLDEN
from gpumd_b200.structures import TIME_UNIT_CONVERSION, fcc, init_velocities
from test_classical_cpu import CLUSTERS, check_cluster, check_vs_fp64, check_vs_oracle, make_cluster

pytestmark = pytest.mark.gpu

POT = {"lj": "LJ", "tersoff": "Tersoff1989", "eam": "EAM"}
CUFENI = GOLDEN / cc.EAM_FILES["cufeni"]


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def compute(eng, kind, path, s, pot=None, prefill=None):
    """One force call through engine.LJ / Tersoff1989 / EAM (created from the potential file unless
    `pot` is given); prefill: values the outputs hold before the call."""
    n = s["type"].shape[0]
    if pot is None:
        pot = getattr(eng, POT[kind])(path, n)
    atom = eng.Atom(s["type"], s["pos"], np.ones(n))
    if prefill is not None:
        atom.potential_per_atom.fill_(prefill[0])
        atom.force_per_atom.fill_(prefill[1])
        atom.virial_per_atom.fill_(prefill[2])
    pot.compute(eng.Box(s["h"], s["pbc"]), atom.type, atom.position_per_atom, atom.potential_per_atom,
                atom.force_per_atom, atom.virial_per_atom)
    pot.check()
    return dict(pe=atom.potential_per_atom.cpu().numpy(), force=atom.force_per_atom.cpu().numpy().reshape(3, n),
                virial=atom.virial_per_atom.cpu().numpy().reshape(9, n)), pot


@pytest.mark.parametrize("case", cc.CASES)
def test_single_point_matches_oracle_and_fp64(oracle, eng, case):
    """Every potential x structure x box form: against the FP32 oracle with the tolerances of the existing
    parity tests, and against the FP64 reference with the oracle's own FP32-FP64 gap added (check_nep)."""
    kind, path, s = cc.make(case)
    n = s["type"].shape[0]
    r32 = cc.oracle32(kind, path, s)
    r64 = cc.reference64(kind, path, s, f32_params=True)
    out, _ = compute(eng, kind, path, s)
    check_vs_oracle(out, r32, n, kind, path)
    check_vs_fp64(out, r64, n, kind, path, gap=cc.gaps(r32, r64))


@pytest.mark.parametrize("name", list(CLUSTERS))
def test_clusters_known_answers(oracle, eng, name):
    """Isolated atom, dimer and equilateral trimer in an open box: closed forms and symmetry."""
    kind, path, s = make_cluster(name)
    out, _ = compute(eng, kind, path, s)
    check_cluster(out, name, s["type"].shape[0])


def test_lj_cutoff_membership_per_pair_type(oracle, eng):
    """Pairs within +-6 ulps of each of the six pair cutoffs of the 3-species table, on a dilute lattice:
    the per-pair-type cutoff test must agree with the oracle's for every pair.  A disagreement moves an
    atom's energy by U(rc)/2 >= 3.2e-5 eV, far above the tolerance."""
    table = cc.lj_table(cc.LJ3)
    s = fcc(4, 22.0, rattle=0.0, seed=1, num_types=1)  # 256 atoms, 15.6 A apart, 88 A box
    pos, n = s["pos"].copy(), s["type"].shape[0]
    types = np.zeros(n, np.int32)
    rng = np.random.default_rng(7)
    kinds = [(a, b) for a in range(3) for b in range(a, 3)]
    dist = []
    for k in range(n // 2):
        i, j = 2 * k, 2 * k + 1
        a, b = kinds[k % 6]
        types[i], types[j] = a, b
        rc = table[a, b, 2]
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        r = rc + rng.integers(-6, 7) * 6e-8 * rc
        pos[:, j] = pos[:, i] + u * r
        dist.append((r, rc))
    s = dict(s, pos=cc.wrap(s["h"], s["pbc"], pos), type=types)
    r32 = cc.oracle32("lj", cc.LJ3, s)
    out, _ = compute(eng, "lj", cc.LJ3, s)
    np.testing.assert_allclose(out["pe"], r32["pe"], rtol=1e-5, atol=1e-7)
    inside = sum(r < rc for r, rc in dist)
    assert 10 < inside < len(dist) - 10  # the construction straddles the cutoffs


# ---------------------------------------------------------------- list dynamics

DYN = {"lj": "lj_3sp-tric", "tersoff": "sic-tric", "eam": "eam_cufeni_a0-tric"}


@pytest.mark.parametrize("kind", list(DYN))
def test_skin_list_reuse_then_rebuild(oracle, eng, kind):
    """Two steps of displacements < skin/2 reuse the list; one atom moved by 0.6 A rebuilds it.  Oracle
    parity after every step."""
    _, path, s = cc.make(DYN[kind])
    n = s["type"].shape[0]
    out, pot = compute(eng, kind, path, s)
    assert pot.num_rebuilds == 1
    rng = np.random.default_rng(3)
    pos = s["pos"].copy()
    for step, amp, expect in ((1, 0.12, 1), (2, 0.12, 1), (3, 0.0, 2)):
        disp = rng.uniform(-1, 1, pos.shape) * amp / np.sqrt(3)
        if step == 3:
            disp[:, 17] = [0.6, 0.0, 0.0]
        pos = cc.wrap(s["h"], s["pbc"], pos + disp)
        t = dict(s, pos=pos)
        out, _ = compute(eng, kind, path, t, pot=pot)
        assert pot.num_rebuilds == expect, (step, pot.num_rebuilds)
        check_vs_oracle(out, cc.oracle32(kind, path, t), n, kind, path)


@pytest.mark.parametrize("kind", list(DYN))
def test_fewer_atoms_than_capacity_equals_a_fresh_handle(oracle, eng, kind):
    """A handle created for N atoms and used on an N-atom system, then called on a different system of
    n < N atoms (Neighbor::update -> invalidate, the block-domain ghost path; column-major lists then have
    stride n): bit-identical to a handle created for n."""
    _, path, big = cc.make(DYN[kind])
    _, _, small = cc.make(DYN[kind].replace("-tric", "-slab"))
    m = small["type"].shape[0] * 3 // 4  # a slab with vacancies: another box, pbc and atom count
    small = dict(small, pos=small["pos"][:, :m], type=small["type"][:m])
    pot = getattr(eng, POT[kind])(path, big["type"].shape[0])
    compute(eng, kind, path, big, pot=pot)
    a, _ = compute(eng, kind, path, small, pot=pot)
    b, _ = compute(eng, kind, path, small)
    for k in ("pe", "force", "virial"):
        assert np.array_equal(a[k], b[k]), k
    check_vs_oracle(a, cc.oracle32(kind, path, small), small["type"].shape[0], kind, path)


@pytest.mark.parametrize("kind", list(DYN))
def test_accumulates_into_outputs_and_is_deterministic(oracle, eng, kind):
    """Potential::compute contract: outputs are added to (b2_body_unpack's +=); repeat calls are
    bit-identical (gather-only kernels)."""
    _, path, s = cc.make(DYN[kind])
    a, pot = compute(eng, kind, path, s)
    b, _ = compute(eng, kind, path, s, pot=pot)
    c, _ = compute(eng, kind, path, s)
    for k in ("pe", "force", "virial"):
        assert np.array_equal(a[k], b[k]) and np.array_equal(a[k], c[k]), k
    d, _ = compute(eng, kind, path, s, pot=pot, prefill=(1.0, 2.0, 3.0))
    for k, v in (("pe", 1.0), ("force", 2.0), ("virial", 3.0)):
        assert np.allclose(d[k] - v, a[k], rtol=0, atol=1e-12), k


@pytest.mark.parametrize("kind", list(DYN))
def test_small_box_is_rejected(eng, kind):
    """A periodic thickness <= 2.5 (rc + 1) returns B200MD_ERR_SMALL_BOX before any kernel runs."""
    from gpumd_b200.lib import B200mdError
    _, path, s = cc.make(DYN[kind])
    rc = cc.cutoff(kind, path)
    H = s["h"].reshape(3, 3).copy()
    H[:, 1] *= 2.45 * (rc + 1) / cc.thickness(s["h"])[1]  # y thickness just below the limit
    t = dict(s, h=H.reshape(9), pos=s["pos"] * 0.0 + 1.0)
    n = s["type"].shape[0]
    pot = getattr(eng, POT[kind])(path, n)
    atom = eng.Atom(t["type"], t["pos"], np.ones(n))
    before = eng.launch_count()
    with pytest.raises(B200mdError, match="error 4"):
        pot.compute(eng.Box(t["h"], t["pbc"]), atom.type, atom.position_per_atom, atom.potential_per_atom,
                    atom.force_per_atom, atom.virial_per_atom)
    assert eng.launch_count() == before
    assert float(atom.force_per_atom.abs().max()) == 0.0


# ---------------------------------------------------------------- MD

def read_thermo(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#")], dtype=np.float64)


def test_eam_nve_conserves_and_tracks_the_reference_gpu(oracle, eng):
    """CuFeNi, 4000 atoms, 300 K, 200 steps of 1 fs: the reference's conservation bound 2e-3 dt^2 N eV,
    oracle parity at the final positions, and thermo.out of the unmodified reference
    gpumd from the same start (tests/golden/refgpu_md_eam_thermo.out) within the time-widening tolerances of
    test_gpu_md.test_nve_trajectory_matches_reference_gpu."""
    from test_gpu_md import run_nve, total_energy
    s = fcc(10, 3.615, rattle=0.0, seed=1, num_types=3, symbols=["Cu", "Fe", "Ni"])
    n = s["type"].shape[0]
    atom, pot, rows = run_nve(eng, s, CUFENI, 200, 1.0, 300.0, seed=42, every=10)
    e = total_energy(rows, n)
    assert np.abs(e - e[0]).max() < 2e-3 * n
    # no atom of a 300 K crystal strays skin/2 = 0.5 A in 200 fs: the list is built once (the 900 K run of
    # test_eam_blocks_follow_the_single_domain_trajectory rebuilds it)
    assert pot.num_rebuilds == 1
    pos = atom.position_per_atom.cpu().numpy().reshape(3, n)
    r = cc.oracle32("eam", CUFENI, dict(s, pos=pos))
    out = dict(pe=atom.potential_per_atom.cpu().numpy(), force=atom.force_per_atom.cpu().numpy().reshape(3, n),
               virial=atom.virial_per_atom.cpu().numpy().reshape(9, n))
    check_vs_oracle(out, r, n, "eam", CUFENI)
    ref = read_thermo(GOLDEN / "refgpu_md_eam_thermo.out")
    mine = rows[1:-1]
    assert mine.shape[0] == ref.shape[0] == 20
    for k in range(20):
        tol = 2e-5 * (1 + k)
        assert abs(mine[k, 0] - ref[k, 0]) < tol * 300.0 * 10, (k, mine[k, 0], ref[k, 0])
        assert abs(mine[k, 1] - ref[k, 2]) < tol * abs(ref[k, 2]), (k, mine[k, 1], ref[k, 2])
        for c in range(3):
            assert abs(mine[k, 2 + c] * 1.602177e+2 - ref[k, 3 + c]) < 2e-3 + 1e-3 * abs(ref[k, 3 + c])
    assert abs(mine[0, 0] - ref[0, 0]) < 2e-3 and abs(mine[0, 1] - ref[0, 2]) / n < 2e-7


def test_sic_tersoff_nve(oracle, eng):
    """Zincblende SiC (every bond through the mixed parameter set) from the perfect lattice, 1000 K, 200 steps
    of 0.5 fs: the reference's bound 2e-3 dt^2 N eV and oracle parity at the final positions.  (A 0.08 A
    rattle of this stiff lattice alone stores ~0.1 eV per degree of freedom: started from it, the run
    fluctuates by 1.7 eV, above the bound's 0.86 eV, whatever the initial temperature.)"""
    from test_gpu_md import run_nve, total_energy
    from cases_classical import _sic
    s = _sic(6, 71, rattle=0.0)
    n = s["type"].shape[0]
    atom, pot, rows = run_nve(eng, s, cc.SIC, 200, 0.5, 1000.0, seed=42, every=10)
    e = total_energy(rows, n)
    assert np.abs(e - e[0]).max() < 2e-3 * 0.25 * n
    pos = atom.position_per_atom.cpu().numpy().reshape(3, n)
    r = cc.oracle32("tersoff", cc.SIC, dict(s, pos=pos))
    out = dict(pe=atom.potential_per_atom.cpu().numpy(), force=atom.force_per_atom.cpu().numpy().reshape(3, n),
               virial=atom.virial_per_atom.cpu().numpy().reshape(9, n))
    check_vs_oracle(out, r, n, "tersoff", cc.SIC)


# ---------------------------------------------------------------- block domains

@pytest.fixture(scope="module")
def mg():
    import torch
    from gpumd_b200 import build
    build.build_lib()
    build.build_mgpu()
    assert torch.cuda.is_available()
    from gpumd_b200 import mgpu
    return mgpu


BLOCKS = {  # name -> (kind, file, structure, grid)
    "eam_221": ("eam", CUFENI, lambda: fcc(10, 3.615, rattle=0.08, seed=81, num_types=3, symbols=["Cu", "Fe", "Ni"]),
                (2, 2, 1)),
    "eam_222": ("eam", CUFENI, lambda: fcc(10, 3.615, rattle=0.08, seed=82, num_types=3, symbols=["Cu", "Fe", "Ni"]),
                (2, 2, 2)),
    "sic_221": ("tersoff", cc.SIC, lambda: cc._sic(6, 83), (2, 2, 1)),
    "sic_222": ("tersoff", cc.SIC, lambda: cc._sic(6, 84), (2, 2, 2)),
    "lj3_221": ("lj", cc.LJ3, lambda: fcc(12, 5.30, rattle=0.1, seed=85, num_types=3, symbols=("Ar", "Ar", "Ar")),
                (2, 2, 1)),
}


@pytest.mark.parametrize("name", list(BLOCKS))
def test_blocks_match_the_whole_system_oracle(oracle, mg, name):
    """Block domains (local mode, ghosts exchanged like the distributed run) against the oracle on the
    whole periodic system; blocks are wider than 2 rc + skin."""
    kind, path, make, grid = BLOCKS[name]
    s = make()
    n = s["type"].shape[0]
    g = mg.DomainGroup(s["h"], s["pbc"], grid, path)
    g.distribute(s["type"], s["pos"], s["mass"])
    assert g.num_local_domains == grid[0] * grid[1] * grid[2]
    out = g.gather_local()
    assert np.array_equal(out["id"], np.arange(n))
    check_vs_oracle(out, cc.oracle32(kind, path, s), n, kind, path)


def test_eam_blocks_follow_the_single_domain_trajectory(oracle, mg):
    """200 NVE steps of CuFeNi on 2x2x2 blocks against one domain from the same start (900 K, so atoms
    cross block faces), then the decomposed state against the oracle at its own positions."""
    from gpumd_b200 import engine
    from test_gpu_md import run_nve
    s = fcc(10, 3.615, rattle=0.02, seed=1, num_types=3, symbols=["Cu", "Fe", "Ni"])
    n = s["type"].shape[0]
    vel = init_velocities(s["mass"], 900.0, seed=42)
    g = mg.DomainGroup(s["h"], s["pbc"], (2, 2, 2), CUFENI, time_step=1.0 / TIME_UNIT_CONVERSION, skin=1.0)
    g.distribute(s["type"], s["pos"], s["mass"], vel)
    g.run(200, check_every=5)
    g.check()
    assert g.migrations >= 1
    th = g.thermo()
    out = g.gather_local()
    assert np.array_equal(out["id"], np.arange(n))
    atom, pot, rows = run_nve(engine, s, CUFENI, 200, 1.0, 900.0, seed=42)
    assert pot.num_rebuilds >= 2  # the first build, then at least one triggered by the skin check
    assert abs(th[0] - rows[-1][0]) < 0.05 and abs(th[1] - rows[-1][1]) < 2e-6 * n
    check_vs_oracle(out, cc.oracle32("eam", CUFENI, dict(s, pos=out["pos"])), n, "eam", CUFENI)

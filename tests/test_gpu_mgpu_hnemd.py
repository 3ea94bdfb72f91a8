"""HNEMD inside the block-domain step of libb200md_mgpu (b200md_mgpu_hnemd_set / _take): the driving force
after the potential, the heat row after the thermostat, kappa at take time.

One 1x1x1 block is the single-domain library bit for bit; the blocks track the reference's own HNEMD run
and the single-domain run across migrations; CUDA-graph replay, blocks that own no atoms, the take
semantics and the two-rank NCCL run are pinned as for the undriven step (test_gpu_mgpu.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import heat_oracle as ho
from conftest import GOLDEN, ROOT
from gpumd_b200.structures import TIME_UNIT_CONVERSION, init_velocities, rocksalt_pbte

pytestmark = pytest.mark.gpu

NEP = GOLDEN / "nep_PbTe.txt"
DT = 1.0 / TIME_UNIT_CONVERSION
FE = (2e-5, 0.0, 0.0)
OI = 10


@pytest.fixture(scope="module")
def mg():
    import torch
    from gpumd_b200 import build
    build.build_lib()
    build.build_mgpu()
    assert torch.cuda.is_available()
    from gpumd_b200 import mgpu
    return mgpu


def volume(s):
    h = np.asarray(s["h"], dtype=np.float64).reshape(9)
    return h[0] * h[4] * h[8]  # the module's Lx Ly Lz


def wrapped_positions(s):
    """The engine's first wrapped positions (its device apply_pbc moves in-box coordinates by an ulp;
    distribute wraps on the host): handing these to the module makes 1x1x1 start where the engine does."""
    from gpumd_b200 import engine
    n = s["type"].shape[0]
    a0, box = engine.Atom(s["type"], s["pos"], s["mass"]), engine.Box(s["h"], s["pbc"])
    engine._lib.check(engine._lib.load().b200md_apply_pbc(n, box._h, box._p, engine._ptr(a0.position_per_atom),
                                                          engine._stream()))
    return a0.position_per_atom.cpu().numpy().reshape(3, n)


def engine_run(s, steps, T, ensemble, fe=FE, oi=OI):
    """test_gpu_md.run_nve's loop on one domain with Force.set_hnemd and HNEMD.process after compute2;
    returns (atom, thermo, kappa[n, 5], rows[n, oi, 5])."""
    import torch
    from gpumd_b200 import engine
    n = s["type"].shape[0]
    atom = engine.Atom(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], T, seed=42))
    box = engine.Box(s["h"], s["pbc"])
    force = engine.Force()
    pot = force.parse_potential(NEP, n)
    force.set_hnemd(fe)
    ens = (engine.Ensemble_BER(n, T, 100.0) if ensemble == "nvt_ber"
           else engine.Ensemble_NHC(n, T, 100.0, DT))
    hn = engine.HNEMD(oi, fe)
    thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
    args = (box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
            atom.virial_per_atom)
    force.compute(*args)
    ens.find_thermo(box.get_volume(), atom, thermo)
    kappa, rows = [], []
    for step in range(steps):
        ens.compute1(DT, box, atom, thermo)
        force.compute(*args)
        ens.compute2(DT, box, atom, thermo)
        hn.process(step, atom)
        if (step + 1) % oi == 0:
            k, r = hn.take(volume(s), T)
            kappa.append(k)
            rows.append(r)
    pot.check()
    return atom, thermo.cpu().numpy(), np.array(kappa), np.array(rows)


def group(mg, s, grid, ensemble, T, skin=1.0, graph=True):
    return mg.DomainGroup(s["h"], s["pbc"], grid, NEP, ensemble=ensemble, temperature=T, temperature_coupling=100.0,
                          time_step=DT, skin=skin, cuda_graph=graph)


def state(g):
    out = g.gather_local()
    return dict(out, thermo=g.thermo())


# ---------------------------------------------------------------- one block is the library

@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("ensemble", ["nvt_ber", "nvt_nhc"])
def test_one_block_is_the_single_domain_library(mg, ensemble, graph):
    """1x1x1, skin 5 (no exchange): the same kernels in the same order on the same atom order as the
    single-domain engine with the drive and the heat sums, so every output is bit-identical after 100 steps."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    n = s["type"].shape[0]
    T = 300.0
    g = group(mg, s, (1, 1, 1), ensemble, T, skin=5.0, graph=graph)
    g.distribute(s["type"], wrapped_positions(s), s["mass"], init_velocities(s["mass"], T, seed=42))
    g.set_hnemd(OI, FE, max_intervals=10)
    g.run(100, check_every=5)
    g.check()
    assert g.migrations == 0
    kappa, rows = g.hnemd_take(T)
    out = state(g)
    atom, th, k_ref, r_ref = engine_run(s, 100, T, ensemble)
    theirs = dict(pos=atom.position_per_atom, vel=atom.velocity_per_atom, force=atom.force_per_atom,
                  virial=atom.virial_per_atom, pe=atom.potential_per_atom)
    for k, v in theirs.items():
        assert np.array_equal(out[k], v.cpu().numpy().reshape(out[k].shape)), k
    assert np.array_equal(out["thermo"][:2], th[:2])
    assert kappa.shape == (10, 5) and rows.shape == (10, OI, 5)
    assert np.array_equal(rows, r_ref)
    assert np.array_equal(kappa, k_ref)


# ---------------------------------------------------------------- the reference's HNEMD run

def read_thermo(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#")], dtype=np.float64)


@pytest.mark.parametrize("grid", [(2, 2, 2), (4, 1, 1)], ids=["222", "411"])
def test_blocks_track_the_reference_hnemd_run(mg, grid):
    """The unmodified reference's PbTe HNEMD run (refgpu_hnemd_pbte_*: nvt_ber 300 K, compute_hnemd 10
    0.00002 0 0, 250 steps), within the tolerances the single-GPU driver meets against it."""
    if not (GOLDEN / "refgpu_hnemd_pbte_kappa.out").exists():
        pytest.skip("refgpu_hnemd_pbte_* not generated yet")
    s = rocksalt_pbte(12, rattle=0.02, seed=31)
    g = group(mg, s, grid, "nvt_ber", 300.0)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=42))
    g.set_hnemd(10, (0.00002, 0.0, 0.0), max_intervals=25)
    mine = []
    for _ in range(25):
        g.run(10, check_every=5)
        mine.append(g.thermo())
    g.check()
    k_mine, _ = g.hnemd_take(300.0)
    ref = read_thermo(GOLDEN / "refgpu_hnemd_pbte_thermo.out")
    mine = np.array(mine)
    for k in range(25):
        tol = 2e-5 * (1 + k)
        assert abs(mine[k, 0] - ref[k, 0]) < tol * 10 * 300.0, (k, mine[k, 0], ref[k, 0])
        assert abs(mine[k, 1] - ref[k, 2]) < tol * abs(ref[k, 2]), (k, mine[k, 1], ref[k, 2])
    k_ref = np.loadtxt(GOLDEN / "refgpu_hnemd_pbte_kappa.out")
    assert k_mine.shape == k_ref.shape == (25, 5)
    assert np.allclose(k_mine, k_ref, rtol=0, atol=2e-2 * np.abs(k_ref).max()), np.abs(k_mine - k_ref).max()


# ---------------------------------------------------------------- migrations

def test_blocks_follow_the_single_domain_hnemd_run(mg):
    """900 K, skin 1 A, 2x2x2, 200 steps with migrations: thermo within the trajectory tolerances of the
    undriven blocks, kappa within those of the reference pin, and the driven forces still sum to zero."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    n = s["type"].shape[0]
    T = 900.0
    g = group(mg, s, (2, 2, 2), "nvt_ber", T)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], T, seed=42))
    g.set_hnemd(OI, FE, max_intervals=20)
    g.run(200, check_every=5)
    g.check()
    assert g.migrations >= 1
    kappa, _ = g.hnemd_take(T)
    out = state(g)
    assert np.array_equal(out["id"], np.arange(n))
    _, th, k_ref, _ = engine_run(s, 200, T, "nvt_ber")
    assert abs(out["thermo"][0] - th[0]) < 0.05 and abs(out["thermo"][1] - th[1]) < 2e-6 * n
    assert kappa.shape == k_ref.shape == (20, 5)
    assert np.allclose(kappa, k_ref, rtol=0, atol=2e-2 * np.abs(k_ref).max()), np.abs(kappa - k_ref).max()
    f = out["force"]
    assert np.abs(f.sum(axis=1)).max() <= 1e-12 * np.abs(f).sum()


# ---------------------------------------------------------------- CUDA graph

@pytest.mark.parametrize("grid", [(2, 2, 1), (4, 1, 1)], ids=["221", "411"])
def test_graph_replay_across_exchanges_is_bit_identical(mg, grid):
    """900 K, skin 1 A, nvt_nhc, 200 steps: every exchange re-captures the step with the drive and the heat
    row inside it; the state, thermo, heat rows and kappa match eager launches bit for bit."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 900.0, seed=42)
    res = []
    for graph in (False, True):
        g = group(mg, s, grid, "nvt_nhc", 900.0, graph=graph)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        g.set_hnemd(OI, FE, max_intervals=20)
        g.run(200, check_every=5)
        g.check()
        assert g.migrations >= 1
        res.append((g.migrations, g.hnemd_take(900.0), state(g)))
    assert res[0][0] == res[1][0]
    assert res[0][1][0].shape == (20, 5)
    assert np.array_equal(res[0][1][0], res[1][1][0]) and np.array_equal(res[0][1][1], res[1][1][1])
    for k in ("pos", "vel", "force", "virial", "pe", "thermo"):
        assert np.array_equal(res[0][2][k], res[1][2][k]), k


# ---------------------------------------------------------------- blocks that own no atoms

def empty_block_hnemd_checks():
    """Body of test_blocks_that_own_no_atoms (run in a child process)."""
    from gpumd_b200 import mgpu
    from test_gpu_mgpu import vacuum_slab
    s = vacuum_slab()
    n = s["type"].shape[0]
    vel = init_velocities(s["mass"], 300.0, seed=42)
    res = {}
    for grid in ((4, 1, 1), (1, 1, 1)):
        g = mgpu.DomainGroup(s["h"], s["pbc"], grid, NEP, ensemble="nvt_ber", temperature=300.0,
                             temperature_coupling=100.0, time_step=DT, skin=1.0, cuda_graph=True)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        if grid == (4, 1, 1):
            assert [g.info(1, k) for k in range(4)] == [n, 0, 0, 0] and g.info(2, 2) == 0
        g.set_hnemd(OI, FE, max_intervals=10)
        g.run(100, check_every=5)
        g.check()
        res[grid] = (g.hnemd_take(300.0)[0], g.gather_local())
    (k4, o4), (k1, o1) = res[(4, 1, 1)], res[(1, 1, 1)]
    assert k4.shape == k1.shape == (10, 5)
    assert np.abs(o4["pos"] - o1["pos"]).max() < 1e-5
    assert np.allclose(k4, k1, rtol=0, atol=2e-2 * np.abs(k1).max()), np.abs(k4 - k1).max()
    print("empty blocks: ok")


def test_blocks_that_own_no_atoms(mg):
    """The vacuum slab of test_gpu_mgpu.py on 4x1x1 (blocks that own no atoms, one that holds none) with
    HNEMD: no launch error, kappa as on one block.  A child process: a failed launch would leave an error
    that every later launch check of the process reports."""
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_gpu_mgpu_hnemd; "
            "test_gpu_mgpu_hnemd.empty_block_hnemd_checks()")
    r = subprocess.run([sys.executable, "-c", code, str(ROOT), str(ROOT / "tests")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "empty blocks: ok" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


# ---------------------------------------------------------------- take semantics

def test_take_returns_the_intervals_finished_since_the_last_one(mg):
    """run(15) take run(5) take == run(20) take, bit for bit; an overflowing run is refused before it
    launches anything, so the group goes on exactly as if it had not been called."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 300.0, seed=42)

    def fresh(max_intervals):
        g = group(mg, s, (2, 1, 1), "nvt_nhc", 300.0)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        g.set_hnemd(OI, FE, max_intervals=max_intervals)
        return g

    a = fresh(4)
    a.run(15)
    k1, r1 = a.hnemd_take(300.0)
    a.run(5)
    k2, r2 = a.hnemd_take(300.0)
    assert k1.shape == k2.shape == (1, 5) and r1.shape == (1, OI, 5)
    b = fresh(4)
    b.run(20)
    kb, rb = b.hnemd_take(300.0)
    assert kb.shape == (2, 5)
    assert np.array_equal(np.concatenate([k1, k2]), kb) and np.array_equal(np.concatenate([r1, r2]), rb)
    assert b.hnemd_take(300.0)[0].shape == (0, 5)  # nothing finished since
    c = fresh(2)
    c.run(15)
    before = state(c)
    with pytest.raises(mg.MgpuError, match="max_intervals"):
        c.run(15)  # 30 steps: 3 intervals untaken
    after = state(c)
    for k in ("pos", "vel", "force", "thermo"):
        assert np.array_equal(before[k], after[k]), k
    c.run(5)
    kc, rc = c.hnemd_take(300.0)
    assert np.array_equal(kc, kb) and np.array_equal(rc, rb)
    for k in ("pos", "vel", "force", "virial", "pe", "thermo"):
        assert np.array_equal(state(c)[k], state(b)[k]), k


def test_set_drives_the_forces_at_the_current_positions(mg):
    """After distribute, set re-evaluates the forces with the drive: on 2x2x2 the blocks' forces are the
    restatement's drive of their undriven forces and virials (one global net force removed); on 1x1x1 they
    are the single-domain engine's driven forces bit for bit."""
    from gpumd_b200 import engine
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    n = s["type"].shape[0]
    fe = (2e-3, -1e-3, 5e-4)
    g = group(mg, s, (2, 2, 2), "nvt_ber", 300.0)
    g.distribute(s["type"], s["pos"], s["mass"])
    before = g.gather_local()
    g.set_hnemd(OI, fe)
    after = g.gather_local()
    assert np.array_equal(after["virial"], before["virial"]) and np.array_equal(after["pe"], before["pe"])
    want = ho.hnemd_drive(before["virial"], before["force"], fe)
    assert np.allclose(after["force"], want, rtol=1e-13, atol=1e-13 * np.abs(want).max())
    assert np.abs(after["force"].sum(axis=1)).max() <= 1e-12 * np.abs(after["force"]).sum()

    one = group(mg, s, (1, 1, 1), "nvt_ber", 300.0, skin=5.0)
    one.distribute(s["type"], wrapped_positions(s), s["mass"])
    one.set_hnemd(OI, fe)
    atom, box = engine.Atom(s["type"], s["pos"], s["mass"]), engine.Box(s["h"], s["pbc"])
    force = engine.Force()
    force.parse_potential(NEP, n)
    force.set_hnemd(fe)
    force.compute(box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
                  atom.virial_per_atom)
    assert np.array_equal(one.gather_local()["force"], atom.force_per_atom.cpu().numpy().reshape(3, n))


def test_zero_fe_is_a_group_that_never_had_hnemd(mg):
    """set with fe = 0 switches the drive and the heat row off: the next steps are bit-identical to a group
    that never had HNEMD, with the same launches per step (eager, so that every step is counted)."""
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    vel = init_velocities(s["mass"], 900.0, seed=42)

    def run(fes, steps):
        g = group(mg, s, (2, 2, 1), "nvt_nhc", 900.0, graph=False)
        g.distribute(s["type"], s["pos"], s["mass"], vel)
        for fe in fes:
            g.set_hnemd(OI, fe)
        g.run(steps, check_every=5)
        g.check()
        return g

    zero = (0.0, 0.0, 0.0)
    assert run([FE], 1).launches_per_step > run([], 1).launches_per_step
    plain, switched = run([], 60), run([FE, zero], 60)
    with pytest.raises(mg.MgpuError, match="HNEMD is off"):
        switched.hnemd_take(900.0)
    assert plain.launches_per_step == switched.launches_per_step
    assert plain.migrations == switched.migrations
    a, b = state(plain), state(switched)
    for k in ("pos", "vel", "force", "virial", "pe", "thermo"):
        assert np.array_equal(a[k], b[k]), k


def test_bad_arguments_are_refused(mg):
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    g = group(mg, s, (2, 1, 1), "nvt_ber", 300.0)
    with pytest.raises(mg.MgpuError, match="distribute first"):
        g.set_hnemd(OI, FE)
    g.distribute(s["type"], s["pos"], s["mass"])
    for oi, fe, mx in ((0, FE, 10), (-1, FE, 10), (OI, FE, 0), (OI, (np.nan, 0.0, 0.0), 10),
                       (OI, (0.0, np.inf, 0.0), 10), (OI, (0.0, 0.0, -np.inf), 10), (1 << 20, FE, 1 << 20)):
        with pytest.raises(mg.MgpuError):
            g.set_hnemd(oi, fe, max_intervals=mx)
    with pytest.raises(mg.MgpuError, match="HNEMD is off"):
        g.hnemd_take(300.0)
    g.set_hnemd(OI, FE, max_intervals=1)
    for T in (0.0, -1.0, np.nan):
        with pytest.raises(mg.MgpuError, match="temperature"):
            g.hnemd_take(T)
    g.run(19)  # one whole interval and a partial one: the most max_intervals = 1 admits
    with pytest.raises(mg.MgpuError, match="max_intervals"):
        g.run(1)
    assert g.hnemd_take(300.0)[0].shape == (1, 5)


# ---------------------------------------------------------------- two ranks over NCCL

WORKER = r"""
import os, sys
import numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2_ROOT"])
from gpumd_b200 import mgpu
from gpumd_b200.structures import TIME_UNIT_CONVERSION, init_velocities, rocksalt_pbte
rank = int(os.environ["RANK"]); torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("nccl")
s = rocksalt_pbte(12, rattle=0.02, seed=1)
g = mgpu.DomainGroup(s["h"], s["pbc"], (2, 1, 1), os.environ["B2_MODEL"], ensemble="nvt_nhc", temperature=300.0,
                     temperature_coupling=100.0, time_step=1.0 / TIME_UNIT_CONVERSION, skin=1.0, cuda_graph=True,
                     distributed=True)
g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=42))
g.set_hnemd(10, (2e-5, 0.0, 0.0), max_intervals=10)
g.run(100, check_every=5); g.check()
kappa, rows = g.hnemd_take(300.0)
np.savez(os.path.join(os.environ["B2_OUT"], f"rank{rank}.npz"), kappa=kappa, rows=rows, **g.owned(0))
dist.barrier(); dist.destroy_process_group()
"""


def test_two_ranks_over_nccl_match_the_local_run(mg, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    (tmp_path / "worker.py").write_text(WORKER)
    env = dict(os.environ, B2_ROOT=str(ROOT), B2_MODEL=str(NEP), B2_OUT=str(tmp_path))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", "29534", str(tmp_path / "worker.py")],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    parts = [np.load(tmp_path / f"rank{k}.npz") for k in range(2)]
    s = rocksalt_pbte(12, rattle=0.02, seed=1)
    g = group(mg, s, (2, 1, 1), "nvt_nhc", 300.0)
    g.distribute(s["type"], s["pos"], s["mass"], init_velocities(s["mass"], 300.0, seed=42))
    g.set_hnemd(10, (2e-5, 0.0, 0.0), max_intervals=10)
    g.run(100, check_every=5)
    kappa, rows = g.hnemd_take(300.0)
    for p in parts:  # every rank takes the global sums
        assert np.array_equal(p["kappa"], kappa) and np.array_equal(p["rows"], rows)
    ids = np.concatenate([p["id"] for p in parts])
    pos = np.concatenate([p["pos"] for p in parts], axis=1)[:, np.argsort(ids)]
    assert np.array_equal(pos, g.gather_local()["pos"])

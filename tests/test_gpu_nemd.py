"""Direct NEMD on the device: the heat_lan / heat_nhc / heat_bdp baths and the group-averaged `compute`
against the numpy restatements of tests/nemd_oracle.py, determinism, CUDA-graph capture, and the
`b200md` driver on the reference's graphene_kappa_nemd case."""
import shutil
import subprocess

import numpy as np
import pytest

import nemd_oracle as no
from conftest import GOLDEN
from gpumd_b200.structures import TIME_UNIT_CONVERSION, graphene_sheet, init_velocities, write_xyz

pytestmark = pytest.mark.gpu
DT = 1.0 / TIME_UNIT_CONVERSION


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def _state(eng, n, seed, groups):
    rng = np.random.default_rng(seed)
    mass = rng.uniform(10.0, 200.0, n)
    vel = rng.normal(size=(3, n)) * 0.05
    atom = eng.Atom(np.zeros(n, np.int32), rng.uniform(0, 50, (3, n)), mass, vel)
    atom.potential_per_atom.copy_(eng.torch.as_tensor(rng.normal(size=n) - 4.0))
    atom.force_per_atom.copy_(eng.torch.as_tensor(rng.normal(size=3 * n)))
    atom.virial_per_atom.copy_(eng.torch.as_tensor(rng.normal(size=9 * n)))
    label = rng.integers(0, groups, n).astype(np.int32)
    return atom, mass, label


def _host(atom):
    return [t.cpu().numpy() for t in (atom.mass, atom.potential_per_atom, atom.force_per_atom,
                                      atom.virial_per_atom, atom.velocity_per_atom)]


@pytest.mark.parametrize("groups,n", [(1, 5000), (9, 300_000), (1500, 100_000)])
def test_compute_matches_group_sums(eng, groups, n):
    atom, mass, label = _state(eng, n, groups, groups)
    label[label % 7 == 3] = 0  # some empty groups (with 9 or 1500 groups)
    label[-1] = groups - 1     # the last group keeps the group count
    comp = eng.Compute(label, 2, 3, no.QUANTITIES)
    assert comp.num_columns == 23
    cols = no.per_atom_columns(*_host(atom))
    sizes = np.bincount(label, minlength=groups)
    for step in range(5):  # samples after steps 1, 3, 5; output after the third
        assert comp.process(step, atom) is None
    out = comp.process(5, atom)
    ref = no.group_sums(label, groups, cols)  # three identical samples
    ref[0] /= np.where(sizes > 0, sizes, np.nan)
    assert out.shape == (23, groups)
    empty = sizes == 0
    assert np.all(np.isnan(out[0, empty])) and np.all(out[1:, empty] == 0)
    assert np.allclose(out[:, ~empty], ref[:, ~empty], rtol=1e-12, atol=1e-12 * np.abs(ref[:, ~empty]).max())


def test_compute_selects_columns_in_the_reference_order(eng):
    atom, _, label = _state(eng, 3000, 5, 4)
    comp = eng.Compute(label, 1, 1, ["momentum", "jk", "temperature"])
    out = comp.process(0, atom)
    ref = no.group_sums(label, 4, no.per_atom_columns(*_host(atom)))[no.select(["temperature", "jk", "momentum"])]
    ref[0] /= np.bincount(label, minlength=4)
    assert out.shape == (7, 4) and np.allclose(out, ref, rtol=1e-12)


def test_compute_is_deterministic(eng):
    atom, _, label = _state(eng, 200_000, 8, 9)
    a = eng.Compute(label, 1, 1, no.QUANTITIES).process(0, atom)
    b = eng.Compute(label, 1, 1, no.QUANTITIES).process(0, atom)
    assert np.array_equal(a, b)


def _slabs(n, groups=6):
    return (np.arange(n) * groups // n).astype(np.int32)


def test_heat_nhc_matches_restatement_step_by_step(eng):
    n, src, snk, T, Tc, dT = 6000, 1, 4, 300.0, 100.0, 20.0
    atom, mass, _ = _state(eng, n, 11, 1)
    label = _slabs(n)
    ens = eng.Ensemble_HEAT_NHC(label, src, snk, T, Tc, dT, DT)
    idx = [np.flatnonzero(label == g) for g in (src, snk)]
    chains = [no.nhc_init(no.K_B * temp, DT * Tc, 3.0 * i.shape[0]) for i, temp in zip(idx, (T + dT, T - dT))]
    energy = np.zeros(2)
    v = atom.velocity_per_atom.cpu().numpy().reshape(3, n).copy()
    for k in range(6):
        ens.half(k % 2, atom)
        for g in range(2):
            vc, ek2 = no.vc_and_ke(mass, v, idx[g])
            kT = no.K_B * (T + dT if g == 0 else T - dT)
            f = no.nhc_chain(chains[g], ek2, 3.0 * idx[g].shape[0], kT, 0.5 * DT)
            energy[g] += ek2 * 0.5 * (1 - f * f)
            v[:, idx[g]] = vc[:, None] + f * (v[:, idx[g]] - vc[:, None])
        st = ens.state()
        for g in range(2):
            assert np.allclose(st["chain"][g], chains[g], rtol=1e-10, atol=1e-14)
        assert np.allclose(st["energy"], energy, rtol=1e-9, atol=1e-14)
        assert np.allclose(atom.velocity_per_atom.cpu().numpy().reshape(3, n), v, rtol=1e-12, atol=1e-15)


def test_heat_bdp_factors_follow_the_mt19937_stream(eng):
    n, src, snk, T, Tc, dT = 6000, 0, 5, 300.0, 100.0, 30.0
    atom, mass, _ = _state(eng, n, 12, 1)
    label = _slabs(n)
    ens = eng.Ensemble_HEAT_BDP(label, src, snk, T, Tc, dT)
    mt = no.BdpOracle(12345678)
    idx = [np.flatnonzero(label == g) for g in (src, snk)]
    energy = np.zeros(2)
    v = atom.velocity_per_atom.cpu().numpy().reshape(3, n).copy()
    for _ in range(5):
        ens.half(0, atom)  # before step 1: nothing
        ens.half(1, atom)
        for g, (vc, f, de) in enumerate(no.bdp_factors(mt, mass, v, idx[0], idx[1], T, dT, Tc)):
            energy[g] += de
            v[:, idx[g]] = vc[:, None] + f * (v[:, idx[g]] - vc[:, None])
        assert np.allclose(ens.energy_transferred(), energy, rtol=1e-9)
        assert np.allclose(atom.velocity_per_atom.cpu().numpy().reshape(3, n), v, rtol=1e-11, atol=1e-15)


def test_heat_lan_without_noise_only_accounts(eng):
    n = 4000
    atom, _, _ = _state(eng, n, 13, 1)
    v0 = atom.velocity_per_atom.clone()
    ens = eng.Ensemble_HEAT_LAN(_slabs(n), 1, 3, 300.0, 1e300, 10.0)  # c1 = 1, c2 = 0
    for k in range(4):
        ens.half(k % 2, atom)
    assert eng.torch.equal(atom.velocity_per_atom, v0)
    assert np.array_equal(ens.energy_transferred(), [0.0, 0.0])


def test_heat_lan_noise_statistics_and_energy_accounting(eng):
    n, src, snk, T, dT, Tc = 60_000, 1, 4, 300.0, 60.0, 1.0
    atom, mass, _ = _state(eng, n, 14, 1)
    atom.velocity_per_atom.zero_()
    label = _slabs(n)
    ens = eng.Ensemble_HEAT_LAN(label, src, snk, T, Tc, dT)
    ens.half(0, atom)
    v = atom.velocity_per_atom.cpu().numpy().reshape(3, n)
    c1 = np.exp(-0.5 / Tc)
    ke = 0.5 * mass * (v * v).sum(0)
    for g, temp in ((src, T + dT), (snk, T - dT)):
        i = label == g
        t_mean = (2 * ke[i] / (3 * no.K_B)).mean()
        expect = (1 - c1 * c1) * temp
        assert abs(t_mean - expect) < 5 * expect * np.sqrt(2 / 3 / i.sum())
    assert np.all(v[:, (label != src) & (label != snk)] == 0)
    e = ens.energy_transferred()
    assert np.isclose(e[0], -ke[label == src].sum(), rtol=1e-12)
    assert np.isclose(e[1], -ke[label == snk].sum(), rtol=1e-12)
    # a second kick: the total transferred still equals minus the change in bath-group kinetic energy
    ens.half(1, atom)
    v = atom.velocity_per_atom.cpu().numpy().reshape(3, n)
    ke2 = 0.5 * mass * (v * v).sum(0)
    assert np.isclose(ens.energy_transferred().sum(), -ke2[(label == src) | (label == snk)].sum(), rtol=1e-11)


def test_heat_lan_is_deterministic(eng):
    out = []
    for _ in range(2):
        atom, _, _ = _state(eng, 20_000, 15, 1)
        ens = eng.Ensemble_HEAT_LAN(_slabs(20_000), 0, 5, 300.0, 10.0, 30.0)
        for k in range(6):
            ens.half(k % 2, atom)
        out.append((atom.velocity_per_atom.cpu().numpy(), ens.energy_transferred()))
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


@pytest.mark.parametrize("kind", ["LAN", "NHC", "BDP"])
def test_heat_step_and_compute_capture_into_a_cuda_graph(eng, kind):
    """No host synchronisation inside a step: compute1 / compute2 and a compute sample are captured on a
    side stream and replayed; the replay matches the same calls made eagerly."""
    torch = eng.torch
    n = 10_000
    label = _slabs(n)
    box = eng.Box(np.diag([50.0, 50.0, 50.0]).reshape(9))

    def make():
        atom, _, _ = _state(eng, n, 16, 1)
        cls = getattr(eng, f"Ensemble_HEAT_{kind}")
        ens = cls(label, 1, 4, 300.0, 50.0, 20.0, DT) if kind == "NHC" else cls(label, 1, 4, 300.0, 50.0, 20.0)
        return atom, ens, eng.Compute(label, 1, 1, no.QUANTITIES)

    atom_e, ens_e, comp_e = make()
    for _ in range(2):
        ens_e.compute1(DT, box, atom_e)
        ens_e.compute2(DT, box, atom_e)
        comp_e.sample(atom_e)
    atom_g, ens_g, comp_g = make()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ens_g.compute1(DT, box, atom_g)
            ens_g.compute2(DT, box, atom_g)
            comp_g.sample(atom_g)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(atom_g.velocity_per_atom, atom_e.velocity_per_atom)
    assert torch.equal(atom_g.position_per_atom, atom_e.position_per_atom)
    assert np.array_equal(ens_g.energy_transferred(), ens_e.energy_transferred())
    assert np.array_equal(comp_g.take(2), comp_e.take(2))


# ---- the `b200md` driver -----------------------------------------------------------------------

def _run_exe(tmp_path, run_in, timeout=900):
    from gpumd_b200 import build
    exe = build.build_host()
    (tmp_path / "run.in").write_text(run_in)
    return subprocess.run([str(exe)], cwd=tmp_path, capture_output=True, text=True, timeout=timeout)


def _graphene(tmp_path, nx=100, ny=101, vel=True):
    s = graphene_sheet(nx, ny)
    write_xyz(tmp_path / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=42) if vel else None)
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    return s


def test_driver_runs_the_references_graphene_kappa_nemd_case(tmp_path):
    """tests/gpumd/graphene_kappa_nemd/run.in of the reference, unchanged, on the same 40 400-atom sheet
    (velocities from `velocity 300`): file shapes as in its compute1 / shc1 / thermo1.out, the fixed
    group at 0 K, the bath groups near the reference's temperatures and energies."""
    _graphene(tmp_path, vel=False)
    run_in = ("potential potential.txt\nvelocity 300\n\nensemble nvt_ber 300 300 100\nfix 0\ntime_step 1\n"
              "dump_thermo 100\nrun 1000\n\nensemble heat_lan 300 100 10 1 8\nfix 0\n"
              "compute 0 10 100 temperature\ncompute_shc 2 250 1 1000 400.0 group 0 4\nrun 1000\n")
    r = _run_exe(tmp_path, run_in)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ref_c = np.loadtxt(GOLDEN / "ref_graphene_nemd_compute1.out").reshape(1, -1)
    mine_c = np.loadtxt(tmp_path / "compute.out").reshape(1, -1)
    assert mine_c.shape == ref_c.shape == (1, 11)
    thermo = [ln for ln in open(tmp_path / "thermo.out") if not ln.startswith("#")]
    ref_t = [ln for ln in open(GOLDEN / "ref_graphene_nemd_thermo1.out") if not ln.startswith("#")]
    assert len(thermo) == len(ref_t) == 10
    shc = [ln for ln in open(tmp_path / "shc.out") if not ln.startswith("#") and ln.strip()]
    ref_s = [ln for ln in open(GOLDEN / "ref_graphene_nemd_shc1.out") if not ln.startswith("#") and ln.strip()]
    assert len(shc) == len(ref_s)
    t = mine_c[0]
    print("compute.out:", " ".join(f"{x:.4g}" for x in t), "| reference:", " ".join(f"{x:.4g}" for x in ref_c[0]))
    assert t[0] == 0.0
    assert abs(t[1] - 308.8255) < 3.0 and abs(t[8] - 290.608) < 3.0
    assert abs(t[9] - ref_c[0, 9]) < 0.15 * abs(ref_c[0, 9]) and abs(t[10] - ref_c[0, 10]) < 0.15 * abs(ref_c[0, 10])


def test_driver_heat_bdp_and_nhc_with_all_compute_columns(tmp_path):
    _graphene(tmp_path, 10, 91)
    for kind in ("nhc", "bdp"):
        d = tmp_path / kind
        d.mkdir()
        shutil.copyfile(tmp_path / "model.xyz", d / "model.xyz")
        shutil.copyfile(tmp_path / "potential.txt", d / "potential.txt")
        r = _run_exe(d, f"potential potential.txt\nensemble heat_{kind} 300 100 10 1 8\nfix 0\ntime_step 1\n"
                        "compute 0 10 10 temperature potential force virial jp jk momentum\nrun 300\n"
                        "ensemble nve\nrun 20\n")
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        c = np.loadtxt(d / "compute.out")
        assert c.shape == (3, 23 * 9 + 2)  # the second run has no `compute` (reset after a run)
        assert np.all(c[:, 0] == 0.0) and np.all(np.isfinite(c)) and np.all(c[:, -2:] != 0.0)


def test_driver_heat_lan_with_a_moving_group(tmp_path):
    s = _graphene(tmp_path, 10, 91)
    r = _run_exe(tmp_path, "potential potential.txt\nensemble heat_lan 300 100 10 2 5\nfix 0\n"
                           "move 8 0 0.001 0\ntime_step 1\ncompute 0 5 4 temperature jp jk\nrun 100\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    c = np.loadtxt(tmp_path / "compute.out")
    assert c.shape == (5, 7 * 9 + 2) and np.all(c[:, 0] == 0) and np.all(c[:, 8] == 0)
    assert s["group"].max() == 8


@pytest.mark.parametrize("line,msg", [
    ("ensemble heat_lan 300 100 10 1", "ensemble heat_lan should have 5 parameters."),
    ("ensemble heat_nhc 0 100 10 1 8", "Temperature should > 0."),
    ("ensemble heat_bdp 300 0.5 10 1 8", "Temperature coupling should >= 1."),
    ("ensemble heat_lan 300 100 300 1 8", "|Temperature difference| is too large."),
    ("ensemble heat_lan 300 100 10 x 8", "Group ID for heat source should be an integer."),
    ("ensemble heat_lan 300 100 10 3 3", "Source and sink cannot be the same group."),
    ("ensemble heat_lan 300 100 10 -1 3", "Group ID for heat source should >= 0."),
    ("ensemble heat_lan 300 100 10 1 9", "Group ID for heat sink should < #groups."),
    ("ensemble heat_nhc 300 100 10 1 8\nfix 0\nmove 2 0 0 0\nrun 10", "only allowed to use"),
    ("compute 0 10", "compute should have at least 4 parameters."),
    ("compute 1 10 10 temperature", "grouping method exceeds the bound."),
    ("compute 0 0 10 temperature", "sampling interval of compute should > 0."),
    ("compute 0 10 x temperature", "output interval of compute should be integer."),
    ("compute 0 10 10 heat", "Invalid property for compute."),
])
def test_driver_rejects_bad_nemd_input(tmp_path, line, msg):
    _graphene(tmp_path, 10, 91)
    r = _run_exe(tmp_path, f"potential potential.txt\n{line}\n", timeout=120)
    assert r.returncode == 1 and "Input Error" in r.stderr and msg in r.stderr, r.stderr


def test_driver_heat_bath_needs_a_grouping_method(tmp_path):
    s = graphene_sheet(10, 11)
    s.pop("group")
    write_xyz(tmp_path / "model.xyz", s, ["C"])
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\nensemble heat_lan 300 100 10 1 2\n", timeout=120)
    assert r.returncode == 1 and "Cannot heat/cold without grouping method." in r.stderr, r.stderr


def test_driver_seeded_heat_lan_run_is_deterministic(tmp_path):
    outs = []
    for k in range(2):
        d = tmp_path / str(k)
        d.mkdir()
        _graphene(d, 10, 91)
        r = _run_exe(d, "potential potential.txt\nensemble heat_lan 300 100 10 1 8\nfix 0\ntime_step 1\n"
                        "compute 0 10 10 temperature potential jp jk\nrun 200\n")
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append((d / "compute.out").read_text())
    assert outs[0] == outs[1]


# ---- the driver against the unmodified reference gpumd (scripts/run_reference_gpumd.py, nemd_* cases) ----

def _reference_runs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("run_reference_gpumd",
                                                  GOLDEN.parent.parent / "scripts" / "run_reference_gpumd.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.NEMD_GRAPHENE_RUN, mod.NEMD_PBTE_RUN


def _rows(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#") and ln.strip()], dtype=np.float64)


def _compute_gap(mine, ref, widths, num_groups):
    """Largest |mine - ref| of each column block (widths x num_groups columns, then the two energies),
    relative to the largest |ref| of that block."""
    gaps, c = [], 0
    for k in [w * num_groups for w in widths] + [2]:
        blk = slice(c, c + k)
        gaps.append(np.abs(mine[:, blk] - ref[:, blk]).max() / np.abs(ref[:, blk]).max())
        c += k
    assert c == ref.shape[1]
    return np.array(gaps)


@pytest.mark.parametrize("kind", ["lan", "nhc", "bdp"])
def test_driver_graphene_nemd_matches_reference(tmp_path, kind):
    """FP64 Tersoff, 200 nvt_ber steps then 600 heat_<kind> steps with every `compute` quantity and SHC,
    against the reference gpumd on the same inputs: thermo.out (including the stale rows a heat run
    prints), compute.out and shc.out.  heat_lan uses the reference's next two rand() values, heat_bdp the
    -DDEBUG MT19937 seed (B200MD_DEBUG_SEED)."""
    import os
    graphene_run, _ = _reference_runs()
    s = graphene_sheet()
    write_xyz(tmp_path / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    from gpumd_b200 import build
    (tmp_path / "run.in").write_text("potential potential.txt\n" + graphene_run.format(kind=kind))
    r = subprocess.run([str(build.build_host())], cwd=tmp_path, capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, B200MD_DEBUG_SEED="1"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    ref = f"refgpu_nemd_graphene_{kind}"
    t_mine, t_ref = _rows(tmp_path / "thermo.out"), _rows(GOLDEN / f"{ref}_thermo.out")
    assert t_mine.shape == t_ref.shape == (26, 18)
    assert np.all(t_ref[20:] == t_ref[19]) and np.all(t_mine[20:] == t_mine[19])  # stale during the heat run
    assert np.allclose(t_mine[:, :3], t_ref[:, :3], rtol=1e-5, atol=1e-6 * np.abs(t_ref[:, :3]).max())
    c_mine, c_ref = _rows(tmp_path / "compute.out"), _rows(GOLDEN / f"{ref}_compute.out")
    assert c_mine.shape == c_ref.shape == (6, 23 * 9 + 2)
    assert np.all(c_mine[:, 0] == 0.0) and np.all(c_ref[:, 0] == 0.0)  # the fixed group
    gap = _compute_gap(c_mine, c_ref, (1, 1, 3, 9, 3, 3, 3), 9)
    print(f"{kind}: compute.out gap per block (T U f W jp jk p E):", " ".join(f"{g:.2e}" for g in gap))
    assert np.allclose(c_mine[:, :9], c_ref[:, :9], rtol=1e-5, atol=0)  # group temperatures
    assert np.all(gap < 1e-5)
    s_mine, s_ref = _rows(tmp_path / "shc.out"), _rows(GOLDEN / f"{ref}_shc.out")
    assert s_mine.shape == s_ref.shape == (399, 3)
    assert np.array_equal(s_mine[:, 0], s_ref[:, 0])
    assert np.allclose(s_mine[:, 1:], s_ref[:, 1:], rtol=1e-4, atol=1e-5 * np.abs(s_ref[:, 1:]).max())


def test_driver_pbte_nemd_with_fix_and_move_matches_reference(tmp_path):
    """FP32 NEP, six slabs along x: nvt_ber, then heat_lan with slab 0 fixed and slab 1 moving, `compute`
    of temperature, jp and jk, against the reference gpumd within 2 % of each block's largest value."""
    from gpumd_b200.structures import nep_type_order, rocksalt_pbte
    _, pbte_run = _reference_runs()
    s = rocksalt_pbte(12, rattle=0.02, seed=32)
    s["group"] = np.minimum((s["pos"][0] / s["h"][0] * 6).astype(np.int32), 5)
    write_xyz(tmp_path / "model.xyz", s, nep_type_order(GOLDEN / "nep_PbTe.txt"),
              init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "nep_PbTe.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\n" + pbte_run)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    t_mine, t_ref = _rows(tmp_path / "thermo.out"), _rows(GOLDEN / "refgpu_nemd_pbte_lan_thermo.out")
    assert t_mine.shape == t_ref.shape == (10, 18)
    assert np.allclose(t_mine[:, :3], t_ref[:, :3], rtol=2e-3)
    c_mine, c_ref = _rows(tmp_path / "compute.out"), _rows(GOLDEN / "refgpu_nemd_pbte_lan_compute.out")
    assert c_mine.shape == c_ref.shape == (3, 7 * 6 + 2)
    assert np.all(c_mine[:, [0, 1]] == 0.0) and np.all(c_ref[:, [0, 1]] == 0.0)  # fixed and moving slabs
    gap = _compute_gap(c_mine, c_ref, (1, 3, 3), 6)
    print("pbte: compute.out gap per block (T jp jk E):", " ".join(f"{g:.2e}" for g in gap))
    assert np.all(gap < 0.02)

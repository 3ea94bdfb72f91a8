"""The benchmark workloads on the device, every atom against the tiled oracle (tests/fullsize.py), and the
cell, brick and type-tile scans at their exact tile boundaries.

The systems are built as bench.py builds them (its constructors are restated here, with the atom counts
asserted): C3 PbTe NEP 50^3 cells, C2 LJ argon 63^3 cells, C5 Tersoff Si per GPU and at 63^3 cells, C4
UNEP-v1 per GPU, and the 2-GPU PbTe / Si arms as block domains in local mode.  At these sizes the list
build runs paths the small exact tests reach once or never:
  * k_scan_cells (block_scan_1024) carries its sum across tiles of 4096 cells: C3 has 73^3 = 389 017
    cells, about 95 tiles;
  * k_brick_scan uses the same scan over the warp-schedule bricks: C3 has 7 x 37 x 37 = 9 583;
  * k_tile_scan carries its sum across groups of 32 blocks of 256 atoms: C4 has 3 969 blocks.
`test_reach` restates make_grid and b2_make_bricks to show that every case gets there.

Outputs are compared per atom: NEP with the FP32 oracle under check_fv and with the FP64 oracle widened
by the FP32 oracle's own distance from it (the check_nep convention), plus its radial and angular lists
bit for bit; LJ with the FP32 oracle; Tersoff (FP64 throughout) at rtol 1e-9.  The totals of energy and
virial, and the thermo vector of the device state, are compared with float64 sums of the oracle outputs.

The small seam cases (dilute, so that the whole-system oracle stays cheap) hit 4095 / 4096 / 4097 / 8192 /
8193 cells, 4095 / 4096 / 4097 bricks, and 8191 / 8192 / 8193 / 16385 atoms (32 / 32 / 33 / 65 blocks of
type-tile counts)."""
import math

import numpy as np
import pytest

import cases_classical as cc
import fullsize
from conftest import GOLDEN, TOL, assert_close
from gpumd_b200.structures import (TIME_UNIT_CONVERSION, diamond, fcc, init_velocities, nep_type_order,
                                   rocksalt_pbte)
from test_classical_cpu import check_vs_oracle
from test_gpu_nep_schedule import Dev, check_schedule
from test_gpu_nep_species import check_tile_rule
from test_kernel_bodies_cpu import check_fv, check_nep

pytestmark = pytest.mark.gpu

PBTE = GOLDEN / "nep_PbTe.txt"
UNEP = GOLDEN / "nep_UNEP_v1.txt"
SKIN = 1.0        # Neighbor::skin of the single-GPU potentials
DOMAIN_SKIN = 3.0  # bench.py's ghost-list skin of the block domains
TIMES = {}        # oracle wall times, printed at the end of the module
PEAK = {}         # device memory in use (all processes) above the free memory a case started from, GiB


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    yield engine
    fullsize.shutdown()
    if TIMES:
        print("\ntiled oracle, %d workers: " % fullsize.num_workers()
              + ", ".join(f"{k} {v:.1f} s" for k, v in TIMES.items()))
    if PEAK:
        print("device memory used per case: " + ", ".join(f"{k} {v:.1f} GiB" for k, v in PEAK.items()))


@pytest.fixture(scope="module")
def mg(eng):
    from gpumd_b200 import build, mgpu
    build.build_mgpu()
    return mgpu


_START = {}


def need_memory(gib, tag):
    """The GPU is shared: skip, saying why, when fewer than `gib` GiB are free."""
    import torch
    free, total = torch.cuda.mem_get_info()
    if free < gib * 2**30:
        pytest.skip(f"needs {gib} GiB of device memory, {free / 2**30:.1f} of {total / 2**30:.1f} GiB free")
    _START[tag] = free


def note_memory(tag):
    import torch
    torch.cuda.synchronize()
    used = (_START[tag] - torch.cuda.mem_get_info()[0]) / 2**30
    PEAK[tag] = max(PEAK.get(tag, 0.0), used)


def tiled(tag, pot, s, pos, lists=False):
    r = fullsize.evaluate(pot, s["type"], s["h"], s["pbc"], pos, lists=lists)
    TIMES[tag] = TIMES.get(tag, 0.0) + r["seconds"]
    return r


# ---------------------------------------------------------------- the bench systems (bench.py, restated)

def bench_pbte(cells=50):
    """bench.crystal: rocksalt PbTe, rattle 0.02, 300 K."""
    s = rocksalt_pbte(cells, rattle=0.02, seed=1)
    s["vel"] = init_velocities(s["mass"], 300.0, seed=42)
    return s


def bench_side(workload, reps):
    """bench.side_structure for one GPU (world = 1) or for the x-slabs of `reps[0] / 16` GPUs."""
    if workload == "lj":
        s, T0 = fcc(reps, 5.30, rattle=0.0, seed=1), 80.0
    elif workload == "unep":
        s, T0 = fcc(reps, 3.9, rattle=0.0, seed=7, num_types=16, symbols=nep_type_order(UNEP)), 300.0
    else:
        s, T0 = diamond(reps, a=5.431, rattle=0.0, seed=1), 300.0
    s["vel"] = init_velocities(s["mass"], T0, seed=42)
    return s


class Run:
    """One bench-style single-GPU run: engine.Force + the ensemble step of bench.py."""

    def __init__(self, eng, s, potfile, ensemble="nve", dt_fs=1.0, T0=300.0):
        import torch
        self.eng, self.s, self.n = eng, s, s["type"].shape[0]
        self.atom = eng.Atom(s["type"], s["pos"], s["mass"], s["vel"])
        self.box = eng.Box(s["h"], s["pbc"])
        self.force = eng.Force()
        self.pot = self.force.parse_potential(potfile, self.n)
        self.ens = eng.Ensemble_BER(self.n, T0, 100.0) if ensemble == "nvt_ber" else eng.Ensemble_NVE(self.n)
        self.thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
        self.dt = dt_fs / TIME_UNIT_CONVERSION
        self.args = (self.box, self.atom.position_per_atom, self.atom.type, self.atom.potential_per_atom,
                     self.atom.force_per_atom, self.atom.virial_per_atom)
        self.force.compute(*self.args)
        self.pot.check()

    def steps(self, k):
        for _ in range(k):
            self.ens.compute1(self.dt, self.box, self.atom, self.thermo)
            self.force.compute(*self.args)
            self.ens.compute2(self.dt, self.box, self.atom, self.thermo)
        self.pot.check()

    def state(self):
        import torch
        n, a = self.n, self.atom
        th = torch.zeros(8, dtype=torch.float64, device="cuda")
        self.ens.find_thermo(self.box.get_volume(), a, th)
        return dict(pos=a.position_per_atom.cpu().numpy().reshape(3, n), vel=a.velocity_per_atom.cpu().numpy()
                    .reshape(3, n), pe=a.potential_per_atom.cpu().numpy(),
                    force=a.force_per_atom.cpu().numpy().reshape(3, n),
                    virial=a.virial_per_atom.cpu().numpy().reshape(9, n), thermo=th.cpu().numpy())


# ---------------------------------------------------------------- checks

def check_repeat(run, out):
    """Determinism: the potential called again at the same positions gives bit-identical outputs.  (Through
    Force.compute the positions would first pass apply_pbc again, whose round trip through fractional
    coordinates, like the reference's, moves most of them by an ulp.)"""
    a = run.atom
    for t in (a.potential_per_atom, a.force_per_atom, a.virial_per_atom):
        t.zero_()
    run.pot.compute(run.box, a.type, a.position_per_atom, a.potential_per_atom, a.force_per_atom, a.virial_per_atom)
    run.pot.check()
    again = run.state()
    assert np.array_equal(again["pos"], out["pos"])
    for k in ("pe", "force", "virial"):
        assert np.array_equal(again[k], out[k]), k


def check_totals(out, r, s, gap=None):
    """Total energy and virial against float64 sums of the oracle's per-atom outputs, and the device's thermo
    vector against the oracle's find_thermo on the oracle outputs and the device velocities.  gap: the FP32
    oracle's (pe, virial) per-atom outputs, when r is the FP64 oracle (the difference is added)."""
    from oracle import oracle_py
    n = s["type"].shape[0]
    e_scale = np.abs(r["pe"]).sum()
    e_gap = 0.0 if gap is None else abs(gap["pe"].sum() - r["pe"].sum())
    assert abs(out["pe"].sum() - r["pe"].sum()) <= TOL["energy"]["atol"] + TOL["energy"]["rtol"] * e_scale + 2 * e_gap
    assert abs(out["pe"].sum() - r["pe"].sum()) / n < TOL["energy_per_atom"] + 2 * e_gap / n
    # FP32 rounding is relative to the terms summed: every component gets the scale of each atom's largest
    # component (the off-diagonal totals of a crystal cancel to nothing)
    v_scale = np.full(9, np.abs(r["virial"]).max(axis=0).sum())
    v_gap = 0.0 if gap is None else np.abs(gap["virial"].sum(axis=1) - r["virial"].sum(axis=1))
    dv = np.abs(out["virial"].sum(axis=1) - r["virial"].sum(axis=1))
    assert np.all(dv <= TOL["virial"]["atol"] + 1e-5 * v_scale + 2 * v_gap), (dv, v_scale)
    vol = abs(np.linalg.det(s["h"].reshape(3, 3)))
    t_ref = oracle_py.find_thermo(n, vol, s["mass"], r["pe"], out["vel"], r["virial"])
    th = out["thermo"]
    assert abs(th[0] - t_ref[0]) <= 1e-9 * t_ref[0]
    assert abs(th[1] - t_ref[1]) <= TOL["energy"]["atol"] + TOL["energy"]["rtol"] * e_scale + 2 * e_gap
    k_scale = (s["mass"][None, :] * out["vel"] ** 2).sum(axis=1) / vol
    p_tol = (1e-5 * v_scale[:3] + 2 * (v_gap[:3] if gap is not None else 0.0)) / vol + 1e-9 * k_scale
    assert np.all(np.abs(th[2:5] - t_ref[2:5]) <= p_tol + 1e-12), (th[2:5], t_ref[2:5])


def check_nep_state(tag, pot, out, s, potfile, lists=True, gaps=None):
    """Every atom of a NEP state against the FP32 and FP64 tiled oracle (check_nep's conventions), the lists
    bit for bit, the totals and the thermo vector.  gaps: the FP32 oracle's (force, virial) distance from
    FP64 measured on an earlier state of the same run; given, only the FP32 oracle runs (its FP64 twin costs
    as much again).  Returns the gaps of this state."""
    n = s["type"].shape[0]
    st = dict(s, pos=out["pos"])
    r32 = tiled(tag, fullsize.nep(potfile, 32), st, out["pos"], lists=lists)
    r64 = None if gaps else tiled(tag, fullsize.nep(potfile, 64), st, out["pos"])
    if lists:
        NNr, NLr, NNa, NLa = pot.export_neighbors()
        fullsize.assert_same_lists(NNr, NLr, r32["NN_radial"], r32["NL_radial"], s["h"], out["pos"], "radial")
        fullsize.assert_same_lists(NNa, NLa, r32["NN_angular"], r32["NL_angular"], s["h"], out["pos"], "angular")
    assert abs(out["pe"].sum() - r32["pe"].sum()) / n < TOL["energy_per_atom"]
    if r64 is not None:
        gap = abs(r32["pe"].sum() - r64["pe"].sum()) / n
        assert abs(out["pe"].sum() - r64["pe"].sum()) / n < TOL["energy_per_atom"] + 2 * gap
        gaps = (np.abs(r32["force"] - r64["force"]).max(), np.abs(r32["virial"] - r64["virial"]).max())
    gap_f, gap_v = gaps
    check_fv(out, r32, gap_f=gap_f, gap_v=gap_v)
    if r64 is not None:
        check_fv(out, r64, gap_f=gap_f, gap_v=gap_v)
    # site energies: the energy tolerance with check_fv's scaling by the largest magnitude (deep wells of
    # several eV cancel in FP32 like large forces do)
    assert_close(out["pe"], r32["pe"], rtol=TOL["energy"]["rtol"],
                 atol=TOL["energy"]["rtol"] * max(1.0, np.abs(r32["pe"]).max()), what="pe")
    if "thermo" in out:
        check_totals(out, r32, st)
        if r64 is not None:
            check_totals(out, r64, st, gap=r32)
    return gaps


def displace(pos, lo, hi, seed):
    """Every atom moved by lo..hi A in a random direction."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=pos.shape)
    d *= rng.uniform(lo, hi, pos.shape[1]) / np.linalg.norm(d, axis=0)
    return pos + d


# ---------------------------------------------------------------- restated grid rules (b2_neighbor.cu/.cuh)

def make_grid(h, cell):
    """make_grid for an orthogonal box: bins per direction and their count."""
    L = np.diag(np.asarray(h, dtype=np.float64).reshape(3, 3))
    nb = [max(1, int(math.floor(L[d] / cell))) for d in range(3)]
    return nb, nb[0] * nb[1] * nb[2]


def make_bricks(nb, n):
    """b2_make_bricks: (bx, by, bz), brick count."""
    ncell = nb[0] * nb[1] * nb[2]
    span = (32 * ncell + n // 2) // n
    bx = 1 if span < 1 else min(span, nb[0])
    return (bx, 2, 2), -(-nb[0] // bx) * -(-nb[1] // 2) * -(-nb[2] // 2)


def tile_blocks(n):
    return -(-n // 256)


# C3 (1 000 000 atoms), C4 (1 016 064 per GPU), the 2-GPU PbTe arm: the NEP cases at bench size
REACH = {
    "C3": (lambda: np.diag([50 * 6.570] * 3).reshape(9), 1_000_000, 8.0, True, False),
    "C4": (lambda: np.diag([16 * 3.9, 126 * 3.9, 126 * 3.9]).reshape(9), 1_016_064, 6.0, False, True),
}


@pytest.mark.parametrize("case", list(REACH))
def test_reach(eng, case):
    """Every NEP case at bench size has more than 4 x 4096 cells, the few-species one more than 4096 bricks,
    the one with type tiles more than 32 blocks of 256 atoms (so each scan carries across its tiles)."""
    h, n, rc, sched, tiles = REACH[case]
    nb, ncell = make_grid(h(), 0.5 * (rc + SKIN))
    assert ncell > 4 * 4096
    if sched:
        assert make_bricks(nb, n)[1] > 4096
    if tiles:
        assert tile_blocks(n) > 32


# ---------------------------------------------------------------- C3: PbTe NEP, 1 000 000 atoms

def test_c3_pbte_every_atom(oracle, eng):
    """bench.py's headline: (a) the first force call, (b) after 20 NVE steps of the bench step, (c) after
    every atom moved 0.55-0.7 A (over skin/2: the lists rebuild from a sorted order that is not the
    identity).  Also the determinism, force-sum and neighbour-symmetry checks of the former full-size test."""
    need_memory(12, "C3")
    s = bench_pbte(50)
    n = s["type"].shape[0]
    assert n == 1_000_000
    run = Run(eng, s, PBTE)
    pot = run.pot
    sch = pot.export_schedule()
    nb, ncell = make_grid(s["h"], 0.5 * (pot.rc + SKIN))
    assert sch["nb"] == nb and ncell == 73 ** 3
    brick, count = make_bricks(nb, n)
    assert sch["brick"] == list(brick) and count == 9583 and len(sch["cell_start"]) == ncell + 1
    check_schedule(pot, n)
    note_memory("C3")
    out = run.state()
    assert np.abs(out["force"].sum(axis=1)).max() < 2e-3
    # (a)
    check_nep_state("C3", pot, out, s, PBTE)
    check_repeat(run, out)
    # (b)
    run.steps(20)
    out = run.state()
    assert np.abs(out["force"].sum(axis=1)).max() < 2e-3
    check_nep_state("C3", pot, out, s, PBTE)
    # (c)
    import torch
    before = pot.num_rebuilds
    moved = displace(out["pos"], 0.55, 0.7, seed=3)
    run.atom.position_per_atom.copy_(torch.as_tensor(moved.reshape(-1), device="cuda"))
    run.force.compute(*run.args)
    pot.check()
    assert pot.num_rebuilds > before
    out = run.state()
    check_schedule(pot, n)
    check_nep_state("C3", pot, out, s, PBTE)


# ---------------------------------------------------------------- C2: LJ argon, 1 000 188 atoms

def check_lj(tag, out, s):
    st = dict(s, pos=out["pos"])
    r = tiled(tag, fullsize.lj(cc.LJ1), st, out["pos"])
    check_vs_oracle(out, r, s["type"].shape[0], "lj", cc.LJ1)
    check_totals(out, r, st)


def test_c2_lj_every_atom(oracle, eng):
    need_memory(8, "C2")
    s = bench_side("lj", (63, 63, 63))
    n = s["type"].shape[0]
    assert n == 1_000_188
    run = Run(eng, s, cc.LJ1, dt_fs=5.0, T0=80.0)
    note_memory("C2")
    out = run.state()
    assert np.abs(out["force"].sum(axis=1)).max() < 2e-3
    check_lj("C2", out, s)
    check_repeat(run, out)
    run.steps(20)
    out = run.state()
    assert np.abs(out["force"].sum(axis=1)).max() < 2e-3
    check_lj("C2", out, s)


# ---------------------------------------------------------------- C5: Tersoff Si

def check_tersoff(tag, eng, run, out, s):
    from oracle import oracle_py
    st = dict(s, pos=out["pos"])
    r = tiled(tag, fullsize.tersoff(cc.SI), st, out["pos"])
    check_vs_oracle(out, r, s["type"].shape[0], "tersoff", cc.SI)
    check_totals(out, r, st)
    heat = eng.compute_heat(run.atom).view(5, run.n).sum(dim=1).cpu().numpy()
    ref = oracle_py.compute_heat(r["virial"], out["vel"]).sum(axis=1)
    assert_close(heat, ref, rtol=1e-9, atol=1e-9 * np.abs(oracle_py.compute_heat(r["virial"], out["vel"])).sum(),
                 what="heat current")


def test_c5_si_per_gpu(oracle, eng):
    """bench.py --workload si on one GPU (16 x 63 x 63 cells), the first call and after 10 NVE steps with the
    heat current of the bench's measurement."""
    need_memory(8, "C5")
    s = bench_side("si", (16, 63, 63))
    assert s["type"].shape[0] == 508_032
    run = Run(eng, s, cc.SI)
    note_memory("C5")
    check_tersoff("C5", eng, run, run.state(), s)
    run.steps(10)
    out = run.state()
    check_tersoff("C5", eng, run, out, s)


def test_c5_si_63(oracle, eng):
    """63^3 cells (2 000 376 atoms, C5's 4-GPU total on one GPU), rattled 0.05 A: every atom, the force sum and
    a bit-identical repeat (the former full-size Tersoff test)."""
    need_memory(16, "C5_63")
    s = diamond(63, a=5.431, rattle=0.05, seed=1)
    s["vel"] = init_velocities(s["mass"], 300.0, seed=42)
    assert s["type"].shape[0] == 2_000_376
    run = Run(eng, s, cc.SI)
    note_memory("C5_63")
    out = run.state()
    assert np.abs(out["force"].sum(axis=1)).max() < 1e-8
    check_tersoff("C5", eng, run, out, s)
    check_repeat(run, out)


# ---------------------------------------------------------------- C4: UNEP-v1, 16 species

def test_c4_unep_every_atom(oracle, eng):
    """bench.py --workload unep on one GPU (16 x 126 x 126 cells, nvt_ber): the first call and after 10 steps,
    on the tensor-core hidden layer with its type tiles.  After the steps only the FP32 oracle runs, with the
    FP32-FP64 gap of the first call (UNEP costs 170 us per atom and evaluation on one core)."""
    need_memory(16, "C4")
    s = bench_side("unep", (16, 126, 126))
    n = s["type"].shape[0]
    assert n == 1_016_064
    run = Run(eng, s, UNEP, ensemble="nvt_ber")
    note_memory("C4")
    pot = run.pot
    assert pot.num_tiles > 0 and pot.tc_ctas > 0
    assert pot.instances["mlp_dimp"] == 0 and pot.instances["utable"] in (1, 2)
    assert pot.export_schedule() is None  # 16 species: no warp schedule
    check_tile_rule(*pot.export_tiles(), s["type"], 16)
    assert tile_blocks(n) == 3969
    gaps = check_nep_state("C4", pot, run.state(), s, UNEP)
    run.steps(10)
    check_nep_state("C4", pot, run.state(), s, UNEP, gaps=gaps)


# ---------------------------------------------------------------- the 2-GPU arms as block domains

BLOCK_ARMS = {
    "pbte": (PBTE, lambda: rocksalt_pbte((100, 50, 50), rattle=0.02, seed=1), 2_000_000, 300.0, 24),
    "si": (cc.SI, lambda: diamond((32, 63, 63), a=5.431, rattle=0.0, seed=1), 1_016_064, 300.0, 12),
}


@pytest.mark.parametrize("arm", list(BLOCK_ARMS))
def test_blocks_every_atom(oracle, mg, arm):
    """grid (2, 1, 1) in local mode with the bench's 3 A ghost skin: 10 steps, then every owned atom."""
    path, make, n_expect, T0, gib = BLOCK_ARMS[arm]
    need_memory(gib, "blocks_" + arm)
    s = make()
    n = s["type"].shape[0]
    assert n == n_expect
    s["vel"] = init_velocities(s["mass"], T0, seed=42)
    g = mg.DomainGroup(s["h"], s["pbc"], (2, 1, 1), path, ensemble="nve", temperature=T0,
                       temperature_coupling=100.0, time_step=1.0 / TIME_UNIT_CONVERSION, skin=DOMAIN_SKIN)
    g.distribute(s["type"], s["pos"], s["mass"], s["vel"])
    assert g.num_local_domains == 2
    g.run(10, 5)
    g.check()
    note_memory("blocks_" + arm)
    out = g.gather_local()
    assert np.array_equal(out["id"], np.arange(n))
    if arm == "pbte":
        check_nep_state("blocks", None, out, s, path, lists=False)
    else:
        r = tiled("blocks", fullsize.tersoff(path), dict(s, pos=out["pos"]), out["pos"])
        check_vs_oracle(out, r, n, "tersoff", path)


# ---------------------------------------------------------------- the scans at their seams (small)

def dilute(shape, cell, pbc, keep, seed, types=(0.3, 0.7), n=None):
    """Atoms on a jittered grid of ~3.2 A sites (nearest pairs >= 2.6 A) in a box of shape[d] cells of `cell`
    A: periodic directions are shape[d] * cell + 0.2 A long, open ones (shape[d] + 0.5) * cell.  Each site
    is kept with probability `keep` (or exactly n sites are kept); species drawn with the `types` weights."""
    rng = np.random.default_rng(seed)
    L = np.array([shape[d] * cell + 0.2 if pbc[d] else (shape[d] + 0.5) * cell for d in range(3)])
    axes = []
    for d in range(3):
        m = max(1, int(L[d] // 3.2))
        axes.append((np.arange(m) + 0.5) * (L[d] / m))
    g = np.stack(np.meshgrid(*axes, indexing="ij"), 0).reshape(3, -1)
    if n is None:
        g = g[:, rng.random(g.shape[1]) < keep]
    else:
        assert g.shape[1] >= n
        g = g[:, np.sort(rng.choice(g.shape[1], n, replace=False))]
    pos = g + rng.uniform(-0.3, 0.3, g.shape)
    m = pos.shape[1]
    t = rng.choice(len(types), m, p=np.asarray(types) / np.sum(types)).astype(np.int32)
    return dict(pos=np.ascontiguousarray(pos), type=t, h=np.diag(L).reshape(9), pbc=np.asarray(pbc, np.int32))


# target -> (cells per direction, pbc)
NCELL = {
    4095: ((5, 7, 117), (1, 1, 1)),
    4096: ((8, 8, 64), (1, 1, 1)),
    4097: ((17, 241, 1), (1, 1, 0)),
    8192: ((8, 16, 64), (1, 1, 1)),
    8193: ((3, 2731, 1), (0, 1, 0)),
}


def _nep_pot(eng, monkeypatch, n, env=None):
    for k in ("B200MD_NEP_MLP", "B200MD_NEP_SCHED", "B200MD_NEP_TEAM", "B200MD_NEP_RADIAL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    pot = eng.NEP(PBTE, n)
    pot.set_accumulate(False)
    return pot


@pytest.mark.parametrize("target", list(NCELL))
def test_cell_scan_seams_nep(oracle, eng, monkeypatch, target):
    shape, pbc = NCELL[target]
    s = dilute(shape, 4.5, pbc, keep=0.2, seed=target)
    n = s["type"].shape[0]
    nb, ncell = make_grid(s["h"], 4.5)
    assert ncell == target and nb == list(shape)
    pot = _nep_pot(eng, monkeypatch, n)
    check_nep(oracle, Dev(eng, pot), "nep_PbTe.txt", s, n)
    sch = pot.export_schedule()
    assert sch["nb"] == nb and len(sch["cell_start"]) == target + 1
    assert np.array_equal(np.diff(sch["cell_start"]) >= 0, np.ones(target, bool))
    check_schedule(pot, n)


@pytest.mark.parametrize("target", list(NCELL))
def test_cell_scan_seams_lj(oracle, eng, target):
    shape, pbc = NCELL[target]
    s = dilute(shape, 5.5, pbc, keep=0.2, seed=target + 1, types=(1.0,))
    n = s["type"].shape[0]
    assert make_grid(s["h"], 0.5 * (10.0 + SKIN))[1] == target
    pot = eng.LJ(cc.LJ1, n)
    atom = eng.Atom(s["type"], s["pos"], np.ones(n))
    pot.compute(eng.Box(s["h"], s["pbc"]), atom.type, atom.position_per_atom, atom.potential_per_atom,
                atom.force_per_atom, atom.virial_per_atom)
    pot.check()
    out = dict(pe=atom.potential_per_atom.cpu().numpy(), force=atom.force_per_atom.cpu().numpy().reshape(3, n),
               virial=atom.virial_per_atom.cpu().numpy().reshape(9, n))
    check_vs_oracle(out, cc.oracle32("lj", cc.LJ1, s), n, "lj", cc.LJ1)


# target brick count -> cells per direction (bx = nb[0] at this density, so the count is the y-z bricks)
BRICKS = {4095: (5, 125, 130), 4096: (5, 128, 127), 4097: (5, 33, 482)}


@pytest.mark.parametrize("target", list(BRICKS))
def test_brick_scan_seams(oracle, eng, monkeypatch, target):
    shape = BRICKS[target]
    s = dilute(shape, 4.5, (1, 1, 1), keep=0.09, seed=target)
    n = s["type"].shape[0]
    nb, ncell = make_grid(s["h"], 4.5)
    brick, count = make_bricks(nb, n)
    assert nb == list(shape) and count == target and brick[0] == shape[0]
    pot = _nep_pot(eng, monkeypatch, n)
    check_nep(oracle, Dev(eng, pot), "nep_PbTe.txt", s, n)
    sch = pot.export_schedule()
    assert sch["nb"] == nb and sch["brick"] == list(brick)
    check_schedule(pot, n)


@pytest.mark.parametrize("n", [8191, 8192, 8193, 16385])
def test_tile_scan_seams(oracle, eng, monkeypatch, n):
    """PbTe on the tensor-core hidden layer (B200MD_NEP_MLP=tc builds type tiles), 30 % Te / 70 % Pb: 32, 32,
    33 and 65 blocks of 256 atoms."""
    s = dilute((26, 26, 26), 4.5, (1, 1, 1), keep=None, seed=n, n=n)
    assert s["type"].shape[0] == n and 0 < (s["type"] == 0).sum() < (s["type"] == 1).sum()
    pot = _nep_pot(eng, monkeypatch, n, {"B200MD_NEP_MLP": "tc"})
    check_nep(oracle, Dev(eng, pot), "nep_PbTe.txt", s, n)
    assert pot.num_tiles > 0 and pot.tc_ctas > 0
    slot, tile_type = pot.export_tiles()
    check_tile_rule(slot, tile_type, s["type"], 2)
    assert tile_blocks(n) == {8191: 32, 8192: 32, 8193: 33, 16385: 65}[n]
    check_schedule(pot, n)

"""The warp schedule of the one- and two-species NEP kernels (B2NeighborView::seg_order; B200MD_NEP_SCHED=0
selects the identity schedule) changes which warp evaluates which 32 consecutive sorted atoms and nothing
else.  So every observable -- energies, forces, virials, the exported lists and descriptors -- must be
bit-identical between the two settings, on every box shape and calling mode, and the default must still sit
within the oracle's tolerances.  After each list rebuild the schedule read back from the device is a
permutation of the segments, equals the ordering rule stated in numpy (test_nep_schedule_cpu.expected_order)
and is the same in a second run."""
import numpy as np
import pytest

from cases import shear, slab
from conftest import GOLDEN
from gpumd_b200.structures import diamond, rocksalt_pbte
from test_kernel_bodies_cpu import check_nep
from test_nep_schedule_cpu import expected_order

pytestmark = pytest.mark.gpu

KEYS = ("pe", "force", "virial")
MODELS = {
    # model file, large structure, small (supercell path) structure
    "PbTe": ("nep_PbTe.txt", lambda: rocksalt_pbte(6, rattle=0.05, seed=1),      # 1728 atoms = 54 segments
             lambda: rocksalt_pbte(3, rattle=0.05, seed=1)),                    # 19.7 A
    "carbon": ("nep_C_2022_NEP4.txt", lambda: diamond(5, a=3.57, rattle=0.05, seed=3, symbol="C"),  # 1000 atoms
               lambda: diamond(3, a=3.57, rattle=0.05, seed=3, symbol="C")),    # 10.7 A
}
BOXES = {"ortho": lambda s: s, "triclinic": shear, "slab": slab}


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def make_pot(eng, monkeypatch, model, n, sched):
    """The switch is read when the handle is created."""
    if sched:
        monkeypatch.delenv("B200MD_NEP_SCHED", raising=False)
    else:
        monkeypatch.setenv("B200MD_NEP_SCHED", "0")
    pot = eng.NEP(GOLDEN / model, n)
    pot.set_accumulate(False)
    return pot


def call(eng, pot, s, observables=True):
    """One store-mode compute on NaN-filled outputs; with the exported lists and descriptors."""
    import torch
    n = s["type"].shape[0]
    bufs = [torch.full((k * n,), np.nan, dtype=torch.float64, device="cuda") for k in (1, 3, 9)]
    ty = torch.as_tensor(np.ascontiguousarray(s["type"], np.int32), device="cuda")
    p = torch.as_tensor(np.ascontiguousarray(s["pos"], np.float64).reshape(-1), device="cuda")
    pot.compute(eng.Box(s["h"], s["pbc"]), ty, p, *bufs)
    pot.check()
    out = dict(pe=bufs[0].cpu().numpy(), force=bufs[1].cpu().numpy().reshape(3, n),
               virial=bufs[2].cpu().numpy().reshape(9, n))
    if observables and n == pot.N2:  # the export hooks size their outputs by the handle's atom count
        out["lists"] = pot.export_neighbors()
        out["q"] = pot.export_descriptors()
    return out


def same(a, b, what):
    for k in KEYS:
        assert np.array_equal(a[k], b[k], equal_nan=True), (what, k)
    if "lists" in a:
        for x, y in zip(a["lists"], b["lists"]):
            assert np.array_equal(x, y), (what, "lists")
        assert np.array_equal(a["q"], b["q"]), (what, "descriptors")


def check_schedule(pot, n_eval):
    """The device's schedule is a permutation of the segments and follows the ordering rule."""
    sch = pot.export_schedule()
    assert sch is not None
    nseg = (n_eval + 31) // 32
    assert sch["cell_start"][-1] == n_eval
    assert np.array_equal(np.sort(sch["seg_order"]), np.arange(nseg))
    assert np.array_equal(sch["seg_order"], expected_order(n_eval, sch["nb"], sch["brick"], sch["cell_start"]))
    return sch["seg_order"]


class Dev:
    """check_nep's device adapter over an existing handle."""

    def __init__(self, eng, pot):
        self.eng, self.pot = eng, pot

    def compute(self, type_, h, pbc, pos):
        return 0, call(self.eng, self.pot, dict(type=type_, h=h, pbc=pbc, pos=pos), observables=False)

    def neighbors(self, mn_r, mn_a):
        return self.pot.export_neighbors(mn_r, mn_a)

    def descriptors(self, dim):
        return self.pot.export_descriptors()


@pytest.mark.parametrize("box", list(BOXES) + ["small"])
@pytest.mark.parametrize("case", list(MODELS))
def test_schedule_changes_no_result(oracle, eng, case, box, monkeypatch):
    model, large, small = MODELS[case]
    s = small() if box == "small" else BOXES[box](large())
    n = s["type"].shape[0]
    off = make_pot(eng, monkeypatch, model, n, sched=False)
    assert off.export_schedule() is None
    ref = call(eng, off, s)
    on = make_pot(eng, monkeypatch, model, n, sched=True)
    out = call(eng, on, s)
    same(out, ref, "default against B200MD_NEP_SCHED=0")
    # a small box evaluates a supercell: the schedule covers all its replicas
    n_eval = int(on.export_schedule()["cell_start"][-1])
    assert n_eval == n if box != "small" else n_eval > n and n_eval % n == 0
    order = check_schedule(on, n_eval)
    if box != "small":
        assert not np.array_equal(order, np.arange(order.size)), "the default schedule is the identity"
    # the oracle, through the same checks as every other kernel path
    e_tol = 1e-6 * 8.0 if case == "carbon" else None  # -7.9 eV/atom: FP32 rounding is relative
    check_nep(oracle, Dev(eng, on), model, s, n, energy_tol=e_tol)
    # a second handle builds the same schedule, and a forced rebuild reproduces it and the result
    again = make_pot(eng, monkeypatch, model, n, sched=True)
    same(call(eng, again, s), ref, "second run")
    assert np.array_equal(check_schedule(again, n_eval), order)
    before = on.num_rebuilds
    on.invalidate(n)
    same(call(eng, on, s), ref, "after invalidate")
    assert on.num_rebuilds == before + 1
    assert np.array_equal(check_schedule(on, n_eval), order)


@pytest.mark.parametrize("n", [1, 31, 33, 1001, 1700])
def test_atom_counts_that_are_no_multiple_of_32(eng, n, monkeypatch):
    """The last segment is partly filled (or the only one)."""
    model, large, _ = MODELS["PbTe"]
    s = large()
    idx = np.random.default_rng(n).permutation(s["type"].shape[0])[:n]
    s = dict(s, type=np.ascontiguousarray(s["type"][idx]), pos=np.ascontiguousarray(s["pos"][:, idx]))
    ref = call(eng, make_pot(eng, monkeypatch, model, n, sched=False), s)
    on = make_pot(eng, monkeypatch, model, n, sched=True)
    same(call(eng, on, s), ref, f"n = {n}")
    check_schedule(on, n)


@pytest.mark.parametrize("case", list(MODELS))
def test_calling_modes_on_one_handle(eng, case, monkeypatch):
    """Owned range, active region, a changing atom count and a permuted atom set after invalidate: the same
    sequence on a handle of each setting, compared call by call; the schedule is rebuilt with every list."""
    model, large, _ = MODELS[case]
    s = large()
    N = s["type"].shape[0]
    off = make_pot(eng, monkeypatch, model, N, sched=False)
    on = make_pot(eng, monkeypatch, model, N, sched=True)
    rng = np.random.default_rng(5)

    def both(sub, what):
        a, b = call(eng, off, sub), call(eng, on, sub)
        same(b, a, what)
        check_schedule(on, sub["type"].shape[0])
        return b

    full = both(s, "all atoms")
    for m in (1, 100, N - 1):
        for p in (off, on):
            p.set_owned(m)
        out = both(s, f"set_owned({m})")
        for k in KEYS:
            assert np.array_equal(out[k][..., :m], full[k][..., :m]) and np.isnan(out[k][..., m:]).all()
    for p in (off, on):
        p.set_owned(0)
    lo, hi = s["pos"].min(axis=1) + 1.0, s["pos"].max(axis=1) - 1.0
    for p in (off, on):
        p.set_active_region(lo, hi)
    out = both(s, "active region")
    outer = ~((s["pos"] >= lo[:, None]) & (s["pos"] < hi[:, None])).all(axis=0)
    assert outer.sum() >= 10 and np.all(out["q"][:, outer] == 0.0)
    for p in (off, on):
        p.set_active_region(None)
    same(both(s, "region off"), full, "region off against the first call")
    for n in (N, 127, 129, 500, N):
        idx = rng.permutation(N)[:n]
        sub = dict(s, type=np.ascontiguousarray(s["type"][idx]), pos=np.ascontiguousarray(s["pos"][:, idx]))
        both(sub, f"n = {n}")
    perm = rng.permutation(N)
    sp = dict(s, type=np.ascontiguousarray(s["type"][perm]), pos=np.ascontiguousarray(s["pos"][:, perm]))
    for p in (off, on):
        p.invalidate(N)
    both(sp, "permuted after invalidate")


def test_schedule_on_a_larger_crystal_across_md_rebuilds(eng, monkeypatch):
    """13 824 atoms (432 segments, bricks of several segments per row) through NVE steps hot enough to
    trigger displacement rebuilds: trajectories of the two settings stay bit-identical, and the schedule
    follows the rule after the rebuilds."""
    import torch
    from gpumd_b200.structures import TIME_UNIT_CONVERSION, init_velocities
    s = rocksalt_pbte(12, rattle=0.05, seed=2)
    n = s["type"].shape[0]
    vel = init_velocities(s["mass"], 1200.0, seed=4)
    runs = {}
    for sched in (False, True):
        if sched:
            monkeypatch.delenv("B200MD_NEP_SCHED", raising=False)
        else:
            monkeypatch.setenv("B200MD_NEP_SCHED", "0")
        atom = eng.Atom(s["type"], s["pos"], s["mass"], vel)
        box = eng.Box(s["h"], s["pbc"])
        force = eng.Force()
        pot = force.parse_potential(GOLDEN / "nep_PbTe.txt", n)
        ens = eng.Ensemble_NVE(n)
        thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
        fargs = (box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
                 atom.virial_per_atom)
        force.compute(*fargs)
        dt = 2.0 / TIME_UNIT_CONVERSION
        for _ in range(200):
            ens.compute1(dt, box, atom, thermo)
            force.compute(*fargs)
            ens.compute2(dt, box, atom, thermo)
        pot.check()
        runs[sched] = dict(pot=pot, pos=atom.position_per_atom.cpu().numpy(),
                           f=atom.force_per_atom.cpu().numpy(), v=atom.virial_per_atom.cpu().numpy(),
                           pe=atom.potential_per_atom.cpu().numpy())
    assert runs[True]["pot"].num_rebuilds >= 2  # the first build and at least one by displacement
    assert runs[True]["pot"].num_rebuilds == runs[False]["pot"].num_rebuilds
    for k in ("pos", "f", "v", "pe"):
        assert np.array_equal(runs[True][k], runs[False][k]), k
    order = check_schedule(runs[True]["pot"], n)
    assert not np.array_equal(order, np.arange(order.size))

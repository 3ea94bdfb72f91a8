"""The NEP handle's calling modes on every kernel path it dispatches: store mode
(b200md_nep_set_accumulate(p, 0), what the `b200md` driver, engine.Force and every block domain use), the
owned range (set_owned), the active region (set_active_region) and an atom count that changes from call to
call on one handle (block domains after each exchange).  Each mode is checked against the default mode on
zeroed outputs bit for bit, and against the oracle; then short trajectories in store mode on small cells and
the lane-team kernels, and the driver on a small cell."""
import shutil
import subprocess

import numpy as np
import pytest

from cases import NEP_CASES, NEP_CASES_SYNTH, NEP_SMALL_CASES, shear, slab
from conftest import GOLDEN, TOL, assert_close
from gpumd_b200.structures import diamond, init_velocities, rocksalt_pbte, write_xyz
from test_few_species_cpu import FEW_SPECIES_CASES
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)
from test_kernel_bodies_cpu import check_fv, check_nep

pytestmark = pytest.mark.gpu

NAN3 = (np.nan,) * 3
KEYS = ("pe", "force", "virial")


def _pbte(make):
    """PbTe, 1728 atoms (39.4 A): an active region with rc = 8 A of margin inside it still holds atoms."""
    return "nep_PbTe.txt", lambda: make(rocksalt_pbte(6, rattle=0.05, seed=1))


# kernel path -> (switches, (model file, structure factory))
PATHS = {
    "fused": ({}, _pbte(lambda s: s)),  # k_angular_fused, the default for PbTe
    "fused_triclinic": ({}, _pbte(shear)),
    "fused_slab": ({}, _pbte(slab)),
    "mlp_tc": ({"B200MD_NEP_MLP": "tc"}, _pbte(lambda s: s)),
    "mlp_simt": ({"B200MD_NEP_MLP": "simt"}, _pbte(lambda s: s)),
    "team_1sp": ({"B200MD_NEP_TEAM": "1"}, FEW_SPECIES_CASES["zbl_k17"]),
    "team_2sp": ({"B200MD_NEP_TEAM": "1"}, _pbte(lambda s: s)),
    "radial_v1": ({"B200MD_NEP_RADIAL": "v1"}, _pbte(lambda s: s)),
    "many_smem": ({}, NEP_CASES["UNEP"]),  # per-type radial accumulators in shared memory
    "raddirect": ({"B200MD_NEP_RADDIRECT": "1"}, NEP_CASES["UNEP"]),
    "synth50": ({}, NEP_CASES_SYNTH["synth50"]),  # per-pair radial contraction by necessity
    "revslot": ({"B200MD_NEP_REVSLOT": "1"}, NEP_CASES["UNEP"]),
    "radreg": ({"B200MD_NEP_RADREG": "1"}, NEP_CASES["UNEP"]),
    "small_PbTe_C1": ({}, NEP_SMALL_CASES["PbTe_C1"]),  # supercell path
    "small_BaZrO3_40": ({}, NEP_SMALL_CASES["BaZrO3_40"]),
}
PBTE_PATHS = ["fused", "mlp_tc", "mlp_simt", "team_2sp", "radial_v1"]


def _setup(path, monkeypatch):
    env, (model, make) = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return model, make()


def _buffers(n, fill):
    import torch
    return [torch.full((k * n,), float(f), dtype=torch.float64, device="cuda") for k, f in zip((1, 3, 9), fill)]


def _compute(eng, pot, s, bufs):  # noqa: F811
    """One b200md_nep_compute into the device buffers `bufs` (pe, force, virial) as they are."""
    import torch
    n = s["type"].shape[0]
    ty = torch.as_tensor(np.ascontiguousarray(s["type"], np.int32), device="cuda")
    p = torch.as_tensor(np.ascontiguousarray(s["pos"], np.float64).reshape(-1), device="cuda")
    pot.compute(eng.Box(s["h"], s["pbc"]), ty, p, *bufs)
    pot.check()
    return dict(pe=bufs[0].cpu().numpy(), force=bufs[1].cpu().numpy().reshape(3, n),
                virial=bufs[2].cpu().numpy().reshape(9, n))


def _call(eng, pot, s, fill=(0.0, 0.0, 0.0)):  # noqa: F811
    return _compute(eng, pot, s, _buffers(s["type"].shape[0], fill))


def _same(a, b, sel=slice(None), what=""):
    for k in KEYS:
        x, y = a[k][..., sel], b[k][..., sel]
        assert np.array_equal(x, y), (what, k, np.nanmax(np.abs(x - y)) if x.size else 0)


class StoreNep(GpuNep):
    """GpuNep in store mode on NaN-filled outputs (check_nep's device adapter)."""

    def __init__(self, eng, model, n):  # noqa: F811
        super().__init__(eng, model, n)
        self.pot.set_accumulate(False)

    def compute(self, type_, h, pbc, pos):
        return 0, _call(self.eng, self.pot, dict(type=type_, h=h, pbc=pbc, pos=pos), NAN3)


@pytest.mark.parametrize("path", list(PATHS))
def test_store_mode(oracle, eng, path, monkeypatch):  # noqa: F811
    """set_accumulate(0) on NaN-filled outputs: the oracle's answer, bit-identical to accumulate mode on zeros,
    unchanged by a second call into the same arrays; back in accumulate mode the outputs are added to."""
    model, s = _setup(path, monkeypatch)
    n = s["type"].shape[0]
    ref = _call(eng, eng.NEP(GOLDEN / model, n), s)
    dev = StoreNep(eng, model, n)
    out = check_nep(oracle, dev, model, s, n)
    _same(out, ref, what="store")
    bufs = _buffers(n, NAN3)
    _compute(eng, dev.pot, s, bufs)
    _same(_compute(eng, dev.pot, s, bufs), ref, what="second store into the same arrays")
    dev.pot.set_accumulate(True)
    fill = (1.0, 2.0, 3.0)
    out = _call(eng, dev.pot, s, fill)
    for k, f in zip(KEYS, fill):
        assert np.array_equal(out[k], ref[k] + f), k


@pytest.mark.parametrize("owned", [0, 100])
@pytest.mark.parametrize("path", PBTE_PATHS)
def test_store_mode_across_box_changes(oracle, eng, path, owned, monkeypatch):  # noqa: F811
    """One handle, store mode, set_owned: large, small (supercell: the handle grows), small, large, small.
    Every call equals the oracle on the owned atoms and leaves the rest as they were."""
    env, _ = PATHS[path]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = rocksalt_pbte(3, rattle=0.05, seed=1)  # 216 atoms, 19.7 A: a small box
    n = s["type"].shape[0]
    m = owned or n
    pot = eng.NEP(GOLDEN / "nep_PbTe.txt", n)
    pot.set_accumulate(False)
    pot.set_owned(owned)
    orc = oracle.NepOracle(GOLDEN / "nep_PbTe.txt")
    for scale in (2.4, 1.0, 1.0, 2.4, 1.0):
        h, pos = s["h"] * scale, s["pos"] * scale
        r = orc.compute(s["type"], h, s["pbc"], pos, precision=32)
        out = _call(eng, pot, dict(type=s["type"], h=h, pbc=s["pbc"], pos=pos), NAN3)
        for k in KEYS:
            assert np.isnan(out[k][..., m:]).all() and np.isfinite(out[k][..., :m]).all(), (scale, k)
        assert abs(out["pe"][:m].sum() - r["pe"][:m].sum()) / m < TOL["energy_per_atom"], scale
        check_fv(dict(force=out["force"][:, :m], virial=out["virial"][:, :m]),
                 dict(force=r["force"][:, :m], virial=r["virial"][:, :m]))


@pytest.mark.parametrize("path", list(PATHS))
def test_owned_range(eng, path, monkeypatch):  # noqa: F811
    """set_owned(m), m = 1, 127, 128, 129, n - 1, in store and accumulate mode: atoms below m get exactly the
    full evaluation (plus the prefill when accumulating), the others keep the prefill; set_owned(0) restores
    all atoms."""
    model, s = _setup(path, monkeypatch)
    n = s["type"].shape[0]
    ref = _call(eng, eng.NEP(GOLDEN / model, n), s)
    pot = eng.NEP(GOLDEN / model, n)
    fill = (7.0, -8.0, 9.0)
    for accumulate in (False, True):
        pot.set_accumulate(accumulate)
        for m in sorted({m for m in (1, 127, 128, 129, n - 1) if 0 < m < n}):
            pot.set_owned(m)
            out = _call(eng, pot, s, fill)
            for k, f in zip(KEYS, fill):
                want = ref[k][..., :m] + f if accumulate else ref[k][..., :m]
                assert np.array_equal(out[k][..., :m], want), (accumulate, m, k)
                assert np.all(out[k][..., m:] == f), (accumulate, m, k)
    pot.set_owned(0)
    pot.set_accumulate(False)
    _same(_call(eng, pot, s, NAN3), ref, what="set_owned(0)")


def _inner_atoms(s, lo, hi, margin):
    """Atoms at least `margin` inside [lo, hi) and, along periodic directions, from the cell faces: every
    atom within `margin` of them lies inside the region, with no periodic wrap in between."""
    pos = s["pos"]
    H = s["h"].reshape(3, 3)
    inside = ((pos - lo[:, None] >= margin) & (hi[:, None] - pos >= margin)).all(axis=0)
    frac = np.linalg.solve(H, pos)
    thick = 1.0 / np.linalg.norm(np.linalg.inv(H), axis=1)  # distance between opposite faces
    for d in range(3):
        if s["pbc"][d]:
            inside &= np.minimum(frac[d], 1.0 - frac[d]) * thick[d] >= margin
    return np.nonzero(inside)[0]


@pytest.mark.parametrize("path", list(PATHS))
def test_active_region(eng, path, monkeypatch):  # noqa: F811
    """set_active_region(lo, hi) 1 A inside the atoms' bounding box: atoms at least rc inside the region (so
    that every atom their result depends on is active) get the full evaluation bit for bit -- the region
    only empties the lists of the atoms outside it, and no inner atom's summation order changes; atoms
    outside get no descriptors and empty lists.  A small box ignores the region (its supercell images lie
    outside the caller's coordinates).  set_active_region(None) restores the full result."""
    model, s = _setup(path, monkeypatch)
    n = s["type"].shape[0]
    pot = eng.NEP(GOLDEN / model, n)
    pot.set_accumulate(False)
    ref = _call(eng, pot, s, NAN3)
    q_ref = pot.export_descriptors()
    lists_ref = pot.export_neighbors()
    lo, hi = s["pos"].min(axis=1) + 1.0, s["pos"].max(axis=1) - 1.0
    pot.set_active_region(lo, hi)
    out = _call(eng, pot, s, NAN3)
    q = pot.export_descriptors()
    NNr, NLr, NNa, NLa = pot.export_neighbors()
    if path.startswith("small_"):
        _same(out, ref, what="small box with a region")
        assert np.array_equal(q, q_ref)
        for a, b in zip((NNr, NLr, NNa, NLa), lists_ref):
            assert np.array_equal(a, b)
    else:
        inner = _inner_atoms(s, lo, hi, pot.rc + 0.01)
        outer = np.nonzero(~((s["pos"] >= lo[:, None]) & (s["pos"] < hi[:, None])).all(axis=0))[0]
        assert inner.size >= 10 and outer.size >= 10, (inner.size, outer.size)
        _same(out, ref, inner, what="inner atoms")
        assert np.array_equal(q[:, inner], q_ref[:, inner])
        assert np.all(q[:, outer] == 0.0)
        assert np.all(NNr[outer] == 0) and np.all(NNa[outer] == 0)
        assert np.all(NLr[outer] == -1) and np.all(NLa[outer] == -1)
        assert np.array_equal(NNr[inner], lists_ref[0][inner]) and np.array_equal(NNa[inner], lists_ref[2][inner])
    pot.set_active_region(None)
    _same(_call(eng, pot, s, NAN3), ref, what="region switched off")


def _subset(s, n, nt, rng):
    """n atoms of s.  Two-species models get species counts that make type tiles (128 atoms) of 0, 1, 127,
    128 and 129 atoms over the sequence of atom counts; one species stays one species; many species keep
    theirs."""
    idx = rng.permutation(s["type"].shape[0])[:n]
    t = s["type"][idx].copy()
    if nt == 2:
        n0 = {1: 1, 127: 0, 128: 128, 129: 1, 257: 128}.get(n, n // 2)
        t = np.r_[np.zeros(n0, np.int32), np.ones(n - n0, np.int32)]
    return dict(s, type=np.ascontiguousarray(t, np.int32), pos=np.ascontiguousarray(s["pos"][:, idx]))


@pytest.mark.parametrize("path", list(PATHS))
def test_changing_atom_count_on_one_handle(oracle, eng, path, monkeypatch):  # noqa: F811
    """A handle created for N atoms, called in store mode with N, 1, 127, 128, 129, 257 and N atoms, then with
    the atoms permuted after invalidate(N) (the migration path of a block domain): every call bit-identical
    to a fresh handle created for that count, which itself matches the oracle."""
    model, s = _setup(path, monkeypatch)
    N = s["type"].shape[0]
    pot = eng.NEP(GOLDEN / model, N)
    pot.set_accumulate(False)
    nt = pot.num_types
    rng = np.random.default_rng(11)
    counts = [c for c in (N, 1, 127, 128, 129, 2 * 128 + 1, N) if c <= N]
    for n in counts:
        sub = _subset(s, n, nt, rng) if n < N else s
        # A mean over few atoms no longer averages out the FP32 rounding of single site energies (a lone
        # UNEP-v1 atom: 1.9e-6 eV from the FP32 restatement, the same bits in the host build of the
        # bodies): below one 128-atom tile the bound is the reference suite's rtol on the site energies.
        e_tol = None
        if n < 128:
            e64 = oracle.NepOracle(GOLDEN / model).compute(sub["type"], sub["h"], sub["pbc"], sub["pos"],
                                                           precision=64)["pe"]
            e_tol = max(TOL["energy_per_atom"], TOL["energy"]["rtol"] * np.abs(e64).mean())
        fresh = check_nep(oracle, GpuNep(eng, model, n), model, sub, n, energy_tol=e_tol)
        _same(_call(eng, pot, sub, NAN3), fresh, what=f"n = {n}")
    perm = rng.permutation(N)
    sp = dict(s, type=np.ascontiguousarray(s["type"][perm]), pos=np.ascontiguousarray(s["pos"][:, perm]))
    pot.invalidate(N)
    fresh = GpuNep(eng, model, N).compute(sp["type"], sp["h"], sp["pbc"], sp["pos"])[1]
    _same(_call(eng, pot, sp, NAN3), fresh, what="permuted after invalidate")


def _si64():
    return diamond(2, a=5.431, rattle=0.05, seed=3)  # 64 atoms, 10.9 A: a small box for rc = 5 A


TRAJECTORIES = {
    "PbTe_C1": ({}, "nep_PbTe.txt", lambda: rocksalt_pbte(3, rattle=0.02, seed=1)),
    "Si64": ({}, "nep_Si_2022_NEP4_3body.txt", _si64),
    "PbTe_team": ({"B200MD_NEP_TEAM": "1"}, "nep_PbTe.txt", lambda: rocksalt_pbte(4, rattle=0.02, seed=1)),
}


@pytest.mark.parametrize("case", list(TRAJECTORIES))
def test_store_mode_trajectory(oracle, eng, case, monkeypatch):  # noqa: F811
    """100 NVE steps through engine.Force (store mode, no zeroing pass): the reference's energy bound and, at
    the last step, forces and virials of an oracle evaluation at the final positions."""
    from test_gpu_md import run_nve, total_energy
    env, model, make = TRAJECTORIES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    s = make()
    n = s["type"].shape[0]
    atom, pot, rows = run_nve(eng, s, GOLDEN / model, 100, 1.0, 300.0, every=10)
    e = total_energy(rows, n)
    assert np.abs(e - e[0]).max() < 2e-3 * 1.0 ** 2 * n  # reference bound: 2e-3*dt^2*N eV
    pos = atom.position_per_atom.cpu().numpy().reshape(3, n)
    r = oracle.NepOracle(GOLDEN / model).compute(s["type"], s["h"], s["pbc"], pos)
    check_fv(dict(force=atom.force_per_atom.cpu().numpy().reshape(3, n),
                  virial=atom.virial_per_atom.cpu().numpy().reshape(9, n)), r)


def test_driver_small_cell_forces(eng, tmp_path):  # noqa: F811
    """`b200md`, 50 NVE steps of a 64-atom Si cell (supercell path, store mode): the forces of the last
    dump_xyz frame equal a fresh evaluation at that frame's positions."""
    from gpumd_b200 import build
    from gpumd_b200.structures import read_xyz
    exe = build.build_host()
    s = _si64()
    n = s["type"].shape[0]
    write_xyz(tmp_path / "model.xyz", s, ["Si"], init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "nep_Si_2022_NEP4_3body.txt", tmp_path / "potential.txt")
    (tmp_path / "run.in").write_text(
        "potential potential.txt\nensemble nve\ntime_step 1\n"
        "dump_xyz 50 dump.xyz precision double force\nrun 50\n")
    r = subprocess.run([str(exe)], cwd=tmp_path, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert (tmp_path / "dump.xyz").read_text().count("Lattice=") == 1
    frame = read_xyz(tmp_path / "dump.xyz", ["Si"])
    assert frame["forces"].shape == (3, n)
    fresh = _call(eng, eng.NEP(GOLDEN / "nep_Si_2022_NEP4_3body.txt", n),
                  dict(type=frame["type"], h=frame["h"], pbc=frame["pbc"], pos=frame["pos"]))
    assert_close(frame["forces"], fresh["force"], rtol=TOL["force"]["rtol"],
                 atol=TOL["force"]["atol"] * max(1.0, np.abs(fresh["force"]).max()), what="force")

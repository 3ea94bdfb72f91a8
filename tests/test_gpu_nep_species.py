"""Species bookkeeping of the NEP handle on every kernel path: atom types that change between calls at the
same positions (Monte Carlo swaps and composition changes between MD steps), the type tiles of the
tensor-core hidden layer, and that layer with many tiles per persistent CTA.

The few-species kernels carry a neighbour's species in its skin-list entry, and the tensor-core layer picks
weights by the species of a 128-atom tile; both are built at a list rebuild.  A changed type must therefore
rebuild the lists, which these tests check bit for bit against a fresh handle and against the oracle.  The
hidden layer's output (site energy, dU/dq and the radial U table) is checked atom by atom against an FP64
restatement written from the model file, so that one wrong tile cannot hide inside force tolerances."""
import numpy as np
import pytest

import cases_classical as cc
from cases import NEP_CASES, NEP_CASES_SYNTH, NEP_SMALL_CASES, _random_alloy, bazro3_supercell
from conftest import GOLDEN, TOL
from gpumd_b200.structures import TIME_UNIT_CONVERSION, fcc, init_velocities, nep_type_order, rocksalt_pbte
from test_classical_cpu import check_vs_oracle
from test_few_species_cpu import FEW_SPECIES_CASES
from test_gpu_classical import compute as classical_compute
from test_gpu_nep_modes import KEYS, NAN3, PATHS, _call, _same
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)
from test_kernel_bodies_cpu import check_fv, check_nep

pytestmark = pytest.mark.gpu

# Scaled bound of the hidden layer against the FP64 restatement: |got - ref| <= C_MLP * sum |terms|, the
# terms including the propagation of the first GEMM's rounding through tanh.  FP32 accumulation (SIMT) and
# 3xTF32 products with FP32 accumulators (tensor cores) with tanhf both stay below it on every model here.
C_MLP = 1e-6


# ------------------------------------------------------------------------------------------ type changes

def _swap(t, rng, frac=0.05):
    """Canonical Monte Carlo: `frac` of the atoms exchange species with an atom of another species."""
    t = t.copy()
    n = t.size
    done = 0
    for _ in range(50 * n):
        if done >= max(1, int(frac * n / 2)):
            break
        i, j = rng.integers(0, n, 2)
        if t[i] != t[j]:
            t[i], t[j] = t[j], t[i]
            done += 1
    assert done > 0
    return t


def _sgc(t, nt, rng, frac=0.05):
    """Semi-grand canonical: `frac` of the atoms take another species (the composition changes)."""
    t = t.copy()
    idx = rng.choice(t.size, max(1, int(frac * t.size)), replace=False)
    t[idx] = (t[idx] + rng.integers(1, nt, idx.size)) % nt
    return t


def _vanish(t, nt):
    """Every atom of species 0 becomes the last species: species 0 owns no atom (and no tile) any more."""
    t = t.copy()
    t[t == 0] = nt - 1
    return t


def type_pair(kind, t, nt, seed=5):
    """(T1, T2): the types of the first and of the second call."""
    rng = np.random.default_rng(seed)
    t = np.ascontiguousarray(t, np.int32)
    if kind == "swap":
        return t, _swap(t, rng)
    if kind == "sgc":
        return t, _sgc(t, nt, rng)
    if kind == "vanish":
        return t, _vanish(t, nt)
    return _vanish(t, nt), t  # "appear": species 0 comes (back) into the system


KINDS = ["swap", "sgc", "vanish", "appear"]

# every path of test_gpu_nep_modes with more than one species (one species has nothing to change), and
# BaZrO3 at 1080 atoms on its default tensor-core layer
TYPE_PATHS = dict({k: v for k, v in PATHS.items() if k != "team_1sp"},
                  BaZrO3=({}, NEP_CASES["BaZrO3"]))


def _env(monkeypatch, env):
    for k in ("B200MD_NEP_MLP", "B200MD_NEP_TEAM", "B200MD_NEP_RADIAL", "B200MD_NEP_RADDIRECT",
              "B200MD_NEP_REVSLOT", "B200MD_NEP_RADREG", "B200MD_NEP_TC_CTAS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("path", list(TYPE_PATHS))
def test_types_changed_without_moving_atoms(oracle, eng, path, kind, monkeypatch):  # noqa: F811
    """One handle in store mode computes types T1, then T2 at the same positions: bit-identical to a fresh
    handle given T2, which matches the oracle.  The change rebuilds the lists exactly once; T2 again does
    not rebuild."""
    env, (model, make) = TYPE_PATHS[path]
    _env(monkeypatch, env)
    s = make()
    n = s["type"].shape[0]
    pot = eng.NEP(GOLDEN / model, n)
    pot.set_accumulate(False)
    t1, t2 = type_pair(kind, s["type"], pot.num_types)
    assert not np.array_equal(t1, t2)
    _call(eng, pot, dict(s, type=t1), NAN3)
    r0 = pot.num_rebuilds
    out = _call(eng, pot, dict(s, type=t2), NAN3)
    r1 = pot.num_rebuilds
    s2 = dict(s, type=t2)
    # below one 128-atom tile the mean no longer averages out the FP32 rounding of single site energies: the
    # bound is then the reference suite's rtol on them (as in test_gpu_nep_modes)
    e_tol = None
    if n < 128:
        e64 = oracle.NepOracle(GOLDEN / model).compute(t2, s["h"], s["pbc"], s["pos"], precision=64)["pe"]
        e_tol = max(TOL["energy_per_atom"], TOL["energy"]["rtol"] * np.abs(e64).mean())
    fresh = check_nep(oracle, GpuNep(eng, model, n), model, s2, n, energy_tol=e_tol)
    _same(out, fresh, what=f"{kind}: T1 then T2 on one handle")
    assert r1 == r0 + 1, (r0, r1)
    _same(_call(eng, pot, s2, NAN3), fresh, what="T2 again")
    assert pot.num_rebuilds == r0 + 1


CLASSICAL = {"lj": "lj_3sp-ortho", "eam": "eam_cufeni_a0-ortho", "tersoff": "sic-ortho"}


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("pot_kind", list(CLASSICAL))
def test_classical_types_changed_without_moving_atoms(oracle, eng, pot_kind, kind):  # noqa: F811
    """LJ with 3 species, EAM CuFeNi and Tersoff SiC read the species at compute time; a change still
    rebuilds once (the lists are shared), and the result equals a fresh handle and the oracle."""
    _, path, s = cc.make(CLASSICAL[pot_kind])
    nt = int(s["type"].max()) + 1
    t1, t2 = type_pair(kind, s["type"], nt)
    _, pot = classical_compute(eng, pot_kind, path, dict(s, type=t1))
    r0 = pot.num_rebuilds
    s2 = dict(s, type=t2)
    out, _ = classical_compute(eng, pot_kind, path, s2, pot=pot)
    r1 = pot.num_rebuilds
    fresh, _ = classical_compute(eng, pot_kind, path, s2)
    _same(out, fresh, what=kind)
    assert r1 == r0 + 1, (r0, r1)
    classical_compute(eng, pot_kind, path, s2, pot=pot)
    assert pot.num_rebuilds == r0 + 1
    check_vs_oracle(out, cc.oracle32(pot_kind, path, s2), s2["type"].shape[0], pot_kind, path)


def _unep_alloy(cells, seed):
    return _random_alloy("nep_UNEP_v1.txt", cells, 3.9, seed)


MCMD = {
    "PbTe": ("nep_PbTe.txt", lambda: rocksalt_pbte(4, rattle=0.02, seed=3)),
    "UNEP": ("nep_UNEP_v1.txt", lambda: _unep_alloy(6, 21)),
}


@pytest.mark.parametrize("case", list(MCMD))
def test_mcmd_like_trajectory(eng, case, monkeypatch):  # noqa: F811
    """NVE through engine.Force, and every 20 steps 5 % of the unlike pairs swap species (MCMD): the forces
    at every swap equal a fresh handle's bit for bit."""
    import torch
    _env(monkeypatch, {})
    model, make = MCMD[case]
    s = make()
    n = s["type"].shape[0]
    atom = eng.Atom(s["type"], s["pos"], np.full(n, 100.0), init_velocities(np.full(n, 100.0), 600.0, seed=8))
    box = eng.Box(s["h"], s["pbc"])
    force = eng.Force()
    pot = force.parse_potential(GOLDEN / model, n)
    ens = eng.Ensemble_NVE(n)
    thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
    args = (box, atom.position_per_atom, atom.type, atom.potential_per_atom, atom.force_per_atom,
            atom.virial_per_atom)
    force.compute(*args)
    dt = 1.0 / TIME_UNIT_CONVERSION
    rng = np.random.default_rng(4)
    for block in range(5):
        for _ in range(20):
            ens.compute1(dt, box, atom, thermo)
            force.compute(*args)
            ens.compute2(dt, box, atom, thermo)
        t = _swap(atom.type.cpu().numpy(), rng)
        atom.type.copy_(torch.as_tensor(t, device="cuda"))
        before = pot.num_rebuilds
        force.compute(*args)
        pot.check()
        pos = atom.position_per_atom.cpu().numpy().reshape(3, n)
        _, fresh = GpuNep(eng, model, n).compute(t, s["h"], s["pbc"], pos)
        got = dict(pe=atom.potential_per_atom.cpu().numpy(), force=atom.force_per_atom.cpu().numpy().reshape(3, n),
                   virial=atom.virial_per_atom.cpu().numpy().reshape(9, n))
        _same(got, fresh, what=f"swap {block}")
        assert pot.num_rebuilds == before + 1, block


# ------------------------------------------------------------------- the hidden layer in FP64 from the file

def load_ann(path):
    """The hidden layer and radial coefficients of a nep.txt (layout: tests/golden/make_synthetic_models.py),
    every parameter rounded to float32 as the library reads it."""
    lines = [ln.split() for ln in open(path) if ln.strip()]
    head = lines[0]
    version = 5 if head[0].startswith("nep5") else 4
    nt = int(head[1])
    hdr, k = {}, 1
    while lines[k][0] != "ANN":
        hdr[lines[k][0]] = lines[k][1:]
        k += 1
    nneu = int(lines[k][1])
    nr1, na1 = int(hdr["n_max"][0]) + 1, int(hdr["n_max"][1]) + 1
    kr1, ka1 = int(hdr["basis_size"][0]) + 1, int(hdr["basis_size"][1]) + 1
    lm = hdr["l_max"]
    num_L = int(lm[0]) + (int(lm[1]) != 0) + (int(lm[2]) != 0)
    dim = nr1 + na1 * num_L
    n_ann = (dim + 2) * nneu * nt + 1 if version == 4 else ((dim + 2) * nneu + 1) * nt + 1
    ntsq = nt * nt
    n_para = n_ann + ntsq * (nr1 * kr1 + na1 * ka1)
    v = np.array([float(ln[0]) for ln in lines[k + 1:k + 1 + n_para + dim]], np.float32)
    assert v.size == n_para + dim
    w0, b0, w1, bt = [], [], [], []
    p = 0
    for _ in range(nt):
        w0.append(v[p:p + nneu * dim].reshape(nneu, dim))
        p += nneu * dim
        b0.append(v[p:p + nneu])
        p += nneu
        w1.append(v[p:p + nneu])
        p += nneu
        if version == 5:
            bt.append(v[p])
            p += 1
    b1 = v[p]
    bias = np.array([np.float32(b + b1) for b in bt] if version == 5 else [b1] * nt, np.float32)
    cr = v[n_ann:n_ann + ntsq * nr1 * kr1].reshape(nr1, kr1, nt, nt)  # [(n*kr1 + k)*nt^2 + t1*nt + t2]
    k1 = next(x for x in (9, 13, 17) if x >= kr1)
    c_r = np.zeros((nt, nt, nr1, k1))
    c_r[..., :kr1] = cr.transpose(2, 3, 0, 1)
    f64 = lambda a: np.asarray(a, np.float64)  # noqa: E731
    return dict(nt=nt, nneu=nneu, dim=dim, nr1=nr1, K1R=k1, w0=f64(w0), b0=f64(b0), w1=f64(w1), bias=f64(bias),
                c_r=c_r, q_scaler=f64(v[n_para:n_para + dim]), zbl="zbl" in head[0])


def mlp_fp64(m, types, x, fp_got):
    """Per atom in FP64 from the scaled descriptors x[dim, n] the layer saw: site energy, dU/dq (times
    q_scaler) and the U table (from the exported dU/dq, so that it isolates the contraction), each with
    the sum of the magnitudes of its terms."""
    n = types.size
    E, SE = np.zeros(n), np.zeros(n)
    fp, Sfp = np.zeros((m["dim"], n)), np.zeros((m["dim"], n))
    U, SU = np.zeros((m["nt"], m["K1R"], n)), np.zeros((m["nt"], m["K1R"], n))
    qs = np.abs(m["q_scaler"])[:, None]
    for t in range(m["nt"]):
        idx = np.nonzero(types == t)[0]
        if idx.size == 0:
            continue
        X = x[:, idx]
        w0, b0, w1 = m["w0"][t], m["b0"][t][:, None], m["w1"][t][:, None]
        a = np.tanh(w0 @ X - b0)
        Z = np.abs(w0) @ np.abs(X) + np.abs(b0)  # magnitude of the first GEMM's terms
        g = 1.0 - a * a
        E[idx] = (w1 * a).sum(axis=0) - m["bias"][t]
        SE[idx] = (np.abs(w1) * (np.abs(a) + g * Z)).sum(axis=0) + abs(m["bias"][t])
        fp[:, idx] = (w0.T @ (w1 * g)) * m["q_scaler"][:, None]
        Sfp[:, idx] = (np.abs(w0).T @ (np.abs(w1) * (g + 2 * np.abs(a) * g * Z))) * qs
        F = fp_got[:m["nr1"], idx].astype(np.float64)  # [nr1, m]
        c = m["c_r"][t]  # [t2, nr1, K]
        U[:, :, idx] = np.einsum("snk,ni->ski", c, F)
        SU[:, :, idx] = np.einsum("snk,ni->ski", np.abs(c), np.abs(F))
    return dict(E=E, SE=SE, fp=fp, Sfp=Sfp, U=U, SU=SU)


def check_mlp(m, pot, types, pe, what=""):
    """The exported hidden layer against mlp_fp64 atom by atom; a failure names the atom, its tile and the
    CTA that computed it (tensor-core layer).  Returns the worst ratio |err| / sum|terms|."""
    x = pot.export_descriptors().astype(np.float64)
    fp_got, u_got = pot.export_mlp()
    ref = mlp_fp64(m, types, x, fp_got)
    where = ""
    if pot.num_tiles:
        slot, _ = pot.export_tiles()
        ctas = pot.tc_ctas

        def where(i):  # noqa: F811
            return f" atom {i}, tile {slot[i] // 128}, CTA {(slot[i] // 128) % ctas} of {ctas}"
    else:
        def where(i):  # noqa: F811
            return f" atom {i}"
    worst = 0.0
    items = [("dU/dq", fp_got, ref["fp"], ref["Sfp"]), ("U", u_got, ref["U"], ref["SU"])]
    if not m["zbl"]:
        items.append(("E", pe, ref["E"], ref["SE"]))
    for name, got, want, S in items:
        got = np.asarray(got, np.float64)
        assert np.isfinite(got).all(), (what, name)
        err = np.abs(got - want)
        ratio = err / np.maximum(S, 1e-300)
        bad = err > C_MLP * S
        if bad.any():
            flat = np.argmax(np.where(bad, ratio, -1.0))
            i = np.unravel_index(flat, err.shape)[-1]
            raise AssertionError(f"{what} {name}: |{got.flat[flat]} - {want.flat[flat]}| = {err.flat[flat]:.3e} > "
                                 f"{C_MLP} * {S.flat[flat]:.3e};{where(i)}; {int(bad.sum())} entries out")
        worst = max(worst, float(np.max(np.where(S > 0, ratio, 0.0))))
    return worst


def _alloy(model, cells, a, seed):
    return lambda: _random_alloy(model, cells, a, seed)


# model -> (file, structure factory); the shapes of the tensor-core layer per model are in DESIGN 3.4
MLP_MODELS = {
    "PbTe": ("nep_PbTe.txt", lambda: rocksalt_pbte(4, rattle=0.05, seed=1)),
    "BaZrO3": NEP_CASES["BaZrO3"],
    "BaTiO3": ("nep_BaTiO3.txt", _alloy("nep_BaTiO3.txt", 5, 4.0, 12)),
    "UNEP": NEP_CASES["UNEP"],
    "pertype_cutoff": NEP_CASES_SYNTH["pertype_cutoff"],
    "synth50": NEP_CASES_SYNTH["synth50"],
    "2sp_namax17": FEW_SPECIES_CASES["namax17"],
    "1sp_nep5": FEW_SPECIES_CASES["nep5_1sp"],  # NEP5: per-species bias
}


def u_slabs(m):
    """Slabs of the U-table GEMM inside the tensor-core layer (0: the table is left to a SIMT kernel)."""
    K1R, nt, nr1, nneu, dim = m["K1R"], m["nt"], m["nr1"], m["nneu"], m["dim"]
    N3 = (nt * ((K1R + 3) // 4 * 4) + 15) // 16 * 16
    K3 = (nr1 + 7) // 8 * 8
    if N3 > 256 or K3 > 16:
        return 0
    SC = max((nneu + 15) // 16 * 16, (dim + 15) // 16 * 16)
    return -(-N3 // SC)


@pytest.mark.parametrize("mlp", ["tc", "simt"])
@pytest.mark.parametrize("name", list(MLP_MODELS))
def test_hidden_layer_against_fp64(eng, name, mlp, monkeypatch):  # noqa: F811
    """Site energy (models without ZBL), dU/dq and the U table of every atom against the FP64 restatement,
    on the tensor-core and on the SIMT hidden layer."""
    _env(monkeypatch, {"B200MD_NEP_MLP": mlp})
    model, make = MLP_MODELS[name]
    s = make()
    n = s["type"].shape[0]
    m = load_ann(GOLDEN / model)
    pot = eng.NEP(GOLDEN / model, n)
    out = _call(eng, pot, s)
    assert (pot.tc_ctas > 0) == (mlp == "tc") and (pot.num_tiles > 0) == (mlp == "tc")
    worst = check_mlp(m, pot, s["type"], out["pe"], what=f"{name}/{mlp}")
    print(f"{name}/{mlp}: worst |err| / sum|terms| = {worst:.3e}, U-GEMM slabs {u_slabs(m)}")
    if name == "UNEP":
        assert u_slabs(m) == 3
    if name == "pertype_cutoff":
        assert u_slabs(m) == 2


# ---------------------------------------------------------------------------- many tiles per CTA

def _walks(tile_type, ctas):
    """Species of the tiles each CTA walks (tile c, c + ctas, ...)."""
    return [tile_type[c::ctas] for c in range(ctas)]


CAP_MODELS = {
    "PbTe": ("nep_PbTe.txt", lambda: rocksalt_pbte(8, rattle=0.05, seed=1), {"B200MD_NEP_MLP": "tc"}),
    "BaZrO3": ("nep_BaZrO3.txt", lambda: bazro3_supercell(4), {}),
    "UNEP": ("nep_UNEP_v1.txt", lambda: _unep_alloy(8, 22), {}),
    "pertype_cutoff": ("nep_synth_pertype_cutoff.txt", _alloy("nep_synth_pertype_cutoff.txt", 8, 4.0, 10), {}),
    "synth50": ("nep_synth_50types.txt", _alloy("nep_synth_50types.txt", 5, 4.2, 9), {}),
}


@pytest.mark.parametrize("name", list(CAP_MODELS))
def test_many_tiles_per_cta(eng, name, monkeypatch):  # noqa: F811
    """B200MD_NEP_TC_CTAS = 1, 2, 5 and unset: each capped CTA walks at least 3 tiles with a species change
    between two of them, and pe, force, virial, q, dU/dq and U are bit-identical across the caps; the
    hidden layer matches the FP64 restatement."""
    model, make, env = CAP_MODELS[name]
    s = make()
    n = s["type"].shape[0]
    m = load_ann(GOLDEN / model)
    res = {}
    for cap in (1, 2, 5, None):
        _env(monkeypatch, dict(env, **({"B200MD_NEP_TC_CTAS": str(cap)} if cap else {})))
        pot = eng.NEP(GOLDEN / model, n)
        out = _call(eng, pot, s)
        tiles, ctas = pot.num_tiles, pot.tc_ctas
        _, tile_type = pot.export_tiles()
        if cap:
            assert ctas == cap and tiles >= 3 * ctas, (cap, tiles, ctas)
            assert any(np.any(np.diff(w) != 0) for w in _walks(tile_type, ctas)), cap
        fp, u = pot.export_mlp()
        res[cap] = dict(out, q=pot.export_descriptors(), fp=fp, u=u)
        if cap is None:
            check_mlp(m, pot, s["type"], out["pe"], what=name)
    for cap in (1, 2, 5):
        for k in KEYS + ("q", "fp", "u"):
            assert np.array_equal(res[cap][k], res[None][k], equal_nan=True), (cap, k)


LARGE = {
    "UNEP": ("nep_UNEP_v1.txt", lambda: _unep_alloy(18, 23)),  # 23 328 atoms
    "BaZrO3": ("nep_BaZrO3.txt", lambda: bazro3_supercell(10)),  # 40 000 atoms
}


@pytest.mark.parametrize("name", list(LARGE))
def test_more_tiles_than_ctas_at_production_size(oracle, eng, name, monkeypatch):  # noqa: F811
    """Without a cap, at sizes where the tiles outnumber the CTAs: forces and virials against the FP64
    oracle (with the FP32 restatement's distance from it, as for block domains), the energy per atom, and
    the SIMT hidden layer."""
    model, make = LARGE[name]
    s = make()
    n = s["type"].shape[0]
    _env(monkeypatch, {})
    pot = eng.NEP(GOLDEN / model, n)
    out = _call(eng, pot, s)
    assert pot.num_tiles > pot.tc_ctas > 0, (pot.num_tiles, pot.tc_ctas)
    check_mlp(load_ann(GOLDEN / model), pot, s["type"], out["pe"], what=name)
    _env(monkeypatch, {"B200MD_NEP_MLP": "simt"})
    simt = _call(eng, eng.NEP(GOLDEN / model, n), s)
    orc = oracle.NepOracle(GOLDEN / model)
    r32 = orc.compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32)
    r64 = orc.compute(s["type"], s["h"], s["pbc"], s["pos"], precision=64)
    gap_f = np.abs(r32["force"] - r64["force"]).max()
    gap_v = np.abs(r32["virial"] - r64["virial"]).max()
    for got in (out, simt):
        check_fv(got, r64, gap_f=gap_f, gap_v=gap_v)
        gap_e = abs(r32["pe"].sum() - r64["pe"].sum()) / n
        assert abs(got["pe"].sum() - r64["pe"].sum()) / n < TOL["energy_per_atom"] + 2 * gap_e
    check_fv(out, simt)


# ------------------------------------------------------------------------------ the rule of the tiles

def check_tile_rule(slot, tile_type, types, nt, whole=True):
    """Slots unique, each in a tile of the atom's species, buckets in ascending species order, each
    starting at the running sum of the counts padded to 128, empty species without a tile.  whole=False
    (supercell): `types` are the first replica's, the buckets hold more atoms of the same species."""
    assert np.unique(slot).size == slot.size
    assert np.array_equal(tile_type[slot // 128], types)
    assert np.all(np.diff(tile_type) >= 0)
    present = np.bincount(types, minlength=nt) > 0
    assert np.array_equal(np.isin(np.arange(nt), tile_type), present)
    if not whole:
        return
    counts = np.bincount(types, minlength=nt)
    per = (counts + 127) // 128
    assert np.array_equal(tile_type, np.repeat(np.arange(nt), per))
    start = 128 * np.r_[0, np.cumsum(per)[:-1]]
    for t in range(nt):
        assert np.array_equal(np.sort(slot[types == t]), start[t] + np.arange(counts[t])), t


def _rule_structure():
    """8 788 UNEP atoms: species 0 and 15 absent, species 5 with exactly 1280 = 10 * 128 atoms, species 7
    with one atom, the rest drawn from the other species."""
    s = fcc(13, 3.9, rattle=0.08, seed=24)
    n = s["type"].shape[0]
    rng = np.random.default_rng(24)
    t = rng.choice([1, 2, 3, 4, 6, 8, 9, 10, 11, 12, 13, 14], n).astype(np.int32)
    idx = rng.permutation(n)
    t[idx[:1280]] = 5
    t[idx[1280]] = 7
    s["type"] = t
    s["symbols"] = nep_type_order(GOLDEN / "nep_UNEP_v1.txt")
    return s


def test_type_tiles_follow_the_rule(eng, monkeypatch):  # noqa: F811
    """More than 8192 atoms (the count scan carries across chunks of blocks), absent first and last species,
    a bucket of exactly 10 tiles and one of one atom; then after a displacement rebuild, after invalidate
    to fewer atoms, and through the supercell of a small box.  Two handles agree on every slot."""
    _env(monkeypatch, {})
    model = "nep_UNEP_v1.txt"
    s = _rule_structure()
    n = s["type"].shape[0]
    counts = np.bincount(s["type"], minlength=16)
    assert n > 8192 and counts[0] == 0 and counts[15] == 0 and counts[5] == 1280 and counts[7] == 1
    pots = [eng.NEP(GOLDEN / model, n) for _ in range(2)]
    slots = []
    for pot in pots:
        _call(eng, pot, s)
        slot, tile_type = pot.export_tiles()
        assert pot.num_tiles == tile_type.size == ((counts + 127) // 128).sum()
        check_tile_rule(slot, tile_type, s["type"], 16)
        slots.append(slot)
    assert np.array_equal(slots[0], slots[1])
    pot = pots[0]
    # displacement rebuild
    pos = s["pos"].copy()
    pos[0, 17] += 0.6
    r0 = pot.num_rebuilds
    _call(eng, pot, dict(s, pos=pos))
    assert pot.num_rebuilds == r0 + 1
    check_tile_rule(*pot.export_tiles(), s["type"], 16)
    # fewer atoms after invalidate: species 5 keeps its 1280 atoms at the front
    m = 6000
    order = np.r_[np.nonzero(s["type"] == 5)[0], np.nonzero(s["type"] != 5)[0]][:m]
    sub = dict(s, type=np.ascontiguousarray(s["type"][order]), pos=np.ascontiguousarray(s["pos"][:, order]))
    pot.invalidate(m)
    _call(eng, pot, sub)
    slot, tile_type = pot.export_tiles(m)
    check_tile_rule(slot, tile_type, sub["type"], 16)
    # supercell of a small box (BaZrO3, 40 atoms, 27 replicas)
    model, make = NEP_SMALL_CASES["BaZrO3_40"]
    s = make()
    n = s["type"].shape[0]
    pot = eng.NEP(GOLDEN / model, n)
    _call(eng, pot, s)
    slot, tile_type = pot.export_tiles()
    assert pot.num_tiles == tile_type.size > 0
    check_tile_rule(slot, tile_type, s["type"], 3, whole=False)


# ---------------------------------------------------------------------------------- NVE under a cap

def test_nve_with_rebuilds_under_a_cta_cap(eng, monkeypatch):  # noqa: F811
    """BaZrO3, 80 steps hot enough for displacement rebuilds, with B200MD_NEP_TC_CTAS=3 and without: the
    thermo rows and the final state are bit-identical."""
    from test_gpu_md import run_nve
    s = bazro3_supercell(3)
    s["mass"] = np.full(s["type"].shape[0], 50.0)
    runs = {}
    for cap in ("3", None):
        _env(monkeypatch, {"B200MD_NEP_TC_CTAS": cap} if cap else {})
        atom, pot, rows = run_nve(eng, s, GOLDEN / "nep_BaZrO3.txt", 80, 2.0, 1500.0, every=10)
        assert pot.num_tiles >= 3 * 3 and (pot.tc_ctas == 3 if cap else pot.tc_ctas > 3)
        runs[cap] = dict(rows=rows, rebuilds=pot.num_rebuilds, pos=atom.position_per_atom.cpu().numpy(),
                         vel=atom.velocity_per_atom.cpu().numpy(), f=atom.force_per_atom.cpu().numpy(),
                         v=atom.virial_per_atom.cpu().numpy(), pe=atom.potential_per_atom.cpu().numpy())
    assert runs["3"]["rebuilds"] >= 2 and runs["3"]["rebuilds"] == runs[None]["rebuilds"]
    for k in ("rows", "pos", "vel", "f", "v", "pe"):
        assert np.array_equal(runs["3"][k], runs[None][k]), k

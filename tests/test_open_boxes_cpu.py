"""Open boundaries beyond `slab()`: clusters, wires and ribbons with an open x or y direction, atoms outside
the box along open directions (below 0, beyond L, a cluster entirely outside, an open direction thinner than
one cell), small-box supercells that replicate only the periodic directions, N = 1, 2 and 3, and the latched
list-overflow bits at count = MN + 1 against the legal count = MN.

Open directions are never wrapped, so a molecule or nanoparticle in MD drifts out of its box.  The cell list
clamps such atoms into the end cells of the open direction (b2_cell_of), where the reference wraps the cell
id; both give the same pairs only while every atom stays inside.  Every structure here has teeth: along each
open direction the atoms stick out of the box on both sides and span more than half its length, so a
minimum image applied to an open direction, or a cell chosen by wrapping, changes the pair set.

The host build of the kernel bodies (tests/emu) and the FP32 / FP64 oracle run the structures here;
tests/test_gpu_open_boxes.py runs the same structures through every device kernel path."""
import numpy as np
import pytest

import cases_classical as cc
from cases import NEP_CASES, shear
from conftest import GOLDEN, assert_close
from gpumd_b200.structures import diamond, nep_type_order, rocksalt_pbte
from test_classical_cpu import check_vs_fp64, check_vs_oracle, emu_handle
from test_few_species_cpu import alloy
from test_kernel_bodies_cpu import check_fv, check_nep


# ---------------------------------------------------------------- structures

def open_box(s, pbc, frac=0.9, length=None, offset=None):
    """Crystal `s` (orthogonal box, atoms inside it) with the directions where `pbc` is 0 opened: the box
    length there becomes `length` (default `frac` of the crystal's extent) and the atoms are centred on it,
    so that they stick out by the same amount on both sides.  `offset` (3 values) then moves all atoms."""
    s = dict(s)
    H = s["h"].reshape(3, 3).copy()
    pos = s["pos"].copy()
    for d in range(3):
        if not pbc[d]:
            ext = H[d, d]
            L = frac * ext if length is None else length
            pos[d] -= 0.5 * (ext - L)
            H[d, d] = L
    if offset is not None:
        pos += np.asarray(offset, np.float64)[:, None]
    s.update(pos=np.ascontiguousarray(pos), h=H.reshape(9), pbc=np.array(pbc, np.int32))
    return s


def pbte(reps, seed):
    return rocksalt_pbte(reps, rattle=0.05, seed=seed)


def water_cluster(m=5, seed=63):
    """m^3 water molecules (O-H 0.9572 A, H-O-H 104.52 deg) on a 3.1 A grid, orientations and a 0.1 A jitter
    drawn from `seed`; types in the order of nep_water.txt (O, H)."""
    order = nep_type_order(GOLDEN / "nep_water.txt")
    rng = np.random.default_rng(seed)
    th = np.deg2rad(104.52) / 2
    local = 0.9572 * np.array([[0.0, 0.0, 0.0], [np.sin(th), np.cos(th), 0.0], [-np.sin(th), np.cos(th), 0.0]])
    pos, types = [], []
    for g in np.stack(np.meshgrid(*[np.arange(m)] * 3, indexing="ij"), -1).reshape(-1, 3):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        pos.append(local @ q.T + (g + 0.5) * 3.1 + rng.normal(0, 0.1, 3))
        types += [order.index("O"), order.index("H"), order.index("H")]
    L = 3.1 * m
    return dict(pos=np.ascontiguousarray(np.concatenate(pos).T), type=np.array(types, np.int32),
                h=np.diag([L] * 3).reshape(9), pbc=np.array([1, 1, 1], np.int32))


def _alloy_of(model, seed):
    """alloy() with the species drawn over all of the model's types (its symbols only set the masses)."""
    s = alloy(model, seed=seed)
    nt = len(nep_type_order(GOLDEN / model))
    s["type"] = np.random.default_rng(seed).integers(0, nt, s["type"].shape[0]).astype(np.int32)
    return s


PBTE = "nep_PbTe.txt"
# name -> (model, factory).  PbTe (rc 8 A, cells of 4.5 A): a 26.3 A crystal in a 23.7 A open box has five
# cells per open direction, where clamping and wrapping pick different cells for the atoms outside.
OPEN_PBTE = {
    "cluster_000": lambda: open_box(pbte(4, 61), (0, 0, 0)),
    "ribbon_010": lambda: open_box(pbte(4, 62), (0, 1, 0)),
    "slab_011": lambda: open_box(pbte(4, 63), (0, 1, 1)),
    "slab_101": lambda: open_box(pbte(4, 64), (1, 0, 1)),
    # periodic direction thinner than 2.5 (rc + 1): the small-box supercell replicates z only / x only
    "wire_001_short": lambda: open_box(pbte((4, 4, 2), 65), (0, 0, 1)),
    "wire_100_short": lambda: open_box(pbte((2, 4, 4), 66), (1, 0, 0)),
    # open z 4 A thick (< 0.5 (rc + 1): one cell), the crystal 13.1 A thick around it
    "thin_open_z": lambda: open_box(pbte((4, 4, 2), 67), (1, 1, 0), length=4.0),
    # every atom outside the box: x below 0, z beyond L
    "outside": lambda: open_box(pbte(4, 68), (0, 0, 0), offset=(-30.0, 0.0, 28.0)),
}
NEP_OPEN = {f"PbTe_{k}-{shape}": (PBTE, (lambda f=f, sh=sh: sh(f())))
            for k, f in OPEN_PBTE.items() for shape, sh in (("ortho", lambda s: s), ("tric", shear))}
NEP_OPEN.update({
    # 1 species, 4- and 5-body terms, rc 4.2 A
    "carbon_particle": ("nep_C_2022_NEP4.txt",
                        lambda: open_box(diamond(4, a=3.57, rattle=0.05, seed=69, symbol="C"), (0, 0, 0))),
    "water_cluster": ("nep_water.txt", lambda: open_box(water_cluster(), (0, 0, 0), frac=0.75)),
    "water_ribbon-tric": ("nep_water.txt", lambda: shear(open_box(water_cluster(6, 70), (1, 0, 0), frac=0.75))),
    "2sp_nep5_flexzbl_wire": ("nep_synth_2sp_nep5_flexzbl.txt",
                              lambda: open_box(alloy("nep_synth_2sp_nep5_flexzbl.txt", seed=71), (0, 0, 1))),
    "1sp_zbl_k17_cluster": ("nep_synth_1sp_zbl_k17.txt",
                            lambda: open_box(alloy("nep_synth_1sp_zbl_k17.txt", seed=72), (0, 0, 0))),
})
# three and more species (shared-memory accumulators, per-pair contraction, U-table GEMM at 256 columns)
NEP_OPEN_MANY = {
    "3sp_nep5_flexzbl": ("nep_synth_3sp_nep5_flexzbl.txt",
                         lambda: open_box(alloy("nep_synth_3sp_nep5_flexzbl.txt", seed=73), (0, 0, 0))),
    "3sp_nep5_flexzbl_ribbon-tric": ("nep_synth_3sp_nep5_flexzbl.txt", lambda: shear(
        open_box(alloy("nep_synth_3sp_nep5_flexzbl.txt", seed=74), (0, 1, 0)))),
    "4sp_typewise_zbl": ("nep_synth_4sp_typewise_zbl.txt",
                         lambda: open_box(alloy("nep_synth_4sp_typewise_zbl.txt", seed=75), (0, 0, 0))),
    "16sp_k13": ("nep_synth_16sp_k13.txt",
                 lambda: open_box(alloy("nep_synth_16sp_k13.txt", seed=76), (0, 1, 1))),
    "UNEP": ("nep_UNEP_v1.txt", lambda: open_box(NEP_CASES["UNEP"][1](), (0, 0, 0))),
    "synth50": ("nep_synth_50types.txt", lambda: open_box(_alloy_of("nep_synth_50types.txt", 78), (0, 0, 0))),
}


def few_atoms(n, rc, which):
    """N = 1 (a lone atom), N = 2 at 0.7 rc, N = 3 collinear (cos = -1 exactly at the middle atom, 0.45 rc
    apart: every pair radial, the end pair beyond an angular cutoff of rc / 2) in a 40 A open box, with the
    atoms near a corner so that two of them are outside it."""
    d = {1: [0.0], 2: [0.0, 0.7 * rc], 3: [0.0, 0.45 * rc, 0.9 * rc]}[n]
    pos = np.zeros((3, n))
    pos[0] = np.asarray(d) - 0.6 * rc
    pos[1] = 0.3 if which else -0.3
    pos[2] = 39.5
    return dict(pos=pos, h=np.diag([40.0] * 3).reshape(9), pbc=np.array([0, 0, 0], np.int32))


def teeth(s, rc):
    """The open directions of `s`, each checked for teeth: atoms on both sides outside the box (or all of them
    outside), an extent above half the box length, and a pair set within rc that a minimum image along that
    direction would change."""
    H = s["h"].reshape(3, 3)
    f = np.linalg.solve(H, s["pos"])
    pbc = np.asarray(s["pbc"]).astype(bool)
    n = f.shape[1]
    sub = np.random.default_rng(0).permutation(n)[:400]

    def pairs(per):
        df = f[:, sub, None] - f[:, None, sub]
        df[per] -= np.round(df[per])
        d = np.einsum("ab,bij->aij", H, df)
        return ((d * d).sum(axis=0) < rc * rc).sum()

    base = pairs(pbc)
    opened = []
    for d in np.nonzero(~pbc)[0]:
        lo, hi = f[d].min(), f[d].max()
        assert (lo < 0 and hi > 1) or lo > 1 or hi < 0, (d, lo, hi)
        assert hi - lo > 0.5, (d, hi - lo)
        per = pbc.copy()
        per[d] = True
        assert pairs(per) > base, d
        opened.append(int(d))
    return opened


@pytest.mark.parametrize("case", list(NEP_OPEN) + list(NEP_OPEN_MANY))
def test_open_structures_have_teeth(oracle, case):
    model, make = {**NEP_OPEN, **NEP_OPEN_MANY}[case]
    assert teeth(make(), model_cutoffs(model)[0])


def test_clamped_and_wrapped_cells_differ(oracle):
    """The PbTe cluster: with five cells per open direction, wrapping the cell id of an atom below 0 would
    put it four cells away from the neighbours it has in cell 0; clamping keeps it next to them.  The
    thin open direction has one cell (nb = 1)."""
    s = NEP_OPEN["PbTe_cluster_000-ortho"][1]()
    cell = 0.5 * (8.0 + 1.0)
    nb = np.floor(np.diag(s["h"].reshape(3, 3)) / cell).astype(int)
    assert (nb == 5).all()
    k = np.floor(s["pos"] / np.diag(s["h"].reshape(3, 3))[:, None] * nb[:, None]).astype(int)
    assert (k < 0).any() and (k >= nb[:, None]).any()
    t = NEP_OPEN["PbTe_thin_open_z-ortho"][1]()
    assert np.floor(t["h"][8] / cell) == 0  # make_grid raises it to nb = 1


@pytest.mark.parametrize("team", ["0", "1"])
@pytest.mark.parametrize("case", list(NEP_OPEN))
def test_open_boxes_bodies_match_oracle(oracle, emu, case, team, monkeypatch):
    """Host build of the generic kernel bodies (team: the lane-team bodies, one lane on the host): exact
    neighbour lists, descriptors, E/F/virial against the FP32 and FP64 oracle."""
    monkeypatch.setenv("B200MD_NEP_TEAM", team)
    model, make = NEP_OPEN[case]
    s = make()
    n = s["type"].shape[0]
    check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)


@pytest.mark.parametrize("case", list(NEP_OPEN_MANY))
def test_open_boxes_many_species_bodies_match_oracle(oracle, emu, case):
    model, make = NEP_OPEN_MANY[case]
    s = make()
    n = s["type"].shape[0]
    check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)


# ---------------------------------------------------------------- N = 1, 2, 3

FEW_ATOM_MODELS = {"1sp": "nep_synth_1sp_zbl_k17.txt", "2sp": PBTE, "3sp": "nep_synth_3sp_nep5_flexzbl.txt",
                   "16sp": "nep_synth_16sp_k13.txt"}


def model_cutoffs(model):
    toks = next(ln for ln in open(GOLDEN / model) if ln.startswith("cutoff")).split()
    return float(toks[1]), float(toks[2])


def few_atom_case(model, n, which=0):
    rc_r, _ = model_cutoffs(model)
    s = few_atoms(n, rc_r, which)
    nt = len(nep_type_order(GOLDEN / model))
    s["type"] = (np.arange(n) * 7 + which) % nt
    s["type"] = s["type"].astype(np.int32)
    return s


def lone_atom_energy(model, t):
    """ann(q = 0): the site energy of an atom without neighbours, from the model's weights in FP64."""
    from test_gpu_nep_species import load_ann
    m = load_ann(GOLDEN / model)
    return float((m["w1"][t] * np.tanh(-m["b0"][t])).sum() - m["bias"][t])


def check_few_atoms(oracle, dev, model, s):
    n = s["type"].shape[0]
    out = check_nep(oracle, dev, model, s, n)
    if n == 1:
        assert abs(out["pe"][0] - lone_atom_energy(model, int(s["type"][0]))) < 1e-6 * max(1.0, abs(out["pe"][0]))
        assert not out["force"].any() and not out["virial"].any()
    else:
        assert np.abs(out["force"].sum(axis=1)).max() < 1e-5 * max(1.0, np.abs(out["force"]).max())
        assert np.abs(out["force"]).max() > 0
    if n == 3:  # collinear along x: no force or virial component off the axis
        assert not out["force"][1:].any()
        assert not out["virial"][[1, 2, 3, 4, 5, 6, 7, 8]].any()
    return out


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("case", list(FEW_ATOM_MODELS))
def test_one_two_three_atoms(oracle, emu, case, n, which):
    model = FEW_ATOM_MODELS[case]
    s = few_atom_case(model, n, which)
    check_few_atoms(oracle, emu.nep(GOLDEN / model, n), model, s)


# ---------------------------------------------------------------- LJ / Tersoff / EAM

# potential -> (kind, file, crystal): periodic thicknesses above 2.5 (rc + 1) (the classical potentials have
# no supercell path), the open directions 0.9 of the crystal's extent
CLASSICAL = {
    "lj": ("lj", cc.LJ3, lambda: cc._lj3_alloy(81)),
    "tersoff": ("tersoff", cc.SIC, lambda: cc._sic(5, 82)),
    "eam": ("eam", GOLDEN / cc.EAM_FILES["cufeni"], lambda: cc._eam("cufeni", 3.615, 83)),
}
CLASSICAL_PBC = {"000": (0, 0, 0), "011": (0, 1, 1), "101": (1, 0, 1), "010": (0, 1, 0), "001": (0, 0, 1)}
CLASSICAL_CASES = [f"{p}-{b}-{sh}" for p in CLASSICAL for b in CLASSICAL_PBC for sh in ("ortho", "tric")]


def classical_case(case):
    pot, b, sh = case.split("-")
    kind, path, make = CLASSICAL[pot]
    s = open_box(make(), CLASSICAL_PBC[b])
    return kind, path, shear(s) if sh == "tric" else s


@pytest.mark.parametrize("case", CLASSICAL_CASES)
def test_classical_open_boxes_bodies(oracle, emu, case):
    """Host build of the LJ / Tersoff / EAM bodies against the FP32 oracle and the FP64 references, with the
    tolerances of test_gpu_classical.py."""
    kind, path, s = classical_case(case)
    assert teeth(s, cc.cutoff(kind, path))
    n = s["type"].shape[0]
    r32 = cc.oracle32(kind, path, s)
    r64 = cc.reference64(kind, path, s, f32_params=True)
    rc, out = emu_handle(emu, kind, path, n).compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    check_vs_oracle(out, r32, n, kind, path)
    check_vs_fp64(out, r64, n, kind, path, gap=cc.gaps(r32, r64))


# ---------------------------------------------------------------- list overflow

def fib_sphere(m, r, centre):
    """m points spread over a sphere of radius r (Fibonacci lattice)."""
    k = np.arange(m) + 0.5
    z = 1 - 2 * k / m
    phi = np.pi * (1 + 5 ** 0.5) * k
    rho = np.sqrt(1 - z * z)
    return np.asarray(centre)[:, None] + r * np.stack([rho * np.cos(phi), rho * np.sin(phi), z])


def shell(m, r, types=None):
    """One atom at the centre of a shell of m atoms at distance r, in an all-open 40 A box: the centre has
    exactly m neighbours within any cutoff above r, every shell atom far fewer."""
    pos = np.concatenate([np.array([[20.0], [20.0], [20.0]]), fib_sphere(m, r, (20.0, 20.0, 20.0))], axis=1)
    t = np.zeros(m + 1, np.int32) if types is None else types(m + 1)
    return dict(pos=np.ascontiguousarray(pos), type=t, h=np.diag([40.0] * 3).reshape(9),
                pbc=np.array([0, 0, 0], np.int32))


def small_mn_model(model, tmp_path, mnr, mna):
    """A copy of `model` with the MN fields of its `cutoff` line set to (mnr, mna): MN = ceil(1.25 field)."""
    lines = (GOLDEN / model).read_text().splitlines()
    k = next(i for i, ln in enumerate(lines) if ln.startswith("cutoff"))
    lines[k] = " ".join(lines[k].split()[:-2] + [str(mnr), str(mna)])
    out = tmp_path / f"mn_{mnr}_{mna}_{model}"
    out.write_text("\n".join(lines) + "\n")
    return out


# (MN fields, MN_radial, MN_angular): 16 -> 20, 8 -> 10
MNR_FIELD, MNA_FIELD, MN_R, MN_A = 16, 8, 20, 10


def skin_capacity(rc, mn_radial):
    """The skin-list capacity of a NEP handle: MN_radial ((rc + 1) / rc)^3, truncated (b2_nep.cu)."""
    return int(mn_radial * (rc + 1.0) ** 3 / rc ** 3)


def overflow_shell(model, bit, extra):
    """The shell whose centre has capacity + extra entries in the list of error bit `bit` (1 skin, 2 radial,
    4 angular) and no more than its capacity in the other lists: skin entries at rc_r + 0.5 (outside the
    radial cutoff), radial at (rc_a + rc_r) / 2, angular at 0.75 rc_a."""
    rc_r, rc_a = model_cutoffs(model)
    nt = len(nep_type_order(GOLDEN / model))
    mn = {1: skin_capacity(rc_r, MN_R), 2: MN_R, 4: MN_A}[bit]
    r = {1: rc_r + 0.5, 2: 0.5 * (rc_r + rc_a), 4: 0.75 * rc_a}[bit]
    return shell(mn + extra, r, lambda m: (np.arange(m) % nt).astype(np.int32))


def overflow_models(tmp_path):
    """1 species, 2 species (the few-species kernels) and 3 species."""
    return {name: small_mn_model(model, tmp_path, MNR_FIELD, MNA_FIELD)
            for name, model in (("1sp", "nep_synth_1sp_zbl_k17.txt"), ("2sp", PBTE),
                                ("3sp", "nep_synth_3sp_nep5_flexzbl.txt"))}


def test_overflow_shells_reach_one_list_only(oracle, tmp_path):
    """The construction: at count = MN + 1 the centre exceeds exactly one capacity, every other count of every
    atom stays within its capacity (so one error bit, and one atom, is what the tests below see)."""
    for name, model in overflow_models(tmp_path).items():
        rc_r, rc_a = model_cutoffs(model.name.split("_", 3)[3])
        for bit in (1, 2, 4):
            s = overflow_shell(model.name.split("_", 3)[3], bit, 1)
            r = oracle.NepOracle(model).compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32, lists=True)
            skin, _ = oracle.neighbor_list(s["h"], s["pbc"], s["pos"], rc_r + 1.0, mn=1024)
            caps = {1: skin_capacity(rc_r, MN_R), 2: MN_R, 4: MN_A}
            counts = {1: skin, 2: r["NN_radial"], 4: r["NN_angular"]}
            for b, c in counts.items():
                over = np.nonzero(c > caps[b])[0]
                assert list(over) == ([0] if b == bit else []), (name, bit, b, c.max(), caps[b])
            assert counts[bit][0] == caps[bit] + 1


@pytest.mark.parametrize("team", ["0", "1"])
@pytest.mark.parametrize("bit", [1, 2, 4])
@pytest.mark.parametrize("name", ["1sp", "2sp", "3sp"])
def test_list_overflow_bits_bodies(oracle, emu, tmp_path, name, bit, team, monkeypatch):
    """count = MN + 1 at one atom latches exactly that list's bit; count = MN latches nothing and the result
    equals the oracle's."""
    monkeypatch.setenv("B200MD_NEP_TEAM", team)
    model = overflow_models(tmp_path)[name]
    base = model.name.split("_", 3)[3]
    s = overflow_shell(base, bit, 1)
    dev = emu.nep(model, s["type"].shape[0])
    dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert emu.E.emu_nep_error_bits(dev.h) == bit
    s = overflow_shell(base, bit, 0)
    n = s["type"].shape[0]
    dev = emu.nep(model, n)
    check_nep(oracle, dev, model, s, n)
    assert emu.E.emu_nep_error_bits(dev.h) == 0


TERSOFF_MAXL = 32  # B2_TERSOFF_MAXL


def tersoff_shell(extra):
    """Si: the centre with 32 + extra neighbours at 2.5 A (inside the 3.0 A cutoff)."""
    return shell(TERSOFF_MAXL + extra, 2.5)


def test_tersoff_angular_overflow_bodies(oracle, emu):
    """Tersoff's local list holds 32 neighbours: 33 latch B2_ERR_ANGULAR_OVERFLOW, 32 are legal and match the
    oracle."""
    s = tersoff_shell(1)
    n = s["type"].shape[0]
    dev = emu.tersoff(cc.SI, n)
    rc, _ = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc != 0 and emu.E.emu_tersoff_error_bits(dev.h) == 4
    s = tersoff_shell(0)
    n = s["type"].shape[0]
    dev = emu.tersoff(cc.SI, n)
    rc, out = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0 and emu.E.emu_tersoff_error_bits(dev.h) == 0
    check_vs_oracle(out, cc.oracle32("tersoff", cc.SI, s), n, "tersoff", cc.SI)


# LJ and EAM: the skin list is their only list.  Its capacity is k ((rc + 1) / rc)^3 entries, k = 700 (LJ) /
# 400 (EAM) (b2_setup.h), or with B200MD_TIGHT_LISTS=1 what a sphere of
# rc + 1 holds at 0.06 / 0.2 atoms per A^3, plus 32.  The shell then puts ~930 / ~620 (~370 / ~320) atoms
# 0.5 A outside the cutoff of the centre: about one atom per 1.1 A^2 of the sphere at most, a finite, if
# unphysical, density.
SKIN_POT = {"lj": (cc.LJ1, 700, 0.06), "eam": (GOLDEN / cc.EAM_FILES["cu_zhou"], 400, 0.2)}


def classical_skin_capacity(kind, tight):
    """The expressions of b2_setup.h (EAM holds its cutoff in float)."""
    path, k, dens = SKIN_POT[kind]
    rc = cc.cutoff(kind, path)
    if kind == "eam":
        rc = float(np.float32(rc))
    rs = rc + 1.0
    return int(4.19 * rs * rs * rs * dens) + 32 if tight else int(k * rs * rs * rs / (rc * rc * rc))


def skin_shell(kind, extra, tight):
    path = SKIN_POT[kind][0]
    return shell(classical_skin_capacity(kind, tight) + extra, cc.cutoff(kind, path) + 0.5)


@pytest.mark.parametrize("kind", list(SKIN_POT))
def test_classical_skin_overflow_bodies(oracle, emu, kind, monkeypatch):
    """count = capacity + 1 latches B2_ERR_SKIN_OVERFLOW; count = capacity is legal and matches the oracle, for
    the default and the B200MD_TIGHT_LISTS=1 capacity."""
    path = SKIN_POT[kind][0]
    for tight in (False, True):
        if tight:
            monkeypatch.setenv("B200MD_TIGHT_LISTS", "1")
        else:
            monkeypatch.delenv("B200MD_TIGHT_LISTS", raising=False)
        s = skin_shell(kind, 1, tight)
        dev = emu_handle(emu, kind, path, s["type"].shape[0])
        rc, _ = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
        assert rc != 0 and getattr(emu.E, f"emu_{kind}_error_bits")(dev.h) == 1
        s = skin_shell(kind, 0, tight)
        n = s["type"].shape[0]
        dev = emu_handle(emu, kind, path, n)
        rc, out = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
        assert rc == 0 and getattr(emu.E, f"emu_{kind}_error_bits")(dev.h) == 0
        r = cc.oracle32(kind, path, s)
        if tight:
            check_vs_oracle(out, r, n, kind, path)
        else:  # ~1.2 A apart: site energies of 1e4 - 1e5 eV, so only the relative parts of the tolerances apply
            assert_close(out["pe"], r["pe"], rtol=1e-5, atol=1e-5, what="pe")
            check_fv(out, r)

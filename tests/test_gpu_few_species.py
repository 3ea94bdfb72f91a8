"""The one- and two-species NEP kernels (k_desc_radial2, k_desc_angular2, k_force_angular2, k_force_final2 and
the hidden-layer kernels before them) on every model feature and kernel instance they dispatch: species count
1 or 2, K1 = 9 / 13 / 17, orthogonal / triclinic / open boundaries, tensor-core or SIMT hidden layer.  These
kernels are device-only, so the host build of the kernel bodies never runs them.  Each case asserts exact
neighbour lists, the descriptors, and E/F/virial against the FP32 and the FP64 oracle (check_nep)."""
import numpy as np
import pytest

from cases import NEP_CASES, shear, slab
from conftest import GOLDEN
from gpumd_b200.structures import fcc
from test_few_species_cpu import FEW_SPECIES_CASES, alloy
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)
from test_kernel_bodies_cpu import check_nep

pytestmark = pytest.mark.gpu

# the synthetic one- and two-species models, plus the shipped PbTe (2 species, K1 = 9/9) and carbon
# (1 species, K1 = 13/9, 4- and 5-body terms) models
MODELS = dict(FEW_SPECIES_CASES, PbTe=NEP_CASES["PbTe"], carbon=NEP_CASES["carbon"])
BOXES = {"ortho": lambda s: s, "triclinic": shear, "slab": slab}


def _run(oracle, eng, model, s):  # noqa: F811
    n = s["type"].shape[0]
    return check_nep(oracle, GpuNep(eng, model, n), model, s, n)


@pytest.mark.parametrize("mlp", ["tc", "simt"])
@pytest.mark.parametrize("box", list(BOXES))
@pytest.mark.parametrize("case", list(MODELS))
def test_few_species_kernels_match_oracle(oracle, eng, case, box, mlp, monkeypatch):  # noqa: F811
    """Every model x box shape (ORTHO = true / false instances; open z) x hidden layer (k_mlp_tc or k_mlp)."""
    monkeypatch.setenv("B200MD_NEP_MLP", mlp)
    model, make = MODELS[case]
    _run(oracle, eng, model, BOXES[box](make()))


@pytest.mark.parametrize("case", list(MODELS))
def test_few_species_simt_u_table(oracle, eng, case, monkeypatch):  # noqa: F811
    """The U table from k_utable instead of k_mlp_tc's third GEMM."""
    monkeypatch.setenv("B200MD_NEP_UTABLE", "simt")
    model, make = MODELS[case]
    _run(oracle, eng, model, make())


@pytest.mark.parametrize("box", list(BOXES))
@pytest.mark.parametrize("case", list(MODELS))
def test_few_species_kernels_equal_generic_kernels(eng, case, box, monkeypatch):  # noqa: F811
    """B200MD_NEP_RADIAL=v1 runs the generic kernels; the few-species kernels keep their per-pair arithmetic op
    for op (DESIGN.md 3.2, 3.4), so energies, forces and virials are bit-identical."""
    model, make = MODELS[case]
    s = BOXES[box](make())
    n = s["type"].shape[0]
    a = GpuNep(eng, model, n).compute(s["type"], s["h"], s["pbc"], s["pos"])[1]
    monkeypatch.setenv("B200MD_NEP_RADIAL", "v1")
    b = GpuNep(eng, model, n).compute(s["type"], s["h"], s["pbc"], s["pos"])[1]
    for k in ("pe", "force", "virial"):
        assert np.array_equal(a[k], b[k]), (k, np.abs(a[k] - b[k]).max())


@pytest.mark.parametrize("species", [0, 1])
@pytest.mark.parametrize("case", ["nep5_flexzbl", "pertype_cut", "PbTe"])
def test_two_species_model_with_one_species_present(oracle, eng, case, species):  # noqa: F811
    """A species absent from the structure: its type tiles are empty and every pair takes one cutoff row."""
    model, make = MODELS[case]
    s = make()
    s["type"] = np.full_like(s["type"], species)
    _run(oracle, eng, model, s)


def _dilute_37(seed=7):
    """37 atoms in a 24 A box (N below one 128-atom tile): one atom without neighbours, a dimer (1 angular
    neighbour each), a triangle (2 each), and 31 atoms at least 1.8 A apart that keep 4.5 A from those six
    and 5.5 A from the lone atom."""
    rng = np.random.default_rng(seed)
    L = 24.0
    fixed = [(12.0, 12.0, 12.0),                                     # lone atom
             (3.0, 3.0, 3.0), (4.8, 3.0, 3.0),                       # dimer, 1.8 A (inside the ZBL range)
             (3.0, 20.0, 3.0), (5.2, 20.0, 3.0), (4.1, 21.9, 3.0)]   # triangle, sides 2.2 A
    pos = [np.array(p) for p in fixed]

    def dist(a, b):
        d = a - b
        d -= L * np.round(d / L)
        return np.sqrt((d * d).sum())

    while len(pos) < 37:
        p = rng.uniform(0, L, 3)
        if dist(p, pos[0]) > 5.5 and all(dist(p, q) > 4.5 for q in pos[1:6]) and \
           all(dist(p, q) > 1.8 for q in pos[6:]):
            pos.append(p)
    pos = np.array(pos).T
    return dict(pos=np.ascontiguousarray(pos), type=rng.integers(0, 2, 37).astype(np.int32),
                h=np.diag([L] * 3).reshape(9).astype(np.float64), pbc=np.array([1, 1, 1], np.int32))


@pytest.mark.parametrize("case", ["nep5_flexzbl", "zbl_k17", "pertype_cut"])
def test_dilute_box_with_0_1_2_angular_neighbours(oracle, eng, case):  # noqa: F811
    """N = 37 in a large box: the prefetch guards of the angular loops (nn > 1, m + 2 < nn) with lists of
    length 0, 1 and 2, and a tile that is mostly padding."""
    model, _ = MODELS[case]
    s = _dilute_37()
    if case == "zbl_k17":
        s["type"][:] = 0
    r = oracle.NepOracle(GOLDEN / model).compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32, lists=True)
    assert r["NN_radial"][0] == 0 and list(r["NN_angular"][:6]) == [0, 1, 1, 2, 2, 2]
    _run(oracle, eng, model, s)


@pytest.mark.parametrize("case", ["nep5_flexzbl", "nep5_1sp"])
def test_atom_count_not_a_multiple_of_128(oracle, eng, case):  # noqa: F811
    """N = 1000: 1372 fcc sites with 372 drawn out at random (a partial last tile per species)."""
    model, _ = MODELS[case]
    s = alloy(model, cells=7, seed=51)
    keep = np.sort(np.random.default_rng(52).permutation(s["type"].shape[0])[:1000])
    s = dict(s, pos=np.ascontiguousarray(s["pos"][:, keep]), type=s["type"][keep])
    _run(oracle, eng, model, s)


@pytest.mark.parametrize("case", ["pertype_cut", "nep5_flexzbl"])
def test_dense_two_species_reverse_slot_tail(oracle, eng, case):  # noqa: F811
    """fcc a = 2.9 A: nearly every atom has more than 8 angular neighbours, so the reverse-slot search of
    k_force_angular2 runs its tail loop (q = 8 ... cj) for almost every pair."""
    model, _ = MODELS[case]
    s = alloy(model, cells=7, a=2.9, rattle=0.1, seed=53)
    r = oracle.NepOracle(GOLDEN / model).compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32, lists=True)
    assert (r["NN_angular"] > 8).mean() > 0.99 and r["NN_angular"].max() > 24
    _run(oracle, eng, model, s)


def test_per_species_cutoff_boundary_membership(oracle, eng):  # noqa: F811
    """Pairs placed within a few ulps of each of the three radial (5.0 / 4.6 / 4.2 A) and angular
    (4.0 / 3.7 / 3.4 A) pair cutoffs of the per-species-cutoff model: the few-species kernels pick the cutoff
    by the neighbour's type tag, and the lists must equal the oracle's exactly."""
    model = "nep_synth_2sp_pertype_cut.txt"
    base = fcc(4, 8.0, rattle=0.0, seed=1)  # 256 atoms, 5.66 A nearest neighbours
    pos = base["pos"].copy()
    n = pos.shape[1]
    ty = np.zeros(n, np.int32)
    rng = np.random.default_rng(9)
    kinds = [((0, 0), 5.0), ((0, 1), 4.6), ((1, 1), 4.2), ((0, 0), 4.0), ((1, 0), 3.7), ((1, 1), 3.4)]
    for k in range(120):
        i, j = 2 * k, 2 * k + 1
        (ti, tj), rc = kinds[k % 6]
        ty[i], ty[j] = ti, tj
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        eps = rng.integers(-6, 7) * 0.5 * float(np.spacing(np.float32(rc)))
        pos[:, j] = pos[:, i] + u * (rc + eps)
    pos = np.mod(pos, base["h"][0])
    r = oracle.NepOracle(GOLDEN / model).compute(ty, base["h"], base["pbc"], pos, precision=32, lists=True)
    dev = GpuNep(eng, model, n)
    dev.compute(ty, base["h"], base["pbc"], pos)
    NNr, NLr, NNa, NLa = dev.neighbors(r["NL_radial"].shape[1], r["NL_angular"].shape[1])
    assert np.array_equal(NNr, r["NN_radial"]) and np.array_equal(NLr, r["NL_radial"])
    assert np.array_equal(NNa, r["NN_angular"]) and np.array_equal(NLa, r["NL_angular"])
    # the construction produced boundary cases on both sides of every one of the six cutoffs
    for kind in range(6):
        ks = range(kind, 120, 6)
        lists = (NNr, NLr) if kind < 3 else (NNa, NLa)
        inside = [(2 * k + 1) in lists[1][2 * k, :lists[0][2 * k]] for k in ks]
        assert 0 < sum(inside) < len(inside), kinds[kind]


@pytest.mark.parametrize("case", ["pertype_cut", "zbl_k17"])
def test_angular_list_overflow_is_reported(eng, case, tmp_path):  # noqa: F811
    """More angular neighbours than MN_angular: check() raises (B2_ERR_ANGULAR_OVERFLOW) instead of returning
    numbers.  The model is a copy with `cutoff ... 100 8` (MN_angular = 10); the structure has ~35."""
    model, make = MODELS[case]
    lines = (GOLDEN / model).read_text().splitlines()
    k = next(i for i, ln in enumerate(lines) if ln.startswith("cutoff"))
    lines[k] = " ".join(lines[k].split()[:-1] + ["8"])
    small = tmp_path / model
    small.write_text("\n".join(lines) + "\n")
    s = make()
    dev = GpuNep(eng, small, s["type"].shape[0])
    with pytest.raises(Exception, match=r"bits=4\b"):
        dev.compute(s["type"], s["h"], s["pbc"], s["pos"])

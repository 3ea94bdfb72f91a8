"""NEP models with three to sixteen species on the features and kernel instances no shipped many-species model
reaches: NEP5 per-species bias, flexible / universal / typewise ZBL with more than two species, K1 = 13 and 17,
n_max_angular = 17, the fused neighbour split with K1 = 13 / 17, the per-pair radial contraction chosen by
itself, the U-table GEMM at its 256-column limit, unstaged angular coefficients, and hidden layers of 64 to
128 padded descriptor components (synthetic models, tests/golden/make_synthetic_models.py).  The oracle is
pinned to the reference's own codes on them (NEP_CPU where it reads the model, else the reference gpumd), and
the host build of the generic kernel bodies is checked against the oracle on orthogonal, triclinic and open
boxes.  tests/test_gpu_many_species.py runs the same cases through the device kernels."""
import numpy as np
import pytest

from cases import shear, slab
from conftest import GOLDEN, assert_close
from test_few_species_cpu import alloy

# name -> (model file, structure factory).  The 8 A models need a box above 2.5 * (8 + 1) A (else the
# small-box supercell path runs): 8 fcc cells of 3.1 A, 2048 atoms.  The others: 6 cells, 864 atoms.
MANY_SPECIES_CASES = {
    # NEP5 (per-species bias), flexible ZBL with its 6 pair rows, K1 = 13/13, 4- and 5-body terms
    "3sp_nep5_flexzbl": ("nep_synth_3sp_nep5_flexzbl.txt",
                         lambda: alloy("nep_synth_3sp_nep5_flexzbl.txt", seed=71)),
    # universal ZBL with the typewise outer cutoff: Li / Mg / Al / Si, 10 pairs, 6 of them below the 2.2 A cap
    "4sp_typewise_zbl": ("nep_synth_4sp_typewise_zbl.txt",
                         lambda: alloy("nep_synth_4sp_typewise_zbl.txt", seed=72)),
    # universal ZBL, K1 = 17/17, rc 8 A: the neighbour split fused into the radial descriptor pass
    "5sp_zbl_k17_rc8": ("nep_synth_5sp_zbl_k17_rc8.txt",
                        lambda: alloy("nep_synth_5sp_zbl_k17_rc8.txt", cells=8, seed=73)),
    # n_max_angular = 17, K1 = 17/17: 64-thread angular force blocks
    "3sp_namax17": ("nep_synth_3sp_namax17.txt", lambda: alloy("nep_synth_3sp_namax17.txt", seed=74)),
    # 16 species, K1 = 13/9: per-pair radial contraction by default, U-table GEMM with nt * KP = 256 columns,
    # angular coefficients read from global memory
    "16sp_k13": ("nep_synth_16sp_k13.txt", lambda: alloy("nep_synth_16sp_k13.txt", seed=75)),
    # 8 species, K1 = 13/13, n_max 19 15, D = 116 (k_mlp<128>), rc 8 A: fused split, no tensor-core layer
    "8sp_wide": ("nep_synth_8sp_wide.txt", lambda: alloy("nep_synth_8sp_wide.txt", cells=8, seed=76)),
}

BOXES = {"ortho": lambda s: s, "triclinic": shear, "slab": slab}

# B200MD_NEP_RADREG=1: NT of the register-accumulator instance (NT * K1 <= 160 registers)
RADREG_NT = {"3sp_nep5_flexzbl": 4, "5sp_zbl_k17_rc8": 8, "3sp_namax17": 4, "8sp_wide": 8}


def check_case(oracle, dev, case, s):
    """check_nep on a case; the 8 A models (~300 radial neighbours) with the FP32 restatement's own distance
    from FP64 added to the descriptor tolerance (check_nep's q_gap)."""
    from test_kernel_bodies_cpu import check_nep
    model, _ = MANY_SPECIES_CASES[case]
    return check_nep(oracle, dev, model, s, s["type"].shape[0], q_gap="rc8" in case or case == "8sp_wide")

# NEP_CPU (oracle/_ref/libnep_cpu_ref.so) reads these models as they are; its results on the case's structure
# with seed 41 are stored in tests/golden/ref_nep_cpu_many_species.npz (tests/golden/make_fixtures.py).
# Two are not among them: the reference sizes its per-atom arrays for n_max <= 16 (MAX_NUM_N = 17), which
# 3sp_namax17 and 8sp_wide exceed, and for D <= 103 (MAX_DIM), which 8sp_wide (D = 116) exceeds.
NEP_CPU_MANY_SPECIES = ["3sp_nep5_flexzbl", "5sp_zbl_k17_rc8", "16sp_k13"]

# typewise ZBL, which NEP_CPU evaluates differently from nep.cu (rc_inner = rc_outer / 2 there, 0 in nep.cu),
# and flexible ZBL, so that its (1, 2) row is pinned by both reference codes: single points of the unmodified
# reference gpumd on an H100 80GB HBM3, scripts/run_reference_gpumd.py -> tests/golden/refgpu_<case>.npz
REFGPU_MANY_SPECIES = {
    "sp_4sp_typewise_zbl": "nep_synth_4sp_typewise_zbl.txt",
    "sp_3sp_nep5_flexzbl": "nep_synth_3sp_nep5_flexzbl.txt",
}

# covalent radii of the typewise-ZBL model's species in the reference's table (nep.cu, COVALENT_RADIUS)
COVALENT = {"Li": 1.6, "Mg": 1.66667, "Al": 1.50667, "Si": 1.46667}


def nep_cpu_many_species_structure(case):
    model, _ = MANY_SPECIES_CASES[case]
    return alloy(model, cells=8 if "rc8" in case else 6, seed=41)


@pytest.mark.parametrize("case", NEP_CPU_MANY_SPECIES)
def test_oracle_matches_reference_nep_cpu_many_species(oracle, case):
    """FP64 restatement vs the reference's NEP_CPU, with the tolerances of
    test_few_species_cpu.py::test_oracle_matches_reference_nep_cpu_few_species."""
    model, _ = MANY_SPECIES_CASES[case]
    s = nep_cpu_many_species_structure(case)
    g = np.load(GOLDEN / "ref_nep_cpu_many_species.npz")
    ref = {k: g[f"{case}_{k}"] for k in ("pe", "force", "virial")}
    r = oracle.NepOracle(GOLDEN / model).compute(s["type"], s["h"], s["pbc"], s["pos"], precision=64)
    n = s["type"].shape[0]
    assert ref["pe"].shape == (n,)
    assert abs(r["pe"].sum() - ref["pe"].sum()) / n < 1e-7
    assert_close(r["force"], ref["force"], rtol=1e-6, atol=5e-7, what="force")
    assert_close(r["virial"], ref["virial"], rtol=1e-5, atol=5e-6, what="virial")


@pytest.mark.parametrize("case", list(REFGPU_MANY_SPECIES))
def test_oracle_matches_reference_gpu_many_species(oracle, case):
    """FP32 restatement vs the reference gpumd's own single point, with the tolerances of
    test_few_species_cpu.py::test_oracle_matches_reference_gpu_few_species (force atol scaled by the largest
    force component, which the ZBL pairs make large)."""
    d = np.load(GOLDEN / f"refgpu_{case}.npz")
    n = d["type"].shape[0]
    r = oracle.NepOracle(GOLDEN / REFGPU_MANY_SPECIES[case]).compute(
        d["type"], d["h"], d["pbc"], d["pos"], precision=32)
    assert abs(r["pe"].sum() - float(d["energy"])) / n < 2e-7
    fs = max(1.0, np.abs(d["force"]).max())
    assert_close(r["force"], d["force"], rtol=1e-5, atol=1e-5 * fs, what="force")
    v = r["virial"].sum(axis=1)
    v33 = np.array([v[0], v[3], v[4], v[6], v[1], v[5], v[7], v[8], v[2]])
    assert_close(v33, d["virial"], rtol=1e-5, atol=5e-3, what="virial")


def zbl_outer_cutoffs(model):
    """[nt, nt] outer ZBL cutoff of every species pair as nep.cu takes it: the flexible table's rc_outer of
    row ta * nt - ta (ta - 1) / 2 + (tb - ta) (ta <= tb), min(factor * (r_a + r_b), rc_outer) for typewise
    ZBL, else the global rc_outer."""
    lines = [ln.split() for ln in open(GOLDEN / model) if ln.strip()]
    syms = lines[0][2:]
    nt = len(syms)
    zbl = next(ln for ln in lines[1:4] if ln[0] == "zbl")
    rc = np.zeros((nt, nt))
    if zbl[1:] == ["0", "0"]:
        table = np.array([float(ln[0]) for ln in lines[-5 * nt * (nt + 1):]]).reshape(-1, 10)
        for ta in range(nt):
            for tb in range(ta, nt):
                rc[ta, tb] = rc[tb, ta] = table[ta * nt - ta * (ta - 1) // 2 + (tb - ta), 1]
    elif len(zbl) == 4:
        for ta in range(nt):
            for tb in range(nt):
                rc[ta, tb] = min(float(zbl[3]) * (COVALENT[syms[ta]] + COVALENT[syms[tb]]), float(zbl[2]))
    else:
        rc[:] = float(zbl[2])
    return rc


def test_many_species_features_are_active(oracle):
    """The structures reach what the models exist for.  Every ordered species pair, (1, 2) included, has more
    than 100 radial pairs, so a wrong coefficient row or cutoff changes the result.  In the ZBL models every
    unordered species pair has pairs inside its own outer ZBL cutoff, so a wrong flexible-ZBL row or typewise
    cutoff does too; the six flexible rows and the typewise cutoffs are distinct."""
    for case, (model, make) in MANY_SPECIES_CASES.items():
        s = make()
        t = s["type"]
        nt = int(open(GOLDEN / model).readline().split()[1])
        assert np.array_equal(np.unique(t), np.arange(nt)), case
        r = oracle.NepOracle(GOLDEN / model).compute(t, s["h"], s["pbc"], s["pos"], precision=32, lists=True)
        counts = np.zeros((nt, nt), int)
        for i in range(t.size):
            np.add.at(counts[t[i]], t[r["NL_radial"][i, :r["NN_radial"][i]]], 1)
        assert counts.min() > 100, (case, counts.min())
        if "zbl" not in case:
            continue
        rc = zbl_outer_cutoffs(model)
        pos, L = s["pos"], s["h"][0]
        inside = np.zeros((nt, nt), int)
        for i in range(t.size):
            d = pos - pos[:, i:i + 1]
            d -= L * np.round(d / L)
            r2 = (d * d).sum(axis=0)
            r2[i] = np.inf
            np.add.at(inside[t[i]], t[r2 < rc[t[i], t] ** 2], 1)
        assert inside.min() >= 10, (case, inside)
        if "flexzbl" in case or "typewise" in case:
            iu = np.triu_indices(nt)
            assert np.unique(rc[iu]).size >= (nt * (nt + 1) // 2 if "flexzbl" in case else 4), (case, rc)


@pytest.mark.parametrize("box", list(BOXES))
@pytest.mark.parametrize("case", list(MANY_SPECIES_CASES))
def test_many_species_bodies_match_oracle(oracle, emu, case, box):
    """Host build of the generic kernel bodies (k_split, k_desc_radial, k_desc_angular, k_mlp, k_utable,
    k_force_angular, k_force_final), every model x box shape."""
    model, make = MANY_SPECIES_CASES[case]
    s = BOXES[box](make())
    check_case(oracle, emu.nep(GOLDEN / model, s["type"].shape[0]), case, s)


@pytest.mark.parametrize("switch", ["B200MD_NEP_RADREG", "B200MD_NEP_RADDIRECT"])
@pytest.mark.parametrize("case", ["3sp_nep5_flexzbl", "5sp_zbl_k17_rc8", "8sp_wide", "3sp_namax17"])
def test_many_species_radial_opt_ins_bodies(oracle, emu, case, switch, monkeypatch):
    """The register-accumulator and per-pair-contraction bodies of k_desc_radial with K1 = 13 and 17."""
    monkeypatch.setenv(switch, "1")
    model, make = MANY_SPECIES_CASES[case]
    s = make()
    check_case(oracle, emu.nep(GOLDEN / model, s["type"].shape[0]), case, s)

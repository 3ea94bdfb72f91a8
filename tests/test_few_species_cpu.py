"""One- and two-species NEP models with the features no shipped fixture carries: NEP5 per-species bias,
flexible / universal / typewise ZBL, per-species cutoffs, K1 = 13 and 17, n_max_angular = 17 (synthetic
models, tests/golden/make_synthetic_models.py).  The oracle is pinned to the reference's own codes on them
(NEP_CPU where it reads the model, else the reference gpumd), and the host build of the kernel bodies is
checked against the oracle.  tests/test_gpu_few_species.py runs the same cases through the device kernels."""
import numpy as np
import pytest

from conftest import GOLDEN, assert_close
from gpumd_b200.structures import fcc, nep_type_order


def alloy(model, cells=6, a=3.1, rattle=0.15, seed=1):
    """fcc with the species of `model` drawn i.i.d.: 864 atoms, 18.6 A box for the default 6 cells.  At
    a = 3.1 A the nearest neighbours sit at 2.19 A, inside every ZBL outer cutoff of the models, and an
    atom has ~35 angular neighbours (well above the 8 the reverse-slot search unrolls)."""
    nt = len(nep_type_order(GOLDEN / model))
    return fcc(cells, a, rattle=rattle, seed=seed, num_types=nt, symbols=("Ar",) * nt)


# name -> (model file, structure factory)
FEW_SPECIES_CASES = {
    # NEP5 (per-species bias), flexible ZBL table, K1 = 13/13, 4- and 5-body terms
    "nep5_flexzbl": ("nep_synth_2sp_nep5_flexzbl.txt", lambda: alloy("nep_synth_2sp_nep5_flexzbl.txt", seed=31)),
    # universal ZBL with the typewise outer cutoff (three distinct pair cutoffs below 2.2 A)
    "typewise_zbl": ("nep_synth_2sp_typewise_zbl.txt", lambda: alloy("nep_synth_2sp_typewise_zbl.txt", seed=32)),
    # per-species radial / angular cutoffs: three distinct pair cutoffs each
    "pertype_cut": ("nep_synth_2sp_pertype_cut.txt", lambda: alloy("nep_synth_2sp_pertype_cut.txt", seed=33)),
    # one species, universal ZBL, K1 = 17/17
    "zbl_k17": ("nep_synth_1sp_zbl_k17.txt", lambda: alloy("nep_synth_1sp_zbl_k17.txt", seed=34)),
    # one species, NEP5, K1 = 9/13, 4- and 5-body terms
    "nep5_1sp": ("nep_synth_1sp_nep5.txt", lambda: alloy("nep_synth_1sp_nep5.txt", seed=35)),
    # n_max_angular = 17, K1A = 17: 64-thread angular force blocks, > 48 KB of descriptor staging
    "namax17": ("nep_synth_2sp_namax17.txt", lambda: alloy("nep_synth_2sp_namax17.txt", seed=36)),
}

# NEP_CPU (oracle/_ref/libnep_cpu_ref.so) reads these models as they are; its results on alloy(model, seed=41)
# are stored in tests/golden/ref_nep_cpu_few_species.npz (tests/golden/make_fixtures.py)
NEP_CPU_FEW_SPECIES = {
    "nep5_flexzbl": "nep_synth_2sp_nep5_flexzbl.txt",
    "zbl_k17": "nep_synth_1sp_zbl_k17.txt",
    "nep5_1sp": "nep_synth_1sp_nep5.txt",
}

# features NEP_CPU cannot pin (typewise ZBL: it takes rc_inner = rc_outer / 2 where nep.cu takes 0; per-species
# cutoffs: it reads global cutoffs only): single points of the unmodified reference gpumd on an H100 80GB HBM3,
# scripts/run_reference_gpumd.py -> tests/golden/refgpu_<case>.npz
REFGPU_FEW_SPECIES = {
    "sp_typewise_zbl": "nep_synth_2sp_typewise_zbl.txt",
    "sp_pertype_cut": "nep_synth_2sp_pertype_cut.txt",
    "sp_nep5_flexzbl": "nep_synth_2sp_nep5_flexzbl.txt",
}


def nep_cpu_few_species_structure(model):
    return alloy(model, seed=41)


@pytest.mark.parametrize("case", list(NEP_CPU_FEW_SPECIES))
def test_oracle_matches_reference_nep_cpu_few_species(oracle, case):
    """FP64 restatement vs the reference's NEP_CPU, with the tolerances of
    test_oracle_pins.py::test_oracle_matches_reference_nep_cpu."""
    model = NEP_CPU_FEW_SPECIES[case]
    s = nep_cpu_few_species_structure(model)
    g = np.load(GOLDEN / "ref_nep_cpu_few_species.npz")
    ref = {k: g[f"{case}_{k}"] for k in ("pe", "force", "virial")}
    r = oracle.NepOracle(GOLDEN / model).compute(s["type"], s["h"], s["pbc"], s["pos"], precision=64)
    n = s["type"].shape[0]
    assert ref["pe"].shape == (n,)
    assert abs(r["pe"].sum() - ref["pe"].sum()) / n < 1e-7
    assert_close(r["force"], ref["force"], rtol=1e-6, atol=5e-7, what="force")
    assert_close(r["virial"], ref["virial"], rtol=1e-5, atol=5e-6, what="virial")


@pytest.mark.parametrize("case", list(REFGPU_FEW_SPECIES))
def test_oracle_matches_reference_gpu_few_species(oracle, case):
    """FP32 restatement vs the reference gpumd's own single point, with the tolerances of
    test_oracle_pins.py::test_oracle_matches_reference_gpu_large_box.  The force atol is scaled by the largest
    force component when that exceeds 1 eV/A, as in check_fv: the ZBL pairs of the flexible-ZBL structure
    reach 280 eV/A, and an atom's force is a sum of such terms taken in a different order by the two codes
    (the largest difference, 1.4e-4 eV/A, is 5e-7 of the largest component)."""
    d = np.load(GOLDEN / f"refgpu_{case}.npz")
    n = d["type"].shape[0]
    r = oracle.NepOracle(GOLDEN / REFGPU_FEW_SPECIES[case]).compute(
        d["type"], d["h"], d["pbc"], d["pos"], precision=32)
    assert abs(r["pe"].sum() - float(d["energy"])) / n < 2e-7
    fs = max(1.0, np.abs(d["force"]).max())
    assert_close(r["force"], d["force"], rtol=1e-5, atol=1e-5 * fs, what="force")
    v = r["virial"].sum(axis=1)
    v33 = np.array([v[0], v[3], v[4], v[6], v[1], v[5], v[7], v[8], v[2]])
    assert_close(v33, d["virial"], rtol=1e-5, atol=5e-3, what="virial")


def test_few_species_features_are_active(oracle):
    """The structures reach what the models exist for: pairs inside the ZBL outer cutoffs, and many radial
    pairs of each of the three species combinations of the per-species-cutoff model (otherwise a wrong choice
    of pair cutoff goes unnoticed)."""
    for case in ("nep5_flexzbl", "typewise_zbl", "zbl_k17"):
        model, make = FEW_SPECIES_CASES[case]
        s = make()
        pos, L = s["pos"], s["h"][0]
        d = pos[:, :, None] - pos[:, None, :]
        d -= L * np.round(d / L)
        r = np.sqrt((d * d).sum(axis=0))
        np.fill_diagonal(r, 10.0)
        assert (r < 1.9).sum() > 20, case
    model, make = FEW_SPECIES_CASES["pertype_cut"]
    s = make()
    r = oracle.NepOracle(GOLDEN / model).compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32, lists=True)
    t = s["type"]
    for t1, t2 in ((0, 0), (0, 1), (1, 1)):
        pairs = [(i, j) for i in range(len(t)) if t[i] == t1
                 for j in r["NL_radial"][i, :r["NN_radial"][i]] if t[j] == t2]
        assert len(pairs) > 100, (t1, t2)


@pytest.mark.parametrize("case", list(FEW_SPECIES_CASES))
def test_few_species_bodies_match_oracle(oracle, emu, case):
    """Host build of the kernel bodies (the generic ones: the few-species kernels are device-only)."""
    from test_kernel_bodies_cpu import check_nep
    model, make = FEW_SPECIES_CASES[case]
    s = make()
    n = s["type"].shape[0]
    check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)

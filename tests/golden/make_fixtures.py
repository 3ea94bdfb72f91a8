"""Regenerate tests/golden/ from the read-only reference tree (run in the build container).

Everything copied here is DATA the reference's own tests/examples pin this path with
(SURVEY.md 8c): potential files, input structures and the checked-in known-answer outputs.
No reference source code is copied.  /root/reference does not exist on the GPU box, so the
tests only ever read the committed copies.

    python tests/golden/make_fixtures.py [few_species | many_species]
"""
import gzip
import shutil
import sys
from pathlib import Path

import numpy as np

REF = Path("/root/reference")
OUT = Path(__file__).resolve().parent

COPIES = {
    # PbTe 250-atom known-answer single point: examples/gpumd_static (E, virial, per-atom forces)
    "examples/gpumd_static/model.xyz": "gpumd_static_model.xyz",
    "examples/gpumd_static/dump.xyz": "gpumd_static_dump.xyz",
    "examples/gpumd_static/neighbor.out": "gpumd_static_neighbor.out",
    "examples/nep_train/nep.txt": "nep_PbTe_static.txt",
    # the PbTe model BASELINE.json's metric is quoted on
    "tests/gpumd/dump_observer/PbTe_species/PbTe.txt": "nep_PbTe.txt",
    # BaZrO3 40-atom golden regression (tests_pytest/test_regression.py:35-44)
    "tests_pytest/fixtures/models/nep_BaZrO3.txt": "nep_BaZrO3.txt",
    "tests_pytest/fixtures/structures/BaZrO3-nat40-rattled.xyz": "BaZrO3-nat40-rattled.xyz",
    # the other structure / model pairs of the reference's property tests (tests_pytest/conftest.py:
    # invariances, finite-difference forces): 3-type ZBL perovskite, 1-type carbon with 17/13 basis
    # functions and a 100-neuron layer, 2-type water with the 4-body term
    "tests_pytest/fixtures/models/nep_BaTiO3.txt": "nep_BaTiO3.txt",
    "tests_pytest/fixtures/structures/BaTiO3-nat40-rattled.xyz": "BaTiO3-nat40-rattled.xyz",
    "tests_pytest/fixtures/models/nep_C.txt": "nep_C_pytest.txt",
    "tests_pytest/fixtures/structures/C-nat16-rattled.xyz": "C-nat16-rattled.xyz",
    "tests_pytest/fixtures/models/nep_water.txt": "nep_water.txt",
    "tests_pytest/fixtures/structures/water-nat63-from-md.xyz": "water-nat63-from-md.xyz",
    # carbon 64 000-atom NVE trajectory golden (tests/gpumd/carbon): thermo + neighbour maxima
    "potentials/nep/C_2022_NEP4.txt": "nep_C_2022_NEP4.txt",
    "tests/gpumd/carbon/thermo1.out": "carbon_thermo1.out",
    "tests/gpumd/carbon/neighbor1.out": "carbon_neighbor1.out",
    "tests/gpumd/carbon/run.in": "carbon_run.in",
    # LJ argon parameters (config C2)
    "potentials/lj/Ar_10A.txt": "lj_Ar_10A.txt",
    "potentials/tersoff/Si_Tersoff_1989.txt": "tersoff_Si_1989.txt",
}
# Stored gzip-compressed (files in the repository stay below 1 MB); gpumd_b200.build.unpack_fixtures(),
# run by build(), writes the plain-text file next to each one.
GZ_COPIES = {
    # UNEP-v1 16-metal alloy model (config C4): 16 types, universal ZBL, 4- and 5-body terms
    "potentials/nep/Song-2024-UNEP-v1-AgAlAuCrCuMgMoNiPbPdPtTaTiVWZr.txt": "nep_UNEP_v1.txt.gz",
    # the silicon models of potentials/nep (tests/test_reference_models_cpu.py)
    "potentials/nep/Si_2022_NEP4_3body.txt": "nep_Si_2022_NEP4_3body.txt.gz",
    "potentials/nep/Si_2022_NEP4_4body.txt": "nep_Si_2022_NEP4_4body.txt.gz",
    "potentials/nep/Si_2022_NEP4_5body.txt": "nep_Si_2022_NEP4_5body.txt.gz",
}


def main():
    for src, dst in COPIES.items():
        shutil.copyfile(REF / src, OUT / dst)
        print("copied", src, "->", dst)
    for src, dst in GZ_COPIES.items():
        with gzip.GzipFile(OUT / dst, "wb", compresslevel=9, mtime=0) as f:
            f.write((REF / src).read_bytes())
        print("compressed", src, "->", dst)
    g = np.load(REF / "tests_pytest/fixtures/golden/bulk_bazro3.npz")
    np.savez(OUT / "bulk_bazro3.npz", **{k: g[k] for k in g})
    # The carbon model.xyz is 4 MB of text; keep the positions as integers in units of 1e-11 A (the
    # precision of the file), split into 1e-4 A steps and remainders: pos = (pos_q * 1e7 + pos_r) / 1e11
    lines = (REF / "tests/gpumd/carbon/model.xyz").read_text().splitlines()
    n = int(lines[0])
    pos = np.array([[float(v) for v in ln.split()[1:4]] for ln in lines[2 : 2 + n]])
    e11 = np.rint(pos * 1e11).astype(np.int64)
    q = e11 // 10**7
    np.savez_compressed(OUT / "carbon_model.npz", header=np.array(lines[1]), pos_q=q.astype(np.int32),
                        pos_r=(e11 - q * 10**7).astype(np.int32))
    print("wrote carbon_model.npz", pos.shape)
    nep_cpu_goldens()
    nep_cpu_goldens_few_species()
    nep_cpu_goldens_many_species()


def nep_cpu_goldens():
    """Energies, forces and virials of the reference's own NEP_CPU (oracle/_ref/libnep_cpu_ref.so,
    built by `make -C oracle` where the reference tree is present) for the inputs of
    tests/test_oracle_pins.py::test_oracle_matches_reference_nep_cpu."""
    root = OUT.parents[1]
    sys.path[:0] = [str(root), str(root / "tests")]
    from oracle import oracle_py
    from test_oracle_pins import NEP_CPU_CASES, nep_cpu_structure
    assert oracle_py.ref_available(), "oracle/_ref/libnep_cpu_ref.so not built"
    out = {}
    for model, structure in NEP_CPU_CASES:
        s = nep_cpu_structure(model, structure)
        r = oracle_py.RefNepCpu(OUT / model).compute(s["type"], s["h"], s["pos"])
        for k in ("pe", "force", "virial"):
            out[f"{structure}_{k}"] = np.asarray(r[k], dtype=np.float64)
    np.savez_compressed(OUT / "ref_nep_cpu.npz", **out)
    print("wrote ref_nep_cpu.npz", sorted(out))


def nep_cpu_goldens_few_species():
    """The same for the synthetic one- and two-species models NEP_CPU reads (NEP5, flexible and universal
    ZBL): inputs of tests/test_few_species_cpu.py::test_oracle_matches_reference_nep_cpu_few_species."""
    root = OUT.parents[1]
    sys.path[:0] = [str(root), str(root / "tests")]
    from oracle import oracle_py
    from test_few_species_cpu import NEP_CPU_FEW_SPECIES, nep_cpu_few_species_structure
    assert oracle_py.ref_available(), "oracle/_ref/libnep_cpu_ref.so not built"
    out = {}
    for case, model in NEP_CPU_FEW_SPECIES.items():
        s = nep_cpu_few_species_structure(model)
        r = oracle_py.RefNepCpu(OUT / model).compute(s["type"], s["h"], s["pos"])
        for k in ("pe", "force", "virial"):
            out[f"{case}_{k}"] = np.asarray(r[k], dtype=np.float64)
    np.savez_compressed(OUT / "ref_nep_cpu_few_species.npz", **out)
    print("wrote ref_nep_cpu_few_species.npz", sorted(out))


def nep_cpu_goldens_many_species():
    """The same for the synthetic models of three to sixteen species NEP_CPU reads: inputs of
    tests/test_many_species_cpu.py::test_oracle_matches_reference_nep_cpu_many_species."""
    root = OUT.parents[1]
    sys.path[:0] = [str(root), str(root / "tests")]
    from oracle import oracle_py
    from test_many_species_cpu import MANY_SPECIES_CASES, NEP_CPU_MANY_SPECIES, nep_cpu_many_species_structure
    assert oracle_py.ref_available(), "oracle/_ref/libnep_cpu_ref.so not built"
    out = {}
    for case in NEP_CPU_MANY_SPECIES:
        s = nep_cpu_many_species_structure(case)
        r = oracle_py.RefNepCpu(OUT / MANY_SPECIES_CASES[case][0]).compute(s["type"], s["h"], s["pos"])
        for k in ("pe", "force", "virial"):
            out[f"{case}_{k}"] = np.asarray(r[k], dtype=np.float64)
    np.savez_compressed(OUT / "ref_nep_cpu_many_species.npz", **out)
    print("wrote ref_nep_cpu_many_species.npz", sorted(out))


if __name__ == "__main__":
    if sys.argv[1:] == ["few_species"]:  # only the NEP_CPU results of the synthetic few-species models
        nep_cpu_goldens_few_species()
    elif sys.argv[1:] == ["many_species"]:  # ... of the synthetic models of three or more species
        nep_cpu_goldens_many_species()
    else:
        main()

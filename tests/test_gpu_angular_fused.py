"""k_angular_fused: descriptor, hidden layer, U table and angular partial forces of a one- or two-species
model in one kernel, the default where the model fits its budget.  It calls the bodies the five-kernel
SIMT pipeline calls (B200MD_NEP_MLP=simt), so energies, forces and virials must be bit-identical to that
pipeline, and both must match the oracle.  The profiler's stage names show which path ran."""
import numpy as np
import pytest

from gpumd_b200.structures import rocksalt_pbte
from test_few_species_cpu import alloy
from test_gpu_few_species import BOXES, MODELS, _dilute_37
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)
from test_kernel_bodies_cpu import check_nep

pytestmark = pytest.mark.gpu

# the models of MODELS within the fused kernel's budget (zero-padded descriptor of 32, two blocks per SM
# of shared memory); the others exceed it: nep5_flexzbl, pertype_cut and nep5_1sp by their descriptor
# width (48), namax17 by its shared-memory rows, carbon by both
FUSED = {"PbTe", "zbl_k17", "typewise_zbl"}
FUSED_STAGES = {"k_desc_radial", "k_angular_fused", "k_force_final"}
SPLIT_STAGES = {"k_desc_radial", "k_desc_angular", "k_mlp", "k_force_angular", "k_force_final"}


def _run(oracle, eng, model, s, mlp, monkeypatch):  # noqa: F811
    """E/F/virial (checked against the oracle) and the NEP stages that ran."""
    if mlp is None:
        monkeypatch.delenv("B200MD_NEP_MLP", raising=False)
    else:
        monkeypatch.setenv("B200MD_NEP_MLP", mlp)
    n = s["type"].shape[0]
    dev = GpuNep(eng, model, n)
    dev.pot.profile(True)
    out = check_nep(oracle, dev, model, s, n)
    stages = set(dev.pot.profile_read()) - {"neighbor_update"}
    dev.pot.profile(False)
    return out, stages


def _fused_equals_simt(oracle, eng, case, s, monkeypatch):  # noqa: F811
    model = MODELS[case][0]
    a, sa = _run(oracle, eng, model, s, None, monkeypatch)
    if case not in FUSED:  # the five kernels with the tensor-core layer: checked against the oracle only
        assert sa == SPLIT_STAGES, sa
        return
    b, sb = _run(oracle, eng, model, s, "simt", monkeypatch)
    assert sa == FUSED_STAGES, sa
    assert sb == SPLIT_STAGES, sb
    for k in ("pe", "force", "virial"):
        assert np.array_equal(a[k], b[k]), (k, np.abs(a[k] - b[k]).max())


@pytest.mark.parametrize("box", list(BOXES))
@pytest.mark.parametrize("case", list(MODELS))
def test_fused_equals_simt_pipeline(oracle, eng, case, box, monkeypatch):  # noqa: F811
    """Every few-species model x box shape (ORTHO = true / false instances; open z).  The models over the
    budget take the five-kernel path by default and still match the oracle."""
    _fused_equals_simt(oracle, eng, case, BOXES[box](MODELS[case][1]()), monkeypatch)


@pytest.mark.parametrize("case", ["zbl_k17", "typewise_zbl"])
def test_fused_dilute_box(oracle, eng, case, monkeypatch):  # noqa: F811
    """37 atoms with angular lists of 0, 1 and 2 entries: the prefetch guards of both pair loops, and one
    block that is mostly beyond N."""
    s = _dilute_37()
    if case == "zbl_k17":
        s["type"][:] = 0
    _fused_equals_simt(oracle, eng, case, s, monkeypatch)


@pytest.mark.parametrize("case", ["PbTe", "typewise_zbl"])
def test_fused_partial_last_block(oracle, eng, case, monkeypatch):  # noqa: F811
    """N = 1000: a partial last 128-atom block (PbTe: the 5x5x5 rock-salt crystal; the synthetic model:
    1372 fcc sites with 372 drawn out at random)."""
    if case == "PbTe":
        s = rocksalt_pbte(5, rattle=0.05, seed=5)
    else:
        s = alloy(MODELS[case][0], cells=7, seed=51)
        keep = np.sort(np.random.default_rng(52).permutation(s["type"].shape[0])[:1000])
        s = dict(s, pos=np.ascontiguousarray(s["pos"][:, keep]), type=s["type"][keep])
    assert s["type"].shape[0] == 1000
    _fused_equals_simt(oracle, eng, case, s, monkeypatch)


@pytest.mark.parametrize("species", [0, 1])
@pytest.mark.parametrize("case", ["PbTe", "typewise_zbl"])
def test_fused_two_species_model_with_one_species_present(oracle, eng, case, species, monkeypatch):  # noqa: F811
    """A species absent from the structure: every warp holds one type's weight rows."""
    s = MODELS[case][1]()
    s["type"] = np.full_like(s["type"], species)
    _fused_equals_simt(oracle, eng, case, s, monkeypatch)


@pytest.mark.parametrize("mlp", ["simt", "tc"])
def test_explicit_hidden_layer_keeps_five_kernels(oracle, eng, mlp, monkeypatch):  # noqa: F811
    """B200MD_NEP_MLP=simt / =tc select the separate angular kernels even for a model within the budget."""
    model, make = MODELS["PbTe"]
    _, stages = _run(oracle, eng, model, make(), mlp, monkeypatch)
    assert stages == SPLIT_STAGES, stages

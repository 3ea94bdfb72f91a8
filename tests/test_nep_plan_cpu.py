"""The NEP kernel-path plan (nep_plan, b2_setup.h) for every shipped model: the choices the GPU tests observe
through b200md_nep_info, here on the host build, which runs the library's own plan function."""
import pytest

from conftest import GOLDEN
from test_many_species_cpu import MANY_SPECIES_CASES, RADREG_NT

MODELS = sorted({p.name.removesuffix(".gz") for p in GOLDEN.glob("nep*.txt*")})
# models k_angular_fused runs by default: <= 2 species, a padded descriptor of 32, within the shared-memory budget;
# value: the instance (FUSED_SHAPE_RT 1, FUSED_SHAPE_4B 2)
FUSED = {"nep_PbTe.txt": 2, "nep_water.txt": 2, "nep_synth_1sp_zbl_k17.txt": 2, "nep_synth_2sp_typewise_zbl.txt": 1}
FUSED_MAX_SMEM = 113 * 1024
# the per-pair radial contraction without a switch: the shared-memory accumulators do not fit
RAD_DIRECT = {"nep_synth_50types.txt", "nep_synth_16sp_k13.txt"}
MANY = {v[0]: k for k, v in MANY_SPECIES_CASES.items()}


def _plan(emu, model, monkeypatch, env):
    for k in ("TEAM", "REVSLOT", "RADREG", "RADDIRECT", "MLP", "CVEC", "RADIAL"):
        monkeypatch.delenv(f"B200MD_NEP_{k}", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(f"B200MD_NEP_{k}", v)
    return emu.nep(GOLDEN / model, 64).plan


@pytest.mark.parametrize("model", MODELS)
def test_nep_plan_of_shipped_models(oracle, emu, model, monkeypatch):
    nt = int((GOLDEN / model).read_text().split()[1])
    p = _plan(emu, model, monkeypatch, {})
    assert not p["team"] and not p["rev_slot"] and p["radial_v2"] == (nt <= 2)
    assert p["fused_shape"] == FUSED.get(model, 0) and p["ang_fused"] == (model in FUSED)
    if p["ang_fused"]:
        assert nt <= 2 and p["fused_smem"] <= FUSED_MAX_SMEM
    assert p["rad_direct"] == (model in RAD_DIRECT) and p["rad_nt"] == (-1 if model in RAD_DIRECT else 0)
    if p["rad_direct"]:
        assert p["rad_smem"] == 0 and p["c_r4"]
    # B200MD_NEP_MLP: the separate angular kernels
    assert not _plan(emu, model, monkeypatch, {"MLP": "simt"})["ang_fused"]
    # lane teams for one- and two-species models only, and then neither the plane-based nor the fused kernels
    p = _plan(emu, model, monkeypatch, {"TEAM": "1"})
    assert p["team"] == (nt <= 2) and not (p["team"] and (p["radial_v2"] or p["ang_fused"]))
    # reverse slots only with the neighbour split as its own kernel
    p = _plan(emu, model, monkeypatch, {"REVSLOT": "1"})
    assert p["rev_slot"] == (nt > 2 and not p["fuse_split"])
    if nt > 2:
        p = _plan(emu, model, monkeypatch, {"RADREG": "1"})
        if model in RAD_DIRECT:
            assert p["rad_nt"] == -1
        elif MANY.get(model) in RADREG_NT:
            assert p["rad_nt"] == RADREG_NT[MANY[model]]
        p = _plan(emu, model, monkeypatch, {"RADDIRECT": "1", "CVEC": "0"})
        assert p["rad_direct"] and p["rad_nt"] == -1 and p["c_r4"]

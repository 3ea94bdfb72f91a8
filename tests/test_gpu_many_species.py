"""The NEP kernels of models with three or more species (k_split, k_desc_radial<NT, K1, SPLIT>,
k_desc_angular<K1, 5>, k_mlp<DIMP, STAGE> / k_mlp_tc / k_utable<K1>, k_force_angular<K1, BLOCK>,
k_force_final<0, K1, 6, 1>) on every model feature and kernel instance they dispatch: K1 = 13 / 17, the fused
neighbour split, the per-pair radial contraction, the U-table GEMM at its 256-column limit, unstaged angular
coefficients, 64-thread angular force blocks, every SIMT hidden-layer width, orthogonal / triclinic / open
boundaries.  Each case asserts exact neighbour lists, the descriptors, E/F/virial against the FP32 and FP64
oracle (check_nep), the hidden layer against its FP64 restatement (check_mlp), and the instance it is named
for (b200md_nep_info 11-18), so that a change of a threshold cannot move a case onto another path unnoticed."""
import numpy as np
import pytest

from cases import NEP_CASES, NEP_CASES_SYNTH
from conftest import GOLDEN
from gpumd_b200.structures import fcc
from test_gpu_nep_modes import _call
from test_gpu_nep_species import MLP_MODELS, _env, check_mlp, check_tile_rule, load_ann
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)
from test_many_species_cpu import BOXES, MANY_SPECIES_CASES, check_case

pytestmark = pytest.mark.gpu

# Every test here takes the `oracle` fixture: its `make -C oracle all` also unpacks the compressed models.

# per model: the instances of the default path with the SIMT hidden layer, and whether the tensor-core layer
# fits (tc) and computes the U table as its third GEMM (tc3: nt * KP <= 256 and n_max_radial < 16).
# ang_block: k_force_angular<K1A, ang_block>; radial_nt / split: k_desc_radial<radial_nt, K1R, split>; the K1 of
# each model are listed in DESIGN.md 7.
EXPECT = {
    "3sp_nep5_flexzbl": dict(ang_block=128, radial_nt=0, split=0, cstage=1, dimp=64, tc=1, tc3=1),
    "4sp_typewise_zbl": dict(ang_block=128, radial_nt=0, split=0, cstage=1, dimp=112, tc=0, tc3=1),
    "5sp_zbl_k17_rc8": dict(ang_block=128, radial_nt=0, split=1, cstage=1, dimp=80, tc=1, tc3=1),
    "3sp_namax17": dict(ang_block=64, radial_nt=0, split=0, cstage=1, dimp=96, tc=1, tc3=1),
    "16sp_k13": dict(ang_block=128, radial_nt=-1, split=0, cstage=0, dimp=32, tc=1, tc3=1),
    "8sp_wide": dict(ang_block=64, radial_nt=0, split=1, cstage=1, dimp=128, tc=0, tc3=0),
}
# B200MD_NEP_RADREG=1: NT of the register-accumulator instance (NT * K1 <= 160 registers)
RADREG_NT = {"3sp_nep5_flexzbl": 4, "5sp_zbl_k17_rc8": 8, "3sp_namax17": 4, "8sp_wide": 8}


def expected(case, mlp, **over):
    e = EXPECT[case]
    tc = mlp == "tc" and e["tc"]
    out = dict(ang_block=e["ang_block"], radial_nt=e["radial_nt"], split=e["split"],
               utable=1 if tc and e["tc3"] else 2, cstage=e["cstage"], revslot=0,
               mlp_dimp=0 if tc else e["dimp"], mlp_stage=-1 if tc else 1)
    out.update(over)
    return out


def run_case(oracle, eng, case, s, mlp, **over):  # noqa: F811
    """check_nep and check_mlp on a fresh handle, and its instances; returns (pot, outputs)."""
    model, _ = MANY_SPECIES_CASES[case]
    dev = GpuNep(eng, model, s["type"].shape[0])
    out = check_case(oracle, dev, case, s)
    pot = dev.pot
    assert pot.instances == expected(case, mlp, **over), (case, mlp)
    assert (pot.num_tiles > 0) == (mlp == "tc" and bool(EXPECT[case]["tc"]))
    check_mlp(load_ann(GOLDEN / model), pot, s["type"], out["pe"], what=f"{case}/{mlp}")
    return pot, out


@pytest.mark.parametrize("mlp", ["tc", "simt"])
@pytest.mark.parametrize("box", list(BOXES))
@pytest.mark.parametrize("case", list(MANY_SPECIES_CASES))
def test_many_species_kernels_match_oracle(oracle, eng, case, box, mlp, monkeypatch):  # noqa: F811
    """Every model x box shape x hidden layer (k_mlp_tc, or k_mlp where the model does not fit the tensor cores:
    4sp_typewise_zbl and 8sp_wide then run k_mlp<112 | 128> with B200MD_NEP_MLP=tc too, without type tiles)."""
    _env(monkeypatch, {"B200MD_NEP_MLP": mlp})
    _, make = MANY_SPECIES_CASES[case]
    run_case(oracle, eng, case, BOXES[box](make()), mlp)


@pytest.mark.parametrize("case", list(MANY_SPECIES_CASES))
def test_many_species_simt_u_table(oracle, eng, case, monkeypatch):  # noqa: F811
    """B200MD_NEP_UTABLE=simt: the U table from k_utable<9 | 13 | 17> after the tensor-core hidden layer."""
    _env(monkeypatch, {"B200MD_NEP_UTABLE": "simt"})
    _, make = MANY_SPECIES_CASES[case]
    run_case(oracle, eng, case, make(), "tc", utable=2)


def _same(a, b, what):
    for k in ("pe", "force", "virial", "q"):
        assert np.array_equal(a[k], b[k]), (what, k, np.abs(a[k] - b[k]).max())


def _compute(eng, case, s, env, monkeypatch):  # noqa: F811
    _env(monkeypatch, env)
    model, _ = MANY_SPECIES_CASES[case]
    dev = GpuNep(eng, model, s["type"].shape[0])
    _, out = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    return dev, dict(out, q=dev.pot.export_descriptors())


@pytest.mark.parametrize("switch", ["B200MD_NEP_RADREG", "B200MD_NEP_RADDIRECT"])
@pytest.mark.parametrize("case", list(RADREG_NT))
def test_many_species_radial_opt_ins(oracle, eng, case, switch, monkeypatch):  # noqa: F811
    """k_desc_radial with its accumulators in registers (<4 | 8, 13 | 17, *>) and with the per-pair contraction
    (<-1, 13 | 17, *>): oracle parity, and agreement with the default shared-memory accumulators within FP32
    rounding: |dF| <= 1e-5 max|F| and |dW| <= 1e-5 max|W| (the sums are the same, in another association)."""
    _env(monkeypatch, {switch: "1"})
    _, make = MANY_SPECIES_CASES[case]
    s = make()
    nt = RADREG_NT[case] if switch == "B200MD_NEP_RADREG" else -1
    _, out = run_case(oracle, eng, case, s, "tc", radial_nt=nt)
    _, ref = _compute(eng, case, s, {}, monkeypatch)
    for k in ("force", "virial"):
        assert np.abs(out[k] - ref[k]).max() <= 1e-5 * np.abs(ref[k]).max(), k
    assert abs(out["pe"].sum() - ref["pe"].sum()) / s["type"].shape[0] < 1e-6


@pytest.mark.parametrize("case", [c for c in EXPECT if EXPECT[c]["cstage"]])
def test_unstaged_angular_coefficients_are_bit_identical(oracle, eng, case, monkeypatch):  # noqa: F811
    """B200MD_NEP_CSTAGE=0: k_desc_angular reads the coefficients from global memory instead of shared memory;
    the arithmetic is the same, so every output is bit-identical."""
    s = MANY_SPECIES_CASES[case][1]()
    _, ref = _compute(eng, case, s, {}, monkeypatch)
    dev, out = _compute(eng, case, s, {"B200MD_NEP_CSTAGE": "0"}, monkeypatch)
    assert dev.pot.instances["cstage"] == 0
    _same(out, ref, "CSTAGE=0")


@pytest.mark.parametrize("case", list(MANY_SPECIES_CASES))
def test_reverse_slots_are_bit_identical(oracle, eng, case, monkeypatch):  # noqa: F811
    """B200MD_NEP_REVSLOT=1: direct reverse slots instead of a search per pair in the angular pair reduction,
    bit-identical.  The models with the fused split ignore the switch: k_split, which writes those slots, does not
    run there."""
    s = MANY_SPECIES_CASES[case][1]()
    _, ref = _compute(eng, case, s, {}, monkeypatch)
    dev, out = _compute(eng, case, s, {"B200MD_NEP_REVSLOT": "1"}, monkeypatch)
    inst = dev.pot.instances
    assert inst["split"] == EXPECT[case]["split"] and inst["revslot"] == 1 - EXPECT[case]["split"], inst
    _same(out, ref, "REVSLOT=1")


@pytest.mark.parametrize("case", list(MANY_SPECIES_CASES))
def test_second_call_on_the_same_handle(oracle, eng, case, monkeypatch):  # noqa: F811
    """The same input again on one handle: no rebuild, bit-identical outputs (the outputs accumulate, so the
    second call starts from zeroed buffers of its own)."""
    s = MANY_SPECIES_CASES[case][1]()
    dev, a = _compute(eng, case, s, {}, monkeypatch)
    _, b = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert dev.rebuilds == 1
    _same(dict(b, q=dev.pot.export_descriptors()), a, "second call")


# every many-species model, old and new, with the SIMT hidden layer
WIDTH_MODELS = dict({c: v for c, v in MANY_SPECIES_CASES.items()}, BaZrO3=NEP_CASES["BaZrO3"],
                    BaTiO3=MLP_MODELS["BaTiO3"], UNEP=NEP_CASES["UNEP"], synth50=NEP_CASES_SYNTH["synth50"],
                    pertype_cutoff=NEP_CASES_SYNTH["pertype_cutoff"])


def test_simt_hidden_layer_reaches_every_width(oracle, eng, monkeypatch):  # noqa: F811
    """B200MD_NEP_MLP=simt across the many-species models runs k_mlp<DIMP, STAGE> for every DIMP from 16 to
    128 and both STAGE values (weights in shared memory; in global memory for UNEP-v1's 16 x 80 neurons),
    each checked against the FP64 hidden layer."""
    _env(monkeypatch, {"B200MD_NEP_MLP": "simt"})
    seen = set()
    for name, (model, make) in WIDTH_MODELS.items():
        s = make()
        pot = GpuNep(eng, model, s["type"].shape[0]).pot
        out = _call(eng, pot, s)
        inst = pot.instances
        assert pot.num_tiles == 0 and inst["utable"] == 2, name
        seen.add((inst["mlp_dimp"], inst["mlp_stage"]))
        check_mlp(load_ann(GOLDEN / model), pot, s["type"], out["pe"], what=name)
    assert {d for d, _ in seen} == set(range(16, 129, 16)), sorted(seen)
    assert {st for _, st in seen} == {0, 1}, sorted(seen)


def _tile_edges():
    """16-species structure on 2048 fcc sites: species 7 absent, the others with 127, 128 and 129 atoms in
    turn, except the last with 77 (N = 1868, not a multiple of 128)."""
    present = [t for t in range(16) if t != 7]
    counts = {t: 127 + k % 3 for k, t in enumerate(present)}
    counts[15] = 77
    s = fcc(8, 3.1, rattle=0.15, seed=77)
    rng = np.random.default_rng(77)
    types = np.concatenate([np.full(c, t, np.int32) for t, c in counts.items()])
    keep = np.sort(rng.permutation(s["type"].shape[0])[:types.size])
    return dict(s, pos=np.ascontiguousarray(s["pos"][:, keep]), type=rng.permutation(types), mass=s["mass"][keep])


def test_type_tiles_with_an_absent_species_and_partial_tiles(oracle, eng, monkeypatch):  # noqa: F811
    """The tensor-core layer of the 16-species model (U table as its third GEMM with 256 columns) on type tiles
    of 127, 128 and 129 atoms, a species without atoms in the middle of the type range and N % 128 != 0: every
    slot follows the tile rule, and the results match the oracle and the FP64 hidden layer."""
    _env(monkeypatch, {})
    s = _tile_edges()
    n = s["type"].shape[0]
    counts = np.bincount(s["type"], minlength=16)
    assert n % 128 and counts[7] == 0 and {127, 128, 129} <= set(counts)
    pot, _ = run_case(oracle, eng, "16sp_k13", s, "tc")
    slot, tile_type = pot.export_tiles()
    assert pot.num_tiles == tile_type.size == ((counts + 127) // 128).sum()
    check_tile_rule(slot, tile_type, s["type"], 16)

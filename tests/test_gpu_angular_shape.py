"""k_angular_fused on every angular model shape it is compiled for and on its run-time-shape instance.

The shapes of NEP4's default n_max = 4 4 with l_max = 4 2 0 (4-body block) and 4 0 0 (3-body only) run
instances in which the channel counts and invariant blocks are compile-time constants; every other shape
within the fused budget runs the instance that reads them from the model.  Whichever runs, energies,
forces, virials and the descriptor must be bit-identical to the five-kernel SIMT pipeline
(B200MD_NEP_MLP=simt), on one- and two-species models, K1 = 9, 13 and 17, orthogonal and triclinic boxes.
Models are written with random parameters for the shape under test."""
import numpy as np
import pytest

from cases import shear
from test_few_species_cpu import alloy
from test_gpu_parity import GpuNep, eng  # noqa: F401  (module fixture: the library, built)

pytestmark = pytest.mark.gpu

FUSED_STAGES = {"k_desc_radial", "k_angular_fused", "k_force_final"}

# name -> (n_max, l_max, instance): the first two are compiled-in shapes, the others take the run-time
# instance (NEP.fused_shape: 1 run-time shape, 2 / 3 n_max 4 4 with l_max 4 2 0 / 4 0 0)
SHAPES = {
    "fixed_4body": ((4, 4), (4, 2, 0), 2),   # dim 30
    "fixed_3body": ((4, 4), (4, 0, 0), 3),   # dim 25
    "rt_5body": ((3, 3), (4, 2, 1), 1),      # dim 28: 4- and 5-body blocks
    "rt_nr1": ((6, 4), (4, 2, 0), 1),        # dim 32: the 4-body layout with another radial count
    "rt_na1": ((4, 3), (4, 0, 0), 1),        # dim 21: 3-body only, four angular channels
}
SPECIES = {1: ["Si"], 2: ["Cu", "O"]}


def write_model(path, symbols, n_max, basis, l_max, nneu=30, seed=0):
    """A nep4 model file (NEP::NEP's layout) with random parameters."""
    rng = np.random.default_rng(seed)
    nt = len(symbols)
    nr1, na1 = n_max[0] + 1, n_max[1] + 1
    kr1, ka1 = basis[0] + 1, basis[1] + 1
    dim = nr1 + na1 * (l_max[0] + (1 if l_max[1] else 0) + (1 if l_max[2] else 0))
    vals = []
    for _ in range(nt):
        vals += list(rng.normal(0.0, 0.4, nneu * dim)) + list(rng.normal(0.0, 0.3, nneu))
        vals += list(rng.normal(0.0, 0.5, nneu))
    vals.append(rng.normal(0.0, 1.0))
    vals += list(rng.normal(0.0, 0.3, nt * nt * (nr1 * kr1 + na1 * ka1)))
    vals += list(rng.uniform(0.05, 0.6, dim))
    with open(path, "w") as f:
        f.write("nep4 %d %s\ncutoff 5 4 100 60\n" % (nt, " ".join(symbols)))
        f.write("n_max %d %d\nbasis_size %d %d\nl_max %d %d %d\nANN %d 0\n" % (*n_max, *basis, *l_max, nneu))
        for v in vals:
            f.write("%.7e\n" % v)
    return path


def _run(eng, model, s, mlp, monkeypatch):  # noqa: F811
    if mlp is None:
        monkeypatch.delenv("B200MD_NEP_MLP", raising=False)
    else:
        monkeypatch.setenv("B200MD_NEP_MLP", mlp)
    n = s["type"].shape[0]
    dev = GpuNep(eng, model, n)
    dev.pot.profile(True)
    _, out = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    stages = set(dev.pot.profile_read()) - {"neighbor_update"}
    out["q"] = dev.pot.export_descriptors()
    return out, stages, dev.pot.fused_shape


@pytest.mark.parametrize("box", ["ortho", "triclinic"])
@pytest.mark.parametrize("k1", [9, 13, 17])
@pytest.mark.parametrize("nt", [1, 2])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_fused_shape_equals_simt(eng, shape, nt, k1, box, tmp_path, monkeypatch):  # noqa: F811
    n_max, l_max, instance = SHAPES[shape]
    model = write_model(tmp_path / "nep.txt", SPECIES[nt], n_max, (k1 - 1, k1 - 1), l_max,
                        seed=100 * nt + k1)
    s = alloy(model, seed=7 + k1)
    if box == "triclinic":
        s = shear(s)
    a, sa, ia = _run(eng, model, s, None, monkeypatch)
    b, sb, ib = _run(eng, model, s, "simt", monkeypatch)
    assert sa == FUSED_STAGES and "k_angular_fused" not in sb
    assert (ia, ib) == (instance, 0)
    assert np.abs(a["force"]).max() > 0
    for key in ("pe", "force", "virial", "q"):
        assert np.array_equal(a[key], b[key]), key

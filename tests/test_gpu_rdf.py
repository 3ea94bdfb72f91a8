"""compute_rdf on the GPU: one sample through the C-ABI equals the brute-force oracle's integer counts
times the reference's FP64 factors bit for bit (both counting paths: block-private shared-memory tables
and, for many species, 64-bit global atomics), the 1 M-atom benchmark crystal against scipy's cKDTree,
the per-sample volume, determinism, and the driver keyword against the reference's own silicon_liquid
rdf1.out."""
import shutil
import subprocess
import types

import numpy as np
import pytest

import rdf_support as R
from conftest import GOLDEN
from gpumd_b200.structures import fcc, init_velocities, rocksalt_pbte, write_xyz

pytestmark = pytest.mark.gpu

SMEM_BUDGET = 64 * 1024  # b2_rdf.cu: tables up to this many bytes of 32-bit counters count in shared memory


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def _sample(eng, s, rc, num_bins, boxes=None):
    """samples through engine.RDF (the C-ABI); boxes: [(h, pos)] of further samples"""
    import torch
    rdf = eng.RDF(rc, num_bins, s["type"])
    atom = types.SimpleNamespace(type=torch.as_tensor(np.ascontiguousarray(s["type"], np.int32), device="cuda"))
    for h, pos in [(s["h"], s["pos"])] + list(boxes or []):
        atom.position_per_atom = torch.as_tensor(np.ascontiguousarray(pos, np.float64).reshape(-1), device="cuda")
        rdf.process(eng.Box(h, s["pbc"]), atom)
    return rdf


CASES = {k: (v[0], v[1]) for k, v in R.rdf_cases().items()}


@pytest.mark.parametrize("num_bins", [21, 500])
@pytest.mark.parametrize("case", list(CASES))
def test_one_sample_equals_oracle_counts_times_the_factors(eng, case, num_bins):
    s, rc = CASES[case]
    ti, na = R.species(s["type"])
    T = len(ti)
    shared = T * (T + 1) // 2 * num_bins * 4 <= SMEM_BUDGET
    assert shared == (case != "fifty_species")  # fifty species count with global atomics
    out = _sample(eng, s, rc, num_bins).postprocess(1)
    counts = R.oracle_counts(s, rc, num_bins)
    f = R.factors(R.volume(s["h"]), s["type"].size, rc, num_bins, na)
    assert counts[:, 0].sum() > 10000
    assert np.array_equal(out, counts * f), np.abs(out - counts * f).max()


def test_pairs_exactly_on_bin_edges(eng):
    """a simple cubic lattice of spacing 2 A with rc 8 A and 32 bins (dr = 0.25): every distance 2, 4, 6 and
    8 A (d2 = 4, 16, 36, 64) is exactly an upper bin edge ((w+1) dr)^2, so those pairs belong to bins 7, 15,
    23 and 31 by the reference's `<=`; d2 = 64 = rc^2 is kept"""
    g = np.arange(10) * 2.0
    pos = np.stack(np.meshgrid(g, g, g, indexing="ij")).reshape(3, -1)
    s = dict(h=np.diag([20.0, 20.0, 20.0]).reshape(9), pbc=np.array([1, 1, 1], np.int32),
             type=(np.arange(pos.shape[1]) % 2).astype(np.int32), pos=pos)
    rc, nb = 8.0, 32
    counts = R.oracle_counts(s, rc, nb)
    n = pos.shape[1]
    assert [counts[w, 0] for w in (7, 15, 23, 31)] == [6 * n, 6 * n, 30 * n, 6 * n]  # 30: (3,0,0), (2,2,1)
    _, na = R.species(s["type"])
    out = _sample(eng, s, rc, nb).postprocess(1)
    assert np.array_equal(out, counts * R.factors(R.volume(s["h"]), n, rc, nb, na))


def test_two_samples_at_different_volumes(eng):
    s, rc = CASES["pbte_tric"]
    nb = 100
    scale = 1.03
    s2 = dict(s, h=np.asarray(s["h"]) * scale, pos=np.asarray(s["pos"]) * scale)
    out = _sample(eng, s, rc, nb, boxes=[(s2["h"], s2["pos"])]).postprocess(2)
    _, na = R.species(s["type"])
    n = s["type"].size
    c1, c2 = R.oracle_counts(s, rc, nb), R.oracle_counts(s2, rc, nb)
    f1, f2 = R.factors(R.volume(s["h"]), n, rc, nb, na), R.factors(R.volume(s2["h"]), n, rc, nb, na)
    assert R.volume(s2["h"]) != R.volume(s["h"])
    assert np.array_equal(out, (c1 * f1 + c2 * f2) / 2)


def test_million_atom_benchmark_crystal_against_ckdtree(eng):
    """bench.py's 1 M-atom PbTe crystal at rc 6 A, 100 bins: the per-bin pair counts against cKDTree's
    pairs binned in numpy.  A difference is allowed only for pairs within a few ulps of a bin edge"""
    from scipy.spatial import cKDTree
    s = rocksalt_pbte(50, rattle=0.02, seed=1)
    n, rc, nb = s["type"].size, 6.0, 100
    out = _sample(eng, s, rc, nb).postprocess(1)
    _, na = R.species(s["type"])
    f = R.factors(R.volume(s["h"]), n, rc, nb, na)
    mine = np.rint(out[:, 0] / f[:, 0]).astype(np.int64)
    assert np.array_equal(mine * f[:, 0], out[:, 0])
    L = np.diag(np.asarray(s["h"]).reshape(3, 3)).copy()
    pos = np.asarray(s["pos"]).T.copy()
    pairs = cKDTree(pos, boxsize=L).query_pairs(rc * 1.0001, output_type="ndarray")
    d = pos[pairs[:, 1]] - pos[pairs[:, 0]]
    d -= L * np.rint(d / L)
    d2 = (d * d).sum(axis=1)
    dr = rc / nb
    edges = (np.arange(nb + 1) * dr) ** 2
    w = np.searchsorted(edges, d2, side="left") - 1  # edges[w] < d2 <= edges[w + 1]
    keep = (d2 <= rc * rc) & (w >= 0) & (w < nb)
    theirs = 2 * np.bincount(w[keep], minlength=nb)
    gap = np.abs(mine - theirs)
    k = np.clip(np.searchsorted(edges, d2), 1, nb)  # the edges on both sides of every d2
    near = np.minimum(np.abs(d2 - edges[k - 1]), np.abs(d2 - edges[k])) <= 8 * np.spacing(edges[-1])
    print(f"1 M atoms: {mine.sum() // 2} pairs, {gap.sum()} counts differ, {near.sum()} pairs near an edge")
    assert gap.sum() <= 2 * near.sum()


def _run_exe(d, run_in, timeout=900):
    from gpumd_b200 import build
    (d / "run.in").write_text(run_in)
    return subprocess.run([str(build.build_host())], cwd=d, capture_output=True, text=True, timeout=timeout)


def _pbte_model(d, reps=6, seed=21, vel=True):
    s = rocksalt_pbte(reps, rattle=0.05, seed=seed)
    write_xyz(d / "model.xyz", s, ["Te", "Pb"], init_velocities(s["mass"], 300.0, seed=seed) if vel else None)
    shutil.copyfile(GOLDEN / "nep_PbTe.txt", d / "potential.txt")
    return s


def test_driver_static_sample_prints_the_oracle_values(tmp_path):
    """time_step 0, run 1, compute_rdf ... 1: rdf.out is the oracle's counts x factors in %.5f, with the
    reference's header and radius column"""
    s = _pbte_model(tmp_path, vel=False)
    rc, nb = 6.0, 120
    r = _run_exe(tmp_path, f"potential potential.txt\nensemble nve\ntime_step 0\ncompute_rdf {rc} {nb} 1\nrun 1\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    lines = open(tmp_path / "rdf.out").read().splitlines()
    assert lines[0] == "#radius total Te-Te Te-Pb Pb-Pb" and len(lines) == nb + 1
    s = dict(s, pos=np.asarray(s["pos"]))
    _, na = R.species(s["type"])
    g = R.oracle_counts(s, rc, nb) * R.factors(R.volume(s["h"]), s["type"].size, rc, nb, na)
    dr = rc / nb
    want = ["%.5f" % (b * dr + dr / 2) + "".join(" %.5f" % v for v in g[b]) for b in range(nb)]
    assert lines[1:] == want


def test_driver_is_deterministic_and_resets_the_keyword(tmp_path):
    """NVE 200 steps sampled every 20: two runs write identical rdf.out; a repeated keyword acts as its
    last occurrence and a second run without it appends nothing"""
    outs = []
    for k in range(2):
        d = tmp_path / str(k)
        d.mkdir()
        _pbte_model(d)
        r = _run_exe(d, "potential potential.txt\nensemble nve\ntime_step 1\ncompute_rdf 5 30 1\n"
                        "compute_rdf 6 100 20\nrun 200\nrun 50\n")
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append(open(d / "rdf.out").read())
    assert outs[0] == outs[1]
    lines = outs[0].splitlines()
    assert len(lines) == 101 and lines[0].startswith("#radius") and lines[1].startswith("0.03000 ")
    g = np.array([ln.split() for ln in lines[1:]], np.float64)
    assert g[:, 1].max() > 3.0 and g[:15, 1].max() == 0.0  # the first shell of the crystal, nothing below 0.9 A


def _rdf_rows(text):
    lines = text.splitlines()
    return lines[0], np.array([ln.split() for ln in lines[1:]], np.float64)


@pytest.mark.parametrize("num_bins", R.RDF_BINS)
@pytest.mark.parametrize("case", list(CASES))
def test_driver_static_sample_matches_the_reference_binary(tmp_path, case, num_bins):
    """time_step 0, run 1, compute_rdf rc bins 1 on the inputs the unmodified reference gpumd ran
    (tests/golden/refgpu_rdf_<case>_<bins>.out, scripts/run_reference_gpumd.py): the same header, every value
    within one unit of the 5th decimal (the reference sums per-pair atomics in any order, this engine
    multiplies exact counts)"""
    s, rc, sym, pot = R.rdf_cases()[case]
    write_xyz(tmp_path / "model.xyz", s, sym)
    shutil.copyfile(pot, tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\n" + R.RDF_STATIC.format(rc=rc, nb=num_bins))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    head, g = _rdf_rows(open(tmp_path / "rdf.out").read())
    head_ref, g_ref = _rdf_rows(open(GOLDEN / f"refgpu_rdf_{case}_{num_bins}.out").read())
    assert head == head_ref and g.shape == g_ref.shape == (num_bins, 1 + R.num_rdfs(len(R.species(s["type"])[0])))
    assert np.array_equal(g[:, 0], g_ref[:, 0])
    gap = np.abs(g[:, 1:] - g_ref[:, 1:]).max()
    print(f"{case} {num_bins} bins: largest gap to the reference binary {gap:.1e}, g max {g[:, 1].max():.3f}")
    assert gap <= 1.000001e-5


# largest |g - g_ref| of the NVE run observed on an H100 80GB HBM3 (700 W): 0, every printed digit agrees.
# Three times a gap of 0 would forbid any rounding, so the bound is one unit of the 5th decimal, the bound of
# the static samples
NVE_GAP_OBSERVED = 0.0
NVE_GAP_BOUND = max(3 * NVE_GAP_OBSERVED, 1.000001e-5)


def test_driver_nve_run_matches_the_reference_binary(tmp_path):
    """200 NVE steps of PbTe sampled every 20 from the same positions and velocities as the reference run
    (tests/golden/refgpu_rdf_pbte_nve.out): FP32 forces summed in another order make the trajectories drift
    apart in principle; on an H100 the printed values agree to every digit (NVE_GAP_OBSERVED)"""
    s, vel, sym, pot = R.rdf_nve_case()
    write_xyz(tmp_path / "model.xyz", s, sym, vel)
    shutil.copyfile(pot, tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\n" + R.RDF_NVE_RUN)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    head, g = _rdf_rows(open(tmp_path / "rdf.out").read())
    head_ref, g_ref = _rdf_rows(open(GOLDEN / "refgpu_rdf_pbte_nve.out").read())
    assert head == head_ref == "#radius total Te-Te Te-Pb Pb-Pb" and g.shape == g_ref.shape == (100, 5)
    assert np.array_equal(g[:, 0], g_ref[:, 0])
    gap = np.abs(g[:, 1:] - g_ref[:, 1:]).max()
    print(f"PbTe NVE 200 steps: largest gap {gap:.2e}, g max {g_ref[:, 1:].max():.3f}")
    assert gap <= NVE_GAP_BOUND


@pytest.mark.parametrize("line,msg", [
    ("compute_rdf 5 100", "compute_rdf should have 3 parameters."),
    ("compute_rdf x 100 10", "radial cutoff should be a number."),
    ("compute_rdf 0 100 10", "radial cutoff should be positive."),
    ("compute_rdf 16 100 10", "The box has a thickness < 2.5 RDF radial cutoffs in a periodic direction."),
    ("compute_rdf 5 1.5 10", "number of bins should be an integer."),
    ("compute_rdf 5 20 10", "A larger nbins is recommended."),
    ("compute_rdf 5 501 10", "A smaller nbins is recommended."),
    ("compute_rdf 5 100 x", "interval step per sample should be an integer."),
    ("compute_rdf 5 100 -2", "interval step per sample should be positive."),
    ("compute_rdf 5 100 200\nensemble nve\nrun 100", "fewer steps than one sample interval"),
])
def test_driver_rejects_bad_rdf_input(tmp_path, line, msg):
    _pbte_model(tmp_path)  # 39.4 A: rc 16 is above the thickness / 2.5
    r = _run_exe(tmp_path, f"potential potential.txt\n{line}\n", timeout=120)
    assert r.returncode == 1 and "Input Error" in r.stderr and msg in r.stderr, r.stderr


def test_driver_silicon_liquid_rdf_matches_the_references_result(tmp_path):
    """compute_rdf 5 100 100 over the NVE half of the reference's silicon_liquid case, from its restart1.xyz,
    against its rdf1.out.  A chaotic liquid on another platform: the header and radii agree exactly, the
    values statistically"""
    shutil.copyfile(GOLDEN / "ref_silicon_liquid_restart1.xyz", tmp_path / "model.xyz")
    shutil.copyfile(GOLDEN / "nep_Si_2022_NEP4_3body.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\ntime_step 2\nensemble nve\ncompute_rdf 5 100 100\nrun 1000\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    mine, ref = open(tmp_path / "rdf.out").read().splitlines(), open(GOLDEN / "ref_silicon_liquid_rdf1.out").read().splitlines()
    assert mine[0] == ref[0] == "#radius total Si-Si" and len(mine) == len(ref) == 101
    g = np.array([ln.split() for ln in mine[1:]], np.float64)
    g_ref = np.array([ln.split() for ln in ref[1:]], np.float64)
    assert np.array_equal(g[:, 0], g_ref[:, 0])
    assert np.array_equal(g[:, 1], g[:, 2])  # one species: total = Si-Si
    gap = np.abs(g[:, 1] - g_ref[:, 1])
    peak, peak_ref = g[:, 0][np.argmax(g[:, 1])], g_ref[:, 0][np.argmax(g_ref[:, 1])]
    print(f"silicon_liquid rdf: max gap {gap.max():.4f}, mean gap {gap.mean():.4f}, "
          f"peak {peak:.3f} A (reference {peak_ref:.3f} A), peak height {g[:, 1].max():.3f} "
          f"(reference {g_ref[:, 1].max():.3f})")
    assert abs(peak - peak_ref) <= 0.1 and gap.mean() < 0.05 and gap.max() < 0.4

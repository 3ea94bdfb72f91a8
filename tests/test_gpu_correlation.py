"""compute_dos / compute_sdc / compute_msd on the device: the blocked correlation kernels against the
numpy restatement of tests/correlation_oracle.py, determinism, CUDA-graph capture (also of SHC, which
runs on the same engine), input errors, the unwrapped positions, and the `b200md` driver against the
unmodified reference gpumd and against the reference's own graphene_dos and silicon_liquid results."""
import shutil
import subprocess

import numpy as np
import pytest

import correlation_oracle as co
from conftest import GOLDEN
from gpumd_b200.structures import TIME_UNIT_CONVERSION, graphene_sheet, init_velocities, write_xyz

pytestmark = pytest.mark.gpu
DT = 1.0 / TIME_UNIT_CONVERSION


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def _close(mine, ref, tol=1e-12):
    """|mine - ref| <= tol * max |ref| (the sums are reordered; single entries can cross zero), NaN where
    the reference has NaN."""
    mine, ref = np.asarray(mine), np.asarray(ref)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(mine), nan)
    scale = np.abs(ref[~nan]).max() if (~nan).any() else 0.0
    gap = np.abs(mine[~nan] - ref[~nan]).max() if (~nan).any() else 0.0
    assert gap <= tol * scale, (gap, scale)


def _groups(n, num_groups, seed):
    """Random labels with some empty groups; the contents lists in Group::find_contents order."""
    rng = np.random.default_rng(seed)
    label = rng.integers(0, num_groups, n)
    if num_groups > 1:
        label[label % 7 == 3] = 0
    return label, [np.flatnonzero(label == g) for g in range(num_groups)]


def _run(eng, kind, n, Nc, interval, steps, groups=None, seed=0, save_at=(), num_dos_points=23):
    """Random frames through engine.DOS / SDC / MSD; returns the outputs, the frames, the masses and the
    outputs of postprocess() called after the steps in save_at."""
    torch = eng.torch
    rng = np.random.default_rng(seed)
    mass = rng.uniform(1.0, 200.0, n)
    atom = eng.Atom(np.zeros(n, np.int32), rng.uniform(0, 10, (3, n)), mass)
    frames = rng.normal(size=(steps, 3, n)) * (0.05 if kind != "msd" else 3.0)
    if kind == "dos":
        obj = eng.DOS(interval, Nc, 400.0, steps, DT, atom, groups, num_dos_points=num_dos_points)
    elif kind == "sdc":
        obj = eng.SDC(interval, Nc, steps, DT, n, groups)
    else:
        obj = eng.MSD(interval, Nc, steps, DT, n, groups)
    mid = {}
    for step in range(steps):
        x = torch.as_tensor(frames[step].reshape(-1), device="cuda")
        if kind == "msd":
            obj.process(step, x)
        else:
            atom.velocity_per_atom.copy_(x)
            obj.process(step, atom)
        if step in save_at:
            mid[step] = obj.postprocess()
    return obj.postprocess(), frames, mass, mid


def _expected(kind, frames, mass, Nc, interval, groups, n, upto=None, num_dos_points=23):
    s = co.sampled(frames if upto is None else frames[:upto + 1], interval)
    s = np.asarray(s)
    if groups is None:
        label, sizes = np.zeros(n, np.int64), [n]
    else:
        label = np.full(n, -1)
        for g, idx in enumerate(groups):
            label[idx] = g
        sizes = [len(g) for g in groups]
        keep = label >= 0
        s, mass, label = s[:, :, keep], mass[keep], label[keep]
    acc, origins = co.ring_correlate(s, Nc, kind == "msd", mass if kind == "dos" else None, label, len(sizes))
    out_a, out_b = [], []
    for g, size in enumerate(sizes):
        if kind == "dos":
            a, b = co.dos_post(acc[g], size, DT * interval, 400.0, num_dos_points)
        elif kind == "sdc":
            a, b = co.sdc_post(acc[g], size, origins, DT * interval)
        else:
            a, b = co.msd_post(acc[g], size, origins, DT * interval)
        out_a.append(a)
        out_b.append(b)
    return np.array(out_a), np.array(out_b)


# Nc = 37 is not a multiple of the block of 16 origins; 2 * (37 + 20) steps end mid-block; 999 atoms are
# not a multiple of 32
CASES = [
    ("whole", 999, 37, 2, 114, None),
    ("one_group", 999, 37, 3, 3 * 37, "one"),   # exactly one time origin
    ("nine_groups", 4000, 20, 1, 75, 9),
    ("many_groups", 6000, 10, 2, 50, 1500),
]


@pytest.mark.parametrize("kind", ["dos", "sdc", "msd"])
@pytest.mark.parametrize("name,n,Nc,interval,steps,grouping", CASES, ids=[c[0] for c in CASES])
def test_kernels_match_restatement(eng, kind, name, n, Nc, interval, steps, grouping):
    groups = None
    if grouping == "one":
        groups = [np.random.default_rng(5).permutation(n)[: n // 3]]
    elif grouping is not None:
        _, groups = _groups(n, grouping, 11)
        assert any(len(g) == 0 for g in groups)
    (a, b), frames, mass, _ = _run(eng, kind, n, Nc, interval, steps, groups, seed=len(name))
    ea, eb = _expected(kind, frames, mass, Nc, interval, groups, n)
    assert a.shape == ea.shape and b.shape == eb.shape
    if kind == "dos" and groups is not None and len(groups) > 1:
        empty = np.array([len(g) == 0 for g in groups])
        assert np.all(np.isnan(a[empty])) and np.all(np.isfinite(a[~empty]))  # 0 / 0, as the reference
    _close(a, ea)
    _close(b, eb)


def test_msd_saved_mid_block_covers_every_origin_so_far(eng):
    """postprocess() during the run (save_every): origins from sample 19 on; the saves after steps 40 and
    77 fall inside a block of 16 origins."""
    n, Nc, steps = 500, 20, 100
    _, groups = _groups(n, 4, 3)
    (a, b), frames, mass, mid = _run(eng, "msd", n, Nc, 1, steps, groups, seed=9, save_at=(40, 77))
    for step, (ma, mb) in mid.items():
        ea, eb = _expected("msd", frames, mass, Nc, 1, groups, n, upto=step)
        _close(ma, ea)
        _close(mb, eb)
    ea, eb = _expected("msd", frames, mass, Nc, 1, groups, n)
    _close(a, ea)
    _close(b, eb)


@pytest.mark.parametrize("kind", ["dos", "msd"])
def test_two_runs_are_bit_identical(eng, kind):
    _, groups = _groups(3000, 9, 4)
    r1, _, _, _ = _run(eng, kind, 3000, 30, 1, 90, groups, seed=1)
    r2, _, _, _ = _run(eng, kind, 3000, 30, 1, 90, groups, seed=1)
    assert r1[0].tobytes() == r2[0].tobytes() and r1[1].tobytes() == r2[1].tobytes()


@pytest.mark.parametrize("kind", ["sdc", "msd", "shc"])
def test_sample_call_captures_into_a_cuda_graph(eng, kind):
    """The last step completes the first block of 16 origins (step 34 at Nc = 20; step 114 at SHC's
    Nc = 100), so the captured call gathers and flushes; one replay equals the eager call: no host
    synchronisation or allocation in a sample."""
    torch = eng.torch
    n, Nc = 2000, 100 if kind == "shc" else 20
    steps = Nc + 15
    rng = np.random.default_rng(8)
    frames = [torch.as_tensor(f.reshape(-1), device="cuda") for f in rng.normal(size=(steps, 3, n))]
    atom = eng.Atom(np.zeros(n, np.int32), np.zeros((3, n)), np.ones(n))
    if kind == "shc":
        atom.virial_per_atom.copy_(torch.as_tensor(rng.normal(size=9 * n), device="cuda"))

    def make():
        if kind == "shc":
            return eng.SHC(1, Nc, 0, steps, num_atoms=n)
        return eng.SDC(1, Nc, steps, DT, n) if kind == "sdc" else eng.MSD(1, Nc, steps, DT, n)

    def call(obj, step):
        if kind == "msd":
            obj.process(step, frames[step])
        else:
            atom.velocity_per_atom.copy_(frames[step])
            obj.process(step, atom)

    eager = make()
    for step in range(steps):
        call(eager, step)
    graphed = make()
    for step in range(steps - 1):
        call(graphed, step)
    if kind != "msd":
        atom.velocity_per_atom.copy_(frames[steps - 1])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            if kind != "msd":
                graphed.process(steps - 1, atom)
            else:
                graphed.process(steps - 1, frames[steps - 1])
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    args = (DT, 10, 400.0) if kind == "shc" else ()
    a, b = eager.postprocess(*args), graphed.postprocess(*args)
    assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def test_bad_arguments_are_rejected(eng):
    L = eng._lib
    n = 100
    atom = eng.Atom(np.zeros(n, np.int32), np.zeros((3, n)), np.ones(n))
    for make, msg in [
        (lambda: eng.SDC(1, 0, 100, DT, n), "number of correlation steps should be positive"),
        (lambda: eng.MSD(0, 10, 100, DT, n), "sample interval should be positive"),
        (lambda: eng.MSD(2, 10, 19, DT, n), "MSD correlation times sampling interval"),
        (lambda: eng.SDC(2, 10, 19, DT, n), "no time origin"),
        (lambda: eng.DOS(1, 10, 400.0, 9, DT, atom), "no time origin"),
        (lambda: eng.DOS(20, 10, 400.0, 1000, DT, atom), "Nyquist"),
        (lambda: eng.DOS(1, 10, 400.0, 100, DT, atom, num_dos_points=0), "number of DOS points"),
        (lambda: eng.DOS(1, 10, -1.0, 100, DT, atom), "maximal angular frequency"),
        (lambda: eng.SDC(1, 10, 100, DT, groups=[np.array([0, 1, -3])]), "negative atom index"),
        (lambda: eng.DOS(1, 10, 400.0, 100, DT, atom, groups=[np.array([5, 100])]), ">= n"),
    ]:
        with pytest.raises(L.B200mdError, match=msg):
            make()
    sdc = eng.SDC(1, 10, 100, DT, groups=[np.array([3, 150])])
    with pytest.raises(L.B200mdError, match="n must exceed"):
        sdc.process(0, atom)
    msd = eng.MSD(1, 10, 100, DT, n)
    with pytest.raises(L.B200mdError, match="no time origin was sampled"):
        msd.postprocess()


def test_out_of_memory_ring_names_its_size(eng):
    """A ring of 1000 + 15 frames of 10^9 atoms (24 TB; 49 TB for SHC's six rows) cannot be allocated."""
    with pytest.raises(eng._lib.B200mdError, match="ring of Nc .* 1000000000 atoms"):
        eng.SDC(1, 1000, 1000, DT, 10**9)
    with pytest.raises(eng._lib.B200mdError, match="shc ring of Nc .* 1000000000 atoms, 48720"):
        eng.SHC(1, 1000, 0, 1000, num_atoms=10**9)


def test_unwrapped_positions_across_box_crossings_and_runs(eng):
    """engine.UnwrappedPosition around compute1 of NVE with a constant force, the positions wrapped into
    the box after every step (as Force::compute does), over two runs: it equals the host restatement
    u += x_new - x_old bit for bit, and differs from the wrapped positions by whole box lengths."""
    torch = eng.torch
    n, L = 300, 10.0
    rng = np.random.default_rng(6)
    atom = eng.Atom(np.zeros(n, np.int32), rng.uniform(0, L, (3, n)), np.full(n, 4.0),
                    rng.normal(size=(3, n)) * 0.3)
    atom.force_per_atom.copy_(torch.as_tensor(rng.normal(size=3 * n) * 0.01))
    box = eng.Box(np.diag([L, L, L]).reshape(9))
    unwrapped = eng.UnwrappedPosition(atom)
    host = atom.position_per_atom.cpu().numpy().copy()
    for run in range(2):
        ens = eng.Ensemble_NVE(n)
        for _ in range(60):
            x_old = atom.position_per_atom.cpu().numpy()
            unwrapped.begin(atom)
            ens.compute1(DT * 5, box, atom)
            unwrapped.end(atom)
            x_new = atom.position_per_atom.cpu().numpy()
            host += x_new - x_old
            atom.position_per_atom.copy_(torch.remainder(atom.position_per_atom, L))
    u = unwrapped.unwrapped_position.cpu().numpy()
    assert np.array_equal(u, host)
    shift = (u - atom.position_per_atom.cpu().numpy()) / L
    assert np.abs(shift).max() >= 1.0  # some atoms crossed the box
    assert np.allclose(shift, np.round(shift), atol=1e-9)


# ---- the `b200md` driver -----------------------------------------------------------------------

def _run_exe(d, run_in, timeout=900):
    from gpumd_b200 import build
    (d / "run.in").write_text(run_in)
    return subprocess.run([str(build.build_host())], cwd=d, capture_output=True, text=True, timeout=timeout)


def _rows(path):
    return np.array([ln.split() for ln in open(path) if not ln.startswith("#") and ln.strip()], dtype=np.float64)


def _graphene(d):
    s = graphene_sheet()
    write_xyz(d / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", d / "potential.txt")


def _reference_runs():
    import importlib.util
    spec = importlib.util.spec_from_file_location("run_reference_gpumd",
                                                  GOLDEN.parent.parent / "scripts" / "run_reference_gpumd.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _column_gap(mine, ref):
    """Largest |mine - ref| of each column over the largest |ref| of that column."""
    assert mine.shape == ref.shape
    return np.abs(mine - ref).max(axis=0) / np.maximum(np.abs(ref).max(axis=0), 1e-300)


GRAPHENE_FILES = {"dos": ["mvac.out", "dos.out"], "dos_groups": ["mvac.out", "dos.out"],
                  "sdc_msd": ["sdc.out", "msd.out", "msd_step500.out", "msd_step1000.out"]}


@pytest.mark.parametrize("case", list(GRAPHENE_FILES))
def test_driver_graphene_correlations_match_reference(tmp_path, case):
    """FP64 Tersoff graphene (40 400 atoms, 9 groups), 200 nvt_ber steps then 1000 nve steps with the
    correlation keywords, against the unmodified reference gpumd on the same input: every column within
    1e-5 of its largest magnitude."""
    mod = _reference_runs()
    _graphene(tmp_path)
    r = _run_exe(tmp_path, "potential potential.txt\n" + mod.CORR_GRAPHENE_PRE + mod.CORR_GRAPHENE_RUNS[case])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    for f in GRAPHENE_FILES[case]:
        ref_path = GOLDEN / f"refgpu_corr_graphene_{case}_{f}"
        mine, ref = _rows(tmp_path / f), _rows(ref_path)
        assert mine.shape == ref.shape, f
        assert np.array_equal(mine[:, 0], ref[:, 0]), f
        gap = _column_gap(mine, ref)
        print(case, f, "largest column gap", f"{gap.max():.2e}")
        assert np.all(gap <= 1e-5), (f, gap)
        heads = [ln for ln in open(tmp_path / f) if ln.startswith("#")]
        assert heads == [ln for ln in open(ref_path) if ln.startswith("#")], f


def test_driver_silicon_nep_correlations_match_reference(tmp_path):
    """NEP Si (FP32 force path), liquid from the reference's silicon_liquid/restart1.xyz, 400 nve steps
    with compute_sdc and compute_msd, against the unmodified reference gpumd."""
    mod = _reference_runs()
    shutil.copyfile(GOLDEN / "ref_silicon_liquid_restart1.xyz", tmp_path / "model.xyz")
    shutil.copyfile(GOLDEN / "nep_Si_2022_NEP4_3body.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\n" + mod.CORR_SI_RUN)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    gaps = {}
    for f in ("sdc.out", "msd.out", "msd_step300.out"):
        mine, ref = _rows(tmp_path / f), _rows(GOLDEN / f"refgpu_corr_si_sdc_msd_{f}")
        assert mine.shape == ref.shape and np.array_equal(mine[:, 0], ref[:, 0]), f
        gaps[f] = _column_gap(mine, ref).max()
    print("NEP Si largest column gaps:", {k: f"{v:.2e}" for k, v in gaps.items()})
    # observed 6.6e-4 of a column's largest value (sdc.out) on an H100: the FP32 forces of a liquid
    # drift apart over 400 steps; three times that
    assert max(gaps.values()) < 2e-3


def test_driver_silicon_liquid_statistics_match_the_references_results(tmp_path):
    """The NVE half of the reference's silicon_liquid case from its restart1.xyz.  Its sdc1.out /
    msd1.out come from a chaotic liquid and another platform: only the first rows and the final SDC are
    compared."""
    shutil.copyfile(GOLDEN / "ref_silicon_liquid_restart1.xyz", tmp_path / "model.xyz")
    shutil.copyfile(GOLDEN / "nep_Si_2022_NEP4_3body.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\ntime_step 2\nensemble nve\ncompute_sdc 2 100\n"
                           "compute_msd 2 100\nrun 1000\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    sdc, ref_sdc = _rows(tmp_path / "sdc.out"), _rows(GOLDEN / "ref_silicon_liquid_sdc1.out")
    msd, ref_msd = _rows(tmp_path / "msd.out"), _rows(GOLDEN / "ref_silicon_liquid_msd1.out")
    assert sdc.shape == ref_sdc.shape == (100, 7) and msd.shape == ref_msd.shape == (100, 7)
    vac0 = np.abs(sdc[0, 1:4] / ref_sdc[0, 1:4] - 1).max()
    msd1 = np.abs(msd[1, 1:4] / ref_msd[1, 1:4] - 1).max()
    d_end = np.abs(sdc[-1, 4:7].mean() / ref_sdc[-1, 4:7].mean() - 1)
    print(f"silicon_liquid: VAC(0) {vac0:.2e}, MSD(dt) {msd1:.2e}, final SDC {d_end:.2e} (relative)")
    # observed on an H100: 4.9e-3, 4.9e-3 and 2.8e-3
    assert vac0 < 0.02 and msd1 < 0.02 and d_end < 0.05


def test_driver_graphene_dos_run_in_matches_the_references_results(tmp_path):
    """The reference's graphene_dos run.in unchanged (npt_ber 10 000 steps, then nve with
    compute_dos 5 200 400.0 for 10 000 steps) on its model.xyz: the DOS sum rule within 1 %, the main peak
    of each direction within two bins of its dos1.out, and mvac at short lags close to its mvac1.out."""
    shutil.copyfile(GOLDEN / "ref_graphene_dos_model.xyz", tmp_path / "model.xyz")
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\nvelocity 300\n\n"
                           "ensemble npt_ber 300 300 100 0 0 0 53.4059 53.4059 53.4059 2000\ntime_step 1\n"
                           "dump_thermo 100\nrun 10000\n\nensemble nve\ncompute_dos 5 200 400.0\nrun 10000\n",
                 timeout=1500)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    dos, ref = _rows(tmp_path / "dos.out"), _rows(GOLDEN / "ref_graphene_dos_dos1.out")
    assert dos.shape == ref.shape == (200, 4)
    n = 8640
    total = dos[:, 1:].sum(axis=0) * 2.0 / (2 * np.pi)
    print("sum rule per direction:", total, "reference:", ref[:, 1:].sum(axis=0) * 2.0 / (2 * np.pi))
    assert np.all(np.abs(total / n - 1) < 0.01)
    peaks, ref_peaks = np.argmax(dos[:, 1:], axis=0), np.argmax(ref[:, 1:], axis=0)
    print("main peaks (bin):", peaks, "reference:", ref_peaks)
    assert np.all(np.abs(peaks - ref_peaks) <= 2)
    mvac, ref_mvac = _rows(tmp_path / "mvac.out"), _rows(GOLDEN / "ref_graphene_dos_mvac1.out")
    assert mvac.shape == ref_mvac.shape == (200, 4)
    gap = np.abs(mvac[:5, 1:] - ref_mvac[:5, 1:]).max()
    print(f"mvac gap over the first 5 lags: {gap:.3e}")
    assert gap < 0.05  # observed 0.015 on an H100


@pytest.mark.parametrize("line,msg", [
    ("compute_dos 5 100", "compute_dos should have at least 3 parameters."),
    ("compute_dos 0 100 400", "sample interval should be positive."),
    ("compute_dos 5 100 -4", "maximal angular frequency should be positive."),
    ("compute_dos 5 100 400 num_dos_points 0", "number of DOS points must be > 0."),
    ("compute_dos 5 100 400 group 0 9", "Group ID should < number of groups."),
    ("compute_dos 50 100 400\nensemble nve\nrun 5000", "Nyquist"),
    ("compute_dos 5 100 400\nensemble nve\nrun 100", "no time origin"),
    ("compute_sdc 2 x", "number of correlation steps should be an integer."),
    ("compute_sdc 2 10 group 0 -1", "group ID should >= 0."),
    ("compute_sdc 2 10 foo", "Unrecognized argument in compute_sdc."),
    ("compute_msd 2 10 all_groups 1", "Grouping method should < number of grouping methods."),
    ("compute_msd 2 10 group 0 1 all_groups 0", "Cannot compute MSD over a single group and all groups"),
    ("compute_msd 2 100\nensemble nve\nrun 100", "MSD correlation times sampling interval"),
])
def test_driver_rejects_bad_correlation_input(tmp_path, line, msg):
    s = graphene_sheet(10, 91)
    write_xyz(tmp_path / "model.xyz", s, ["C"])
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, f"potential potential.txt\n{line}\n", timeout=120)
    assert r.returncode == 1 and "Input Error" in r.stderr and msg in r.stderr, r.stderr


def test_driver_resets_the_keywords_and_keeps_unwrapping(tmp_path):
    """A second run without the keywords writes nothing more; a third with compute_msd continues from
    the unwrapped positions the first one started."""
    s = graphene_sheet(10, 91)
    write_xyz(tmp_path / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=1))
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", tmp_path / "potential.txt")
    r = _run_exe(tmp_path, "potential potential.txt\nensemble nve\ntime_step 1\ncompute_dos 2 20 400\n"
                           "compute_sdc 2 20\ncompute_msd 2 20\nrun 100\nrun 50\ncompute_msd 2 20\nrun 60\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert _rows(tmp_path / "mvac.out").shape == (20, 4) and _rows(tmp_path / "dos.out").shape == (20, 4)
    assert _rows(tmp_path / "sdc.out").shape == (20, 7)
    assert _rows(tmp_path / "msd.out").shape == (40, 7)
    assert open(tmp_path / "msd.out").read().count("# compute_msd 2 20") == 2

"""The measurement and dump keywords of the `b200md` driver (gpumd_b200/host/measure.cpp): a keyword given
twice before one `run` acts as its last occurrence alone, and every keyword holds for one run only."""
import shutil
import subprocess

import pytest

from conftest import GOLDEN
from gpumd_b200.structures import graphene_sheet, init_velocities, write_xyz

pytestmark = pytest.mark.gpu

# keyword: (first occurrence, the occurrence that replaces it); both fit one 120-step run of the sheet
REPEATS = {
    "dump_thermo": ("dump_thermo 5", "dump_thermo 7"),
    "dump_xyz": ("dump_xyz 5 first.xyz", "dump_xyz 40 dump.xyz precision double velocity force"),
    "dump_restart": ("dump_restart 50", "dump_restart 70"),
    "compute_hac": ("compute_hac 2 20 1", "compute_hac 3 10 2"),
    "compute": ("compute 0 5 2 temperature", "compute 0 10 3 potential jp momentum"),
    "compute_shc": ("compute_shc 1 100 1 10 400.0", "compute_shc 1 110 0 20 200.0 group 0 1"),
    "compute_dos": ("compute_dos 2 20 400", "compute_dos 3 15 300 num_dos_points 30"),
    "compute_sdc": ("compute_sdc 2 20", "compute_sdc 3 15 group 0 1"),
    "compute_msd": ("compute_msd 2 20", "compute_msd 3 15 save_every 60"),
}
REPEATS["all"] = tuple("\n".join(v[k] for v in REPEATS.values()) for k in (0, 1))

PRE = "potential potential.txt\nensemble nvt_ber 300 300 100\ntime_step 1\n"


def _run(d, run_in, timeout=600):
    from gpumd_b200 import build
    exe = build.build_host()
    s = graphene_sheet(10, 11)  # 440 atoms, grouping method 0 with two groups
    write_xyz(d / "model.xyz", s, ["C"], init_velocities(s["mass"], 300.0, seed=42))
    shutil.copyfile(GOLDEN / "Graphene_Lindsay_2010_modified.txt", d / "potential.txt")
    (d / "run.in").write_text(run_in)
    return subprocess.run([str(exe)], cwd=d, capture_output=True, text=True, timeout=timeout)


def _outputs(d):
    return {p.name: p.read_bytes() for p in d.iterdir() if p.name not in ("model.xyz", "potential.txt", "run.in")}


@pytest.mark.parametrize("keyword", list(REPEATS))
def test_repeated_keyword_acts_as_its_last_occurrence_for_one_run(tmp_path, keyword):
    """The keyword twice, then a second run without it, writes exactly the files of a single run with only
    the second occurrence: no earlier occurrence samples or writes, and the second run adds nothing."""
    first, second = REPEATS[keyword]
    both, last = tmp_path / "both", tmp_path / "last"
    both.mkdir()
    last.mkdir()
    r = _run(both, PRE + f"{first}\n{second}\nrun 120\nrun 20\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    r = _run(last, PRE + f"{second}\nrun 120\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    mine, ref = _outputs(both), _outputs(last)
    assert ref and sorted(mine) == sorted(ref)
    for name in ref:
        assert mine[name] == ref[name], name


def test_repeated_compute_hnemd_is_an_input_error_within_a_run_only(tmp_path):
    r = _run(tmp_path, PRE + "compute_hnemd 10 0 1e-5 0\ncompute_hnemd 20 0 1e-5 0\nrun 20\n")
    assert r.returncode == 1 and "Cannot have more than one HNEMD method within one run." in r.stderr, r.stderr
    r = _run(tmp_path, PRE + "compute_hnemd 10 0 1e-5 0\nrun 20\ncompute_hnemd 5 0 1e-5 0\nrun 20\nrun 20\n")
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert len((tmp_path / "kappa.out").read_text().splitlines()) == 2 + 4

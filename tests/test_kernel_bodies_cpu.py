"""The kernel BODIES of libb200md (gpumd_b200/csrc/*.cuh), compiled for the host by tests/emu and
checked against the oracle.  This is the GPU-less proxy for tests/test_gpu_parity.py: same inputs,
same assertions, but the device scheduling (blocks, shared memory, atomics, scans) is emulated by
serial loops.  Neighbour sets must be bit-exact; E/F/virial within the reference suite's own
tolerances."""
import numpy as np
import pytest

from cases import NEP_CASES, NEP_CASES_SYNTH
from conftest import GOLDEN, TOL, assert_close
from gpumd_b200.structures import fcc, rocksalt_pbte


def check_fv(out, ref, noise=1.0, gap_f=0.0, gap_v=0.0):
    """force: rtol 1e-4 + atol 1e-5 eV/A, virial: rtol 1e-4 + atol 2e-5 eV (SURVEY.md 8d), with the
    atol scaled by the largest component when that exceeds 1 -- FP32 accumulation noise is
    relative to the magnitude of the terms being summed, not to the (possibly cancelling) result.
    `noise` widens the atol for potentials whose per-pair terms cancel heavily (stated at the call).
    gap_f / gap_v: the FP32 restatement's own distance from the FP64 truth on this input (max over
    components); a second FP32 evaluation with a different summation order cannot be expected to
    sit closer to either of them than they sit to each other, so it is added to the atol."""
    fs = noise * max(1.0, np.abs(ref["force"]).max())
    vs = noise * max(1.0, np.abs(ref["virial"]).max())
    assert_close(out["force"], ref["force"], rtol=TOL["force"]["rtol"],
                 atol=TOL["force"]["atol"] * fs + gap_f, what="force")
    assert_close(out["virial"], ref["virial"], rtol=TOL["virial"]["rtol"],
                 atol=TOL["virial"]["atol"] * vs + gap_v, what="virial")


def check_nep(oracle, dev, model, s, n, energy_tol=None, q_gap=False):
    """energy_tol: eV/atom bound against the FP32 restatement (default 1e-6, SURVEY 8d).  Callers with
    deep-well models (|E|/N of several eV) pass 1e-6 * |E|/N: FP32 rounding is relative.
    q_gap: for models with ~300 radial neighbours (rc = 8 A), whose FP32 radial sums cancel to 1e-5 of their
    terms: each descriptor component's atol gets twice the FP32 restatement's own largest distance from the
    FP64 descriptors (another FP32 summation order may sit on the other side of the FP64 value), and the
    descriptors are also checked against FP64."""
    energy_tol = TOL["energy_per_atom"] if energy_tol is None else energy_tol
    orc = oracle.NepOracle(GOLDEN / model)
    r32 = orc.compute(s["type"], s["h"], s["pbc"], s["pos"], precision=32, lists=True, descriptors=True)
    r64 = orc.compute(s["type"], s["h"], s["pbc"], s["pos"], precision=64, descriptors=q_gap)
    rc, out = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    NNr, NLr, NNa, NLa = dev.neighbors(r32["NL_radial"].shape[1], r32["NL_angular"].shape[1])
    assert np.array_equal(NNr, r32["NN_radial"]) and np.array_equal(NLr, r32["NL_radial"])
    assert np.array_equal(NNa, r32["NN_angular"]) and np.array_equal(NLa, r32["NL_angular"])
    q = dev.descriptors(orc.info["dim"])
    if q_gap:
        q_atol = 2e-6 + 2 * np.abs(r32["q"] - r64["q"]).max(axis=1, keepdims=True)
        assert_close(q, r64["q"], rtol=2e-5, atol=q_atol, what="descriptor vs FP64")
    else:
        q_atol = 2e-6
    assert_close(q, r32["q"], rtol=2e-5, atol=q_atol, what="descriptor")
    # |dE|/N <= 1e-6 eV against the FP32 restatement (the reference GPU's arithmetic); against the
    # FP64 truth allow the FP32 pair-math noise itself (the restatement's own f32-f64 gap) on top
    gap = abs(r32["pe"].sum() - r64["pe"].sum()) / n
    assert abs(out["pe"].sum() - r32["pe"].sum()) / n < energy_tol
    assert abs(out["pe"].sum() - r64["pe"].sum()) / n < energy_tol + 2 * gap
    # the reference suite's total-energy tolerance (rtol 1e-5, tests_pytest/conftest.py:51-62) applied to
    # the magnitude that is being summed: site energies of opposite sign can cancel in the total (the
    # water fixture: sum |E_i| = 289 eV, E = -1.0 eV), and FP32 noise does not cancel with them
    e_scale = np.abs(r64["pe"]).sum()
    assert abs(out["pe"].sum() - r32["pe"].sum()) <= TOL["energy"]["atol"] + TOL["energy"]["rtol"] * e_scale
    gap_f = np.abs(r32["force"] - r64["force"]).max()
    gap_v = np.abs(r32["virial"] - r64["virial"]).max()
    check_fv(out, r32, gap_f=gap_f, gap_v=gap_v)
    check_fv(out, r64, gap_f=gap_f, gap_v=gap_v)
    return out


@pytest.mark.parametrize("team", ["0", "1"])
@pytest.mark.parametrize("case", list(NEP_CASES))
def test_nep_bodies_match_oracle(oracle, emu, case, team, monkeypatch):
    """team: thread-per-atom radial passes (default) or the lane-team bodies (<= 2 types; the host
    build runs them with a team of one lane)."""
    monkeypatch.setenv("B200MD_NEP_TEAM", team)
    model, make = NEP_CASES[case]
    s = make()
    n = s["type"].shape[0]
    dev = emu.nep(GOLDEN / model, n)
    check_nep(oracle, dev, model, s, n)


@pytest.mark.parametrize("case", list(NEP_CASES_SYNTH))
def test_synthetic_models_match_oracle(oracle, emu, case):
    """50 species (radial descriptor by per-pair contraction, the path a model like NEP89 takes) and the
    per-type `cutoff` form."""
    model, make = NEP_CASES_SYNTH[case]
    s = make()
    n = s["type"].shape[0]
    check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)


@pytest.mark.parametrize("case", ["UNEP", "BaZrO3"])
def test_per_pair_radial_contraction_matches_oracle(oracle, emu, case, monkeypatch):
    """B200MD_NEP_RADDIRECT=1 forces k_desc_radial<-1,...>'s body on the shipped many-type models."""
    monkeypatch.setenv("B200MD_NEP_RADDIRECT", "1")
    model, make = NEP_CASES[case]
    s = make()
    n = s["type"].shape[0]
    check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)


@pytest.mark.parametrize("switch", ["B200MD_NEP_REVSLOT", "B200MD_NEP_RADREG"])
@pytest.mark.parametrize("case", ["UNEP", "BaZrO3"])
def test_many_type_opt_ins_match_oracle(oracle, emu, case, switch, monkeypatch):
    """The many-type opt-in paths (direct reverse slots in the angular pair reduction; radial accumulators
    in registers) produce the same results as the defaults (measured slower, kept as A/B switches)."""
    monkeypatch.setenv(switch, "1")
    model, make = NEP_CASES[case]
    s = make()
    n = s["type"].shape[0]
    out = check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)
    monkeypatch.delenv(switch)
    ref = emu.nep(GOLDEN / model, n).compute(s["type"], s["h"], s["pbc"], s["pos"])[1]
    assert np.array_equal(out["force"], ref["force"]) and np.array_equal(out["virial"], ref["virial"])


def test_nep_accumulates_into_outputs(oracle, emu):
    """Potential::compute contract: outputs are += (nep.cu:653,755-770)."""
    s = rocksalt_pbte(4, rattle=0.05, seed=1)
    n = s["type"].shape[0]
    dev = emu.nep(GOLDEN / "nep_PbTe.txt", n)
    _, a = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    # second call on the same handle: no rebuild, same answer
    _, b = dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert dev.rebuilds == 1
    assert np.array_equal(a["force"], b["force"]) and np.array_equal(a["pe"], b["pe"])


def _store_mode_cases():
    from cases import NEP_SMALL_CASES
    from test_few_species_cpu import FEW_SPECIES_CASES
    return {"PbTe": NEP_CASES["PbTe"], "zbl_k17": FEW_SPECIES_CASES["zbl_k17"], "BaZrO3": NEP_CASES["BaZrO3"],
            "PbTe_C1": NEP_SMALL_CASES["PbTe_C1"]}


@pytest.mark.parametrize("team", ["0", "1"])
@pytest.mark.parametrize("case", ["PbTe", "zbl_k17", "BaZrO3", "PbTe_C1"])
def test_final_bodies_store_mode_and_owned_range(emu, case, team, monkeypatch):
    """b200md_nep_set_accumulate(p, 0) on the final bodies (thread per atom with one, two and many types; the
    lane-team bodies for one and two types; the supercell fold of a small box): outputs prefilled with NaN
    must come out equal to accumulate mode on zeros.  With set_owned(m) only atoms below m are written, in
    both modes; accumulate mode adds to the prefill."""
    monkeypatch.setenv("B200MD_NEP_TEAM", team)
    model, make = _store_mode_cases()[case]
    s = make()
    n = s["type"].shape[0]
    args = (s["type"], s["h"], s["pbc"], s["pos"])
    dev = emu.nep(GOLDEN / model, n)
    _, ref = dev.compute(*args)
    assert all(np.isfinite(ref[k]).all() for k in ref)
    dev.set_mode(accumulate=False)
    for _ in range(2):  # a second store on the same handle
        _, out = dev.compute(*args, prefill=(np.nan,) * 3)
        for k in ("pe", "force", "virial"):
            assert np.array_equal(out[k], ref[k]), k
    m = 129 if n > 129 else n - 1
    for accumulate, fill in ((False, (7.0, 7.0, 7.0)), (True, (1.0, 2.0, 3.0))):
        dev.set_mode(accumulate=accumulate, n_owned=m)
        _, out = dev.compute(*args, prefill=fill)
        for k, f in zip(("pe", "force", "virial"), fill):
            want = ref[k][..., :m] + f if accumulate else ref[k][..., :m]
            assert np.array_equal(out[k][..., :m], want), (k, accumulate)
            assert np.all(out[k][..., m:] == f), (k, accumulate)
    dev.set_mode(accumulate=False, n_owned=0)
    _, out = dev.compute(*args, prefill=(np.nan,) * 3)
    for k in ("pe", "force", "virial"):
        assert np.array_equal(out[k], ref[k]), k


def test_skin_list_reuse_and_rebuild(oracle, emu):
    """Move atoms by less than skin/2: no rebuild, sets still exact.  Move one atom further:
    the predicated rebuild fires and the sets are exact again."""
    s = rocksalt_pbte(4, rattle=0.05, seed=1)
    n = s["type"].shape[0]
    dev = emu.nep(GOLDEN / "nep_PbTe.txt", n)
    orc = oracle.NepOracle(GOLDEN / "nep_PbTe.txt")
    rng = np.random.default_rng(3)
    pos = s["pos"].copy()
    dev.compute(s["type"], s["h"], s["pbc"], pos)
    for step, amp, expect in ((1, 0.12, 1), (2, 0.12, 1), (3, 0.0, 2)):
        disp = rng.uniform(-1, 1, pos.shape) * amp / np.sqrt(3)
        if step == 3:
            disp[:, 17] = [0.6, 0.0, 0.0]  # > skin/2 from the snapshot for sure
        pos = np.mod(pos + disp, s["h"][0])
        r = orc.compute(s["type"], s["h"], s["pbc"], pos, precision=32, lists=True)
        rc, out = dev.compute(s["type"], s["h"], s["pbc"], pos)
        assert rc == 0 and dev.rebuilds == expect, (step, dev.rebuilds)
        NNr, NLr, NNa, NLa = dev.neighbors(r["NL_radial"].shape[1], r["NL_angular"].shape[1])
        assert np.array_equal(NLr, r["NL_radial"]) and np.array_equal(NLa, r["NL_angular"])
        assert_close(out["force"], r["force"], **TOL["force"], what="force")


def test_changed_types_rebuild(oracle, emu):
    """Same positions, 5 % of the unlike pairs swapped: exactly one rebuild (a changed type triggers it like a
    displacement), none when the same types come again; the result equals a fresh handle's bit for bit and
    the oracle's."""
    s = rocksalt_pbte(4, rattle=0.05, seed=1)
    n = s["type"].shape[0]
    t2 = s["type"].copy()
    rng = np.random.default_rng(5)
    pb, te = rng.permutation(np.nonzero(t2 == 0)[0])[:13], rng.permutation(np.nonzero(t2 == 1)[0])[:13]
    t2[pb], t2[te] = 1, 0
    dev = emu.nep(GOLDEN / "nep_PbTe.txt", n)
    dev.compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert dev.rebuilds == 1
    rc, out = dev.compute(t2, s["h"], s["pbc"], s["pos"])
    assert rc == 0 and dev.rebuilds == 2
    _, fresh = emu.nep(GOLDEN / "nep_PbTe.txt", n).compute(t2, s["h"], s["pbc"], s["pos"])
    for k in ("pe", "force", "virial"):
        assert np.array_equal(out[k], fresh[k]), k
    dev.compute(t2, s["h"], s["pbc"], s["pos"])
    assert dev.rebuilds == 2
    r = oracle.NepOracle(GOLDEN / "nep_PbTe.txt").compute(t2, s["h"], s["pbc"], s["pos"], precision=32)
    assert_close(out["force"], r["force"], **TOL["force"], what="force")
    assert abs(out["pe"].sum() - r["pe"].sum()) / n < TOL["energy_per_atom"]


def test_cutoff_boundary_membership(oracle, emu):
    """Pairs placed within a few ulps of the radial and angular cutoffs: membership is decided by
    the reference's FP32 expression, so the CUDA-side test and the oracle must agree exactly."""
    base = rocksalt_pbte(4, a=7.4, rattle=0.0, seed=1)  # dilute lattice: 3.7 A nearest neighbours
    pos = base["pos"].copy()
    n = pos.shape[1]
    rng = np.random.default_rng(5)
    # move the odd atom of 120 pairs so that |r| straddles rc_radial (8) or rc_angular (4)
    for k in range(120):
        i, j = 2 * k, 2 * k + 1
        rc = 8.0 if k % 2 == 0 else 4.0
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        eps = (rng.integers(-6, 7)) * 4.8e-7 * (rc / 8.0)
        pos[:, j] = pos[:, i] + u * (rc + eps)
    pos = np.mod(pos, base["h"][0])
    orc = oracle.NepOracle(GOLDEN / "nep_PbTe.txt")
    r = orc.compute(base["type"], base["h"], base["pbc"], pos, precision=32, lists=True)
    dev = emu.nep(GOLDEN / "nep_PbTe.txt", n)
    rc, _ = dev.compute(base["type"], base["h"], base["pbc"], pos)
    assert rc == 0
    NNr, NLr, NNa, NLa = dev.neighbors(r["NL_radial"].shape[1], r["NL_angular"].shape[1])
    assert np.array_equal(NLr, r["NL_radial"]) and np.array_equal(NLa, r["NL_angular"])
    # the construction really produced boundary cases: some of the engineered pairs are in, some out
    eng = [(2 * k + 1) in NLr[2 * k, :NNr[2 * k]] for k in range(0, 120, 2)]
    assert 5 < sum(eng) < 55


@pytest.mark.parametrize("case", ["PbTe_C1", "PbTe_static_golden", "BaZrO3_40", "PbTe_thin"])
def test_small_box_through_supercell(oracle, emu, case):
    """Boxes thinner than 2.5*(rc+skin) (the reference's nep_small_box.cuh path): the library
    evaluates the smallest admissible supercell and keeps the first replica.  Same assertions as the
    large-box cases; lists then hold one entry per periodic image, like the reference's."""
    from cases import NEP_SMALL_CASES
    model, make = NEP_SMALL_CASES[case]
    s = make()
    n = s["type"].shape[0]
    check_nep(oracle, emu.nep(GOLDEN / model, n), model, s, n)


def test_reference_goldens_directly(emu):
    """The reference's checked-in known answers (small boxes), no oracle in between."""
    from cases import check_reference_goldens
    check_reference_goldens(lambda model, n: emu.nep(GOLDEN / model, n), assert_close, TOL)


def write_potential(path, head, rows):
    """A potential file: the first line, then one line per row of numbers (repr: the values round-trip)."""
    path.write_text("\n".join([head] + [" ".join(repr(float(x)) for x in r) for r in rows]) + "\n")
    return path


def write_lj(path, para, symbols):
    """An `lj` file of the table para[a][b] = (epsilon, sigma, cutoff)."""
    nt = para.shape[0]
    return write_potential(path, f"lj {nt} {' '.join(symbols)}", para.reshape(nt * nt, 3))


def test_lj_bodies_match_oracle(oracle, emu, tmp_path):
    s = fcc(6, 5.30, rattle=0.1, seed=2)  # 31.8 A box > 2.5*(10+1)
    n = s["type"].shape[0]
    para = np.array([[[1.032e-2, 3.405, 10.0]]])
    r = oracle.lj_compute(para, s["type"], s["h"], s["pbc"], s["pos"])
    rc, out = emu.lj(write_lj(tmp_path / "lj.txt", para, ["Ar"]), n).compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    assert_close(out["pe"], r["pe"], rtol=1e-5, atol=1e-7, what="pe")
    assert_close(out["force"], r["force"], **TOL["force"], what="force")
    assert_close(out["virial"], r["virial"], **TOL["virial"], what="virial")


def test_lj_two_types(oracle, emu, tmp_path):
    s = fcc(6, 5.30, rattle=0.1, seed=9, num_types=2, symbols=("Ar", "Ar"))
    n = s["type"].shape[0]
    para = np.array([[[1.0e-2, 3.4, 10.0], [0.8e-2, 3.2, 9.0]], [[0.8e-2, 3.2, 9.0], [1.2e-2, 3.0, 8.0]]])
    r = oracle.lj_compute(para, s["type"], s["h"], s["pbc"], s["pos"])
    path = write_lj(tmp_path / "lj.txt", para, ["Ar", "Ar"])
    rc, out = emu.lj(path, n).compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    assert_close(out["force"], r["force"], **TOL["force"], what="force")
    assert_close(out["pe"], r["pe"], rtol=1e-5, atol=1e-7, what="pe")


def test_integrate_bodies(oracle, emu):
    rng = np.random.default_rng(1)
    n = 200
    mass = rng.uniform(1, 200, n)
    pos, vel, f = rng.normal(size=(3, n)) * 5 + 10, rng.normal(size=(3, n)), rng.normal(size=(3, n))
    for step1 in (True, False):
        a = oracle.velocity_verlet(step1, 0.098, mass, pos, vel, f)
        b = emu.velocity_verlet(step1, 0.098, mass, pos, vel, f)
        # FP64, same operations; the host build may or may not contract a*b+c, so allow 1 ulp here
        # (the GPU test compares bit for bit against the FMA form nvcc emits)
        assert np.allclose(a[0], b[0], rtol=4e-16, atol=0) and np.allclose(a[1], b[1], rtol=4e-16, atol=1e-18)
    # `fix` / `move` groups (ensemble.cu:111-174): group 1 frozen, group 2 dragged at a constant velocity
    label = rng.integers(0, 4, n).astype(np.int32)
    mv = np.array([0.3, -0.2, 0.1])
    for step1 in (True, False):
        a = oracle.velocity_verlet_groups(step1, 0.098, mass, pos, vel, f, label, 1, 2, mv)
        b = emu.velocity_verlet_groups(step1, 0.098, mass, pos, vel, f, label, 1, 2, mv)
        assert np.allclose(a[0], b[0], rtol=4e-16, atol=0) and np.allclose(a[1], b[1], rtol=4e-16, atol=1e-18)
        assert np.all(a[1][:, (label == 1) | (label == 2)] == 0.0)
        assert np.array_equal(a[0][:, label == 1], pos[:, label == 1])
        if step1:
            assert np.allclose(a[0][:, label == 2], pos[:, label == 2] + mv[:, None] * 0.098, rtol=1e-15)
    pe, vir = rng.normal(size=n), rng.normal(size=(9, n))
    assert np.allclose(oracle.find_thermo(n, 123.0, mass, pe, vel, vir),
                       emu.find_thermo(n, 123.0, mass, pe, vel, vir), rtol=1e-13)
    h = np.array([20.0, 2.0, 0.0, 0.0, 21.0, 1.0, 0.0, 0.0, 22.0])
    p = rng.uniform(-5, 27, (3, n))
    assert np.allclose(oracle.apply_pbc(h, [1, 0, 1], p), emu.apply_pbc(h, [1, 0, 1], p), rtol=0, atol=1e-13)


@pytest.mark.parametrize("case", ["Si", "SiC_like"])
def test_tersoff_bodies_match_oracle(oracle, emu, case, tmp_path):
    """Tersoff-1989 is FP64 end to end in the reference; our fused kernel only re-orders the
    arithmetic (radial functions evaluated once per neighbour), so agreement is at 1e-10."""
    from gpumd_b200.structures import diamond
    path = GOLDEN / "tersoff_Si_1989.txt"
    if case == "Si":
        nt, para = oracle.tersoff_parameters(path)
        s = diamond(4, a=5.431, rattle=0.08, seed=12)  # 512 atoms, 21.7 A box
        types = s["type"]
    else:  # two types: Si parameters twice with perturbed second set and chi != 1 (mixing rules)
        _, p0 = oracle.tersoff_parameters(path)
        p1 = p0 * np.array([1.05, 0.97, 1.02, 0.98, 1.0, 1.0, 1.0, 1.0, 1.0, 0.98, 0.99])
        nt, para = 2, np.concatenate([p0, p1, [0.9776]])
        path = write_potential(tmp_path / "tersoff.txt", "tersoff_1989 2 Si C", [p0, p1, [0.9776]])
        s = diamond(4, a=5.431, rattle=0.08, seed=13)
        types = (np.arange(s["type"].shape[0]) % 2).astype(np.int32)
    n = types.shape[0]
    r = oracle.tersoff_compute(nt, para, types, s["h"], s["pbc"], s["pos"])
    rc, out = emu.tersoff(path, n).compute(types, s["h"], s["pbc"], s["pos"])
    assert rc == 0
    assert_close(out["pe"], r["pe"], rtol=1e-10, atol=1e-11, what="pe")
    assert_close(out["force"], r["force"], rtol=1e-9, atol=1e-10, what="force")
    assert_close(out["virial"], r["virial"], rtol=1e-9, atol=1e-10, what="virial")
    assert np.abs(out["force"].sum(axis=1)).max() < 1e-9  # Newton's third law
    # heat current from the per-atom virial
    vel = np.random.default_rng(2).normal(size=(3, n))
    assert np.allclose(emu.compute_heat(out["virial"], vel), oracle.compute_heat(out["virial"], vel),
                       rtol=1e-14, atol=0)


def test_tersoff_energy_is_physical(oracle):
    """Sanity pin of the restatement: cohesive energy of perfect diamond Si with Tersoff-1989 (T3)
    is -4.6297 eV/atom (Tersoff, PRB 39, 5566) and forces vanish by symmetry."""
    from gpumd_b200.structures import diamond
    nt, para = oracle.tersoff_parameters(GOLDEN / "tersoff_Si_1989.txt")
    s = diamond(3, a=5.432, rattle=0.0)
    r = oracle.tersoff_compute(nt, para, s["type"], s["h"], s["pbc"], s["pos"])
    assert abs(r["pe"].mean() + 4.6297) < 2e-3
    assert np.abs(r["force"]).max() < 1e-9


@pytest.mark.parametrize("potfile,ntypes", [("eam_Cu_Zhou_2004.txt", 1), ("eam_zhou_2004_CuFeNi.txt", 3),
                                            ("eam_Cu_Dai_2006.txt", 1)])
def test_eam_bodies_match_oracle(oracle, emu, potfile, ntypes):
    model, nt, para = oracle.eam_parameters(GOLDEN / potfile)
    assert nt == ntypes
    s = fcc(6, 3.615, rattle=0.08, seed=31, num_types=nt, symbols=["Cu", "Fe", "Ni"][:nt])
    n = s["type"].shape[0]  # 864 atoms, 21.7 A box (rc 6.5 / 4.3 A)
    r = oracle.eam_compute(model, nt, para, s["type"], s["h"], s["pbc"], s["pos"])
    rc, out = emu.eam(GOLDEN / potfile, n).compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    assert_close(out["pe"], r["pe"], rtol=2e-6, atol=1e-6, what="pe")
    check_fv(out, r)
    assert np.abs(out["force"].sum(axis=1)).max() < 1e-3


def test_eam_cohesive_energy_is_physical(oracle):
    """Pin of the restatement: Zhou-2004 Cu gives Ec = -3.54 eV/atom at a0 = 3.615 A (the value the
    parametrisation was fitted to)."""
    model, nt, para = oracle.eam_parameters(GOLDEN / "eam_Cu_Zhou_2004.txt")
    s = fcc(6, 3.615, rattle=0.0)
    r = oracle.eam_compute(model, nt, para, s["type"], s["h"], s["pbc"], s["pos"])
    assert abs(r["pe"].mean() + 3.54) < 0.01
    assert np.abs(r["force"]).max() < 1e-5


def test_bdp_body_matches_oracle(oracle, emu):
    """b2_bdp.cuh (host build): same uniform stream as the oracle bit for bit, and the same velocity
    scale factors along a sequence of steps (libm exp/log/sqrt on both sides here: exact)."""
    E = emu.E
    st = E.emu_bdp_create(12345678)
    o = oracle.BdpOracle(12345678)
    assert [E.emu_bdp_rand01(st) for _ in range(500)] == [o.rand01() for _ in range(500)]
    E.emu_bdp_destroy(st)
    st = E.emu_bdp_create(12345678)
    o = oracle.BdpOracle(12345678)
    rng = np.random.default_rng(0)
    for n_atoms, tc in [(64000, 100.0), (250, 10.0), (3, 100.0), (1, 0.05)]:
        for _ in range(20):
            t = float(rng.uniform(200, 400))
            a = E.emu_bdp_factor(st, t, 3 * n_atoms, 300.0, tc)
            b = o.factor(t, n_atoms, 300.0, tc)
            assert a == pytest.approx(b, rel=1e-15), (n_atoms, tc)
    E.emu_bdp_destroy(st)

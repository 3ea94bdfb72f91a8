"""LJ, Tersoff-1989 and EAM without a GPU: the plain FP64 references of tests/cases_classical.py checked
against their own derivatives, the FP32 oracle against them, the host build of the kernel bodies against
the oracle, known-answer clusters, and the oracle pinned to the unmodified reference gpumd's output
(tests/golden/refgpu_sp_*.npz, written on an H100 by scripts/run_reference_gpumd.py)."""
import numpy as np
import pytest

import cases_classical as cc
from conftest import GOLDEN, TOL, assert_close
from test_kernel_bodies_cpu import check_fv

DAI_NOISE = 4.0  # Dai-2006's pair polynomial cancels to ~1e-2 of its terms (test_gpu_parity.test_eam_matches_oracle)


def _energy(kind, path, s):
    return cc.reference64(kind, path, s)["pe"].sum()


# ---------------------------------------------------------------- FP64 references are self-consistent

SELF_CHECK = ["lj_3sp-tric", "lj_3sp-slab", "sic-tric", "si_expanded-slab", "eam_cufeni_compressed-tric",
              "eam_cu_zhou_expanded-slab", "eam_cu_zhou_a0-tric", "eam_cu_dai_a0-slab"]


@pytest.mark.parametrize("case", SELF_CHECK)
def test_fp64_reference_forces_are_energy_gradients(oracle, case):
    """Central differences of the total energy (h = 1e-6 A) against the reference's forces.  The steps are
    small because LJ and EAM are truncated without a shift: a pair crossing its cutoff inside the
    difference stencil would add U(rc) / 2h."""
    kind, path, s = cc.make(case)
    r = cc.reference64(kind, path, s)
    h = 1e-6
    for i in (3, 101):
        for d in range(3):
            sp, sm = dict(s), dict(s)
            sp["pos"], sm["pos"] = s["pos"].copy(), s["pos"].copy()
            sp["pos"][d, i] += h
            sm["pos"][d, i] -= h
            fd = -(_energy(kind, path, sp) - _energy(kind, path, sm)) / (2 * h)
            assert abs(fd - r["force"][d, i]) < 1e-6 + 1e-6 * abs(r["force"][d, i]), (i, d, fd, r["force"][d, i])


@pytest.mark.parametrize("case", SELF_CHECK)
def test_fp64_reference_virial_is_strain_derivative(oracle, case):
    """-dE/de_ab (box and positions strained together by (1 + e), e = 1e-8) against the summed virial,
    all nine components.  With e = 1e-6, some pair of the 864-atom LJ slab crosses its cutoff inside
    the stencil (see above)."""
    kind, path, s = cc.make(case)
    r = cc.reference64(kind, path, s)
    W = cc.v33(r["virial"]).reshape(3, 3)
    H = s["h"].reshape(3, 3)
    e = 1e-8
    wmax = max(1.0, np.abs(W).max())
    for a in range(3):
        for b in range(3):
            eps = np.zeros((3, 3))
            eps[a, b] = e
            es = []
            for sign in (1, -1):
                M = np.eye(3) + sign * eps
                t = dict(s, h=(M @ H).reshape(9), pos=M @ s["pos"])
                es.append(_energy(kind, path, t))
            fd = -(es[0] - es[1]) / (2 * e)
            assert abs(fd - W[a, b]) < 2e-5 * wmax, (a, b, fd, W[a, b])


def test_inputs_reach_the_branches_they_are_for(oracle):
    """Zhou-2004 Cu at a = 3.3 / 3.615 / 4.0 A sits in the power/log, middle and low-density embedding
    branches; stretched Si puts most bonds into Tersoff's 2.7-3.0 A switching region; SiC bonds are all
    Si-C (the mixed parameter set)."""
    path = GOLDEN / cc.EAM_FILES["cu_zhou"]
    for tag, branch in (("compressed", 2), ("a0", 1), ("expanded", 0)):
        _, _, s = cc.make(f"eam_cu_zhou_{tag}-ortho")
        rho = cc.eam64(path, s, return_rho=True)["rho"]
        assert np.all(cc.zhou_branch(path, rho) == branch), tag
    _, _, s = cc.make("si_expanded-tric")
    d = [r for _, _, _, r in cc._pairs(s, 3.0)]
    assert sum(((x > 2.7) & (x < 3.0)).sum() for x in d) > 500
    _, _, s = cc.make("sic-ortho")
    for i, j, _, r in cc._pairs(s, 2.51):
        assert np.all(s["type"][j] != s["type"][i])


def test_lj_table_is_symmetric_with_a_large_truncation_jump():
    t = cc.lj_table(cc.LJ3)
    assert t.shape == (3, 3, 3) and np.array_equal(t, t.transpose(1, 0, 2))
    assert len({tuple(t[a, b]) for a in range(3) for b in range(a, 3)}) == 6
    eps, sig, rc = t[1, 1]
    sr6 = (sig / rc) ** 6
    assert abs(4 * eps * (sr6 * sr6 - sr6)) > 1.5e-3 and abs(rc - 2.5 * sig) < 1e-12


# ---------------------------------------------------------------- FP32 oracle vs FP64

def check_vs_fp64(out, r64, n, kind, path, gap=(0.0, 0.0, 0.0), energy_tol=2e-6):
    """LJ / EAM: |dE|/N, per-atom energy and check_fv against the FP64 reference, widened by `gap`
    (another FP32 evaluation's own distance from FP64).  Tersoff is FP64 throughout: 1e-10 / 1e-9."""
    if kind == "tersoff":
        assert_close(out["pe"], r64["pe"], rtol=1e-10, atol=1e-11, what="pe")
        assert_close(out["force"], r64["force"], rtol=1e-9, atol=1e-10, what="force")
        assert_close(out["virial"], r64["virial"], rtol=1e-9, atol=1e-10, what="virial")
        return
    noise = DAI_NOISE if "Dai" in str(path) else 1.0
    assert abs(out["pe"].sum() - r64["pe"].sum()) / n < energy_tol + 2 * gap[2]
    assert_close(out["pe"], r64["pe"], rtol=1e-5, atol=1e-5 * noise + gap[2], what="pe")
    check_fv(out, r64, noise=noise, gap_f=gap[0], gap_v=gap[1])


@pytest.mark.parametrize("case", cc.CASES)
def test_oracle_matches_fp64_reference(oracle, case):
    """The FP32 restatement against the FP64 references (EAM with the file's parameters rounded to float,
    as both FP32 codes hold them: the tolerances then measure arithmetic only)."""
    kind, path, s = cc.make(case)
    n = s["type"].shape[0]
    r32 = cc.oracle32(kind, path, s)
    r64 = cc.reference64(kind, path, s, f32_params=True)
    check_vs_fp64(r32, r64, n, kind, path)


# ---------------------------------------------------------------- host build of the kernel bodies

def emu_handle(emu, kind, path, n):
    from oracle import oracle_py
    if kind == "lj":
        return emu.lj(cc.lj_table(path), n)
    if kind == "tersoff":
        nt, p = oracle_py.tersoff_parameters(path)
        return emu.tersoff(nt, p, n)
    model, nt, p = oracle_py.eam_parameters(path)
    return emu.eam(model, nt, p, n)


def check_vs_oracle(out, r, n, kind, path):
    """The existing tolerances of test_{lj,tersoff,eam}_bodies_match_oracle, force / virial atol scaled by
    the largest component (check_fv)."""
    if kind == "tersoff":
        assert_close(out["pe"], r["pe"], rtol=1e-10, atol=1e-11, what="pe")
        assert_close(out["force"], r["force"], rtol=1e-9, atol=1e-10, what="force")
        assert_close(out["virial"], r["virial"], rtol=1e-9, atol=1e-10, what="virial")
        assert np.abs(out["force"].sum(axis=1)).max() < 1e-9
        return
    if kind == "lj":
        assert_close(out["pe"], r["pe"], rtol=1e-5, atol=1e-7, what="pe")
        check_fv(out, r)
    else:
        noise = DAI_NOISE if "Dai" in str(path) else 1.0
        assert_close(out["pe"], r["pe"], rtol=1e-5, atol=1e-5, what="pe")
        assert abs(out["pe"].sum() - r["pe"].sum()) / n < 2e-6
        check_fv(out, r, noise=noise)
    assert np.abs(out["force"].sum(axis=1)).max() < 1e-3


@pytest.mark.parametrize("case", cc.CASES)
def test_kernel_bodies_match_oracle(oracle, emu, case):
    kind, path, s = cc.make(case)
    n = s["type"].shape[0]
    r = cc.oracle32(kind, path, s)
    rc, out = emu_handle(emu, kind, path, n).compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    check_vs_oracle(out, r, n, kind, path)


# ---------------------------------------------------------------- known answers: isolated clusters

def _tersoff_pair(p, r):
    """Tersoff-1989 dimer (zeta = 0, b = 1): f_c (f_R - f_A); p = A B lambda mu ... R S."""
    A, B, lam, mu, R, S = p[0], p[1], p[2], p[3], p[9], p[10]
    fc = 1.0 if r < R else (0.0 if r > S else 0.5 + 0.5 * np.cos(np.pi * (r - R) / (S - R)))
    return fc * (A * np.exp(-lam * r) - B * np.exp(-mu * r))


def _mixed(p0, p1, chi):
    """Tersoff's mixing rules (PRB 39, 5566): geometric A, B (times chi), R, S; arithmetic lambda, mu."""
    g = lambda k: np.sqrt(p0[k] * p1[k])
    m = np.array(p0, dtype=np.float64)
    m[0], m[1], m[2], m[3], m[9], m[10] = g(0), chi * g(1), 0.5 * (p0[2] + p1[2]), 0.5 * (p0[3] + p1[3]), g(9), g(10)
    return m


def _eam_F(model, P, t, rho):
    if model == "dai":
        return -P[0] * np.sqrt(rho)
    return cc._zhou_embed(P[t], rho)[0]


# (potential kind, file, cluster, bond length, types) -> closed-form total energy or None (symmetry only)
CLUSTERS = {
    "lj_atom": ("lj", cc.LJ3, "atom", 3.0, [1]),
    "lj_dimer_11": ("lj", cc.LJ3, "dimer", 3.7, [1, 1]),
    "lj_dimer_02": ("lj", cc.LJ3, "dimer", 3.4, [0, 2]),
    "lj_trimer": ("lj", cc.LJ3, "trimer", 3.9, [2, 2, 2]),
    "tersoff_atom": ("tersoff", cc.SIC, "atom", 2.0, [0]),
    "tersoff_si2_switching": ("tersoff", cc.SI, "dimer", 2.85, [0, 0]),
    "tersoff_si2": ("tersoff", cc.SI, "dimer", 2.35, [0, 0]),
    "tersoff_sic": ("tersoff", cc.SIC, "dimer", 1.9, [0, 1]),
    "tersoff_trimer": ("tersoff", cc.SI, "trimer", 2.4, [0, 0, 0]),
    "eam_zhou_atom": ("eam", GOLDEN / cc.EAM_FILES["cu_zhou"], "atom", 2.5, [0]),
    "eam_zhou_dimer": ("eam", GOLDEN / cc.EAM_FILES["cu_zhou"], "dimer", 2.3, [0, 0]),
    "eam_alloy_dimer": ("eam", GOLDEN / cc.EAM_FILES["cufeni"], "dimer", 2.5, [0, 2]),
    "eam_zhou_trimer": ("eam", GOLDEN / cc.EAM_FILES["cu_zhou"], "trimer", 2.5, [0, 0, 0]),
    "eam_dai_dimer": ("eam", GOLDEN / cc.EAM_FILES["cu_dai"], "dimer", 2.6, [0, 0]),
    "eam_dai_trimer": ("eam", GOLDEN / cc.EAM_FILES["cu_dai"], "trimer", 2.6, [0, 0, 0]),
}


def cluster_energy(kind, path, which, r, types, f32_params=False):
    """Closed forms (from the published functional forms, not from any code) of the total energy.
    f32_params: EAM parameters rounded to float, as the FP32 codes hold them (see cc.eam64)."""
    model, _, P = cc.eam_read(path) if kind == "eam" else (None, None, None)
    if f32_params and kind == "eam":
        P = P.astype(np.float32).astype(np.float64)
    if which == "atom":
        return _eam_F(model, P, types[0], 0.0) if kind == "eam" else 0.0
    if kind == "lj":
        eps, sig, _ = cc.lj_table(path)[types[0], types[1]]
        u = 4 * eps * ((sig / r) ** 12 - (sig / r) ** 6)
        return u if which == "dimer" else 3 * u
    if kind == "tersoff":
        if which != "dimer":
            return None
        from oracle import oracle_py
        nt, p = oracle_py.tersoff_parameters(path)
        if types[0] == types[1]:
            return _tersoff_pair(p[11 * types[0]:11 * types[0] + 11], r)
        return _tersoff_pair(_mixed(p[:11], p[11:22], p[22]), r)
    ta, tb = types[0], types[1]
    phi, _, fb, _, _ = cc._eam_pair_terms(model, P, ta, np.array([tb]), np.array([r]))
    fa = cc._eam_pair_terms(model, P, tb, np.array([ta]), np.array([r]))[2]
    if which == "dimer":
        return _eam_F(model, P, ta, fb[0]) + _eam_F(model, P, tb, fa[0]) + phi[0]
    return 3 * _eam_F(model, P, ta, 2 * fb[0]) + 3 * phi[0]


def check_cluster(out, name, n, fp32=True):
    """Known answer (closed form or symmetry) for one cluster; shared with the device test."""
    kind, path, which, r, types = CLUSTERS[name]
    e = cluster_energy(kind, path, which, r, types, f32_params=fp32)
    tol = 1e-12 if kind == "tersoff" else 3e-6  # FP64 / FP32 pair math
    if e is not None:
        assert abs(out["pe"].sum() - e) <= tol * max(1.0, abs(e)), (out["pe"].sum(), e)
    assert np.abs(out["force"].sum(axis=1)).max() <= tol * max(1.0, np.abs(out["force"]).max())
    if which == "atom":
        assert np.all(out["force"] == 0) and np.all(out["virial"] == 0)
    if which == "trimer":  # equilateral, one species: equal energies, equal force magnitudes
        assert np.ptp(out["pe"]) <= tol * max(1.0, np.abs(out["pe"]).max())
        fm = np.linalg.norm(out["force"], axis=0)
        assert np.ptp(fm) <= 10 * tol * max(1.0, fm.max())
    if which == "dimer":  # the force lies along the bond
        assert np.abs(out["force"][1:]).max() <= tol * max(1.0, np.abs(out["force"]).max())


def make_cluster(name):
    kind, path, which, r, types = CLUSTERS[name]
    return kind, path, cc.cluster(kind, which, r, types)


@pytest.mark.parametrize("name", list(CLUSTERS))
def test_clusters_known_answers(oracle, emu, name):
    """Open box (pbc 0 0 0): the oracle and the host kernel bodies against the closed forms; the Si dimer
    goes through b = 1 (zeta < 1e-16) and, at 2.85 A, the cosine switching function."""
    kind, path, s = make_cluster(name)
    n = s["type"].shape[0]
    r = cc.oracle32(kind, path, s)
    check_cluster(r, name, n)
    check_cluster(cc.reference64(kind, path, s), name, n, fp32=False)
    rc, out = emu_handle(emu, kind, path, n).compute(s["type"], s["h"], s["pbc"], s["pos"])
    assert rc == 0
    check_cluster(out, name, n)


def test_eam_dimer_closed_form_is_the_papers(oracle):
    """The Zhou dimer closed form written out directly: E = 2 F(f(r)) + phi(r) at r = 2.3 A (low-density
    embedding branch)."""
    _, _, P = cc.eam_read(GOLDEN / cc.EAM_FILES["cu_zhou"])
    re, fe, rho_e, rho_s, al, be, A, B, ka, la = P[0][:10]
    r = 2.3
    phi = A * np.exp(-al * (r / re - 1)) / (1 + (r / re - ka) ** 20) - B * np.exp(-be * (r / re - 1)) / (1 + (r / re - la) ** 20)
    f = fe * np.exp(-be * (r / re - 1)) / (1 + (r / re - la) ** 20)
    assert f < 0.85 * rho_e
    x = f / (0.85 * rho_e) - 1
    F = sum(P[0][10 + k] * x ** k for k in range(4))
    assert abs(cluster_energy("eam", GOLDEN / cc.EAM_FILES["cu_zhou"], "dimer", r, [0, 0]) - (2 * F + phi)) < 1e-12


# ---------------------------------------------------------------- oracle pinned to the reference GPU code

REFGPU = {  # fixture -> (kind, potential file)
    "sp_lj3_tric": ("lj", cc.LJ3),
    "sp_sic": ("tersoff", cc.SIC),
    "sp_sic_slab": ("tersoff", cc.SIC),
    "sp_eam_dai": ("eam", GOLDEN / cc.EAM_FILES["cu_dai"]),
    "sp_eam_cu_compressed": ("eam", GOLDEN / cc.EAM_FILES["cu_zhou"]),
    "sp_eam_alloy_tric": ("eam", GOLDEN / cc.EAM_FILES["cufeni"]),
}


@pytest.mark.parametrize("case", list(REFGPU))
def test_oracle_matches_reference_gpu(oracle, case):
    """tests/golden/refgpu_<case>.npz: energy, per-atom forces and the summed virial written by the
    unmodified reference gpumd on an H100 from our inputs.  Tolerances of test_{lj,tersoff,eam}_oracle_
    matches_reference_gpu (test_oracle_pins.py); the force atol is scaled by the largest component."""
    kind, path = REFGPU[case]
    d = np.load(GOLDEN / f"refgpu_{case}.npz")
    n = d["type"].shape[0]
    s = dict(type=d["type"], h=d["h"], pbc=d["pbc"], pos=d["pos"])
    r = cc.oracle32(kind, path, s)
    fs = max(1.0, np.abs(d["force"]).max())
    E = float(d["energy"])
    if kind == "lj":
        assert abs(r["pe"].sum() - E) / n < 1e-9
        assert_close(r["force"], d["force"], rtol=1e-6, atol=5e-7 * fs, what="force")
        assert_close(cc.v33(r["virial"]), d["virial"], rtol=1e-6, atol=1e-4, what="virial")
    elif kind == "tersoff":
        assert abs(r["pe"].sum() - E) < 1e-9 * abs(E)
        assert_close(r["force"], d["force"], rtol=1e-10, atol=1e-10 * fs, what="force")
        assert_close(cc.v33(r["virial"]), d["virial"], rtol=1e-10, atol=1e-8, what="virial")
    else:  # Dai-2006: the summation-order noise factor of test_gpu_parity.test_eam_matches_oracle
        noise = DAI_NOISE if "Dai" in str(path) else 1.0
        assert abs(r["pe"].sum() - E) / n < 1e-6
        assert_close(r["force"], d["force"], rtol=1e-5, atol=1e-5 * noise * fs, what="force")
    assert (s["pbc"] == 0).any() == case.endswith("slab")

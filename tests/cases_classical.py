"""Inputs and plain FP64 references for the LJ, Tersoff-1989 and EAM kernels.

Structures: each potential on its crystals in three box forms (orthogonal, `shear()`, `slab()`), every
periodic thickness > 2.5 (rc + 1) after shearing.  References: brute-force pair sums in float64 with the
fractional-coordinate minimum image (triclinic boxes and open directions alike), written from the
published functional forms -- not from the oracle's FP32 arithmetic -- so that a misreading shared by
the oracle and the kernels shows up against them.  Per-atom energy, force [3, N] and 9-component virial
[9, N] in GPUMD's order (xx yy zz xy xz yz yx zx zy) and GPUMD's per-atom partition."""
import numpy as np

from cases import shear, slab
from conftest import GOLDEN
from gpumd_b200.structures import diamond, fcc

LJ3 = GOLDEN / "lj_synth_3types.txt"
LJ1 = GOLDEN / "lj_Ar_10A.txt"
SI = GOLDEN / "tersoff_Si_1989.txt"
SIC = GOLDEN / "tersoff_SiC_1989.txt"
EAM_FILES = {"cu_zhou": "eam_Cu_Zhou_2004.txt", "cufeni": "eam_zhou_2004_CuFeNi.txt", "cu_dai": "eam_Cu_Dai_2006.txt"}

BOXES = {"ortho": lambda s: s, "tric": shear, "slab": slab}


def lj_table(path):
    """(nt, nt, 3) epsilon, sigma, cutoff from an `lj` potential file."""
    toks = open(path).read().split()
    nt = int(toks[1])
    return np.array([float(v) for v in toks[2 + nt:2 + nt + 9 * nt * nt]]).reshape(nt, nt, 3)


def thickness(h):
    """Distance between opposite faces of the cell (h: lattice vectors as columns)."""
    H = np.asarray(h, dtype=np.float64).reshape(3, 3)
    a, b, c = H[:, 0], H[:, 1], H[:, 2]
    vol = abs(np.linalg.det(H))
    return np.array([vol / np.linalg.norm(np.cross(b, c)), vol / np.linalg.norm(np.cross(c, a)),
                     vol / np.linalg.norm(np.cross(a, b))])


def _lj3_alloy(seed):
    s = fcc(6, 5.30, rattle=0.1, seed=seed, num_types=3, symbols=("Ar", "Ar", "Ar"))
    s["symbols"] = ["Ar", "Ne", "Kr"]
    return s


def _sic(reps, seed, rattle=0.08):
    """Zincblende SiC: the diamond lattice with the first fcc sub-lattice Si, the second C."""
    s = diamond(reps, a=4.36, rattle=rattle, seed=seed)
    s["type"] = np.tile(np.array([0, 0, 0, 0, 1, 1, 1, 1], np.int32), reps ** 3)
    s["mass"] = np.where(s["type"] == 0, 28.085, 12.011)
    s["symbols"] = ["Si", "C"]
    return s


def _eam(key, a, seed):
    nt = 3 if key == "cufeni" else 1
    cells = 7 if a < 3.5 else 6
    return fcc(cells, a, rattle=0.08, seed=seed, num_types=nt, symbols=["Cu", "Fe", "Ni"][:nt])


# name -> (kind, potential file, structure factory without the box form)
STRUCTURES = {
    "lj_ar": ("lj", LJ1, lambda: fcc(6, 5.30, rattle=0.1, seed=41)),  # 864 atoms, 31.8 A
    "lj_3sp": ("lj", LJ3, lambda: _lj3_alloy(42)),
    # Si at a0; Si stretched so that most bonds sit in the 2.7-3.0 A switching region; SiC (mixed set only)
    "si": ("tersoff", SI, lambda: diamond(4, a=5.431, rattle=0.08, seed=43)),  # 512 atoms, 21.7 A
    "si_expanded": ("tersoff", SI, lambda: diamond(4, a=6.5, rattle=0.25, seed=44)),
    "sic": ("tersoff", SIC, lambda: _sic(5, 45)),  # 1000 atoms, 21.8 A
}
for _k in EAM_FILES:
    for _a, _tag in ((3.615, "a0"), (3.3, "compressed"), (4.0, "expanded")):
        STRUCTURES[f"eam_{_k}_{_tag}"] = ("eam", GOLDEN / EAM_FILES[_k],
                                          (lambda k=_k, a=_a: _eam(k, a, 46)))

CASES = [f"{name}-{box}" for name in STRUCTURES for box in BOXES]


def make(case):
    """case 'name-box' -> (kind, potential file, structure)."""
    name, box = case.rsplit("-", 1)
    kind, path, factory = STRUCTURES[name]
    return kind, path, BOXES[box](factory())


def cutoff(kind, path):
    if kind == "lj":
        return lj_table(path)[..., 2].max()
    if kind == "tersoff":
        from oracle import oracle_py
        nt, p = oracle_py.tersoff_parameters(path)
        return max(p[10], p[21]) if nt == 2 else p[10]
    from oracle import oracle_py
    model, nt, p = oracle_py.eam_parameters(path)
    return max(p[20::21]) if model == 0 else max(p[1], p[2])


# ---------------------------------------------------------------- known-answer clusters (open box)

def cluster(kind, which, r, types=None):
    """`atom`, `dimer` (bond length r) or equilateral `trimer` (side r) in a 40 A box, pbc 0 0 0."""
    pos = {"atom": [[0, 0, 0]], "dimer": [[0, 0, 0], [r, 0, 0]],
           "trimer": [[0, 0, 0], [r, 0, 0], [0.5 * r, 0.5 * np.sqrt(3.0) * r, 0]]}[which]
    pos = np.asarray(pos, dtype=np.float64) + np.array([17.3, 18.1, 19.7])
    n = pos.shape[0]
    t = np.zeros(n, np.int32) if types is None else np.asarray(types[:n], np.int32)
    return dict(pos=np.ascontiguousarray(pos.T), type=t, h=np.diag([40.0, 40.0, 40.0]).reshape(9),
                pbc=np.array([0, 0, 0], np.int32), mass=np.full(n, 30.0))


# ---------------------------------------------------------------- FP64 references

def _pairs(s, rc):
    """Yield (i, j[], r_ij[3, m], d[m]) over all ordered pairs j != i with |r_ij| < rc, r_ij = r_j - r_i
    under the fractional minimum image (periodic directions only)."""
    H = np.asarray(s["h"], dtype=np.float64).reshape(3, 3)
    Hi = np.linalg.inv(H)
    pbc = np.asarray(s["pbc"]).astype(bool)
    pos = np.asarray(s["pos"], dtype=np.float64)
    n = pos.shape[1]
    idx = np.arange(n)
    for i in range(n):
        d = pos - pos[:, i:i + 1]
        f = Hi @ d
        f[pbc] -= np.round(f[pbc])
        d = H @ f
        r = np.sqrt((d * d).sum(axis=0))
        m = (r < rc) & (idx != i)
        yield i, idx[m], d[:, m], r[m]


_VMAP = [(0, 0), (1, 1), (2, 2), (0, 1), (0, 2), (1, 2), (1, 0), (2, 0), (2, 1)]


def _virial(d, c):
    """sum_j r^a r^b c_j for the 9 GPUMD components."""
    return np.array([(d[a] * d[b] * c).sum() for a, b in _VMAP])


def lj64(table, s):
    """Truncated, unshifted 12-6 LJ with a cutoff per type pair (the reference's form)."""
    n = s["type"].shape[0]
    ty = np.asarray(s["type"])
    pe, f, v = np.zeros(n), np.zeros((3, n)), np.zeros((9, n))
    for i, j, d, r in _pairs(s, table[..., 2].max()):
        p = table[ty[i], ty[j]]
        eps, sig, rc = p[:, 0], p[:, 1], p[:, 2]
        keep = r < rc
        j, d, r, eps, sig = j[keep], d[:, keep], r[keep], eps[keep], sig[keep]
        sr6 = (sig / r) ** 6
        u = 4 * eps * (sr6 * sr6 - sr6)
        du = 4 * eps * (-12 * sr6 * sr6 + 6 * sr6) / r  # dU/dr
        pe[i] = 0.5 * u.sum()
        f[:, i] = (d * (du / r)).sum(axis=1)
        v[:, i] = _virial(d, -0.5 * du / r)
    return dict(pe=pe, force=f, virial=v)


def eam_read(path):
    toks = open(path).read().split()
    nt = int(toks[1])
    vals = np.array([float(t) for t in toks[2 + nt:]])
    if toks[0] == "eam_zhou_2004":
        return "zhou", nt, vals[:21 * nt].reshape(nt, 21)
    return "dai", 1, vals[:9]


def _zhou(p, r):
    """Zhou, Johnson & Wadley (PRB 69, 144113): phi_aa(r), f_a(r) and their derivatives."""
    re, fe, _, _, al, be, A, B, ka, la = p[:10]
    x = r / re
    t1, t2 = (x - ka) ** 20, (x - la) ** 20
    dt1, dt2 = 20 * (x - ka) ** 19 / re, 20 * (x - la) ** 19 / re
    e1, e2 = np.exp(-al * (x - 1)), np.exp(-be * (x - 1))
    phi = A * e1 / (1 + t1) - B * e2 / (1 + t2)
    dphi = (A * e1 * (-al / re) / (1 + t1) - A * e1 * dt1 / (1 + t1) ** 2
            - B * e2 * (-be / re) / (1 + t2) + B * e2 * dt2 / (1 + t2) ** 2)
    fr = fe * e2 / (1 + t2)
    dfr = fe * e2 * (-be / re) / (1 + t2) - fe * e2 * dt2 / (1 + t2) ** 2
    return phi, dphi, fr, dfr


def _zhou_embed(p, rho):
    rho_e, rho_s = p[2], p[3]
    Fn, Fm, eta, Fe = p[10:14], p[14:18], p[18], p[19]
    rho_n, rho_0 = 0.85 * rho_e, 1.15 * rho_e
    if rho < rho_n:
        x = rho / rho_n - 1
        return sum(Fn[k] * x ** k for k in range(4)), sum(k * Fn[k] * x ** (k - 1) for k in range(1, 4)) / rho_n
    if rho < rho_0:
        x = rho / rho_e - 1
        return sum(Fm[k] * x ** k for k in range(4)), sum(k * Fm[k] * x ** (k - 1) for k in range(1, 4)) / rho_e
    y = rho / rho_s
    F = Fe * (1 - eta * np.log(y)) * y ** eta
    dF = Fe * (-eta / rho * y ** eta + (1 - eta * np.log(y)) * eta * y ** eta / rho)
    return F, dF


def zhou_branch(path, rho, t=0):
    """0: rho < 0.85 rho_e, 1: middle polynomial, 2: rho >= 1.15 rho_e (power/log form)."""
    _, _, P = eam_read(path)
    rho_e = P[t][2]
    return np.where(rho < 0.85 * rho_e, 0, np.where(rho < 1.15 * rho_e, 1, 2))


def _eam_pair_terms(model, P, ti, tj, r):
    """phi(r), phi'(r), f_{tj}(r) [density at i], f'_{tj}, f'_{ti} [density at j]."""
    if model == "dai":
        A, dd, c, c0, c1, c2, c3, c4, B = P
        poly = c0 + r * (c1 + r * (c2 + r * (c3 + r * c4)))
        dpoly = c1 + r * (2 * c2 + r * (3 * c3 + r * 4 * c4))
        inside_c = r <= c
        phi = np.where(inside_c, (r - c) ** 2 * poly, 0.0)
        dphi = np.where(inside_c, 2 * (r - c) * poly + (r - c) ** 2 * dpoly, 0.0)
        inside_d = r <= dd
        fr = np.where(inside_d, (r - dd) ** 2 + B * B * (r - dd) ** 4, 0.0)
        dfr = np.where(inside_d, 2 * (r - dd) + 4 * B * B * (r - dd) ** 3, 0.0)
        return phi, dphi, fr, dfr, dfr
    phi, dphi = np.zeros_like(r), np.zeros_like(r)
    fj, dfj, dfi = np.zeros_like(r), np.zeros_like(r), np.zeros_like(r)
    for b in np.unique(tj):
        m = tj == b
        pa, dpa, fa, dfa = _zhou(P[ti], r[m])
        pb, dpb, fb, dfb = _zhou(P[b], r[m])
        fj[m], dfj[m], dfi[m] = fb, dfb, dfa
        if b == ti:
            phi[m], dphi[m] = pa, dpa
        else:  # phi_ab = (f_b / f_a phi_aa + f_a / f_b phi_bb) / 2
            phi[m] = 0.5 * (fb / fa * pa + fa / fb * pb)
            dphi[m] = 0.5 * ((dfb * fa - fb * dfa) / fa ** 2 * pa + fb / fa * dpa
                             + (dfa * fb - fa * dfb) / fb ** 2 * pb + fa / fb * dpb)
    return phi, dphi, fj, dfj, dfi


def eam64(path, s, return_rho=False, f32_params=False):
    """f32_params: the file's parameters rounded to float first, as the reference (and the kernels)
    hold them.  Dai-2006's pair polynomial cancels to ~1e-2 of its terms, so that rounding alone moves
    its energy by ~4e-5 eV/atom; with it the FP32 restatement sits within 5e-7 eV/atom."""
    model, nt, P = eam_read(path)
    if f32_params:
        P = P.astype(np.float32).astype(np.float64)
    rc = max(P[:, 20]) if model == "zhou" else max(P[1], P[2])
    n = s["type"].shape[0]
    ty = np.asarray(s["type"])
    pairs = list(_pairs(s, rc))
    terms = [_eam_pair_terms(model, P, ty[i], ty[j], r) for i, j, d, r in pairs]
    rho = np.array([t[2].sum() for t in terms])
    F, dF = np.zeros(n), np.zeros(n)
    for i in range(n):
        if model == "dai":
            F[i] = -P[0] * np.sqrt(rho[i])
            dF[i] = -0.5 * P[0] / np.sqrt(rho[i]) if rho[i] > 0 else 0.0
        else:
            F[i], dF[i] = _zhou_embed(P[ty[i]], rho[i])
    pe, f, v = F.copy(), np.zeros((3, n)), np.zeros((9, n))
    for (i, j, d, r), (phi, dphi, fj, dfj, dfi) in zip(pairs, terms):
        pe[i] += 0.5 * phi.sum()
        dE = dphi + dF[i] * dfj + dF[j] * dfi  # d(total E)/dr of the pair
        f[:, i] = (d * (dE / r)).sum(axis=1)
        v[:, i] = _virial(d, -(0.5 * dphi + dF[j] * dfi) / r)
    out = dict(pe=pe, force=f, virial=v)
    if return_rho:
        out["rho"] = rho
    return out


def reference64(kind, path, s, f32_params=False):
    """FP64 truth: the numpy references for LJ and EAM, the oracle's FP64 Tersoff (the reference's own
    Tersoff is FP64, and the oracle is self-checked by finite differences in test_classical_cpu.py)."""
    if kind == "lj":
        return lj64(lj_table(path), s)
    if kind == "eam":
        return eam64(path, s, f32_params=f32_params)
    from oracle import oracle_py
    nt, p = oracle_py.tersoff_parameters(path)
    return oracle_py.tersoff_compute(nt, p, s["type"], s["h"], s["pbc"], s["pos"])


def oracle32(kind, path, s):
    """The FP32 restatement of the reference (oracle/*.c), loaded from the potential file."""
    from oracle import oracle_py
    if kind == "lj":
        return oracle_py.lj_compute(lj_table(path), s["type"], s["h"], s["pbc"], s["pos"])
    if kind == "tersoff":
        nt, p = oracle_py.tersoff_parameters(path)
        return oracle_py.tersoff_compute(nt, p, s["type"], s["h"], s["pbc"], s["pos"])
    model, nt, p = oracle_py.eam_parameters(path)
    return oracle_py.eam_compute(model, nt, p, s["type"], s["h"], s["pbc"], s["pos"])


def wrap(h, pbc, pos):
    """Positions mapped into the box along its periodic directions (the reference's apply_pbc)."""
    from oracle import oracle_py
    return oracle_py.apply_pbc(h, pbc, pos)


def gaps(r32, r64):
    return (np.abs(r32["force"] - r64["force"]).max(), np.abs(r32["virial"] - r64["virial"]).max(),
            np.abs(r32["pe"] - r64["pe"]).max())


def v33(virial):
    """Summed GPUMD 9-virial -> row-major 3x3 (xx xy xz / yx yy yz / zx zy zz)."""
    v = np.asarray(virial).sum(axis=1)
    return np.array([v[0], v[3], v[4], v[6], v[1], v[5], v[7], v[8], v[2]])

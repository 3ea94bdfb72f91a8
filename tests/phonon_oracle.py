"""Numpy restatement of the reference's phonon calculation (src/phonon/hessian.cu, src/force/force_constant.cu):
kpoints.in parsing, the k-path and its omega2.out header, the force constants by both finite-difference schemes
(the reference's neighbour displacement and the basis displacement libb200md uses), D(k), and the output
layouts.  Positions are [3, n], h [9] row-major with the lattice vectors as columns."""
import numpy as np

PI = 3.14159265358979                      # src/utilities/common.cuh:20
TIME_UNIT_CONVERSION = 1.018051e+1         # src/utilities/common.cuh:26
NATURAL_TO_THZ2 = 1.0e6 / (TIME_UNIT_CONVERSION * TIME_UNIT_CONVERSION)


def parse_kpoints(text):
    """hessian.cu:116-153: (segments of fractional k-points, names per segment).  A blank line closes a
    segment, a line whose first token starts with '#' is skipped, a line needs 4 tokens."""
    segs, names, cur, cur_names = [], [], [], []
    for line in text.split("\n"):
        t = line.split()
        if not t:
            if cur:
                segs.append(cur), names.append(" ".join(cur_names))
                cur, cur_names = [], []
            continue
        if t[0][0] == "#":
            continue
        if len(t) < 4:
            raise ValueError("kpoints.in file at least 4 parameters for each line.")
        cur.append([float(x) for x in t[:3]])
        cur_names.append(t[3])
    if cur:
        segs.append(cur), names.append(" ".join(cur_names))
    return segs, names


def inverse(h):
    """The inverse box matrix (Box::get_inverse, src/model/box.cu:60-78), h [9] -> [3, 3]."""
    h = np.asarray(h, dtype=np.float64).reshape(9)
    return np.linalg.inv(h.reshape(3, 3))


def kpath(segs, h, cxyz, inv=None):
    """hessian.cu:155-197: Cartesian k-points [nk, 3], kpath [nk], kpath at the high-symmetry points."""
    inv = inverse(h) if inv is None else np.asarray(inv).reshape(3, 3)
    rec = 2.0 * PI * np.asarray(cxyz, dtype=np.float64)[None, :] * inv.T   # rec[j][i] = 2 pi c_i inv[i][j]
    pts = [[rec @ np.asarray(k) for k in s] for s in segs]
    ks, path, sym = [pts[0][0]], [0.0], [0.0]
    for s in pts:
        for a, b in zip(s[:-1], s[1:]):
            for j in range(1, 101):
                k = a + (j * 0.01) * (b - a)
                path.append(path[-1] + np.linalg.norm(k - ks[-1] if j > 1 else k - a))
                ks.append(k)
            sym.append(path[-1])
    return np.array(ks), np.array(path), np.array(sym)


def header(sym, names):
    return "#" + "".join(" %.6f" % s for s in sym) + " " + "|".join(names)


def mic(h, pbc, r):
    """apply_mic (src/model/box.cuh:37-82) on r [3, m]."""
    H = np.asarray(h, dtype=np.float64).reshape(3, 3)
    s = np.linalg.solve(H, r)
    for d in range(3):
        if pbc[d]:
            s[d] -= np.rint(s[d])
    return H @ s


def geometry(x, h, pbc, nb, cutoff):
    """r12 [nb, n, 3] = x[n2] - x[n1] under the minimum image, and the mask |r12| <= cutoff."""
    r = np.stack([mic(h, pbc, x - x[:, [b]]).T for b in range(nb)])
    return r, (r * r).sum(axis=2) <= cutoff * cutoff


def h_basis(forces, x, nb, d, mask):
    """The basis-displacement scheme: H[n1][n2][a*3+b] = (F_n2^b(n1 at -d along a) - F_n2^b(+d)) / 2d."""
    n = x.shape[1]
    H = np.zeros((nb, n, 9))
    for n1 in range(nb):
        for a in range(3):
            f = []
            for s in (-d, d):
                y = x.copy()
                y[a, n1] += s
                f.append(forces(y))
            H[n1, :, a * 3:a * 3 + 3] = ((f[0] - f[1]) / (2 * d)).T
    return H * mask[:, :, None]


def h_neighbour(forces, x, nb, d, mask):
    """The reference's scheme (force_constant.cu:80-133): H[n1][n2][a*3+b] = (F_n1^a(n2 at -d along b) -
    F_n1^a(+d)) / 2d, for n2 within the cutoff."""
    n = x.shape[1]
    H = np.zeros((nb, n, 9))
    for n1 in range(nb):
        for n2 in np.nonzero(mask[n1])[0]:
            for b in range(3):
                f = []
                for s in (-d, d):
                    y = x.copy()
                    y[b, n2] += s
                    f.append(forces(y)[:, n1])
                H[n1, n2, b::3] = (f[0] - f[1]) / (2 * d)
    return H


def dynamical(H, r12, mask, mass, kpts, gamma_only=False):
    """hessian.cu:391-419 (find_D without the phase for one k-point): D [nk, dim, dim] (row, col)."""
    nb, n = H.shape[:2]
    dim = 3 * nb
    D = np.zeros((len(kpts), dim, dim), dtype=complex)
    for k, kv in enumerate(kpts):
        for b1 in range(nb):
            for n2 in range(n):
                if not mask[b1, n2]:
                    continue
                b2 = n2 % nb
                ph = 1.0 if gamma_only else np.exp(1j * np.dot(kv, r12[b1, n2]))
                D[k, 3 * b1:3 * b1 + 3, 3 * b2:3 * b2 + 3] += H[b1, n2].reshape(3, 3) * ph / np.sqrt(mass[b1] * mass[b2])
    return D


def omega2_lines(path, omega2):
    return ["%.6f " % p + "".join("%g " % w for w in row) for p, row in zip(path, omega2)]

"""numpy restatements of the direct-NEMD pieces (src/integrate/ensemble_{lan,nhc,bdp}.cu heat branches,
src/integrate/ensemble.cu:700-879, src/measure/compute.cu), the yardsticks of tests/test_gpu_nemd.py."""
import numpy as np

from oracle.oracle_py import BdpOracle  # noqa: F401  std::mt19937 + resamplekin, pinned to libstdc++

K_B = 8.617343e-5
VIRIAL_ROWS = [0, 3, 4, 6, 1, 5, 7, 8, 2]  # xx xy xz yx yy yz zx zy zz, compute.cu:416-433
QUANTITIES = ("temperature", "potential", "force", "virial", "jp", "jk", "momentum")


def contents(label):
    """Group::find_contents: sizes per group and the atom indices sorted by group, then index."""
    label = np.asarray(label, np.int64)
    return np.bincount(label), np.argsort(label, kind="stable")


def per_atom_columns(mass, pe, force, virial, vel):
    """[23, N]: the per-atom quantities of compute.cu:85-175 in the reference's column order."""
    n = mass.shape[0]
    f, w, v = force.reshape(3, n), virial.reshape(9, n)[VIRIAL_ROWS], vel.reshape(3, n)
    v2 = (v * v).sum(0)
    e = mass * v2 * 0.5 + pe
    jp = np.stack([(w[3 * r:3 * r + 3] * v).sum(0) for r in range(3)])
    return np.concatenate([(mass * v2 / (3 * K_B))[None], pe[None], f, w, jp, v * e[None], v * mass[None]])


def select(quantities):
    width = dict(zip(QUANTITIES, (1, 1, 3, 9, 3, 3, 3)))
    cols, q = [], 0
    for name in QUANTITIES:
        if name in quantities:
            cols += list(range(q, q + width[name]))
        q += width[name]
    return cols


def group_sums(label, num_groups, columns):
    """[C, Ng] sums of each column over each group (the reference's find_group_sum_*)."""
    out = np.zeros((columns.shape[0], num_groups))
    for g in range(num_groups):
        out[:, g] = columns[:, label == g].sum(axis=1)
    return out


def vc_and_ke(mass, vel, idx):
    """gpu_find_vc_and_ke (ensemble.cu:700-782) for one group: centre-of-mass velocity and twice the
    relative kinetic energy."""
    m, v = mass[idx], vel[:, idx]
    mc = m.sum()
    vc = (v * m).sum(1) / mc
    return vc, (m * (v * v).sum(0)).sum() - mc * (vc * vc).sum()


def nhc_init(kT, tau, dof):
    """Ensemble_NHC heat constructor, ensemble_nhc.cu:70-86: eta[4], v_eta[4], Q[4]."""
    s = np.array([0, 0, 0, 0, 1.0, -1.0, 1.0, -1.0] + [kT * tau * tau] * 4)
    s[8] *= dof
    return s


def nhc_chain(state, ek2, dof, kT, dt_half):
    """The reference's nhc() (ensemble_nhc.cu:101-171); updates state in place, returns the factor."""
    M = 4
    w = [0.784513610477560, 0.235573213359357, -1.17767998417887, 1.31518632068391, -1.17767998417887,
         0.235573213359357, 0.784513610477560]
    eta, ve, Q = state[:4], state[4:8], state[8:12]
    factor = 1.0
    for a in range(7):
        dt2 = dt_half * w[a] / 4.0
        dt4, dt8 = 0.5 * dt2, 0.25 * dt2
        for _ in range(4):
            ve[M - 1] += dt4 * (ve[M - 2] ** 2 / Q[M - 2] - kT)
            for m in range(M - 2, -1, -1):
                damp = np.exp(-dt8 * ve[m + 1] / Q[m + 1])
                G = ek2 - dof * kT if m == 0 else ve[m - 1] ** 2 / Q[m - 1] - kT
                ve[m] = damp * (damp * ve[m] + dt4 * G)
            eta += dt2 * ve / Q
            f = np.exp(-dt2 * ve[0] / Q[0])
            ek2 *= f * f
            factor *= f
            for m in range(M - 1):
                damp = np.exp(-dt8 * ve[m + 1] / Q[m + 1])
                G = ek2 - dof * kT if m == 0 else ve[m - 1] ** 2 / Q[m - 1] - kT
                ve[m] = damp * (damp * ve[m] + dt4 * G)
            ve[M - 1] += dt4 * (ve[M - 2] ** 2 / Q[M - 2] - kT)
    return factor


def nhc_energy(state, ek2, dof, kT):
    """Conserved extended energy of a chain driving a kinetic energy ek2 / 2 (Martyna-Tuckerman)."""
    eta, ve, Q = state[:4], state[4:8], state[8:12]
    return 0.5 * ek2 + (0.5 * ve * ve / Q).sum() + dof * kT * eta[0] + kT * eta[1:].sum()


class HeatLan:
    """heat_lan's bath (Ensemble_LAN heat branch, ensemble_lan.cu:43-85,128-195, with the groups' gpu_langevin
    of langevin_utilities.cuh:127-149): two XORWOW streams, curand_init(seed_source, m, 0) for the m-th
    source atom and curand_init(seed_sink, m, 0) for the m-th sink atom, m the position within the group
    in `contents` order.  Each half kicks v <- c1 v + c2_g / sqrt(m) xi on the source then the sink
    (c1 = exp(-1/2 / Tc), c2_g = sqrt((1 - c1^2) k_B (T +- dT))), with no momentum correction, and adds
    1/2 sum m (v_before^2 - v_after^2) to the group's energy.  Other atoms are untouched."""

    def __init__(self, mass, label, source, sink, T, Tc, dT, seed_source, seed_sink):
        from curand_oracle import XorwowStates
        self.mass = np.asarray(mass, dtype=np.float64)
        sizes, order = contents(label)
        start = np.concatenate([[0], np.cumsum(sizes)])
        self.atoms = [order[start[g]:start[g + 1]] for g in (source, sink)]
        self.c1 = float(np.exp(-0.5 / Tc))
        self.c2 = [float(np.sqrt((1.0 - self.c1 * self.c1) * K_B * t)) for t in (T + dT, T - dT)]
        self.noise = [XorwowStates(seed, np.arange(idx.shape[0]))
                      for seed, idx in zip((seed_source, seed_sink), self.atoms)]
        self.energy = np.zeros(2)

    def half(self, vel):
        v = np.array(vel, dtype=np.float64)
        for g in range(2):
            idx = self.atoms[g]
            m = self.mass[idx]
            v0 = v[:, idx]
            v1 = self.c1 * v0 + (self.c2[g] * np.sqrt(1.0 / m))[None, :] * self.noise[g].normal_double(3)
            v[:, idx] = v1
            self.energy[g] += (0.5 * m * (v0 * v0 - v1 * v1).sum(axis=0)).sum()
        return v


def bdp_factors(mt, mass, vel, src, snk, T, dT, Tc):
    """integrate_heat_bdp_2 (ensemble_bdp.cu:103-149): factors and energies of source then sink; mt is a
    BdpOracle (one stream for both groups)."""
    out = []
    for idx, temp in ((src, T + dT), (snk, T - dT)):
        vc, ke2 = vc_and_ke(mass, vel, idx)
        dN = 3 * (idx.shape[0] - 1)
        ek = 0.5 * ke2
        f = np.sqrt(mt.resamplekin(ek, dN * K_B * temp * 0.5, dN, Tc) / ek)
        out.append((vc, f, ek * (1.0 - f * f)))
    return out

"""float64 restatement of one whole MD step of each ensemble, with `fix` / `move` groups: the pieces of
oracle/oracle_py.py (velocity_verlet_groups, find_thermo, nhc_state / nhc_chain, berendsen_factor,
BdpOracle, berendsen_pressure, apply_pbc) put together in the reference's order.  The yardstick of
tests/test_gpu_ensemble_steps.py, which restates every step from the device's own state before it.

Group rules shared by every ensemble (src/integrate/ensemble.cu:111-174, 645-651):
  - atoms of the fixed group keep their position and have zero velocity;
  - atoms of the moving group translate by move_velocity * dt in step 1 and store zero velocity;
  - the temperature counts the other n_temperature = N - N_fixed - N_move atoms.
"""
import numpy as np

from curand_oracle import XorwowStates
from oracle import oracle_py as O

K_B = 8.617343e-5                    # src/utilities/common.cuh:21
PRESSURE_UNIT_CONVERSION = 1.602177e+2  # src/utilities/common.cuh:25
KINDS = ("nve", "nvt_ber", "nvt_nhc", "nvt_bdp", "npt_ber", "nvt_lan", "nvt_bao")
LANGEVIN_SEED = 1804289383  # glibc's first rand(): the seed of an unseeded run's first Langevin ensemble


def pressure_parameters(target_pressure, elastic_modulus, tau_p):
    """`ensemble npt_ber T T tau p.. C.. tau_p` in natural units: 6 target pressures and 6 couplings,
    coupling 1 / (3 tau_p C) and 0 for C > 2000 GPa (integrate.cu:700-712, 1150-1153)."""
    p = np.atleast_1d(np.asarray(target_pressure, dtype=np.float64))
    c = np.ones(6)
    c[:p.shape[0]] = np.atleast_1d(np.asarray(elastic_modulus, dtype=np.float64))
    p0 = np.zeros(6)
    p0[:p.shape[0]] = p
    pc = np.where(c > 2.0e3, 0.0, 1.0 / (float(tau_p) * 3.0 * c))
    return p.shape[0], p0 / PRESSURE_UNIT_CONVERSION, pc * PRESSURE_UNIT_CONVERSION


class EnsembleStep:
    """One ensemble, its thermostat state carried from step to step.  Arrays are SoA float64: pos and vel
    [3, N], force [3, N], virial [9, N], h[9] row-major with the lattice vectors as columns."""

    def __init__(self, kind, mass, time_step, pbc=(1, 1, 1), label=None, fixed_group=-1, move_group=-1,
                 move_velocity=(0.0, 0.0, 0.0), temperature=300.0, temperature_coupling=100.0,
                 seed=None, target_pressure=None, elastic_modulus=None, tau_p=None):
        if kind not in KINDS:
            raise ValueError(kind)
        self.kind = kind
        self.mass = np.ascontiguousarray(mass, dtype=np.float64)
        n = self.mass.shape[0]
        self.n = n
        self.dt = float(time_step)
        self.pbc = np.asarray(pbc, dtype=np.int32)
        self.fixed_group, self.move_group = int(fixed_group), int(move_group)
        if label is None and max(self.fixed_group, self.move_group) >= 0:
            raise ValueError("fix / move need group labels")
        # no groups: every atom in group 0, and no group is -1
        self.label = np.zeros(n, np.int32) if label is None else np.asarray(label, dtype=np.int32)
        self.move_velocity = np.asarray(move_velocity, dtype=np.float64)
        # ensemble.cu:645-651
        self.n_temperature = n - sum(int((self.label == g).sum()) for g in (self.fixed_group, self.move_group)
                                     if g >= 0)
        self.temperature, self.temperature_coupling = float(temperature), float(temperature_coupling)
        if kind == "nvt_nhc":
            # Ensemble_NHC::Ensemble_NHC (ensemble_nhc.cu:31-50): the chain's dN = 3N counts every atom,
            # fixed and moving ones included (ensemble_nhc.cu:185-198)
            self.chain = O.nhc_state(n, self.temperature, self.temperature_coupling, self.dt)
        if kind == "nvt_bdp":
            # integrate_nvt_bdp_2 (ensemble_bdp.cu:87-95): ndeg = 3 (N - N_fixed - N_move)
            self.ndeg = 3 * self.n_temperature
            if self.ndeg < 3:
                raise ValueError("nvt_bdp needs at least one atom outside the fixed and moving groups")
            self.bdp = O.BdpOracle(12345678 if seed is None else seed)
        if kind == "npt_ber":
            self.num_p, self.p0, self.pc = pressure_parameters(target_pressure, elastic_modulus, tau_p)
        if kind in ("nvt_lan", "nvt_bao"):
            # ensemble_lan.cu:35-39 / ensemble_bao.cu:35-39: c1 = exp(-1/2 / tau) for the half kicks of
            # nvt_lan, exp(-1 / tau) for nvt_bao's whole O step; curand_init(seed, i, 0) per atom
            self.c1 = float(np.exp((-0.5 if kind == "nvt_lan" else -1.0) / self.temperature_coupling))
            self.noise = XorwowStates(LANGEVIN_SEED if seed is None else seed, np.arange(n))

    # ---- the pieces
    def velocity_verlet(self, step1, pos, vel, force):
        """Ensemble::velocity_verlet, ensemble.cu:348-397 (ensemble.cu:111-174 with groups)."""
        return O.velocity_verlet_groups(step1, self.dt, self.mass, pos, vel, force, self.label,
                                        self.fixed_group, self.move_group, self.move_velocity)

    def find_thermo(self, h, pe, vel, virial):
        """Ensemble::find_thermo, ensemble.cu:636-673: T over the integrated atoms, U, 6 stresses."""
        volume = abs(float(np.linalg.det(np.asarray(h, dtype=np.float64).reshape(3, 3))))
        return O.find_thermo(self.n_temperature, volume, self.mass, pe, vel, virial)

    def nhc_half(self, t_now, vel):
        """The thermostat half of integrate_nvt_nhc_1 / _2 (ensemble_nhc.cu:173-237): the chain with
        ek2 = T * 3N * k_B (T over the integrated atoms, 3N over all atoms, :194-196)."""
        ek2 = t_now * 3.0 * self.n * K_B
        factor = O.nhc_chain(self.chain, ek2, K_B * self.temperature, 3.0 * self.n, 0.5 * self.dt)
        return vel * factor

    def langevin(self, vel):
        """gpu_langevin + gpu_find_momentum + gpu_correct_momentum (langevin_utilities.cuh:26-127):
        v <- c1 v + c2 / sqrt(m) xi on every atom, fixed ones included, with xi drawn x, y, z per atom and
        c2 = sqrt((1 - c1^2) k_B T) from the target temperature of this kick; then the total momentum
        (float64 sums) is removed."""
        c2 = np.sqrt((1.0 - self.c1 * self.c1) * K_B * self.temperature)
        xi = self.noise.normal_double(3)
        v = self.c1 * vel + (c2 * np.sqrt(1.0 / self.mass))[None, :] * xi
        return v - (v * self.mass).sum(axis=1, keepdims=True) / self.mass.sum()

    def baoab(self, which, pos, vel, force):
        """gpu_operator_A (which 0) / gpu_operator_B (which 1) with the fixed group frozen."""
        return O.baoab_operator(which, self.dt, self.mass, pos, vel, force, self.label, self.fixed_group)

    # ---- the two halves around the force call
    def compute1(self, h, pos, vel, force):
        """Ensemble::compute1 up to the force call: (pos, vel)."""
        if self.kind == "nvt_lan":  # ensemble_lan.cu:197-227: kick, then velocity-Verlet step 1
            vel = self.langevin(vel)
        if self.kind == "nvt_bao":  # ensemble_bao.cu:419-479: B A O A
            pos, vel = self.baoab(1, pos, vel, force)
            pos, vel = self.baoab(0, pos, vel, force)
            vel = self.langevin(vel)
            return self.baoab(0, pos, vel, force)
        if self.kind == "nvt_nhc":  # find_thermo, then the chain (ensemble_nhc.cu:184-195)
            vel = self.nhc_half(self.find_thermo(h, np.zeros(self.n), vel, np.zeros((9, self.n)))[0], vel)
        return self.velocity_verlet(True, pos, vel, force)

    def compute2(self, h, pos, vel, force, pe, virial):
        """Ensemble::compute2 after the force call: (pos, vel, h, thermo[8]).  thermo is the one
        find_thermo leaves: before any thermostat or barostat acts on the state, except for nvt_lan,
        whose second kick comes before find_thermo."""
        h = np.array(h, dtype=np.float64).reshape(9)
        pos = np.array(pos, dtype=np.float64)
        if self.kind == "nvt_bao":  # Ensemble_BAO::compute2, ensemble_bao.cu:481: B, then thermo
            _, vel = self.baoab(1, pos, vel, force)
            return pos, vel, h, self.find_thermo(h, pe, vel, virial)
        _, vel = self.velocity_verlet(False, pos, vel, force)
        if self.kind == "nvt_lan":  # Ensemble_LAN::compute2, ensemble_lan.cu:229: step 2, kick, then thermo
            vel = self.langevin(vel)
        thermo = self.find_thermo(h, pe, vel, virial)
        T, Tc = self.temperature, self.temperature_coupling
        if self.kind in ("nvt_ber", "npt_ber"):  # Ensemble_BER::compute2, ensemble_ber.cu:195-233
            vel = vel * O.berendsen_factor(T, Tc, thermo[0])
        elif self.kind == "nvt_nhc":  # ensemble_nhc.cu:225-236
            vel = self.nhc_half(thermo[0], vel)
        elif self.kind == "nvt_bdp":  # ensemble_bdp.cu:91-100
            vel = vel * self.bdp.factor(thermo[0], self.n_temperature, T, Tc)
        if self.kind == "npt_ber":  # ensemble_ber.cu:235-285, with the stress before the scaling above
            h, mu = O.berendsen_pressure(h, self.pbc, thermo, self.p0, self.pc, self.num_p)
            pos = mu.reshape(3, 3) @ pos
        return pos, vel, h, thermo

    def step(self, h, pos, vel, force_before, force_after, pe_after, virial_after):
        """One whole step: compute1, the force driver's wrap into the box (Force::compute, force.cu:771-801),
        compute2 with the forces the force call returned.  Returns (pos, vel, h, thermo[8])."""
        pos, vel = self.compute1(h, pos, vel, force_before)
        pos = O.apply_pbc(h, self.pbc, pos)
        return self.compute2(h, pos, vel, force_after, pe_after, virial_after)

"""Numpy restatements of the reference's HNEMD drive and heat-current sum, and of its SHC ring,
correlation and post-processing (src/force/force.cu:228-312,857-897; src/measure/hnemd_kappa.cu;
src/measure/shc.cu).  Test infrastructure only."""
import math

import numpy as np

KAPPA_UNIT_CONVERSION = 1.573769e+5   # src/utilities/common.cuh:27
TIME_UNIT_CONVERSION = 1.018051e+1    # src/utilities/common.cuh:26
PI = 3.14159265358979                 # src/utilities/common.cuh:19


def hnemd_drive(virial, force, fe):
    """gpu_add_driving_force + gpu_sum_force + gpu_correct_force (force.cu:228-312, 857-897).
    virial[9, n] in GPUMD order (xx yy zz xy xz yz yx zx zy), force[3, n]; returns the new force."""
    w = np.asarray(virial, dtype=np.float64)
    f = np.array(force, dtype=np.float64)
    fx, fy, fz = (float(x) for x in fe)
    # xx xy xz / yx yy yz / zx zy zz = 0 3 4 / 6 1 5 / 7 8 2
    f[0] += fx * w[0] + fy * w[6] + fz * w[7]
    f[1] += fx * w[3] + fy * w[1] + fz * w[8]
    f[2] += fx * w[4] + fy * w[5] + fz * w[2]
    ftot = f.sum(axis=1)
    f -= (ftot * (1.0 / f.shape[1]))[:, None]
    return f


def hnemd_heat_row(virial, vel):
    """compute_heat + gpu_sum_heat (hnemd_kappa.cu:52-106): the five summed heat-current components."""
    return compute_heat_np(virial, vel).sum(axis=1)


def compute_heat_np(virial, vel):
    """gpu_compute_heat (compute_heat.cu:32-63) in numpy: [5, n] = jx_in jx_out jy_in jy_out jz."""
    w = np.asarray(virial, dtype=np.float64)
    v = np.asarray(vel, dtype=np.float64)
    return np.stack([w[0] * v[0] + w[3] * v[1], w[4] * v[2], w[6] * v[0] + w[1] * v[1], w[5] * v[2],
                     w[7] * v[0] + w[8] * v[1] + w[2] * v[2]])


def hnemd_kappa(rows, volume, temperature, fe):
    """The output branch of HNEMD::process (hnemd_kappa.cu:108-131): rows[output_interval, 5] of heat
    sums -> the kappa.out row (W/mK), xx_in xx_out yy_in yy_out zz."""
    rows = np.asarray(rows, dtype=np.float64)
    oi = rows.shape[0]
    fe_norm = math.sqrt(fe[0] * fe[0] + fe[1] * fe[1] + fe[2] * fe[2])
    factor = KAPPA_UNIT_CONVERSION / oi
    factor /= volume * temperature * fe_norm
    return rows.sum(axis=0) * factor


class ShcRing:
    """SHC::process as the reference computes it (shc.cu:162-310): per output group a ring of Nc frames
    of (s_x, s_y, s_z, v_x, v_y, v_z); from sample_step Nc-1 on, gpu_find_k (shc.cu:81-130) adds
    sum_j s(now) v(slot b) to k_negative[(cs - b) mod Nc] and sum_j v(now) s(slot b) to
    k_positive[...], cs = sample_step mod Nc.  groups: list of index arrays (find_contents order)."""

    def __init__(self, sample_interval, Nc, direction, groups):
        self.si, self.Nc, self.dir = int(sample_interval), int(Nc), int(direction)
        self.groups = [np.asarray(g, dtype=np.int64) for g in groups]
        self.ring = [np.zeros((Nc, 6, len(g))) for g in self.groups]
        self.k = np.zeros((len(groups), 4, Nc))  # neg_i neg_o pos_i pos_o
        self.num_time_origins = 0

    def process(self, step, virial, vel):
        if (step + 1) % self.si:
            return
        sample_step = step // self.si
        cs = sample_step % self.Nc
        rows = [[0, 3, 4], [6, 1, 5], [7, 8, 2]][self.dir]  # shc.cu:188
        w, v = np.asarray(virial), np.asarray(vel)
        for g, idx in enumerate(self.groups):
            self.ring[g][cs] = np.concatenate([w[rows][:, idx], v[:, idx]])
        if sample_step < self.Nc - 1:
            return
        self.num_time_origins += 1
        for g in range(len(self.groups)):
            r = self.ring[g]
            now = r[cs]
            for b in range(self.Nc):
                lag = cs - b if b <= cs else cs + self.Nc - b
                self.k[g, 0, lag] += np.sum(now[0] * r[b, 3] + now[1] * r[b, 4])
                self.k[g, 1, lag] += np.sum(now[2] * r[b, 5])
                self.k[g, 2, lag] += np.sum(now[3] * r[b, 0] + now[4] * r[b, 1])
                self.k[g, 3, lag] += np.sum(now[5] * r[b, 2])


def shc_average_k(k, Nc, num_time_origins):
    """SHC::average_k (shc.cu:312-348): k[4, Nc] = neg_i neg_o pos_i pos_o -> ki, ko [2Nc-1] in A eV/ps."""
    k = np.asarray(k, dtype=np.float64)
    scalar = 1000.0 / TIME_UNIT_CONVERSION / num_time_origins
    ki, ko = np.zeros(2 * Nc - 1), np.zeros(2 * Nc - 1)
    ki[:Nc - 1] = k[0, Nc - 1:0:-1] * scalar
    ko[:Nc - 1] = k[1, Nc - 1:0:-1] * scalar
    ki[Nc - 1:] = k[2] * scalar
    ko[Nc - 1:] = k[3] * scalar
    return ki, ko


def shc_window(ki, ko, Nc):
    """The Hann window of SHC::find_shc (shc.cu:356-359); the windowed ki, ko are what shc.out lists."""
    nc = np.arange(2 * Nc - 1)
    hann = (np.cos(PI * (nc + 1 - Nc) / Nc) + 1.0) * 0.5
    return np.asarray(ki) * hann, np.asarray(ko) * hann


def shc_transform(ki_w, ko_w, Nc, dt_in_ps, num_omega, max_omega):
    """The cosine transform of SHC::find_shc (shc.cu:362-376) of windowed ki, ko: omega (THz rad),
    shc_i, shc_o (A eV = A eV/ps/THz)."""
    nc = np.arange(2 * Nc - 1)
    omega = (np.arange(num_omega) + 1) * (max_omega / num_omega)
    c = np.cos(omega[:, None] * ((nc + 1 - Nc) * dt_in_ps)[None, :])
    return omega, c @ np.asarray(ki_w) * 2.0 * dt_in_ps, c @ np.asarray(ko_w) * 2.0 * dt_in_ps


def shc_brute_force(s_series, v_series, Nc):
    """The SHC correlations as the double sum they stand for: for every time origin t >= Nc-1 and lag
    0..Nc-1, the sum over atoms of s(t) . v(t-lag) (negative) and v(t) . s(t-lag) (positive), with no
    ring.  s_series, v_series [K, 3, G] of one group -> k[4, Nc] = neg_i neg_o pos_i pos_o, and the
    number of origins."""
    K = s_series.shape[0]
    k = np.zeros((4, Nc))
    if K < Nc:
        return k, 0
    s_now, v_now = s_series[Nc - 1:], v_series[Nc - 1:]
    for lag in range(Nc):
        s_past, v_past = s_series[Nc - 1 - lag:K - lag], v_series[Nc - 1 - lag:K - lag]
        k[0, lag] = np.sum(s_now[:, 0] * v_past[:, 0] + s_now[:, 1] * v_past[:, 1])
        k[1, lag] = np.sum(s_now[:, 2] * v_past[:, 2])
        k[2, lag] = np.sum(v_now[:, 0] * s_past[:, 0] + v_now[:, 1] * s_past[:, 1])
        k[3, lag] = np.sum(v_now[:, 2] * s_past[:, 2])
    return k, K - Nc + 1

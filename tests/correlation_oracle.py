"""Numpy restatement of the reference's time-correlation measurements (compute_dos, compute_sdc,
compute_msd; src/measure/dos.cu, sdc.cu, msd.cu): the per-sample ring arithmetic of gpu_find_vac /
gpu_find_msd and the host post-processing, in the reference's order of operations."""
import numpy as np

PI = 3.14159265358979                # src/utilities/common.cuh:19
TIME_UNIT_CONVERSION = 1.018051e+1   # src/utilities/common.cuh:26


def ring_correlate(frames, Nc, msd=False, weights=None, labels=None, num_groups=1):
    """frames [S, 3, G]: the sampled vectors in order.  The reference's ring of Nc frames: sample s goes
    to slot s % Nc and, from s = Nc - 1 on, is correlated with every slot (dos.cu:84-143, msd.cu:89-149).
    Returns acc [3, Nc] (summed over the atoms) and the number of time origins; with labels [G] (group
    of each atom), acc [num_groups, 3, Nc] of the per-group sums."""
    frames = np.asarray(frames, dtype=np.float64)
    S, _, G = frames.shape
    w = np.ones(G) if weights is None else np.asarray(weights, dtype=np.float64)
    ring = np.zeros((Nc, 3, G))
    if labels is not None:
        per_atom, origins = ring_correlate_per_atom(frames, Nc, msd, w)
        acc = np.zeros((num_groups, 3, Nc))
        np.add.at(acc, np.asarray(labels), per_atom.transpose(2, 0, 1))
        return acc, origins
    acc = np.zeros((3, Nc))
    origins = 0
    for s in range(S):
        cs = s % Nc
        ring[cs] = frames[s]
        if s < Nc - 1:
            continue
        origins += 1
        for bid in range(Nc):
            lag = cs - bid if bid <= cs else cs + Nc - bid
            if msd:
                d = frames[s] - ring[bid]
                acc[:, lag] += (d * d).sum(axis=1)
            else:
                acc[:, lag] += (w * frames[s] * ring[bid]).sum(axis=1)
    return acc, origins


def ring_correlate_per_atom(frames, Nc, msd, w):
    """ring_correlate without the sum over atoms: [3, Nc, G]."""
    S, _, G = frames.shape
    ring = np.zeros((Nc, 3, G))
    acc = np.zeros((3, Nc, G))
    origins = 0
    for s in range(S):
        cs = s % Nc
        ring[cs] = frames[s]
        if s < Nc - 1:
            continue
        origins += 1
        for bid in range(Nc):
            lag = cs - bid if bid <= cs else cs + Nc - bid
            d = frames[s] - ring[bid]
            acc[:, lag] += d * d if msd else w * frames[s] * ring[bid]
    return acc, origins


def brute_force(frames, Nc, msd=False, weights=None):
    """The same sums as direct double sums over time origins s >= Nc - 1 and lags."""
    frames = np.asarray(frames, dtype=np.float64)
    S, _, G = frames.shape
    w = np.ones(G) if weights is None else np.asarray(weights, dtype=np.float64)
    acc = np.zeros((3, Nc))
    for s in range(Nc - 1, S):
        for lag in range(Nc):
            a, b = frames[s], frames[s - lag]
            acc[:, lag] += ((a - b) ** 2).sum(axis=1) if msd else (w * a * b).sum(axis=1)
    return acc, max(S - Nc + 1, 0)


def sampled(step_frames, sample_interval):
    """The frames a run samples: after the steps with (step + 1) % sample_interval == 0."""
    return [f for step, f in enumerate(step_frames) if (step + 1) % sample_interval == 0]


def dos_post(acc, group_size, dt_natural, omega_max, num_dos_points):
    """normalize_vac + find_dos (dos.cu:414-427, 450-481) for one group: mvac [3, Nc], dos [3, n]."""
    Nc = acc.shape[1]
    dt_in_ps = dt_natural * TIME_UNIT_CONVERSION / 1000.0
    with np.errstate(invalid="ignore", divide="ignore"):
        mvac = acc / acc[:, :1]
    vac = mvac.copy()
    for nc in range(Nc):
        hann = (np.cos((PI * nc) / Nc) + 1.0) * 0.5
        vac[:, nc] *= hann if nc == 0 else 2.0 * hann
    d_omega = omega_max / num_dos_points
    dos = np.zeros((3, num_dos_points))
    for nw in range(num_dos_points):
        omega = d_omega + nw * d_omega
        s = np.zeros(3)
        for nc in range(Nc):
            s += vac[:, nc] * np.cos(omega * nc * dt_in_ps)
        dos[:, nw] = s * (dt_in_ps * 2.0 * group_size)
    return mvac, dos


def sdc_post(acc, num_atoms, origins, dt_natural):
    """SDC::postprocess (sdc.cu:239-285): vac in A^2/ps^2 and its running integral in A^2/ps."""
    with np.errstate(divide="ignore", invalid="ignore"):  # an empty group: 1 / 0, then 0 * inf, as in C
        vac = acc * (np.float64(1.0) / (np.float64(num_atoms) * np.float64(origins)))
    dt2 = dt_natural * 0.5
    sdc = np.zeros_like(vac)
    for nc in range(1, vac.shape[1]):
        sdc[:, nc] = sdc[:, nc - 1] + (vac[:, nc - 1] + vac[:, nc]) * dt2
    conv = 1.0e3 / TIME_UNIT_CONVERSION
    return vac * (conv * conv), sdc * conv


def msd_post(acc, num_atoms, origins, dt_natural):
    """MSD::write (msd.cu:369-445): msd in A^2 and the finite-difference sdc in A^2/ps; zeros for an
    empty group."""
    scaler = 1.0 / (float(num_atoms) * float(origins)) if num_atoms > 0 and origins > 0 else 0.0
    msd = acc * scaler
    sdc = np.zeros_like(msd)
    sdc[:, 1:] = (msd[:, 1:] - msd[:, :-1]) * (0.5 / dt_natural)
    return msd, sdc * (1.0e3 / TIME_UNIT_CONVERSION)

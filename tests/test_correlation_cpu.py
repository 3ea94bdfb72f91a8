"""The numpy restatement of compute_dos / compute_sdc / compute_msd (tests/correlation_oracle.py) against
brute-force sums and closed forms; no GPU needed."""
import numpy as np
import pytest

import correlation_oracle as co

DT = 1.0 / co.TIME_UNIT_CONVERSION  # 1 fs in natural units


@pytest.mark.parametrize("msd", [False, True])
@pytest.mark.parametrize("S,Nc", [(23, 7), (7, 7), (40, 10), (31, 1)])
def test_ring_matches_brute_force(msd, S, Nc):
    """The reference's ring bookkeeping, including runs that are not a multiple of Nc and exactly one
    time origin (S = Nc)."""
    rng = np.random.default_rng(S * 10 + Nc)
    frames = rng.normal(size=(S, 3, 13))
    w = None if msd else rng.uniform(1, 50, 13)
    acc, origins = co.ring_correlate(frames, Nc, msd, w)
    ref, ref_origins = co.brute_force(frames, Nc, msd, w)
    assert origins == ref_origins == S - Nc + 1
    assert np.allclose(acc, ref, rtol=1e-13, atol=0)


def test_sampled_frames_follow_the_interval():
    assert co.sampled(list(range(10)), 3) == [2, 5, 8]


def _oscillators(n, S, dt_ps, omegas, damping, seed):
    """S frames of n atoms whose velocities oscillate at the given angular frequencies (rad/ps)."""
    rng = np.random.default_rng(seed)
    w = rng.choice(omegas, size=(3, n))
    phase = rng.uniform(0, 2 * np.pi, (3, n))
    t = np.arange(S)[:, None, None] * dt_ps
    return np.cos(w * t + phase) * np.exp(-damping * t)


def test_dos_sum_rule():
    """sum dos * d_omega / 2pi = N per direction on a fine grid up to the Nyquist frequency (the
    reference's graphene_dos1.out gives 8624 for N = 8640)."""
    n, Nc, interval = 64, 100, 5
    dt_natural = DT * interval
    dt_ps = dt_natural * co.TIME_UNIT_CONVERSION / 1000.0
    frames = _oscillators(n, 400, dt_ps, [30.0, 75.0, 140.0], 2.0, 1)
    acc, _ = co.ring_correlate(frames, Nc, weights=np.full(n, 12.0))
    omega_max = np.pi / dt_ps  # the Nyquist limit dos.cu:286-288 allows
    npts = 4000
    _, dos = co.dos_post(acc, n, dt_natural, omega_max, npts)
    total = dos.sum(axis=1) * (omega_max / npts) / (2 * np.pi)
    assert np.allclose(total, n, rtol=2e-3), total


def test_dos_of_one_frequency_peaks_there():
    n, Nc, interval = 200, 200, 2
    dt_natural = DT * interval
    dt_ps = dt_natural * co.TIME_UNIT_CONVERSION / 1000.0
    frames = _oscillators(n, 500, dt_ps, [60.0], 0.0, 2)
    acc, _ = co.ring_correlate(frames, Nc)
    mvac, dos = co.dos_post(acc, n, dt_natural, 200.0, 400)
    assert np.allclose(mvac[:, 0], 1.0)
    omega = np.arange(1, 401) * 0.5
    assert np.all(np.abs(omega[np.argmax(dos, axis=1)] - 60.0) <= 1.0)


def test_dos_of_an_empty_group_is_nan_like_the_reference():
    mvac, dos = co.dos_post(np.zeros((3, 10)), 0, DT, 100.0, 20)
    assert np.all(np.isnan(mvac)) and np.all(np.isnan(dos))


def test_sdc_of_an_exponential_vac():
    """vac(t) = v0^2 exp(-t / tau) integrates to v0^2 tau (1 - exp(-t / tau)); the trapezoid rule is
    within O(dt^2 / tau^2) of it."""
    Nc, n, origins, v0sq, tau = 400, 10, 7, 3.0e-3, 40 * DT
    t = np.arange(Nc) * DT
    acc = np.tile(n * origins * v0sq * np.exp(-t / tau), (3, 1))
    vac, sdc = co.sdc_post(acc, n, origins, DT)
    conv = 1.0e3 / co.TIME_UNIT_CONVERSION
    assert np.allclose(vac, v0sq * np.exp(-t / tau) * conv * conv, rtol=1e-13)
    exact = v0sq * tau * (1 - np.exp(-t / tau)) * conv
    assert np.allclose(sdc, exact, rtol=1e-3, atol=1e-6 * exact.max())


def test_ballistic_msd():
    """x(t) = x0 + v t: msd(lag) = <(v lag dt)^2> per direction, and the finite-difference sdc grows
    linearly."""
    rng = np.random.default_rng(3)
    n, S, Nc, interval = 50, 60, 20, 2
    dt_natural = DT * interval
    x0, v = rng.uniform(0, 10, (3, n)), rng.normal(size=(3, n)) * 0.01
    frames = x0[None] + v[None] * (np.arange(S)[:, None, None] * dt_natural)
    acc, origins = co.ring_correlate(frames, Nc, msd=True)
    msd, sdc = co.msd_post(acc, n, origins, dt_natural)
    lag = np.arange(Nc) * dt_natural
    assert np.allclose(msd, (v ** 2).mean(axis=1)[:, None] * lag ** 2, rtol=1e-9, atol=1e-20)
    assert sdc[0, 0] == 0.0
    empty, _ = co.msd_post(acc, 0, origins, dt_natural)
    assert np.all(empty == 0.0)

"""HNEMD / SHC post-processing and the restatements the device tests compare against (no GPU needed).

  - the cosine transform of find_shc reproduces the reference's own shc.out of its graphene HNEMD
    regression case (tests/gpumd/graphene_kappa_hnemd/shc1.out, tests/golden/ref_graphene_hnemd_shc1.out);
  - the reference's ring-based SHC bookkeeping (ShcRing: Nc slots, gpu_find_k lag indexing) equals the
    double sum over time origins and atoms it stands for;
  - the kappa.out factor and units against a hand computation."""
import math

import numpy as np
import pytest

import heat_oracle as ho
from conftest import GOLDEN


def read_shc_out(path):
    head, rows = {}, []
    for ln in open(path):
        if ln.startswith("#"):
            parts = ln[1:].split()
            head[parts[0]] = parts[1:]
        elif ln.strip():
            rows.append([float(x) for x in ln.split()])
    return head, np.array(rows)


def test_find_shc_reproduces_reference_shc_out():
    head, rows = read_shc_out(GOLDEN / "ref_graphene_hnemd_shc1.out")
    Nc = (int(head["num_correlation_rows"][0]) + 1) // 2
    num_omega = int(head["num_frequency_rows"][0])
    dt_in_ps = float(head["dt_output"][0])
    max_omega = float(head["compute_shc"][4])
    assert (Nc, num_omega, max_omega) == (250, 1000, 400.0)
    corr, freq = rows[:2 * Nc - 1], rows[2 * Nc - 1:]
    assert freq.shape == (num_omega, 3)
    # the correlation rows are already windowed (find_shc windows ki / ko in place before printing)
    assert np.allclose(corr[:, 0], (np.arange(2 * Nc - 1) + 1 - Nc) * dt_in_ps, rtol=1e-5, atol=1e-12)
    omega, si, so = ho.shc_transform(corr[:, 1], corr[:, 2], Nc, dt_in_ps, num_omega, max_omega)
    assert np.allclose(omega, freq[:, 0], rtol=1e-5)
    # %g keeps 6 significant digits of every input row: the transform of the rounded rows agrees with
    # the printed spectrum to that precision, relative to the spectrum's scale
    for got, want in ((si, freq[:, 1]), (so, freq[:, 2])):
        assert np.allclose(got, want, rtol=2e-5, atol=2e-5 * np.abs(want).max())
    # the window itself: zero at both ends of the 2Nc-1 rows, one at lag 0
    wi, _ = ho.shc_window(np.ones(2 * Nc - 1), np.ones(2 * Nc - 1), Nc)
    assert wi[Nc - 1] == 1.0 and wi[0] < 1e-3 and wi[-1] < 1e-3


@pytest.mark.parametrize("sample_interval,steps", [(1, 137), (3, 3 * 130 + 2), (2, 2 * 100)])
def test_ring_restatement_equals_brute_force(sample_interval, steps):
    """Three groups of unequal size (one of a single atom), sample counts that do not fill a whole
    number of rings, and exactly Nc samples (one time origin)."""
    rng = np.random.default_rng(sample_interval)
    n, Nc, direction = 40, 100, 1
    groups = [np.array([7]), rng.permutation(n)[:13], np.arange(20, 40)]
    ring = ho.ShcRing(sample_interval, Nc, direction, groups)
    rows = [[0, 3, 4], [6, 1, 5], [7, 8, 2]][direction]
    s_hist, v_hist = [], []
    for step in range(steps):
        w, v = rng.normal(size=(9, n)), rng.normal(size=(3, n))
        ring.process(step, w, v)
        if (step + 1) % sample_interval == 0:
            s_hist.append(w[rows])
            v_hist.append(v)
    s_hist, v_hist = np.array(s_hist), np.array(v_hist)
    for g, idx in enumerate(groups):
        k, origins = ho.shc_brute_force(s_hist[:, :, idx], v_hist[:, :, idx], Nc)
        assert origins == ring.num_time_origins == steps // sample_interval - Nc + 1
        assert np.allclose(ring.k[g], k, rtol=1e-12, atol=1e-12 * np.abs(k).max())


def test_average_k_orders_negative_then_positive_lags():
    Nc = 100
    k = np.arange(4 * Nc, dtype=float).reshape(4, Nc)
    ki, ko = ho.shc_average_k(k, Nc, 2)
    scalar = 1000.0 / ho.TIME_UNIT_CONVERSION / 2
    assert ki.shape == (2 * Nc - 1,)
    assert ki[0] == k[0, Nc - 1] * scalar and ki[Nc - 2] == k[0, 1] * scalar  # t = -(Nc-1) .. -1
    assert ki[Nc - 1] == k[2, 0] * scalar and ko[-1] == k[3, Nc - 1] * scalar  # t = 0 .. Nc-1


def test_kappa_factor_by_hand():
    """kappa = sum of the interval's heat sums * 1.573769e5 / output_interval / (V T |fe|): two rows
    of J = (1, 2, 3, 4, 5) eV A^2/ps-equivalent natural units in a 1000 A^3 box at 300 K with
    fe = (0, 3e-5, 4e-5) (|fe| = 5e-5 /A)."""
    rows = np.array([[1.0, 2.0, 3.0, 4.0, 5.0]] * 2)
    kappa = ho.hnemd_kappa(rows, 1000.0, 300.0, (0.0, 3e-5, 4e-5))
    by_hand = np.array([2.0, 4.0, 6.0, 8.0, 10.0]) * 1.573769e5 / 2 / (1000.0 * 300.0 * 5e-5)
    assert np.allclose(kappa, by_hand, rtol=1e-15)
    assert math.isclose(kappa[0], 10491.793333333333, rel_tol=1e-12)


def test_drive_restatement_removes_the_net_force():
    rng = np.random.default_rng(1)
    n = 1001
    w, f = rng.normal(size=(9, n)), rng.normal(size=(3, n))
    fe = (1e-3, -2e-3, 5e-4)
    out = ho.hnemd_drive(w, f, fe)
    assert np.abs(out.sum(axis=1)).max() < 1e-12 * np.abs(out).sum()
    Wt = np.stack([[w[0], w[3], w[4]], [w[6], w[1], w[5]], [w[7], w[8], w[2]]])  # rows x y z of W
    drive = np.einsum("abn,a->bn", Wt, np.array(fe))
    want = f + drive
    want -= want.mean(axis=1, keepdims=True)
    assert np.allclose(out, want, rtol=1e-13, atol=1e-13)

"""compute_rdf without a GPU: the brute-force oracle (oracle/rdf_oracle.c) on hand-built pairs, the
bit-symmetry the unordered counting rests on, and the device's bin rule, half-shell cell walk and fold
built for the host (tests/emu/rdf_emu.cpp) against the oracle."""
import numpy as np
import pytest

import rdf_support as R
from gpumd_b200.structures import fcc, rocksalt_pbte


def _two(h, pbc, p1, p2, types=(0, 0)):
    return dict(h=np.asarray(h, np.float64).reshape(9), pbc=np.asarray(pbc, np.int32),
                type=np.asarray(types, np.int32), pos=np.array([p1, p2], np.float64).T.copy())


BOX = np.diag([20.0, 20.0, 20.0]).reshape(9)


@pytest.mark.parametrize("num_bins", [21, 100, 500])
def test_pairs_on_the_bin_edges(num_bins):
    """d2 exactly on ((w+1) dr)^2 belongs to bin w (<=), exactly on (w dr)^2 to bin w - 1 (>), for every edge"""
    rc = 5.0
    dr = rc / num_bins
    for w in range(num_bins):
        up = ((w + 1) * dr) * ((w + 1) * dr)
        assert R.ref_bin(up, rc, num_bins) == w
        assert R.emu_bin(up, rc, num_bins) == w
        nxt = np.nextafter(up, np.inf)
        assert R.emu_bin(nxt, rc, num_bins) == R.ref_bin(nxt, rc, num_bins)
        if w > 0:
            lo = (w * dr) * (w * dr)
            assert R.ref_bin(lo, rc, num_bins) == w - 1 == R.emu_bin(lo, rc, num_bins)
    # random d2 over the whole range, and a pair placed so that its d2 is exactly an edge
    rng = np.random.default_rng(3)
    for d2 in rng.uniform(0, rc * rc * 1.1, 2000):
        assert R.emu_bin(d2, rc, num_bins) == R.ref_bin(d2, rc, num_bins)
    # pairs placed exactly on edges: atoms at 0 and x, so x12 = x exactly and d2 = fl(x * x), the edge itself
    for w in (0, 3, num_bins // 2, num_bins - 1):
        x = (w + 1) * dr  # d2 = ((w+1) dr)^2, the upper edge of bin w: bin w by `<=`
        s = _two(BOX, (1, 1, 1), (0.0, 0.0, 0.0), (x, 0.0, 0.0))
        assert (x - 0.0) * (x - 0.0) == ((w + 1) * dr) * ((w + 1) * dr)
        c = R.oracle_counts(s, rc, num_bins)
        assert c[:, 0].sum() == 2 and c[w, 0] == 2, w
        assert np.array_equal(R.ordered_from_unordered(R.emu_counts(s, rc, num_bins), 1), c)
        if w > 0:
            x = w * dr  # d2 = (w dr)^2, the lower edge of bin w: not in bin w (`>`), in bin w - 1
            s = _two(BOX, (1, 1, 1), (0.0, 0.0, 0.0), (x, 0.0, 0.0))
            c = R.oracle_counts(s, rc, num_bins)
            assert c[:, 0].sum() == 2 and c[w - 1, 0] == 2 and c[w, 0] == 0, w
            assert np.array_equal(R.ordered_from_unordered(R.emu_counts(s, rc, num_bins), 1), c)


def test_pair_beyond_the_last_bin_but_inside_rc_is_dropped():
    """rc = 5, 77 bins: dr = rc / 77 and (77 dr)^2 rounds below rc^2, so a pair in between lands in no bin"""
    rc, nb = 5.0, 77
    dr = rc / nb
    last = (nb * dr) * (nb * dr)
    assert last < rc * rc  # the rounding this case relies on
    d2 = np.nextafter(last, np.inf)
    assert d2 <= rc * rc
    assert R.ref_bin(d2, rc, nb) == -1 == R.emu_bin(d2, rc, nb)
    s = _two(BOX, (1, 1, 1), (2.0, 2.0, 2.0), (2.0, 2.0, 2.0 + 5.0))
    assert R.oracle_counts(s, rc, nb).sum() == 0  # d2 = rc^2 exactly: the last bin's edge is below it
    u = R.emu_counts(s, rc, nb)
    assert u.sum() == 0


def test_coincident_atoms_land_in_no_bin():
    s = _two(BOX, (1, 1, 1), (3.0, 4.0, 5.0), (3.0, 4.0, 5.0))
    assert R.oracle_counts(s, 5.0, 50).sum() == 0
    assert R.emu_counts(s, 5.0, 50).sum() == 0
    assert R.ref_bin(0.0, 5.0, 50) == -1 == R.emu_bin(0.0, 5.0, 50)


def test_triclinic_minimum_image():
    """two atoms near opposite faces of a sheared cell: the pair is counted at its minimum-image distance"""
    h = np.array([[15.0, 4.0, -3.0], [0.0, 14.0, 5.0], [0.0, 0.0, 16.0]])
    frac1, frac2 = np.array([0.02, 0.5, 0.5]), np.array([0.97, 0.52, 0.49])
    s = _two(h, (1, 1, 1), h @ frac1, h @ frac2)
    d = h @ (frac2 - frac1 - np.round(frac2 - frac1))
    rc, nb = 5.0, 100
    c = R.oracle_counts(s, rc, nb)
    w = int(np.linalg.norm(d) / (rc / nb))
    assert c[:, 0].sum() == 2 and c[w, 0] == 2
    assert np.array_equal(R.ordered_from_unordered(R.emu_counts(s, rc, nb), 1), c)


def test_open_direction_with_atoms_outside_the_box():
    """pbc T T F: no image along z, and atoms beyond both faces of the box still pair with each other"""
    h = np.diag([15.0, 15.0, 15.0])
    rc, nb = 5.0, 50
    # across the open z faces: 14 A apart in the box, no image, so no pair
    s = _two(h, (1, 1, 0), (1.0, 1.0, 0.5), (1.0, 1.0, 14.5))
    assert R.oracle_counts(s, rc, nb).sum() == 0 and R.emu_counts(s, rc, nb).sum() == 0
    # both below the box, and one below with one inside
    for z1, z2 in ((-4.0, -1.5), (-2.0, 1.0), (16.0, 19.5)):
        s = _two(h, (1, 1, 0), (1.0, 1.0, z1), (1.0, 14.0, z2))
        c = R.oracle_counts(s, rc, nb)
        assert c[:, 0].sum() == 2, (z1, z2)
        assert np.array_equal(R.ordered_from_unordered(R.emu_counts(s, rc, nb), 1), c)


def _systems():
    pbte = rocksalt_pbte(4, rattle=0.15, seed=5)  # 512 atoms, 26.3 A
    alloy = R.random_types(fcc(5, 3.6, rattle=0.12, seed=6), 3, seed=7)  # 500 atoms, 18 A
    return {
        "pbte_ortho": (pbte, 6.0),
        "pbte_tric": (R.triclinic(pbte), 5.0),
        "alloy_tric": (R.triclinic(alloy, (0.2, 0.1, -0.15)), 4.2),
        "pbte_slab": (R.open_slab(pbte), 6.0),
        "one_type_missing": (R.random_types(alloy, 3, seed=8, absent=(1,)), 4.5),
    }


@pytest.mark.parametrize("case", list(_systems()))
def test_ordered_counts_are_twice_the_unordered_ones(case):
    """2 u(a,a) / u(a<b) / 2 sum u give the oracle's ordered counts exactly, and no pair has a d2 that
    differs between i -> j and j -> i"""
    s, rc = _systems()[case]
    T = len(R.species(s["type"])[0])
    for nb in (21, 500):
        ordered = R.oracle_counts(s, rc, nb)
        u, asym = R.oracle_unordered(s, rc, nb)
        assert asym == 0
        assert np.array_equal(R.ordered_from_unordered(u, T), ordered)
        assert ordered[:, 0].sum() > 1000


@pytest.mark.parametrize("case", list(_systems()))
def test_host_built_walk_and_bin_rule_give_the_oracles_counts(case):
    s, rc = _systems()[case]
    for nb in (21, 500):
        u = R.emu_counts(s, rc, nb)
        assert np.array_equal(u, R.oracle_unordered(s, rc, nb)[0])


def test_normalisation_matches_a_hand_calculation():
    """one sample folded on the host (b2_body_rdf_fold): count x 1 / (N (N / V) dV) for the total and
    count x 1 / (N_a (N_b / V) dV) for (a, b), dV = r_mid^2 4 pi dr; a second sample at another volume adds
    its own factors"""
    rc, nb = 5.0, 25
    T, num_atoms, n = 2, np.array([3, 5], np.int32), 8
    rng = np.random.default_rng(1)
    u = rng.integers(0, 1000, (3, nb)).astype(np.uint64)
    V1, V2 = 1000.0, 1331.0
    dr = rc / nb
    acc = R.emu_fold(u, rc, nb, V1, n, num_atoms)
    ordered = R.ordered_from_unordered(u.astype(np.int64), T)
    for w in range(nb):
        dV = ((w + 0.5) * dr) ** 2 * 4 * np.pi * dr
        assert acc[w, 0] == pytest.approx(ordered[w, 0] * V1 / (n * n * dV), rel=1e-14)
        assert acc[w, 1] == pytest.approx(ordered[w, 1] * V1 / (3 * 3 * dV), rel=1e-14)
        assert acc[w, 2] == pytest.approx(ordered[w, 2] * V1 / (3 * 5 * dV), rel=1e-14)
        assert acc[w, 3] == pytest.approx(ordered[w, 3] * V1 / (5 * 5 * dV), rel=1e-14)
    # bit for bit: the oracle's factor times the count
    assert np.array_equal(acc, ordered * R.factors(V1, n, rc, nb, num_atoms))
    acc2 = R.emu_fold(u, rc, nb, V2, n, num_atoms, acc)
    assert np.array_equal(acc2, acc + ordered * R.factors(V2, n, rc, nb, num_atoms))
    assert R.volume(np.diag([10.0, 11.0, 12.0]).reshape(9)) == 1320.0

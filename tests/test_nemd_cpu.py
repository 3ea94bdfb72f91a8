"""The restatements of tests/nemd_oracle.py against brute-force versions (no GPU)."""
import numpy as np

import nemd_oracle as no


def test_group_sums_match_bincount():
    rng = np.random.default_rng(3)
    n = 2000
    label = rng.integers(0, 40, n)
    label[label == 7] = 8  # group 7 empty
    cols = no.per_atom_columns(rng.random(n) + 1, rng.normal(size=n), rng.normal(size=3 * n),
                               rng.normal(size=9 * n), rng.normal(size=3 * n))
    assert cols.shape == (23, n)
    sums = no.group_sums(label, 40, cols)
    for c in range(23):
        assert np.allclose(sums[c], np.bincount(label, weights=cols[c], minlength=40), rtol=1e-12, atol=1e-12)
    assert np.all(sums[:, 7] == 0)
    sizes, cont = no.contents(label)
    assert sizes.sum() == n and np.all(label[cont][:-1] <= label[cont][1:])


def test_per_atom_columns_by_hand():
    m, pe = np.array([2.0]), np.array([-1.5])
    v = np.array([1.0, 2.0, 3.0])
    W = np.arange(1.0, 10.0)  # GPUMD virial rows xx yy zz xy xz yz yx zx zy
    c = no.per_atom_columns(m, pe, np.array([4.0, 5.0, 6.0]), W, v)[:, 0]
    assert np.isclose(c[0], 2 * 14 / (3 * no.K_B)) and c[1] == -1.5 and list(c[2:5]) == [4, 5, 6]
    assert list(c[5:14]) == [1, 4, 5, 7, 2, 6, 8, 9, 3]
    assert list(c[14:17]) == [1 + 8 + 15, 7 + 4 + 18, 8 + 18 + 9]
    e = 0.5 * 2 * 14 - 1.5
    assert np.allclose(c[17:20], v * e) and np.allclose(c[20:23], 2 * v)
    assert no.select(["jk", "temperature"]) == [0, 17, 18, 19]


def test_nhc_chain_conserves_its_extended_energy():
    """A chain coupled to a kinetic energy that only it changes: the extended energy is conserved."""
    kT, dof, tau = no.K_B * 310.0, 3.0 * 500, 100.0 / 10.18
    s = no.nhc_init(kT, tau, dof)
    ek2 = dof * no.K_B * 250.0
    e0 = no.nhc_energy(s, ek2, dof, kT)
    for _ in range(200):
        f = no.nhc_chain(s, ek2, dof, kT, 0.5 / 10.18)
        ek2 *= f * f
    assert abs(no.nhc_energy(s, ek2, dof, kT) - e0) < 1e-8 * abs(e0)
    assert ek2 / (dof * no.K_B) > 250.0  # heated toward 310 K


def test_bdp_stream_matches_numpy_randomstate():
    """The generator heat_bdp's restatement draws from: init_genrand seeding (std::mt19937) and the raw
    32-bit stream against numpy's legacy RandomState, which uses the same generator and seeding.  Its
    doubles are pinned bit for bit to libstdc++'s own objects in tests/test_oracle_pins.py; the whole
    heat_bdp stream is checked against the reference gpumd by the nemd_graphene_bdp driver test."""
    mt = no.BdpOracle(12345678)
    raw = np.random.RandomState(12345678).randint(0, 2 ** 32, size=1500, dtype=np.uint64)
    assert np.array_equal(np.array([mt.raw() for _ in range(1500)], dtype=np.uint64), raw)


def test_resamplekin_stream_is_reproducible_and_unbiased():
    a, b = no.BdpOracle(12345678), no.BdpOracle(12345678)
    x = [a.resamplekin(100.0, 120.0, 300, 100.0) for _ in range(50)]
    assert x == [b.resamplekin(100.0, 120.0, 300, 100.0) for _ in range(50)]
    # tau -> 0: the new kinetic energy is a canonical sample with mean sigma
    c = no.BdpOracle(1)
    draws = np.array([c.resamplekin(100.0, 120.0, 30, 0.0) for _ in range(4000)])
    assert abs(draws.mean() - 120.0) < 4 * 120.0 * np.sqrt(2 / 30 / 4000)


def heat_lan_setup(n=500, seed=3):
    rng = np.random.default_rng(seed)
    mass = rng.uniform(1.0, 200.0, n)
    label = rng.integers(0, 5, n).astype(np.int32)  # interleaved: the group contents are not contiguous
    vel = rng.normal(size=(3, n)) * 0.01
    return mass, label, vel


def test_heat_lan_kicks_only_source_and_sink_and_accounts_the_energy():
    import curand_oracle as X
    mass, label, vel = heat_lan_setup()
    bath = no.HeatLan(mass, label, 1, 3, 300.0, 10.0, 30.0, 1804289383, 846930886)
    sizes, order = no.contents(label)
    src, snk = order[label[order] == 1], order[label[order] == 3]
    assert np.array_equal(bath.atoms[0], src) and np.array_equal(bath.atoms[1], snk)
    streams = [X.XorwowStates(1804289383, np.arange(sizes[1])), X.XorwowStates(846930886, np.arange(sizes[3]))]
    v = vel
    energy = np.zeros(2)
    for _ in range(5):
        v1 = bath.half(v)
        other = (label != 1) & (label != 3)
        assert np.array_equal(v1[:, other], v[:, other])
        for g, (idx, T) in enumerate(((src, 330.0), (snk, 270.0))):
            c2 = np.sqrt((1 - bath.c1 ** 2) * no.K_B * T)
            want = bath.c1 * v[:, idx] + c2 * np.sqrt(1.0 / mass[idx]) * streams[g].normal_double(3)
            assert np.array_equal(v1[:, idx], want)
            energy[g] += 0.5 * (mass[idx] * ((v[:, idx] ** 2).sum(0) - (want ** 2).sum(0))).sum()
        v = v1
    assert np.allclose(bath.energy, energy, rtol=1e-13, atol=0)


def test_heat_lan_without_friction_or_noise_changes_nothing():
    mass, label, vel = heat_lan_setup(seed=4)
    bath = no.HeatLan(mass, label, 0, 4, 300.0, np.inf, 10.0, 1, 2)
    assert bath.c1 == 1.0 and bath.c2 == [0.0, 0.0]
    assert np.array_equal(bath.half(vel), vel) and np.all(bath.energy == 0.0)

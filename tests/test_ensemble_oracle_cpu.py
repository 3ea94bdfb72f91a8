"""Pins on tests/ensemble_oracle.py, the float64 whole-step restatement the GPU ensemble tests trust:
it is the composition of the oracle_py pieces in the reference's order, its group rules hold, NVE on
analytic harmonic forces conserves energy to O(dt^2), and nvt_bdp's stream depends on the degrees of
freedom it is given."""
import numpy as np
import pytest

from ensemble_oracle import K_B, EnsembleStep, pressure_parameters

DT = 1.0 / 10.18051  # 1 fs in natural units


def random_state(n=257, seed=0, triclinic=False):
    rng = np.random.default_rng(seed)
    h = np.diag([20.0, 21.0, 22.0])
    if triclinic:
        h[0, 1], h[0, 2], h[1, 2] = 2.0, -1.5, 1.0
    mass = rng.uniform(10.0, 200.0, n)
    pos = h @ rng.uniform(0.02, 0.98, (3, n))
    vel = rng.normal(size=(3, n)) * np.sqrt(K_B * 300.0 / mass)
    f0, f1 = rng.normal(size=(3, n)), rng.normal(size=(3, n))
    pe, vir = rng.normal(size=n) - 3.0, rng.normal(size=(9, n)) * 0.1
    label = rng.integers(0, 4, n).astype(np.int32)
    return dict(h=h.reshape(9), mass=mass, pos=pos, vel=vel, f0=f0, f1=f1, pe=pe, vir=vir, label=label)


GROUPS = {"none": {}, "fix": dict(fixed_group=1),
          "fix_move": dict(fixed_group=1, move_group=2, move_velocity=(0.03, -0.02, 0.01))}


@pytest.mark.parametrize("groups", list(GROUPS))
@pytest.mark.parametrize("kind", ["nve", "nvt_ber", "nvt_nhc", "nvt_bdp", "npt_ber1", "npt_ber3", "npt_ber6"])
def test_step_is_the_composition_of_the_oracle_pieces(oracle, kind, groups):
    """Three consecutive steps of EnsembleStep against the same oracle_py calls written out in the
    reference's order (thermostat state carried by hand), bit for bit."""
    s = random_state(triclinic=kind == "npt_ber6")
    g = GROUPS[groups]
    label = s["label"] if g else None
    extra, num_p = {}, 0
    if kind.startswith("npt_ber"):
        num_p = int(kind[-1])
        p, c = [0.1, -0.2, 0.3, 0.05, -0.04, 0.02][:num_p], [40.0, 60.0, 2500.0, 30.0, 30.0, 30.0][:num_p]
        extra = dict(target_pressure=p, elastic_modulus=c, tau_p=200.0)
    e = EnsembleStep(kind[:7], s["mass"], DT, label=label, temperature=310.0, temperature_coupling=50.0,
                     **extra, **g)
    fg, mg = g.get("fixed_group", -1), g.get("move_group", -1)
    mv = np.asarray(g.get("move_velocity", (0.0, 0.0, 0.0)))
    lab = label if label is not None else np.zeros(len(s["mass"]), np.int32)
    n = len(s["mass"])
    n_t = n - sum(int((lab == k).sum()) for k in (fg, mg) if k >= 0)
    assert e.n_temperature == n_t
    chain = oracle.nhc_state(n, 310.0, 50.0, DT)
    bdp = oracle.BdpOracle(12345678)
    h, pos, vel = s["h"].copy(), s["pos"].copy(), s["vel"].copy()
    vol = lambda h: abs(np.linalg.det(h.reshape(3, 3)))  # noqa: E731
    for k in range(3):
        f0, f1 = (s["f0"], s["f1"]) if k % 2 == 0 else (s["f1"], s["f0"])
        got = e.step(h, pos, vel, f0, f1, s["pe"], s["vir"])
        v = vel
        if kind == "nvt_nhc":
            t = oracle.find_thermo(n_t, vol(h), s["mass"], np.zeros(n), v, np.zeros((9, n)))[0]
            v = v * oracle.nhc_chain(chain, t * 3 * n * K_B, K_B * 310.0, 3.0 * n, 0.5 * DT)
        p, v = oracle.velocity_verlet_groups(True, DT, s["mass"], pos, v, f0, lab, fg, mg, mv)
        p = oracle.apply_pbc(h, (1, 1, 1), p)
        _, v = oracle.velocity_verlet_groups(False, DT, s["mass"], p, v, f1, lab, fg, mg, mv)
        th = oracle.find_thermo(n_t, vol(h), s["mass"], s["pe"], v, s["vir"])
        if kind == "nvt_ber" or kind.startswith("npt_ber"):
            v = v * oracle.berendsen_factor(310.0, 50.0, th[0])
        elif kind == "nvt_nhc":
            v = v * oracle.nhc_chain(chain, th[0] * 3 * n * K_B, K_B * 310.0, 3.0 * n, 0.5 * DT)
        elif kind == "nvt_bdp":
            v = v * bdp.factor(th[0], n_t, 310.0, 50.0)
        hn = h
        if kind.startswith("npt_ber"):
            _, p0, pc = pressure_parameters(extra["target_pressure"], extra["elastic_modulus"], 200.0)
            hn, mu = oracle.berendsen_pressure(h, (1, 1, 1), th, p0, pc, num_p)
            p = mu.reshape(3, 3) @ p
            assert not np.array_equal(hn, h)
        for a, b in zip(got, (p, v, hn, th)):
            assert np.array_equal(a, b), (kind, groups, k)
        pos, vel, h = got[0], got[1], got[2]
        # the group rules
        if fg >= 0:
            assert np.all(vel[:, lab == fg] == 0.0)
        if mg >= 0:
            assert np.all(vel[:, lab == mg] == 0.0)


def test_group_rules_of_one_step(oracle):
    """Fixed atoms keep their position bit for bit, moving atoms translate by mv dt (one FMA) and store
    zero velocity, and the temperature counts the other atoms only."""
    s = random_state(seed=3)
    mv = (0.03, -0.02, 0.01)
    e = EnsembleStep("nve", s["mass"], DT, label=s["label"], fixed_group=0, move_group=3, move_velocity=mv)
    p1, v1 = e.compute1(s["h"], s["pos"], s["vel"], s["f0"])
    fixed, moving = s["label"] == 0, s["label"] == 3
    assert np.array_equal(p1[:, fixed], s["pos"][:, fixed])
    assert np.all(v1[:, fixed | moving] == 0.0)
    for d in range(3):
        assert np.allclose(p1[d, moving], s["pos"][d, moving] + mv[d] * DT, rtol=1e-15, atol=0)
    _, _, _, th = e.compute2(s["h"], p1, v1, s["f1"], s["pe"], s["vir"])
    _, v2 = oracle.velocity_verlet_groups(False, DT, s["mass"], p1, v1, s["f1"], s["label"], 0, 3, mv)
    ke2 = (s["mass"] * (v2 ** 2).sum(axis=0)).sum()
    n_t = int((~(fixed | moving)).sum())
    assert th[0] == pytest.approx(ke2 / (3 * n_t * K_B), rel=1e-13)


def test_bdp_rejects_no_integrated_atoms():
    s = random_state(n=8, seed=1)
    label = np.zeros(8, np.int32)
    label[4:] = 1
    with pytest.raises(ValueError):
        EnsembleStep("nvt_bdp", s["mass"], DT, label=label, fixed_group=0, move_group=1, move_velocity=(0, 0, 0))


def test_npt_ber_coupling_of_a_stiff_direction_is_zero():
    num_p, p0, pc = pressure_parameters([1.0, 2.0, 3.0], [50.0, 2000.0, 2000.5], 100.0)
    assert num_p == 3 and pc[2] == 0.0 and pc[1] > 0.0
    assert p0[0] == 1.0 / 1.602177e+2


@pytest.mark.parametrize("kind", ["nve", "nvt_ber", "nvt_nhc", "nvt_bdp", "npt_ber"])
def test_open_direction_and_stiff_direction_keep_their_box(kind):
    """npt_ber with 3 components leaves an open direction and a direction with modulus > 2000 GPa
    bit for bit alone; the other ensembles never touch the box."""
    s = random_state(seed=5)
    extra = dict(target_pressure=[0.1, -0.1, 0.2], elastic_modulus=[40.0, 3000.0, 40.0], tau_p=100.0) \
        if kind == "npt_ber" else {}
    e = EnsembleStep(kind, s["mass"], DT, pbc=(1, 1, 0), **extra)
    _, _, h, _ = e.step(s["h"], s["pos"], s["vel"], s["f0"], s["f1"], s["pe"], s["vir"])
    assert np.array_equal(h[[1, 2, 3, 4, 5, 6, 7, 8]], s["h"][[1, 2, 3, 4, 5, 6, 7, 8]])
    assert (h[0] != s["h"][0]) == (kind == "npt_ber")


@pytest.mark.parametrize("pbc", [(1, 1, 1), (1, 1, 0)])
def test_deform_overrides_the_pressure_and_the_open_direction(oracle, pbc):
    """`deform` in the 3-component barostat: the deformed directions grow by their rate per step, open or
    not; the others keep the pressure rule (periodic) or their length (open)."""
    h = np.diag([40.0, 41.0, 42.0]).reshape(9)
    thermo = np.array([300.0, -1.0, 0.010, 0.012, 0.008, 0.0, 0.0, 0.0])
    p0, pc = np.array([0.003, 0.002, 0.001]), np.array([0.5, 0.4, 0.3])
    plain, mu0 = oracle.berendsen_pressure(h, pbc, thermo, p0, pc, 3)
    hn, mu = oracle.berendsen_pressure(h, pbc, thermo, p0, pc, 3, deform=(1, 0, 1), deform_rate=(1e-3, 5.0, -2e-3))
    assert hn[0] == pytest.approx(40.001, rel=1e-15) and hn[8] == pytest.approx(41.998, rel=1e-15)
    assert mu[0] == hn[0] / 40.0 and mu[8] == hn[8] / 42.0
    assert hn[4] == plain[4] and mu[4] == mu0[4]  # y is not deformed: its rate is not read
    assert hn[4] != 41.0
    assert np.array_equal(hn[[1, 2, 3, 5, 6, 7]], np.zeros(6))
    assert np.array_equal(oracle.berendsen_pressure(h, pbc, thermo, p0, pc, 3, deform=(0, 0, 0),
                                                    deform_rate=(1.0, 1.0, 1.0))[0], plain)


def harmonic_run(dt, steps, k_spring=2.0, n=64, seed=7):
    """NVE on independent 3D oscillators f = -k (r - r0); returns the total energy after every step."""
    rng = np.random.default_rng(seed)
    mass = rng.uniform(20.0, 60.0, n)
    r0 = rng.uniform(20.0, 80.0, (3, n))
    h = np.diag([100.0, 100.0, 100.0]).reshape(9)
    e = EnsembleStep("nve", mass, dt, pbc=(0, 0, 0))
    pos = r0 + rng.normal(size=(3, n)) * 0.1
    vel = rng.normal(size=(3, n)) * np.sqrt(K_B * 300.0 / mass)
    force = -k_spring * (pos - r0)
    out = []
    for _ in range(steps):
        p1, v1 = e.compute1(h, pos, vel, force)
        f1 = -k_spring * (p1 - r0)
        pe = 0.5 * k_spring * ((p1 - r0) ** 2).sum(axis=0)
        pos, vel, h, th = e.compute2(h, p1, v1, f1, pe, np.zeros((9, n)))
        force = f1
        out.append(1.5 * n * K_B * th[0] + th[1])
    return np.array(out)


def test_nve_conserves_harmonic_energy_to_second_order():
    """Velocity-Verlet's energy error on a harmonic system is O(dt^2) and does not drift: halving dt
    cuts the fluctuation about fourfold, over the same simulated time."""
    t_total = 40.0  # natural time units, several periods (omega ~ sqrt(2 / 40) ~ 0.22)
    dt = 0.1
    e1 = harmonic_run(dt, int(t_total / dt))
    e2 = harmonic_run(dt / 2, int(t_total / (dt / 2)))
    w1, w2 = np.abs(e1 - e1[0]).max(), np.abs(e2 - e2[0]).max()
    assert w1 < 1e-3 * abs(e1[0])
    assert 3.5 < w1 / w2 < 4.5, (w1, w2)
    assert abs(e2[-1] - e2[0]) <= w2  # no drift beyond the fluctuation


def counted_factors(oracle, n_integrated, steps=3, t_now=290.0):
    """The first `steps` BDP factors for ndeg = 3 n_integrated and how many 32-bit numbers the generator had drawn after
    each of them."""
    o = oracle.BdpOracle(12345678)
    raw, count = o.raw, [0]

    def counting():
        count[0] += 1
        return raw()
    o.raw = counting
    out = []
    for _ in range(steps):
        out.append((o.factor(t_now, n_integrated, 300.0, 100.0), count[0]))
    return out


@pytest.mark.parametrize("n_atoms,k", [(1728, 1), (1728, 3), (1728, 200), (3, 1), (2, 1)])
def test_bdp_stream_depends_on_the_degrees_of_freedom(oracle, n_atoms, k):
    """resamplekin draws one Gaussian and sumnoises(ndeg - 1): a Gamma variate of order (ndeg - 1) // 2
    plus, for even ndeg, a second Gaussian (the cached partner of the first).  Taking k atoms out of
    ndeg changes the factor from the first step; an odd k flips the parity, so the generator falls out
    of step by the second; and below 12 degrees of freedom the Gamma variate's own draw count changes."""
    a = counted_factors(oracle, n_atoms)
    b = counted_factors(oracle, n_atoms - k)
    assert a[0][0] != b[0][0]
    if k % 2:
        assert [c for _, c in a[1:]] != [c for _, c in b[1:]]
    if 3 * n_atoms <= 12:
        assert a[0][1] != b[0][1]


# ---------------------------------------------------------------- nvt_lan / nvt_bao

def zero_momentum_state(n=256, seed=11):
    """Atom i + n/2 is atom i, in the same group, with the velocity and forces negated: the momentum of each half is the exact
    negative of the other's after any step, and numpy's pairwise sum splits 256 atoms into these two
    halves, so the total momentum is exactly zero."""
    s = random_state(n=n, seed=seed)
    half = n // 2
    s["mass"] = np.concatenate([s["mass"][:half]] * 2)
    s["label"] = np.concatenate([s["label"][:half]] * 2)
    for k in ("vel", "f0", "f1"):
        s[k] = np.concatenate([s[k][:, :half], -s[k][:, :half]], axis=1)
    return s


@pytest.mark.parametrize("groups", ["none", "fix"])
def test_langevin_without_friction_or_noise_is_nve(groups):
    """c1 = 1 (infinite coupling time) and c2 = 0 leave a kick v <- c1 v + c2 / sqrt(m) xi and the
    momentum removal with nothing to do on a state of zero total momentum: nvt_lan is then nve bit for
    bit, and nvt_bao (B A A | force | B) is nve up to the rounding of two half drifts instead of one."""
    s = zero_momentum_state()
    g = GROUPS[groups]
    label = s["label"] if g else None
    nve = EnsembleStep("nve", s["mass"], DT, label=label, **g)
    want = nve.step(s["h"], s["pos"], s["vel"], s["f0"], s["f1"], s["pe"], s["vir"])
    for kind in ("nvt_lan", "nvt_bao"):
        e = EnsembleStep(kind, s["mass"], DT, label=label, temperature=300.0, temperature_coupling=np.inf, **g)
        assert e.c1 == 1.0
        got = e.step(s["h"], s["pos"], s["vel"], s["f0"], s["f1"], s["pe"], s["vir"])
        for a, b, what in zip(got, want, ("pos", "vel", "h", "thermo")):
            if kind == "nvt_lan" or what == "h":
                assert np.array_equal(a, b), (kind, what)
            else:
                assert np.allclose(a, b, rtol=1e-14, atol=1e-14 * np.abs(b).max()), (kind, what)


@pytest.mark.parametrize("kind", ["nvt_lan", "nvt_bao"])
def test_langevin_kick_removes_the_momentum_and_draws_per_atom(kind):
    """After every kick the total momentum is zero to rounding; the noise of atom i is normal number
    3c..3c+2 of curand_init(seed, i, 0), x then y then z, on every atom whatever its group."""
    import curand_oracle as X
    s = random_state(seed=9)
    e = EnsembleStep(kind, s["mass"], DT, label=s["label"], fixed_group=1, temperature=300.0,
                     temperature_coupling=20.0)
    v = s["vel"]
    stream = X.XorwowStates(1804289383, np.arange(len(s["mass"])))
    c2 = np.sqrt((1 - e.c1 ** 2) * K_B * 300.0)
    for _ in range(4):
        xi = stream.normal_double(3)
        raw = e.c1 * v + c2 * np.sqrt(1.0 / s["mass"]) * xi
        v = e.langevin(v)
        p = (v * s["mass"]).sum(axis=1)
        assert np.abs(p).max() < 1e-13 * (np.abs(v) * s["mass"]).sum()
        shift = raw - v  # one momentum shift for all atoms
        assert np.allclose(shift, shift[:, :1], rtol=0, atol=1e-15)


@pytest.mark.parametrize("kind", ["nvt_lan", "nvt_bao"])
def test_langevin_fixed_atom_rules(kind):
    """Fixed atoms keep their position bit for bit.  nvt_bao's B step leaves their velocity at zero at
    the end of each step; nvt_lan's last kick draws noise for them too (the reference kicks every atom)."""
    s = random_state(seed=4)
    e = EnsembleStep(kind, s["mass"], DT, label=s["label"], fixed_group=2, temperature=300.0,
                     temperature_coupling=30.0)
    fixed = s["label"] == 2
    h, pos, vel = s["h"], s["pos"], s["vel"]
    for k in range(3):
        p1, v1 = e.compute1(h, pos, vel, s["f0"])
        assert np.array_equal(p1[:, fixed], pos[:, fixed]), k
        pos, vel, h, th = e.compute2(h, p1, v1, s["f1"], s["pe"], s["vir"])
        assert np.array_equal(pos[:, fixed], p1[:, fixed])
        if kind == "nvt_bao":
            assert np.all(vel[:, fixed] == 0.0)
        else:
            assert np.all(vel[:, fixed] != 0.0)

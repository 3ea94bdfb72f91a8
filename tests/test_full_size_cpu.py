"""The tiled oracle (tests/fullsize.py) against the whole-system oracle, on systems small enough for both.

Every system is rattled after wrapping, so that atoms stick out of [0, L), and the tiles start at an offset
so that they cross the periodic faces.  The tiles keep the periodic box and the atoms' own coordinates, so
every displacement and every neighbour order is the whole system's: the outputs and the NEP neighbour lists
are bit-identical, in FP32 and FP64 (which implies the 1e-10 / conftest.TOL agreement the GPU tests rely
on).  A halo of only rc for NEP (its forces reach 2 rc) must fail the same comparison: the pin can fail."""
import numpy as np
import pytest

import cases_classical as cc
import fullsize
from conftest import GOLDEN, TOL, assert_close
from gpumd_b200.structures import diamond, fcc, nep_type_order, rocksalt_pbte
from test_kernel_bodies_cpu import check_fv

CUFENI = GOLDEN / cc.EAM_FILES["cufeni"]


def _stick_out(s, seed, sigma=0.05):
    """A second rattle after the wrap: some atoms then lie below 0 or at or above L."""
    s = dict(s)
    s["pos"] = s["pos"] + np.random.default_rng(seed).normal(0.0, sigma, s["pos"].shape)
    L = np.diag(s["h"].reshape(3, 3))
    out = ((s["pos"] < 0) | (s["pos"] >= L[:, None])).any(axis=0)
    assert out.sum() > 0
    return s


def _unep(reps, seed):
    s = fcc(reps, 3.9, rattle=0.05, seed=seed, num_types=16, symbols=nep_type_order(GOLDEN / "nep_UNEP_v1.txt"))
    return s


# name -> (potential factory, structure factory, tiles per direction, tile offset in A)
SYSTEMS = {
    "pbte_20": (lambda p: fullsize.nep(GOLDEN / "nep_PbTe.txt", p), lambda: rocksalt_pbte(20, rattle=0.03, seed=3),
                (3, 2, 2), (11.3, 27.9, 5.1)),
    "unep_13": (lambda p: fullsize.nep(GOLDEN / "nep_UNEP_v1.txt", p), lambda: _unep(13, 5), (2, 2, 2),
                (7.7, 19.1, 3.3)),
    "lj_12": (lambda p: fullsize.lj(cc.LJ1), lambda: fcc(12, 5.30, rattle=0.05, seed=4), (2, 2, 2), (9.4, 30.2, 1.7)),
    "si_10": (lambda p: fullsize.tersoff(cc.SI), lambda: diamond(10, a=5.431, rattle=0.05, seed=6), (3, 3, 3),
              (4.1, 13.3, 17.0)),
    "cufeni_12": (lambda p: fullsize.eam(CUFENI),
                  lambda: fcc(12, 3.615, rattle=0.05, seed=8, num_types=3, symbols=["Cu", "Fe", "Ni"]), (2, 2, 2),
                  (3.2, 10.9, 20.0)),
}


def _whole(pot, s, lists=False):
    """The whole-system oracle, the same potentials as the tiles."""
    from oracle import oracle_py
    if pot["kind"] == "nep":
        return oracle_py.NepOracle(pot["path"]).compute(s["type"], s["h"], s["pbc"], s["pos"],
                                                          precision=pot["precision"], lists=lists)
    if pot["kind"] == "lj":
        return oracle_py.lj_compute(pot["para"], s["type"], s["h"], s["pbc"], s["pos"])
    if pot["kind"] == "tersoff":
        return oracle_py.tersoff_compute(pot["nt"], pot["para"], s["type"], s["h"], s["pbc"], s["pos"])
    return oracle_py.eam_compute(pot["model"], pot["nt"], pot["para"], s["type"], s["h"], s["pbc"], s["pos"])


def check_fp64(a, b, rtol=1e-10):
    for k in ("pe", "force", "virial"):
        assert_close(a[k], b[k], rtol=rtol, atol=rtol * np.abs(b[k]).max(), what=k)


def check_fp32(a, b):
    assert_close(a["pe"], b["pe"], what="pe", **TOL["energy"])
    check_fv(a, b)


def check_same(a, b):
    """Bit-identical outputs; on a difference, first the tolerance checks, which say by how much."""
    for k in ("pe", "force", "virial"):
        if not np.array_equal(a[k], b[k]):
            check_fp64(a, b, rtol=1e-10)
            check_fp32(a, b)
            raise AssertionError(f"{k}: within the tolerances but not bit-identical, max |diff| = "
                                 f"{np.abs(a[k] - b[k]).max():.3e}")


@pytest.fixture(scope="module", autouse=True)
def _pool():
    yield
    fullsize.shutdown()


# NEP in both precisions; the LJ and EAM oracles compute in FP32 and the Tersoff oracle in FP64 only
PRECISIONS = [(name, p) for name in SYSTEMS for p in ((32, 64) if name in ("pbte_20", "unep_13") else
                                                      (64,) if name == "si_10" else (32,))]


@pytest.mark.parametrize("name,precision", PRECISIONS)
def test_tiles_match_the_whole_system(oracle, name, precision):
    make_pot, make, tiles, offset = SYSTEMS[name]
    pot = make_pot(precision)
    s = _stick_out(make(), seed=len(name) + precision)
    lists = pot["kind"] == "nep" and precision == 32
    whole = _whole(pot, s, lists=lists)
    tiled = fullsize.evaluate(pot, s["type"], s["h"], s["pbc"], s["pos"], lists=lists, tiles=tiles,
                              offset=offset)
    assert tiled["tiles"] == list(tiles)
    check_same(tiled, whole)
    if lists:
        for which in ("radial", "angular"):
            fullsize.assert_same_lists(tiled[f"NN_{which}"], tiled[f"NL_{which}"], whole[f"NN_{which}"],
                                       whole[f"NL_{which}"], s["h"], s["pos"], what=which)


def test_default_tiling_matches_the_whole_system(oracle):
    """The tiling the GPU tests use (tile_counts, no offset) on PbTe FP64."""
    pot = fullsize.nep(GOLDEN / "nep_PbTe.txt", 64)
    s = _stick_out(rocksalt_pbte(20, rattle=0.03, seed=9), seed=9)
    tiled = fullsize.evaluate(pot, s["type"], s["h"], s["pbc"], s["pos"])
    assert np.prod(tiled["tiles"]) > 1
    check_same(tiled, _whole(pot, s))


def test_a_halo_of_rc_fails_the_pin(oracle):
    """NEP forces depend on atoms up to 2 rc away (through the neighbours' descriptors): with a halo of rc
    plus the margin, the atoms near the tile faces get wrong forces, and the FP64 pin fails by far."""
    make_pot, make, tiles, offset = SYSTEMS["pbte_20"]
    pot = make_pot(64)
    s = _stick_out(make(), seed=100)
    whole = _whole(pot, s)
    short = fullsize.evaluate(pot, s["type"], s["h"], s["pbc"], s["pos"], halo=pot["rc"] + fullsize.MARGIN,
                              tiles=tiles, offset=offset)
    with pytest.raises(AssertionError):
        check_fp64(short, whole)
    err = np.abs(short["force"] - whole["force"]).max()
    assert err > 1e-3 * np.abs(whole["force"]).max(), err
    # and the energies alone, which only reach rc, are still right
    assert_close(short["pe"], whole["pe"], rtol=1e-10, atol=1e-10 * np.abs(whole["pe"]).max(), what="pe")


def test_tiles_cover_every_atom_once():
    """The tiling itself: every atom is owned once, and a sub-system holds exactly the atoms with an image
    within the halo of its tile, in ascending global id."""
    s = _stick_out(rocksalt_pbte(6, rattle=0.03, seed=2), seed=2)
    h, pos = s["h"], s["pos"]
    L = np.diag(h.reshape(3, 3))
    n = pos.shape[1]
    owned = np.zeros(n, np.int64)
    halo, tiles, off = 9.0, (2, 3, 1), np.array([5.0, 1.0, 30.0])
    w = L / tiles
    for own, gid, where in fullsize.subsystems(h, pos, halo, tiles, offset=off):
        owned[own] += 1
        assert np.all(np.diff(gid) > 0) and np.array_equal(gid[where], own)
        # the tile's box from its owned atoms' wrapped coordinates; an atom belongs to the sub-system iff its
        # minimum-image distance to that box is below the halo along every direction
        u = off[:, None] + np.mod(pos[:, own] - off[:, None], L[:, None])
        lo = off + np.floor((u.min(axis=1) - off) / w) * w
        centre = lo + w / 2
        d = pos - centre[:, None]
        d -= np.round(d / L[:, None]) * L[:, None]
        inside = np.all(np.abs(d) < (w / 2 + halo)[:, None], axis=0)
        edge = np.any(np.abs(np.abs(d) - (w / 2 + halo)[:, None]) < 1e-9, axis=0)
        assert np.array_equal(np.isin(np.arange(n), gid) | edge, inside | edge)
    assert np.all(owned == 1)

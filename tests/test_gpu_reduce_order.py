"""The summation order of the deterministic grid reductions (gpumd_b200/csrc/b2_reduce.cuh), pinned bit for
bit against a numpy restatement.  The inputs span 24 decades with random signs, so another order of the same
terms gives other bits.  Each case is a sum whose per-atom terms are the raw inputs, at sizes below one
block, between, and above the block cap (the grid-stride loops wrap)."""
import numpy as np
import pytest

BLK = 256
CHUNK = 4 * BLK  # entries per segment of the group sums (b2_nemd.cu)


@pytest.fixture(scope="module")
def eng():
    import torch
    from gpumd_b200 import build, engine
    build.build_lib()
    assert torch.cuda.is_available()
    return engine


def wide(rng, shape):
    return rng.choice([-1.0, 1.0], shape) * 10.0 ** rng.uniform(-12.0, 12.0, shape)


def bits(x):
    return np.asarray(x, np.float64).view(np.int64)


def tree(v):
    """the shuffle-down tree over the last axis (32 lanes): what lane 0 ends with"""
    v = v.copy()
    for o in (16, 8, 4, 2, 1):
        v[..., :o] = v[..., :o] + v[..., o:2 * o]
    return v[..., 0]


def thread_sums(x, blocks):
    """grid-stride accumulation from 0.0: thread j adds x[j], x[j + blocks * BLK], ... in order"""
    span = blocks * BLK
    s = np.zeros(span)
    for row in np.concatenate([x, np.zeros(-len(x) % span)]).reshape(-1, span):
        s = s + row
    return s


def block_totals(s):
    """per-thread values -> one total per block: warp trees, then the warps in order from 0.0"""
    w = tree(s.reshape(-1, BLK // 32, 32))
    acc = np.zeros(w.shape[0])
    for k in range(BLK // 32):
        acc = acc + w[:, k]
    return acc


def warp_ordered(p):
    """one warp: lane l adds p[l], p[l + 32], ... from 0.0, then the tree"""
    acc = np.zeros(32)
    for row in np.concatenate([p, np.zeros(-len(p) % 32)]).reshape(-1, 32):
        acc = acc + row
    return tree(acc)


def grid_sum(x, cap):
    blocks = min(max(1, -(-len(x) // BLK)), cap)
    return warp_ordered(block_totals(thread_sums(x, blocks)))


def test_inputs_tell_summation_orders_apart():
    """no GPU needed: on these inputs a serial sum, or the same order on another grid, gives other bits"""
    x = wide(np.random.default_rng(0), 50_000)
    serial = 0.0
    for v in x:
        serial += v
    assert bits(grid_sum(x, 1056)) != bits(serial) and bits(grid_sum(x, 1056)) != bits(grid_sum(x, 100))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [100, 50_000, 400_000])  # cap: 1056 blocks = 270 336 atoms
def test_find_thermo_potential_sum(eng, n):
    import torch
    rng = np.random.default_rng(n)
    pe = wide(rng, n)
    atom = eng.Atom(np.zeros(n, np.int32), rng.uniform(0.0, 10.0, (3, n)), np.ones(n))
    atom.potential_per_atom.copy_(torch.as_tensor(pe))
    thermo = torch.zeros(8, dtype=torch.float64, device="cuda")
    eng.Ensemble_NVE(n).find_thermo(1000.0, atom, thermo)
    assert bits(thermo[1].item()) == bits(grid_sum(pe, 1056))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [7, 15, 20])  # n = 2^k; cap: 264 blocks = 67 584 atoms
def test_hnemd_drive_force_sum(eng, k):
    """With fe = 0 the drive leaves f as it is and subtracts ftot / n; an atom with f = 0 then holds
    -ftot * 2^-k, exactly."""
    import torch
    n = 1 << k
    rng = np.random.default_rng(k)
    f = wide(rng, (3, n))
    f[:, 0] = 0.0
    d_f = torch.as_tensor(f.reshape(-1), device="cuda")
    eng.hnemd_drive(n, (0.0, 0.0, 0.0), torch.as_tensor(rng.normal(size=9 * n), device="cuda"), d_f)
    ftot = -d_f.cpu().numpy().reshape(3, n)[:, 0] * n
    assert np.array_equal(bits(ftot), bits([grid_sum(f[d], 264) for d in range(3)]))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [100, 50_000, 400_000])  # cap: 1024 blocks = 262 144 atoms
def test_sd_trial_energy_sum(eng, n):
    import torch
    rng = np.random.default_rng(n + 1)
    atom = eng.Atom(np.zeros(n, np.int32), rng.uniform(0.0, 20.0, (3, n)), np.ones(n))
    atom.force_per_atom.copy_(torch.as_tensor(rng.normal(size=3 * n)))
    mz = eng.Minimizer("sd", n, 1e-30, 10)
    mz.sd_begin(atom)
    ut = wide(rng, n)
    mz.trial_potential.copy_(torch.as_tensor(ut))
    rec = mz.sd_step(atom)
    assert bits(rec[eng.MIN_UTRIAL]) == bits(grid_sum(ut, 1024))


@pytest.mark.gpu
def test_group_compute_potential_sums(eng):
    """Groups below one block, over a few segments, and over more than 32 segments (the warp's lanes
    wrap); a segment is a group's overlap with a chunk of CHUNK entries of the group contents."""
    import torch
    sizes = [100, 5000, 40_000, 1, 300]
    rng = np.random.default_rng(5)
    label = rng.permutation(np.repeat(np.arange(len(sizes)), sizes)).astype(np.int32)
    n = label.shape[0]
    pe = wide(rng, n)
    atom = eng.Atom(np.zeros(n, np.int32), rng.uniform(0.0, 10.0, (3, n)), np.ones(n))
    atom.potential_per_atom.copy_(torch.as_tensor(pe))
    out = eng.Compute(label, 1, 1, ["potential"]).process(0, atom)
    contents = np.argsort(label, kind="stable")
    want, pos = [], 0
    for size in sizes:
        partial, end = [], pos + size
        while pos < end:
            stop = min(end, (pos // CHUNK + 1) * CHUNK)
            partial.append(block_totals(thread_sums(pe[contents[pos:stop]], 1))[0])
            pos = stop
        want.append(0.0 + warp_ordered(np.array(partial)))
    assert np.array_equal(bits(out[0]), bits(want))

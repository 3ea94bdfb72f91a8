"""The ordering rule of the NEP warp schedule (b2_neighbor.cuh: B2NeighborView::seg_order), without a GPU.

A segment is 32 consecutive cell-sorted atoms.  The rule: key every segment by the cell (cx, cy, cz) of its
first atom; order by brick (cz / bz, cx / bx, cy / by), inside a brick by (cz % bz, cy % by, cx), ties by
segment number.  `expected_order` states that rule as a sort in numpy; the kernels build the same order from
`cell_start` alone (b2_brick_segments), and their bodies are compiled for the host here and compared with it
on random cell occupancies, including empty cells, grids that the bricks do not divide, and a last segment
that is not full."""
import ctypes as C
import subprocess

import numpy as np
import pytest

from conftest import ROOT

SHIM = r"""
#include "b2_neighbor.cuh"
extern "C" int sched_host(int n, const int* nb, const int* cell_start, int* dims, int* seg_order, int* brick_start)
{
  B2Grid g;
  for (int d = 0; d < 3; ++d) {
    g.nb[d] = nb[d];
    g.scale[d] = nb[d];
  }
  g.ncell = nb[0] * nb[1] * nb[2];
  const B2Bricks br = b2_make_bricks(g, n);
  dims[0] = br.bx;
  dims[1] = br.by;
  dims[2] = br.bz;
  B2NeighborView v{};
  v.n = n;
  v.cell_start = const_cast<int*>(cell_start);
  v.seg_order = seg_order;
  v.brick_start = brick_start;
  int run = 0;
  for (int b = 0; b < br.count; ++b) { // k_brick_scan: exclusive scan of the brick counts
    brick_start[b] = run;
    run += b2_body_brick_count(b, v, g, br);
  }
  for (int b = 0; b < br.count; ++b) // k_seg_order
    b2_body_seg_order(b, v, g, br);
  return run;
}
"""


def expected_order(n, nb, brick, cell_start):
    """The schedule as the rule states it: a sort of the segment numbers by their key."""
    nseg = (n + 31) // 32
    seg = np.arange(nseg)
    cell = np.searchsorted(np.asarray(cell_start), 32 * seg, side="right") - 1  # cell of the first atom
    cx, cy, cz = cell % nb[0], cell // nb[0] % nb[1], cell // (nb[0] * nb[1])
    bx, by, bz = brick
    return np.lexsort((seg, cx, cy % by, cz % bz, cy // by, cx // bx, cz // bz))  # last key is the primary


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    d = tmp_path_factory.mktemp("sched")
    (d / "shim.cpp").write_text(SHIM)
    lib = d / "libsched.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas",
                    "-I", str(ROOT / "gpumd_b200" / "csrc"), "-o", str(lib), str(d / "shim.cpp")], check=True)
    L = C.CDLL(str(lib))
    ip = C.POINTER(C.c_int)
    L.sched_host.argtypes = [C.c_int, ip, ip, ip, ip, ip]
    L.sched_host.restype = C.c_int

    def run(n, nb, cell_start):
        nb_a = np.asarray(nb, np.int32)
        cs = np.ascontiguousarray(cell_start, np.int32)
        dims = np.zeros(3, np.int32)
        order = np.full((n + 31) // 32, -1, np.int32)
        start = np.zeros(int(np.prod(nb)) + 1, np.int32)
        p = lambda a: a.ctypes.data_as(ip)  # noqa: E731
        total = L.sched_host(n, p(nb_a), p(cs), p(dims), p(order), p(start))
        return total, [int(x) for x in dims], order

    return run


# (cells per direction, mean atoms per cell, fraction of empty cells)
CASES = {
    "cube_dense": ((10, 10, 10), 2.6, 0.0),
    "odd_grid": ((7, 5, 9), 2.6, 0.1),           # bricks of 2 x 2 rows do not divide 5 and 9 rows
    "sparse": ((12, 6, 6), 0.4, 0.7),            # many empty cells, segments span several rows
    "one_cell_rows": ((1, 8, 8), 40.0, 0.0),     # a row is one cell holding more than a segment
    "flat": ((16, 16, 1), 3.0, 0.2),             # a single layer of cells (open direction, thin box)
    "tiny": ((5, 5, 5), 0.2, 0.5),               # fewer atoms than one segment per brick
}


@pytest.mark.parametrize("case", list(CASES))
def test_host_compiled_bodies_follow_the_rule(shim, case):
    nb, mean, empty = CASES[case]
    rng = np.random.default_rng(sum(map(ord, case)))
    for _ in range(5):
        count = rng.poisson(mean, size=int(np.prod(nb)))
        count[rng.random(count.shape) < empty] = 0
        if count.sum() == 0:
            count[rng.integers(count.size)] = 1
        cell_start = np.r_[0, np.cumsum(count)]
        n = int(cell_start[-1])
        total, brick, order = shim(n, nb, cell_start)
        nseg = (n + 31) // 32
        assert total == nseg
        assert np.array_equal(np.sort(order), np.arange(nseg)), "not a permutation of the segments"
        assert brick[1] == brick[2] == 2 and 1 <= brick[0] <= nb[0]
        assert np.array_equal(order, expected_order(n, nb, brick, cell_start))


def test_brick_width_is_the_cells_one_segment_spans(shim):
    """2.6 atoms per cell (PbTe at 4.5 A cells): 32 atoms span 12 cells; never wider than a row."""
    nb = (72, 4, 4)
    count = np.full(int(np.prod(nb)), 0)
    count[::5] = 13  # 2.6 per cell
    cell_start = np.r_[0, np.cumsum(count)]
    assert shim(int(cell_start[-1]), nb, cell_start)[1][0] == 12
    nb = (6, 4, 4)
    cell_start = np.arange(int(np.prod(nb)) + 1)  # one atom per cell: 32 cells per segment, rows of 6
    assert shim(int(cell_start[-1]), nb, cell_start)[1][0] == 6

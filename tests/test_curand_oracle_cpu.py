"""The XORWOW restatement of tests/curand_oracle.py against cuRAND itself: curand_kernel.h compiled for the
host (QUALIFIERS redefined to __host__ __device__) draws the same numbers bit for bit, and the jump
matrices the restatement computes by squaring equal the toolkit's precalculated table.  Also the glibc
rand() values the b200md driver seeds its Langevin generators from."""
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

import curand_oracle as X

SEEDS = [0, 1804289383, 846930886, 2 ** 32 + 5, 2 ** 63 + 12345]
SUBSEQUENCES = [0, 1, 255, 256, 257, 4095, 4096, 100_002, 2 ** 20 + 3]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return exe if Path(exe).exists() else None


def _include_dir():
    exe = _nvcc()
    return Path(exe).resolve().parent.parent / "include" if exe else None


needs_nvcc = pytest.mark.skipif(_nvcc() is None, reason="nvcc (and cuRAND's headers) not installed")

HOST_CURAND = r"""
#define QUALIFIERS static __forceinline__ __host__ __device__
#include <curand_kernel.h>
#include <cstdio>
#include <cstring>
// stdin: lines "seed subsequence offset draws calls kind" (kind 0: curand_normal_double, 1: curand);
// stdout: per line, calls x draws values as hexadecimal bit patterns
int main()
{
  unsigned long long seed, sub, off;
  int draws, calls, kind;
  while (scanf("%llu %llu %llu %d %d %d", &seed, &sub, &off, &draws, &calls, &kind) == 6) {
    curandState s;
    curand_init(seed, sub, off, &s);
    for (int c = 0; c < calls; ++c) {
      for (int k = 0; k < draws; ++k) {
        if (kind == 0) {
          double x = curand_normal_double(&s);
          unsigned long long b;
          memcpy(&b, &x, 8);
          printf("%016llx ", b);
        } else {
          printf("%08x ", curand(&s));
        }
      }
    }
    printf("\n");
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def host_curand(tmp_path_factory):
    d = tmp_path_factory.mktemp("curand")
    (d / "host_curand.cu").write_text(HOST_CURAND)
    exe = d / "host_curand"
    r = subprocess.run([_nvcc(), "-O2", "-x", "cu", str(d / "host_curand.cu"), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr

    def run(queries):
        inp = "".join(f"{s} {q} {o} {k} {c} {kind}\n" for s, q, o, k, c, kind in queries)
        out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout
        return [[int(t, 16) for t in line.split()] for line in out.splitlines()]
    return run


def as_bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


@needs_nvcc
@pytest.mark.parametrize("seed", SEEDS)
def test_normals_match_host_curand_bit_for_bit(host_curand, seed):
    """Every subsequence, 1 to 9 normals from a fresh state (odd counts leave the cached value)."""
    queries = [(seed, q, 0, k, 1, 0) for q in SUBSEQUENCES for k in range(1, 10)]
    want = host_curand(queries)
    st = X.XorwowStates(seed, SUBSEQUENCES)
    got = st.normal_double(9)  # [9, len(SUBSEQUENCES)]: the first k of 9 draws are the k-draw answer
    for (s, q, _, k, _, _), w in zip(queries, want):
        j = SUBSEQUENCES.index(q)
        assert as_bits(got[:k, j]).tolist() == w, (seed, q, k)


@needs_nvcc
@pytest.mark.parametrize("seed", SEEDS)
def test_three_draw_calls_match_host_curand(host_curand, seed):
    """What the Langevin kernels do: three normals per atom per call, seven calls on one state, so
    the cached second value of a pair crosses from one call into the next every other call."""
    want = host_curand([(seed, q, 0, 3, 7, 0) for q in SUBSEQUENCES])
    st = X.XorwowStates(seed, SUBSEQUENCES)
    got = np.concatenate([st.normal_double(3) for _ in range(7)])
    for j, w in enumerate(want):
        assert as_bits(got[:, j]).tolist() == w, (seed, SUBSEQUENCES[j])


@needs_nvcc
def test_u32_draws_and_offsets_match_host_curand(host_curand):
    """curand() itself, and curand_init's offset skip-ahead (a plain power of the step matrix)."""
    cases = [(s, q, o) for s in SEEDS[:3] for q in (0, 3, 100_002) for o in (0, 1, 5, 1000, 2 ** 40 + 7)]
    want = host_curand([(s, q, o, 6, 1, 1) for s, q, o in cases])
    for (s, q, o), w in zip(cases, want):
        st = X.XorwowStates(s, [q], offset=o)
        got = [int(st.next_u32()[0]) for _ in range(6)]
        assert got == w, (s, q, o)
        # skipping ahead is the same as drawing
        if o <= 1000:
            st2 = X.XorwowStates(s, [q])
            for _ in range(o):
                st2.next_u32()
            assert [int(st2.next_u32()[0]) for _ in range(6)] == w


def _precalc_table():
    text = (_include_dir() / "curand_precalc.h").read_text()
    m = re.search(r"precalc_xorwow_matrix_host\s*\[\s*32\s*\]\s*\[\s*800\s*\]\s*=\s*\{(.*?)\};", text, re.S)
    assert m, "precalc_xorwow_matrix_host not found in curand_precalc.h"
    words = [int(t.rstrip("uUlL"), 0) for t in re.findall(r"0x[0-9a-fA-F]+[uUlL]*|\b\d+[uUlL]*\b", m.group(1))]
    assert len(words) == 32 * 800
    return np.array(words, np.uint64).astype(np.uint32).reshape(32, 160, 5)


@needs_nvcc
def test_jump_matrices_equal_the_toolkit_table():
    """Entry k of precalc_xorwow_matrix_host is M^(4^k * 2^67): the restatement's J_0 and J_2 (computed
    by squaring the one-step matrix, no table involved) are its first two entries."""
    table = _precalc_table()
    assert np.array_equal(X.jump_matrix(0), table[0])
    assert np.array_equal(X.jump_matrix(2), table[1])
    assert np.array_equal(X.jump_matrix(4), table[2])


def test_jump_commutes_with_stepping():
    """M J = J M (both powers of M), and a subsequence jump leaves d alone: the state at subsequence 1
    stepped once is the state at subsequence 0 stepped once and then jumped."""
    a = X.XorwowStates(1804289383, [0])
    a.next_u32()
    b = X.XorwowStates(1804289383, [1])
    b.next_u32()
    assert np.array_equal(X.apply(X.jump_matrix(0), a.v), b.v) and np.array_equal(a.d, b.d)


def test_vectorised_states_equal_one_by_one():
    subs = np.array([0, 7, 256, 4097, 100_002])
    st = X.XorwowStates(2 ** 63 + 12345, subs)
    got = np.concatenate([st.normal_double(3) for _ in range(3)])
    for j, q in enumerate(subs):
        one = X.XorwowStates(2 ** 63 + 12345, [q])
        want = np.concatenate([one.normal_double(3) for _ in range(3)])[:, 0]
        assert np.array_equal(got[:, j], want)


def test_glibc_rand_defaults():
    """After srand(1) glibc's rand() gives 1804289383 then 846930886: the seeds of an unseeded run's
    first Langevin ensemble (and of heat_lan's source and sink)."""
    r = X.GlibcRand()
    r.srand(1)
    assert [r.rand(), r.rand()] == [1804289383, 846930886]

"""cuRAND's XORWOW generator (curandState, curand_kernel.h) restated in numpy, vectorised over atoms:
curand_init(seed, subsequence, offset), curand() and curand_normal_double(), the noise of nvt_lan,
nvt_bao and heat_lan.  Written from the algorithm (Marsaglia's xorwow, cuRAND's seeding and its
Box-Muller transform); tests/test_curand_oracle_cpu.py holds it to cuRAND itself built for the host,
bit for bit, and its jump matrices to the toolkit's precalculated table.

The 160-bit state v is linear over GF(2): one step is a 160x160 bit matrix M, and a subsequence is
2^67 steps, so curand_init's jump to subsequence s is the product of J_b = M^(2^(67+b)) over the set
bits b of s.  The Weyl counter d advances by 362437 per step and is unchanged by a subsequence jump
(362437 * 2^67 = 0 mod 2^32).  A matrix is kept in cuRAND's own layout: row r = 32 k + j holds the five
output words for input bit j of word k, so applying it XORs together the rows of the set input bits.

Host and device differ in one place: the device computes sin(pi v), cos(pi v) with sincospi, the host
with sin(v * pi), cos(v * pi).  This restatement follows the host (glibc's libm, through `math`), so
it equals host-built cuRAND bit for bit and sits a few ulp from the device.
"""
import math

import numpy as np

WEYL = 362437
TWO_POW_53_INV = 1.1102230246251565e-16  # CURAND_2POW53_INV_DOUBLE
PI = 3.1415926535897932                  # CURAND_PI_DOUBLE
_U32 = np.uint32


def _step(v):
    """One xorwow step of the linear part: v [5, m] uint32 -> new v (d is handled apart)."""
    t = v[0] ^ (v[0] >> _U32(2))
    out = np.empty_like(v)
    out[:4] = v[1:]
    out[4] = (v[4] ^ (v[4] << _U32(4))) ^ (t ^ (t << _U32(1)))
    return out


def apply(matrix, v):
    """matrix [160, 5] applied to the state vectors v [5, m]: XOR of the rows of the set input bits."""
    out = np.zeros_like(v)
    for r in range(160):
        bit = (v[r >> 5] >> _U32(r & 31)) & _U32(1)
        if not bit.any():
            continue
        out ^= matrix[r][:, None] & np.negative(bit)[None, :]  # -1 = all ones where the bit is set
    return out


def square(matrix):
    """matrix^2: each row (the image of one input bit) mapped once more."""
    return np.ascontiguousarray(apply(matrix, np.ascontiguousarray(matrix.T)).T)


def step_matrix():
    """M: the images of the 160 unit vectors under one step."""
    e = np.zeros((5, 160), np.uint32)
    for r in range(160):
        e[r >> 5, r] = _U32(1) << _U32(r & 31)
    return np.ascontiguousarray(_step(e).T)


_POW2 = []  # _POW2[k] = M^(2^k), grown on demand


def power_of_two(k):
    """M^(2^k), by k squarings of M (cached for the process)."""
    if not _POW2:
        _POW2.append(step_matrix())
    while len(_POW2) <= k:
        _POW2.append(square(_POW2[-1]))
    return _POW2[k]


def jump_matrix(b):
    """J_b = M^(2^(67+b)): skips 2^b subsequences."""
    return power_of_two(67 + b)


class XorwowStates:
    """n generator states (curandStateXORWOW) as numpy arrays: v [5, n], d [n], the Box-Muller flag
    [n] and the cached second normal [n]."""

    def __init__(self, seed, subsequence, offset=0):
        """curand_init(seed, subsequence[i], offset) for every i (_curand_init_scratch)."""
        sub = np.atleast_1d(np.asarray(subsequence, dtype=np.uint64))
        n = sub.shape[0]
        seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        s0 = (seed & 0xFFFFFFFF) ^ 0xaad26b49
        s1 = (seed >> 32) ^ 0xf7dcefdd
        t0 = (1099087573 * s0) & 0xFFFFFFFF
        t1 = (2591861531 * s1) & 0xFFFFFFFF
        v0 = [(123456789 + t0) & 0xFFFFFFFF, 362436069 ^ t0, (521288629 + t1) & 0xFFFFFFFF, 88675123 ^ t1,
              (5783321 + t0) & 0xFFFFFFFF]
        self.v = np.repeat(np.array(v0, np.uint32)[:, None], n, axis=1)
        self.d = np.full(n, (6615241 + t1 + t0) & 0xFFFFFFFF, np.uint32)
        b = 0
        rest = sub.copy()
        while rest.any():
            sel = np.nonzero(rest & np.uint64(1))[0]
            if sel.size:
                self.v[:, sel] = apply(jump_matrix(b), self.v[:, sel])
            rest >>= np.uint64(1)
            b += 1
        self.flag = np.zeros(n, np.uint32)
        self.extra = np.zeros(n, np.float64)
        if offset:
            self.skipahead(offset)

    @property
    def n(self):
        return self.d.shape[0]

    def skipahead(self, offset):
        """skipahead(offset): M^offset on v (a product of M^(2^k)), d += 362437 offset."""
        offset = int(offset)
        k = 0
        while offset >> k:
            if (offset >> k) & 1:
                self.v = apply(power_of_two(k), self.v)
            k += 1
        self.d = (self.d + _U32((WEYL * offset) & 0xFFFFFFFF)).astype(np.uint32)

    def next_u32(self, idx=None):
        """curand(): one 32-bit draw for the states idx (all by default)."""
        idx = slice(None) if idx is None else idx
        v = self.v[:, idx]
        nv = _step(v)
        self.v[:, idx] = nv
        d = self.d[idx] + _U32(WEYL)
        self.d[idx] = d
        return nv[4] + d

    def normal_double(self, k=1):
        """k successive curand_normal_double() per state: [k, n] float64."""
        out = np.empty((k, self.n))
        for c in range(k):
            need = np.nonzero(self.flag == 0)[0]
            have = np.nonzero(self.flag != 0)[0]
            out[c, have] = self.extra[have]
            self.flag[have] = 0
            if need.size:
                x0, x1, y0, y1 = (self.next_u32(need).astype(np.uint64) for _ in range(4))
                zx = x0 ^ (x1 << np.uint64(21))
                zy = y0 ^ (y1 << np.uint64(21))
                u = zx.astype(np.float64) * TWO_POW_53_INV + TWO_POW_53_INV / 2.0
                w = zy.astype(np.float64) * (TWO_POW_53_INV * 2.0) + TWO_POW_53_INV
                s = np.sqrt(-2.0 * _log(u))
                out[c, need] = _sin(w * PI) * s
                self.extra[need] = _cos(w * PI) * s
                self.flag[need] = 1
        return out

    def copy(self):
        c = object.__new__(XorwowStates)
        c.v, c.d, c.flag, c.extra = self.v.copy(), self.d.copy(), self.flag.copy(), self.extra.copy()
        return c


# glibc's libm element by element: numpy's own vector sin / cos / log may differ from it in the last bit
def _libm(f):
    uf = np.frompyfunc(f, 1, 1)
    return lambda x: uf(x).astype(np.float64)


_log, _sin, _cos = _libm(math.log), _libm(math.sin), _libm(math.cos)


class GlibcRand:
    """glibc's srand() / rand() through ctypes: the stream the b200md driver seeds its Langevin
    generators from (the first two values after srand(1) are 1804289383 and 846930886)."""

    def __init__(self):
        import ctypes
        import ctypes.util
        self.libc = ctypes.CDLL(ctypes.util.find_library("c") or "libc.so.6")

    def srand(self, seed):
        self.libc.srand(int(seed) & 0xFFFFFFFF)

    def rand(self):
        return int(self.libc.rand())

// b2_common.cuh -- shared definitions for libb200md (sm_90a).
//
// Kernel BODIES in this library are written as `B2_HD` functions of (thread index, params) so
// that tests/emu can compile the very same arithmetic for the host and check it against the
// oracle without a GPU.  The emulation build is test infrastructure only: the shipped library
// contains no host execution path (b2_api.cu returns an error if CUDA is unavailable).
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __device__ __forceinline__
#define B2_HOST_DEVICE __host__ __device__ // sizes both the kernels and the host setup (b2_setup.h) compute
#define B2_LDG(p) __ldg(p)
// streaming (evict-first) load / store for data that is touched once per kernel -- the neighbour
// lists -- so that it does not displace the gathered records and U rows from L1 / L2
#define B2_LDCS(p) __ldcs(p)
#define B2_STCS(p, v) __stcs((p), (v))
#else
#define B2_HD static inline
#define B2_HOST_DEVICE
#define B2_LDG(p) (*(p))
#define B2_LDCS(p) (*(p))
#define B2_STCS(p, v) (*(p) = (v))
#endif

#if !defined(__CUDACC__)
struct float4 {
  float x, y, z, w;
};
struct int4 {
  int x, y, z, w;
};
#endif

#if defined(__CUDA_ARCH__)
#define B2_ATOMIC_OR(p, v) atomicOr((p), (v))
#else
#define B2_ATOMIC_OR(p, v) (*(p) |= (v))
#endif

// ---- lane teams: kernels that spread ONE atom's neighbour loop over B2_TEAM adjacent lanes.
// Consecutive list entries are (mostly) consecutive cell-sorted atoms, so a team's gathers fall
// into a few 128-byte lines instead of one line per lane.  The host build (tests/emu) uses a team
// of one, for which every primitive is the identity.
#if defined(__CUDACC__)
#define B2_TEAM 8
__device__ __forceinline__ unsigned b2_team_mask() { return 0xFFu << (threadIdx.x & 24u); }
__device__ __forceinline__ float b2_team_sum(float v)
{
  const unsigned m = b2_team_mask();
  v += __shfl_xor_sync(m, v, 1);
  v += __shfl_xor_sync(m, v, 2);
  v += __shfl_xor_sync(m, v, 4);
  return v;
}
// bit l = predicate of team lane l
__device__ __forceinline__ unsigned b2_team_ballot(bool p)
{
  return (__ballot_sync(b2_team_mask(), p) >> (threadIdx.x & 24u)) & 0xFFu;
}
#define B2_POPC(x) __popc(x)
#else
#define B2_TEAM 1
static inline float b2_team_sum(float v) { return v; }
static inline unsigned b2_team_ballot(bool p) { return p ? 1u : 0u; }
#define B2_POPC(x) __builtin_popcount(x)
#endif

// Box passed by value to kernels: GPUMD's Box::cpu_h / float_h (src/model/box.cuh:18-35).
constexpr int B2_MAX_TYPES = 94; // NUM_ELEMENTS, src/utilities/common.cuh:18
constexpr int B2_NQMAX = 5;      // radial channels in groups of four: up to n_max_radial = 19

struct B2Box {
  double h[18]; // h[0..8] row-major (lattice vectors are columns), h[9..17] inverse
  float hf[18];
  int pbc[3];
  int ortho;
  double thickness[3];
  double volume;
};

// sorted-atom record: one 32-byte sector per neighbour gather
struct __attribute__((aligned(32))) B2Atom {
  double x, y, z;
  int type;
  int pad;
};

// FP32 minimum image with the reference's semantics (src/model/box.cuh:84-129): orthogonal boxes
// shift once by +-L when |x| > L/2; triclinic boxes go through fractional coordinates.  The fma
// nesting of the triclinic branch is the one nvcc's default contraction produces for the
// reference expression a*x + b*y + c*z = fma(c,z, fma(a,x, b*y)).
B2_HD void b2_mic(const B2Box& b, float& x, float& y, float& z)
{
  if (b.ortho) {
    if (b.pbc[0]) {
      const float L = b.hf[0], hl = L * 0.5f;
      if (x < -hl)
        x += L;
      else if (x > hl)
        x -= L;
    }
    if (b.pbc[1]) {
      const float L = b.hf[4], hl = L * 0.5f;
      if (y < -hl)
        y += L;
      else if (y > hl)
        y -= L;
    }
    if (b.pbc[2]) {
      const float L = b.hf[8], hl = L * 0.5f;
      if (z < -hl)
        z += L;
      else if (z > hl)
        z -= L;
    }
  } else {
    float sx = fmaf(b.hf[11], z, fmaf(b.hf[9], x, b.hf[10] * y));
    float sy = fmaf(b.hf[14], z, fmaf(b.hf[12], x, b.hf[13] * y));
    float sz = fmaf(b.hf[17], z, fmaf(b.hf[15], x, b.hf[16] * y));
    if (b.pbc[0])
      sx -= nearbyintf(sx);
    if (b.pbc[1])
      sy -= nearbyintf(sy);
    if (b.pbc[2])
      sz -= nearbyintf(sz);
    x = fmaf(b.hf[2], sz, fmaf(b.hf[0], sx, b.hf[1] * sy));
    y = fmaf(b.hf[5], sz, fmaf(b.hf[3], sx, b.hf[4] * sy));
    z = fmaf(b.hf[8], sz, fmaf(b.hf[6], sx, b.hf[7] * sy));
  }
}

// FP64 minimum image (src/model/box.cuh:37-82), used where the reference uses it
// (gpu_find_force_many_body, src/force/potential.cu:211-217).
B2_HD void b2_mic(const B2Box& b, double& x, double& y, double& z)
{
  if (b.ortho) {
    if (b.pbc[0]) {
      const double L = b.h[0];
      if (x < -L * 0.5)
        x += L;
      else if (x > L * 0.5)
        x -= L;
    }
    if (b.pbc[1]) {
      const double L = b.h[4];
      if (y < -L * 0.5)
        y += L;
      else if (y > L * 0.5)
        y -= L;
    }
    if (b.pbc[2]) {
      const double L = b.h[8];
      if (z < -L * 0.5)
        z += L;
      else if (z > L * 0.5)
        z -= L;
    }
  } else {
    double sx = b.h[9] * x + b.h[10] * y + b.h[11] * z;
    double sy = b.h[12] * x + b.h[13] * y + b.h[14] * z;
    double sz = b.h[15] * x + b.h[16] * y + b.h[17] * z;
    if (b.pbc[0])
      sx -= nearbyint(sx);
    if (b.pbc[1])
      sy -= nearbyint(sy);
    if (b.pbc[2])
      sz -= nearbyint(sz);
    x = b.h[0] * sx + b.h[1] * sy + b.h[2] * sz;
    y = b.h[3] * sx + b.h[4] * sy + b.h[5] * sz;
    z = b.h[6] * sx + b.h[7] * sy + b.h[8] * sz;
  }
}

// Pair displacement exactly as every reference kernel forms it (e.g. src/force/nep.cu:467-470):
// FP64 subtract, narrow to FP32, FP32 minimum image.
B2_HD void b2_r12(
  const B2Box& b, const B2Atom& a1, const B2Atom& a2, float& x12, float& y12, float& z12)
{
  x12 = (float)(a2.x - a1.x);
  y12 = (float)(a2.y - a1.y);
  z12 = (float)(a2.z - a1.z);
  b2_mic(b, x12, y12, z12);
}

// Per-thread register copy of what the pair geometry needs.  Orthogonal boxes (the common case)
// get a branch-free minimum image with identical results to b2_mic: exactly one of the two
// comparisons can be true, and an open direction has an infinite half-length.
struct B2Geo {
  int ortho;
  float Lx, Ly, Lz, hx, hy, hz;
};

B2_HD B2Geo b2_geo(const B2Box& b)
{
  B2Geo g;
  g.ortho = b.ortho;
  g.Lx = b.hf[0];
  g.Ly = b.hf[4];
  g.Lz = b.hf[8];
  g.hx = b.pbc[0] ? b.hf[0] * 0.5f : INFINITY;
  g.hy = b.pbc[1] ? b.hf[4] * 0.5f : INFINITY;
  g.hz = b.pbc[2] ? b.hf[8] * 0.5f : INFINITY;
  return g;
}

B2_HD void b2_r12(
  const B2Geo& g, const B2Box& b, const B2Atom& a1, const B2Atom& a2, float& x12, float& y12,
  float& z12)
{
  x12 = (float)(a2.x - a1.x);
  y12 = (float)(a2.y - a1.y);
  z12 = (float)(a2.z - a1.z);
  if (g.ortho) {
    x12 += (x12 < -g.hx) ? g.Lx : ((x12 > g.hx) ? -g.Lx : 0.0f);
    y12 += (y12 < -g.hy) ? g.Ly : ((y12 > g.hy) ? -g.Ly : 0.0f);
    z12 += (z12 < -g.hz) ? g.Lz : ((z12 > g.hz) ? -g.Lz : 0.0f);
  } else {
    b2_mic(b, x12, y12, z12);
  }
}

// 32-byte record through the read-only path as two 128-bit loads
B2_HD B2Atom b2_load_atom(const B2Atom* p)
{
#if defined(__CUDA_ARCH__)
  const int4* q = reinterpret_cast<const int4*>(p);
  const int4 lo = __ldg(q), hi = __ldg(q + 1);
  B2Atom a;
  a.x = __hiloint2double(lo.y, lo.x);
  a.y = __hiloint2double(lo.w, lo.z);
  a.z = __hiloint2double(hi.y, hi.x);
  a.type = hi.z;
  a.pad = hi.w;
  return a;
#else
  return *p;
#endif
}

// sin(pi x), cos(pi x)
B2_HD void b2_sincospi(float x, float& s, float& c)
{
#if defined(__CUDA_ARCH__)
  sincospif(x, &s, &c);
#else
  s = sinf(3.14159265358979f * x);
  c = cosf(3.14159265358979f * x);
#endif
}

// 1/sqrt(x): hardware approximation (<= 2 ulp) on the device.  -DB2_EXACT_RSQRT builds the
// correctly rounded 1/sqrt (diagnostic builds only: gpumd_b200.build.build_lib(variant=...)).
B2_HD float b2_rsqrt(float x)
{
#if defined(__CUDA_ARCH__) && !defined(B2_EXACT_RSQRT)
  return rsqrtf(x);
#else
  return 1.0f / sqrtf(x);
#endif
}

B2_HD float b2_cospi(float x)
{
#if defined(__CUDA_ARCH__)
  return cospif(x);
#else
  return cosf(3.14159265358979f * x);
#endif
}

// d^2 with the fma nesting nvcc emits for `x*x + y*y + z*z` (checked on the PTX of the reference
// expression, DESIGN.md "FP32 membership"): fma(z,z, fma(x,x, y*y)).  Membership tests against a
// cutoff use this so neighbour sets are bit-identical to the reference's.
B2_HD float b2_d2(float x, float y, float z) { return fmaf(z, z, fmaf(x, x, y * y)); }

// error bits latched on the device
enum {
  B2_ERR_SKIN_OVERFLOW = 1,
  B2_ERR_RADIAL_OVERFLOW = 2,
  B2_ERR_ANGULAR_OVERFLOW = 4,
  B2_ERR_CELL_RANGE = 8,
};

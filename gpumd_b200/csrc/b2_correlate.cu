// b2_correlate.cu -- the one time-correlation engine: per-atom vectors of the output groups gathered
// into a device ring of frames and correlated over Nc lags, for
//
//   b200md_dos_*  <- DOS: mass-weighted velocity autocorrelation and phonon DOS, src/measure/dos.cu:39-503
//   b200md_sdc_*  <- SDC: velocity autocorrelation and its running integral, src/measure/sdc.cu:34-338
//   b200md_msd_*  <- MSD: mean-square displacement of unwrapped positions, src/measure/msd.cu:52-542
//   b200md_shc_*  <- SHC: spectral heat current, the virial row of the transport direction against the
//                    velocity, SHC::preprocess / process / average_k / find_shc, src/measure/shc.cu:34-396
//   b200md_unwrap_begin / _end <- the unwrapped-position update around Integrate::compute1,
//                                 src/integrate/integrate.cu:295-375
//
// The reference correlates every sample with its whole ring of Nc stored frames (gpu_find_vac /
// gpu_find_msd: Nc blocks of 128 threads, each streaming one frame; shc.cu:249-309 likewise), so it
// reads Nc frames per sample.  Here the ring keeps Nc + CORR_B - 1 frames and the correlation is
// deferred: one flush correlates up to CORR_B pending time origins with all Nc lags and reads each ring
// frame once.  A flush happens when CORR_B origins are pending and before every finish.  The per-group
// sums have a fixed order and use no atomics: the results do not depend on scheduling.
#include "../../include/b200md.h"
#include "b2_host.h"
#include <algorithm>
#include <cmath>
#include <new>
#include <string>
#include <vector>

#ifndef B200MD_CORR_BLOCK
#define B200MD_CORR_BLOCK 16
#endif

namespace b2 {

// What a flush correlates.  Each kind fixes the frame width, the accumulators, the update and the
// output rows of k_corr:
//   Vac  frame v_x v_y v_z; per component sum_j w_j v_now . v_past (gpu_find_vac, dos.cu:84-143 and
//        sdc.cu:71-128; w = the mass for DOS, 1 for SDC); 3 rows
//   Msd  frame x_x x_y x_z; per component sum_j (x_now - x_past)^2 (gpu_find_msd, msd.cu:89-149); 3 rows
//   Shc  frame s_x s_y s_z v_x v_y v_z (the virial row of the transport direction, shc.cu:188-191);
//        blockIdx.y = 0 correlates s(now) . v(past) (gpu_find_k's "negative" call), 1 correlates
//        v(now) . s(past) ("positive"), each into an in-plane (x + y) and an out-of-plane (z) sum;
//        4 rows: negative in, out, positive in, out
enum class CorrKind { Vac, Msd, Shc };
__host__ __device__ constexpr int corr_width(CorrKind k) { return k == CorrKind::Shc ? 6 : 3; }
__host__ __device__ constexpr int corr_rows(CorrKind k) { return k == CorrKind::Shc ? 4 : 3; }

namespace {

constexpr int CORR_B = B200MD_CORR_BLOCK; // time origins per correlation flush
constexpr int CORR_CHUNK = 256;           // atoms one warp correlates (never straddles an output group)
constexpr int CORR_WARPS = 4;             // warps per block of k_corr
constexpr int RED_ROWS = 32, RED_LANES = 32; // k_corr_reduce: 32 output entries x 32 chunk lanes

constexpr double PI = 3.14159265358979;             // common.cuh:19
constexpr double TIME_UNIT_CONVERSION = 1.018051e+1; // common.cuh:26

// the base pointers of the source rows of one frame
struct Rows {
  const double* p[6];
};

// frame[c * G + j] = src.p[c][contents[j]] for c < ncomp <= 6 (Group::find_contents order); contents
// NULL: the atoms 0 .. G-1
__global__ void __launch_bounds__(256) k_corr_gather(
  int G, int ncomp, const int* __restrict__ contents, Rows src, double* frame)
{
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < G) {
    const int m = contents ? contents[j] : j;
#pragma unroll
    for (int c = 0; c < 6; ++c)
      if (c < ncomp)
        frame[(size_t)c * G + j] = src.p[c][m];
  }
}

// Blocked correlation of P <= CORR_B consecutive time origins k0 .. k0+P-1 with lags 0 .. Nc-1.  One
// warp owns one chunk (start, length) of ring atoms.  Each lane keeps three "now" components of every
// origin in registers (times the atom's mass for DOS) and walks the past frames f = k0+CORR_B-1 down
// to k0-Nc+1 once: frame f adds to lag k0+p-f of origin p.  The accumulators of CORR_B consecutive
// lags rotate through registers; after frame f the lag k0-f is complete, is reduced over the warp and
// stored to partial[chunk][corr_rows(K)][Nc].  A slot holds one lag from the moment it is cleared until
// it is stored, so lags < 0 (frames newer than an origin, possibly stale) and lags >= Nc never reach
// partial.  Origins p >= P are skipped (Msd) or carry zero "now" values (dot products).
template <CorrKind K>
__global__ void __launch_bounds__(CORR_WARPS * 32) k_corr(
  int G, int Nc, int R, int k0, int P, int nchunks, const int2* __restrict__ chunks,
  const double* __restrict__ mass, const double* __restrict__ ring, double* partial)
{
  constexpr int W = corr_width(K), NOUT = corr_rows(K), NACC = K == CorrKind::Shc ? 2 : 3;
  const int lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * CORR_WARPS + (threadIdx.x >> 5);
  if (chunk >= nchunks)
    return; // whole warps only: no block-wide synchronisation below
  const int half = K == CorrKind::Shc ? blockIdx.y : 0;
  const int now_c = 3 * half, past_c = K == CorrKind::Shc ? 3 - now_c : 0; // first frame component
  const int2 ch = chunks[chunk];
  double* out = partial + (size_t)chunk * NOUT * Nc + 2 * half * Nc;
  const size_t g = (size_t)G, frame = W * g; // a component, a frame
  const int T = Nc + CORR_B - 1;              // number of past frames
  for (int sub = 0; sub < ch.y; sub += 32) {
    const bool ok = sub + lane < ch.y;
    const int j = ch.x + sub + lane;
    const double w = (K == CorrKind::Vac && ok && mass) ? mass[j] : 1.0;
    double n[3][CORR_B];
#pragma unroll
    for (int p = 0; p < CORR_B; ++p) {
#pragma unroll
      for (int c = 0; c < 3; ++c)
        n[c][p] = 0.0;
      if (ok && p < P) {
        const double* fr = ring + (size_t)((k0 + p) % R) * frame + now_c * g + j;
#pragma unroll
        for (int c = 0; c < 3; ++c)
          n[c][p] = K == CorrKind::Vac ? w * fr[c * g] : fr[c * g]; // dos.cu:113: mass * v_now * v_past
      }
    }
    double a[NACC][CORR_B];
#pragma unroll
    for (int q = 0; q < CORR_B; ++q)
#pragma unroll
      for (int c = 0; c < NACC; ++c)
        a[c][q] = 0.0;
    for (int tb = 0; tb < T; tb += CORR_B) {
#pragma unroll
      for (int u = 0; u < CORR_B; ++u) {
        const int t = tb + u;
        double x[3] = {0.0, 0.0, 0.0}; // the past frame
        if (ok && t < T) {
          const int f = k0 + CORR_B - 1 - t; // >= k0 - Nc + 1 >= 0
          const double* fr = ring + (size_t)(f % R) * frame + past_c * g + j;
#pragma unroll
          for (int c = 0; c < 3; ++c)
            x[c] = fr[c * g];
        }
#pragma unroll
        for (int p = 0; p < CORR_B; ++p) {
          const int q = (p + u + 1) % CORR_B; // register slot of lag p + t - (CORR_B - 1)
          if constexpr (K == CorrKind::Vac) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
              a[c][q] = fma(n[c][p], x[c], a[c][q]);
          } else if constexpr (K == CorrKind::Msd) {
            if (ok && p < P) {
#pragma unroll
              for (int c = 0; c < 3; ++c) {
                const double d = n[c][p] - x[c];
                a[c][q] = fma(d, d, a[c][q]);
              }
            }
          } else {
            a[0][q] = fma(n[1][p], x[1], fma(n[0][p], x[0], a[0][q]));
            a[1][q] = fma(n[2][p], x[2], a[1][q]);
          }
        }
        const int q = (u + 1) % CORR_B, lag = t - (CORR_B - 1);
        double s[NACC];
#pragma unroll
        for (int c = 0; c < NACC; ++c) {
          s[c] = a[c][q];
          a[c][q] = 0.0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
          for (int c = 0; c < NACC; ++c)
            s[c] += __shfl_down_sync(0xffffffffu, s[c], o);
        if (lane == 0 && lag >= 0 && lag < Nc)
#pragma unroll
          for (int c = 0; c < NACC; ++c)
            out[c * Nc + lag] = sub == 0 ? s[c] : out[c * Nc + lag] + s[c];
      }
    }
  }
}

// acc[group][r] += sum of partial[chunk][r] over the group's chunks, r < row.  Block (group, tile of
// RED_ROWS entries); lane c of a row sums the chunks c, c + RED_LANES, ... in order, then the lanes are
// added in a fixed tree: the order does not depend on scheduling.
__global__ void __launch_bounds__(RED_ROWS * RED_LANES) k_corr_reduce(
  int ngroups, int row, const int* __restrict__ group_chunk, const double* __restrict__ partial, double* acc)
{
  __shared__ double s[RED_LANES][RED_ROWS + 1];
  const int x = threadIdx.x % RED_ROWS, c0 = threadIdx.x / RED_ROWS;
  const int r = blockIdx.x * RED_ROWS + x;
  for (int gr = blockIdx.y; gr < ngroups; gr += gridDim.y) { // gridDim.y <= 65535
    double v = 0.0;
    if (r < row)
      for (int c = group_chunk[gr] + c0; c < group_chunk[gr + 1]; c += RED_LANES)
        v += partial[(size_t)c * row + r];
    s[c0][x] = v;
    __syncthreads();
    for (int o = RED_LANES / 2; o > 0; o >>= 1) {
      if (c0 < o)
        s[c0][x] += s[c0 + o][x];
      __syncthreads();
    }
    if (c0 == 0 && r < row)
      acc[(size_t)gr * row + r] += s[0][x];
    __syncthreads();
  }
}

// gpu_copy_position + gpu_update_unwrapped_position, integrate.cu:295-330
__global__ void __launch_bounds__(256) k_copy3(int n, const double* __restrict__ x, double* y)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const size_t s = (size_t)n;
    y[i] = x[i];
    y[s + i] = x[s + i];
    y[2 * s + i] = x[2 * s + i];
  }
}

__global__ void __launch_bounds__(256) k_unwrap_add(
  int n, const double* __restrict__ x_new, const double* __restrict__ x_old, double* u)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const size_t s = (size_t)n;
    u[i] += x_new[i] - x_old[i];
    u[s + i] += x_new[s + i] - x_old[s + i];
    u[2 * s + i] += x_new[2 * s + i] - x_old[2 * s + i];
  }
}

} // namespace
} // namespace b2

using namespace b2;

// shared by DOS, SDC, MSD and SHC: the ring of gathered frames, the pending time origins and the
// per-group running sums acc[group][row][lag]
struct b200md_corr {
  const char* name = "";
  CorrKind kind = CorrKind::Vac;
  int xrow[3] = {0, 1, 2}; // the rows of the first source a frame starts with (SHC: its virial row)
  int Nc = 0, sample_interval = 1, ngroups = 0, G = 0, R = 0;
  int max_index = -1;       // largest atom index in contents (identity: G - 1)
  int k0 = 0, pending = 0;  // first pending time origin and how many there are
  int num_time_origins = 0; // sdc.cu:208, msd.cu:320, shc.cu:249-251
  int nchunks = 0;
  double dt_natural = 0.0; // time_step * sample_interval (not SHC, which gets its time step at finish)
  std::vector<int> sizes;
  DevBuf<int> contents;    // empty: the whole system in atom order
  DevBuf<int2> chunks;     // (ring start, length) per warp
  DevBuf<int> group_chunk; // chunks of group g: [group_chunk[g], group_chunk[g+1])
  DevBuf<double> mass;     // DOS: the masses in ring order (gpu_copy_mass, dos.cu:39-46,326-336)
  DevBuf<double> ring, partial, acc;
};
struct b200md_dos : b200md_corr {
  double omega_max = 0.0;
  int num_dos_points = 0;
};
struct b200md_sdc : b200md_corr {};
struct b200md_msd : b200md_corr {};
struct b200md_shc : b200md_corr {};

namespace {

std::string fn(const b200md_corr* p, const char* what) { return std::string("b200md_") + p->name + what; }

// the checks every create makes, then the device buffers; B200MD_OK or an error code with the message set
int corr_init(
  b200md_corr* p, int Nc, int sample_interval, int number_of_steps, double time_step, int num_groups,
  const int* group_sizes, const int* contents)
{
  if (!group_sizes || num_groups < 1 || (!contents && num_groups != 1)) {
    set_error(fn(p, "_create: bad argument"));
    return B200MD_ERR_ARG;
  }
  if (sample_interval < 1) { // dos.cu:168-170, sdc.cu:316-318, msd.cu:497-499
    set_error(fn(p, "_create: sample interval should be positive"));
    return B200MD_ERR_ARG;
  }
  if (Nc < 1) { // dos.cu:176-178, sdc.cu:325-327, msd.cu:506-508
    set_error(fn(p, "_create: number of correlation steps should be positive"));
    return B200MD_ERR_ARG;
  }
  if (p->kind != CorrKind::Shc && !(time_step > 0.0)) { // SHC gets its time step at finish
    set_error(fn(p, "_create: time_step should be positive"));
    return B200MD_ERR_ARG;
  }
  // msd.cu:217-219 for MSD.  The first time origin is sample Nc - 1; for DOS, SDC and SHC the reference
  // divides by zero without one (dos.cu:418-424, sdc.cu:240, shc.cu:323), so a run too short for it is
  // refused too
  if (number_of_steps / sample_interval < Nc) {
    set_error(fn(p, p->kind == CorrKind::Msd ? "_create: MSD correlation times sampling interval should be <= "
                                               "number of MD steps (the run gives no time origin)"
                                             : "_create: the run gives no time origin (need number_of_steps / "
                                               "sample_interval >= Nc)"));
    return B200MD_ERR_ARG;
  }
  long long G = 0;
  for (int gr = 0; gr < num_groups; ++gr) {
    if (group_sizes[gr] < 0) {
      set_error(fn(p, "_create: negative group size"));
      return B200MD_ERR_ARG;
    }
    G += group_sizes[gr];
  }
  if (G < 1 || G > 0x7fffffff) {
    set_error(fn(p, "_create: the groups must hold between 1 and 2^31-1 atoms"));
    return B200MD_ERR_ARG;
  }
  int max_index = (int)G - 1;
  if (contents) {
    max_index = -1;
    for (long long j = 0; j < G; ++j) {
      if (contents[j] < 0) {
        set_error(fn(p, "_create: negative atom index in contents"));
        return B200MD_ERR_ARG;
      }
      max_index = contents[j] > max_index ? contents[j] : max_index;
    }
  }
  p->Nc = Nc;
  p->sample_interval = sample_interval;
  p->dt_natural = time_step * sample_interval;
  p->ngroups = num_groups;
  p->G = (int)G;
  p->R = Nc + CORR_B - 1;
  p->max_index = max_index;
  p->sizes.assign(group_sizes, group_sizes + num_groups);
  std::vector<int2> chunks;
  std::vector<int> group_chunk(num_groups + 1, 0);
  int start = 0;
  for (int gr = 0; gr < num_groups; ++gr) {
    group_chunk[gr] = (int)chunks.size();
    for (long long o = 0; o < group_sizes[gr]; o += CORR_CHUNK) // long long: o + CORR_CHUNK may pass 2^31
      chunks.push_back(make_int2(start + (int)o, (int)std::min<long long>(group_sizes[gr] - o, CORR_CHUNK)));
    start += group_sizes[gr];
  }
  group_chunk[num_groups] = (int)chunks.size();
  p->nchunks = (int)chunks.size();
  const int width = corr_width(p->kind), rows = corr_rows(p->kind);
  const bool ok =
    p->ring.reserve((size_t)p->R * width * p->G) == cudaSuccess &&
    p->partial.reserve((size_t)p->nchunks * rows * Nc) == cudaSuccess &&
    p->acc.reserve((size_t)num_groups * rows * Nc) == cudaSuccess &&
    p->chunks.reserve(chunks.size()) == cudaSuccess &&
    p->group_chunk.reserve(group_chunk.size()) == cudaSuccess &&
    (!contents || p->contents.reserve((size_t)G) == cudaSuccess);
  if (!ok) {
    cudaGetLastError(); // clear the allocation error
    set_error(std::string("out of device memory (") + p->name + " ring of Nc + " + std::to_string(CORR_B - 1) +
              " frames of " + std::to_string(G) + " atoms, " +
              std::to_string((double)p->R * width * 8 * G / 1e9) + " GB)");
    return B200MD_ERR_CUDA;
  }
  // the ring starts as zeros: a partial flush reads not-yet-written frames (for lags < 0 only)
  if (cudaMemset(p->ring.p, 0, sizeof(double) * p->R * width * (size_t)p->G) != cudaSuccess ||
      cudaMemset(p->acc.p, 0, sizeof(double) * num_groups * rows * (size_t)Nc) != cudaSuccess ||
      cudaMemcpy(p->chunks.p, chunks.data(), sizeof(int2) * chunks.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(p->group_chunk.p, group_chunk.data(), sizeof(int) * group_chunk.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
      (contents && cudaMemcpy(p->contents.p, contents, sizeof(int) * (size_t)G, cudaMemcpyHostToDevice) != cudaSuccess)) {
    set_error(fn(p, "_create: CUDA error while initialising"));
    return B200MD_ERR_CUDA;
  }
  return B200MD_OK;
}

int corr_flush(b200md_corr* p, cudaStream_t st)
{
  if (p->pending == 0)
    return B200MD_OK;
  if (p->nchunks > 0) {
    auto* corr = p->kind == CorrKind::Vac ? k_corr<CorrKind::Vac>
               : p->kind == CorrKind::Msd ? k_corr<CorrKind::Msd>
                                          : k_corr<CorrKind::Shc>;
    const dim3 grid(grid_for(p->nchunks, CORR_WARPS), p->kind == CorrKind::Shc ? 2 : 1); // SHC: two halves
    corr<<<grid, CORR_WARPS * 32, 0, st>>>(
      p->G, p->Nc, p->R, p->k0, p->pending, p->nchunks, p->chunks.p, p->mass.p, p->ring.p, p->partial.p);
    B2_LAUNCHED();
    const int row = corr_rows(p->kind) * p->Nc;
    const dim3 rgrid(grid_for(row, RED_ROWS), std::min(p->ngroups, 65535));
    k_corr_reduce<<<rgrid, RED_ROWS * RED_LANES, 0, st>>>(p->ngroups, row, p->group_chunk.p, p->partial.p, p->acc.p);
    B2_LAUNCHED();
  }
  p->k0 += p->pending;
  p->pending = 0;
  return B200MD_OK;
}

// process() of dos.cu:236-244, sdc.cu:173-223, msd.cu:285-361, shc.cu:162-310: every sample_interval
// steps gather a frame, the rows xrow of d_x[.][stride] and, for SHC, the three rows of d_v[3][stride];
// from sample Nc - 1 on, each sample is a time origin
int corr_sample(b200md_corr* p, int step, int n, int stride, const double* d_x, const double* d_v, void* stream)
{
  if (!p || step < 0 || n <= p->max_index || stride < n || !d_x || (p->kind == CorrKind::Shc && !d_v)) {
    set_error(std::string("b200md_") + (p ? p->name : "corr") +
              "_sample: bad argument (n must exceed every atom index of the groups)");
    return B200MD_ERR_ARG;
  }
  if ((step + 1) % p->sample_interval != 0)
    return B200MD_OK;
  const int k = step / p->sample_interval; // sample_step
  cudaStream_t st = (cudaStream_t)stream;
  const int width = corr_width(p->kind);
  Rows src = {};
  for (int c = 0; c < 3; ++c) {
    src.p[c] = d_x + (size_t)p->xrow[c] * stride;
    if (width == 6)
      src.p[3 + c] = d_v + (size_t)c * stride;
  }
  k_corr_gather<<<grid_for(p->G, 256), 256, 0, st>>>(
    p->G, width, p->contents.p, src, p->ring.p + (size_t)(k % p->R) * width * p->G);
  B2_LAUNCHED();
  if (k >= p->Nc - 1) {
    if (p->pending == 0)
      p->k0 = k;
    ++p->pending;
    ++p->num_time_origins;
    if (p->pending == CORR_B)
      return corr_flush(p, st);
  }
  return B200MD_OK;
}

// flush, then copy acc[group][corr_rows][Nc] to the host (synchronises)
int corr_take(b200md_corr* p, std::vector<double>& acc, void* stream)
{
  if (p->num_time_origins == 0) {
    set_error(fn(p, "_finish: no time origin was sampled"));
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = corr_flush(p, st);
  if (rc != B200MD_OK)
    return rc;
  acc.resize((size_t)p->ngroups * corr_rows(p->kind) * p->Nc);
  B2_CUDA(cudaMemcpyAsync(acc.data(), p->acc.p, sizeof(double) * acc.size(), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200MD_OK;
}

// new T + corr_init; *out only on success
template <typename T>
int corr_create(
  const char* name, CorrKind kind, int Nc, int sample_interval, int number_of_steps, double time_step,
  int num_groups, const int* group_sizes, const int* contents, T** out)
{
  if (!out) {
    set_error(std::string("b200md_") + name + "_create: bad argument");
    return B200MD_ERR_ARG;
  }
  T* p = new (std::nothrow) T;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->name = name;
  p->kind = kind;
  const int rc = corr_init(p, Nc, sample_interval, number_of_steps, time_step, num_groups, group_sizes, contents);
  if (rc != B200MD_OK) {
    delete p;
    return rc;
  }
  *out = p;
  return B200MD_OK;
}

} // namespace

extern "C" {

int b200md_dos_create(
  int Nc, int sample_interval, int number_of_steps, double time_step, double omega_max, int num_dos_points,
  int num_groups, const int* group_sizes, const int* contents, int n, const double* d_mass, b200md_dos** out)
{
  if (!out || !d_mass || n < 1) {
    set_error("b200md_dos_create: bad argument");
    return B200MD_ERR_ARG;
  }
  if (!(omega_max > 0.0)) { // dos.cu:184-186
    set_error("b200md_dos_create: maximal angular frequency should be positive");
    return B200MD_ERR_ARG;
  }
  if (num_dos_points < 1) { // dos.cu:275-277 (the default, -1, is Nc: dos.cu:304-306)
    set_error("b200md_dos_create: number of DOS points must be > 0");
    return B200MD_ERR_ARG;
  }
  const double dt_in_ps = time_step * sample_interval * TIME_UNIT_CONVERSION / 1000.0;
  if (time_step > 0.0 && sample_interval > 0 && 1.0 / dt_in_ps < omega_max / PI) { // dos.cu:284-288
    set_error("b200md_dos_create: Velocity sampling rate < Nyquist frequency.");
    return B200MD_ERR_ARG;
  }
  b200md_dos* p = nullptr;
  int rc = corr_create("dos", CorrKind::Vac, Nc, sample_interval, number_of_steps, time_step, num_groups, group_sizes,
                       contents, &p);
  if (rc != B200MD_OK)
    return rc;
  p->omega_max = omega_max;
  p->num_dos_points = num_dos_points;
  if (p->max_index >= n) {
    set_error("b200md_dos_create: an atom index of the groups is >= n");
    rc = B200MD_ERR_ARG;
  } else if (p->mass.reserve((size_t)p->G) != cudaSuccess) {
    cudaGetLastError();
    set_error("out of device memory (DOS masses)");
    rc = B200MD_ERR_CUDA;
  } else {
    k_corr_gather<<<grid_for(p->G, 256), 256>>>(p->G, 1, p->contents.p, Rows{{d_mass}}, p->mass.p);
    ++g_launch_count;
    if (cudaDeviceSynchronize() != cudaSuccess) {
      set_error("b200md_dos_create: CUDA error while gathering the masses");
      rc = B200MD_ERR_CUDA;
    }
  }
  if (rc != B200MD_OK) {
    delete p;
    return rc;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_dos_destroy(b200md_dos* p) { delete p; }

int b200md_dos_sample(b200md_dos* p, int step, int n, int stride, const double* d_velocity, void* stream)
{
  return corr_sample(p, step, n, stride, d_velocity, nullptr, stream);
}

int b200md_dos_finish(b200md_dos* p, double* mvac, double* dos, void* stream)
{
  if (!p || !mvac || !dos) {
    set_error("b200md_dos_finish: bad argument");
    return B200MD_ERR_ARG;
  }
  std::vector<double> acc;
  const int rc = corr_take(p, acc, stream);
  if (rc != B200MD_OK)
    return rc;
  const int Nc = p->Nc, nw_all = p->num_dos_points;
  const double dt_in_ps = p->dt_natural * TIME_UNIT_CONVERSION / 1000.0; // dos.cu:284-285
  const double d_omega = p->omega_max / nw_all;
  for (int gr = 0; gr < p->ngroups; ++gr) {
    for (int c = 0; c < 3; ++c) {
      double* v = acc.data() + ((size_t)gr * 3 + c) * Nc;
      const double v0 = v[0];
      for (int nc = 0; nc < Nc; nc++) { // normalize_vac, dos.cu:414-427 (0 / 0 for an empty group)
        v[nc] /= v0;
        mvac[((size_t)gr * 3 + c) * Nc + nc] = v[nc];
      }
      for (int nc = 0; nc < Nc; nc++) { // find_dos, dos.cu:450-481
        const double hann_window = (cos((PI * nc) / Nc) + 1.0) * 0.5;
        const double multiply_factor = (nc == 0) ? hann_window : 2.0 * hann_window;
        v[nc] *= multiply_factor;
      }
      for (int nw = 0; nw < nw_all; nw++) {
        const double omega = d_omega + nw * d_omega;
        double d = 0.0;
        for (int nc = 0; nc < Nc; nc++) {
          const double cos_factor = cos(omega * nc * dt_in_ps);
          d += v[nc] * cos_factor;
        }
        d *= dt_in_ps * 2.0 * p->sizes[gr];
        dos[((size_t)gr * 3 + c) * nw_all + nw] = d;
      }
    }
  }
  return B200MD_OK;
}

int b200md_sdc_create(
  int Nc, int sample_interval, int number_of_steps, double time_step, int num_groups,
  const int* group_sizes, const int* contents, b200md_sdc** out)
{
  return corr_create("sdc", CorrKind::Vac, Nc, sample_interval, number_of_steps, time_step, num_groups, group_sizes,
                     contents, out);
}

void b200md_sdc_destroy(b200md_sdc* p) { delete p; }

int b200md_sdc_sample(b200md_sdc* p, int step, int n, int stride, const double* d_velocity, void* stream)
{
  return corr_sample(p, step, n, stride, d_velocity, nullptr, stream);
}

int b200md_sdc_finish(b200md_sdc* p, double* vac, double* sdc, void* stream)
{
  if (!p || !vac || !sdc) {
    set_error("b200md_sdc_finish: bad argument");
    return B200MD_ERR_ARG;
  }
  std::vector<double> acc;
  const int rc = corr_take(p, acc, stream);
  if (rc != B200MD_OK)
    return rc;
  const int Nc = p->Nc;
  const double sdc_unit_conversion = 1.0e3 / TIME_UNIT_CONVERSION; // sdc.cu:257-258
  const double vac_unit_conversion = sdc_unit_conversion * sdc_unit_conversion;
  const double dt2 = p->dt_natural * 0.5;
  for (int gr = 0; gr < p->ngroups; ++gr) {
    const double vac_scaler = 1.0 / ((double)p->sizes[gr] * (double)p->num_time_origins); // sdc.cu:240
    for (int c = 0; c < 3; ++c) {
      const size_t o = ((size_t)gr * 3 + c) * Nc;
      double* v = acc.data() + o;
      for (int nc = 0; nc < Nc; nc++)
        v[nc] *= vac_scaler;
      double s = 0.0; // sdc.cu:247-255
      for (int nc = 0; nc < Nc; nc++) {
        if (nc > 0)
          s = s + (v[nc - 1] + v[nc]) * dt2;
        vac[o + nc] = v[nc] * vac_unit_conversion;
        sdc[o + nc] = s * sdc_unit_conversion;
      }
    }
  }
  return B200MD_OK;
}

int b200md_msd_create(
  int Nc, int sample_interval, int number_of_steps, double time_step, int num_groups,
  const int* group_sizes, const int* contents, b200md_msd** out)
{
  return corr_create("msd", CorrKind::Msd, Nc, sample_interval, number_of_steps, time_step, num_groups, group_sizes,
                     contents, out);
}

void b200md_msd_destroy(b200md_msd* p) { delete p; }

int b200md_msd_sample(b200md_msd* p, int step, int n, int stride, const double* d_unwrapped, void* stream)
{
  return corr_sample(p, step, n, stride, d_unwrapped, nullptr, stream);
}

int b200md_msd_finish(b200md_msd* p, double* msd, double* sdc, void* stream)
{
  if (!p || !msd || !sdc) {
    set_error("b200md_msd_finish: bad argument");
    return B200MD_ERR_ARG;
  }
  std::vector<double> acc;
  const int rc = corr_take(p, acc, stream);
  if (rc != B200MD_OK)
    return rc;
  const int Nc = p->Nc;
  const double sdc_unit_conversion = 1.0e3 / TIME_UNIT_CONVERSION; // msd.cu:399
  const double dt2inv = 0.5 / p->dt_natural;
  for (int gr = 0; gr < p->ngroups; ++gr) { // MSD::write, msd.cu:373-397
    const int num_atoms = p->sizes[gr];
    double msd_scaler = 0.0; // an empty group gives rows of zeros
    if (num_atoms > 0 && p->num_time_origins > 0)
      msd_scaler = 1.0 / ((double)num_atoms * (double)p->num_time_origins);
    for (int c = 0; c < 3; ++c) {
      const size_t o = ((size_t)gr * 3 + c) * Nc;
      for (int nc = 0; nc < Nc; nc++)
        msd[o + nc] = acc[o + nc] * msd_scaler;
      sdc[o] = 0.0;
      for (int nc = 1; nc < Nc; nc++)
        sdc[o + nc] = (msd[o + nc] - msd[o + nc - 1]) * dt2inv * sdc_unit_conversion;
    }
  }
  return B200MD_OK;
}

int b200md_shc_create(
  int Nc, int sample_interval, int direction, int number_of_steps, int num_groups,
  const int* group_sizes, const int* contents, b200md_shc** out)
{
  // SHC::parse, shc.cu:466-542
  if (sample_interval < 1 || sample_interval > 50) {
    set_error("b200md_shc_create: sample_interval should be in [1, 50]");
    return B200MD_ERR_ARG;
  }
  if (Nc < 100 || Nc > 1000) {
    set_error("b200md_shc_create: Nc should be in [100, 1000]");
    return B200MD_ERR_ARG;
  }
  if (direction < 0 || direction > 2) {
    set_error("b200md_shc_create: direction should be 0 (x), 1 (y) or 2 (z)");
    return B200MD_ERR_ARG;
  }
  const int rc = corr_create("shc", CorrKind::Shc, Nc, sample_interval, number_of_steps, 0.0, num_groups,
                             group_sizes, contents, out);
  if (rc == B200MD_OK) {
    const int tensor[3][3] = {{0, 3, 4}, {6, 1, 5}, {7, 8, 2}}; // shc.cu:188
    std::copy(tensor[direction], tensor[direction] + 3, (*out)->xrow);
  }
  return rc;
}

void b200md_shc_destroy(b200md_shc* p) { delete p; }

int b200md_shc_sample(
  b200md_shc* p, int step, int n, int stride, const double* d_virial, const double* d_velocity,
  void* stream)
{
  return corr_sample(p, step, n, stride, d_virial, d_velocity, stream);
}

int b200md_shc_finish(
  b200md_shc* p, double time_step, int num_omega, double max_omega, double* ki, double* ko,
  double* shc_i, double* shc_o, void* stream)
{
  if (!p || num_omega < 0 || !(max_omega > 0.0) || !ki || !ko || (num_omega > 0 && (!shc_i || !shc_o))) {
    set_error("b200md_shc_finish: bad argument (num_omega >= 0, max_omega > 0)");
    return B200MD_ERR_ARG;
  }
  std::vector<double> acc;
  const int rc = corr_take(p, acc, stream);
  if (rc != B200MD_OK)
    return rc;
  const int Nc = p->Nc, Nk = 2 * Nc - 1;
  const double scalar = 1000.0 / TIME_UNIT_CONVERSION / p->num_time_origins;
  const double dt_in_ps = time_step * p->sample_interval * TIME_UNIT_CONVERSION / 1000.0;
  const double d_omega = max_omega / num_omega;
  for (int gr = 0; gr < p->ngroups; ++gr) {
    const double* a = acc.data() + (size_t)gr * 4 * Nc; // neg_i, neg_o, pos_i, pos_o
    double* gi = ki + (size_t)gr * Nk;
    double* go = ko + (size_t)gr * Nk;
    for (int nc = 0; nc < Nc - 1; ++nc) { // average_k, shc.cu:312-348
      gi[nc] = a[Nc - nc - 1] * scalar;
      go[nc] = a[Nc + Nc - nc - 1] * scalar;
    }
    for (int nc = 0; nc < Nc; ++nc) {
      gi[nc + Nc - 1] = a[2 * Nc + nc] * scalar;
      go[nc + Nc - 1] = a[3 * Nc + nc] * scalar;
    }
    // find_shc, shc.cu:350-396: Hann window, then the cosine transform (the windowed ki / ko are
    // what shc.out lists)
    for (int nc = 0; nc < Nk; ++nc) {
      const double hann_window = (cos(PI * (nc + 1 - Nc) / Nc) + 1.0) * 0.5;
      gi[nc] *= hann_window;
      go[nc] *= hann_window;
    }
    double* si = shc_i + (size_t)gr * num_omega;
    double* so = shc_o + (size_t)gr * num_omega;
    for (int nw = 0; nw < num_omega; ++nw) {
      const double omega = (nw + 1) * d_omega;
      double s_i = 0.0, s_o = 0.0;
      for (int nc = 0; nc < Nk; nc++) {
        const double t_in_ps = (nc + 1 - Nc) * dt_in_ps;
        const double cos_factor = cos(omega * t_in_ps);
        s_i += gi[nc] * cos_factor;
        s_o += go[nc] * cos_factor;
      }
      si[nw] = s_i * 2.0 * dt_in_ps;
      so[nw] = s_o * 2.0 * dt_in_ps;
    }
  }
  return B200MD_OK;
}

int b200md_unwrap_begin(int n, const double* d_position, double* d_position_old, void* stream)
{
  if (n < 1 || !d_position || !d_position_old) {
    set_error("b200md_unwrap_begin: bad argument");
    return B200MD_ERR_ARG;
  }
  k_copy3<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(n, d_position, d_position_old);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_unwrap_end(int n, const double* d_position, const double* d_position_old, double* d_unwrapped, void* stream)
{
  if (n < 1 || !d_position || !d_position_old || !d_unwrapped) {
    set_error("b200md_unwrap_end: bad argument");
    return B200MD_ERR_ARG;
  }
  k_unwrap_add<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(n, d_position, d_position_old, d_unwrapped);
  B2_LAUNCHED();
  return B200MD_OK;
}

} // extern "C"

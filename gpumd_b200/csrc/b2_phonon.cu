// b2_phonon.cu -- harmonic phonons: force constants by finite differences, dynamical matrices and their
// eigenvalues, all on the device.
//
//   b200md_phonon_begin / _step   <- Hessian::find_H (src/phonon/hessian.cu:272-302) with find_H12
//                                    (src/force/force_constant.cu:80-133)
//   b200md_phonon_dynamical       <- Hessian::find_dispersion's D(k) sums (hessian.cu:391-419) and find_D
//                                    (hessian.cu:431-458)
//   b200md_phonon_eig             <- eig_hermitian_Jacobi_batch / eig_hermitian_QR (dispersion) and
//                                    eigenvectors_symmetric_Jacobi (one k-point), hessian.cu:347-374,460-492
//
// The reference displaces every neighbour n2 of a basis atom n1 and reads back F_n1 (6 force calls per pair,
// each followed by three blocking copies).  Here the basis atom n1 is displaced by -d and +d along a; one
// force call then gives -dF_n2^b/du_n1^a for every n2 at once, which for a conservative force field is the
// reference's H[n1][n2][a*3+b].  That is 6 * num_basis force calls in all.  Between two force calls runs one
// kernel (k_sweep): it keeps F(-), or writes (F(-) - F(+)) / 2d into H, and moves the next atom; the
// displaced coordinate is always set from a saved copy of the positions, which the last step restores
// entirely.  Nothing synchronises with the host inside the sweep.
//
// The eigensolver is a cyclic Jacobi method with the round-robin parallel ordering, one CTA per matrix and
// the matrix in shared memory: Hermitian (eigenvalues only) or real symmetric (with eigenvectors), up to
// dim = 96.  Eigenvalues come out in ascending order, eigenvectors as columns of a column-major matrix.
#include "../../include/b200md.h"
#include "b2_host.h"
#include <cfloat>
#include <cmath>
#include <new>
#include <string>
#include <vector>

namespace b2 {
namespace {

constexpr int BLK = 256;
constexpr int JBLK = 256;          // threads of one eigensolver CTA
constexpr int MAX_DIM = 3 * B200MD_PHONON_MAX_BASIS;
constexpr int MAX_SWEEPS = 40;     // Jacobi sweeps (about 10 reach rounding level at dim 96)

// r12 = x[n2] - x[n1] under the minimum image (Hessian::is_too_far, hessian.cu:255-270) for every
// (basis atom, atom) pair, and the mask of pairs within the phonon cutoff.  Sums and products are rounded
// one by one, as the reference's host code evaluates them.
__global__ void __launch_bounds__(BLK) k_geometry(
  int n, int nb, B2Box box, double cut2, const double* __restrict__ x, double* __restrict__ r12,
  unsigned char* __restrict__ mask)
{
  const long long t = (long long)blockIdx.x * BLK + threadIdx.x;
  if (t >= (long long)nb * n)
    return;
  const int n1 = (int)(t / n), n2 = (int)(t % n);
  const size_t N = (size_t)n;
  double dx = x[n2] - x[n1], dy = x[N + n2] - x[N + n1], dz = x[2 * N + n2] - x[2 * N + n1];
  b2_mic(box, dx, dy, dz);
  const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
  r12[t * 3 + 0] = dx;
  r12[t * 3 + 1] = dy;
  r12[t * 3 + 2] = dz;
  mask[t] = d2 > cut2 ? 0 : 1;
}

// One step of the sweep, after force call `call` (-1: before the first).  Call j displaces basis atom
// j / 6 along a = (j % 6) / 2 by -d (j even) or +d (j odd).  Even calls keep F(-); odd calls write
// H[n1][n2][a*3+b] = (F_n2^b(-) - F_n2^b(+)) / 2d, zero beyond the cutoff.  Thread 0 then sets the position
// of the atom for the next call from the saved copy x0.  After the last call the positions are x0 again.
__global__ void __launch_bounds__(BLK) k_sweep(
  int n, int calls, int call, double d, const double* __restrict__ f, double* __restrict__ fm,
  double* __restrict__ H, const unsigned char* __restrict__ mask, double* __restrict__ x,
  const double* __restrict__ x0)
{
  const int i = blockIdx.x * BLK + threadIdx.x;
  const size_t N = (size_t)n;
  if (call >= 0 && i < n) {
    if ((call & 1) == 0) {
      fm[i] = f[i];
      fm[N + i] = f[N + i];
      fm[2 * N + i] = f[2 * N + i];
    } else {
      const int n1 = call / 6, a = (call % 6) / 2;
      const size_t t = (size_t)n1 * N + i;
      const bool near = mask[t] != 0;
      const double d2 = d * 2;
#pragma unroll
      for (int b = 0; b < 3; ++b)
        H[t * 9 + a * 3 + b] = near ? (fm[b * N + i] - f[b * N + i]) / d2 : 0.0;
    }
  }
  if (call == calls - 1) { // the last call: every position back to the saved copy
    if (i < n) {
      x[i] = x0[i];
      x[N + i] = x0[N + i];
      x[2 * N + i] = x0[2 * N + i];
    }
    return;
  }
  if (i != 0)
    return;
  // the force call wraps the displaced atom into the box, which in a triclinic box can move its other
  // coordinates too: all three are set from the saved copy
  if (call >= 0 && (call & 1)) { // the atom of this pair of calls goes back
    const int n1 = call / 6;
    x[n1] = x0[n1];
    x[N + n1] = x0[N + n1];
    x[2 * N + n1] = x0[2 * N + n1];
  }
  const int next = call + 1, n1 = next / 6, a = (next % 6) / 2;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const size_t k = (size_t)c * N + n1;
    x[k] = c != a ? x0[k] : ((next & 1) ? x0[k] + d : x0[k] + (-d));
  }
}

// D(k) for every k-point (hessian.cu:391-419, or find_D at one k-point without the phase): one thread per
// (k, basis atom b1, basis atom b2) block of 3 x 3 entries, summed over the atoms n2 = b2 + c * nb in
// increasing order.  Column-major in each k-point's dim x dim matrix.
__global__ void __launch_bounds__(BLK) k_dynamical(
  int n, int nb, int nk, int gamma_only, const double* __restrict__ kpt, const double* __restrict__ mass,
  const double* __restrict__ H, const double* __restrict__ r12, const unsigned char* __restrict__ mask,
  double* __restrict__ DR, double* __restrict__ DI)
{
  const int t = blockIdx.x * BLK + threadIdx.x;
  if (t >= nk * nb * nb)
    return;
  const int k = t / (nb * nb), b1 = (t / nb) % nb, b2 = t % nb;
  const double kx = kpt[3 * k], ky = kpt[3 * k + 1], kz = kpt[3 * k + 2];
  const double mf = 1.0 / sqrt(mass[b1] * mass[b2]);
  double re[9], im[9];
#pragma unroll
  for (int e = 0; e < 9; ++e)
    re[e] = im[e] = 0.0;
  for (int n2 = b2; n2 < n; n2 += nb) {
    const size_t p = (size_t)b1 * n + n2;
    if (!mask[p])
      continue;
    const double* h = H + p * 9;
    if (gamma_only) {
#pragma unroll
      for (int e = 0; e < 9; ++e)
        re[e] = __dadd_rn(re[e], __dmul_rn(h[e], mf));
    } else {
      const double* r = r12 + p * 3;
      const double kr = __dadd_rn(__dadd_rn(__dmul_rn(kx, r[0]), __dmul_rn(ky, r[1])), __dmul_rn(kz, r[2]));
      double s, c;
      sincos(kr, &s, &c);
#pragma unroll
      for (int e = 0; e < 9; ++e) {
        re[e] = __dadd_rn(re[e], __dmul_rn(__dmul_rn(h[e], c), mf));
        im[e] = __dadd_rn(im[e], __dmul_rn(__dmul_rn(h[e], s), mf));
      }
    }
  }
  const int dim = 3 * nb;
  const size_t off = (size_t)k * dim * dim;
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const size_t idx = off + (size_t)(b2 * 3 + b) * dim + b1 * 3 + a;
      DR[idx] = re[a * 3 + b];
      if (!gamma_only)
        DI[idx] = im[a * 3 + b];
    }
}

// Cyclic Jacobi, one CTA per dim x dim matrix.  Input: the lower triangle of a column-major matrix (real
// part re, imaginary part im when CPLX), mirrored into a full Hermitian matrix in shared memory.  Each round
// of a sweep rotates dim/2 disjoint pairs (p, q) of the round-robin ordering at once: the rotation
// J = [[c, s e^{i phi}], [-s e^{-i phi}, c]] on (p, q), phi the phase of A_pq, annihilates A_pq; the rows are
// rotated, then the columns (and the eigenvector columns), then A_pq is set to zero.  A pair is skipped
// when |A_pq| <= eps sqrt(|A_pp A_qq|) or |A_pq| <= 1e-18 ||A||_F; the sweeps stop when a sweep rotates
// nothing.  w: eigenvalues ascending; v (VEC): the eigenvectors as columns, column-major; info: the sweeps
// taken, or -1 when MAX_SWEEPS sweeps still rotated (not converged).
template <bool CPLX, bool VEC>
__global__ void __launch_bounds__(JBLK) k_jacobi(
  int dim, const double* __restrict__ are, const double* __restrict__ aim, double* __restrict__ w,
  double* __restrict__ v, int* __restrict__ info)
{
  extern __shared__ double sm[];
  double* A = sm;             // real part, row-major
  double* B = sm + dim * dim; // imaginary part (CPLX) or the eigenvectors (VEC), row-major
  __shared__ double pc[MAX_DIM / 2], psr[MAX_DIM / 2], psi[MAX_DIM / 2], red[JBLK / 32];
  __shared__ int pp[MAX_DIM / 2], pq[MAX_DIM / 2];
  __shared__ int rotated;
  __shared__ double floor_abs;
  const size_t off = (size_t)blockIdx.x * dim * dim;
  const int dd = dim * dim;
  double norm2 = 0.0;
  for (int t = threadIdx.x; t < dd; t += JBLK) {
    const int r = t % dim, c = t / dim; // element (r, c) of the column-major input
    if (r >= c) {
      const double x = are[off + t], y = (CPLX && r != c) ? aim[off + t] : 0.0;
      A[r * dim + c] = x;
      A[c * dim + r] = x;
      if (CPLX) {
        B[r * dim + c] = y;
        B[c * dim + r] = -y;
      }
      norm2 += (r == c ? 1.0 : 2.0) * (x * x + y * y);
    }
    if (VEC)
      B[t] = r == c ? 1.0 : 0.0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    norm2 += __shfl_down_sync(0xffffffffu, norm2, o);
  if ((threadIdx.x & 31) == 0)
    red[threadIdx.x >> 5] = norm2;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < JBLK / 32; ++k)
      s += red[k];
    floor_abs = 1e-18 * sqrt(s);
  }
  const int m = dim + (dim & 1), half = m / 2;
  int sweeps = -1;
  for (int sweep = 0; sweep < MAX_SWEEPS; ++sweep) {
    if (threadIdx.x == 0)
      rotated = 0;
    __syncthreads();
    for (int round = 0; round < m - 1; ++round) {
      for (int k = threadIdx.x; k < half; k += JBLK) {
        int p = k == 0 ? round : (round + k) % (m - 1);
        int q = k == 0 ? m - 1 : (round - k + m - 1) % (m - 1);
        if (p > q) {
          const int s = p;
          p = q;
          q = s;
        }
        int rp = -1;
        if (q < dim) {
          const double xr = A[p * dim + q], xi = CPLX ? B[p * dim + q] : 0.0;
          const double r = CPLX ? hypot(xr, xi) : fabs(xr);
          const double app = A[p * dim + p], aqq = A[q * dim + q];
          if (r > floor_abs && r > DBL_EPSILON * sqrt(fabs(app) * fabs(aqq))) {
            const double theta = (aqq - app) / (2.0 * r);
            const double tn = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(1.0 + theta * theta));
            const double c = 1.0 / sqrt(1.0 + tn * tn), s = tn * c;
            pc[k] = c;
            psr[k] = s * (xr / r);
            psi[k] = CPLX ? s * (xi / r) : 0.0;
            rp = p;
            rotated = 1;
          }
        }
        pp[k] = rp;
        pq[k] = q;
      }
      __syncthreads();
      // rows: A_pj <- c A_pj - s e^{i phi} A_qj,  A_qj <- s e^{-i phi} A_pj + c A_qj
      for (int t = threadIdx.x; t < half * dim; t += JBLK) {
        const int k = t / dim, j = t % dim, p = pp[k];
        if (p < 0)
          continue;
        const int q = pq[k];
        const double c = pc[k], sr = psr[k], si = psi[k];
        const double ar = A[p * dim + j], br = A[q * dim + j];
        if (CPLX) {
          const double ai = B[p * dim + j], bi = B[q * dim + j];
          A[p * dim + j] = c * ar - (sr * br - si * bi);
          B[p * dim + j] = c * ai - (sr * bi + si * br);
          A[q * dim + j] = (sr * ar + si * ai) + c * br;
          B[q * dim + j] = (sr * ai - si * ar) + c * bi;
        } else {
          A[p * dim + j] = c * ar - sr * br;
          A[q * dim + j] = sr * ar + c * br;
        }
      }
      __syncthreads();
      // columns: A_ip <- c A_ip - s e^{-i phi} A_iq,  A_iq <- s e^{i phi} A_ip + c A_iq  (and V <- V J)
      for (int t = threadIdx.x; t < half * dim; t += JBLK) {
        const int k = t / dim, i = t % dim, p = pp[k];
        if (p < 0)
          continue;
        const int q = pq[k];
        const double c = pc[k], sr = psr[k], si = psi[k];
        const double ar = A[i * dim + p], br = A[i * dim + q];
        if (CPLX) {
          const double ai = B[i * dim + p], bi = B[i * dim + q];
          A[i * dim + p] = c * ar - (sr * br + si * bi);
          B[i * dim + p] = c * ai - (sr * bi - si * br);
          A[i * dim + q] = (sr * ar - si * ai) + c * br;
          B[i * dim + q] = (sr * ai + si * ar) + c * bi;
        } else {
          A[i * dim + p] = c * ar - sr * br;
          A[i * dim + q] = sr * ar + c * br;
          if (VEC) {
            const double vp = B[i * dim + p], vq = B[i * dim + q];
            B[i * dim + p] = c * vp - sr * vq;
            B[i * dim + q] = sr * vp + c * vq;
          }
        }
      }
      __syncthreads();
      for (int k = threadIdx.x; k < half; k += JBLK) {
        const int p = pp[k];
        if (p < 0)
          continue;
        const int q = pq[k];
        A[p * dim + q] = A[q * dim + p] = 0.0;
        if (CPLX)
          B[p * dim + q] = B[q * dim + p] = B[p * dim + p] = B[q * dim + q] = 0.0;
      }
      __syncthreads();
    }
    const int any = rotated;
    __syncthreads();
    if (!any) {
      sweeps = sweep + 1;
      break;
    }
  }
  if (threadIdx.x == 0)
    info[blockIdx.x] = sweeps;
  // ascending order; equal values keep their index order
  for (int i = threadIdx.x; i < dim; i += JBLK) {
    const double di = A[i * dim + i];
    int rank = 0;
    for (int j = 0; j < dim; ++j) {
      const double dj = A[j * dim + j];
      rank += (dj < di || (dj == di && j < i)) ? 1 : 0;
    }
    w[(size_t)blockIdx.x * dim + rank] = di;
    if (VEC)
      for (int r = 0; r < dim; ++r)
        v[off + (size_t)rank * dim + r] = B[r * dim + i];
  }
}

template <bool CPLX, bool VEC>
int launch_jacobi(
  int dim, int batch, const double* re, const double* im, double* w, double* v, int* info, cudaStream_t st)
{
  const size_t smem = (size_t)((CPLX || VEC) ? 2 : 1) * dim * dim * sizeof(double);
  B2_CUDA(cudaFuncSetAttribute(k_jacobi<CPLX, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_jacobi<CPLX, VEC><<<batch, JBLK, smem, st>>>(dim, re, im, w, v, info);
  B2_LAUNCHED();
  return B200MD_OK;
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_phonon {
  int n = 0, nb = 0, nk = 0, calls = 0, next = 0;
  double d = 0.0;
  DevBuf<double> H, r12, fm, x0, kpt, mass, DR, DI, W, V;
  DevBuf<unsigned char> mask;
  DevBuf<int> info;
};

extern "C" {

int b200md_jacobi_eig(
  int dim, int batch, int hermitian, const double* d_re, const double* d_im, double* d_w, double* d_v,
  int* d_info, void* stream)
{
  if (dim < 1 || dim > MAX_DIM || batch < 1 || !d_re || !d_w || !d_info || (hermitian && (!d_im || d_v)) ||
      (hermitian != 0 && hermitian != 1)) {
    set_error("b200md_jacobi_eig: 1 <= dim <= 96, batch >= 1, d_info given; hermitian 1 needs the imaginary "
              "parts and gives no eigenvectors");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (hermitian)
    return launch_jacobi<true, false>(dim, batch, d_re, d_im, d_w, nullptr, d_info, st);
  if (d_v)
    return launch_jacobi<false, true>(dim, batch, d_re, nullptr, d_w, d_v, d_info, st);
  return launch_jacobi<false, false>(dim, batch, d_re, nullptr, d_w, nullptr, d_info, st);
}

int b200md_phonon_create(
  int n, int num_basis, int num_kpoints, const double* kpoints, double displacement, b200md_phonon** out)
{
  if (!out || n <= 0 || num_basis < 1 || num_basis > B200MD_PHONON_MAX_BASIS || num_basis > n ||
      num_kpoints < 1 || !kpoints || !(displacement > 0.0) || 9LL * num_basis * n > (1LL << 40)) {
    set_error("b200md_phonon_create: n > 0, 1 <= num_basis <= 32 and <= n, num_kpoints >= 1 with their "
              "coordinates, displacement > 0");
    return B200MD_ERR_ARG;
  }
  b200md_phonon* p = new (std::nothrow) b200md_phonon;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->n = n;
  p->nb = num_basis;
  p->nk = num_kpoints;
  p->calls = 6 * num_basis;
  p->next = -1;
  p->d = displacement;
  const size_t N = (size_t)n, pairs = (size_t)num_basis * N, dim = 3 * (size_t)num_basis;
  const size_t nd = dim * dim * (size_t)num_kpoints;
  cudaError_t e = p->H.reserve(pairs * 9);
  if (e == cudaSuccess)
    e = p->r12.reserve(pairs * 3);
  if (e == cudaSuccess)
    e = p->mask.reserve(pairs);
  if (e == cudaSuccess)
    e = p->fm.reserve(3 * N);
  if (e == cudaSuccess)
    e = p->x0.reserve(3 * N);
  if (e == cudaSuccess)
    e = p->kpt.reserve(3 * (size_t)num_kpoints);
  if (e == cudaSuccess)
    e = p->mass.reserve(num_basis);
  if (e == cudaSuccess)
    e = p->DR.reserve(nd);
  if (e == cudaSuccess && num_kpoints > 1)
    e = p->DI.reserve(nd);
  if (e == cudaSuccess)
    e = p->W.reserve(dim * num_kpoints);
  if (e == cudaSuccess && num_kpoints == 1)
    e = p->V.reserve(dim * dim);
  if (e == cudaSuccess)
    e = p->info.reserve(num_kpoints);
  if (e == cudaSuccess)
    e = cudaMemcpy(p->kpt.p, kpoints, 3 * (size_t)num_kpoints * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error(std::string("b200md_phonon_create: ") + cudaGetErrorString(e));
    delete p;
    return B200MD_ERR_CUDA;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_phonon_destroy(b200md_phonon* p) { delete p; }

int b200md_phonon_begin(
  b200md_phonon* p, int n, const double h[9], const int pbc[3], double cutoff, double* d_position,
  const double* d_mass, void* stream)
{
  if (!p || n != p->n || !h || !pbc || !d_position || !d_mass || !(cutoff > 0.0)) {
    set_error("b200md_phonon_begin: null argument, cutoff <= 0, or atom count differs from creation");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = (size_t)n;
  B2_CUDA(cudaMemcpyAsync(p->x0.p, d_position, 3 * N * sizeof(double), cudaMemcpyDeviceToDevice, st));
  B2_CUDA(cudaMemcpyAsync(p->mass.p, d_mass, p->nb * sizeof(double), cudaMemcpyDeviceToDevice, st));
  k_geometry<<<grid_for((long long)p->nb * n, BLK), BLK, 0, st>>>(
    n, p->nb, make_box(h, pbc), cutoff * cutoff, d_position, p->r12.p, p->mask.p);
  B2_LAUNCHED();
  k_sweep<<<grid_for(n, BLK), BLK, 0, st>>>(
    n, p->calls, -1, p->d, nullptr, p->fm.p, p->H.p, p->mask.p, d_position, p->x0.p);
  B2_LAUNCHED();
  p->next = 0;
  return B200MD_OK;
}

int b200md_phonon_step(b200md_phonon* p, int call, double* d_position, const double* d_force, void* stream)
{
  if (!p || call != p->next || call < 0 || call >= p->calls || !d_position || !d_force) {
    set_error("b200md_phonon_step: calls must follow b200md_phonon_begin in order 0 .. 6 num_basis - 1");
    return B200MD_ERR_ARG;
  }
  k_sweep<<<grid_for(p->n, BLK), BLK, 0, (cudaStream_t)stream>>>(
    p->n, p->calls, call, p->d, d_force, p->fm.p, p->H.p, p->mask.p, d_position, p->x0.p);
  B2_LAUNCHED();
  p->next = call + 1 < p->calls ? call + 1 : -1;
  return B200MD_OK;
}

int b200md_phonon_dynamical(b200md_phonon* p, void* stream)
{
  if (!p) {
    set_error("b200md_phonon_dynamical: null handle");
    return B200MD_ERR_ARG;
  }
  k_dynamical<<<grid_for((long long)p->nk * p->nb * p->nb, BLK), BLK, 0, (cudaStream_t)stream>>>(
    p->n, p->nb, p->nk, p->nk == 1, p->kpt.p, p->mass.p, p->H.p, p->r12.p, p->mask.p, p->DR.p, p->DI.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_phonon_eig(b200md_phonon* p, void* stream)
{
  if (!p) {
    set_error("b200md_phonon_eig: null handle");
    return B200MD_ERR_ARG;
  }
  const int dim = 3 * p->nb;
  const int rc = p->nk == 1 ? b200md_jacobi_eig(dim, 1, 0, p->DR.p, nullptr, p->W.p, p->V.p, p->info.p, stream)
                            : b200md_jacobi_eig(dim, p->nk, 1, p->DR.p, p->DI.p, p->W.p, nullptr, p->info.p, stream);
  if (rc != B200MD_OK)
    return rc;
  // the end of the calculation: one synchronisation to report a matrix the sweeps did not diagonalise
  std::vector<int> info(p->nk);
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(cudaMemcpyAsync(info.data(), p->info.p, p->nk * sizeof(int), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  for (int k = 0; k < p->nk; ++k)
    if (info[k] < 0) {
      set_error("b200md_phonon_eig: the Jacobi eigensolver did not converge in " + std::to_string(MAX_SWEEPS) +
                " sweeps at k-point " + std::to_string(k));
      return B200MD_ERR_NOT_CONVERGED;
    }
  return B200MD_OK;
}

int b200md_phonon_read(b200md_phonon* p, int what, double* host, void* stream)
{
  if (!p || !host || what < B200MD_PHONON_H || what > B200MD_PHONON_V ||
      (what == B200MD_PHONON_D_IMAG && p->nk == 1) || (what == B200MD_PHONON_V && p->nk != 1)) {
    set_error("b200md_phonon_read: null argument, or an array this calculation does not have (the imaginary "
              "part of D with one k-point, eigenvectors with more)");
    return B200MD_ERR_ARG;
  }
  const size_t dim = 3 * (size_t)p->nb, n9 = (size_t)p->nb * p->n * 9, nd = dim * dim * p->nk;
  const double* src[] = {p->H.p, p->DR.p, p->DI.p, p->W.p, p->V.p};
  const size_t count[] = {n9, nd, nd, dim * p->nk, dim * dim};
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(cudaMemcpyAsync(host, src[what], count[what] * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return B200MD_OK;
}

} // extern "C"

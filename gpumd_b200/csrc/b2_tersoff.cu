// b2_tersoff.cu -- Tersoff-1989 potential (FP64) and the per-atom heat current of libb200md;
// C-ABI entry points b200md_tersoff_*, b200md_compute_heat.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_neighbor_host.h"
#include "b2_nep.cuh" // b2_body_unpack
#include "b2_tersoff.cuh"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

namespace b2 {
namespace {

__global__ void __launch_bounds__(64) k_tersoff_partial(B2TersoffView P, B2Box box)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_tersoff_partial(i, P, box);
}

__global__ void __launch_bounds__(128) k_tersoff_reduce(B2TersoffView P, B2Box box)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_tersoff_reduce(i, P, box);
}

__global__ void __launch_bounds__(256) k_unpack_t(
  int n, const int* __restrict__ perm, const double* __restrict__ acc, double* pe, double* force,
  double* virial)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    b2_body_unpack(i, n, perm, acc, pe, force, virial);
}

__global__ void __launch_bounds__(256) k_heat(
  int n, int stride, const double* __restrict__ w, const double* __restrict__ v, double* heat,
  int hstride)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    b2_body_heat(i, stride, w, v, heat, hstride);
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_tersoff {
  int nt = 0, n = 0;
  double rc = 0.0;
  std::vector<std::string> symbols;
  Neighbor nb;
  DevBuf<int> nn, nl;
  DevBuf<double> f12, acc;
  B2TersoffView view;
};

#define B2_TRY(expr)        \
  do {                      \
    const int rc_ = (expr); \
    if (rc_ != B200MD_OK)   \
      return rc_;           \
  } while (0)

extern "C" {

int b200md_tersoff_create(const char* path, int num_atoms, b200md_tersoff** out)
{
  if (!path || !out || num_atoms <= 0) {
    set_error("b200md_tersoff_create: bad argument");
    return B200MD_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("b200md_tersoff_create: no CUDA device (libb200md has no CPU fallback)");
    return B200MD_ERR_CUDA;
  }
  TersoffFile file;
  const std::string err = load_tersoff(path, file);
  if (!err.empty())
    return load_error(err);
  b200md_tersoff* p = new (std::nothrow) b200md_tersoff;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->nt = file.nt;
  p->symbols = file.symbols;
  p->rc = file.rc;
  p->n = num_atoms;
  const size_t N = (size_t)num_atoms;
  int rc = p->nb.init(num_atoms, p->rc, file.mn_skin);
  if (rc != B200MD_OK) {
    delete p;
    return rc;
  }
  if (p->nn.reserve(N) != cudaSuccess || p->nl.reserve(N * B2_TERSOFF_MAXL) != cudaSuccess ||
      p->f12.reserve(3 * N * B2_TERSOFF_MAXL) != cudaSuccess ||
      p->acc.reserve(13 * N) != cudaSuccess) {
    delete p;
    set_error("out of device memory");
    return B200MD_ERR_CUDA;
  }
  B2TersoffView& P = p->view;
  P = file.view;
  P.n = num_atoms;
  P.atoms = p->nb.atoms.p;
  P.nn_skin = p->nb.nn_skin.p;
  P.nl_skin = p->nb.nl_skin.p;
  P.nn = p->nn.p;
  P.nl = p->nl.p;
  P.f12 = p->f12.p;
  P.acc = p->acc.p;
  P.flags = p->nb.flags.p;
  cudaDeviceSynchronize();
  *out = p;
  return B200MD_OK;
}

void b200md_tersoff_destroy(b200md_tersoff* p) { delete p; }
double b200md_tersoff_rc(const b200md_tersoff* p) { return p->rc; }
const char* b200md_tersoff_symbol(const b200md_tersoff* p, int t)
{
  return (t >= 0 && t < p->nt) ? p->symbols[t].c_str() : "";
}
int b200md_tersoff_info(const b200md_tersoff* p, int what)
{
  if (what == 0)
    return p->nt;
  if (what == 6) {
    int bits = 0, rebuilds = 0;
    const_cast<b200md_tersoff*>(p)->nb.check(0, &bits, &rebuilds);
    return rebuilds;
  }
  return -1;
}

int b200md_tersoff_compute(
  b200md_tersoff* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  const B2Box box = make_box(h, pbc);
  B2_TRY(p->nb.update(box, d_type, d_position, n, st));
  p->n = n;
  p->view.n = n;
  k_tersoff_partial<<<grid_for(n, 64), 64, 0, st>>>(p->view, box);
  B2_LAUNCHED();
  k_tersoff_reduce<<<grid_for(n, 128), 128, 0, st>>>(p->view, box);
  B2_LAUNCHED();
  k_unpack_t<<<grid_for(n, 256), 256, 0, st>>>(
    n, p->nb.perm.p, p->acc.p, d_potential, d_force, d_virial);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_tersoff_invalidate(b200md_tersoff* p, int n_new, void* stream)
{
  B2_TRY(p->nb.invalidate(n_new, (cudaStream_t)stream));
  p->n = n_new;
  p->view.n = n_new;
  return B200MD_OK;
}

int b200md_tersoff_check(b200md_tersoff* p, void* stream)
{
  int bits = 0, rebuilds = 0;
  B2_TRY(p->nb.check((cudaStream_t)stream, &bits, &rebuilds));
  if (bits) {
    set_error("Tersoff neighbour capacity exceeded on the device (skin list or 32 local neighbours)");
    return B200MD_ERR_OVERFLOW;
  }
  return B200MD_OK;
}

int b200md_compute_heat(
  int n, int stride, const double* d_virial, const double* d_velocity, double* d_heat,
  int heat_stride, void* stream)
{
  k_heat<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(
    n, stride, d_virial, d_velocity, d_heat, heat_stride);
  B2_LAUNCHED();
  return B200MD_OK;
}

} // extern "C"

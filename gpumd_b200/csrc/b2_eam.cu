// b2_eam.cu -- analytic EAM potentials (Zhou-2004 alloy form, Dai-2006) of libb200md;
// C-ABI entry points b200md_eam_*.
#include "../../include/b200md.h"
#include "b2_eam.cuh"
#include "b2_host.h"
#include "b2_neighbor_host.h"
#include "b2_nep.cuh" // b2_body_unpack
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <vector>

namespace b2 {
namespace {

__global__ void __launch_bounds__(128) k_eam_density(B2EamView P, B2Box box)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_eam_density(i, P, box);
}

__global__ void __launch_bounds__(128) k_eam_force(B2EamView P, B2Box box)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_eam_force(i, P, box);
}

__global__ void __launch_bounds__(256) k_unpack_e(
  int n, const int* __restrict__ perm, const double* __restrict__ acc, double* pe, double* force,
  double* virial)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    b2_body_unpack(i, n, perm, acc, pe, force, virial);
}

} // namespace
} // namespace b2

using namespace b2;

struct b200md_eam {
  int nt = 0, n = 0, model = 0;
  double rc = 0.0;
  std::vector<std::string> symbols;
  Neighbor nb;
  DevBuf<float> zp, Fp;
  DevBuf<double> acc;
  B2EamView view;
};

#define B2_TRY(expr)        \
  do {                      \
    const int rc_ = (expr); \
    if (rc_ != B200MD_OK)   \
      return rc_;           \
  } while (0)

extern "C" {

int b200md_eam_create(const char* path, int num_atoms, b200md_eam** out)
{
  if (!path || !out || num_atoms <= 0) {
    set_error("b200md_eam_create: bad argument");
    return B200MD_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("b200md_eam_create: no CUDA device (libb200md has no CPU fallback)");
    return B200MD_ERR_CUDA;
  }
  EamFile file;
  const std::string err = load_eam(path, file);
  if (!err.empty())
    return load_error(err);
  b200md_eam* p = new (std::nothrow) b200md_eam;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  p->nt = file.nt;
  p->model = file.view.model;
  p->symbols = file.symbols;
  p->rc = file.rc;
  p->n = num_atoms;
  const size_t N = (size_t)num_atoms;
  int r = p->nb.init(num_atoms, file.rc, file.mn_skin);
  if (r != B200MD_OK) {
    delete p;
    return r;
  }
  if (p->zp.reserve(file.zp.size()) != cudaSuccess || p->Fp.reserve(N) != cudaSuccess ||
      p->acc.reserve(13 * N) != cudaSuccess) {
    delete p;
    set_error("out of device memory");
    return B200MD_ERR_CUDA;
  }
  cudaMemcpy(p->zp.p, file.zp.data(), sizeof(float) * file.zp.size(), cudaMemcpyHostToDevice);
  B2EamView& P = p->view;
  P = file.view;
  P.zp = p->zp.p;
  P.n = num_atoms;
  P.atoms = p->nb.atoms.p;
  P.nn_skin = p->nb.nn_skin.p;
  P.nl_skin = p->nb.nl_skin.p;
  P.Fp = p->Fp.p;
  P.acc = p->acc.p;
  cudaDeviceSynchronize();
  *out = p;
  return B200MD_OK;
}

void b200md_eam_destroy(b200md_eam* p) { delete p; }
double b200md_eam_rc(const b200md_eam* p) { return p->rc; }
const char* b200md_eam_symbol(const b200md_eam* p, int t)
{
  return (t >= 0 && t < p->nt) ? p->symbols[t].c_str() : "";
}
int b200md_eam_info(const b200md_eam* p, int what)
{
  if (what == 0)
    return p->nt;
  if (what == 6) {
    int bits = 0, rebuilds = 0;
    const_cast<b200md_eam*>(p)->nb.check(0, &bits, &rebuilds);
    return rebuilds;
  }
  return -1;
}

int b200md_eam_compute(
  b200md_eam* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  const B2Box box = make_box(h, pbc);
  B2_TRY(p->nb.update(box, d_type, d_position, n, st));
  p->n = n;
  p->view.n = n;
  k_eam_density<<<grid_for(n, 128), 128, 0, st>>>(p->view, box);
  B2_LAUNCHED();
  k_eam_force<<<grid_for(n, 128), 128, 0, st>>>(p->view, box);
  B2_LAUNCHED();
  k_unpack_e<<<grid_for(n, 256), 256, 0, st>>>(
    n, p->nb.perm.p, p->acc.p, d_potential, d_force, d_virial);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_eam_invalidate(b200md_eam* p, int n_new, void* stream)
{
  B2_TRY(p->nb.invalidate(n_new, (cudaStream_t)stream));
  p->n = n_new;
  p->view.n = n_new;
  return B200MD_OK;
}

int b200md_eam_check(b200md_eam* p, void* stream)
{
  int bits = 0, rebuilds = 0;
  B2_TRY(p->nb.check((cudaStream_t)stream, &bits, &rebuilds));
  if (bits) {
    set_error("EAM neighbour-list capacity exceeded on the device");
    return B200MD_ERR_OVERFLOW;
  }
  return B200MD_OK;
}

} // extern "C"

// b2_mgpu.cu -- libb200md_mgpu.so: block / slab domain decomposition of the MD hot path in C++,
// CUDA and NCCL (see include/b200md_mgpu.h for the design and what it replaces).  A client of the
// libb200md C-ABI: potentials, integrator kernels and thermo are the single-GPU entry points acting
// on the owned part of one set of local SoA arrays [owned | ghosts].
//
// Local frame of a domain with grid coordinate c_d in a decomposed direction d (P_d > 1):
//   x_local = x_global - (c_d * w_d - halo),  w_d = L_d / P_d
// so owned atoms sit in [halo, halo + w_d), ghosts in [0, halo) and [halo + w_d, w_d + 2 halo), and
// the local box is open along d.  Neighbouring frames differ by exactly +-w_d (periodic wrap
// included), so a position sent to the lower neighbour is shifted by +w_d, to the upper one by -w_d.
// Undecomposed directions keep the global length and periodicity.
//
// Ghosts are exchanged in stages x, y, z; stage d selects among the owned atoms AND the ghosts of
// the earlier stages, which is what carries edge and corner ghosts without diagonal messages.
#include "../../include/b200md.h"
#include "../../include/b200md_mgpu.h"
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <nccl.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <vector>

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg)
{
  g_err = msg;
  return code;
}

#define MG_CUDA(call)                                                                        \
  do {                                                                                       \
    const cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess)                                                                   \
      return fail(B200MD_ERR_CUDA, std::string("CUDA error ") + cudaGetErrorString(e_) +     \
                                     " in " #call);                                          \
  } while (0)
#define MG_NCCL(call)                                                                        \
  do {                                                                                       \
    const ncclResult_t r_ = (call);                                                          \
    if (r_ != ncclSuccess)                                                                   \
      return fail(B200MD_ERR_CUDA, std::string("NCCL error ") + ncclGetErrorString(r_) +     \
                                     " in " #call);                                          \
  } while (0)
#define MG_B2(call)                                                                          \
  do {                                                                                       \
    const int r_ = (call);                                                                   \
    if (r_ != B200MD_OK)                                                                     \
      return fail(r_, std::string(b200md_last_error()) + " (" #call ")");                    \
  } while (0)
#define MG_TRY(call)          \
  do {                        \
    const int r_ = (call);    \
    if (r_ != B200MD_OK)      \
      return r_;              \
  } while (0)

template <typename T>
struct DBuf {
  T* p = nullptr;
  size_t n = 0;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  ~DBuf() { release(); }
  void release()
  {
    if (p)
      cudaFree(p);
    p = nullptr;
    n = 0;
  }
  cudaError_t reserve(size_t count) // grows only, contents not preserved
  {
    if (count <= n)
      return cudaSuccess;
    release();
    const cudaError_t e = cudaMalloc((void**)&p, (count ? count : 1) * sizeof(T));
    if (e == cudaSuccess)
      n = count;
    return e;
  }
};

constexpr int BLK = 256;
inline int grid_for(long long n, int b) { return (int)((n + b - 1) / b); }
long long g_own_launches = 0; // kernels launched by this module (libb200md counts its own)
#define MG_COUNT() (++g_own_launches)

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
// flags for the three destinations of stage `d`: lo[i] = coordinate < lo_edge, hi[i] = >= hi_edge
__global__ void __launch_bounds__(BLK) k_flag_faces(
  int m, const double* __restrict__ coord, double lo_edge, double hi_edge, char* lo, char* hi, char* stay)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) {
    const double c = coord[i];
    const char l = c < lo_edge, h = c >= hi_edge;
    lo[i] = l;
    hi[i] = h;
    if (stay)
      stay[i] = !(l | h);
  }
}

// out[r*m + k] = in[r*stride + idx[k]] (+ shift on row `shift_row`), r < rows
__global__ void __launch_bounds__(BLK) k_gather_rows(
  int m, int rows, const int* __restrict__ idx, int stride, const double* __restrict__ in, int shift_row,
  double shift, double* out)
{
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < (long long)m * rows) {
    const int r = (int)(e / m), k = (int)(e - (long long)r * m);
    double v = in[(size_t)r * stride + idx[k]];
    if (r == shift_row)
      v += shift;
    out[e] = v;
  }
}

// out[r*out_stride + out_off + k] = in[r*m + k]
__global__ void __launch_bounds__(BLK) k_scatter_rows(
  int m, int rows, const double* __restrict__ in, int out_stride, int out_off, double* out)
{
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < (long long)m * rows) {
    const int r = (int)(e / m), k = (int)(e - (long long)r * m);
    out[(size_t)r * out_stride + out_off + k] = in[e];
  }
}

__global__ void __launch_bounds__(BLK) k_int_to_double(int m, const int* in, double* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m)
    out[i] = (double)in[i];
}
__global__ void __launch_bounds__(BLK) k_ll_to_double(int m, const long long* in, double* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m)
    out[i] = (double)in[i];
}
__global__ void __launch_bounds__(BLK) k_double_to_int(int m, const double* in, int* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m)
    out[i] = (int)in[i];
}
__global__ void __launch_bounds__(BLK) k_double_to_ll(int m, const double* in, long long* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m)
    out[i] = (long long)in[i];
}

// largest squared displacement of the owned atoms since the last exchange (minimum image in the
// undecomposed periodic directions, whose coordinates are wrapped every step)
__global__ void __launch_bounds__(BLK) k_max_disp2(
  int n, int stride, const double* __restrict__ pos, const double* __restrict__ ref, double Lx, double Ly,
  double Lz, unsigned int* out_bits)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float d2 = 0.0f;
  if (i < n) {
    const double L[3] = {Lx, Ly, Lz};
    double s = 0.0;
    for (int d = 0; d < 3; ++d) {
      double v = pos[(size_t)d * stride + i] - ref[(size_t)d * n + i];
      if (L[d] > 0.0)
        v -= L[d] * rint(v / L[d]);
      s += v * v;
    }
    d2 = (float)s;
  }
  for (int o = 16; o > 0; o >>= 1)
    d2 = fmaxf(d2, __shfl_xor_sync(0xffffffffu, d2, o));
  if ((threadIdx.x & 31) == 0 && d2 > 0.0f)
    atomicMax(out_bits, __float_as_uint(d2)); // non-negative floats order like their bit patterns
}

__global__ void k_add8(double* acc, const double* in, int n)
{
  const int i = threadIdx.x;
  if (i < n)
    acc[i] += in[i];
}

// ---------------------------------------------------------------------------------------------
// potentials behind one face
// ---------------------------------------------------------------------------------------------
struct Pot {
  int kind = -1; // 0 nep, 1 lj, 2 tersoff_1989, 3 eam
  void* h = nullptr;
  double rc = 0.0;
  bool many_body = true;

  int create(const char* file, int cap)
  {
    std::ifstream in(file);
    if (!in.is_open())
      return fail(B200MD_ERR_IO, std::string("Failed to open ") + file);
    std::string name;
    in >> name;
    if (name.rfind("nep", 0) == 0) {
      kind = 0;
      MG_B2(b200md_nep_create(file, cap, (b200md_nep**)&h));
      MG_B2(b200md_nep_set_accumulate((b200md_nep*)h, 0));
      rc = b200md_nep_rc((b200md_nep*)h);
    } else if (name == "lj") {
      kind = 1;
      many_body = false;
      MG_B2(b200md_lj_create(file, cap, (b200md_lj**)&h));
      rc = b200md_lj_rc((b200md_lj*)h);
    } else if (name == "tersoff_1989") {
      kind = 2;
      MG_B2(b200md_tersoff_create(file, cap, (b200md_tersoff**)&h));
      rc = b200md_tersoff_rc((b200md_tersoff*)h);
    } else if (name == "eam_zhou_2004" || name == "eam_dai_2006") {
      kind = 3;
      MG_B2(b200md_eam_create(file, cap, (b200md_eam**)&h));
      rc = b200md_eam_rc((b200md_eam*)h);
    } else {
      return fail(B200MD_ERR_ARG, "illegal potential model '" + name + "' for the b200md backend");
    }
    return B200MD_OK;
  }
  ~Pot()
  {
    if (!h)
      return;
    switch (kind) {
      case 0: b200md_nep_destroy((b200md_nep*)h); break;
      case 1: b200md_lj_destroy((b200md_lj*)h); break;
      case 2: b200md_tersoff_destroy((b200md_tersoff*)h); break;
      case 3: b200md_eam_destroy((b200md_eam*)h); break;
    }
  }
  int compute(
    int n, const double* lh, const int* lpbc, const int* type, const double* pos, double* pe,
    double* f, double* v, cudaStream_t st)
  {
    switch (kind) {
      case 0: MG_B2(b200md_nep_compute((b200md_nep*)h, n, lh, lpbc, type, pos, pe, f, v, st)); break;
      case 1: MG_B2(b200md_lj_compute((b200md_lj*)h, n, lh, lpbc, type, pos, pe, f, v, st)); break;
      case 2:
        MG_B2(b200md_tersoff_compute((b200md_tersoff*)h, n, lh, lpbc, type, pos, pe, f, v, st));
        break;
      default: MG_B2(b200md_eam_compute((b200md_eam*)h, n, lh, lpbc, type, pos, pe, f, v, st)); break;
    }
    return B200MD_OK;
  }
  int invalidate(int n, cudaStream_t st)
  {
    switch (kind) {
      case 0: MG_B2(b200md_nep_invalidate((b200md_nep*)h, n, st)); break;
      case 1: MG_B2(b200md_lj_invalidate((b200md_lj*)h, n, st)); break;
      case 2: MG_B2(b200md_tersoff_invalidate((b200md_tersoff*)h, n, st)); break;
      default: MG_B2(b200md_eam_invalidate((b200md_eam*)h, n, st)); break;
    }
    return B200MD_OK;
  }
  int set_owned(int n)
  {
    if (kind == 0)
      MG_B2(b200md_nep_set_owned((b200md_nep*)h, n)); // the others compute ghost outputs, unused
    return B200MD_OK;
  }
  int set_active(const double lo[3], const double hi[3])
  {
    if (kind == 0)
      MG_B2(b200md_nep_set_active_region((b200md_nep*)h, lo, hi));
    return B200MD_OK;
  }
  int check(cudaStream_t st)
  {
    switch (kind) {
      case 0: MG_B2(b200md_nep_check((b200md_nep*)h, st)); break;
      case 1: MG_B2(b200md_lj_check((b200md_lj*)h, st)); break;
      case 2: MG_B2(b200md_tersoff_check((b200md_tersoff*)h, st)); break;
      default: MG_B2(b200md_eam_check((b200md_eam*)h, st)); break;
    }
    return B200MD_OK;
  }
  int rebuilds() const
  {
    switch (kind) {
      case 0: return b200md_nep_info((b200md_nep*)h, 6);
      case 1: return b200md_lj_info((b200md_lj*)h, 6);
      case 2: return b200md_tersoff_info((b200md_tersoff*)h, 6);
      default: return b200md_eam_info((b200md_eam*)h, 6);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// one spatial domain
// ---------------------------------------------------------------------------------------------
constexpr int MIG_ROWS = 12; // pos3 vel3 force3 mass type id, all as doubles
constexpr int GHOST_ROWS = 5; // pos3 type mass

struct Stage {
  bool active = false;
  int m_cand = 0;                  // atoms [0, m_cand) of the local order are candidates
  DBuf<int> idx_lo, idx_hi;        // local indices sent to the lower / upper neighbour
  int n_lo = 0, n_hi = 0;          // their counts
  int n_from_hi = 0, n_from_lo = 0; // ghosts received, stored [from_hi | from_lo] at ghost_start
  int ghost_start = 0;
};

struct Domain {
  int rank = 0, c[3] = {0, 0, 0};
  int nb_lo[3], nb_hi[3];
  double origin[3] = {0, 0, 0};
  double lh[9];
  int lpbc[3];
  int cap = 0, n_own = 0, n_loc = 0;
  // main local arrays, stride n_loc
  DBuf<double> pos, vel, force, virial, pe, mass;
  DBuf<int> type;
  DBuf<long long> id;
  // compact owned copies used while the atom set changes (stride n_own) + scratch twins
  DBuf<double> own_d, own_d2; // [MIG_ROWS * cap]
  // candidate arrays while ghosts are collected, stride cap: pos3 type mass as doubles
  DBuf<double> cand;
  DBuf<double> ref; // owned positions at the last exchange [3*n_own]
  Stage st[3];
  // message buffers
  DBuf<double> send_lo, send_hi, recv_hi, recv_lo;
  // selection scratch
  DBuf<char> flag_lo, flag_hi, flag_stay;
  DBuf<int> idx_tmp, count_dev;
  DBuf<unsigned char> cub_tmp;
  size_t cub_bytes = 0;
  Pot pot;
  b200md_nhc* nhc = nullptr;
  b200md_bdp* bdp = nullptr;
  DBuf<double> thermo;
  DBuf<unsigned char> thermo_scratch;
  DBuf<double> heat, heat5;
  DBuf<unsigned int> disp_bits;
  // HNEMD: this block's total of the driven forces (then the global one), its heat-current rows and
  // the ring row the next one goes to, and the scratch of both reductions
  DBuf<double> hn_ftot, hn_rows;
  DBuf<unsigned int> hn_row;
  DBuf<unsigned char> hn_scratch;
  ~Domain()
  {
    if (nhc)
      b200md_nhc_destroy(nhc);
    if (bdp)
      b200md_bdp_destroy(bdp);
  }
};

} // namespace

struct b200md_mgpu {
  b200md_mgpu_config cfg;
  std::string potential_file;
  int world = 1;
  double L[3], w[3], halo = 0.0, volume = 0.0;
  bool distributed = false;
  ncclComm_t comm = nullptr;
  cudaStream_t stream = nullptr;
  std::vector<std::unique_ptr<Domain>> dom; // local domains (1 when distributed, world otherwise)
  long long n_global = 0;
  int migrations = 0;
  int steps_since_exchange = 0;
  DBuf<double> thermo_sum; // local mode: the domains' sums of thermo[8] or of the HNEMD force total
  // HNEMD (b200md_mgpu_hnemd_set): each domain's heat rows form a ring of hn_ring rows; the hn_pending
  // steps sampled since the last take start at ring row hn_first
  bool hn_on = false;
  double hn_fe[3] = {0, 0, 0};
  int hn_oi = 1, hn_max = 0, hn_ring = 0, hn_first = 0;
  long long hn_pending = 0;
  DBuf<double> hn_gather; // distributed: every rank's ring, gathered at take time
  DBuf<int> cnt_dev;
  // profiling
  bool prof = false;
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  double prof_ms[4] = {0, 0, 0, 0};
  int prof_steps = 0;
  // CUDA graph of one step
  cudaGraphExec_t graph = nullptr;
  double graph_dt = 0.0;
  long long launches_per_step = 0; // kernels of one step (this module's + libb200md's)
  cudaEvent_t t0 = nullptr, t1 = nullptr;

  ~b200md_mgpu()
  {
    if (graph)
      cudaGraphExecDestroy(graph);
    dom.clear();
    for (auto& e : ev)
      if (e)
        cudaEventDestroy(e);
    if (t0)
      cudaEventDestroy(t0);
    if (t1)
      cudaEventDestroy(t1);
    if (comm)
      ncclCommDestroy(comm);
    if (stream)
      cudaStreamDestroy(stream);
  }
  Domain* find(int rank)
  {
    for (auto& d : dom)
      if (d->rank == rank)
        return d.get();
    return nullptr;
  }
};

namespace {

using Group = b200md_mgpu;

int rank_of(const int grid[3], int cx, int cy, int cz) { return (cx * grid[1] + cy) * grid[2] + cz; }

// ---- deterministic compaction: indices i in [0, m) with flag[i] != 0, ascending ----
int select(Domain& D, int m, const char* flags, int* out, int* count_host, cudaStream_t st)
{
  cub::CountingInputIterator<int> it(0);
  size_t need = 0;
  MG_CUDA(cub::DeviceSelect::Flagged(nullptr, need, it, flags, out, D.count_dev.p, m, st));
  if (need > D.cub_bytes) {
    MG_CUDA(cudaStreamSynchronize(st));
    MG_CUDA(D.cub_tmp.reserve(need));
    D.cub_bytes = D.cub_tmp.n;
  }
  need = D.cub_bytes;
  if (m > 0)
    MG_CUDA(cub::DeviceSelect::Flagged(D.cub_tmp.p, need, it, flags, out, D.count_dev.p, m, st));
  else
    MG_CUDA(cudaMemsetAsync(D.count_dev.p, 0, sizeof(int), st));
  MG_CUDA(cudaMemcpyAsync(count_host, D.count_dev.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  MG_CUDA(cudaStreamSynchronize(st));
  return B200MD_OK;
}

// ---- message exchange of one stage for all local domains ----
// every domain has filled send_lo (n_lo_rows doubles) / send_hi; sizes to receive are known
struct Msg {
  size_t send_lo = 0, send_hi = 0, recv_hi = 0, recv_lo = 0; // in doubles
};

int exchange_payload(Group& G, int d, const std::vector<Msg>& msg)
{
  cudaStream_t st = G.stream;
  if (G.distributed) {
    Domain& D = *G.dom[0];
    const Msg& m = msg[0];
    MG_NCCL(ncclGroupStart());
    if (m.send_lo)
      MG_NCCL(ncclSend(D.send_lo.p, m.send_lo, ncclDouble, D.nb_lo[d], G.comm, st));
    if (m.send_hi)
      MG_NCCL(ncclSend(D.send_hi.p, m.send_hi, ncclDouble, D.nb_hi[d], G.comm, st));
    if (m.recv_hi)
      MG_NCCL(ncclRecv(D.recv_hi.p, m.recv_hi, ncclDouble, D.nb_hi[d], G.comm, st));
    if (m.recv_lo)
      MG_NCCL(ncclRecv(D.recv_lo.p, m.recv_lo, ncclDouble, D.nb_lo[d], G.comm, st));
    MG_NCCL(ncclGroupEnd());
    return B200MD_OK;
  }
  // local: what I send to my lower neighbour is what it receives from its upper neighbour
  for (size_t k = 0; k < G.dom.size(); ++k) {
    Domain& D = *G.dom[k];
    const Msg& m = msg[k];
    if (m.send_lo) {
      Domain* peer = G.find(D.nb_lo[d]);
      MG_CUDA(cudaMemcpyAsync(
        peer->recv_hi.p, D.send_lo.p, m.send_lo * sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
    if (m.send_hi) {
      Domain* peer = G.find(D.nb_hi[d]);
      MG_CUDA(cudaMemcpyAsync(
        peer->recv_lo.p, D.send_hi.p, m.send_hi * sizeof(double), cudaMemcpyDeviceToDevice, st));
    }
  }
  return B200MD_OK;
}

// counts: every domain tells its two neighbours how many entries follow
int exchange_counts(Group& G, int d, const std::vector<int>& n_lo, const std::vector<int>& n_hi,
                    std::vector<int>& from_hi, std::vector<int>& from_lo)
{
  const size_t K = G.dom.size();
  from_hi.assign(K, 0);
  from_lo.assign(K, 0);
  if (G.distributed) {
    Domain& D = *G.dom[0];
    int h[4] = {n_lo[0], n_hi[0], 0, 0};
    MG_CUDA(G.cnt_dev.reserve(4));
    MG_CUDA(cudaMemcpyAsync(G.cnt_dev.p, h, 2 * sizeof(int), cudaMemcpyHostToDevice, G.stream));
    MG_NCCL(ncclGroupStart());
    MG_NCCL(ncclSend(G.cnt_dev.p, 1, ncclInt, D.nb_lo[d], G.comm, G.stream));
    MG_NCCL(ncclSend(G.cnt_dev.p + 1, 1, ncclInt, D.nb_hi[d], G.comm, G.stream));
    MG_NCCL(ncclRecv(G.cnt_dev.p + 2, 1, ncclInt, D.nb_hi[d], G.comm, G.stream));
    MG_NCCL(ncclRecv(G.cnt_dev.p + 3, 1, ncclInt, D.nb_lo[d], G.comm, G.stream));
    MG_NCCL(ncclGroupEnd());
    MG_CUDA(cudaMemcpyAsync(h + 2, G.cnt_dev.p + 2, 2 * sizeof(int), cudaMemcpyDeviceToHost, G.stream));
    MG_CUDA(cudaStreamSynchronize(G.stream));
    from_hi[0] = h[2];
    from_lo[0] = h[3];
    return B200MD_OK;
  }
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    for (size_t q = 0; q < K; ++q) {
      if (G.dom[q]->rank == D.nb_hi[d])
        from_hi[k] = n_lo[q]; // my upper neighbour's "to lower" message
      if (G.dom[q]->rank == D.nb_lo[d])
        from_lo[k] = n_hi[q];
    }
  }
  return B200MD_OK;
}

int reserve_msg(Domain& D, size_t s_lo, size_t s_hi, size_t r_hi, size_t r_lo, cudaStream_t st)
{
  if (s_lo > D.send_lo.n || s_hi > D.send_hi.n || r_hi > D.recv_hi.n || r_lo > D.recv_lo.n) {
    MG_CUDA(cudaStreamSynchronize(st));
    MG_CUDA(D.send_lo.reserve(s_lo + s_lo / 4 + 64));
    MG_CUDA(D.send_hi.reserve(s_hi + s_hi / 4 + 64));
    MG_CUDA(D.recv_hi.reserve(r_hi + r_hi / 4 + 64));
    MG_CUDA(D.recv_lo.reserve(r_lo + r_lo / 4 + 64));
  }
  return B200MD_OK;
}

// ---------------------------------------------------------------------------------------------
// migration + ghost lists (rare; a few host synchronisations for the message sizes)
// ---------------------------------------------------------------------------------------------
// own_d rows: 0-2 pos, 3-5 vel, 6-8 force, 9 mass, 10 type, 11 id; stride = n_own
int sync_owned(Group& G, Domain& D)
{
  cudaStream_t st = G.stream;
  const int n = D.n_own, s = D.n_loc;
  if (n == 0)
    return B200MD_OK;
  for (int r = 0; r < 3; ++r) {
    MG_CUDA(cudaMemcpyAsync(D.own_d.p + (size_t)r * n, D.pos.p + (size_t)r * s, sizeof(double) * n,
                            cudaMemcpyDeviceToDevice, st));
    MG_CUDA(cudaMemcpyAsync(D.own_d.p + (size_t)(3 + r) * n, D.vel.p + (size_t)r * s,
                            sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
    MG_CUDA(cudaMemcpyAsync(D.own_d.p + (size_t)(6 + r) * n, D.force.p + (size_t)r * s,
                            sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
  }
  MG_CUDA(cudaMemcpyAsync(D.own_d.p + (size_t)9 * n, D.mass.p, sizeof(double) * n,
                          cudaMemcpyDeviceToDevice, st));
  k_int_to_double<<<grid_for(n, BLK), BLK, 0, st>>>(n, D.type.p, D.own_d.p + (size_t)10 * n); MG_COUNT();
  k_ll_to_double<<<grid_for(n, BLK), BLK, 0, st>>>(n, D.id.p, D.own_d.p + (size_t)11 * n); MG_COUNT();
  return B200MD_OK;
}

int migrate_stage(Group& G, int d)
{
  cudaStream_t st = G.stream;
  const size_t K = G.dom.size();
  std::vector<int> n_lo(K), n_hi(K), n_stay(K), from_hi, from_lo;
  std::vector<std::unique_ptr<DBuf<int>>> idx_stay(K);
  for (auto& b : idx_stay)
    b.reset(new DBuf<int>);
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    const int n = D.n_own;
    MG_CUDA(D.flag_lo.reserve(D.cap));
    MG_CUDA(D.flag_hi.reserve(D.cap));
    MG_CUDA(D.flag_stay.reserve(D.cap));
    MG_CUDA(D.idx_tmp.reserve(D.cap));
    MG_CUDA(D.st[d].idx_lo.reserve(D.cap));
    MG_CUDA(D.st[d].idx_hi.reserve(D.cap));
    MG_CUDA(idx_stay[k]->reserve(D.cap));
    if (n > 0) {
      k_flag_faces<<<grid_for(n, BLK), BLK, 0, st>>>(
        n, D.own_d.p + (size_t)d * n, G.halo, G.halo + G.w[d], D.flag_lo.p, D.flag_hi.p, D.flag_stay.p); MG_COUNT();
    }
    MG_TRY(select(D, n, D.flag_lo.p, D.st[d].idx_lo.p, &n_lo[k], st));
    MG_TRY(select(D, n, D.flag_hi.p, D.st[d].idx_hi.p, &n_hi[k], st));
    MG_TRY(select(D, n, D.flag_stay.p, idx_stay[k]->p, &n_stay[k], st));
  }
  MG_TRY(exchange_counts(G, d, n_lo, n_hi, from_hi, from_lo));
  std::vector<Msg> msg(K);
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    const int n = D.n_own;
    msg[k].send_lo = (size_t)MIG_ROWS * n_lo[k];
    msg[k].send_hi = (size_t)MIG_ROWS * n_hi[k];
    msg[k].recv_hi = (size_t)MIG_ROWS * from_hi[k];
    msg[k].recv_lo = (size_t)MIG_ROWS * from_lo[k];
    MG_TRY(reserve_msg(D, msg[k].send_lo, msg[k].send_hi, msg[k].recv_hi, msg[k].recv_lo, st));
    if (n_lo[k]) {
      k_gather_rows<<<grid_for((long long)n_lo[k] * MIG_ROWS, BLK), BLK, 0, st>>>(
        n_lo[k], MIG_ROWS, D.st[d].idx_lo.p, n, D.own_d.p, d, +G.w[d], D.send_lo.p); MG_COUNT();
    }
    if (n_hi[k]) {
      k_gather_rows<<<grid_for((long long)n_hi[k] * MIG_ROWS, BLK), BLK, 0, st>>>(
        n_hi[k], MIG_ROWS, D.st[d].idx_hi.p, n, D.own_d.p, d, -G.w[d], D.send_hi.p); MG_COUNT();
    }
  }
  MG_TRY(exchange_payload(G, d, msg));
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    const int n = D.n_own;
    const int n_new = n_stay[k] + from_hi[k] + from_lo[k];
    if (n_new > D.cap)
      return fail(B200MD_ERR_OVERFLOW, "a domain's atom count exceeds its capacity (raise capacity_factor)");
    // own_d2 = [stay | from_hi | from_lo] with stride n_new
    if (n_stay[k]) {
      k_gather_rows<<<grid_for((long long)n_stay[k] * MIG_ROWS, BLK), BLK, 0, st>>>(
        n_stay[k], MIG_ROWS, idx_stay[k]->p, n, D.own_d.p, -1, 0.0, D.cand.p); MG_COUNT(); // cand as scratch
    }
    if (n_stay[k]) {
      k_scatter_rows<<<grid_for((long long)n_stay[k] * MIG_ROWS, BLK), BLK, 0, st>>>(
        n_stay[k], MIG_ROWS, D.cand.p, n_new, 0, D.own_d2.p); MG_COUNT();
    }
    if (from_hi[k]) {
      k_scatter_rows<<<grid_for((long long)from_hi[k] * MIG_ROWS, BLK), BLK, 0, st>>>(
        from_hi[k], MIG_ROWS, D.recv_hi.p, n_new, n_stay[k], D.own_d2.p); MG_COUNT();
    }
    if (from_lo[k]) {
      k_scatter_rows<<<grid_for((long long)from_lo[k] * MIG_ROWS, BLK), BLK, 0, st>>>(
        from_lo[k], MIG_ROWS, D.recv_lo.p, n_new, n_stay[k] + from_hi[k], D.own_d2.p); MG_COUNT();
    }
    std::swap(D.own_d.p, D.own_d2.p);
    std::swap(D.own_d.n, D.own_d2.n);
    D.n_own = n_new;
  }
  MG_CUDA(cudaStreamSynchronize(st)); // idx_stay buffers die here
  return B200MD_OK;
}

int ghost_stage(Group& G, int d, std::vector<int>& m_now)
{
  cudaStream_t st = G.stream;
  const size_t K = G.dom.size();
  std::vector<int> n_lo(K), n_hi(K), from_hi, from_lo;
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    Stage& S = D.st[d];
    S.active = true;
    S.m_cand = m_now[k];
    const int m = S.m_cand;
    // within `halo` of the lower face: coordinate < 2 halo; of the upper face: >= w
    if (m > 0) {
      k_flag_faces<<<grid_for(m, BLK), BLK, 0, st>>>(
        m, D.cand.p + (size_t)d * D.cap, 2.0 * G.halo, G.w[d], D.flag_lo.p, D.flag_hi.p, nullptr); MG_COUNT();
    }
    MG_TRY(select(D, m, D.flag_lo.p, S.idx_lo.p, &S.n_lo, st));
    MG_TRY(select(D, m, D.flag_hi.p, S.idx_hi.p, &S.n_hi, st));
    n_lo[k] = S.n_lo;
    n_hi[k] = S.n_hi;
  }
  MG_TRY(exchange_counts(G, d, n_lo, n_hi, from_hi, from_lo));
  std::vector<Msg> msg(K);
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    Stage& S = D.st[d];
    S.n_from_hi = from_hi[k];
    S.n_from_lo = from_lo[k];
    S.ghost_start = m_now[k];
    if (m_now[k] + from_hi[k] + from_lo[k] > D.cap)
      return fail(B200MD_ERR_OVERFLOW, "owned + ghost atoms exceed a domain's capacity (raise capacity_factor)");
    msg[k].send_lo = (size_t)GHOST_ROWS * S.n_lo;
    msg[k].send_hi = (size_t)GHOST_ROWS * S.n_hi;
    msg[k].recv_hi = (size_t)GHOST_ROWS * from_hi[k];
    msg[k].recv_lo = (size_t)GHOST_ROWS * from_lo[k];
    MG_TRY(reserve_msg(D, msg[k].send_lo, msg[k].send_hi, msg[k].recv_hi, msg[k].recv_lo, st));
    if (S.n_lo) {
      k_gather_rows<<<grid_for((long long)S.n_lo * GHOST_ROWS, BLK), BLK, 0, st>>>(
        S.n_lo, GHOST_ROWS, S.idx_lo.p, D.cap, D.cand.p, d, +G.w[d], D.send_lo.p); MG_COUNT();
    }
    if (S.n_hi) {
      k_gather_rows<<<grid_for((long long)S.n_hi * GHOST_ROWS, BLK), BLK, 0, st>>>(
        S.n_hi, GHOST_ROWS, S.idx_hi.p, D.cap, D.cand.p, d, -G.w[d], D.send_hi.p); MG_COUNT();
    }
  }
  MG_TRY(exchange_payload(G, d, msg));
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    Stage& S = D.st[d];
    if (S.n_from_hi) {
      k_scatter_rows<<<grid_for((long long)S.n_from_hi * GHOST_ROWS, BLK), BLK, 0, st>>>(
        S.n_from_hi, GHOST_ROWS, D.recv_hi.p, D.cap, S.ghost_start, D.cand.p); MG_COUNT();
    }
    if (S.n_from_lo) {
      k_scatter_rows<<<grid_for((long long)S.n_from_lo * GHOST_ROWS, BLK), BLK, 0, st>>>(
        S.n_from_lo, GHOST_ROWS, D.recv_lo.p, D.cap, S.ghost_start + S.n_from_hi, D.cand.p); MG_COUNT();
    }
    m_now[k] += S.n_from_hi + S.n_from_lo;
  }
  return B200MD_OK;
}

// own_d (compact owned state) -> ghosts -> main arrays
int rebuild_local(Group& G)
{
  cudaStream_t st = G.stream;
  const size_t K = G.dom.size();
  for (int d = 0; d < 3; ++d)
    if (G.cfg.grid[d] > 1)
      MG_TRY(migrate_stage(G, d));
  std::vector<int> m_now(K);
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    const int n = D.n_own;
    m_now[k] = n;
    for (int d = 0; d < 3; ++d)
      D.st[d].active = false;
    // candidates start as the owned atoms: pos3, type, mass
    for (int r = 0; r < 3; ++r)
      MG_CUDA(cudaMemcpyAsync(D.cand.p + (size_t)r * D.cap, D.own_d.p + (size_t)r * n,
                              sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
    MG_CUDA(cudaMemcpyAsync(D.cand.p + (size_t)3 * D.cap, D.own_d.p + (size_t)10 * n, sizeof(double) * n,
                            cudaMemcpyDeviceToDevice, st));
    MG_CUDA(cudaMemcpyAsync(D.cand.p + (size_t)4 * D.cap, D.own_d.p + (size_t)9 * n, sizeof(double) * n,
                            cudaMemcpyDeviceToDevice, st));
  }
  for (int d = 0; d < 3; ++d)
    if (G.cfg.grid[d] > 1)
      MG_TRY(ghost_stage(G, d, m_now));
  for (size_t k = 0; k < K; ++k) {
    Domain& D = *G.dom[k];
    const int n = D.n_own, s = m_now[k];
    D.n_loc = s;
    MG_CUDA(cudaMemsetAsync(D.vel.p, 0, sizeof(double) * 3 * (size_t)s, st));
    MG_CUDA(cudaMemsetAsync(D.force.p, 0, sizeof(double) * 3 * (size_t)s, st));
    for (int r = 0; r < 3; ++r) {
      MG_CUDA(cudaMemcpyAsync(D.pos.p + (size_t)r * s, D.cand.p + (size_t)r * D.cap, sizeof(double) * s,
                              cudaMemcpyDeviceToDevice, st));
      MG_CUDA(cudaMemcpyAsync(D.vel.p + (size_t)r * s, D.own_d.p + (size_t)(3 + r) * n,
                              sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
      MG_CUDA(cudaMemcpyAsync(D.force.p + (size_t)r * s, D.own_d.p + (size_t)(6 + r) * n,
                              sizeof(double) * n, cudaMemcpyDeviceToDevice, st));
      MG_CUDA(cudaMemcpyAsync(D.ref.p + (size_t)r * n, D.own_d.p + (size_t)r * n, sizeof(double) * n,
                              cudaMemcpyDeviceToDevice, st));
    }
    MG_CUDA(cudaMemcpyAsync(D.mass.p, D.cand.p + (size_t)4 * D.cap, sizeof(double) * s,
                            cudaMemcpyDeviceToDevice, st));
    if (s > 0) {
      k_double_to_int<<<grid_for(s, BLK), BLK, 0, st>>>(s, D.cand.p + (size_t)3 * D.cap, D.type.p); MG_COUNT();
    }
    if (n > 0) {
      k_double_to_ll<<<grid_for(n, BLK), BLK, 0, st>>>(n, D.own_d.p + (size_t)11 * n, D.id.p); MG_COUNT();
    }
    // a block over vacuum may hold no atoms at all: its potential keeps its old list and is not
    // called until an exchange brings atoms in
    if (s > 0)
      MG_TRY(D.pot.invalidate(s, st));
    MG_TRY(D.pot.set_owned(n));
  }
  if (G.graph) { // array strides changed: the captured step is stale
    cudaGraphExecDestroy(G.graph);
    G.graph = nullptr;
  }
  G.steps_since_exchange = 0;
  return B200MD_OK;
}

// ---------------------------------------------------------------------------------------------
// per-step pieces
// ---------------------------------------------------------------------------------------------
int halo_update(Group& G)
{
  cudaStream_t st = G.stream;
  const size_t K = G.dom.size();
  for (int d = 0; d < 3; ++d) {
    if (G.cfg.grid[d] <= 1)
      continue;
    std::vector<Msg> msg(K);
    for (size_t k = 0; k < K; ++k) {
      Domain& D = *G.dom[k];
      const Stage& S = D.st[d];
      msg[k].send_lo = (size_t)3 * S.n_lo;
      msg[k].send_hi = (size_t)3 * S.n_hi;
      msg[k].recv_hi = (size_t)3 * S.n_from_hi;
      msg[k].recv_lo = (size_t)3 * S.n_from_lo;
      if (S.n_lo) {
        k_gather_rows<<<grid_for((long long)S.n_lo * 3, BLK), BLK, 0, st>>>(
          S.n_lo, 3, S.idx_lo.p, D.n_loc, D.pos.p, d, +G.w[d], D.send_lo.p); MG_COUNT();
      }
      if (S.n_hi) {
        k_gather_rows<<<grid_for((long long)S.n_hi * 3, BLK), BLK, 0, st>>>(
          S.n_hi, 3, S.idx_hi.p, D.n_loc, D.pos.p, d, -G.w[d], D.send_hi.p); MG_COUNT();
      }
    }
    MG_TRY(exchange_payload(G, d, msg));
    for (size_t k = 0; k < K; ++k) {
      Domain& D = *G.dom[k];
      const Stage& S = D.st[d];
      if (S.n_from_hi) {
        k_scatter_rows<<<grid_for((long long)S.n_from_hi * 3, BLK), BLK, 0, st>>>(
          S.n_from_hi, 3, D.recv_hi.p, D.n_loc, S.ghost_start, D.pos.p); MG_COUNT();
      }
      if (S.n_from_lo) {
        k_scatter_rows<<<grid_for((long long)S.n_from_lo * 3, BLK), BLK, 0, st>>>(
          S.n_from_lo, 3, D.recv_lo.p, D.n_loc, S.ghost_start + S.n_from_hi, D.pos.p); MG_COUNT();
      }
    }
  }
  return B200MD_OK;
}

int compute_force(Group& G)
{
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    if (D.n_loc == 0)
      continue;
    if (D.pot.kind != 0) // NEP stores its outputs (set_accumulate(0) at creation): no zeroing pass
      MG_B2(b200md_zero_properties(D.n_loc, D.pe.p, D.force.p, D.virial.p, G.stream));
    MG_TRY(D.pot.compute(D.n_loc, D.lh, D.lpbc, D.type.p, D.pos.p, D.pe.p, D.force.p, D.virial.p, G.stream));
  }
  return B200MD_OK;
}

// the sum over all domains of (D.*buf)[0..n), n <= 8, lands in every domain's buffer: one
// ncclAllReduce, or in local mode a sum in domain order
int sum_over_domains(Group& G, DBuf<double> Domain::*buf, int n)
{
  cudaStream_t st = G.stream;
  if (G.distributed) {
    double* p = ((*G.dom[0]).*buf).p;
    MG_NCCL(ncclAllReduce(p, p, n, ncclDouble, ncclSum, G.comm, st));
  } else if (G.dom.size() > 1) {
    MG_CUDA(cudaMemsetAsync(G.thermo_sum.p, 0, n * sizeof(double), st));
    for (auto& dp : G.dom)
      k_add8<<<1, 32, 0, st>>>(G.thermo_sum.p, ((*dp).*buf).p, n); MG_COUNT();
    for (auto& dp : G.dom)
      MG_CUDA(cudaMemcpyAsync(((*dp).*buf).p, G.thermo_sum.p, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  }
  return B200MD_OK;
}

// partial sums over the owned atoms, then the global sum lands in every domain's thermo[]; a block
// that owns no atoms still runs it, because its single thread block writes the zero partial
int find_thermo(Group& G)
{
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    MG_B2(b200md_find_thermo_strided(
      D.n_own, D.n_loc, (int)G.n_global, G.volume, D.mass.p, D.pe.p, D.vel.p, D.virial.p, D.thermo.p,
      D.thermo_scratch.p, G.stream));
  }
  return sum_over_domains(G, &Domain::thermo, 8);
}

// compute_hnemd's drive (force.cu:857-897) on the blocks: f_i += W_i^T fe on the owned atoms with each
// block's total of the new forces, the global total, then f_i -= total / N.  A block that owns no
// atoms contributes the zero total of its single thread block and skips the correction.
int hnemd_drive(Group& G)
{
  cudaStream_t st = G.stream;
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    MG_B2(b200md_hnemd_drive_add(
      D.n_own, D.n_loc, G.hn_fe, D.virial.p, D.force.p, D.hn_scratch.p, D.hn_ftot.p, st));
  }
  MG_TRY(sum_over_domains(G, &Domain::hn_ftot, 3));
  const double one_over_n = 1.0 / (double)G.n_global;
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    MG_B2(b200md_hnemd_drive_correct(D.n_own, D.n_loc, one_over_n, D.hn_ftot.p, D.force.p, st));
  }
  return B200MD_OK;
}

// HNEMD::process (hnemd_kappa.cu:82-106) on the blocks: every block sums the heat current of its owned
// atoms into its own ring row; blocks are summed only at take time
int hnemd_heat(Group& G)
{
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    MG_B2(b200md_hnemd_heat_row(
      D.n_own, D.n_loc, D.virial.p, D.vel.p, D.hn_rows.p, G.hn_ring, D.hn_row.p, D.hn_scratch.p, G.stream));
  }
  return B200MD_OK;
}

int nhc_half(Group& G, double dt)
{
  MG_TRY(find_thermo(G));
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    MG_B2(b200md_nhc_half_step(D.nhc, D.n_own, D.n_loc, dt, D.thermo.p, D.vel.p, G.stream));
  }
  return B200MD_OK;
}

void mark(Group& G, int k)
{
  if (G.prof)
    cudaEventRecord(G.ev[k], G.stream);
}

int one_step(Group& G, double dt)
{
  cudaStream_t st = G.stream;
  const int ens = G.cfg.ensemble;
  const long long l0 = g_own_launches + b200md_launch_count();
  struct Tally {
    Group& G;
    long long l0;
    ~Tally() { G.launches_per_step = g_own_launches + b200md_launch_count() - l0; }
  } tally{G, l0};
  mark(G, 0);
  if (ens == 2)
    MG_TRY(nhc_half(G, dt));
  // blocks that own no atoms skip the per-atom launches (a zero-block grid is a launch error); the
  // thermostat calls still run there, because they advance the chain / random state that every
  // domain keeps a copy of and only scale when there are atoms
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    if (D.n_own == 0)
      continue;
    MG_B2(b200md_velocity_verlet_strided(
      1, D.n_own, D.n_loc, dt, D.mass.p, D.pos.p, D.vel.p, D.force.p, st));
    // wrap only the undecomposed periodic directions (the local box is open in the others)
    MG_B2(b200md_apply_pbc_strided(D.n_own, D.n_loc, D.lh, D.lpbc, D.pos.p, st));
  }
  mark(G, 1);
  MG_TRY(halo_update(G));
  mark(G, 2);
  MG_TRY(compute_force(G));
  if (G.hn_on)
    MG_TRY(hnemd_drive(G));
  mark(G, 3);
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    if (D.n_own > 0)
      MG_B2(b200md_velocity_verlet_strided(
        0, D.n_own, D.n_loc, dt, D.mass.p, D.pos.p, D.vel.p, D.force.p, st));
  }
  if (ens == 2) {
    MG_TRY(nhc_half(G, dt));
  } else {
    MG_TRY(find_thermo(G));
    for (auto& dp : G.dom) {
      Domain& D = *dp;
      if (ens == 1 && D.n_own > 0)
        MG_B2(b200md_berendsen_temperature(
          D.n_own, D.n_loc, G.cfg.temperature, G.cfg.temperature_coupling, D.thermo.p, D.vel.p, st));
      else if (ens == 4)
        MG_B2(b200md_bdp_step(D.bdp, D.n_own, D.n_loc, D.thermo.p, D.vel.p, st));
    }
  }
  if (G.hn_on)
    MG_TRY(hnemd_heat(G));
  mark(G, 4);
  return B200MD_OK;
}

// true on every rank when some owned atom anywhere moved further than 0.7 * skin / 2
int needs_exchange(Group& G, bool* out)
{
  cudaStream_t st = G.stream;
  float worst = 0.0f;
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    MG_CUDA(cudaMemsetAsync(D.disp_bits.p, 0, sizeof(unsigned int), st));
    if (D.n_own > 0) {
      k_max_disp2<<<grid_for(D.n_own, BLK), BLK, 0, st>>>(
        D.n_own, D.n_loc, D.pos.p, D.ref.p, D.lpbc[0] ? G.L[0] : 0.0, D.lpbc[1] ? G.L[1] : 0.0,
        D.lpbc[2] ? G.L[2] : 0.0, D.disp_bits.p); MG_COUNT();
    }
  }
  if (G.distributed)
    MG_NCCL(ncclAllReduce(G.dom[0]->disp_bits.p, G.dom[0]->disp_bits.p, 1, ncclUint32, ncclMax, G.comm, st));
  for (auto& dp : G.dom) {
    unsigned int bits = 0;
    MG_CUDA(cudaMemcpyAsync(&bits, dp->disp_bits.p, sizeof bits, cudaMemcpyDeviceToHost, st));
    MG_CUDA(cudaStreamSynchronize(st));
    float v;
    std::memcpy(&v, &bits, sizeof v);
    worst = v > worst ? v : worst;
  }
  const double lim = 0.7 * 0.5 * G.cfg.skin;
  *out = worst > (float)(lim * lim);
  return B200MD_OK;
}

int exchange(Group& G)
{
  for (auto& dp : G.dom)
    MG_TRY(sync_owned(G, *dp));
  MG_TRY(rebuild_local(G));
  MG_TRY(halo_update(G));
  ++G.migrations;
  return B200MD_OK;
}

} // namespace

// ---------------------------------------------------------------------------------------------
// C-ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

const char* b200md_mgpu_last_error(void) { return g_err.c_str(); }

int b200md_mgpu_unique_id(char out128[128])
{
  ncclUniqueId id;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  MG_NCCL(ncclGetUniqueId(&id));
  std::memcpy(out128, &id, 128);
  return B200MD_OK;
}

int b200md_mgpu_create(const b200md_mgpu_config* cfg, const char* nccl_id128, b200md_mgpu** out)
{
  if (!cfg || !out || !cfg->potential_file)
    return fail(B200MD_ERR_ARG, "b200md_mgpu_create: bad argument");
  const double* h = cfg->h;
  if (h[1] != 0 || h[2] != 0 || h[3] != 0 || h[5] != 0 || h[6] != 0 || h[7] != 0)
    return fail(B200MD_ERR_ARG, "domain decomposition needs an orthogonal box");
  std::unique_ptr<Group> G(new Group);
  G->cfg = *cfg;
  G->potential_file = cfg->potential_file;
  G->cfg.potential_file = G->potential_file.c_str();
  if (G->cfg.skin < 1.0)
    G->cfg.skin = 1.0;
  if (G->cfg.capacity_factor < 1.05)
    G->cfg.capacity_factor = 1.35;
  G->world = cfg->grid[0] * cfg->grid[1] * cfg->grid[2];
  if (G->world < 1)
    return fail(B200MD_ERR_ARG, "grid must be >= 1 in every direction");
  G->distributed = nccl_id128 != nullptr;
  for (int d = 0; d < 3; ++d) {
    G->L[d] = h[4 * d];
    G->w[d] = G->L[d] / cfg->grid[d];
    if (cfg->grid[d] > 1 && !cfg->pbc[d])
      return fail(B200MD_ERR_ARG, "decomposed directions must be periodic");
  }
  G->volume = G->L[0] * G->L[1] * G->L[2];
  MG_CUDA(cudaStreamCreateWithFlags(&G->stream, cudaStreamNonBlocking));
  for (auto& e : G->ev)
    MG_CUDA(cudaEventCreate(&e));
  if (G->distributed) {
    ncclUniqueId id;
    std::memcpy(&id, nccl_id128, 128);
    MG_NCCL(ncclCommInitRank(&G->comm, G->world, id, cfg->rank));
  }
  // the cutoff decides the halo: read it through a throw-away handle
  {
    Pot probe;
    MG_TRY(probe.create(G->potential_file.c_str(), 64));
    G->halo = (probe.many_body ? 2.0 : 1.0) * probe.rc + G->cfg.skin;
  }
  for (int d = 0; d < 3; ++d)
    if (cfg->grid[d] > 1 && G->w[d] < G->halo)
      return fail(B200MD_ERR_ARG, "a domain is narrower than the halo (2*rc + skin): use fewer ranks in that direction");
  const int first = G->distributed ? cfg->rank : 0, last = G->distributed ? cfg->rank + 1 : G->world;
  for (int r = first; r < last; ++r) {
    std::unique_ptr<Domain> D(new Domain);
    D->rank = r;
    D->c[0] = r / (cfg->grid[1] * cfg->grid[2]);
    D->c[1] = (r / cfg->grid[2]) % cfg->grid[1];
    D->c[2] = r % cfg->grid[2];
    for (int k = 0; k < 9; ++k)
      D->lh[k] = 0.0;
    for (int d = 0; d < 3; ++d) {
      int lo[3] = {D->c[0], D->c[1], D->c[2]}, hi[3] = {D->c[0], D->c[1], D->c[2]};
      lo[d] = (D->c[d] - 1 + cfg->grid[d]) % cfg->grid[d];
      hi[d] = (D->c[d] + 1) % cfg->grid[d];
      D->nb_lo[d] = rank_of(cfg->grid, lo[0], lo[1], lo[2]);
      D->nb_hi[d] = rank_of(cfg->grid, hi[0], hi[1], hi[2]);
      if (cfg->grid[d] > 1) {
        D->origin[d] = D->c[d] * G->w[d] - G->halo;
        D->lh[4 * d] = G->w[d] + 2.0 * G->halo;
        D->lpbc[d] = 0;
      } else {
        D->origin[d] = 0.0;
        D->lh[4 * d] = G->L[d];
        D->lpbc[d] = cfg->pbc[d] ? 1 : 0;
      }
    }
    G->dom.push_back(std::move(D));
  }
  MG_CUDA(G->thermo_sum.reserve(8));
  *out = G.release();
  return B200MD_OK;
}

void b200md_mgpu_destroy(b200md_mgpu* g)
{
  if (g) {
    cudaStreamSynchronize(g->stream);
    delete g;
  }
}

int b200md_mgpu_distribute(
  b200md_mgpu* g, int n_global, const int* type, const double* position, const double* mass,
  const double* velocity)
{
  Group& G = *g;
  cudaStream_t st = G.stream;
  G.n_global = n_global;
  G.hn_on = false; // the domains' buffers are about to be re-sized: b200md_mgpu_hnemd_set comes after
  const size_t N = (size_t)n_global;
  // owner of every atom from its wrapped coordinate
  std::vector<int> owner(N);
  std::vector<double> wrapped(3 * N);
  for (size_t i = 0; i < N; ++i) {
    int c[3];
    for (int d = 0; d < 3; ++d) {
      double x = position[d * N + i];
      if (G.cfg.pbc[d]) {
        x = std::fmod(x, G.L[d]);
        if (x < 0)
          x += G.L[d];
      }
      wrapped[d * N + i] = x;
      int q = G.cfg.grid[d] > 1 ? (int)std::floor(x / G.w[d]) : 0;
      if (q >= G.cfg.grid[d])
        q = G.cfg.grid[d] - 1;
      if (q < 0)
        q = 0;
      c[d] = q;
    }
    owner[i] = rank_of(G.cfg.grid, c[0], c[1], c[2]);
  }
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    std::vector<size_t> mine;
    for (size_t i = 0; i < N; ++i)
      if (owner[i] == D.rank)
        mine.push_back(i);
    const int n = (int)mine.size();
    // capacity: owned + a halo shell estimated from the volumes, times the safety factor
    double vol_own = 1.0, vol_loc = 1.0;
    for (int d = 0; d < 3; ++d) {
      vol_own *= D.lh[4 * d] - (G.cfg.grid[d] > 1 ? 2.0 * G.halo : 0.0);
      vol_loc *= D.lh[4 * d];
    }
    const double est = (double)n_global / (double)G.world * (vol_loc / vol_own);
    D.cap = (int)(G.cfg.capacity_factor * (est > n ? est : n)) + 1024;
    const size_t cap = (size_t)D.cap;
    MG_CUDA(D.pos.reserve(3 * cap));
    MG_CUDA(D.vel.reserve(3 * cap));
    MG_CUDA(D.force.reserve(3 * cap));
    MG_CUDA(D.virial.reserve(9 * cap));
    MG_CUDA(D.pe.reserve(cap));
    MG_CUDA(D.mass.reserve(cap));
    MG_CUDA(D.type.reserve(cap));
    MG_CUDA(D.id.reserve(cap));
    MG_CUDA(D.own_d.reserve(MIG_ROWS * cap));
    MG_CUDA(D.own_d2.reserve(MIG_ROWS * cap));
    MG_CUDA(D.cand.reserve(MIG_ROWS * cap));
    MG_CUDA(D.ref.reserve(3 * cap));
    MG_CUDA(D.flag_lo.reserve(cap));
    MG_CUDA(D.flag_hi.reserve(cap));
    MG_CUDA(D.flag_stay.reserve(cap));
    MG_CUDA(D.idx_tmp.reserve(cap));
    MG_CUDA(D.count_dev.reserve(4));
    MG_CUDA(D.disp_bits.reserve(1));
    MG_CUDA(D.thermo.reserve(8));
    for (int d = 0; d < 3; ++d) {
      MG_CUDA(D.st[d].idx_lo.reserve(cap));
      MG_CUDA(D.st[d].idx_hi.reserve(cap));
    }
    const long long sb = b200md_thermo_scratch_bytes(D.cap);
    MG_CUDA(D.thermo_scratch.reserve((size_t)sb));
    MG_CUDA(cudaMemsetAsync(D.thermo_scratch.p, 0, (size_t)sb, st));
    MG_CUDA(cudaMemsetAsync(D.thermo.p, 0, 8 * sizeof(double), st));
    MG_TRY(D.pot.create(G.potential_file.c_str(), D.cap));
    { // ghosts beyond rc + skin of the owned block cannot be a neighbour of an owned atom: no
      // descriptor work for them (they still serve as neighbours)
      double lo[3], hi[3];
      const double reach = D.pot.rc + G.cfg.skin;
      for (int d = 0; d < 3; ++d) {
        const bool cut = G.cfg.grid[d] > 1;
        lo[d] = cut ? G.halo - reach : -1.0e300;
        hi[d] = cut ? G.halo + G.w[d] + reach : 1.0e300;
      }
      MG_TRY(D.pot.set_active(lo, hi));
    }
    if (G.cfg.ensemble == 2)
      MG_B2(b200md_nhc_create(n_global, G.cfg.temperature, G.cfg.temperature_coupling, G.cfg.time_step, &D.nhc));
    else if (G.cfg.ensemble == 4)
      MG_B2(b200md_bdp_create(n_global, G.cfg.temperature, G.cfg.temperature_coupling, G.cfg.bdp_seed, &D.bdp));
    else if (G.cfg.ensemble != 0 && G.cfg.ensemble != 1)
      return fail(B200MD_ERR_ARG, "unsupported ensemble (0 nve, 1 nvt_ber, 2 nvt_nhc, 4 nvt_bdp)");
    // compact owned state on the host -> own_d
    std::vector<double> hbuf((size_t)MIG_ROWS * n);
    for (int k = 0; k < n; ++k) {
      const size_t i = mine[k];
      for (int d = 0; d < 3; ++d) {
        hbuf[(size_t)d * n + k] = wrapped[d * N + i] - D.origin[d];
        hbuf[(size_t)(3 + d) * n + k] = velocity ? velocity[d * N + i] : 0.0;
        hbuf[(size_t)(6 + d) * n + k] = 0.0;
      }
      hbuf[(size_t)9 * n + k] = mass[i];
      hbuf[(size_t)10 * n + k] = (double)type[i];
      hbuf[(size_t)11 * n + k] = (double)i;
    }
    if (n > 0)
      MG_CUDA(cudaMemcpyAsync(D.own_d.p, hbuf.data(), sizeof(double) * hbuf.size(), cudaMemcpyHostToDevice, st));
    MG_CUDA(cudaStreamSynchronize(st));
    D.n_own = n;
    D.n_loc = n;
  }
  MG_TRY(rebuild_local(G));
  MG_TRY(compute_force(G));
  MG_TRY(find_thermo(G));
  MG_CUDA(cudaStreamSynchronize(st));
  return b200md_mgpu_check(g);
}

int b200md_mgpu_run(b200md_mgpu* g, int nsteps, int check_every)
{
  Group& G = *g;
  const double dt = G.cfg.time_step;
  if (check_every < 1)
    check_every = 5;
  if (G.hn_on && nsteps > 0 && (G.hn_pending + nsteps) / G.hn_oi > G.hn_max)
    return fail(B200MD_ERR_OVERFLOW, "b200md_mgpu_run: the run would complete more HNEMD intervals than "
                                     "max_intervals before the next b200md_mgpu_hnemd_take");
  auto stepped = [&G] { // every step enqueued writes one HNEMD heat row
    ++G.steps_since_exchange;
    if (G.hn_on)
      ++G.hn_pending;
  };
  for (int s = 0; s < nsteps; ++s) {
    if (G.steps_since_exchange && G.steps_since_exchange % check_every == 0) {
      bool need = false;
      MG_TRY(needs_exchange(G, &need));
      if (need)
        MG_TRY(exchange(G));
    }
    if (G.cfg.use_cuda_graph && !G.prof) {
      if (!G.graph || G.graph_dt != dt) {
        if (G.graph) {
          cudaGraphExecDestroy(G.graph);
          G.graph = nullptr;
        }
        // one eager step first so that nothing allocates or synchronises inside the capture
        MG_TRY(one_step(G, dt));
        stepped();
        if (++s >= nsteps)
          break;
        cudaGraph_t graph = nullptr;
        MG_CUDA(cudaStreamBeginCapture(G.stream, cudaStreamCaptureModeThreadLocal));
        const int rc = one_step(G, dt);
        const cudaError_t ce = cudaStreamEndCapture(G.stream, &graph);
        if (rc != B200MD_OK)
          return rc;
        MG_CUDA(ce);
        MG_CUDA(cudaGraphInstantiate(&G.graph, graph, nullptr, nullptr, 0));
        MG_CUDA(cudaGraphDestroy(graph));
        G.graph_dt = dt;
      }
      MG_CUDA(cudaGraphLaunch(G.graph, G.stream));
    } else {
      MG_TRY(one_step(G, dt));
      if (G.prof) {
        MG_CUDA(cudaStreamSynchronize(G.stream));
        for (int k = 0; k < 4; ++k) {
          float ms = 0.0f;
          cudaEventElapsedTime(&ms, G.ev[k], G.ev[k + 1]);
          G.prof_ms[k] += ms;
        }
        ++G.prof_steps;
      }
    }
    stepped();
  }
  return B200MD_OK;
}

int b200md_mgpu_run_timed(b200md_mgpu* g, int nsteps, int check_every, double* ms_out)
{
  Group& G = *g;
  if (!G.t0) {
    MG_CUDA(cudaEventCreate(&G.t0));
    MG_CUDA(cudaEventCreate(&G.t1));
  }
  MG_CUDA(cudaStreamSynchronize(G.stream));
  MG_CUDA(cudaEventRecord(G.t0, G.stream));
  MG_TRY(b200md_mgpu_run(g, nsteps, check_every));
  MG_CUDA(cudaEventRecord(G.t1, G.stream));
  MG_CUDA(cudaStreamSynchronize(G.stream));
  float ms = 0.0f;
  MG_CUDA(cudaEventElapsedTime(&ms, G.t0, G.t1));
  if (ms_out)
    *ms_out = ms;
  return B200MD_OK;
}

int b200md_mgpu_thermo(b200md_mgpu* g, double out8[8])
{
  Group& G = *g;
  MG_CUDA(cudaMemcpyAsync(out8, G.dom[0]->thermo.p, 8 * sizeof(double), cudaMemcpyDeviceToHost, G.stream));
  MG_CUDA(cudaStreamSynchronize(G.stream));
  return B200MD_OK;
}

int b200md_mgpu_heat_current(b200md_mgpu* g, double out5[5])
{
  Group& G = *g;
  cudaStream_t st = G.stream;
  double tot[5] = {0, 0, 0, 0, 0};
  for (auto& dp : G.dom) {
    Domain& D = *dp;
    const int n = D.n_own;
    MG_CUDA(D.heat.reserve(5 * (size_t)D.cap));
    MG_CUDA(D.heat5.reserve(5));
    if (n == 0)
      MG_CUDA(cudaMemsetAsync(D.heat5.p, 0, 5 * sizeof(double), st));
    else
      MG_B2(b200md_compute_heat(n, D.n_loc, D.virial.p, D.vel.p, D.heat.p, n, st));
    // five device reductions (cub): rare call (every sample_interval steps)
    for (int k = 0; k < 5 && n > 0; ++k) {
      size_t need = 0;
      MG_CUDA(cub::DeviceReduce::Sum(nullptr, need, D.heat.p + (size_t)k * n, D.heat5.p + k, n, st));
      if (need > D.cub_bytes) {
        MG_CUDA(cudaStreamSynchronize(st));
        MG_CUDA(D.cub_tmp.reserve(need));
        D.cub_bytes = D.cub_tmp.n;
      }
      need = D.cub_bytes;
      MG_CUDA(cub::DeviceReduce::Sum(D.cub_tmp.p, need, D.heat.p + (size_t)k * n, D.heat5.p + k, n, st));
    }
    if (G.distributed)
      MG_NCCL(ncclAllReduce(D.heat5.p, D.heat5.p, 5, ncclDouble, ncclSum, G.comm, st));
    double h5[5];
    MG_CUDA(cudaMemcpyAsync(h5, D.heat5.p, sizeof h5, cudaMemcpyDeviceToHost, st));
    MG_CUDA(cudaStreamSynchronize(st));
    for (int k = 0; k < 5; ++k)
      tot[k] += h5[k];
  }
  for (int k = 0; k < 5; ++k)
    out5[k] = tot[k];
  return B200MD_OK;
}

int b200md_mgpu_hnemd_set(b200md_mgpu* g, int output_interval, const double fe[3], int max_intervals)
{
  if (!g || !fe || output_interval < 1 || max_intervals < 1)
    return fail(B200MD_ERR_ARG, "b200md_mgpu_hnemd_set: need output_interval >= 1, max_intervals >= 1 and fe[3]");
  if (!std::isfinite(fe[0]) || !std::isfinite(fe[1]) || !std::isfinite(fe[2]))
    return fail(B200MD_ERR_ARG, "b200md_mgpu_hnemd_set: fe must be finite");
  if ((long long)(max_intervals + 1LL) * output_interval > INT_MAX / 5)
    return fail(B200MD_ERR_ARG, "b200md_mgpu_hnemd_set: (max_intervals + 1) * output_interval rows are too many");
  Group& G = *g;
  if (G.n_global <= 0)
    return fail(B200MD_ERR_ARG, "b200md_mgpu_hnemd_set: call b200md_mgpu_distribute first");
  cudaStream_t st = G.stream;
  MG_CUDA(cudaStreamSynchronize(st)); // buffers of a previous setting may still be in use
  if (G.graph) { // the step gains or loses launches
    cudaGraphExecDestroy(G.graph);
    G.graph = nullptr;
  }
  G.hn_on = fe[0] != 0.0 || fe[1] != 0.0 || fe[2] != 0.0; // fe = 0: Force::finalize, force.cu:335-339
  for (int d = 0; d < 3; ++d)
    G.hn_fe[d] = fe[d];
  G.hn_oi = output_interval;
  G.hn_max = max_intervals;
  // a take finds at most max_intervals whole intervals and a partial one
  G.hn_ring = (max_intervals + 1) * output_interval;
  G.hn_first = 0;
  G.hn_pending = 0;
  if (G.hn_on) {
    const size_t ring = (size_t)5 * G.hn_ring;
    for (auto& dp : G.dom) {
      Domain& D = *dp;
      const size_t sb = (size_t)std::max(b200md_hnemd_drive_scratch_bytes(D.cap),
                                         b200md_hnemd_heat_row_scratch_bytes(D.cap));
      MG_CUDA(D.hn_ftot.reserve(3));
      MG_CUDA(D.hn_rows.reserve(ring));
      MG_CUDA(D.hn_row.reserve(1));
      MG_CUDA(D.hn_scratch.reserve(sb));
      MG_CUDA(cudaMemsetAsync(D.hn_rows.p, 0, sizeof(double) * ring, st));
      MG_CUDA(cudaMemsetAsync(D.hn_row.p, 0, sizeof(unsigned int), st));
      MG_CUDA(cudaMemsetAsync(D.hn_scratch.p, 0, sb, st));
    }
    if (G.distributed)
      MG_CUDA(G.hn_gather.reserve(ring * G.world));
  }
  // forces at the current positions as the next step's first half expects them (the evaluation before
  // a run's loop, run.cu:217-248); the ghosts' positions are those of the last force call
  MG_TRY(compute_force(G));
  if (G.hn_on)
    MG_TRY(hnemd_drive(G));
  MG_CUDA(cudaStreamSynchronize(st));
  return b200md_mgpu_check(g);
}

int b200md_mgpu_hnemd_take(b200md_mgpu* g, double temperature, int* n_intervals, double* kappa, double* rows)
{
  if (!g || !n_intervals || !kappa || !(temperature > 0.0))
    return fail(B200MD_ERR_ARG, "b200md_mgpu_hnemd_take: need temperature > 0, n_intervals and kappa");
  Group& G = *g;
  if (!G.hn_on)
    return fail(B200MD_ERR_ARG, "b200md_mgpu_hnemd_take: HNEMD is off (b200md_mgpu_hnemd_set with fe != 0)");
  cudaStream_t st = G.stream;
  const int oi = G.hn_oi, m = (int)(G.hn_pending / oi);
  const size_t ring = (size_t)5 * G.hn_ring;
  // the rows of all blocks, summed in block (= rank) order on the host
  std::vector<double> all, sum(ring);
  if (G.distributed) {
    Domain& D = *G.dom[0];
    all.resize(ring * G.world);
    MG_NCCL(ncclAllGather(D.hn_rows.p, G.hn_gather.p, ring, ncclDouble, G.comm, st));
    MG_CUDA(cudaMemcpyAsync(all.data(), G.hn_gather.p, sizeof(double) * all.size(), cudaMemcpyDeviceToHost, st));
  } else {
    all.resize(ring * G.dom.size());
    for (size_t k = 0; k < G.dom.size(); ++k)
      MG_CUDA(cudaMemcpyAsync(all.data() + ring * k, G.dom[k]->hn_rows.p, sizeof(double) * ring,
                              cudaMemcpyDeviceToHost, st));
  }
  MG_CUDA(cudaStreamSynchronize(st));
  const size_t blocks = all.size() / ring;
  for (size_t e = 0; e < ring; ++e) {
    double v = all[e];
    for (size_t k = 1; k < blocks; ++k)
      v += all[ring * k + e];
    sum[e] = v;
  }
  std::vector<double> h((size_t)5 * oi);
  for (int j = 0; j < m; ++j) {
    for (int r = 0; r < oi; ++r) {
      const size_t at = (size_t)((G.hn_first + (long long)j * oi + r) % G.hn_ring);
      for (int k = 0; k < 5; ++k)
        h[(size_t)5 * r + k] = sum[5 * at + k];
    }
    MG_B2(b200md_hnemd_kappa(oi, G.volume, temperature, G.hn_fe, h.data(), kappa + (size_t)5 * j));
    if (rows)
      std::copy(h.begin(), h.end(), rows + (size_t)5 * oi * j);
  }
  G.hn_first = (int)((G.hn_first + (long long)m * oi) % G.hn_ring);
  G.hn_pending -= (long long)m * oi;
  *n_intervals = m;
  return B200MD_OK;
}

long long b200md_mgpu_info(b200md_mgpu* g, int what, int k)
{
  Group& G = *g;
  if (what == 0)
    return (long long)G.dom.size();
  if (what == 3)
    return G.migrations;
  if (what == 6)
    return G.launches_per_step;
  if (k < 0 || k >= (int)G.dom.size())
    return -1;
  Domain& D = *G.dom[k];
  switch (what) {
    case 1: return D.n_own;
    case 2: return D.n_loc;
    case 4: cudaStreamSynchronize(G.stream); return D.pot.rebuilds();
    case 5: return D.rank;
    default: return -1;
  }
}

int b200md_mgpu_get_owned(
  b200md_mgpu* g, int k, long long* id, double* position, double* velocity, double* force,
  double* potential, double* virial)
{
  Group& G = *g;
  if (k < 0 || k >= (int)G.dom.size())
    return fail(B200MD_ERR_ARG, "b200md_mgpu_get_owned: bad domain index");
  Domain& D = *G.dom[k];
  cudaStream_t st = G.stream;
  const size_t n = (size_t)D.n_own, s = (size_t)D.n_loc;
  auto rows = [&](double* out, const double* dev, int r) -> int {
    if (!out)
      return B200MD_OK;
    for (int q = 0; q < r; ++q)
      MG_CUDA(cudaMemcpyAsync(out + q * n, dev + q * s, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    return B200MD_OK;
  };
  if (id)
    MG_CUDA(cudaMemcpyAsync(id, D.id.p, sizeof(long long) * n, cudaMemcpyDeviceToHost, st));
  MG_TRY(rows(position, D.pos.p, 3));
  MG_TRY(rows(velocity, D.vel.p, 3));
  MG_TRY(rows(force, D.force.p, 3));
  MG_TRY(rows(potential, D.pe.p, 1));
  MG_TRY(rows(virial, D.virial.p, 9));
  MG_CUDA(cudaStreamSynchronize(st));
  if (position)
    for (int d = 0; d < 3; ++d)
      for (size_t i = 0; i < n; ++i) {
        double x = position[d * n + i] + D.origin[d];
        if (G.cfg.pbc[d]) {
          x = std::fmod(x, G.L[d]);
          if (x < 0)
            x += G.L[d];
        }
        position[d * n + i] = x;
      }
  return B200MD_OK;
}

int b200md_mgpu_get_local(
  b200md_mgpu* g, int k, int* type, double* position, double h_out[9], int pbc_out[3])
{
  Group& G = *g;
  if (k < 0 || k >= (int)G.dom.size())
    return fail(B200MD_ERR_ARG, "b200md_mgpu_get_local: bad domain index");
  Domain& D = *G.dom[k];
  const size_t s = (size_t)D.n_loc;
  if (type)
    MG_CUDA(cudaMemcpyAsync(type, D.type.p, sizeof(int) * s, cudaMemcpyDeviceToHost, G.stream));
  if (position)
    MG_CUDA(cudaMemcpyAsync(position, D.pos.p, sizeof(double) * 3 * s, cudaMemcpyDeviceToHost, G.stream));
  MG_CUDA(cudaStreamSynchronize(G.stream));
  if (h_out)
    std::memcpy(h_out, D.lh, sizeof D.lh);
  if (pbc_out)
    std::memcpy(pbc_out, D.lpbc, sizeof D.lpbc);
  return B200MD_OK;
}

int b200md_mgpu_profile(b200md_mgpu* g, int enable, double* ms_out, int max_out)
{
  Group& G = *g;
  int n = 0;
  if (ms_out && G.prof_steps > 0)
    for (; n < 4 && n < max_out; ++n)
      ms_out[n] = G.prof_ms[n] / G.prof_steps;
  G.prof = enable != 0;
  for (double& v : G.prof_ms)
    v = 0.0;
  G.prof_steps = 0;
  return n;
}

int b200md_mgpu_check(b200md_mgpu* g)
{
  for (auto& dp : g->dom)
    if (dp->n_loc > 0)
      MG_TRY(dp->pot.check(g->stream));
  return B200MD_OK;
}

} // extern "C"

// b2_rdf.cu -- radial distribution function (compute_rdf): kernels and C-ABI (see b2_rdf.cuh).
//
// One sample = the neighbour module's cell sort with cells of at least rc / 2 (no skin list), one
// counting kernel, one fold kernel.  Nothing is copied to the host and nothing synchronises per sample;
// b200md_rdf_finish does the only copy.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_neighbor_host.h"
#include "b2_rdf.cuh"
#include <vector>

using namespace b2;

namespace {

constexpr int RDF_BLK = 128;
// the block-private table of 32-bit counters ([num_pairs][num_bins]) is used when it fits this budget;
// larger tables (many species) count with 64-bit global atomics directly
constexpr size_t RDF_SMEM_BUDGET = 64 * 1024;

// warp-aggregated increment: lanes that hit the same counter add once (a crystal puts whole warps in
// one shell)
template <bool SHARED>
__device__ __forceinline__ void rdf_add(unsigned* sh, unsigned long long* gl, int k)
{
  const unsigned peers = __match_any_sync(__activemask(), k);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) {
    if (SHARED)
      atomicAdd(sh + k, (unsigned)__popc(peers));
    else
      atomicAdd(gl + k, (unsigned long long)__popc(peers));
  }
}

// block b counts the pairs of the sorted atoms [b chunk, (b+1) chunk)
template <bool SHARED>
__global__ void __launch_bounds__(RDF_BLK, 8) k_rdf_count(
  int n, int chunk, const B2Atom* __restrict__ atoms, const int* __restrict__ cell_start, B2Box box, B2Grid g,
  B2RdfPara p, const int* __restrict__ species_g, unsigned long long* __restrict__ counts)
{
  extern __shared__ unsigned table[];
  __shared__ int species[B2_MAX_TYPES];
  const int table_size = p.num_pairs * p.num_bins;
  for (int t = threadIdx.x; t < B2_MAX_TYPES; t += RDF_BLK)
    species[t] = species_g[t];
  if (SHARED)
    for (int k = threadIdx.x; k < table_size; k += RDF_BLK)
      table[k] = 0;
  __syncthreads();
  const int i0 = blockIdx.x * chunk;
  const int i1 = min(n, i0 + chunk);
  for (int i = i0 + threadIdx.x; i < i1; i += RDF_BLK)
    b2_body_rdf_atom(i, atoms, cell_start, box, g, p, species,
                     [&](int k) { rdf_add<SHARED>(table, counts, k); });
  if (SHARED) {
    __syncthreads();
    for (int k = threadIdx.x; k < table_size; k += RDF_BLK) {
      const unsigned c = table[k];
      if (c)
        atomicAdd(counts + k, (unsigned long long)c);
    }
  }
}

__global__ void k_rdf_fold(
  B2RdfPara p, double volume, int n, const int* __restrict__ num_atoms, unsigned long long* counts, double* acc)
{
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w < p.num_bins)
    b2_body_rdf_fold(w, p, volume, n, num_atoms, counts, acc);
}

} // namespace

struct b200md_rdf {
  B2RdfPara para;
  double rc = 0.0;
  int n = 0;
  std::vector<int> type_index, num_atoms;
  Neighbor cells;
  DevBuf<int> species, d_num_atoms;
  DevBuf<unsigned long long> counts; // [num_pairs][num_bins], zero between samples
  DevBuf<double> acc;                // [num_bins][1 + num_pairs]
  bool shared = false;
  size_t smem = 0;
  int grid = 0, chunk = 0;
  long long samples = 0;
};

namespace {

int rdf_setup(b200md_rdf* p)
{
  const B2RdfPara& q = p->para;
  const size_t table = (size_t)q.num_pairs * q.num_bins;
  const int rc_init = p->cells.init(p->n, p->rc, 0); // cells only: no skin list entries
  if (rc_init != B200MD_OK)
    return rc_init;
  B2_CUDA(p->counts.reserve(table));
  B2_CUDA(p->acc.reserve((size_t)q.num_bins * (1 + q.num_pairs)));
  B2_CUDA(p->species.reserve(B2_MAX_TYPES));
  B2_CUDA(p->d_num_atoms.reserve(q.num_types));
  B2_CUDA(cudaMemset(p->counts.p, 0, table * sizeof(unsigned long long)));
  B2_CUDA(cudaMemset(p->acc.p, 0, (size_t)q.num_bins * (1 + q.num_pairs) * sizeof(double)));
  std::vector<int> sp(B2_MAX_TYPES, -1);
  for (int a = 0; a < q.num_types; ++a)
    sp[p->type_index[a]] = a;
  B2_CUDA(cudaMemcpy(p->species.p, sp.data(), sizeof(int) * B2_MAX_TYPES, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(p->d_num_atoms.p, p->num_atoms.data(), sizeof(int) * q.num_types, cudaMemcpyHostToDevice));

  p->smem = table * sizeof(unsigned);
  p->shared = p->smem <= RDF_SMEM_BUDGET;
  int dev = 0, sms = 0, per_sm = 0;
  B2_CUDA(cudaGetDevice(&dev));
  B2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (p->shared) {
    // the whole budget, not this table's size: the attribute belongs to the kernel, and a later object
    // with a smaller table must not lower the limit under an earlier object's launches
    B2_CUDA(cudaFuncSetAttribute(k_rdf_count<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)RDF_SMEM_BUDGET));
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rdf_count<true>, RDF_BLK, p->smem));
  } else {
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rdf_count<false>, RDF_BLK, 0));
  }
  long long grid = (long long)sms * (per_sm > 0 ? per_sm : 1);
  // a block's 32-bit counters hold at most chunk * (n - 1) pairs: more blocks where that could overflow
  const long long cap = 4294967295LL / (p->n > 1 ? p->n - 1 : 1);
  if (p->shared && (p->n + grid - 1) / grid > cap)
    grid = (p->n + cap - 1) / cap;
  if (grid > p->n)
    grid = p->n;
  p->chunk = (int)((p->n + grid - 1) / grid);
  p->grid = grid_for(p->n, p->chunk);
  return B200MD_OK;
}

} // namespace

extern "C" {

int b200md_rdf_create(
  double rc, int num_bins, int num_types, const int* type_index, const int* num_atoms, int n, b200md_rdf** out)
{
  if (!out || !type_index || !num_atoms || n < 1) {
    set_error("b200md_rdf_create: bad argument");
    return B200MD_ERR_ARG;
  }
  *out = nullptr;
  if (!(rc > 0)) { // rdf.cu:280-282
    set_error("b200md_rdf_create: radial cutoff should be positive.");
    return B200MD_ERR_ARG;
  }
  if (num_bins <= 20) { // rdf.cu:298-304
    set_error("b200md_rdf_create: A larger nbins is recommended.");
    return B200MD_ERR_ARG;
  }
  if (num_bins > 500) {
    set_error("b200md_rdf_create: A smaller nbins is recommended.");
    return B200MD_ERR_ARG;
  }
  if (num_types < 1 || num_types > B2_MAX_TYPES) {
    set_error("b200md_rdf_create: the number of species must be in 1 .. 94");
    return B200MD_ERR_ARG;
  }
  long long sum = 0;
  for (int a = 0; a < num_types; ++a) {
    if (type_index[a] < 0 || type_index[a] >= B2_MAX_TYPES || (a > 0 && type_index[a] <= type_index[a - 1])) {
      set_error("b200md_rdf_create: type_index must ascend strictly within 0 .. 93");
      return B200MD_ERR_ARG;
    }
    if (num_atoms[a] < 1) {
      set_error("b200md_rdf_create: every species listed must have at least one atom");
      return B200MD_ERR_ARG;
    }
    sum += num_atoms[a];
  }
  if (sum != n) {
    set_error("b200md_rdf_create: the species' atom counts do not add up to n");
    return B200MD_ERR_ARG;
  }
  b200md_rdf* p = new b200md_rdf;
  p->para.num_bins = num_bins;
  p->para.num_types = num_types;
  p->para.num_pairs = num_types * (num_types + 1) / 2;
  p->para.dr = rc / num_bins;  // rdf.cu:326
  p->para.rc2 = rc * rc;       // rdf.cu:325
  p->rc = rc;
  p->n = n;
  p->type_index.assign(type_index, type_index + num_types);
  p->num_atoms.assign(num_atoms, num_atoms + num_types);
  const int rc_setup = rdf_setup(p);
  if (rc_setup != B200MD_OK) {
    delete p;
    return rc_setup;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_rdf_destroy(b200md_rdf* p) { delete p; }

int b200md_rdf_sample(
  b200md_rdf* p, const double* box_h, const int* pbc, const int* d_type, const double* d_pos, int n, void* stream)
{
  if (!p || !box_h || !pbc || !d_type || !d_pos) {
    set_error("b200md_rdf_sample: bad argument");
    return B200MD_ERR_ARG;
  }
  if (n != p->n) {
    set_error("b200md_rdf_sample: n differs from the n given at creation");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const B2Box box = make_box(box_h, pbc);
  const B2RdfPara& q = p->para;
  const int rc_sort = p->cells.sort_cells(box, d_type, d_pos, n, 0.5 * p->rc, st); // rdf.cu:131
  if (rc_sort != B200MD_OK)
    return rc_sort;
  const B2NeighborView v = p->cells.view();
  if (p->shared)
    k_rdf_count<true><<<p->grid, RDF_BLK, p->smem, st>>>(n, p->chunk, v.atoms, v.cell_start, box, p->cells.grid, q,
                                                         p->species.p, p->counts.p);
  else
    k_rdf_count<false><<<p->grid, RDF_BLK, 0, st>>>(n, p->chunk, v.atoms, v.cell_start, box, p->cells.grid, q,
                                                    p->species.p, p->counts.p);
  B2_LAUNCHED();
  // rdf.cu:196-199: the volume of this sample
  k_rdf_fold<<<grid_for(q.num_bins, 128), 128, 0, st>>>(q, box.volume, n, p->d_num_atoms.p, p->counts.p, p->acc.p);
  B2_LAUNCHED();
  ++p->samples;
  return B200MD_OK;
}

int b200md_rdf_finish(b200md_rdf* p, int num_repeats, double* out, void* stream)
{
  if (!p || !out) {
    set_error("b200md_rdf_finish: bad argument");
    return B200MD_ERR_ARG;
  }
  if (num_repeats < 1) {
    set_error("b200md_rdf_finish: num_repeats must be positive (the run has no full sampling interval)");
    return B200MD_ERR_ARG;
  }
  const size_t count = (size_t)p->para.num_bins * (1 + p->para.num_pairs);
  cudaStream_t st = (cudaStream_t)stream;
  B2_CUDA(cudaMemcpyAsync(out, p->acc.p, count * sizeof(double), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  for (size_t k = 0; k < count; ++k) // rdf.cu:236-247
    out[k] /= num_repeats;
  return B200MD_OK;
}

} // extern "C"

// b2_neighbor.cu -- kernels and host driver for the cell-sorted skin list (see b2_neighbor.cuh).
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_neighbor.cuh"
#include "b2_neighbor_host.h"

namespace b2 {

namespace {

constexpr int BLK = 256;

__global__ void k_init_perm(int n, int* perm, int* flags)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    perm[i] = i;
  if (i == 0) {
    flags[0] = 1; // first call always builds
    flags[1] = 0;
    flags[2] = 0;
  }
}

__global__ void k_force_rebuild(int* flags) { flags[0] = 1; }

__global__ void k_reset_perm(int n, int* perm, int* flags)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    perm[i] = i;
  if (i == 0)
    flags[0] = 1;
}

__global__ void __launch_bounds__(BLK) k_pack_check(
  B2NeighborView v, B2Box box, const int* __restrict__ type, const double* __restrict__ x,
  const double* __restrict__ y, const double* __restrict__ z, float trigger_d2)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < v.n)
    b2_body_pack_check(i, v, box, type, x, y, z, trigger_d2);
}

// ---- everything below runs only when flags[0] != 0 -----------------------------------------

__global__ void __launch_bounds__(BLK) k_zero_cells(B2NeighborView v, int ncell)
{
  if (!v.flags[0])
    return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < ncell) {
    v.cell_count[c] = 0;
    v.cell_fill[c] = 0;
  }
}

__global__ void __launch_bounds__(BLK) k_cell_count(B2NeighborView v, B2Box box, B2Grid g)
{
  if (!v.flags[0])
    return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < v.n) {
    int cx, cy, cz;
    const int c = b2_cell_of(box, g, v.atoms[i], &cx, &cy, &cz);
    v.cell_of[i] = c;
    atomicAdd(&v.cell_count[c], 1);
  }
}

// single-block (1024 threads) exclusive scan of in(0 .. count-1) into out[0 .. count]: tiles of 1024*4
// with a running carry
template <class In>
__device__ __forceinline__ void block_scan_1024(int count, int* out, In in)
{
  const int ncell = count;
  __shared__ int warp_sums[32];
  __shared__ int carry_s;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0)
    carry_s = 0;
  __syncthreads();
  for (int base = 0; base < ncell; base += 4096) {
    const int idx = base + tid * 4;
    int a[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      a[k] = (idx + k < ncell) ? in(idx + k) : 0;
    const int mine = a[0] + a[1] + a[2] + a[3];
    int incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o)
        incl += t;
    }
    if (lane == 31)
      warp_sums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      int w = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o)
          w += t;
      }
      warp_sums[lane] = w; // inclusive over warps
    }
    __syncthreads();
    const int carry = carry_s;
    int excl = carry + (wid ? warp_sums[wid - 1] : 0) + incl - mine;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (idx + k < ncell)
        out[idx + k] = excl;
      excl += a[k];
    }
    __syncthreads();
    if (tid == 1023)
      carry_s = carry + warp_sums[31];
    __syncthreads();
  }
  if (tid == 0)
    out[ncell] = carry_s;
}

__global__ void __launch_bounds__(1024) k_scan_cells(B2NeighborView v, int ncell)
{
  if (!v.flags[0])
    return;
  block_scan_1024(ncell, v.cell_start, [&](int c) { return v.cell_count[c]; });
}

__global__ void __launch_bounds__(BLK) k_cell_fill(B2NeighborView v)
{
  if (!v.flags[0])
    return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < v.n) {
    const int c = v.cell_of[i];
    const int slot = v.cell_start[c] + atomicAdd(&v.cell_fill[c], 1);
    v.order_tmp[slot] = i;
  }
}

__global__ void __launch_bounds__(BLK) k_sort_cells(B2NeighborView v, int ncell)
{
  if (!v.flags[0])
    return;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < ncell)
    b2_body_sort_cell(c, v);
}

__global__ void __launch_bounds__(BLK) k_commit(B2NeighborView v)
{
  if (!v.flags[0])
    return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < v.n)
    b2_body_commit(i, v);
}

__global__ void __launch_bounds__(128)
  k_skin_list(B2NeighborView v, B2Box box, B2Grid g, float cutoff2)
{
  if (!v.flags[0])
    return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < v.n)
    b2_body_skin_list(i, v, box, g, cutoff2);
}

__global__ void __launch_bounds__(128) k_skin_reverse(B2NeighborView v)
{
  if (!v.flags[0])
    return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < v.n)
    b2_body_skin_reverse(i, v);
}

// ---- type tiles: stable counting sort of the sorted atoms by type, buckets padded to 128 ------
// rank of this thread's atom among the same-type atoms of its block (ascending thread order);
// leaves the per-warp counts in wcnt[warp][type]
__device__ __forceinline__ int block_rank_by_type(
  int t, bool valid, int nt, int (*wcnt)[B2_MAX_TYPES + 2], int& before_warp)
{
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  for (int k = tid; k < (BLK / 32) * (B2_MAX_TYPES + 2); k += BLK)
    (&wcnt[0][0])[k] = 0;
  __syncthreads();
  const unsigned act = __ballot_sync(0xffffffffu, valid);
  int rank = 0;
  if (valid) {
    const unsigned peers = __match_any_sync(act, t);
    rank = __popc(peers & ((1u << lane) - 1u));
    if (rank == 0)
      wcnt[w][t] = __popc(peers);
  }
  __syncthreads();
  before_warp = 0;
  if (valid)
    for (int k = 0; k < w; ++k)
      before_warp += wcnt[k][t];
  return rank;
}

__global__ void __launch_bounds__(BLK) k_tile_count(B2NeighborView v)
{
  if (!v.flags[0])
    return;
  __shared__ int wcnt[BLK / 32][B2_MAX_TYPES + 2];
  const int i = blockIdx.x * BLK + threadIdx.x;
  for (int s = i; s < v.tile_nslot; s += gridDim.x * BLK)
    v.tile_atom[s] = -1;
  const bool valid = i < v.n;
  int before;
  block_rank_by_type(valid ? v.atoms[i].type : 0, valid, v.tile_nt, wcnt, before);
  if (threadIdx.x < v.tile_nt) {
    int c = 0;
    for (int k = 0; k < BLK / 32; ++k)
      c += wcnt[k][threadIdx.x];
    v.tile_blk[(size_t)threadIdx.x * v.tile_nblk + blockIdx.x] = c;
  }
}

// one warp per type: exclusive scan of the block counts; then bucket bases and tile types
__global__ void __launch_bounds__(1024) k_tile_scan(B2NeighborView v)
{
  if (!v.flags[0])
    return;
  __shared__ int count[B2_MAX_TYPES + 2], base[B2_MAX_TYPES + 2];
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  for (int t = w; t < v.tile_nt; t += 32) {
    int* c = v.tile_blk + (size_t)t * v.tile_nblk;
    int run = 0;
    for (int b0 = 0; b0 < v.tile_nblk; b0 += 32) {
      const int b = b0 + lane;
      const int mine = b < v.tile_nblk ? c[b] : 0;
      int inc = mine;
      for (int o = 1; o < 32; o <<= 1) {
        const int up = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o)
          inc += up;
      }
      if (b < v.tile_nblk)
        c[b] = run + inc - mine;
      run += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0)
      count[t] = run;
  }
  __syncthreads();
  if (tid == 0) {
    int slot = 0;
    for (int t = 0; t < v.tile_nt; ++t) {
      base[t] = slot;
      v.tile_meta[1 + t] = slot;
      slot += (count[t] + 127) / 128 * 128;
    }
    base[v.tile_nt] = slot;
    v.tile_meta[0] = slot / 128;
  }
  __syncthreads();
  const int ntile = base[v.tile_nt] / 128;
  for (int k = tid; k < ntile; k += 1024) {
    int t = 0;
    while (t + 1 < v.tile_nt && base[t + 1] <= k * 128)
      ++t;
    v.tile_type[k] = t;
  }
}

__global__ void __launch_bounds__(BLK) k_tile_fill(B2NeighborView v)
{
  if (!v.flags[0])
    return;
  __shared__ int wcnt[BLK / 32][B2_MAX_TYPES + 2];
  const int i = blockIdx.x * BLK + threadIdx.x;
  const bool valid = i < v.n;
  const int t = valid ? v.atoms[i].type : 0;
  int before;
  const int rank = block_rank_by_type(t, valid, v.tile_nt, wcnt, before);
  if (valid)
  {
    const int slot = v.tile_meta[1 + t] + v.tile_blk[(size_t)t * v.tile_nblk + blockIdx.x] + before + rank;
    v.tile_atom[slot] = i;
    v.tile_slot[i] = slot;
  }
}

// ---- warp schedule (b2_neighbor.cuh): segments per brick -> first position of each brick -> order ----
__global__ void __launch_bounds__(1024) k_brick_scan(B2NeighborView v, B2Grid g, B2Bricks br)
{
  if (!v.flags[0])
    return;
  block_scan_1024(br.count, v.brick_start, [&](int b) { return b2_body_brick_count(b, v, g, br); });
}

__global__ void __launch_bounds__(BLK) k_seg_order(B2NeighborView v, B2Grid g, B2Bricks br)
{
  if (!v.flags[0])
    return;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < br.count)
    b2_body_seg_order(b, v, g, br);
}

__global__ void k_rebuild_done(int* flags)
{
  if (flags[0]) {
    flags[0] = 0;
    flags[2] += 1;
  }
}

} // namespace

B2Grid make_grid(const B2Box& box, double cell_size)
{
  B2Grid g;
  for (int d = 0; d < 3; ++d) {
    int nb = (int)floor(box.thickness[d] / cell_size);
    if (nb < 1)
      nb = 1;
    g.nb[d] = nb;
    g.scale[d] = (double)nb;
  }
  g.ncell = g.nb[0] * g.nb[1] * g.nb[2];
  return g;
}

int Neighbor::init(int num_atoms, double rc_, int mn_skin_)
{
  n = num_atoms;
  capacity = num_atoms;
  rc = rc_;
  mn_skin = mn_skin_;
  B2_CUDA(atoms.reserve(n));
  B2_CUDA(atoms_tmp.reserve(n));
  B2_CUDA(snap.reserve((size_t)3 * n));
  B2_CUDA(snap_type.reserve(n));
  B2_CUDA(perm.reserve(n));
  B2_CUDA(perm_tmp.reserve(n));
  B2_CUDA(cell_of.reserve(n));
  B2_CUDA(order_tmp.reserve(n));
  B2_CUDA(nn_skin.reserve(n));
  B2_CUDA(nl_skin.reserve((size_t)skin_pitch() * n));
  B2_CUDA(flags.reserve(4));
  B2_CUDA(cudaMemset(snap.p, 0, sizeof(double) * 3 * (size_t)n));
  B2_CUDA(cudaMemset(snap_type.p, 0, sizeof(int) * (size_t)n));
  k_init_perm<<<grid_for(n, BLK), BLK>>>(n, perm.p, flags.p);
  B2_LAUNCHED();
  have_grid = false;
  return B200MD_OK;
}

B2NeighborView Neighbor::view() const
{
  B2NeighborView v;
  v.n = n;
  v.mn_skin = mn_skin;
  v.atoms = atoms.p;
  v.atoms_tmp = atoms_tmp.p;
  v.plane0 = planes ? plane0.p : nullptr;
  v.plane1 = planes ? plane1.p : nullptr;
  v.planez = planes ? planez.p : nullptr;
  v.tag_types = tag_types ? 1 : 0;
  v.rskin = reverse ? rskin.p : nullptr;
  v.snap = snap.p;
  v.snap_type = snap_type.p;
  v.perm = perm.p;
  v.perm_tmp = perm_tmp.p;
  v.cell_of = cell_of.p;
  v.order_tmp = order_tmp.p;
  v.cell_count = cell_count.p;
  v.cell_fill = cell_fill.p;
  v.cell_start = cell_start.p;
  v.nn_skin = nn_skin.p;
  v.nl_skin = nl_skin.p;
  v.skin_si = skin_row_major ? (size_t)skin_pitch() : 1;
  v.skin_sk = skin_row_major ? 1 : (size_t)n;
  v.flags = flags.p;
  v.tile_nt = tile_nt;
  v.tile_nblk = grid_for(n, BLK);
  v.tile_nslot = n + 128 * tile_nt;
  v.tile_atom = tile_atom.p;
  v.tile_slot = tile_slot.p;
  v.tile_type = tile_type.p;
  v.tile_blk = tile_blk.p;
  v.tile_meta = tile_meta.p;
  v.seg_order = schedule ? seg_order.p : nullptr;
  v.brick_start = brick_start.p;
  return v;
}

int Neighbor::update(
  const B2Box& box, const int* d_type, const double* d_pos, int n_in, cudaStream_t st)
{
  if (n_in <= 0) {
    set_error("no atoms: the neighbour list needs at least one");
    return B200MD_ERR_ARG;
  }
  if (n_in > capacity) {
    set_error("number of atoms exceeds the capacity given at construction");
    return B200MD_ERR_ARG;
  }
  if (n_in != n) {
    const int rc_inv = invalidate(n_in, st);
    if (rc_inv != B200MD_OK)
      return rc_inv;
  }
  // the cell list needs >= 5 half-(rc+skin) cells per periodic direction.  b200md_nep_compute never
  // gets here with a thinner box (it evaluates a supercell instead); LJ / Tersoff / EAM do
  for (int d = 0; d < 3; ++d) {
    if (box.pbc[d] && box.thickness[d] <= 2.5 * (rc + skin)) {
      set_error(
        "periodic box thickness <= 2.5*(rc+1): small boxes are supported for NEP only (supercell "
        "path); this potential needs a larger box or a replicated cell");
      return B200MD_ERR_SMALL_BOX;
    }
  }
  const B2Grid g = make_grid(box, 0.5 * (rc + skin));
  for (int d = 0; d < 3; ++d) {
    if (box.pbc[d] && g.nb[d] < 5) {
      set_error("internal: fewer than 5 cells in a periodic direction");
      return B200MD_ERR_SMALL_BOX;
    }
  }
  if ((size_t)g.ncell + 1 > cell_start.n) {
    const size_t cap = (size_t)(g.ncell * 1.2) + 64;
    B2_CUDA(cudaStreamSynchronize(st));
    B2_CUDA(cell_count.reserve(cap));
    B2_CUDA(cell_fill.reserve(cap));
    B2_CUDA(cell_start.reserve(cap + 1));
    if (schedule)
      B2_CUDA(brick_start.reserve(cap + 1)); // never more bricks than cells
  }
  if (have_grid && (g.nb[0] != grid.nb[0] || g.nb[1] != grid.nb[1] || g.nb[2] != grid.nb[2])) {
    k_force_rebuild<<<1, 1, 0, st>>>(flags.p);
    B2_LAUNCHED();
  }
  grid = g;
  have_grid = true;

  const B2NeighborView v = view();
  const double* x = d_pos;
  const double* y = d_pos + n;
  const double* z = d_pos + 2 * (size_t)n;
  const float trigger = (float)(skin * skin * 0.25);
  const float cutoff = (float)((rc + skin) * (rc + skin));
  const int gn = grid_for(n, BLK), gc = grid_for(g.ncell, BLK);

  k_pack_check<<<gn, BLK, 0, st>>>(v, box, d_type, x, y, z, trigger);
  B2_LAUNCHED();
  k_zero_cells<<<gc, BLK, 0, st>>>(v, g.ncell);
  B2_LAUNCHED();
  k_cell_count<<<gn, BLK, 0, st>>>(v, box, g);
  B2_LAUNCHED();
  k_scan_cells<<<1, 1024, 0, st>>>(v, g.ncell);
  B2_LAUNCHED();
  k_cell_fill<<<gn, BLK, 0, st>>>(v);
  B2_LAUNCHED();
  k_sort_cells<<<gc, BLK, 0, st>>>(v, g.ncell);
  B2_LAUNCHED();
  k_commit<<<gn, BLK, 0, st>>>(v);
  B2_LAUNCHED();
  k_skin_list<<<grid_for(n, 128), 128, 0, st>>>(v, box, g, cutoff);
  B2_LAUNCHED();
  if (reverse) {
    k_skin_reverse<<<grid_for(n, 128), 128, 0, st>>>(v);
    B2_LAUNCHED();
  }
  if (tile_nt > 0) {
    k_tile_count<<<gn, BLK, 0, st>>>(v);
    B2_LAUNCHED();
    k_tile_scan<<<1, 1024, 0, st>>>(v);
    B2_LAUNCHED();
    k_tile_fill<<<gn, BLK, 0, st>>>(v);
    B2_LAUNCHED();
  }
  if (schedule) {
    const B2Bricks br = b2_make_bricks(g, n);
    k_brick_scan<<<1, 1024, 0, st>>>(v, g, br);
    B2_LAUNCHED();
    k_seg_order<<<grid_for(br.count, BLK), BLK, 0, st>>>(v, g, br);
    B2_LAUNCHED();
  }
  k_rebuild_done<<<1, 1, 0, st>>>(flags.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

int Neighbor::sort_cells(
  const B2Box& box, const int* d_type, const double* d_pos, int n_in, double cell_size, cudaStream_t st)
{
  if (n_in <= 0 || n_in > capacity) {
    set_error("sort_cells: the number of atoms must be in 1 .. the capacity given at construction");
    return B200MD_ERR_ARG;
  }
  if (n_in != n) {
    const int rc_inv = invalidate(n_in, st);
    if (rc_inv != B200MD_OK)
      return rc_inv;
  }
  const B2Grid g = make_grid(box, cell_size);
  for (int d = 0; d < 3; ++d) {
    if (box.pbc[d] && g.nb[d] < 5) {
      set_error("sort_cells: fewer than 5 cells in a periodic direction (box thinner than 2.5 cutoffs)");
      return B200MD_ERR_SMALL_BOX;
    }
  }
  if ((size_t)g.ncell + 1 > cell_start.n) {
    const size_t cap = (size_t)(g.ncell * 1.2) + 64;
    B2_CUDA(cudaStreamSynchronize(st));
    B2_CUDA(cell_count.reserve(cap));
    B2_CUDA(cell_fill.reserve(cap));
    B2_CUDA(cell_start.reserve(cap + 1));
  }
  grid = g;
  have_grid = true;
  const B2NeighborView v = view();
  const int gn = grid_for(n, BLK), gc = grid_for(g.ncell, BLK);
  k_force_rebuild<<<1, 1, 0, st>>>(flags.p);
  B2_LAUNCHED();
  k_pack_check<<<gn, BLK, 0, st>>>(v, box, d_type, d_pos, d_pos + n, d_pos + 2 * (size_t)n, 0.0f);
  B2_LAUNCHED();
  k_zero_cells<<<gc, BLK, 0, st>>>(v, g.ncell);
  B2_LAUNCHED();
  k_cell_count<<<gn, BLK, 0, st>>>(v, box, g);
  B2_LAUNCHED();
  k_scan_cells<<<1, 1024, 0, st>>>(v, g.ncell);
  B2_LAUNCHED();
  k_cell_fill<<<gn, BLK, 0, st>>>(v);
  B2_LAUNCHED();
  k_sort_cells<<<gc, BLK, 0, st>>>(v, g.ncell);
  B2_LAUNCHED();
  k_commit<<<gn, BLK, 0, st>>>(v);
  B2_LAUNCHED();
  k_rebuild_done<<<1, 1, 0, st>>>(flags.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

int Neighbor::enable_schedule()
{
  B2_CUDA(seg_order.reserve(((size_t)capacity + 31) / 32));
  schedule = true;
  return B200MD_OK;
}

int Neighbor::enable_planes()
{
  B2_CUDA(plane0.reserve(capacity));
  B2_CUDA(plane1.reserve(capacity));
  B2_CUDA(planez.reserve(capacity));
  planes = true;
  return B200MD_OK;
}

int Neighbor::enable_reverse()
{
  if (skin_row_major || tag_types) {
    set_error("enable_reverse: needs column-major, untagged skin lists");
    return B200MD_ERR_ARG;
  }
  B2_CUDA(rskin.reserve((size_t)capacity * mn_skin));
  reverse = true;
  return B200MD_OK;
}

int Neighbor::enable_type_tiles(int num_types)
{
  if (num_types < 1 || num_types > B2_MAX_TYPES) {
    set_error("enable_type_tiles: bad number of types");
    return B200MD_ERR_ARG;
  }
  tile_nt = num_types;
  B2_CUDA(tile_atom.reserve((size_t)capacity + 128 * (size_t)num_types));
  B2_CUDA(tile_slot.reserve((size_t)capacity));
  B2_CUDA(tile_type.reserve((size_t)capacity / 128 + num_types + 2));
  B2_CUDA(tile_blk.reserve((size_t)num_types * grid_for(capacity, BLK)));
  B2_CUDA(tile_meta.reserve(num_types + 2));
  return B200MD_OK;
}

int Neighbor::invalidate(int n_new, cudaStream_t st)
{
  if (n_new <= 0) {
    set_error("no atoms: the neighbour list needs at least one");
    return B200MD_ERR_ARG;
  }
  if (n_new > capacity) {
    set_error("number of atoms exceeds the capacity given at construction");
    return B200MD_ERR_ARG;
  }
  n = n_new;
  k_reset_perm<<<grid_for(n, BLK), BLK, 0, st>>>(n, perm.p, flags.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

int Neighbor::check(cudaStream_t st, int* err_bits, int* rebuilds)
{
  int host[4] = {0, 0, 0, 0};
  B2_CUDA(cudaMemcpyAsync(host, flags.p, sizeof(int) * 3, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  if (err_bits)
    *err_bits = host[1];
  if (rebuilds)
    *rebuilds = host[2];
  return B200MD_OK;
}

} // namespace b2

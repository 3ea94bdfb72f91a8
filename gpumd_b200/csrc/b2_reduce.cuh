// b2_reduce.cuh -- the one summation order of the deterministic grid reductions outside the force
// kernels (DESIGN.md "Deterministic reductions"): block totals of row k at partial[k * grid + b], summed
// by the last block to arrive.  The grid size is part of the order: it depends on the item count and a
// cap only.
#pragma once
#include "b2_host.h" // grid_for
#include <algorithm>
#include <stddef.h>

namespace b2 {

// a sum, or a maximum for rows that take one (their values are >= 0, so 0.0 is neutral for them too)
__device__ __forceinline__ double b2_combine(bool max, double a, double b) { return max ? fmax(a, b) : a + b; }

// Block stage: thread k stores the block's total of t[k] at out[k * out_stride]; bit k of MAXMASK makes
// row k a maximum.
template <int K, int BLK, unsigned MAXMASK = 0>
__device__ __forceinline__ void b2_block_totals(const double (&t)[K], double* out, size_t out_stride)
{
  static_assert(K <= BLK && BLK % 32 == 0, "one thread per row, whole warps");
  __shared__ double sm[K][BLK / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double v = t[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      v = b2_combine(MAXMASK >> k & 1u, v, __shfl_down_sync(0xffffffffu, v, o));
    if (lane == 0)
      sm[k][wid] = v;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    const int k = threadIdx.x;
    double v = 0.0;
    for (int w = 0; w < BLK / 32; ++w)
      v = b2_combine(MAXMASK >> k & 1u, v, sm[k][w]);
    out[k * out_stride] = v;
  }
}

// True in every thread of the block that arrives last; what every block stored before it arrived is
// then visible to it.  The last block re-arms the ticket for the next launch on the stream.
__device__ __forceinline__ bool b2_last_block(unsigned int* ticket)
{
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    if (last)
      *ticket = 0u;
  }
  __syncthreads();
  if (last)
    __threadfence();
  return last;
}

// One warp combines p[0 .. count): lane l takes items l, l + 32, ... in order from 0.0, then a
// shuffle-down tree; lane 0 holds the result.
__device__ __forceinline__ double b2_warp_ordered(const double* p, int count, bool max = false)
{
  double v = 0.0;
  for (int i = threadIdx.x & 31; i < count; i += 32)
    v = b2_combine(max, v, p[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = b2_combine(max, v, __shfl_down_sync(0xffffffffu, v, o));
  return v;
}

// Grid stage, in the last block: lane 0 of warp k % (BLK / 32) calls put(k, total of row k).  Ends
// with a barrier, so totals put in shared memory are visible to the whole block.
template <int K, int BLK, unsigned MAXMASK = 0, class Put>
__device__ __forceinline__ void b2_grid_totals(const double* partial, Put put)
{
  for (int k = threadIdx.x >> 5; k < K; k += BLK / 32) {
    const double v = b2_warp_ordered(partial + (size_t)k * gridDim.x, gridDim.x, MAXMASK >> k & 1u);
    if ((threadIdx.x & 31) == 0)
      put(k, v);
  }
  __syncthreads();
}

// blocks of a grid-stride reduction over n items: one per blk items, at least one, at most cap
inline int b2_reduce_blocks(int n, int blk, int cap) { return std::max(1, std::min(grid_for(n, blk), cap)); }

// scratch that callers allocate: a 64-byte ticket slot (zero before the first launch), then the partials
constexpr size_t B2_TICKET_BYTES = 64;
inline size_t b2_scratch_bytes(int rows, int blocks) { return B2_TICKET_BYTES + sizeof(double) * rows * blocks; }
inline unsigned int* b2_scratch_ticket(void* s) { return (unsigned int*)s; }
inline double* b2_scratch_partials(void* s) { return (double*)((char*)s + B2_TICKET_BYTES); }

} // namespace b2

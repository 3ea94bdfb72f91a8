// b2_neighbor_host.h -- host-side owner of the cell-sorted skin list (see b2_neighbor.cuh).
#pragma once
#include "b2_host.h"
#include "b2_neighbor.cuh"
#include "b2_setup.h"

namespace b2 {

class Neighbor
{
public:
  int n = 0;        // atoms of the current system (<= capacity)
  int capacity = 0; // atoms the buffers were sized for
  int mn_skin = 0;
  bool skin_row_major = false; // set before init(): rows of skin_pitch() ints instead of columns
  int skin_pitch() const { return (mn_skin + 7) / 8 * 8; }
  double rc = 0.0;
  double skin = 1.0; // src/force/neighbor.cuh:212
  B2Grid grid;
  bool have_grid = false;

  DevBuf<B2Atom> atoms, atoms_tmp;
  DevBuf<int4> plane0, plane1; // see B2NeighborView::plane0 (enable_planes)
  DevBuf<double> planez;
  bool planes = false;
  bool tag_types = false; // see B2NeighborView::tag_types (set before the first update)
  DevBuf<double> snap;
  DevBuf<int> snap_type, perm, perm_tmp, cell_of, order_tmp, cell_count, cell_fill, cell_start, nn_skin,
    nl_skin, flags;
  DevBuf<int> rskin;    // see B2NeighborView::rskin (enable_reverse)
  bool reverse = false;
  int tile_nt = 0; // type tiles (see B2NeighborView) are maintained when > 0
  DevBuf<int> tile_atom, tile_slot, tile_type, tile_blk, tile_meta;
  bool schedule = false; // see B2NeighborView::seg_order (enable_schedule)
  DevBuf<int> seg_order, brick_start;

  // Neighbor::initialize, src/force/neighbor.cu:824-833
  int init(int num_atoms, double rc, int mn_skin);
  // also keep the type-bucketed tile order up to date at every rebuild (num_types <= 94)
  int enable_type_tiles(int num_types);
  // also maintain the 16-byte planes of the sorted records (call after init)
  int enable_planes();
  // also maintain the reverse slots of the skin list (column-major, untagged lists; call after init)
  int enable_reverse();
  // also maintain the warp schedule seg_order at every rebuild (call after init)
  int enable_schedule();
  int num_segments() const { return (n + 31) / 32; }
  int max_tiles() const { return (n + 127) / 128 + tile_nt; }
  // Neighbor::find_neighbor_global, src/force/neighbor.cu:756-800 (fully asynchronous here)
  int update(const B2Box& box, const int* d_type, const double* d_pos, int n, cudaStream_t st);
  int check(cudaStream_t st, int* err_bits, int* rebuilds);
  // cells only, for consumers with their own pair loop (the RDF): re-sort the atoms by cells of at least
  // cell_size, every call, and build no skin list (init with mn_skin = 0).  atoms / cell_start / perm of
  // view() then hold the sorted records of d_pos; update() is not to be mixed with it on one object
  int sort_cells(const B2Box& box, const int* d_type, const double* d_pos, int n, double cell_size,
                 cudaStream_t st);
  // forget the current ordering and lists (the caller changed the atom set or its order)
  int invalidate(int n_new, cudaStream_t st);
  B2NeighborView view() const;
};

} // namespace b2

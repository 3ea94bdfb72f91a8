// b2_neighbor.cuh -- cell-sorted atoms + Verlet ("skin") list for libb200md.
//
// Replaces class Neighbor / find_cell_list / find_neighbor (src/force/neighbor.cu:42-349,
// 640-833, neighbor.cuh:76-136) with a different design:
//   * atoms are physically re-ordered by cell (counting sort, deterministic: ascending caller
//     index inside a cell) into 32-byte B2Atom records, so that one neighbour gather is one
//     sector and threads of a warp share neighbours through L1;
//   * the displacement test, the cell sort and the list build are all PREDICATED on a device
//     flag -- no host round trip per step (the reference does a blocking D2H every step,
//     neighbor.cu:741-754);
//   * the skin list is produced in ascending sorted-index order by construction (the 5x5x5 cell
//     walk visits wrapped cell ids in increasing order), which replaces the per-atom O(NN^2)
//     rank sort (neighbor.cuh:112-136) and keeps binary search valid downstream.
// Semantics kept from the reference: half-(rc+skin) cells searched +-2 (neighbor.cu:117-124,
// 316-317), FP32 membership test d2 < (rc+skin)^2 on FP64-subtracted displacements
// (neighbor.cu:146-152), skin = 1 A (neighbor.cuh:212), rebuild when any atom moved more than
// skin/2 (neighbor.cu:741-754, 776).
#pragma once
#include "b2_common.cuh"

struct B2Grid {
  int nb[3];   // bins per direction
  int ncell;   // nb[0]*nb[1]*nb[2]
  double scale[3]; // fractional coordinate -> bin
};

struct B2NeighborView {
  int n;             // atoms
  int mn_skin;       // skin-list capacity per atom
  B2Atom* atoms;     // [n] sorted records (current positions)
  B2Atom* atoms_tmp; // [n] scratch for re-ordering
  // optional 16-byte PLANES of the same records for the gather-heavy radial NEP kernels:
  // plane0[j] = {x, y}, plane1[j] = {z, type, pad}.  A warp-wide 128-bit gather then touches half as
  // many 128-byte lines as with the 32-byte records (8 atoms per line instead of 4); null = off
  int4* plane0 = nullptr;
  int4* plane1 = nullptr;
  double* planez = nullptr; // z alone (8 bytes, 16 atoms per line) for consumers that get the type elsewhere
  // 1: skin-list entries carry the neighbour's type in bits 30+ (entry = j | type << 30; needs
  //    n < 2^30 and <= 2 types).  The type of an atom is constant between rebuilds (a changed type
  //    rebuilds, b2_body_pack_check), and a consumer that reads it from the entry saves a gather.  Only
  //    the few-type NEP kernels ask for this.
  int tag_types = 0;
  double* snap;      // [3n] positions at the last rebuild, sorted order (x0,y0,z0 SoA)
  // [n] types at the last rebuild, sorted order: a changed type rebuilds, because the type tags of the skin
  // list and the type tiles are built from them.  Neighbor always keeps it; null (a view built without the
  // snapshot) = only displacements rebuild
  int* snap_type = nullptr;
  int* perm;        // [n] sorted index -> caller index
  int* perm_tmp;     // [n]
  int* cell_of;      // [n] cell id of sorted atom (valid during a rebuild)
  int* order_tmp;    // [n] old sorted index per new slot
  int* cell_count;   // [ncell_cap]
  int* cell_fill;    // [ncell_cap]
  int* cell_start;   // [ncell_cap+1]
  int* nn_skin;      // [n]
  int* nl_skin;      // entry k of atom i at nl_skin[i*skin_si + k*skin_sk]: column-major
                     // (si = 1, sk = n) for thread-per-atom kernels, row-major (si = pitch,
                     // sk = 1) for kernels that spread one atom's neighbours over lanes
  size_t skin_si = 1, skin_sk = 0;
  // optional (Neighbor::enable_reverse, column-major untagged lists only): rskin[k*n + i] = the slot of
  // atom i in the skin list of its k-th skin neighbour.  Built once per rebuild; lets a consumer that
  // needs the partner's view of a pair (the angular force reduction) skip the per-step binary search.
  int* rskin = nullptr;
  int* flags;        // [0] rebuild requested, [1] error bits, [2] rebuild counter
  // optional type tiles (Neighbor::enable_type_tiles): the sorted atoms bucketed by type, every
  // bucket padded to a multiple of 128 slots -- row blocks of the tensor-core hidden layer
  int tile_nt = 0;          // 0 = feature off
  int tile_nblk = 0;        // blocks of BLK atoms
  int tile_nslot = 0;       // n + 128 * tile_nt
  int* tile_atom = nullptr; // [tile_nslot] sorted atom index or -1 (padding)
  int* tile_slot = nullptr; // [n] slot of every sorted atom (inverse of tile_atom)
  int* tile_type = nullptr; // [tile_nslot / 128] type of each 128-slot tile
  int* tile_blk = nullptr;  // [tile_nt * tile_nblk] per-block counts, then offsets inside the bucket
  int* tile_meta = nullptr; // [0] number of tiles, [1 + t] first slot of type t
  // optional warp schedule (Neighbor::enable_schedule): a permutation of the SEGMENTS (the 32 consecutive
  // sorted atoms [32 s, 32 s + 32)) that puts the segments of one brick of cells next to each other, so
  // that the warps of a block, and the blocks resident on an SM, gather from the same neighbourhood.
  // No atom moves: a consumer maps warp w to atoms seg_order[w] * 32 + lane, and any permutation is correct
  int* seg_order = nullptr;   // [ceil(n / 32)]
  int* brick_start = nullptr; // [number of bricks] first position of each brick in seg_order
};

// Bricks of the schedule: bx x by x bz cells, numbered y fastest, then x, then z (consecutive blocks, which
// run at the same time on the same or nearby SMs, are then bricks stacked along y over the same cells in x:
// measured faster than x fastest, see DESIGN 6; z outermost keeps consecutive blocks close in memory).  by = bz = 2 rows; bx = the cells that 32
// atoms span at the mean density, so that the four warps of a 128-thread block are the four rows of one
// brick.
struct B2Bricks {
  int bx, by, bz;
  int nx, ny, nz; // bricks per direction
  int count;      // nx*ny*nz
};

inline B2Bricks b2_make_bricks(const B2Grid& g, int n)
{
  B2Bricks b;
  const long long span = ((long long)32 * g.ncell + n / 2) / n; // cells per segment, rounded
  b.bx = span < 1 ? 1 : (span > g.nb[0] ? g.nb[0] : (int)span);
  b.by = 2;
  b.bz = 2;
  b.nx = (g.nb[0] + b.bx - 1) / b.bx;
  b.ny = (g.nb[1] + b.by - 1) / b.by;
  b.nz = (g.nb[2] + b.bz - 1) / b.bz;
  b.count = b.nx * b.ny * b.nz;
  return b;
}

// ---- pack: caller SoA -> sorted B2Atom records, and displacement trigger -------------------
// (gpu_check_atom_distance, neighbor.cu:646-684; the trigger only needs to be conservative)
B2_HD void b2_store_planes(const B2NeighborView& v, int i, const B2Atom& a)
{
#if defined(__CUDA_ARCH__)
  if (v.plane0) {
    int4 lo, hi;
    lo.x = __double2loint(a.x);
    lo.y = __double2hiint(a.x);
    lo.z = __double2loint(a.y);
    lo.w = __double2hiint(a.y);
    hi.x = __double2loint(a.z);
    hi.y = __double2hiint(a.z);
    hi.z = a.type;
    hi.w = 0;
    v.plane0[i] = lo;
    v.plane1[i] = hi;
    v.planez[i] = a.z;
  }
#else
  (void)v;
  (void)i;
  (void)a;
#endif
}

B2_HD void b2_body_pack_check(
  int i, const B2NeighborView& v, const B2Box& box, const int* type, const double* x,
  const double* y, const double* z, float trigger_d2)
{
  const int src = v.perm[i];
  B2Atom a;
  a.x = x[src];
  a.y = y[src];
  a.z = z[src];
  a.type = type[src];
  a.pad = 0;
  v.atoms[i] = a;
  b2_store_planes(v, i, a);
  float dx = (float)(a.x - v.snap[i]);
  float dy = (float)(a.y - v.snap[(size_t)v.n + i]);
  float dz = (float)(a.z - v.snap[(size_t)2 * v.n + i]);
  b2_mic(box, dx, dy, dz);
  // a swapped or changed species (Monte Carlo moves between MD steps) rebuilds like a displacement
  if (dx * dx + dy * dy + dz * dz > trigger_d2 || (v.snap_type && a.type != v.snap_type[i]))
    v.flags[0] = 1; // benign race: every writer stores the same value
}

// ---- cell id of a record (find_cell_id, neighbor.cuh:76-110, with clamping for open
// directions instead of a single bin) ---------------------------------------------------------
B2_HD int b2_cell_of(const B2Box& box, const B2Grid& g, const B2Atom& a, int* cx, int* cy, int* cz)
{
  const double sx = box.h[9] * a.x + box.h[10] * a.y + box.h[11] * a.z;
  const double sy = box.h[12] * a.x + box.h[13] * a.y + box.h[14] * a.z;
  const double sz = box.h[15] * a.x + box.h[16] * a.y + box.h[17] * a.z;
  int c[3];
  c[0] = (int)floor(sx * g.scale[0]);
  c[1] = (int)floor(sy * g.scale[1]);
  c[2] = (int)floor(sz * g.scale[2]);
  for (int d = 0; d < 3; ++d) {
    if (box.pbc[d]) {
      c[d] %= g.nb[d];
      if (c[d] < 0)
        c[d] += g.nb[d];
    } else {
      if (c[d] < 0)
        c[d] = 0;
      if (c[d] >= g.nb[d])
        c[d] = g.nb[d] - 1;
    }
  }
  *cx = c[0];
  *cy = c[1];
  *cz = c[2];
  return c[0] + g.nb[0] * (c[1] + g.nb[1] * c[2]);
}

// ---- per-cell ordering: ascending caller index => run-to-run deterministic layout ----------
B2_HD void b2_body_sort_cell(int c, const B2NeighborView& v)
{
  const int s0 = v.cell_start[c], s1 = v.cell_start[c + 1];
  for (int a = s0 + 1; a < s1; ++a) { // insertion sort, cells hold a handful of atoms
    const int o = v.order_tmp[a];
    const int key = v.perm[o];
    int q = a - 1;
    while (q >= s0 && v.perm[v.order_tmp[q]] > key) {
      v.order_tmp[q + 1] = v.order_tmp[q];
      --q;
    }
    v.order_tmp[q + 1] = o;
  }
  for (int a = s0; a < s1; ++a) {
    const int o = v.order_tmp[a];
    v.perm_tmp[a] = v.perm[o];
    v.atoms_tmp[a] = v.atoms[o];
  }
}

B2_HD void b2_body_commit(int i, const B2NeighborView& v)
{
  const B2Atom a = v.atoms_tmp[i];
  v.atoms[i] = a;
  b2_store_planes(v, i, a);
  v.perm[i] = v.perm_tmp[i];
  v.snap[i] = a.x;
  v.snap[(size_t)v.n + i] = a.y;
  v.snap[(size_t)2 * v.n + i] = a.z;
  if (v.snap_type)
    v.snap_type[i] = a.type;
}

// Offsets -2..+2 of one direction arranged so that the WRAPPED coordinate ascends.
B2_HD void b2_axis_walk(int c, int nb, int pbc, int out[5], int* cnt)
{
  int m = 0;
  if (!pbc) {
    for (int o = -2; o <= 2; ++o) {
      const int k = c + o;
      if (k >= 0 && k < nb)
        out[m++] = k;
    }
  } else {
    // wrapped values of c-2..c+2 (nb >= 5 guaranteed, so they are distinct); emit ascending
    int first = c - 2;
    if (first < 0) {
      // coordinates 0..c+2 come first, then the wrapped tail nb+first..nb-1
      for (int k = 0; k <= c + 2; ++k)
        out[m++] = k;
      for (int k = nb + first; k < nb; ++k)
        out[m++] = k;
    } else if (c + 2 >= nb) {
      for (int k = 0; k <= c + 2 - nb; ++k)
        out[m++] = k;
      for (int k = first; k < nb; ++k)
        out[m++] = k;
    } else {
      for (int k = first; k <= c + 2; ++k)
        out[m++] = k;
    }
  }
  *cnt = m;
}

// ---- skin list (gpu_find_neighbor_ON1, neighbor.cu:85-162) ---------------------------------
B2_HD void b2_body_skin_list(
  int i, const B2NeighborView& v, const B2Box& box, const B2Grid& g, float cutoff2)
{
  const B2Geo geo = b2_geo(box);
  const B2Atom a1 = v.atoms[i];
  int cx, cy, cz;
  b2_cell_of(box, g, a1, &cx, &cy, &cz);
  int wx[5], wy[5], wz[5], nx, ny, nz;
  b2_axis_walk(cx, g.nb[0], box.pbc[0], wx, &nx);
  b2_axis_walk(cy, g.nb[1], box.pbc[1], wy, &ny);
  b2_axis_walk(cz, g.nb[2], box.pbc[2], wz, &nz);
  int count = 0;
  for (int kz = 0; kz < nz; ++kz) {
    for (int ky = 0; ky < ny; ++ky) {
      const int row = g.nb[0] * (wy[ky] + g.nb[1] * wz[kz]);
      for (int kx = 0; kx < nx; ++kx) {
        const int cell = row + wx[kx];
        const int s1 = v.cell_start[cell + 1];
        for (int j = v.cell_start[cell]; j < s1; ++j) {
          if (j == i)
            continue;
          float x12, y12, z12;
          const B2Atom a2 = v.atoms[j];
          b2_r12(geo, box, a1, a2, x12, y12, z12);
          if (b2_d2(x12, y12, z12) < cutoff2) {
            if (count < v.mn_skin)
              v.nl_skin[(size_t)i * v.skin_si + (size_t)count * v.skin_sk] =
                v.tag_types ? (j | (a2.type << 30)) : j;
            ++count;
          }
        }
      }
    }
  }
  if (count > v.mn_skin) {
    B2_ATOMIC_OR(&v.flags[1], (int)B2_ERR_SKIN_OVERFLOW);
    count = v.mn_skin;
  }
  v.nn_skin[i] = count;
}

// ---- reverse slots of the skin list (the relation is symmetric: FP32 distances are exact mirror
//      images under i <-> j) -------------------------------------------------------------------
B2_HD void b2_body_skin_reverse(int i, const B2NeighborView& v)
{
  const size_t N = (size_t)v.n;
  const int nn = v.nn_skin[i];
  for (int k = 0; k < nn; ++k) {
    const int j = v.nl_skin[(size_t)k * N + i];
    int lo = 0, hi = v.nn_skin[j] - 1, rev = 0;
    while (lo <= hi) { // j's list is ascending
      const int mid = (lo + hi) >> 1;
      const int v2 = v.nl_skin[(size_t)mid * N + j];
      if (v2 < i)
        lo = mid + 1;
      else if (v2 > i)
        hi = mid - 1;
      else {
        rev = mid;
        break;
      }
    }
    v.rskin[(size_t)k * N + i] = rev;
  }
}

// ---- warp schedule ---------------------------------------------------------------------------
// Order of the segments: by the brick (cz / bz, cx / bx, cy / by) of the cell of the segment's FIRST atom,
// inside a brick by (cz % bz, cy % by, cx), ties by segment number.  The atoms are sorted by cell with x
// fastest, so the segments that start in the cells [c0, c1) of one row are the consecutive numbers
// ceil(cell_start[c0] / 32) .. ceil(cell_start[c1] / 32) - 1: the order follows from cell_start alone,
// without a sort.  fn(s) is called for the segments of brick b in that order; returns their number.
template <class Fn>
B2_HD int b2_brick_segments(int b, const B2Grid& g, const B2Bricks& br, const int* cell_start, Fn fn)
{
  const int ky = b % br.ny, kx = (b / br.ny) % br.nx, kz = b / (br.nx * br.ny);
  const int x0 = kx * br.bx, x1 = x0 + br.bx < g.nb[0] ? x0 + br.bx : g.nb[0];
  int count = 0;
  for (int rz = 0; rz < br.bz; ++rz) {
    for (int ry = 0; ry < br.by; ++ry) {
      const int cy = ky * br.by + ry, cz = kz * br.bz + rz;
      if (cy >= g.nb[1] || cz >= g.nb[2])
        continue;
      const int row = g.nb[0] * (cy + g.nb[1] * cz);
      const int s1 = (cell_start[row + x1] + 31) >> 5;
      for (int s = (cell_start[row + x0] + 31) >> 5; s < s1; ++s) {
        fn(s);
        ++count;
      }
    }
  }
  return count;
}

B2_HD int b2_body_brick_count(int b, const B2NeighborView& v, const B2Grid& g, const B2Bricks& br)
{
  return b2_brick_segments(b, g, br, v.cell_start, [](int) {});
}

B2_HD void b2_body_seg_order(int b, const B2NeighborView& v, const B2Grid& g, const B2Bricks& br)
{
  int* out = v.seg_order + v.brick_start[b];
  b2_brick_segments(b, g, br, v.cell_start, [&](int s) { *out++ = s; });
}

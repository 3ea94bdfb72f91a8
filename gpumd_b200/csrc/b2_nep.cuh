// b2_nep.cuh -- device math and kernel bodies of the NEP path of libb200md (sm_90a).
//
// What it computes is what the reference computes (src/force/nep.cu:436-975 with
// src/utilities/nep_utilities.cuh); HOW is re-derived for a cell-sorted, gather-only,
// register-resident formulation:
//
//  * radial descriptor: q_n = sum_j sum_k c[t1,t2,n,k] fn_k(r_ij) is accumulated as
//    S[t2][k] = sum_{j of type t2} fn_k(r_ij) (K+1 adds per pair instead of (n_max+1)(K+1) FMAs and
//    coefficient loads, nep.cu:536-545) and contracted with c once per atom;
//  * radial force: the per-pair sums over n (nep.cu:718-733) are pre-contracted per atom into
//    U_i[t][k] = sum_n Fp_i[n] c[t_i,t,n,k]; a pair then costs two (K+1)-term dot products
//    A = fn'.U_i[t_j], B = fn'.U_j[t_i] and one 48-byte gather of U_j (the reference gathers
//    n_max+1 strided Fp values and re-reads 2(n_max+1)(K+1) coefficients per pair);
//  * angular part: dU/ds[n][abc] (3-body + the chain-rule terms of the 4-/5-body invariants) is
//    formed ONCE per atom; a pair then contracts it with g_n, g_n' and uses the closed-form
//    gradients of the real solid harmonics up to L = 4.  The reference re-derives the 4-/5-body
//    prefactors for every pair (nep_utilities.cuh:625-718) and walks generic coefficient tables
//    (nep_utilities.cuh:1342-1434);
//  * the per-atom MLP (apply_ann_one_layer, nep_utilities.cuh:169-194) is a separate pass over
//    128-atom tiles of one type on the tensor cores (b2_nep_tc.cuh); the SIMT body below
//    (b2_body_mlp: type-sorted tiles, zero-padded weight rows) is the fallback for layer sizes the
//    tensor-core kernel does not cover and what tests/emu runs on the host;
//  * the neighbour-set split (nep.cu:436-486) is folded into the radial descriptor pass.
// Summation orders therefore differ from the reference at the FP32 rounding level; the membership
// of the radial/angular neighbour sets does not (b2_r12 / b2_d2 in b2_common.cuh).
#pragma once
#include "b2_common.cuh"

// normalisation of the real harmonics (C3B, nep_utilities.cuh:18-27; L <= 4 part)
#define B2_C3B_LIST                                                                             \
  0.238732414637843f, 0.119366207318922f, 0.119366207318922f, 0.099471839432435f,              \
    0.596831036594608f, 0.596831036594608f, 0.149207759148652f, 0.149207759148652f,            \
    0.139260575205408f, 0.104445431404056f, 0.104445431404056f, 1.044454314040563f,            \
    1.044454314040563f, 0.174075719006761f, 0.174075719006761f, 0.011190581936149f,            \
    0.223811638722978f, 0.223811638722978f, 0.111905819361489f, 0.111905819361489f,            \
    1.566681471060845f, 1.566681471060845f, 0.195835183882606f, 0.195835183882606f
// C4B, C5B (nep_utilities.cuh:40-46)
#define B2_C4B0 (-0.007499480826664f)
#define B2_C4B1 (-0.134990654879954f)
#define B2_C4B2 (0.067495327439977f)
#define B2_C4B3 (0.404971964639861f)
#define B2_C4B4 (-0.809943929279723f)
#define B2_C5B0 (0.026596810706114f)
#define B2_C5B1 (0.053193621412227f)
#define B2_C5B2 (0.026596810706114f)

constexpr int B2_NABC = 24;      // (L_max+1)^2 - 1 for L_max = 4
constexpr int B2_ABC4 = B2_NABC / 4; // float4 groups of one angular channel

// Shared-memory rows of the few-type angular kernels (b2_nep_angular.cuh): WS4 float4s of per-atom weights
// per thread, and k_angular_fused's w0 stride and its whole dynamic shared memory per 128-thread block
B2_HOST_DEVICE constexpr int b2_ang_ws4(int na1) { return B2_ABC4 * na1 + 1; }
B2_HOST_DEVICE constexpr int b2_fused_w0_stride4(int nneu, int dimp) { return (nneu * dimp / 4) | 1; }
B2_HOST_DEVICE constexpr size_t b2_fused_smem_bytes(int nt, int na1, int k1a, int nneu, int dimp)
{
  return (size_t)128 * b2_ang_ws4(na1) * 16 + (size_t)nt * nt * na1 * ((k1a + 3) / 4) * 16 +
         (size_t)nt * b2_fused_w0_stride4(nneu, dimp) * 16 + (size_t)2 * nt * nneu * 4;
}

// list entry = neighbour index | type << 30 (B2NeighborView::tag_types; the radial and angular lists
// of the few-type kernels in b2_nep_radial.cuh / b2_nep_angular.cuh)
constexpr int B2_TAG_SHIFT = 30;
constexpr int B2_TAG_MASK = (1 << B2_TAG_SHIFT) - 1;

struct B2NepView {
  // ---- model (device tables) ----
  int nt;       // number of types
  int nr1, na1; // n_max_radial+1, n_max_angular+1
  int kr1, ka1; // basis_size_radial+1, basis_size_angular+1 (true sizes)
  int K1R, K1A; // padded basis counts the kernels are instantiated for (9, 13 or 17)
  int KP;       // U-table row stride per type: K1R rounded up to a multiple of 4
  int UST;      // U-table stride per atom = nt * KP
  int has222, has1111, num_L; // L_max is 4
  int dim, dim_ang, nneu, DIMP;
  int zbl_enabled, zbl_flexible, zbl_typewise;
  float zbl_rc_inner, zbl_rc_outer, zbl_typewise_factor;
  const float* rc_r;    // [nt*nt] pair cutoff (rc[t1]+rc[t2])*0.5f
  const float* rcinv_r; // [nt*nt] 1.0f / rc_r
  const float* rc2_r;   // [nt*nt] rc_r*rc_r
  const float* rc_a;
  const float* rcinv_a;
  const float* rc2_a;
  const float* c_r;      // [nt*nt][nr1][K1R] zero-padded in k
  const float* c_a;      // [nt*nt][na1][K1A]
  // the same coefficients padded for 128-bit loads (null: scalar loads).  With many types every lane
  // of a warp reads a different (t1, t2) row, so each load instruction costs one L1 wavefront per
  // lane; four coefficients per instruction cut that cost by four.
  const float4* c_a4;    // [nt*nt][na1][(K1A+3)/4]: k = 4q .. 4q+3, zero-padded (always set)
  const float4* c_r4;    // [nt*nt][nqr][K1R]: n = 4*nq .. 4*nq+3 of basis function k, zero-padded; null:
                         // scalar loads in the radial contraction (B200MD_NEP_CVEC=0)
  int nqr;               // (nr1 + 3) / 4  (<= B2_NQMAX)
  // Direct reverse slots for the angular pair reduction (many-type path; null = binary search):
  //   rskin  [mn_skin*n]  slot of i in the skin list of its k-th skin neighbour (per rebuild, b2_neighbor)
  //   aslot  [mn_skin*n]  per step: angular slot of i's k-th skin neighbour, or -1
  //   nla_rs [mn_a*n]     per step: rskin of the skin slot the m-th angular neighbour came from
  // so the slot of i in j's angular list is aslot[nla_rs[m*n+i]*n + j].
  const int* rskin;
  int* aslot;
  int* nla_rs;
  int debug_skip;        // TIMING ONLY (B200MD_DEBUG_SKIP): 1 no radial sum, 2 no angular reduction, 4 no ZBL
  const float* w0p;      // [nt][nneu][DIMP] zero-padded rows
  const float* b0;       // [nt][nneu]
  const float* w1;       // [nt][nneu]
  const float* bias;     // [nt]  b1 (+ typewise bias for NEP5)
  const float* q_scaler; // [DIMP] zero-padded
  const int* zbl_z;      // [nt] atomic numbers
  const float* zbl_para; // flexible ZBL table
  const float* cov_radius; // [94]
  // ---- per-step state ----
  int n;
  int mn_r, mn_a;
  const B2Atom* atoms; // sorted records
  const int* perm;
  const int* nn_skin;
  const int* nl_skin;
  int* nn_r;
  int* nl_r; // [mn_r * n]
  int* nn_a;
  int* nl_a; // [mn_a * n]
  float* q;   // [dim * n]   unscaled descriptors
  float* sfx; // [na1*24 * n] angular sums s[n][abc]
  float* FpR; // [nr1 * n]     dU/dq, radial part (input of k_utable)
  float* FpA; // [dim_ang * n] dU/dq (already multiplied by q_scaler), angular part
  float* U;   // [n * UST]   pre-contracted radial table
  float* f12; // [3 * mn_a * n] as three planes; few-type kernels: [mn_a * n] float4 entries (w unused)
  double* acc; // [13 * n]: pe, fx,fy,fz, virial xx,yy,zz,xy,xz,yz,yx,zx,zy (sorted order)
  int* flags;
  // ---- lane-team path (<= 2 types): row-major skin / radial lists, U table as float4 planes ----
  size_t skin_si, skin_sk; // B2NeighborView::skin_si / skin_sk
  int pitch_r;             // row pitch of nl_r when team != 0 (else nl_r is column-major)
  int team;                // 1: k_team_* kernels own the radial passes
  int u_planes;            // 0: U as AoS rows of UST floats (many-type path, tests/emu); 1: float4 planes
                           //    [(t*KP4+q)*n + i] (lane teams); 2: compact planes of b2_nep_radial.cuh:
                           //    KQ = (K1-1)/4 float4 planes [(t*KQ+q)*n + i] + a float plane [t*n + i]
  int n_own;               // > 0: only caller indices < n_own get outputs (domain decomposition:
                           // the rest are ghosts whose forces the caller discards)
  int overwrite;           // 1: the final kernel STORES pe / force / virial instead of adding to them
                           //    (b200md_nep_set_accumulate(p, 0): the caller skips its zeroing pass)
  int use_active;          // 1: atoms outside [act_lo, act_hi) get empty neighbour sets, i.e. no
  double act_lo[3];        //    descriptor / MLP-gradient / partial-force work: ghosts further than
  double act_hi[3];        //    rc from every owned atom only serve as neighbours (b200md_nep_set_active_region)
  // ---- tensor-core hidden layer (k_mlp_tc; null / 0 when the SIMT k_mlp is used) ----
  const float* tc_img;  // [nt][tc_img_floats] shared-memory images, see NepModel::tc_img
  int tc_img_floats, HN, DK, DN;
  int K3, N3;           // U-table GEMM inside k_mlp_tc (N3 = 0: done by k_utable instead)
  // Tile-major copies of the hidden layer's input and output (non-null when k_mlp_tc is in use):
  //   qt [tile][k/4][row][k%4], fpt the same shape for dU/dq -- a 128-atom tile of one type is ONE
  //   contiguous block of DKT*128 floats, already in the K-major order of the wgmma A operand, so the
  //   kernel fetches it with a single TMA bulk copy and stores dU/dq with fully coalesced float4s.
  //   The descriptor kernels write q there (through tile_slot) instead of the SoA columns.
  const int* tile_slot; // [n] slot (tile*128 + row) of every sorted atom
  float* qt;
  float* fpt;
  int DKT;              // columns per tile row (= DK, a multiple of 8)
  const int* tile_atom; // B2NeighborView::tile_atom / tile_type / tile_meta
  const int* tile_type;
  const int* tile_meta;
  const int* seg_order; // B2NeighborView::seg_order (few-type kernels); null = identity schedule
};

// address of descriptor component k of sorted atom i (slot = P.tile_slot[i] when the tile-major copy is
// in use, ignored otherwise); the same indexing serves dU/dq in P.fpt
B2_HD size_t b2_tile_offset(int DKT, int slot, int k)
{
  return ((size_t)(slot >> 7) * (DKT >> 2) + (k >> 2)) * 512 + (size_t)(slot & 127) * 4 + (k & 3);
}
B2_HD float* b2_q_ptr(const B2NepView& P, int i, int slot, int k)
{
  return P.qt ? P.qt + b2_tile_offset(P.DKT, slot, k) : P.q + (size_t)k * P.n + i;
}

// inside the region whose atoms need descriptors (always true without a region)
B2_HD bool b2_is_active(const B2NepView& P, double x, double y, double z)
{
  if (!P.use_active)
    return true;
  return x >= P.act_lo[0] && x < P.act_hi[0] && y >= P.act_lo[1] && y < P.act_hi[1] &&
         z >= P.act_lo[2] && z < P.act_hi[2];
}

// ---------------------------------------------------------------------------------------------
// neighbour-set split: find_neighbor_list_large_box, nep.cu:436-486
// ---------------------------------------------------------------------------------------------
B2_HD void b2_body_split(int i, const B2NepView& P, const B2Box& box)
{
  const B2Geo geo = b2_geo(box);
  const size_t N = (size_t)P.n;
  const B2Atom a1 = P.atoms[i];
  if (!b2_is_active(P, a1.x, a1.y, a1.z)) {
    P.nn_r[i] = 0;
    P.nn_a[i] = 0;
    if (P.aslot)
      for (int k = 0; k < P.nn_skin[i]; ++k)
        P.aslot[(size_t)k * N + i] = -1;
    return;
  }
  const int nn = P.nn_skin[i];
  const int row = a1.type * P.nt;
  int cr = 0, ca = 0;
  // software pipeline: the record of candidate k+1 and the index of candidate k+2 are in flight
  // while candidate k is tested (the loads are dependent: index -> record)
  int jn = nn > 0 ? P.nl_skin[i] : i;
  B2Atom an = b2_load_atom(&P.atoms[jn]);
  int j2 = nn > 1 ? P.nl_skin[N + i] : i;
  for (int k = 0; k < nn; ++k) {
    const int j = jn;
    const B2Atom a2 = an;
    jn = j2;
    an = b2_load_atom(&P.atoms[jn]);
    j2 = (k + 2 < nn) ? P.nl_skin[(size_t)(k + 2) * N + i] : i;
    float x12, y12, z12;
    b2_r12(geo, box, a1, a2, x12, y12, z12);
    const float d2 = b2_d2(x12, y12, z12);
    const int pair = row + a2.type;
    int as = -1; // angular slot of skin candidate k
    if (d2 < B2_LDG(&P.rc2_r[pair])) {
      if (cr < P.mn_r)
        P.nl_r[(size_t)cr * N + i] = j;
      ++cr;
      if (d2 < B2_LDG(&P.rc2_a[pair])) {
        if (ca < P.mn_a) {
          P.nl_a[(size_t)ca * N + i] = j;
          if (P.aslot)
            P.nla_rs[(size_t)ca * N + i] = P.rskin[(size_t)k * N + i];
          as = ca;
        }
        ++ca;
      }
    }
    if (P.aslot)
      P.aslot[(size_t)k * N + i] = as;
  }
  if (cr > P.mn_r) {
    B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_RADIAL_OVERFLOW);
    cr = P.mn_r;
  }
  if (ca > P.mn_a) {
    B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_ANGULAR_OVERFLOW);
    ca = P.mn_a;
  }
  P.nn_r[i] = cr;
  P.nn_a[i] = ca;
}

// ---------------------------------------------------------------------------------------------
// radial basis.  fc, fc' : nep_utilities.cuh:409-431;  fn, fn' : nep_utilities.cuh:572-623
// ---------------------------------------------------------------------------------------------
template <int K1>
B2_HD void b2_basis(float d, float rc, float rcinv, float* fn)
{
  float fc = 0.0f;
  if (d < rc)
    fc = 0.5f * b2_cospi(d * rcinv) + 0.5f;
  const float y = d * rcinv - 1.0f;
  const float x = 2.0f * y * y - 1.0f;
  const float hfc = 0.5f * fc;
  fn[0] = fc;
  fn[1] = (x + 1.0f) * hfc;
  float t0 = 1.0f, t1 = x;
#pragma unroll
  for (int k = 2; k < K1; ++k) {
    const float t2 = 2.0f * x * t1 - t0;
    t0 = t1;
    t1 = t2;
    fn[k] = (t2 + 1.0f) * hfc;
  }
}

// WITH_FN = false skips fn (the radial force only needs the derivatives)
template <int K1, bool WITH_FN>
B2_HD void b2_basis_d(float d, float rc, float rcinv, float* fn, float* fnp)
{
  float fc = 0.0f, fcp = 0.0f;
  if (d < rc) {
    float s, c;
    b2_sincospi(d * rcinv, s, c);
    fc = 0.5f * c + 0.5f;
    fcp = -1.5707963f * s * rcinv;
  }
  const float y = d * rcinv - 1.0f;
  const float x = 2.0f * y * y - 1.0f;
  const float g = 2.0f * y * rcinv * fc; // d/dr of (x+1)/2, times fc
  const float hfc = 0.5f * fc, hfcp = 0.5f * fcp;
  if (WITH_FN) {
    fn[0] = fc;
    fn[1] = (x + 1.0f) * hfc;
  }
  fnp[0] = fcp;
  fnp[1] = g + (x + 1.0f) * hfcp;
  float t0 = 1.0f, t1 = x;        // T_{k-2}, T_{k-1}
  float u0 = 1.0f, u1 = 2.0f * x; // U_{k-2}, U_{k-1}
#pragma unroll
  for (int k = 2; k < K1; ++k) {
    const float t2 = 2.0f * x * t1 - t0;
    t0 = t1;
    t1 = t2;
    // d T_k / dx = k U_{k-1}
    fnp[k] = ((float)k * u1) * g + (t2 + 1.0f) * hfcp;
    if (WITH_FN)
      fn[k] = (t2 + 1.0f) * hfc;
    const float u2 = 2.0f * x * u1 - u0;
    u0 = u1;
    u1 = u2;
  }
}

// ---------------------------------------------------------------------------------------------
// radial descriptor (radial half of find_descriptor, nep.cu:521-546)
// NT > 0: per-type accumulators in registers (models with <= NT types), updated with a 0/1 mask per
// type -- NT*K1 FMAs per pair.  That is the default for 1 and 2 types; for 16 types x 9 functions it
// needs 211 registers, which costs more than the shared-memory accumulators of NT == 0 save.
// NT == 0: accumulators in the caller-provided scratch `acc` laid out [(t2*K1+k)*stride + lane].
// NT < 0: no per-type accumulators at all -- every pair is contracted with c[t1,t2,n,k] on the spot (45 FMAs
// and K1 128-bit coefficient loads per pair for n_max = 4, K = 8).  Costs more per pair but needs no
// storage that grows with the number of types: the path for models like NEP89 (89 species).
// ---------------------------------------------------------------------------------------------
// SPLIT = true fuses the neighbour-set split (b2_body_split) into this pass: the loop then walks
// the skin list, applies the reference's two FP32 membership tests and emits the radial /
// angular lists on the way.  That pays when few skin candidates fail the test (large rc); with a
// small rc the idle lanes cost more than the separate cheap kernel.
template <int NT, int K1, bool SPLIT>
B2_HD void b2_body_desc_radial(
  int i, const B2NepView& P, const B2Box& box, float* acc, int stride, int lane)
{
  const B2Geo geo = b2_geo(box);
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  if (SPLIT && !b2_is_active(P, a1.x, a1.y, a1.z)) {
    P.nn_r[i] = 0;
    P.nn_a[i] = 0;
    const int slot0 = P.qt ? P.tile_slot[i] : 0;
    for (int n = 0; n < P.nr1; ++n)
      *b2_q_ptr(P, i, slot0, n) = 0.0f;
    return;
  }
  const int nn = SPLIT ? P.nn_skin[i] : P.nn_r[i];
  const int* list = SPLIT ? P.nl_skin : P.nl_r;
  int cr = 0, ca = 0;
  float S[NT > 0 ? NT : 1][K1];
  float Q[B2_NQMAX][4]; // NT < 0: the descriptor components themselves, four per register group
  if (NT > 0) {
#pragma unroll
    for (int t = 0; t < (NT > 0 ? NT : 1); ++t)
#pragma unroll
      for (int k = 0; k < K1; ++k)
        S[t][k] = 0.0f;
  } else if (NT == 0) {
    for (int m = 0; m < P.nt * K1; ++m)
      acc[(size_t)m * stride + lane] = 0.0f;
  } else {
#pragma unroll
    for (int nq = 0; nq < B2_NQMAX; ++nq)
      Q[nq][0] = Q[nq][1] = Q[nq][2] = Q[nq][3] = 0.0f;
  }
  int jn = nn > 0 ? B2_LDCS(&list[i]) : i;
  B2Atom an = b2_load_atom(&P.atoms[jn]);
  int j2 = nn > 1 ? B2_LDCS(&list[(size_t)P.n + i]) : i;
  for (int s = 0; s < nn; ++s) {
    const int j = jn;
    const B2Atom a2 = an;
    jn = j2;
    an = b2_load_atom(&P.atoms[j2]);
    j2 = (s + 2 < nn) ? B2_LDCS(&list[(size_t)(s + 2) * P.n + i]) : i;
    float x12, y12, z12;
    b2_r12(geo, box, a1, a2, x12, y12, z12);
    const float d2 = b2_d2(x12, y12, z12);
    const int t2 = a2.type;
    const int pair = t1 * P.nt + t2;
    if (SPLIT) {
      if (d2 >= B2_LDG(&P.rc2_r[pair]))
        continue;
      if (cr < P.mn_r)
        B2_STCS(&P.nl_r[(size_t)cr * P.n + i], j);
      ++cr;
      if (d2 < B2_LDG(&P.rc2_a[pair])) {
        if (ca < P.mn_a)
          P.nl_a[(size_t)ca * P.n + i] = j;
        ++ca;
      }
    }
    const float d = sqrtf(d2);
    float fn[K1];
    b2_basis<K1>(d, B2_LDG(&P.rc_r[pair]), B2_LDG(&P.rcinv_r[pair]), fn);
    if (NT == 1) {
#pragma unroll
      for (int k = 0; k < K1; ++k)
        S[0][k] += fn[k];
    } else if (NT > 1) {
#pragma unroll
      for (int t = 0; t < (NT > 0 ? NT : 1); ++t) {
        const float m = (t2 == t) ? 1.0f : 0.0f;
#pragma unroll
        for (int k = 0; k < K1; ++k)
          S[t][k] = fmaf(m, fn[k], S[t][k]);
      }
    } else if (NT == 0) {
      float* a = acc + (size_t)(t2 * K1) * stride + lane;
#pragma unroll
      for (int k = 0; k < K1; ++k)
        a[(size_t)k * stride] += fn[k];
    } else {
      // per-pair contraction, the reference's own order (find_descriptor, nep.cu:521-546):
      // g_n = sum_k fn_k c[t1,t2,n,k], then q_n += g_n
#pragma unroll
      for (int nq = 0; nq < B2_NQMAX; ++nq) {
        if (nq < P.nqr) {
          const float4* c4 = P.c_r4 + ((size_t)pair * P.nqr + nq) * K1;
          float g0 = 0.0f, g1 = 0.0f, g2 = 0.0f, g3 = 0.0f;
#pragma unroll
          for (int k = 0; k < K1; ++k) {
            const float4 v = B2_LDG(&c4[k]);
            g0 = fmaf(fn[k], v.x, g0);
            g1 = fmaf(fn[k], v.y, g1);
            g2 = fmaf(fn[k], v.z, g2);
            g3 = fmaf(fn[k], v.w, g3);
          }
          Q[nq][0] += g0;
          Q[nq][1] += g1;
          Q[nq][2] += g2;
          Q[nq][3] += g3;
        }
      }
    }
  }
  if (SPLIT) {
    if (cr > P.mn_r) {
      B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_RADIAL_OVERFLOW);
      cr = P.mn_r;
    }
    if (ca > P.mn_a) {
      B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_ANGULAR_OVERFLOW);
      ca = P.mn_a;
    }
    P.nn_r[i] = cr;
    P.nn_a[i] = ca;
  }
  // contraction with the expansion coefficients
  const int qslot = P.qt ? P.tile_slot[i] : 0;
  if (NT < 0) {
#pragma unroll
    for (int nq = 0; nq < B2_NQMAX; ++nq)
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (4 * nq + c < P.nr1)
          *b2_q_ptr(P, i, qslot, 4 * nq + c) = Q[nq][c];
    return;
  }
  if ((NT == 0 || NT > 2) && P.c_r4) {
    // four radial channels per pass: one 128-bit coefficient load and one read of the accumulator
    // serve four FMAs; per channel the (t outer, k inner) summation order is the scalar path's
    for (int nq = 0; nq < P.nqr; ++nq) {
      float q0 = 0.0f, q1 = 0.0f, q2 = 0.0f, q3 = 0.0f;
      if (NT > 2) {
#pragma unroll
        for (int t = 0; t < (NT > 0 ? NT : 1); ++t) {
          if (t < P.nt) {
            const float4* c4 = P.c_r4 + ((size_t)(t1 * P.nt + t) * P.nqr + nq) * K1;
#pragma unroll
            for (int k = 0; k < K1; ++k) {
              const float av = S[t][k];
              const float4 v = B2_LDG(&c4[k]);
              q0 = fmaf(v.x, av, q0);
              q1 = fmaf(v.y, av, q1);
              q2 = fmaf(v.z, av, q2);
              q3 = fmaf(v.w, av, q3);
            }
          }
        }
      } else
      for (int t = 0; t < P.nt; ++t) {
        const float4* c4 = P.c_r4 + ((size_t)(t1 * P.nt + t) * P.nqr + nq) * K1;
        const float* a = acc + (size_t)(t * K1) * stride + lane;
#pragma unroll
        for (int k = 0; k < K1; ++k) {
          const float av = a[(size_t)k * stride];
          const float4 v = B2_LDG(&c4[k]);
          q0 = fmaf(v.x, av, q0);
          q1 = fmaf(v.y, av, q1);
          q2 = fmaf(v.z, av, q2);
          q3 = fmaf(v.w, av, q3);
        }
      }
      const int n = 4 * nq;
      *b2_q_ptr(P, i, qslot, n) = q0;
      if (n + 1 < P.nr1)
        *b2_q_ptr(P, i, qslot, n + 1) = q1;
      if (n + 2 < P.nr1)
        *b2_q_ptr(P, i, qslot, n + 2) = q2;
      if (n + 3 < P.nr1)
        *b2_q_ptr(P, i, qslot, n + 3) = q3;
    }
    return;
  }
  for (int n = 0; n < P.nr1; ++n) {
    float q = 0.0f;
    if (NT > 0) {
#pragma unroll
      for (int t = 0; t < (NT > 0 ? NT : 1); ++t) {
        if (t < P.nt) {
          const float* c = P.c_r + ((size_t)(t1 * P.nt + t) * P.nr1 + n) * K1;
#pragma unroll
          for (int k = 0; k < K1; ++k)
            q = fmaf(B2_LDG(&c[k]), S[t][k], q);
        }
      }
    } else {
      for (int t = 0; t < P.nt; ++t) {
        const float* c = P.c_r + ((size_t)(t1 * P.nt + t) * P.nr1 + n) * K1;
        const float* a = acc + (size_t)(t * K1) * stride + lane;
#pragma unroll
        for (int k = 0; k < K1; ++k)
          q = fmaf(B2_LDG(&c[k]), a[(size_t)k * stride], q);
      }
    }
    *b2_q_ptr(P, i, qslot, n) = q;
  }
}

// ---------------------------------------------------------------------------------------------
// real solid harmonics on the unit sphere, L = 1..4, in the reference's ordering
// (accumulate_s_one, nep_utilities.cuh:1674-1723 with Z_COEFFICIENT_1..4, :87-103):
// for each L: m = 0, then Re/Im (x+iy)^m times the z-polynomial, m = 1..L.
// ---------------------------------------------------------------------------------------------
B2_HD void b2_harmonics(float x, float y, float z, float* B)
{
  const float x2 = x * x, y2 = y * y, z2 = z * z;
  const float c2 = x2 - y2, s2 = 2.0f * x * y;                       // Re, Im (x+iy)^2
  const float c3 = x * (x2 - 3.0f * y2), s3 = y * (3.0f * x2 - y2); // (x+iy)^3
  const float c4 = c2 * c2 - s2 * s2, s4 = 2.0f * c2 * s2;           // (x+iy)^4
  B[0] = z;
  B[1] = x;
  B[2] = y;
  B[3] = 3.0f * z2 - 1.0f;
  B[4] = x * z;
  B[5] = y * z;
  B[6] = c2;
  B[7] = s2;
  const float p31 = 5.0f * z2 - 1.0f;
  B[8] = (5.0f * z2 - 3.0f) * z;
  B[9] = p31 * x;
  B[10] = p31 * y;
  B[11] = z * c2;
  B[12] = z * s2;
  B[13] = c3;
  B[14] = s3;
  const float p41 = (7.0f * z2 - 3.0f) * z, p42 = 7.0f * z2 - 1.0f;
  B[15] = (35.0f * z2 - 30.0f) * z2 + 3.0f;
  B[16] = p41 * x;
  B[17] = p41 * y;
  B[18] = p42 * c2;
  B[19] = p42 * s2;
  B[20] = z * c3;
  B[21] = z * s3;
  B[22] = c4;
  B[23] = s4;
}

// G = sum_abc W[abc] * grad B_abc evaluated at the unit vector (x,y,z), where B_abc are the
// homogeneous (degree L) forms of the harmonics above (r^2 = 1 substituted after differentiating).
B2_HD void b2_harmonics_grad_dot(
  float x, float y, float z, const float* W, float& gx, float& gy, float& gz)
{
  const float x2 = x * x, y2 = y * y, z2 = z * z;
  const float xy = x * y, xz = x * z, yz = y * z;
  const float c2 = x2 - y2, s2 = 2.0f * xy;
  const float c3 = x * (x2 - 3.0f * y2), s3 = y * (3.0f * x2 - y2);
  // L = 1
  gx = W[1];
  gy = W[2];
  gz = W[0];
  // L = 2: 3z^2-r^2, xz, yz, x^2-y^2, 2xy
  gx += W[3] * (-2.0f * x) + W[4] * z + W[6] * (2.0f * x) + W[7] * (2.0f * y);
  gy += W[3] * (-2.0f * y) + W[5] * z - W[6] * (2.0f * y) + W[7] * (2.0f * x);
  gz += W[3] * (4.0f * z) + W[4] * x + W[5] * y;
  // L = 3: 5z^3-3zr^2, (5z^2-r^2)x, (5z^2-r^2)y, z(x^2-y^2), 2xyz, x^3-3xy^2, 3x^2y-y^3
  {
    const float p = 5.0f * z2 - 1.0f;
    gx += W[8] * (-6.0f * xz) + W[9] * (p - 2.0f * x2) + W[10] * (-2.0f * xy) +
          W[11] * (2.0f * xz) + W[12] * (2.0f * yz) + W[13] * (3.0f * c2) + W[14] * (6.0f * xy);
    gy += W[8] * (-6.0f * yz) + W[9] * (-2.0f * xy) + W[10] * (p - 2.0f * y2) -
          W[11] * (2.0f * yz) + W[12] * (2.0f * xz) - W[13] * (6.0f * xy) + W[14] * (3.0f * c2);
    gz += W[8] * (9.0f * z2 - 3.0f) + W[9] * (8.0f * xz) + W[10] * (8.0f * yz) + W[11] * c2 +
          W[12] * s2;
  }
  // L = 4: 35z^4-30z^2r^2+3r^4, (7z^3-3zr^2)x, (7z^3-3zr^2)y, (7z^2-r^2)(x^2-y^2),
  //        (7z^2-r^2)2xy, z(x^3-3xy^2), z(3x^2y-y^3), x^4-6x^2y^2+y^4, 4xy(x^2-y^2)
  {
    const float a0 = 12.0f - 60.0f * z2;         // d/dx, d/dy prefactor of the m=0 term
    const float p1 = (7.0f * z2 - 3.0f) * z;     // 7z^3 - 3z
    const float p1z = 15.0f * z2 - 3.0f;         // d/dz of (7z^3-3zr^2) at r=1
    const float p2 = 7.0f * z2 - 1.0f;
    gx += W[15] * (a0 * x) + W[16] * (p1 - 6.0f * z * x2) + W[17] * (-6.0f * z * xy) +
          W[18] * (2.0f * x * (p2 - c2)) + W[19] * (2.0f * y * p2 - 4.0f * x2 * y) +
          W[20] * (3.0f * z * c2) + W[21] * (6.0f * z * xy) +
          W[22] * (4.0f * c3) + W[23] * (4.0f * s3);
    gy += W[15] * (a0 * y) + W[16] * (-6.0f * z * xy) + W[17] * (p1 - 6.0f * z * y2) +
          W[18] * (-2.0f * y * (p2 + c2)) + W[19] * (2.0f * x * p2 - 4.0f * x * y2) -
          W[20] * (6.0f * z * xy) + W[21] * (3.0f * z * c2) -
          W[22] * (4.0f * s3) + W[23] * (4.0f * c3);
    gz += W[15] * (z * (80.0f * z2 - 48.0f)) + W[16] * (x * p1z) + W[17] * (y * p1z) +
          W[18] * (12.0f * z * c2) + W[19] * (12.0f * z * s2) + W[20] * c3 + W[21] * s3;
  }
}

// Angular descriptor components of one radial channel from its sums s[abc]: the 3-body invariants
// L = 1..4 (block L-1), then the 4-body (has222) and the 5-body (has1111) one; emit(block, value).
// Component (block, n) sits at q[nr1 + block*na1 + n].
template <class Emit>
B2_HD void b2_ang_invariants(const float* s, int has222, int has1111, Emit emit)
{
  const float C3B[B2_NABC] = {B2_C3B_LIST};
  int st = 0;
#pragma unroll
  for (int L = 1; L <= 4; ++L) {
    float v = 0.0f;
#pragma unroll
    for (int k = 1; k < 2 * L + 1; ++k)
      v = fmaf(C3B[st + k] * s[st + k], s[st + k], v);
    v = 2.0f * v + C3B[st] * s[st] * s[st];
    emit(L - 1, v);
    st += 2 * L + 1;
  }
  int Lidx = 4;
  if (has222) {
    const float* t = &s[3];
    const float v = B2_C4B0 * t[0] * t[0] * t[0] + B2_C4B1 * t[0] * (t[1] * t[1] + t[2] * t[2]) +
                    B2_C4B2 * t[0] * (t[3] * t[3] + t[4] * t[4]) +
                    B2_C4B3 * t[3] * (t[2] * t[2] - t[1] * t[1]) + B2_C4B4 * t[1] * t[2] * t[4];
    emit(Lidx, v);
    ++Lidx;
  }
  if (has1111) {
    const float s0 = s[0] * s[0], tt = s[1] * s[1] + s[2] * s[2];
    emit(Lidx, B2_C5B0 * s0 * s0 + B2_C5B1 * s0 * tt + B2_C5B2 * tt * tt);
  }
}

// dU/ds[abc] of one radial channel: 3-body weights plus the chain-rule terms of the 4- and 5-body
// invariants.  F[L-1] = dU/dq of the L-th 3-body component, F[4] of the 4-body, F[5] of the 5-body one
// (ignored when the model lacks them).
B2_HD void b2_ang_weights(const float* s, const float* F6, int has222, int has1111, float* wv)
{
  const float C3B[B2_NABC] = {B2_C3B_LIST};
  int st = 0;
#pragma unroll
  for (int L = 1; L <= 4; ++L) {
    const float F = F6[L - 1];
    wv[st] = 2.0f * F * C3B[st] * s[st];
#pragma unroll
    for (int k = 1; k < 2 * L + 1; ++k)
      wv[st + k] = 4.0f * F * C3B[st + k] * s[st + k];
    st += 2 * L + 1;
  }
  // the chain-rule terms are added with explicit FMAs: with has222 / has1111 known at compile time the
  // compiler could otherwise fuse the product above into the add instead, which rounds differently
  if (has222) {
    const float F = F6[4];
    const float* t = &s[3];
    wv[3] = fmaf(F, 3.0f * B2_C4B0 * t[0] * t[0] + B2_C4B1 * (t[1] * t[1] + t[2] * t[2]) +
                      B2_C4B2 * (t[3] * t[3] + t[4] * t[4]), wv[3]);
    wv[4] = fmaf(F, 2.0f * B2_C4B1 * t[0] * t[1] - 2.0f * B2_C4B3 * t[3] * t[1] + B2_C4B4 * t[2] * t[4], wv[4]);
    wv[5] = fmaf(F, 2.0f * B2_C4B1 * t[0] * t[2] + 2.0f * B2_C4B3 * t[3] * t[2] + B2_C4B4 * t[1] * t[4], wv[5]);
    wv[6] = fmaf(F, 2.0f * B2_C4B2 * t[0] * t[3] + B2_C4B3 * (t[2] * t[2] - t[1] * t[1]), wv[6]);
    wv[7] = fmaf(F, 2.0f * B2_C4B2 * t[0] * t[4] + B2_C4B4 * t[1] * t[2], wv[7]);
  }
  if (has1111) {
    const float F = F6[5];
    const float tt = s[1] * s[1] + s[2] * s[2];
    wv[0] = fmaf(F, 4.0f * B2_C5B0 * s[0] * s[0] * s[0] + 2.0f * B2_C5B1 * tt * s[0], wv[0]);
    wv[1] = fmaf(F, 2.0f * B2_C5B1 * s[0] * s[0] * s[1] + 4.0f * B2_C5B2 * tt * s[1], wv[1]);
    wv[2] = fmaf(F, 2.0f * B2_C5B1 * s[0] * s[0] * s[2] + 4.0f * B2_C5B2 * tt * s[2], wv[2]);
  }
}

// ---------------------------------------------------------------------------------------------
// angular descriptor (angular half of find_descriptor, nep.cu:549-581, find_q
// nep_utilities.cuh:1819-1872).  Processes the radial index n in chunks of NCH so that the
// NCH*24 accumulators stay in registers; each chunk walks the (short) angular list once.
// ---------------------------------------------------------------------------------------------
template <int K1, int NCH>
// ctab / rs4: the padded angular coefficients c_a4 (B2NepView) and their row stride per type pair in
// float4 units -- the global table (rs4 = na1*KQ) or the block's shared-memory copy
B2_HD void b2_body_desc_angular(
  int i, const B2NepView& P, const B2Box& box, const float4* ctab, int rs4)
{
  const float C3B[B2_NABC] = {B2_C3B_LIST};
  const B2Geo geo = b2_geo(box);
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  const int nn = P.nn_a[i];
  for (int n0 = 0; n0 < P.na1; n0 += NCH) {
    float s[NCH][B2_NABC];
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int abc = 0; abc < B2_NABC; ++abc)
        s[c][abc] = 0.0f;
    // (no software pipelining here: with NCH*24 accumulators live it costs registers)
    for (int m = 0; m < nn; ++m) {
      const int j = P.nl_a[(size_t)m * P.n + i];
      const B2Atom a2 = b2_load_atom(&P.atoms[j]);
      float x12, y12, z12;
      b2_r12(geo, box, a1, a2, x12, y12, z12);
      const float d = sqrtf(b2_d2(x12, y12, z12));
      const int pair = t1 * P.nt + a2.type;
      float fn[K1];
      b2_basis<K1>(d, B2_LDG(&P.rc_a[pair]), B2_LDG(&P.rcinv_a[pair]), fn);
      const float dinv = 1.0f / d;
      float B[B2_NABC];
      b2_harmonics(x12 * dinv, y12 * dinv, z12 * dinv, B);
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        if (n0 + c < P.na1) {
          float g = 0.0f;
          constexpr int KQ = (K1 + 3) / 4;
          const float4* c4 = ctab + (size_t)pair * rs4 + (n0 + c) * KQ;
          float ck[KQ * 4];
#pragma unroll
          for (int q = 0; q < KQ; ++q) {
            const float4 v = c4[q];
            ck[4 * q] = v.x;
            ck[4 * q + 1] = v.y;
            ck[4 * q + 2] = v.z;
            ck[4 * q + 3] = v.w;
          }
#pragma unroll
          for (int k = 0; k < K1; ++k)
            g = fmaf(fn[k], ck[k], g);
#pragma unroll
          for (int abc = 0; abc < B2_NABC; ++abc)
            s[c][abc] = fmaf(g, B[abc], s[c][abc]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      const int n = n0 + c;
      if (n < P.na1) {
        const int qslot = P.qt ? P.tile_slot[i] : 0; // q[nr1 + L*na1 + n] of atom i
        // 3-body invariants, L = 1..4
        int st = 0;
#pragma unroll
        for (int L = 1; L <= 4; ++L) {
          float v = 0.0f;
#pragma unroll
          for (int k = 1; k < 2 * L + 1; ++k)
            v = fmaf(C3B[st + k] * s[c][st + k], s[c][st + k], v);
          v = 2.0f * v + C3B[st] * s[c][st] * s[c][st];
          *b2_q_ptr(P, i, qslot, P.nr1 + (L - 1) * P.na1 + n) = v;
          st += 2 * L + 1;
        }
        int Lidx = 4;
        if (P.has222) {
          const float* t = &s[c][3];
          const float v = B2_C4B0 * t[0] * t[0] * t[0] + B2_C4B1 * t[0] * (t[1] * t[1] + t[2] * t[2]) +
                          B2_C4B2 * t[0] * (t[3] * t[3] + t[4] * t[4]) +
                          B2_C4B3 * t[3] * (t[2] * t[2] - t[1] * t[1]) + B2_C4B4 * t[1] * t[2] * t[4];
          *b2_q_ptr(P, i, qslot, P.nr1 + Lidx * P.na1 + n) = v;
          ++Lidx;
        }
        if (P.has1111) {
          const float s0 = s[c][0] * s[c][0], tt = s[c][1] * s[c][1] + s[c][2] * s[c][2];
          *b2_q_ptr(P, i, qslot, P.nr1 + Lidx * P.na1 + n) =
            B2_C5B0 * s0 * s0 + B2_C5B1 * s0 * tt + B2_C5B2 * tt * tt;
          ++Lidx;
        }
#pragma unroll
        for (int abc = 0; abc < B2_NABC; ++abc)
          P.sfx[(size_t)(n * B2_NABC + abc) * P.n + i] = s[c][abc];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// per-atom MLP (apply_ann_one_layer[_nep5], nep_utilities.cuh:169-194, 285-310; nep.cu:583-657)
// plus the radial pre-contraction U_i[t][k] = sum_n Fp_i[n] c[t_i,t,n,k].
// ---------------------------------------------------------------------------------------------
// The per-atom core: scaled descriptor q[DIMP] (zero-padded) in, site energy out, dU/dq (already
// multiplied by q_scaler) in Fp[DIMP].  w0 / b0 / w1 are the rows of the atom's type.  Shared by
// b2_body_mlp and k_angular_fused (b2_nep_angular.cuh), so both produce the same bits.
template <int DIMP, bool GLOBAL_W>
B2_HD void b2_mlp_row(const float4* w0, int n, float4* w)
{
  const float4* row = w0 + (size_t)n * (DIMP / 4);
#pragma unroll
  for (int d = 0; d < DIMP / 4; ++d)
    w[d] = GLOBAL_W ? B2_LDG(&row[d]) : row[d];
}

// activation of neuron n from its dot product, then its terms of F and of every Fp[d]
template <int DIMP, bool GLOBAL_W>
B2_HD void b2_mlp_neuron(
  float dot, const float4* w, const float* b0, const float* w1, int n, float& F, float* Fp)
{
  const float x1 = tanhf(dot - (GLOBAL_W ? B2_LDG(&b0[n]) : b0[n]));
  const float w1n = GLOBAL_W ? B2_LDG(&w1[n]) : w1[n];
  F = fmaf(w1n, x1, F);
  const float coef = w1n * (1.0f - x1 * x1);
#pragma unroll
  for (int d = 0; d < DIMP / 4; ++d) {
    Fp[4 * d] = fmaf(coef, w[d].x, Fp[4 * d]);
    Fp[4 * d + 1] = fmaf(coef, w[d].y, Fp[4 * d + 1]);
    Fp[4 * d + 2] = fmaf(coef, w[d].z, Fp[4 * d + 2]);
    Fp[4 * d + 3] = fmaf(coef, w[d].w, Fp[4 * d + 3]);
  }
}

// PAIR (k_angular_fused on a fixed angular shape, DIMP = 32): the forward dot products of two neurons are formed together, two
// independent chains of DIMP dependent FMAs in flight instead of one, each still summed in order over d;
// the activations, F and the Fp updates then follow neuron by neuron in the order n, n+1.  Both forms
// give the same bits.  k_mlp keeps one chain: at DIMP >= 64 the second row of weights makes it spill.
template <int DIMP, bool GLOBAL_W, bool PAIR = false>
B2_HD float b2_mlp_core(
  const float* q, const float4* w0, const float* b0, const float* w1, int nneu, float bias,
  const float* q_scaler, float* Fp)
{
#pragma unroll
  for (int d = 0; d < DIMP; ++d)
    Fp[d] = 0.0f;
  float F = 0.0f;
  int n = 0;
  if (PAIR) {
    for (; n + 1 < nneu; n += 2) {
      float4 wa[DIMP / 4], wb[DIMP / 4];
      b2_mlp_row<DIMP, GLOBAL_W>(w0, n, wa);
      b2_mlp_row<DIMP, GLOBAL_W>(w0, n + 1, wb);
      float da = 0.0f, db = 0.0f;
#pragma unroll
      for (int d = 0; d < DIMP / 4; ++d) {
        da = fmaf(wa[d].x, q[4 * d], da);
        db = fmaf(wb[d].x, q[4 * d], db);
        da = fmaf(wa[d].y, q[4 * d + 1], da);
        db = fmaf(wb[d].y, q[4 * d + 1], db);
        da = fmaf(wa[d].z, q[4 * d + 2], da);
        db = fmaf(wb[d].z, q[4 * d + 2], db);
        da = fmaf(wa[d].w, q[4 * d + 3], da);
        db = fmaf(wb[d].w, q[4 * d + 3], db);
      }
      b2_mlp_neuron<DIMP, GLOBAL_W>(da, wa, b0, w1, n, F, Fp);
      b2_mlp_neuron<DIMP, GLOBAL_W>(db, wb, b0, w1, n + 1, F, Fp);
    }
  }
  for (; n < nneu; ++n) {
    float4 w[DIMP / 4];
    b2_mlp_row<DIMP, GLOBAL_W>(w0, n, w);
    float dot = 0.0f;
#pragma unroll
    for (int d = 0; d < DIMP / 4; ++d) {
      dot = fmaf(w[d].x, q[4 * d], dot);
      dot = fmaf(w[d].y, q[4 * d + 1], dot);
      dot = fmaf(w[d].z, q[4 * d + 2], dot);
      dot = fmaf(w[d].w, q[4 * d + 3], dot);
    }
    b2_mlp_neuron<DIMP, GLOBAL_W>(dot, w, b0, w1, n, F, Fp);
  }
  F -= bias;
#pragma unroll
  for (int d = 0; d < DIMP; ++d)
    Fp[d] *= B2_LDG(&q_scaler[d]);
  return F;
}

// w0_all / b0_all / w1_all: [nt][nneu][DIMP], [nt][nneu], [nt][nneu] -- either the global tables
// (GLOBAL_W = true, read through the read-only path) or a shared-memory copy staged by the block.
template <int DIMP, bool GLOBAL_W>
B2_HD void b2_body_mlp(
  int i, const B2NepView& P, const float* w0_all, const float* b0_all, const float* w1_all)
{
  const int t = P.atoms[i].type;
  float q[DIMP], Fp[DIMP];
#pragma unroll
  for (int d = 0; d < DIMP; ++d)
    q[d] = (d < P.dim) ? P.q[(size_t)d * P.n + i] * B2_LDG(&P.q_scaler[d]) : 0.0f;
  const float F = b2_mlp_core<DIMP, GLOBAL_W>(
    q, reinterpret_cast<const float4*>(w0_all + (size_t)t * P.nneu * DIMP), b0_all + (size_t)t * P.nneu,
    w1_all + (size_t)t * P.nneu, P.nneu, B2_LDG(&P.bias[t]), P.q_scaler, Fp);
  P.acc[i] = (double)F;
  // dU/dq: radial part first (input of the U-table contraction), then the angular part
#pragma unroll
  for (int d = 0; d < DIMP; ++d) {
    if (d < P.nr1)
      P.FpR[(size_t)d * P.n + i] = Fp[d];
    else if (d < P.dim)
      P.FpA[(size_t)(d - P.nr1) * P.n + i] = Fp[d];
  }
}

// radial pre-contraction U_i[t2][k] = sum_n Fp_i[n] c[t_i,t2,n,k]  (one AoS row per atom, see
// b2_body_force_radial)
template <int K1>
B2_HD void b2_body_utable(int i, const B2NepView& P)
{
  constexpr int KP = (K1 + 3) / 4 * 4;
  const int t = P.atoms[i].type;
  float* U = P.U + (size_t)i * P.UST;
  for (int t2 = 0; t2 < P.nt; ++t2) {
    const float* c = P.c_r + (size_t)(t * P.nt + t2) * P.nr1 * K1;
    float u[KP];
#pragma unroll
    for (int k = 0; k < KP; ++k)
      u[k] = 0.0f;
    for (int n = 0; n < P.nr1; ++n) {
      const float f = P.FpR[(size_t)n * P.n + i];
#pragma unroll
      for (int k = 0; k < K1; ++k)
        u[k] = fmaf(f, B2_LDG(&c[n * K1 + k]), u[k]);
    }
#pragma unroll
    for (int k = 0; k < KP; ++k)
      U[t2 * KP + k] = u[k];
  }
}

// for (n = 0; n < count; n += step) f(n): fully unrolled when FIXED (count is then a compile-time constant,
// k_angular_fused on a fixed angular shape), otherwise left to the compiler as a run-time loop
template <bool FIXED, class F>
B2_HD void b2_channel_loop(int count, int step, F f)
{
  if constexpr (FIXED) {
#pragma unroll
    for (int n = 0; n < count; n += step)
      f(n);
  } else {
    for (int n = 0; n < count; n += step)
      f(n);
  }
}

// same contraction into the compact planes of the few-type kernels (B2NepView::u_planes == 2):
// KQ = (K1-1)/4 float4 planes U4[(t2*KQ + q)*n + i] and a float plane [t2*n + i] for k = K1-1.
// fr(n) = dU/dq[n] of atom i (type t), n < nr1.  Shared by k_utable and k_angular_fused.  NR1 > 0: nr1 is
// that compile-time constant (k_angular_fused on a fixed model shape), so fr is called with constants.
template <int K1, int NR1 = 0, class FpR>
B2_HD void b2_utable_compact(const B2NepView& P, int i, int t, FpR fr)
{
  constexpr int KQ = (K1 - 1) / 4;
  const int nr1 = NR1 > 0 ? NR1 : P.nr1;
  float4* U4 = reinterpret_cast<float4*>(P.U);
  float* Uf = P.U + (size_t)P.nt * KQ * 4 * P.n;
  for (int t2 = 0; t2 < P.nt; ++t2) {
    const float* c = P.c_r + (size_t)(t * P.nt + t2) * nr1 * K1;
    float u[K1];
#pragma unroll
    for (int k = 0; k < K1; ++k)
      u[k] = 0.0f;
    b2_channel_loop<(NR1 > 0)>(nr1, 1, [&](int n) {
      const float f = fr(n);
#pragma unroll
      for (int k = 0; k < K1; ++k)
        u[k] = fmaf(f, B2_LDG(&c[n * K1 + k]), u[k]);
    });
#pragma unroll
    for (int q = 0; q < KQ; ++q) {
      float4 v;
      v.x = u[4 * q];
      v.y = u[4 * q + 1];
      v.z = u[4 * q + 2];
      v.w = u[4 * q + 3];
      U4[(size_t)(t2 * KQ + q) * P.n + i] = v;
    }
    Uf[(size_t)t2 * P.n + i] = u[K1 - 1];
  }
}

// same contraction, written as float4 planes U4[(t2*KP/4 + q)*n + i] for the lane-team radial force
template <int K1>
B2_HD void b2_body_utable_planes(int i, const B2NepView& P)
{
  constexpr int KP4 = (K1 + 3) / 4;
  const int t = P.atoms[i].type;
  float4* U4 = reinterpret_cast<float4*>(P.U);
  for (int t2 = 0; t2 < P.nt; ++t2) {
    const float* c = P.c_r + (size_t)(t * P.nt + t2) * P.nr1 * K1;
    float u[KP4 * 4];
#pragma unroll
    for (int k = 0; k < KP4 * 4; ++k)
      u[k] = 0.0f;
    for (int n = 0; n < P.nr1; ++n) {
      const float f = P.FpR[(size_t)n * P.n + i];
#pragma unroll
      for (int k = 0; k < K1; ++k)
        u[k] = fmaf(f, B2_LDG(&c[n * K1 + k]), u[k]);
    }
#pragma unroll
    for (int q = 0; q < KP4; ++q) {
      float4 v;
      v.x = u[4 * q];
      v.y = u[4 * q + 1];
      v.z = u[4 * q + 2];
      v.w = u[4 * q + 3];
      U4[(size_t)(t2 * KP4 + q) * P.n + i] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// radial force (find_force_radial, nep.cu:661-772) in the pre-contracted form:
//   F_i   += (A + B) * r12 / d,   A = fn'(d) . U_i[t_j],  B = fn'(d) . U_j[t_i]
//   W_i^ab += r12^a * f21^b,      f21 = -B * r12 / d
// ---------------------------------------------------------------------------------------------
// out[12] = fx,fy,fz, vxx,vyy,vzz,vxy,vxz,vyz,vyx,vzx,vzy (FP32 partial sums of this stage)
// one pair of the radial force; acc = fx,fy,fz,vxx,vyy,vzz,vxy,vxz,vyz
template <int NT, int K1>
B2_HD void b2_radial_pair(
  const B2NepView& P, const B2Geo& geo, const B2Box& box, const B2Atom& a1, int t1,
  const B2Atom& a2, const float* Uj, const float (*Ur)[K1], const float* rcv, const float* rciv,
  const float* Ui, float* acc)
{
  float x12, y12, z12;
  b2_r12(geo, box, a1, a2, x12, y12, z12);
  const float d2 = b2_d2(x12, y12, z12);
  const float dinv = b2_rsqrt(d2);
  const float d = d2 * dinv;
  const int t2 = a2.type;
  float rc, rcinv;
  if (NT == 1) {
    rc = rcv[0];
    rcinv = rciv[0];
  } else if (NT > 1) {
    rc = rcv[0];
    rcinv = rciv[0];
#pragma unroll
    for (int t = 1; t < (NT > 0 ? NT : 1); ++t) {
      rc = (t2 == t) ? rcv[t] : rc;
      rcinv = (t2 == t) ? rciv[t] : rcinv;
    }
  } else {
    const int pair = t1 * P.nt + t2;
    rc = B2_LDG(&P.rc_r[pair]);
    rcinv = B2_LDG(&P.rcinv_r[pair]);
  }
  float fnp[K1];
  b2_basis_d<K1, false>(d, rc, rcinv, nullptr, fnp);
  float A = 0.0f, Bv = 0.0f;
  if (NT == 1) {
#pragma unroll
    for (int k = 0; k < K1; ++k)
      A = fmaf(fnp[k], Ur[0][k], A);
  } else if (NT > 1) {
#pragma unroll
    for (int k = 0; k < K1; ++k) {
      float u = Ur[0][k];
#pragma unroll
      for (int t = 1; t < (NT > 0 ? NT : 1); ++t)
        u = (t2 == t) ? Ur[t][k] : u;
      A = fmaf(fnp[k], u, A);
    }
  } else {
    // own row U_i[t2]: every lane reads a different row, so 128-bit loads (rows are KP = 4*KQ
    // floats, 16-byte aligned) cost a quarter of the L1 wavefronts of K1 scalar ones
    constexpr int KQ = (K1 + 3) / 4;
    const float4* Uit = reinterpret_cast<const float4*>(Ui + t2 * P.KP);
    float u[KQ * 4];
#pragma unroll
    for (int q = 0; q < KQ; ++q) {
      const float4 v = Uit[q];
      u[4 * q] = v.x;
      u[4 * q + 1] = v.y;
      u[4 * q + 2] = v.z;
      u[4 * q + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < K1; ++k)
      A = fmaf(fnp[k], u[k], A);
  }
#pragma unroll
  for (int k = 0; k < K1; ++k)
    Bv = fmaf(fnp[k], Uj[k], Bv);
  const float sA = (A + Bv) * dinv;
  const float sB = -Bv * dinv; // f21 = sB * r12
  acc[0] = fmaf(sA, x12, acc[0]);
  acc[1] = fmaf(sA, y12, acc[1]);
  acc[2] = fmaf(sA, z12, acc[2]);
  acc[3] = fmaf(x12 * x12, sB, acc[3]);
  acc[4] = fmaf(y12 * y12, sB, acc[4]);
  acc[5] = fmaf(z12 * z12, sB, acc[5]);
  acc[6] = fmaf(x12 * y12, sB, acc[6]);
  acc[7] = fmaf(x12 * z12, sB, acc[7]);
  acc[8] = fmaf(y12 * z12, sB, acc[8]);
}

// DEPTH = neighbours whose record and U row are in flight while one is evaluated (1 or 2); the
// loop is latency-bound on those dependent gathers (index -> record / U row)
template <int NT, int K1, int DEPTH>
B2_HD void b2_force_radial_sum(int i, const B2NepView& P, const B2Box& box, float* out)
{
  constexpr int KP4 = (K1 + 3) / 4; // float4 loads per U row (KP = 4*KP4)
  constexpr int NTA = NT > 0 ? NT : 1;
  const B2Geo geo = b2_geo(box);
  const size_t N = (size_t)P.n;
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  const int nn = P.nn_r[i];
  const float* Ui = P.U + (size_t)i * P.UST;
  float Ur[NTA][K1];
  float rcv[NTA], rciv[NTA]; // pair cutoffs of (t1, t) for the few-type path
  if (NT > 0) {
#pragma unroll
    for (int t = 0; t < NTA; ++t) {
      const int pr = t1 * P.nt + (t < P.nt ? t : 0);
      rcv[t] = B2_LDG(&P.rc_r[pr]);
      rciv[t] = B2_LDG(&P.rcinv_r[pr]);
#pragma unroll
      for (int k = 0; k < K1; ++k)
        Ur[t][k] = (t < P.nt) ? Ui[t * P.KP + k] : 0.0f;
    }
  }
  float acc[9];
#pragma unroll
  for (int k = 0; k < 9; ++k)
    acc[k] = 0.0f;
  const float4* Ubase = reinterpret_cast<const float4*>(P.U + (size_t)t1 * P.KP);
  const size_t ust4 = (size_t)P.UST / 4;
  // software pipeline: records / U rows of the next DEPTH neighbours and the index after them
  // are in flight while neighbour s is evaluated
  B2Atom an[DEPTH];
  float4 un[DEPTH][KP4];
#pragma unroll
  for (int p = 0; p < DEPTH; ++p) {
    const int jp = p < nn ? B2_LDCS(&P.nl_r[(size_t)p * N + i]) : i;
    an[p] = b2_load_atom(&P.atoms[jp]);
#pragma unroll
    for (int q = 0; q < KP4; ++q)
      un[p][q] = B2_LDG(&Ubase[(size_t)jp * ust4 + q]);
  }
  int jnext = DEPTH < nn ? B2_LDCS(&P.nl_r[(size_t)DEPTH * N + i]) : i;
  for (int s = 0; s < nn; s += DEPTH) {
#pragma unroll
    for (int p = 0; p < DEPTH; ++p) {
      const B2Atom a2 = an[p];
      float Uj[KP4 * 4];
#pragma unroll
      for (int q = 0; q < KP4; ++q) {
        Uj[4 * q] = un[p][q].x;
        Uj[4 * q + 1] = un[p][q].y;
        Uj[4 * q + 2] = un[p][q].z;
        Uj[4 * q + 3] = un[p][q].w;
      }
      // refill slot p with neighbour s + p + DEPTH, fetch the index after it
      const int jl = jnext;
      an[p] = b2_load_atom(&P.atoms[jl]);
#pragma unroll
      for (int q = 0; q < KP4; ++q)
        un[p][q] = B2_LDG(&Ubase[(size_t)jl * ust4 + q]);
      jnext = (s + p + DEPTH + 1 < nn) ? B2_LDCS(&P.nl_r[(size_t)(s + p + DEPTH + 1) * N + i]) : i;
      if (s + p < nn)
        b2_radial_pair<NT, K1>(P, geo, box, a1, t1, a2, Uj, Ur, rcv, rciv, Ui, acc);
    }
  }
  out[0] = acc[0];
  out[1] = acc[1];
  out[2] = acc[2];
  out[3] = acc[3];
  out[4] = acc[4];
  out[5] = acc[5];
  out[6] = acc[6];
  out[7] = acc[7];
  out[8] = acc[8];
  out[9] = acc[6];  // yx: the radial pair virial r12 (x) f21 is symmetric
  out[10] = acc[7]; // zx
  out[11] = acc[8]; // zy
}

// ---------------------------------------------------------------------------------------------
// angular partial forces (find_partial_force_angular, nep.cu:774-861, accumulate_f12
// nep_utilities.cuh:1523-1672).  `w` is scratch for the per-atom weights dU/ds[n][abc], laid out
// w[(n*24+abc)*stride + lane] (shared memory on the device).
// ---------------------------------------------------------------------------------------------
// STRIDE = threads per block (compile-time so that the scratch offsets are immediates; the host
// build of tests/emu uses 1)
template <int K1, int STRIDE>
B2_HD void b2_body_force_angular(
  int i, const B2NepView& P, const B2Box& box, float* w, int lane, const float4* ctab,
  int rs4) // ctab / rs4 as in b2_body_desc_angular
{
  constexpr size_t stride = STRIDE;
  const float C3B[B2_NABC] = {B2_C3B_LIST};
  const size_t N = (size_t)P.n;
  // dU/dq of this atom: tile-major copy written by k_mlp_tc (component d at fbase + (d/4)*512 + d%4),
  // or the SoA columns FpA[(d - nr1)*N + i] of the SIMT layer
  const float* fbase = P.fpt ? P.fpt + b2_tile_offset(P.DKT, P.tile_slot[i], 0) : nullptr;
  auto FpAt = [&](int da) -> float { // da = index inside the angular part
    if (fbase) {
      const int d = P.nr1 + da;
      return fbase[(size_t)(d >> 2) * 512 + (d & 3)];
    }
    return P.FpA[(size_t)da * N + i];
  };
  // ---- weights: 3-body (calculate_s_one, nep_utilities.cuh:1327-1340) + chain rule of the
  //      4-body (:625-679) and 5-body (:681-718) invariants ----
  for (int n = 0; n < P.na1; ++n) {
    float s[B2_NABC];
#pragma unroll
    for (int abc = 0; abc < B2_NABC; ++abc)
      s[abc] = P.sfx[(size_t)(n * B2_NABC + abc) * N + i];
    float wv[B2_NABC];
    int st = 0;
#pragma unroll
    for (int L = 1; L <= 4; ++L) {
      const float F = FpAt((L - 1) * P.na1 + n);
      wv[st] = 2.0f * F * C3B[st] * s[st];
#pragma unroll
      for (int k = 1; k < 2 * L + 1; ++k)
        wv[st + k] = 4.0f * F * C3B[st + k] * s[st + k];
      st += 2 * L + 1;
    }
    int Lidx = 4;
    if (P.has222) {
      const float F = FpAt(Lidx * P.na1 + n);
      const float* t = &s[3];
      wv[3] += F * (3.0f * B2_C4B0 * t[0] * t[0] + B2_C4B1 * (t[1] * t[1] + t[2] * t[2]) +
                    B2_C4B2 * (t[3] * t[3] + t[4] * t[4]));
      wv[4] += F * (2.0f * B2_C4B1 * t[0] * t[1] - 2.0f * B2_C4B3 * t[3] * t[1] + B2_C4B4 * t[2] * t[4]);
      wv[5] += F * (2.0f * B2_C4B1 * t[0] * t[2] + 2.0f * B2_C4B3 * t[3] * t[2] + B2_C4B4 * t[1] * t[4]);
      wv[6] += F * (2.0f * B2_C4B2 * t[0] * t[3] + B2_C4B3 * (t[2] * t[2] - t[1] * t[1]));
      wv[7] += F * (2.0f * B2_C4B2 * t[0] * t[4] + B2_C4B4 * t[1] * t[2]);
      ++Lidx;
    }
    if (P.has1111) {
      const float F = FpAt(Lidx * P.na1 + n);
      const float tt = s[1] * s[1] + s[2] * s[2];
      wv[0] += F * (4.0f * B2_C5B0 * s[0] * s[0] * s[0] + 2.0f * B2_C5B1 * tt * s[0]);
      wv[1] += F * (2.0f * B2_C5B1 * s[0] * s[0] * s[1] + 4.0f * B2_C5B2 * tt * s[1]);
      wv[2] += F * (2.0f * B2_C5B1 * s[0] * s[0] * s[2] + 4.0f * B2_C5B2 * tt * s[2]);
      ++Lidx;
    }
#pragma unroll
    for (int abc = 0; abc < B2_NABC; ++abc)
      w[(size_t)(n * B2_NABC + abc) * stride + lane] = wv[abc];
  }
  // ---- pairs ----
  const B2Geo geo = b2_geo(box);
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  const int nn = P.nn_a[i];
  const size_t plane = (size_t)P.mn_a * N;
  // gathers one neighbour ahead (record) / two ahead (index), as in the radial kernels
  int jn = nn > 0 ? P.nl_a[i] : i;
  B2Atom an = b2_load_atom(&P.atoms[jn]);
  int j2 = nn > 1 ? P.nl_a[N + i] : i;
  for (int m = 0; m < nn; ++m) {
    const B2Atom a2 = an;
    an = b2_load_atom(&P.atoms[j2]);
    j2 = (m + 2 < nn) ? P.nl_a[(size_t)(m + 2) * N + i] : i;
    float x12, y12, z12;
    b2_r12(geo, box, a1, a2, x12, y12, z12);
    const float d = sqrtf(b2_d2(x12, y12, z12));
    const float dinv = 1.0f / d;
    const int pair = t1 * P.nt + a2.type;
    float fn[K1], fnp[K1];
    b2_basis_d<K1, true>(d, B2_LDG(&P.rc_a[pair]), B2_LDG(&P.rcinv_a[pair]), fn, fnp);
    float W[B2_NABC], Wp[B2_NABC];
#pragma unroll
    for (int abc = 0; abc < B2_NABC; ++abc) {
      W[abc] = 0.0f;
      Wp[abc] = 0.0f;
    }
    for (int n = 0; n < P.na1; ++n) {
      float g = 0.0f, gp = 0.0f;
      constexpr int KQ = (K1 + 3) / 4;
      const float4* c4 = ctab + (size_t)pair * rs4 + n * KQ;
      float ck[KQ * 4];
#pragma unroll
      for (int q = 0; q < KQ; ++q) {
        const float4 v = c4[q];
        ck[4 * q] = v.x;
        ck[4 * q + 1] = v.y;
        ck[4 * q + 2] = v.z;
        ck[4 * q + 3] = v.w;
      }
#pragma unroll
      for (int k = 0; k < K1; ++k) {
        g = fmaf(fn[k], ck[k], g);
        gp = fmaf(fnp[k], ck[k], gp);
      }
      const float* wn = w + (size_t)(n * B2_NABC) * stride + lane;
#pragma unroll
      for (int abc = 0; abc < B2_NABC; ++abc) {
        const float wv = wn[(size_t)abc * stride];
        W[abc] = fmaf(g, wv, W[abc]);
        Wp[abc] = fmaf(gp, wv, Wp[abc]);
      }
    }
    const float xh = x12 * dinv, yh = y12 * dinv, zh = z12 * dinv;
    float B[B2_NABC];
    b2_harmonics(xh, yh, zh, B);
    // radial part: sum_abc (g' - L g / r) w b(rhat)
    float ar = 0.0f, al = 0.0f;
    {
      int st = 0;
#pragma unroll
      for (int L = 1; L <= 4; ++L) {
        float tl = 0.0f;
#pragma unroll
        for (int k = 0; k < 2 * L + 1; ++k) {
          ar = fmaf(Wp[st + k], B[st + k], ar);
          tl = fmaf(W[st + k], B[st + k], tl);
        }
        al = fmaf((float)L, tl, al);
        st += 2 * L + 1;
      }
    }
    float gx, gy, gz;
    b2_harmonics_grad_dot(xh, yh, zh, W, gx, gy, gz);
    const float rad = ar - al * dinv;
    const size_t slot = (size_t)m * N + i;
    P.f12[slot] = fmaf(rad, xh, gx * dinv);
    P.f12[plane + slot] = fmaf(rad, yh, gy * dinv);
    P.f12[2 * plane + slot] = fmaf(rad, zh, gz * dinv);
  }
}

// ---------------------------------------------------------------------------------------------
// F_i = sum_j (f12_ij - f12_ji), W_i = sum_j r_ij (x) f12_ji
// (gpu_find_force_many_body, src/force/potential.cu:170-297; the reverse slot is found by binary
// search in j's ascending list, potential.cu:226-247)
// ---------------------------------------------------------------------------------------------
// m0 / mstep: the neighbours m0, m0+mstep, ... are summed (0, 1 = all; a lane team passes lane, B2_TEAM)
B2_HD void b2_reduce_angular_sum(
  int i, const B2NepView& P, const B2Box& box, float* out, int m0 = 0, int mstep = 1)
{
  const size_t N = (size_t)P.n;
  const size_t plane = (size_t)P.mn_a * N;
  const B2Atom a1 = P.atoms[i];
  const int nn = P.nn_a[i];
  float f[3] = {0.0f, 0.0f, 0.0f};
  float v[9] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f}; // row-major r (x) f21
  for (int m = m0; m < nn; m += mstep) {
    const size_t slot = (size_t)m * N + i;
    const int j = P.nl_a[slot];
    const B2Atom a2 = P.atoms[j];
    double xd = a2.x - a1.x, yd = a2.y - a1.y, zd = a2.z - a1.z;
    b2_mic(box, xd, yd, zd); // potential.cu:211-217: FP64 minimum image, then narrowed
    const float r[3] = {(float)xd, (float)yd, (float)zd};
    int rev = 0;
    if (P.aslot) {
      // direct: j's angular slot for its skin neighbour i (same value the search below finds)
      rev = P.aslot[(size_t)P.nla_rs[slot] * N + j];
      rev = rev < 0 ? 0 : rev;
    } else {
      int lo = 0, hi = P.nn_a[j] - 1;
      while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const int v2 = P.nl_a[(size_t)mid * N + j];
        if (v2 < i)
          lo = mid + 1;
        else if (v2 > i)
          hi = mid - 1;
        else {
          rev = mid;
          break;
        }
      }
    }
    const size_t rslot = (size_t)rev * N + j;
    const float f12[3] = {P.f12[slot], P.f12[plane + slot], P.f12[2 * plane + slot]};
    const float f21[3] = {P.f12[rslot], P.f12[plane + rslot], P.f12[2 * plane + rslot]};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      f[a] += f12[a] - f21[a];
#pragma unroll
      for (int b = 0; b < 3; ++b)
        v[a * 3 + b] = fmaf(r[a], f21[b], v[a * 3 + b]);
    }
  }
  out[0] = f[0];
  out[1] = f[1];
  out[2] = f[2];
  out[3] = v[0];  // xx
  out[4] = v[4];  // yy
  out[5] = v[8];  // zz
  out[6] = v[1];  // xy
  out[7] = v[2];  // xz
  out[8] = v[5];  // yz
  out[9] = v[3];  // yx
  out[10] = v[6]; // zx
  out[11] = v[7]; // zy
}

// ---------------------------------------------------------------------------------------------
// ZBL pair repulsion over the angular list (find_force_ZBL, nep.cu:863-975;
// find_f_and_fp_zbl nep_utilities.cuh:433-508)
// ---------------------------------------------------------------------------------------------
B2_HD void b2_zbl_pair(
  const float* para8 /* a0,b0,...,a3,b3 */, float r1, float r2, float zizj, float a_inv, float d,
  float dinv, float& f, float& fp)
{
  const float x = d * a_inv;
  float phi = 0.0f, phip = 0.0f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float t = para8[2 * k] * expf(-para8[2 * k + 1] * x);
    phi += t;
    phip -= para8[2 * k + 1] * t;
  }
  phi *= zizj;
  phip *= zizj * a_inv;
  phip = phip * dinv - phi * dinv * dinv;
  phi *= dinv;
  float fc, fcp;
  if (d < r1) {
    fc = 1.0f;
    fcp = 0.0f;
  } else if (d < r2) {
    const float pf = 3.1415927f / (r2 - r1);
    fc = cosf(pf * (d - r1)) * 0.5f + 0.5f;
    fcp = -sinf(pf * (d - r1)) * pf * 0.5f;
  } else {
    fc = 0.0f;
    fcp = 0.0f;
  }
  fp = phip * fc + phi * fcp;
  f = phi * fc;
}

B2_HD void b2_zbl_sum(
  int i, const B2NepView& P, const B2Box& box, float* out, float& pe_out, int m0 = 0, int mstep = 1)
{
  const size_t N = (size_t)P.n;
  const B2Geo geo = b2_geo(box);
  const B2Atom a1 = P.atoms[i];
  const int ty1 = a1.type;
  const int zi = B2_LDG(&P.zbl_z[ty1]);
  const float pzi = powf((float)zi, 0.23f);
  const int nn = P.nn_a[i];
  float pe = 0.0f, f[3] = {0.0f, 0.0f, 0.0f};
  float vxx = 0.0f, vyy = 0.0f, vzz = 0.0f, vxy = 0.0f, vxz = 0.0f, vyz = 0.0f;
  for (int m = m0; m < nn; m += mstep) {
    const int j = P.nl_a[(size_t)m * N + i] & B2_TAG_MASK; // the few-type path tags the entries
    const B2Atom a2 = b2_load_atom(&P.atoms[j]);
    float x12, y12, z12;
    b2_r12(geo, box, a1, a2, x12, y12, z12);
    const float d = sqrtf(b2_d2(x12, y12, z12));
    const float dinv = 1.0f / d;
    const int ty2 = a2.type;
    const int zj = B2_LDG(&P.zbl_z[ty2]);
    // Outer cutoff of this pair first: beyond it the switching function and its derivative are exactly
    // zero, every contribution below is +-0 and the sums are unchanged -- so the four exponentials, the
    // power and the sin/cos are skipped.  (The reference evaluates them and multiplies by zero.)
    float para[10];
    float rin = P.zbl_rc_inner, rout = P.zbl_rc_outer;
    if (P.zbl_flexible) {
      const int ta = ty1 < ty2 ? ty1 : ty2, tb = ty1 < ty2 ? ty2 : ty1;
      const int zidx = ta * P.nt - (ta * (ta - 1)) / 2 + (tb - ta);
#pragma unroll
      for (int k = 0; k < 10; ++k)
        para[k] = B2_LDG(&P.zbl_para[10 * zidx + k]);
      rin = para[0];
      rout = para[1];
    } else if (P.zbl_typewise) {
      const float tw =
        (B2_LDG(&P.cov_radius[zi - 1]) + B2_LDG(&P.cov_radius[zj - 1])) * P.zbl_typewise_factor;
      rout = fminf(tw, rout);
      rin = 0.0f;
    }
    if (!(d < rout))
      continue;
    const float a_inv = (pzi + powf((float)zj, 0.23f)) * 2.134563f;
    const float zizj = 14.399645f * (float)zi * (float)zj; // K_C_SP, common.cuh:23
    float fv, fpv;
    if (P.zbl_flexible) {
      b2_zbl_pair(para + 2, rin, rout, zizj, a_inv, d, dinv, fv, fpv);
    } else {
      const float uni[8] = {0.18175f, 3.1998f, 0.50986f, 0.94229f,
                            0.28022f, 0.4029f, 0.02817f, 0.20162f};
      b2_zbl_pair(uni, rin, rout, zizj, a_inv, d, dinv, fv, fpv);
    }
    const float f2 = fpv * dinv * 0.5f; // f12 = r12 * f2, f21 = -f12
    f[0] += 2.0f * (x12 * f2);
    f[1] += 2.0f * (y12 * f2);
    f[2] += 2.0f * (z12 * f2);
    vxx -= x12 * (x12 * f2);
    vyy -= y12 * (y12 * f2);
    vzz -= z12 * (z12 * f2);
    vxy -= x12 * (y12 * f2);
    vxz -= x12 * (z12 * f2);
    vyz -= y12 * (z12 * f2);
    pe += fv * 0.5f;
  }
  pe_out = pe;
  out[0] = f[0];
  out[1] = f[1];
  out[2] = f[2];
  out[3] = vxx;
  out[4] = vyy;
  out[5] = vzz;
  out[6] = vxy;
  out[7] = vxz;
  out[8] = vyz;
  out[9] = vxy;
  out[10] = vxz;
  out[11] = vyz;
}

// ---------------------------------------------------------------------------------------------
// Final force kernel: radial pair forces + angular pair reduction (+ ZBL) for one atom, then ONE
// scatter into the caller's FP64 arrays with += (the accumulate convention of Potential::compute,
// nep.cu:653,755-770).  Each stage keeps its own FP32 partial sums and they are combined in FP64,
// exactly like the reference's separate kernels adding into double arrays.
// ---------------------------------------------------------------------------------------------
template <int NT, int K1, int DEPTH = 1>
B2_HD void b2_body_force_final(
  int i, const B2NepView& P, const B2Box& box, double* pe, double* force, double* virial)
{
  if (P.n_own > 0 && P.perm[i] >= P.n_own)
    return; // ghost atom of a spatial domain
  float r[12], a[12], z[12];
  float zpe = 0.0f;
  if (!(P.debug_skip & 1))
    b2_force_radial_sum<NT, K1, DEPTH>(i, P, box, r);
  else
    for (int k = 0; k < 12; ++k)
      r[k] = 0.0f;
  if (!(P.debug_skip & 2))
    b2_reduce_angular_sum(i, P, box, a);
  else
    for (int k = 0; k < 12; ++k)
      a[k] = 0.0f;
  if (P.zbl_enabled && !(P.debug_skip & 4)) {
    b2_zbl_sum(i, P, box, z, zpe);
  } else {
#pragma unroll
    for (int k = 0; k < 12; ++k)
      z[k] = 0.0f;
  }
  const int dst = P.perm[i];
  const size_t N = (size_t)P.n;
  if (P.overwrite) {
    pe[dst] = P.acc[i] + (double)zpe;
#pragma unroll
    for (int k = 0; k < 3; ++k)
      force[k * N + dst] = (double)r[k] + (double)a[k] + (double)z[k];
#pragma unroll
    for (int k = 0; k < 9; ++k)
      virial[k * N + dst] = (double)r[3 + k] + (double)a[3 + k] + (double)z[3 + k];
    return;
  }
  pe[dst] += P.acc[i] + (double)zpe; // acc[i] = site energy from the MLP pass
#pragma unroll
  for (int k = 0; k < 3; ++k)
    force[k * N + dst] += (double)r[k] + (double)a[k] + (double)z[k];
#pragma unroll
  for (int k = 0; k < 9; ++k)
    virial[k * N + dst] += (double)r[3 + k] + (double)a[3 + k] + (double)z[3 + k];
}

// =============================================================================================
// Lane-team variants of the two radial passes (models with <= 2 types, NT = number of types).
// Team lane l of atom i handles list entries l, l+B2_TEAM, ...; partial sums are combined with
// b2_team_sum.  Lists: skin and radial row-major (see B2NepView::skin_si / pitch_r), angular
// column-major (its consumers are thread-per-atom).  Same arithmetic per pair as the
// thread-per-atom bodies; only the summation order over neighbours differs.
// =============================================================================================
template <int NT, int K1>
B2_HD void b2_team_desc_radial(int i, int l, const B2NepView& P, const B2Box& box)
{
  constexpr int G = B2_TEAM;
  const B2Geo geo = b2_geo(box);
  const size_t N = (size_t)P.n;
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  if (!b2_is_active(P, a1.x, a1.y, a1.z)) { // as in b2_body_desc_radial (uniform over the team)
    if (l == 0) {
      P.nn_r[i] = 0;
      P.nn_a[i] = 0;
    }
    for (int n = l; n < P.nr1; n += G)
      *b2_q_ptr(P, i, P.qt ? P.tile_slot[i] : 0, n) = 0.0f;
    return;
  }
  const int nn = P.nn_skin[i];
  const int* row = P.nl_skin + (size_t)i * P.skin_si;
  int* out_r = P.nl_r + (size_t)i * P.pitch_r;
  float S[NT][K1];
  float rcv[NT], rciv[NT], rc2r[NT], rc2a[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int pr = t1 * P.nt + (t < P.nt ? t : 0);
    rcv[t] = B2_LDG(&P.rc_r[pr]);
    rciv[t] = B2_LDG(&P.rcinv_r[pr]);
    rc2r[t] = B2_LDG(&P.rc2_r[pr]);
    rc2a[t] = B2_LDG(&P.rc2_a[pr]);
#pragma unroll
    for (int k = 0; k < K1; ++k)
      S[t][k] = 0.0f;
  }
  int cr = 0, ca = 0;
  const unsigned below = (1u << l) - 1u;
  // software pipeline as in the thread-per-atom bodies: record one entry ahead, index two ahead
  int jn = l < nn ? row[l] : i;
  B2Atom an = b2_load_atom(&P.atoms[jn]);
  int j2 = l + G < nn ? row[l + G] : i;
  for (int k0 = 0; k0 < nn; k0 += G) {
    const bool valid = k0 + l < nn;
    const int j = jn;
    const B2Atom a2 = an;
    jn = j2;
    an = b2_load_atom(&P.atoms[j2]);
    j2 = (k0 + l + 2 * G < nn) ? row[k0 + l + 2 * G] : i;
    float x12, y12, z12;
    b2_r12(geo, box, a1, a2, x12, y12, z12);
    const float d2 = b2_d2(x12, y12, z12);
    const int t2 = a2.type;
    float rc = rcv[0], rcinv = rciv[0], r2r = rc2r[0], r2a = rc2a[0];
#pragma unroll
    for (int t = 1; t < NT; ++t) {
      rc = (t2 == t) ? rcv[t] : rc;
      rcinv = (t2 == t) ? rciv[t] : rcinv;
      r2r = (t2 == t) ? rc2r[t] : r2r;
      r2a = (t2 == t) ? rc2a[t] : r2a;
    }
    // the reference's membership tests (nep.cu:473-484), list order = ascending sorted index
    const bool inr = valid && d2 < r2r;
    const bool ina = inr && d2 < r2a;
    const unsigned mr = b2_team_ballot(inr), ma = b2_team_ballot(ina);
    if (inr) {
      const int pos = cr + B2_POPC(mr & below);
      if (pos < P.mn_r)
        out_r[pos] = j;
    }
    if (ina) {
      const int pos = ca + B2_POPC(ma & below);
      if (pos < P.mn_a)
        P.nl_a[(size_t)pos * N + i] = j;
    }
    cr += B2_POPC(mr);
    ca += B2_POPC(ma);
    if (inr) {
      float fn[K1];
      b2_basis<K1>(sqrtf(d2), rc, rcinv, fn);
      if (NT == 1) {
#pragma unroll
        for (int k = 0; k < K1; ++k)
          S[0][k] += fn[k];
      } else {
#pragma unroll
        for (int t = 0; t < NT; ++t) {
          const float m = (t2 == t) ? 1.0f : 0.0f;
#pragma unroll
          for (int k = 0; k < K1; ++k)
            S[t][k] = fmaf(m, fn[k], S[t][k]);
        }
      }
    }
  }
  if (l == 0) {
    if (cr > P.mn_r) {
      B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_RADIAL_OVERFLOW);
      cr = P.mn_r;
    }
    if (ca > P.mn_a) {
      B2_ATOMIC_OR(&P.flags[1], (int)B2_ERR_ANGULAR_OVERFLOW);
      ca = P.mn_a;
    }
    P.nn_r[i] = cr;
    P.nn_a[i] = ca;
  }
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int k = 0; k < K1; ++k)
      S[t][k] = b2_team_sum(S[t][k]);
  // contraction with the expansion coefficients, one n per lane
  for (int n = l; n < P.nr1; n += G) {
    float q = 0.0f;
#pragma unroll
    for (int t = 0; t < NT; ++t) {
      if (t < P.nt) {
        const float* c = P.c_r + ((size_t)(t1 * P.nt + t) * P.nr1 + n) * K1;
#pragma unroll
        for (int k = 0; k < K1; ++k)
          q = fmaf(B2_LDG(&c[k]), S[t][k], q);
      }
    }
    *b2_q_ptr(P, i, P.qt ? P.tile_slot[i] : 0, n) = q;
  }
}

// radial pair forces + angular pair reduction (+ ZBL) + the scatter into the caller's arrays;
// the lane-team counterpart of b2_body_force_final
template <int NT, int K1>
B2_HD void b2_team_force_final(
  int i, int l, const B2NepView& P, const B2Box& box, double* pe, double* force, double* virial)
{
  constexpr int G = B2_TEAM;
  constexpr int KP4 = (K1 + 3) / 4;
  if (P.n_own > 0 && P.perm[i] >= P.n_own)
    return; // ghost atom of a spatial domain (uniform over the team)
  const B2Geo geo = b2_geo(box);
  const size_t N = (size_t)P.n;
  const B2Atom a1 = P.atoms[i];
  const int t1 = a1.type;
  const int nn = P.nn_r[i];
  const int* row = P.nl_r + (size_t)i * P.pitch_r;
  const float4* U4 = reinterpret_cast<const float4*>(P.U);
  float Ur[NT][K1];
  float rcv[NT], rciv[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int tt = t < P.nt ? t : 0;
    const int pr = t1 * P.nt + tt;
    rcv[t] = B2_LDG(&P.rc_r[pr]);
    rciv[t] = B2_LDG(&P.rcinv_r[pr]);
    float u[KP4 * 4];
#pragma unroll
    for (int q = 0; q < KP4; ++q) {
      const float4 v = B2_LDG(&U4[(size_t)(tt * KP4 + q) * N + i]);
      u[4 * q] = v.x;
      u[4 * q + 1] = v.y;
      u[4 * q + 2] = v.z;
      u[4 * q + 3] = v.w;
    }
#pragma unroll
    for (int k = 0; k < K1; ++k)
      Ur[t][k] = u[k];
  }
  float fx = 0.0f, fy = 0.0f, fz = 0.0f;
  float vxx = 0.0f, vyy = 0.0f, vzz = 0.0f, vxy = 0.0f, vxz = 0.0f, vyz = 0.0f;
  const float4* Ub = U4 + (size_t)t1 * KP4 * N; // plane q of the neighbour's row for MY type
  int jn = l < nn ? row[l] : i;
  B2Atom an = b2_load_atom(&P.atoms[jn]);
  float4 un[KP4];
#pragma unroll
  for (int q = 0; q < KP4; ++q)
    un[q] = B2_LDG(&Ub[(size_t)q * N + jn]);
  int j2 = l + G < nn ? row[l + G] : i;
  for (int k0 = 0; k0 < nn; k0 += G) {
    const bool valid = k0 + l < nn;
    const B2Atom a2 = an;
    float Uj[KP4 * 4];
#pragma unroll
    for (int q = 0; q < KP4; ++q) {
      Uj[4 * q] = un[q].x;
      Uj[4 * q + 1] = un[q].y;
      Uj[4 * q + 2] = un[q].z;
      Uj[4 * q + 3] = un[q].w;
    }
    an = b2_load_atom(&P.atoms[j2]);
#pragma unroll
    for (int q = 0; q < KP4; ++q)
      un[q] = B2_LDG(&Ub[(size_t)q * N + j2]);
    j2 = (k0 + l + 2 * G < nn) ? row[k0 + l + 2 * G] : i;
    if (!valid)
      continue;
    float x12, y12, z12;
    b2_r12(geo, box, a1, a2, x12, y12, z12);
    const float d2 = b2_d2(x12, y12, z12);
    const float dinv = b2_rsqrt(d2);
    const float d = d2 * dinv;
    const int t2 = a2.type;
    float rc = rcv[0], rcinv = rciv[0];
#pragma unroll
    for (int t = 1; t < NT; ++t) {
      rc = (t2 == t) ? rcv[t] : rc;
      rcinv = (t2 == t) ? rciv[t] : rcinv;
    }
    float fnp[K1];
    b2_basis_d<K1, false>(d, rc, rcinv, nullptr, fnp);
    float A = 0.0f, Bv = 0.0f;
#pragma unroll
    for (int k = 0; k < K1; ++k) {
      float u = Ur[0][k];
#pragma unroll
      for (int t = 1; t < NT; ++t)
        u = (t2 == t) ? Ur[t][k] : u;
      A = fmaf(fnp[k], u, A);
      Bv = fmaf(fnp[k], Uj[k], Bv);
    }
    const float sA = (A + Bv) * dinv;
    const float sB = -Bv * dinv; // f21 = sB * r12
    fx = fmaf(sA, x12, fx);
    fy = fmaf(sA, y12, fy);
    fz = fmaf(sA, z12, fz);
    vxx = fmaf(x12 * x12, sB, vxx);
    vyy = fmaf(y12 * y12, sB, vyy);
    vzz = fmaf(z12 * z12, sB, vzz);
    vxy = fmaf(x12 * y12, sB, vxy);
    vxz = fmaf(x12 * z12, sB, vxz);
    vyz = fmaf(y12 * z12, sB, vyz);
  }
  // this lane's share of the angular pair reduction and of the ZBL pairs
  float a[12], z[12], zpe = 0.0f;
  b2_reduce_angular_sum(i, P, box, a, l, G);
  if (P.zbl_enabled) {
    b2_zbl_sum(i, P, box, z, zpe, l, G);
  } else {
#pragma unroll
    for (int k = 0; k < 12; ++k)
      z[k] = 0.0f;
  }
  float tot[13];
  tot[0] = zpe;
  tot[1] = fx + a[0] + z[0];
  tot[2] = fy + a[1] + z[1];
  tot[3] = fz + a[2] + z[2];
  tot[4] = vxx + a[3] + z[3];
  tot[5] = vyy + a[4] + z[4];
  tot[6] = vzz + a[5] + z[5];
  tot[7] = vxy + a[6] + z[6];
  tot[8] = vxz + a[7] + z[7];
  tot[9] = vyz + a[8] + z[8];
  tot[10] = vxy + a[9] + z[9];   // yx (the radial pair virial is symmetric)
  tot[11] = vxz + a[10] + z[10]; // zx
  tot[12] = vyz + a[11] + z[11]; // zy
#pragma unroll
  for (int k = 0; k < 13; ++k)
    tot[k] = b2_team_sum(tot[k]);
  // scatter (+=, the accumulate convention of Potential::compute, or a store when P.overwrite is
  // set, as in b2_body_force_final): component c by lane c % G
  const int dst = P.perm[i];
#pragma unroll
  for (int c = 0; c < 13; ++c) {
    if (c % G == l) {
      double* out;
      double val;
      if (c == 0) {
        out = &pe[dst];
        val = P.acc[i] + (double)tot[0]; // acc[i] = site energy from the MLP pass
      } else if (c < 4) {
        out = &force[(size_t)(c - 1) * N + dst];
        val = (double)tot[c];
      } else {
        out = &virial[(size_t)(c - 4) * N + dst];
        val = (double)tot[c];
      }
      *out = P.overwrite ? val : *out + val;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// scatter the sorted-order results back to the caller's arrays with += (the accumulate
// convention of Potential::compute, nep.cu:653, 755-770)
// ---------------------------------------------------------------------------------------------
B2_HD void b2_body_unpack(
  int i, int n, const int* perm, const double* acc, double* pe, double* force, double* virial)
{
  const int dst = perm[i];
  const size_t N = (size_t)n;
  pe[dst] += acc[i];
#pragma unroll
  for (int k = 0; k < 3; ++k)
    force[k * N + dst] += acc[(1 + k) * N + i];
#pragma unroll
  for (int k = 0; k < 9; ++k)
    virial[k * N + dst] += acc[(4 + k) * N + i];
}

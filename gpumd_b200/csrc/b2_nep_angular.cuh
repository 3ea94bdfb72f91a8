// b2_nep_angular.cuh -- the angular kernels of the NEP path for models with one or two atom types
// (device only), on the layout of b2_nep_radial.cuh.  Same arithmetic per pair, op for op, as
// b2_body_desc_angular / b2_body_force_angular in b2_nep.cuh (which tests/emu runs on the host and
// which stay the many-type path); what differs is everything around the arithmetic:
//   * neighbours come from the tagged angular list (index | type << B2_TAG_SHIFT, written by
//     k_desc_radial2) and the {x,y} / z position planes: one 16-byte and one 8-byte gather per
//     neighbour instead of a dependent 32-byte record;
//   * the angular pair cutoffs of the <= 2 neighbour types live in registers, the minimum image of an
//     orthogonal box is the branch-free one (b2_rec_r12);
//   * the coefficient rows c_a4 are staged in shared memory once per block;
//   * s[n][abc] travels between the two kernels as float4 planes sfx4[(n*6 + abc/4)*N + i]: the same
//     480 bytes per atom (PbTe) with a quarter of the memory instructions;
//   * the force kernel keeps the per-atom weights dU/ds[n][abc] in shared memory as ONE row per thread,
//     read as float4s (the per-pair W / Wp contraction needs a quarter of the shared-memory loads);
//   * the force kernel also finds, for each pair (i, j), the slot of i in j's angular list and stores
//     it (arev), so that the pair reduction in k_force_final2 (b2_reduce_angular_planes) gathers f21
//     directly instead of walking a binary search of dependent loads;
//   * k_angular_fused runs the descriptor, the hidden layer, the U table and the partial forces of one
//     atom in one thread, so s, dU/dq and the weights never leave the SM (the default where the model
//     fits it, see nep_setup); the two-kernel pair with k_mlp / k_mlp_tc in between stays for the models
//     that do not fit and for B200MD_NEP_MLP=simt / tc.  All of them call the same bodies below.
#pragma once
#include "b2_nep_radial.cuh"

namespace b2 {

constexpr int B2_ABC4 = B2_NABC / 4; // float4 groups of one angular channel

// Shape of the angular model: nr1 radial and na1 angular channels, the 4-body (has222) and 5-body
// (has1111) invariant blocks.  NA1 = 0 reads all four from the model at run time; otherwise they are
// compile-time constants, so the channel loops unroll and dU/dq is indexed with constants.
template <int NR1, int NA1, bool H222, bool H1111>
struct B2AngShape {
  static constexpr bool fixed = NA1 > 0;
  static __device__ __forceinline__ int nr1(const B2NepView& P) { return fixed ? NR1 : P.nr1; }
  static __device__ __forceinline__ int na1(const B2NepView& P) { return fixed ? NA1 : P.na1; }
  static __device__ __forceinline__ int has222(const B2NepView& P) { return fixed ? H222 : P.has222; }
  static __device__ __forceinline__ int has1111(const B2NepView& P) { return fixed ? H1111 : P.has1111; }
  static __device__ __forceinline__ int dim(const B2NepView& P)
  {
    return fixed ? NR1 + NA1 * (4 + (H222 ? 1 : 0) + (H1111 ? 1 : 0)) : P.dim;
  }
  static constexpr int nr1_const = fixed ? NR1 : 0; // 0: run time (b2_utable_compact)
};
using B2AngShapeRT = B2AngShape<0, 0, false, false>;

// angular pair cutoffs of a type-t1 atom against neighbour types 0 .. NT-1, pinned in registers
template <int NT>
__device__ __forceinline__ void b2_ang_cutoffs(const B2NepView& P, int t1, float* rc, float* rcinv)
{
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    const int pr = t1 * P.nt + (t < P.nt ? t : 0);
    rc[t] = __ldg(&P.rc_a[pr]);
    rcinv[t] = __ldg(&P.rcinv_a[pr]);
    B2_PIN_F(rc[t]);
    B2_PIN_F(rcinv[t]);
  }
}

// every block copies the padded angular coefficients c_a4 ([nt*nt][na1][KQ] float4s, <= 2.9 KB with
// two types) to shared memory; the caller syncs
__device__ __forceinline__ void b2_stage_ctab(const B2NepView& P, float4* dst, int KQ)
{
  const int tot = P.nt * P.nt * P.na1 * KQ;
  for (int e = threadIdx.x; e < tot; e += blockDim.x)
    dst[e] = __ldg(&P.c_a4[e]);
}

// ---------------------------------------------------------------------------------------------
// Angular descriptor of sorted atom i (record a1).  The radial index n is processed in chunks of NCH
// channels so that the NCH*24 accumulators stay in registers; each chunk walks the (short) angular
// list once.  NCH = 3 at three blocks per SM (146 registers for PbTe, no spills) measured faster on an
// H100 (400 W, 1 M-atom PbTe: 0.41 ms) than one pass with NCH = 5 at two blocks per SM (198 registers,
// 0.48 ms); NCH = 5 at three blocks spills.
// emit_q(k, v): descriptor component k (nr1 <= k < dim); emit_s(g, v): float4 group g = n*6 + abc/4 of
// the sums s[n][abc].
// ---------------------------------------------------------------------------------------------
template <int NT, int K1, int NCH, bool ORTHO, class SH, class EmitQ, class EmitS>
__device__ __forceinline__ void b2_ang_desc_atom(
  const B2NepView& P, const int4* __restrict__ p0, const double* __restrict__ pz, const B2Box& box,
  int i, const B2Rec& a1, const float4* ctab_s, EmitQ emit_q, EmitS emit_s)
{
  static_assert(NT == 1 || NT == 2, "few-type path");
  constexpr int KQ = (K1 + 3) / 4;
  const B2GeoR geo = b2_geo_pinned(box);
  const unsigned N = (unsigned)P.n;
  const int na1 = SH::na1(P);
  const int t1 = a1.t;
  float rcv[NT], rciv[NT];
  b2_ang_cutoffs<NT>(P, t1, rcv, rciv);
  const float4* crow[NT]; // coefficient rows (t1, t2)
#pragma unroll
  for (int t = 0; t < NT; ++t)
    crow[t] = ctab_s + (t1 * P.nt + (t < P.nt ? t : 0)) * na1 * KQ;
  const int* __restrict__ list = P.nl_a;
  const int nn = P.nn_a[i];
  b2_channel_loop<SH::fixed>(na1, NCH, [&](int n0) {
    float s[NCH][B2_NABC];
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int abc = 0; abc < B2_NABC; ++abc)
        s[c][abc] = 0.0f;
    // list entries two neighbours ahead, positions one ahead
    int e1 = nn > 1 ? __ldg(list + N + i) : i;
    B2Rec rn = b2_rec_load_tagged(p0, pz, nn > 0 ? __ldg(list + i) : i);
    for (int m = 0; m < nn; ++m) {
      const B2Rec a2 = rn;
      rn = b2_rec_load_tagged(p0, pz, e1);
      e1 = (m + 2 < nn) ? __ldg(list + (unsigned)(m + 2) * N + i) : i;
      float x12, y12, z12;
      b2_rec_r12<ORTHO>(geo, box, a1, a2, x12, y12, z12);
      const float d = sqrtf(b2_d2(x12, y12, z12));
      const bool ty = NT > 1 && a2.t != 0;
      float fn[K1];
      b2_basis<K1>(d, ty ? rcv[NT - 1] : rcv[0], ty ? rciv[NT - 1] : rciv[0], fn);
      const float dinv = 1.0f / d;
      float B[B2_NABC];
      b2_harmonics(x12 * dinv, y12 * dinv, z12 * dinv, B);
      const float4* c4 = (ty ? crow[NT - 1] : crow[0]) + n0 * KQ;
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        if (n0 + c < na1) {
          float ck[KQ * 4];
#pragma unroll
          for (int q = 0; q < KQ; ++q) {
            const float4 v = c4[c * KQ + q];
            ck[4 * q] = v.x;
            ck[4 * q + 1] = v.y;
            ck[4 * q + 2] = v.z;
            ck[4 * q + 3] = v.w;
          }
          float g = 0.0f;
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
      if (n < na1) {
        b2_ang_invariants(s[c], SH::has222(P), SH::has1111(P),
                          [&](int blk, float v) { emit_q(SH::nr1(P) + blk * na1 + n, v); });
#pragma unroll
        for (int g = 0; g < B2_ABC4; ++g)
          emit_s(n * B2_ABC4 + g, make_float4(s[c][4 * g], s[c][4 * g + 1], s[c][4 * g + 2], s[c][4 * g + 3]));
      }
    }
  });
}

template <int NT, int K1, int NCH, bool ORTHO>
__global__ void __launch_bounds__(128, 3) k_desc_angular2(
  const B2NepView P, const int4* __restrict__ p0, const int4* __restrict__ p1,
  const double* __restrict__ pz, const B2Box box)
{
  constexpr int KQ = (K1 + 3) / 4;
  extern __shared__ float4 ctab_s[];
  b2_stage_ctab(P, ctab_s, KQ);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n)
    return;
  const unsigned N = (unsigned)P.n;
  const B2Rec a1 = b2_rec_load(p0, p1, i);
  // descriptor component k of this atom: tile-major copy (k_mlp_tc) or SoA columns
  float* const qb = P.qt ? P.qt + b2_tile_offset(P.DKT, P.tile_slot[i], 0) : P.q + i;
  // With the tile-major copy the angular components are collected in shared memory (qs[(k-nr1)*128 + tid],
  // after the coefficient table) and written once at the end as 16-byte groups: written where they are
  // formed, one 4-byte store per component, the groups of a tile row would reach HBM as partial sectors
  // in two passes over the list.
  float* const qs = reinterpret_cast<float*>(ctab_s + P.nt * P.nt * P.na1 * KQ) + threadIdx.x;
  float4* __restrict__ sf4 = reinterpret_cast<float4*>(P.sfx);
  b2_ang_desc_atom<NT, K1, NCH, ORTHO, B2AngShapeRT>(
    P, p0, pz, box, i, a1, ctab_s,
    [&](int k, float v) { *(P.qt ? qs + (size_t)(k - P.nr1) * 128 : qb + (size_t)k * N) = v; },
    [&](int g, float4 v) { sf4[(size_t)g * N + i] = v; });
  if (P.qt) {
    const int klo = P.nr1, khi = P.dim;
    for (int k0 = klo & ~3; k0 < khi; k0 += 4) {
      float* dst = qb + (size_t)(k0 >> 2) * 512;
      if (k0 >= klo && k0 + 4 <= khi) {
        const float* src = qs + (size_t)(k0 - klo) * 128;
        *reinterpret_cast<float4*>(dst) = make_float4(src[0], src[128], src[256], src[384]);
      } else {
        for (int r = 0; r < 4; ++r)
          if (k0 + r >= klo && k0 + r < khi)
            dst[r] = qs[(size_t)(k0 + r - klo) * 128];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Angular partial forces f12 and the reverse slots arev.  Dynamic shared memory: blockDim.x rows of
// WS4 = 6*na1 + 1 float4s (the per-atom weights; the odd row stride keeps the 128-bit accesses of a
// quarter warp on distinct banks), then the coefficient table.
// ---------------------------------------------------------------------------------------------
__host__ __device__ constexpr int b2_ang_ws4(int na1) { return B2_ABC4 * na1 + 1; }

// The pair loop of sorted atom i (record a1): w = its row of weights dU/ds[n][abc] (float4 group
// n*6 + abc/4), ctab_s the staged coefficient table.
template <int NT, int K1, bool ORTHO, class SH>
__device__ __forceinline__ void b2_ang_force_pairs(
  const B2NepView& P, const int4* __restrict__ p0, const double* __restrict__ pz, const B2Box& box,
  int i, const B2Rec& a1, const float4* w, const float4* ctab_s, int* __restrict__ arev)
{
  constexpr int KQ = (K1 + 3) / 4;
  const unsigned N = (unsigned)P.n;
  const int na1 = SH::na1(P);
  const B2GeoR geo = b2_geo_pinned(box);
  const int t1 = a1.t;
  float rcv[NT], rciv[NT];
  b2_ang_cutoffs<NT>(P, t1, rcv, rciv);
  const float4* crow[NT];
#pragma unroll
  for (int t = 0; t < NT; ++t)
    crow[t] = ctab_s + (t1 * P.nt + (t < P.nt ? t : 0)) * na1 * KQ;
  const int* __restrict__ list = P.nl_a;
  const int* __restrict__ cnt = P.nn_a;
  const int nn = cnt[i];
  float4* __restrict__ f4 = reinterpret_cast<float4*>(P.f12);
  // list entries two neighbours ahead; position and list length of the neighbour one ahead
  int e1 = nn > 1 ? __ldg(list + N + i) : i;
  int en = nn > 0 ? __ldg(list + i) : i;
  B2Rec rn = b2_rec_load_tagged(p0, pz, en);
  int cn = __ldg(&cnt[en & B2_TAG_MASK]);
  for (int m = 0; m < nn; ++m) {
    const B2Rec a2 = rn;
    const int j = en & B2_TAG_MASK, cj = cn;
    en = e1;
    rn = b2_rec_load_tagged(p0, pz, en);
    cn = __ldg(&cnt[en & B2_TAG_MASK]);
    e1 = (m + 2 < nn) ? __ldg(list + (unsigned)(m + 2) * N + i) : i;
    // slot of i in j's list: the number of j's neighbours below i (the list is a set); -> 0 when i is
    // missing, as the binary search of b2_reduce_angular_sum.  Independent loads, issued before the
    // pair arithmetic that hides them.
    int below = 0, hit = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int v = q < cj ? (__ldg(list + (unsigned)q * N + j) & B2_TAG_MASK) : INT_MAX;
      below += v < i ? 1 : 0;
      hit |= v == i ? 1 : 0;
    }
    for (int q = 8; q < cj; ++q) {
      const int v = __ldg(list + (unsigned)q * N + j) & B2_TAG_MASK;
      below += v < i ? 1 : 0;
      hit |= v == i ? 1 : 0;
    }
    float x12, y12, z12;
    b2_rec_r12<ORTHO>(geo, box, a1, a2, x12, y12, z12);
    const float d = sqrtf(b2_d2(x12, y12, z12));
    const float dinv = 1.0f / d;
    const bool ty = NT > 1 && a2.t != 0;
    float fn[K1], fnp[K1];
    b2_basis_d<K1, true>(d, ty ? rcv[NT - 1] : rcv[0], ty ? rciv[NT - 1] : rciv[0], fn, fnp);
    float W[B2_NABC], Wp[B2_NABC];
#pragma unroll
    for (int abc = 0; abc < B2_NABC; ++abc) {
      W[abc] = 0.0f;
      Wp[abc] = 0.0f;
    }
    const float4* c4 = ty ? crow[NT - 1] : crow[0];
    b2_channel_loop<SH::fixed>(na1, 1, [&](int n) {
      float ck[KQ * 4];
#pragma unroll
      for (int q = 0; q < KQ; ++q) {
        const float4 v = c4[n * KQ + q];
        ck[4 * q] = v.x;
        ck[4 * q + 1] = v.y;
        ck[4 * q + 2] = v.z;
        ck[4 * q + 3] = v.w;
      }
      float g = 0.0f, gp = 0.0f;
#pragma unroll
      for (int k = 0; k < K1; ++k) {
        g = fmaf(fn[k], ck[k], g);
        gp = fmaf(fnp[k], ck[k], gp);
      }
      const float4* wn = w + n * B2_ABC4;
#pragma unroll
      for (int q = 0; q < B2_ABC4; ++q) {
        const float4 v = wn[q];
        const float wq[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          W[4 * q + r] = fmaf(g, wq[r], W[4 * q + r]);
          Wp[4 * q + r] = fmaf(gp, wq[r], Wp[4 * q + r]);
        }
      }
    });
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
    const unsigned slot = (unsigned)m * N + i;
    f4[slot] = make_float4(fmaf(rad, xh, gx * dinv), fmaf(rad, yh, gy * dinv), fmaf(rad, zh, gz * dinv), 0.0f);
    arev[slot] = hit ? below : 0;
  }
}

template <int NT, int K1, bool ORTHO>
__global__ void __launch_bounds__(128, 3) k_force_angular2(
  const B2NepView P, const int4* __restrict__ p0, const int4* __restrict__ p1,
  const double* __restrict__ pz, const B2Box box, int* __restrict__ arev)
{
  static_assert(NT == 1 || NT == 2, "few-type path");
  constexpr int KQ = (K1 + 3) / 4;
  extern __shared__ float4 fa_smem[];
  const int na1 = P.na1;
  const int WS4 = b2_ang_ws4(na1);
  float4* const ctab_s = fa_smem + blockDim.x * WS4;
  b2_stage_ctab(P, ctab_s, KQ);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n)
    return;
  const unsigned N = (unsigned)P.n;
  float4* const w = fa_smem + threadIdx.x * WS4;
  // dU/dq of this atom: tile-major copy written by k_mlp_tc (component d at fbase + (d/4)*512 + d%4),
  // or the SoA columns FpA[(d - nr1)*N + i] of the SIMT layer
  const float* fbase = P.fpt ? P.fpt + b2_tile_offset(P.DKT, P.tile_slot[i], 0) : P.FpA + i;
  auto FpAt = [&](int da) -> float { // da = index inside the angular part
    if (P.fpt) {
      const int d = P.nr1 + da;
      return fbase[(size_t)(d >> 2) * 512 + (d & 3)];
    }
    return fbase[(size_t)da * N];
  };
  // ---- weights ----
  const float4* __restrict__ sf4 = reinterpret_cast<const float4*>(P.sfx);
  // the sums and dU/dq of NB channels are fetched together before any of them is used, so a warp waits
  // for one memory latency per NB channels instead of one per channel (H100, 400 W, 1 M-atom PbTe:
  // 0.42 ms with NB = 3 against 0.44 with NB = 1 and NB = 5; NB = 5 needs 168 registers and spills)
  constexpr int NB = 3;
  for (int n0 = 0; n0 < na1; n0 += NB) {
    float4 sv[NB][B2_ABC4];
    float Fv[NB][6];
#pragma unroll
    for (int c = 0; c < NB; ++c) {
      const int n = n0 + c;
      if (n < na1) {
#pragma unroll
        for (int g = 0; g < B2_ABC4; ++g)
          sv[c][g] = sf4[(size_t)(n * B2_ABC4 + g) * N + i];
#pragma unroll
        for (int L = 0; L < 4; ++L)
          Fv[c][L] = FpAt(L * na1 + n);
        Fv[c][4] = P.has222 ? FpAt(4 * na1 + n) : 0.0f;
        Fv[c][5] = P.has1111 ? FpAt((4 + (P.has222 ? 1 : 0)) * na1 + n) : 0.0f;
      }
    }
#pragma unroll
    for (int c = 0; c < NB; ++c) {
      const int n = n0 + c;
      if (n >= na1)
        break;
      float s[B2_NABC];
#pragma unroll
      for (int g = 0; g < B2_ABC4; ++g) {
        const float4 v = sv[c][g];
        s[4 * g] = v.x;
        s[4 * g + 1] = v.y;
        s[4 * g + 2] = v.z;
        s[4 * g + 3] = v.w;
      }
      float wv[B2_NABC];
      b2_ang_weights(s, Fv[c], P.has222, P.has1111, wv);
#pragma unroll
      for (int g = 0; g < B2_ABC4; ++g)
        w[n * B2_ABC4 + g] = make_float4(wv[4 * g], wv[4 * g + 1], wv[4 * g + 2], wv[4 * g + 3]);
    }
  }
  // ---- pairs ----
  b2_ang_force_pairs<NT, K1, ORTHO, B2AngShapeRT>(P, p0, pz, box, i, b2_rec_load(p0, p1, i), w, ctab_s, arev);
}

// ---------------------------------------------------------------------------------------------
// k_angular_fused: descriptor, hidden layer, U table and angular partial forces of one sorted atom in
// one thread, for models that fit its budget (b2_fused_smem_bytes, DIMP = 32; nep_setup).  Nothing in
// the chain depends on another atom's result, so s[n][abc], dU/dq and dU/ds stay on the SM:
//   1. descriptor (b2_ang_desc_atom): s goes to the thread's shared-memory row, the angular components
//      of q to the SoA columns P.q (they stay observable, b200md_nep_export_descriptors);
//   2. hidden layer (b2_mlp_core) from the radial part of q that k_desc_radial2 wrote and the angular
//      part, weights from a shared-memory copy; site energy to acc[i];
//   3. U table rows (b2_utable_compact) from the radial part of dU/dq;
//   4. weights dU/ds (b2_ang_weights) in place over s;
//   5. pair loop (b2_ang_force_pairs): f12 and arev.
// Every step calls the body the five-kernel path calls, so the results are bit-identical to it with the
// SIMT hidden layer.  SH (B2AngShape) is the model's angular shape: with a fixed one the channel loops
// unroll, dU/dq and q are indexed with constants, and the angular components of q reach the hidden layer
// from registers instead of being read back from P.q.  B2AngShapeRT takes the shape from the model at run
// time (every other model within the budget).
// Dynamic shared memory: 128 rows of b2_ang_ws4(na1) float4s, the coefficient table, then w0 of each
// type at a stride of b2_fused_w0_stride4 float4s (odd: a warp holding both types reads the two rows
// on distinct banks), b0 and w1.
// ---------------------------------------------------------------------------------------------
__host__ __device__ constexpr int b2_fused_w0_stride4(int nneu, int dimp) { return (nneu * dimp / 4) | 1; }

#ifdef B2_FUSED_STOP
// Diagnostic builds only (build_lib(variant=..., defs=["B2_FUSED_STOP=k"])): k_angular_fused returns after
// step k (1 descriptor, 2 hidden layer, 3 U table, 4 weights) so that the stage profiler times the steps
// before it.  f12 and arev of the atom's pairs are zeroed, so k_force_final2 reads valid slots; the forces
// are then wrong, which is why no default build contains this.
#define B2_FUSED_MAYBE_STOP(k, ...)                                           \
  if (B2_FUSED_STOP == (k)) {                                                 \
    __VA_ARGS__;                                                              \
    for (int m = 0; m < P.nn_a[i]; ++m) {                                     \
      reinterpret_cast<float4*>(P.f12)[(unsigned)m * N + i] = make_float4(0.f, 0.f, 0.f, 0.f); \
      arev[(unsigned)m * N + i] = 0;                                          \
    }                                                                         \
    return;                                                                   \
  }
#else
#define B2_FUSED_MAYBE_STOP(k, ...)
#endif

__host__ __device__ constexpr size_t b2_fused_smem_bytes(int nt, int na1, int k1a, int nneu, int dimp)
{
  return (size_t)128 * b2_ang_ws4(na1) * 16 + (size_t)nt * nt * na1 * ((k1a + 3) / 4) * 16 +
         (size_t)nt * b2_fused_w0_stride4(nneu, dimp) * 16 + (size_t)2 * nt * nneu * 4;
}

template <int NT, int K1, int DIMP, bool ORTHO, class SH>
__global__ void __launch_bounds__(128, 3) k_angular_fused(
  const B2NepView P, const int4* __restrict__ p0, const int4* __restrict__ p1,
  const double* __restrict__ pz, const B2Box box, int* __restrict__ arev)
{
  static_assert(NT == 1 || NT == 2, "few-type path");
  constexpr int KQ = (K1 + 3) / 4;
  extern __shared__ float4 af_smem[];
  const int na1 = SH::na1(P), nr1 = SH::nr1(P), nneu = P.nneu;
  const int WS4 = b2_ang_ws4(na1);
  float4* const ctab_s = af_smem + blockDim.x * WS4;
  float4* const w0_s = ctab_s + P.nt * P.nt * na1 * KQ;
  const int wst4 = b2_fused_w0_stride4(nneu, DIMP);
  float* const b0_s = reinterpret_cast<float*>(w0_s + P.nt * wst4);
  float* const w1_s = b0_s + P.nt * nneu;
  b2_stage_ctab(P, ctab_s, KQ);
  {
    const int row4 = nneu * DIMP / 4;
    const float4* src = reinterpret_cast<const float4*>(P.w0p);
    for (int e = threadIdx.x; e < P.nt * row4; e += blockDim.x) {
      const int t = e / row4;
      w0_s[t * wst4 + (e - t * row4)] = __ldg(&src[e]);
    }
    for (int e = threadIdx.x; e < P.nt * nneu; e += blockDim.x) {
      b0_s[e] = __ldg(&P.b0[e]);
      w1_s[e] = __ldg(&P.w1[e]);
    }
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n)
    return;
  const unsigned N = (unsigned)P.n;
  float4* const row = af_smem + threadIdx.x * WS4;
  const B2Rec a1 = b2_rec_load(p0, p1, i);
  // 1. descriptor; with a fixed shape the angular components of q also stay in q[] for step 2
  float q[DIMP];
  b2_ang_desc_atom<NT, K1, 3, ORTHO, SH>(
    P, p0, pz, box, i, a1, ctab_s,
    [&](int k, float v) {
      P.q[(size_t)k * N + i] = v;
      if constexpr (SH::fixed)
        q[k] = v;
    },
    [&](int g, float4 v) { row[g] = v; });
  B2_FUSED_MAYBE_STOP(1, );
  // 2. hidden layer
  const int t = a1.t;
  float fl[DIMP]; // dU/dq
  {
    float Fp[DIMP];
#pragma unroll
    for (int d = 0; d < DIMP; ++d) {
      if (d < SH::dim(P))
        q[d] = (SH::fixed && d >= nr1 ? q[d] : P.q[(size_t)d * N + i]) * __ldg(&P.q_scaler[d]);
      else
        q[d] = 0.0f;
    }
    // paired neurons only on a fixed shape: the run-time-shape instance measured slower with them
    const float F = b2_mlp_core<DIMP, false, SH::fixed>(q, w0_s + t * wst4, b0_s + t * nneu,
                                                        w1_s + t * nneu, nneu, __ldg(&P.bias[t]),
                                                        P.q_scaler, Fp);
    P.acc[i] = (double)F;
#pragma unroll
    for (int d = 0; d < DIMP; ++d)
      fl[d] = Fp[d];
  }
  B2_FUSED_MAYBE_STOP(2, for (int d = 0; d < DIMP; ++d) asm volatile("" ::"f"(fl[d])));
  // 3. U table
  auto fr = [&](int n) { return fl[n]; };
  switch (P.K1R) {
    case 9: b2_utable_compact<9, SH::nr1_const>(P, i, t, fr); break;
    case 13: b2_utable_compact<13, SH::nr1_const>(P, i, t, fr); break;
    default: b2_utable_compact<17, SH::nr1_const>(P, i, t, fr); break;
  }
  B2_FUSED_MAYBE_STOP(3, for (int d = 0; d < DIMP; ++d) asm volatile("" ::"f"(fl[d])));
  // 4. weights over s
  const float* fa = fl + nr1;
  const int h222 = SH::has222(P), h1111 = SH::has1111(P);
  b2_channel_loop<SH::fixed>(na1, 1, [&](int n) {
    float s[B2_NABC];
#pragma unroll
    for (int g = 0; g < B2_ABC4; ++g) {
      const float4 v = row[n * B2_ABC4 + g];
      s[4 * g] = v.x;
      s[4 * g + 1] = v.y;
      s[4 * g + 2] = v.z;
      s[4 * g + 3] = v.w;
    }
    float F6[6];
#pragma unroll
    for (int L = 0; L < 4; ++L)
      F6[L] = fa[L * na1 + n];
    F6[4] = h222 ? fa[4 * na1 + n] : 0.0f;
    F6[5] = h1111 ? fa[(4 + (h222 ? 1 : 0)) * na1 + n] : 0.0f;
    float wv[B2_NABC];
    b2_ang_weights(s, F6, h222, h1111, wv);
#pragma unroll
    for (int g = 0; g < B2_ABC4; ++g)
      row[n * B2_ABC4 + g] = make_float4(wv[4 * g], wv[4 * g + 1], wv[4 * g + 2], wv[4 * g + 3]);
  });
  B2_FUSED_MAYBE_STOP(4, );
  // 5. pairs
  b2_ang_force_pairs<NT, K1, ORTHO, SH>(P, p0, pz, box, i, a1, row, ctab_s, arev);
}

} // namespace b2

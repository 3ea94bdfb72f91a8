// b2_nep.cu -- NEP potential of libb200md: kernels (thin wrappers over the bodies in b2_nep.cuh),
// template dispatch, device tables, and the C-ABI entry points b200md_nep_*.
#include "../../include/b200md.h"
#include "b2_host.h"
#include "b2_neighbor_host.h"
#include "b2_nep.cuh"
#include "b2_nep_tc.cuh"
#include "b2_nep_radial.cuh"
#include "b2_nep_angular.cuh"
#include "b2_nep_model.h"
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace b2 {

namespace {

constexpr int BLK = 128;
constexpr int MLP_BLK = 256;
// k_angular_fused runs for models with a zero-padded descriptor of 32 (the width whose instances ptxas
// compiles without spills at three blocks per SM; at 48 every instance spills) and where two of its
// blocks fit an SM's 228 KB of shared memory (1 KB reserved per block)
constexpr int FUSED_DIMP = 32;
constexpr size_t FUSED_MAX_SMEM = 113 * 1024;
// Angular shapes k_angular_fused is compiled for (B2AngShape): NEP4's default n_max = 4 4 with l_max = 4 2 0
// (dim 30) and 4 0 0 (dim 25).  Each shape adds 12 instances (NT x K1 x ORTHO, about 15 s of build time);
// every other shape within the budget runs the run-time-shape instance.
enum { FUSED_SHAPE_NONE, FUSED_SHAPE_RT, FUSED_SHAPE_4B, FUSED_SHAPE_3B };

int fused_shape_of(const NepModel& m)
{
  if (m.nr1 == 5 && m.na1 == 5 && !m.has1111)
    return m.has222 ? FUSED_SHAPE_4B : FUSED_SHAPE_3B;
  return FUSED_SHAPE_RT;
}

__global__ void __launch_bounds__(BLK) k_split(B2NepView P, B2Box box)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_split(i, P, box);
}

template <int NT, int K1, bool SPLIT>
__global__ void __launch_bounds__(BLK) k_desc_radial(B2NepView P, B2Box box)
{
  extern __shared__ float dyn_smem[];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_desc_radial<NT, K1, SPLIT>(i, P, box, dyn_smem, blockDim.x, threadIdx.x);
}

// lane-team kernels: B2_TEAM adjacent lanes per atom, BLK / B2_TEAM atoms per block
template <int NT, int K1>
__global__ void __launch_bounds__(BLK) k_team_desc_radial(B2NepView P, B2Box box)
{
  const int i = blockIdx.x * (BLK / B2_TEAM) + threadIdx.x / B2_TEAM;
  if (i < P.n)
    b2_team_desc_radial<NT, K1>(i, threadIdx.x % B2_TEAM, P, box);
}

template <int NT, int K1>
__global__ void __launch_bounds__(BLK)
  k_team_force_final(B2NepView P, B2Box box, double* pe, double* force, double* virial)
{
  const int i = blockIdx.x * (BLK / B2_TEAM) + threadIdx.x / B2_TEAM;
  if (i < P.n)
    b2_team_force_final<NT, K1>(i, threadIdx.x % B2_TEAM, P, box, pe, force, virial);
}

template <int K1, int NCH>
__global__ void __launch_bounds__(BLK, 3) k_desc_angular(B2NepView P, B2Box box, int stage_rs4)
{
  // stage_rs4 > 0: every block first copies the padded angular coefficient table into shared memory,
  // rows re-strided to stage_rs4 (odd) float4s.  With many types each lane reads a different
  // (t1, t2) row: from shared memory that costs bank conflicts only, from L1 one wavefront per lane.
  extern __shared__ float4 ctab_s[];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  constexpr int KQ = (K1 + 3) / 4;
  if (stage_rs4 > 0) {
    const int row4 = P.na1 * KQ, tot = P.nt * P.nt * row4;
    for (int e = threadIdx.x; e < tot; e += blockDim.x) {
      const int r = e / row4;
      ctab_s[r * stage_rs4 + (e - r * row4)] = P.c_a4[e];
    }
    __syncthreads();
    if (i < P.n)
      b2_body_desc_angular<K1, NCH>(i, P, box, ctab_s, stage_rs4);
  } else if (i < P.n) {
    b2_body_desc_angular<K1, NCH>(i, P, box, P.c_a4, P.na1 * KQ);
  }
}

// One tile of MLP_BLK consecutive (cell-sorted) atoms per block.  The tile is counting-sorted by
// type in shared memory so that the lanes of a warp read the same weight rows (broadcast loads).
// STAGE: the weights of all types are first copied to shared memory (models where they fit).
template <int DIMP, bool STAGE>
__global__ void __launch_bounds__(MLP_BLK) k_mlp(B2NepView P)
{
  extern __shared__ float4 mlp_smem4[];
  __shared__ int order[MLP_BLK];
  __shared__ int cnt[B2_MAX_TYPES + 1];
  const int tid = threadIdx.x;
  const int base = blockIdx.x * MLP_BLK;
  const int i = base + tid;
  const float* w0 = P.w0p;
  const float* b0 = P.b0;
  const float* w1 = P.w1;
  if (STAGE) {
    float* sm = reinterpret_cast<float*>(mlp_smem4);
    const int nw0 = P.nt * P.nneu * DIMP, nb = P.nt * P.nneu;
    const float4* src4 = reinterpret_cast<const float4*>(P.w0p);
    for (int k = tid; k < nw0 / 4; k += MLP_BLK)
      mlp_smem4[k] = __ldg(&src4[k]);
    for (int k = tid; k < nb; k += MLP_BLK) {
      sm[nw0 + k] = __ldg(&P.b0[k]);
      sm[nw0 + nb + k] = __ldg(&P.w1[k]);
    }
    w0 = sm;
    b0 = sm + nw0;
    w1 = sm + nw0 + nb;
  }
  int mine = i;
  int t = 0, rank = 0;
  if (P.nt > 1) {
    if (tid <= B2_MAX_TYPES)
      cnt[tid] = 0;
    __syncthreads();
    if (i < P.n) {
      t = P.atoms[i].type;
      rank = atomicAdd(&cnt[t], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int run = 0;
      for (int k = 0; k < P.nt; ++k) {
        const int c = cnt[k];
        cnt[k] = run;
        run += c;
      }
    }
    __syncthreads();
    if (i < P.n)
      order[cnt[t] + rank] = i;
  }
  __syncthreads();
  if (P.nt > 1 && i < P.n)
    mine = order[tid];
  if (i < P.n)
    b2_body_mlp<DIMP, !STAGE>(mine, P, w0, b0, w1);
}

// AoS rows (thread-per-atom consumers gather one row per neighbour): each thread contracts its
// own row, the block transposes it through shared memory so that the global stores are runs of
// consecutive floats instead of one 4-byte store per thread per element (same arithmetic as
// b2_body_utable, which tests/emu runs).
template <int K1>
__global__ void __launch_bounds__(BLK) k_utable(B2NepView P)
{
  constexpr int KP = (K1 + 3) / 4 * 4;
  __shared__ float tile[BLK][KP + 1];
  const int base = blockIdx.x * BLK;
  const int i = base + threadIdx.x;
  if (P.u_planes == 2) { // compact planes of the few-type kernels (b2_nep_radial.cuh)
    if (i < P.n)
      b2_utable_compact<K1>(P, i, P.atoms[i].type, [&](int n) { return P.FpR[(size_t)n * P.n + i]; });
    return;
  }
  if (P.u_planes) {
    if (i < P.n)
      b2_body_utable_planes<K1>(i, P);
    return;
  }
  const int t = i < P.n ? P.atoms[i].type : 0;
  float fp[8]; // nr1 <= n_max_radial + 1; larger models take the loop below in two halves
  const int nr1 = P.nr1;
  for (int t2 = 0; t2 < P.nt; ++t2) {
    float u[KP];
#pragma unroll
    for (int k = 0; k < KP; ++k)
      u[k] = 0.0f;
    if (i < P.n) {
      const float* c = P.c_r + (size_t)(t * P.nt + t2) * nr1 * K1;
      for (int n0 = 0; n0 < nr1; n0 += 8) {
#pragma unroll
        for (int m = 0; m < 8; ++m)
          fp[m] = (n0 + m < nr1) ? P.FpR[(size_t)(n0 + m) * P.n + i] : 0.0f;
#pragma unroll
        for (int m = 0; m < 8; ++m) {
          if (n0 + m < nr1) {
#pragma unroll
            for (int k = 0; k < K1; ++k)
              u[k] = fmaf(fp[m], __ldg(&c[(n0 + m) * K1 + k]), u[k]);
          }
        }
      }
    }
    __syncthreads(); // previous t2's tile has been written out
#pragma unroll
    for (int k = 0; k < KP; ++k)
      tile[threadIdx.x][k] = u[k];
    __syncthreads();
    for (int e = threadIdx.x; e < BLK * KP; e += BLK) {
      const int r = e / KP, k = e - r * KP;
      if (base + r < P.n)
        P.U[(size_t)(base + r) * P.UST + t2 * KP + k] = tile[r][k];
    }
  }
}

// MINB: resident blocks per SM the register allocation is tuned for (latency hiding vs spills)
template <int NT, int K1, int MINB, int DEPTH>
__global__ void __launch_bounds__(BLK, MINB)
  k_force_final(B2NepView P, B2Box box, double* pe, double* force, double* virial)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P.n)
    b2_body_force_final<NT, K1, DEPTH>(i, P, box, pe, force, virial);
}

template <int K1, int NTHR>
__global__ void __launch_bounds__(NTHR) k_force_angular(B2NepView P, B2Box box)
{
  // (a shared-memory copy of the coefficient table as in k_desc_angular needs 256-thread blocks to fit
  // next to the weights; it gained nothing on UNEP-v1 and the second code path slowed the few-type
  // case -- not kept)
  extern __shared__ float dyn_smem[];
  const int i = blockIdx.x * NTHR + threadIdx.x;
  if (i < P.n)
    b2_body_force_angular<K1, NTHR>(i, P, box, dyn_smem, threadIdx.x, P.c_a4, P.na1 * ((K1 + 3) / 4));
}

// parity hooks ---------------------------------------------------------------------------------
__global__ void k_export_list(
  int n, int n_cell, const int* perm, const int* nn, const int* nl, size_t si, size_t sk,
  int mn_out, int* NN_out, int* NL_out, int* flags, int mask)
{
  // n_cell < n: a supercell was evaluated; report the first replica with neighbour indices folded
  // back into the caller's cell (an atom then appears once per periodic image, like in the
  // reference's small-box lists, nep_small_box.cuh:56-150)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int a = perm[i];
  if (a >= n_cell)
    return;
  int cnt = nn[i];
  if (cnt > mn_out) {
    atomicOr(&flags[1], (int)B2_ERR_RADIAL_OVERFLOW);
    cnt = mn_out;
  }
  int* row = NL_out + (size_t)a * mn_out;
  for (int k = 0; k < cnt; ++k) { // insertion sort into ascending caller index
    const int v = perm[nl[(size_t)i * si + (size_t)k * sk] & mask] % n_cell;
    int q = k - 1;
    while (q >= 0 && row[q] > v) {
      row[q + 1] = row[q];
      --q;
    }
    row[q + 1] = v;
  }
  NN_out[a] = cnt;
}

__global__ void k_export_q(B2NepView P, int n_cell, float* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n)
    return;
  const int a = P.perm[i];
  if (a >= n_cell)
    return;
  for (int d = 0; d < P.dim; ++d)
    out[(size_t)d * n_cell + a] = *b2_q_ptr(P, i, P.qt ? P.tile_slot[i] : 0, d) * P.q_scaler[d];
}

__global__ void k_export_tile_slot(int n, int n_cell, const int* perm, const int* tile_slot, int* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  const int a = perm[i];
  if (a < n_cell)
    out[a] = tile_slot[i];
}

// the hidden layer's output in one layout whatever the storage: fp[d*n_cell + a] (dU/dq times q_scaler)
// and u[(t2*K1R + k)*n_cell + a] (the U table); either may be null
__global__ void k_export_mlp(B2NepView P, int n_cell, float* fp, float* u)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P.n)
    return;
  const int a = P.perm[i];
  if (a >= n_cell)
    return;
  const size_t N = (size_t)P.n, M = (size_t)n_cell;
  if (fp) {
    for (int d = 0; d < P.dim; ++d) {
      float v;
      if (P.fpt)
        v = P.fpt[b2_tile_offset(P.DKT, P.tile_slot[i], d)];
      else
        v = d < P.nr1 ? P.FpR[(size_t)d * N + i] : P.FpA[(size_t)(d - P.nr1) * N + i];
      fp[(size_t)d * M + a] = v;
    }
  }
  if (u) {
    const int KQ = P.KP / 4 - 1;
    for (int t2 = 0; t2 < P.nt; ++t2) {
      for (int k = 0; k < P.K1R; ++k) {
        float v;
        if (P.u_planes == 2) // compact planes (b2_nep_radial.cuh): k < K1R - 1 in float4 planes, the last alone
          v = k < 4 * KQ ? P.U[((size_t)(t2 * KQ + k / 4) * N + i) * 4 + (k & 3)]
                         : P.U[(size_t)P.nt * KQ * 4 * N + (size_t)t2 * N + i];
        else if (P.u_planes == 1) // float4 planes [(t2*KP4 + q)*n + i]
          v = P.U[((size_t)((t2 * P.KP + k) / 4) * N + i) * 4 + (k & 3)];
        else // AoS rows of UST floats
          v = P.U[(size_t)i * P.UST + t2 * P.KP + k];
        u[((size_t)t2 * P.K1R + k) * M + a] = v;
      }
    }
  }
}

// ---- small periodic boxes: evaluate a supercell, keep the first replica -----------------------
// replica r = (a*ry + b)*rz + c of atom i sits at index r*n + i, shifted by a*A + b*B + c*C
__global__ void __launch_bounds__(BLK) k_replicate(
  int n, int rx, int ry, int rz, B2Box box, const int* __restrict__ type,
  const double* __restrict__ pos, int* type_out, double* pos_out)
{
  const size_t nR = (size_t)n * rx * ry * rz;
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nR)
    return;
  const int r = (int)(e / n), i = (int)(e - (size_t)r * n);
  const int c = r % rz, b = (r / rz) % ry, a = r / (rz * ry);
  type_out[e] = type[i];
  // lattice vectors are the columns of h (box.cuh:18-35)
  pos_out[e] = pos[i] + a * box.h[0] + b * box.h[1] + c * box.h[2];
  pos_out[nR + e] = pos[(size_t)n + i] + a * box.h[3] + b * box.h[4] + c * box.h[5];
  pos_out[2 * nR + e] = pos[2 * (size_t)n + i] + a * box.h[6] + b * box.h[7] + c * box.h[8];
}

// outputs of the first replica are the outputs of the original cell (+= convention, or a store with
// overwrite); n_own > 0: atoms from n_own on keep what the caller's arrays hold
__global__ void __launch_bounds__(BLK) k_fold_replica(
  int n, size_t nR, const double* __restrict__ acc, double* pe, double* force, double* virial,
  int overwrite, int n_own)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (n_own > 0 && i >= n_own))
    return;
  pe[i] = (overwrite ? 0.0 : pe[i]) + acc[i];
  for (int k = 0; k < 3; ++k)
    force[(size_t)k * n + i] = (overwrite ? 0.0 : force[(size_t)k * n + i]) + acc[nR + (size_t)k * nR + i];
  for (int k = 0; k < 9; ++k)
    virial[(size_t)k * n + i] =
      (overwrite ? 0.0 : virial[(size_t)k * n + i]) + acc[4 * nR + (size_t)k * nR + i];
}

template <typename T>
int upload(DevBuf<T>& buf, const std::vector<T>& host)
{
  const size_t count = host.empty() ? 1 : host.size();
  B2_CUDA(buf.reserve(count));
  if (!host.empty())
    B2_CUDA(cudaMemcpy(buf.p, host.data(), sizeof(T) * host.size(), cudaMemcpyHostToDevice));
  return B200MD_OK;
}

} // namespace

} // namespace b2

using namespace b2;

struct b200md_nep {
  NepModel model;
  Neighbor nb;
  int n = 0;
  DevBuf<float> rc_r, rcinv_r, rc2_r, rc_a, rcinv_a, rc2_a, c_r, c_a, c_a4, c_r4, w0p, b0, w1, bias, q_scaler,
    zbl_para, cov_radius;
  DevBuf<int> zbl_z;
  DevBuf<int> nn_r, nl_r, nn_a, nl_a;
  DevBuf<int> aslot, nla_rs; // see B2NepView::aslot
  DevBuf<int> arev;          // few-type path: slot of i in the angular list of its m-th angular neighbour
  bool rev_slot = false;
  DevBuf<float> q, sfx, FpR, FpA, U, f12;
  DevBuf<double> acc;
  DevBuf<float> tc_img, qt, fpt; // tile-major q / dU/dq for k_mlp_tc (B2NepView::qt)
  int num_sms = 132;
  int tc_ctas_cap = 0;  // B200MD_NEP_TC_CTAS: at most this many CTAs of k_mlp_tc (0: as many as fit)
  int tc_ctas_last = 0; // CTAs of the last k_mlp_tc launch (0: the last compute did not run it)
  int variant = 0;        // B200MD_NEP_VARIANT: kernel tuning variants for A/B measurements
  bool fuse_split = false; // many-type path: neighbour split inside the radial descriptor pass
  bool use_tc = false; // hidden layer on the tensor cores (k_mlp_tc) instead of k_mlp
  bool ang_fused = false; // k_angular_fused instead of k_desc_angular2 + hidden layer + k_force_angular2
  int fused_shape = 0;     // its instance: FUSED_SHAPE_* (b200md_nep_info 10)
  size_t fused_smem = 0;  // its dynamic shared memory per block
  bool slot_map = false;  // k_force_final2: thread per tile slot (type-pure warps); measured slower
                          // (H100, 1 M-atom PbTe: 1.26 vs 1.02 ms), B200MD_NEP_SLOTMAP=1 for A/B runs
  bool rad_direct = false; // many types: contract every pair on the spot (k_desc_radial<-1,...>), see nep_setup
  bool rad_reg = false;   // 3..16 types: radial accumulators in registers (k_desc_radial<4|8|16,...>); slower
                          // than the shared-memory accumulators on UNEP-v1, B200MD_NEP_RADREG=1
  int rad_nt = 0;         // 3+ types: NT of the k_desc_radial instance (-1, 0, 4, 8, 16), see nep_setup
  bool ang_cstage = true; // k_desc_angular: coefficient table staged in shared memory
  bool radial_v2 = false; // few-type radial passes of b2_nep_radial.cuh (planes, branch-free loop)
  bool sched = false;     // their warps follow Neighbor::seg_order (B200MD_NEP_SCHED=0: identity, A/B runs)
  // small periodic boxes (SURVEY 8f rank 1): supercell replication, see b200md_nep_compute
  DevBuf<int> rep_type;
  DevBuf<double> rep_pos, rep_out;
  int rep_n = 0; // atoms of the caller's cell while a supercell is being evaluated (else 0)
  // staging for the host-buffer entry point
  DevBuf<int> h_type;
  DevBuf<double> h_pos, h_out;
  // the caller's set_accumulate / set_owned / set_active_region requests: kept here because
  // nep_setup rebuilds the view (the supercell path grows the handle), copied into it by every compute
  int overwrite = 0, n_own = 0, use_active = 0;
  double act_lo[3] = {0, 0, 0}, act_hi[3] = {0, 0, 0};
  B2NepView view;
  StageProfiler prof;
  int ang_block = BLK;
  size_t ang_smem = 0, rad_smem = 0;
};

namespace {

// thread per atom; NT = 0: per-type accumulators in shared memory (many types)
template <int NT, int K1, bool SPLIT>
int launch_desc_radial(const b200md_nep* p, const B2Box& box, cudaStream_t st)
{
  auto kern = k_desc_radial<NT, K1, SPLIT>;
  if (NT == 0 && p->rad_smem > 48 * 1024)
    B2_CUDA(cudaFuncSetAttribute(
      kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->rad_smem));
  kern<<<grid_for(p->n, BLK), BLK, NT == 0 ? p->rad_smem : 0, st>>>(p->view, box);
  B2_LAUNCHED();
  return B200MD_OK;
}

template <int K1>
int dispatch_desc_radial(const b200md_nep* p, const B2Box& box, cudaStream_t st)
{
  const int team_grid = grid_for(p->n, BLK / B2_TEAM);
  if (p->view.team && p->model.nt == 1) {
    k_team_desc_radial<1, K1><<<team_grid, BLK, 0, st>>>(p->view, box);
  } else if (p->view.team) {
    k_team_desc_radial<2, K1><<<team_grid, BLK, 0, st>>>(p->view, box);
  } else if (p->radial_v2) {
    const B2NepView& P = p->view;
    B2RadialDescArgs A;
    A.n = P.n; A.nt = P.nt; A.nr1 = P.nr1; A.mn_r = P.mn_r; A.mn_a = P.mn_a;
    A.plane0 = p->nb.plane0.p; A.plane1 = p->nb.plane1.p; A.planez = p->nb.planez.p;
    A.nn_skin = P.nn_skin; A.nl_skin = P.nl_skin; A.seg_order = P.seg_order;
    A.nn_r = P.nn_r; A.nl_r = P.nl_r; A.nn_a = P.nn_a; A.nl_a = P.nl_a;
    A.q = P.q; A.flags = P.flags;
    A.tile_slot = P.tile_slot; A.qt = P.qt; A.DKT = P.DKT;
    A.rc_r = P.rc_r; A.rcinv_r = P.rcinv_r; A.rc2_r = P.rc2_r; A.rc2_a = P.rc2_a; A.c_r = P.c_r;
    A.use_active = P.use_active;
    for (int d = 0; d < 3; ++d) {
      A.act_lo[d] = P.act_lo[d];
      A.act_hi[d] = P.act_hi[d];
    }
    const int g = grid_for(p->n, BLK);
    if (p->model.nt == 1 && box.ortho)
      k_desc_radial2<1, K1, true><<<g, BLK, 0, st>>>(A, box);
    else if (p->model.nt == 1)
      k_desc_radial2<1, K1, false><<<g, BLK, 0, st>>>(A, box);
    else if (box.ortho)
      k_desc_radial2<2, K1, true><<<g, BLK, 0, st>>>(A, box);
    else
      k_desc_radial2<2, K1, false><<<g, BLK, 0, st>>>(A, box);
  } else if (p->model.nt == 1) {
    return launch_desc_radial<1, K1, true>(p, box, st);
  } else if (p->model.nt == 2) {
    return launch_desc_radial<2, K1, true>(p, box, st);
  } else {
    // 3+ types: the instance nep_setup chose (p->rad_nt)
    if (!p->fuse_split) {
      k_split<<<grid_for(p->n, BLK), BLK, 0, st>>>(p->view, box);
      B2_LAUNCHED();
    }
#define B2_DR(NT_)                                                 \
  return p->fuse_split ? launch_desc_radial<NT_, K1, true>(p, box, st) \
                       : launch_desc_radial<NT_, K1, false>(p, box, st)
    if (p->rad_nt == -1)
      B2_DR(-1);
    if (p->rad_nt == 4)
      B2_DR(4);
    if constexpr (8 * K1 <= 160) {
      if (p->rad_nt == 8)
        B2_DR(8);
    }
    if constexpr (16 * K1 <= 160) {
      if (p->rad_nt == 16)
        B2_DR(16);
    }
    B2_DR(0);
#undef B2_DR
  }
  B2_LAUNCHED();
  return B200MD_OK;
}

template <int NT, int K1>
int launch_force_final(
  const b200md_nep* p, const B2Box& box, cudaStream_t st, double* pe, double* f, double* v)
{
  const int g = grid_for(p->n, BLK);
  switch (p->variant) {
    // B200MD_NEP_VARIANT: register / occupancy variants for A/B runs
    case 1: k_force_final<NT, K1, 6, 1><<<g, BLK, 0, st>>>(p->view, box, pe, f, v); break;
    case 3: k_force_final<NT, K1, 5, 1><<<g, BLK, 0, st>>>(p->view, box, pe, f, v); break;
    case 2: k_force_final<NT, K1, 4, 2><<<g, BLK, 0, st>>>(p->view, box, pe, f, v); break;
    default:
      // many types: 80 registers / 6 blocks
      if (NT == 0)
        k_force_final<NT, K1, 6, 1><<<g, BLK, 0, st>>>(p->view, box, pe, f, v);
      else
        k_force_final<NT, K1, 5, 1><<<g, BLK, 0, st>>>(p->view, box, pe, f, v);
      break;
  }
  B2_LAUNCHED();
  return B200MD_OK;
}

template <int K1>
int dispatch_force_final(
  const b200md_nep* p, const B2Box& box, cudaStream_t st, double* pe, double* f, double* v)
{
  const int team_grid = grid_for(p->n, BLK / B2_TEAM);
  if (p->view.team && p->model.nt == 1)
    k_team_force_final<1, K1><<<team_grid, BLK, 0, st>>>(p->view, box, pe, f, v);
  else if (p->view.team)
    k_team_force_final<2, K1><<<team_grid, BLK, 0, st>>>(p->view, box, pe, f, v);
  else if (p->radial_v2) {
    // one thread per tile slot when type tiles exist (type-pure warps), else per sorted atom
    B2NepView V = p->view;
    if (!p->slot_map)
      V.tile_atom = nullptr; // B200MD_NEP_SLOTMAP=0: thread per sorted atom (A/B runs)
    const int g = V.tile_atom ? p->nb.max_tiles() : grid_for(p->n, BLK);
    const int4* p0 = p->nb.plane0.p;
    const int4* p1 = p->nb.plane1.p;
    const double* pz = p->nb.planez.p;
    const int* ar = p->arev.p;
    // B200MD_NEP_VARIANT: resident blocks per SM the register allocation targets.  Measured on an
    // H100 (400 W) with 1 M-atom PbTe: 5 blocks / 96 regs 1.02 ms (default), 6 blocks / 80 regs with
    // spills 1.30 ms, 4 blocks / 128 regs (variant 2) 1.00 ms, variant 3 1.02 ms
#define B2_FF2(NT_, ORTHO_)                                                                      \
  do {                                                                                           \
    if (p->variant == 1)                                                                         \
      k_force_final2<NT_, K1, ORTHO_, 6><<<g, BLK, 0, st>>>(V, p0, p1, pz, ar, box, pe, f, v); \
    else if (p->variant == 2)                                                                    \
      k_force_final2<NT_, K1, ORTHO_, 4><<<g, BLK, 0, st>>>(V, p0, p1, pz, ar, box, pe, f, v); \
    else                                                                                         \
      k_force_final2<NT_, K1, ORTHO_, 5><<<g, BLK, 0, st>>>(V, p0, p1, pz, ar, box, pe, f, v); \
  } while (0)
    if (p->model.nt == 1 && box.ortho)
      B2_FF2(1, true);
    else if (p->model.nt == 1)
      B2_FF2(1, false);
    else if (box.ortho)
      B2_FF2(2, true);
    else
      B2_FF2(2, false);
#undef B2_FF2
  }
  else if (p->model.nt == 1)
    return launch_force_final<1, K1>(p, box, st, pe, f, v);
  else if (p->model.nt == 2)
    return launch_force_final<2, K1>(p, box, st, pe, f, v);
  else
    return launch_force_final<0, K1>(p, box, st, pe, f, v);
  B2_LAUNCHED();
  return B200MD_OK;
}

// the few-type angular kernels of b2_nep_angular.cuh (with the plane-based radial passes)
template <int NT, int K1, bool ORTHO>
int launch_angular2(const b200md_nep* p, const B2Box& box, cudaStream_t st, bool force)
{
  const int4* p0 = p->nb.plane0.p;
  const int4* p1 = p->nb.plane1.p;
  const double* pz = p->nb.planez.p;
  const size_t ctab = (size_t)p->model.nt * p->model.nt * p->model.na1 * ((K1 + 3) / 4) * sizeof(float4);
  if (!force) {
    // + the per-thread staging of the angular descriptors when they go to the tile-major copy
    const size_t qs = p->view.qt ? (size_t)p->model.dim_angular * BLK * sizeof(float) : 0;
    auto dk = k_desc_angular2<NT, K1, 3, ORTHO>;
    if (ctab + qs > 48 * 1024)
      B2_CUDA(cudaFuncSetAttribute(dk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(ctab + qs)));
    dk<<<grid_for(p->n, BLK), BLK, ctab + qs, st>>>(p->view, p0, p1, pz, box);
    B2_LAUNCHED();
    return B200MD_OK;
  }
  auto kern = k_force_angular2<NT, K1, ORTHO>;
  const size_t bytes = p->ang_smem + ctab;
  if (bytes > 48 * 1024)
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  kern<<<grid_for(p->n, p->ang_block), p->ang_block, bytes, st>>>(p->view, p0, p1, pz, box, p->arev.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

// k_desc_angular's coefficient table: float4 rows of (na1 * KQ) | 1, one per type pair
int ang_coeff_row(const b200md_nep* p) { return (p->model.na1 * ((p->model.K1A + 3) / 4)) | 1; }

size_t ang_coeff_bytes(const b200md_nep* p)
{
  return (size_t)p->model.nt * p->model.nt * ang_coeff_row(p) * sizeof(float4);
}

// shared-memory copy of the angular coefficients when three blocks of it fit an SM
// (B200MD_NEP_CSTAGE=0: read them from global memory)
bool ang_coeff_staged(const b200md_nep* p) { return p->ang_cstage && ang_coeff_bytes(p) <= 72 * 1024; }

template <int K1>
int launch_angular(const b200md_nep* p, const B2Box& box, cudaStream_t st, bool force)
{
  if (p->radial_v2) {
    if (p->model.nt == 1 && box.ortho)
      return launch_angular2<1, K1, true>(p, box, st, force);
    if (p->model.nt == 1)
      return launch_angular2<1, K1, false>(p, box, st, force);
    if (box.ortho)
      return launch_angular2<2, K1, true>(p, box, st, force);
    return launch_angular2<2, K1, false>(p, box, st, force);
  }
  if (!force) {
    {
      const int rs4 = ang_coeff_row(p);
      const size_t bytes = ang_coeff_bytes(p);
      const bool stage = ang_coeff_staged(p);
      auto kern = k_desc_angular<K1, 5>;
      if (stage && bytes > 48 * 1024)
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
      kern<<<grid_for(p->n, BLK), BLK, stage ? bytes : 0, st>>>(p->view, box, stage ? rs4 : 0);
    }
    B2_LAUNCHED();
    return B200MD_OK;
  }
  void (*kern)(B2NepView, B2Box) = k_force_angular<K1, 128>;
  if (p->ang_block == 64)
    kern = k_force_angular<K1, 64>;
  else if (p->ang_block == 32)
    kern = k_force_angular<K1, 32>;
  if (p->ang_smem > 48 * 1024)
    B2_CUDA(cudaFuncSetAttribute(
      kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->ang_smem));
  kern<<<grid_for(p->n, p->ang_block), p->ang_block, p->ang_smem, st>>>(p->view, box);
  B2_LAUNCHED();
  return B200MD_OK;
}

template <int NT, int K1, int DIMP, bool ORTHO, class SH>
int launch_fused_inst(const b200md_nep* p, const B2Box& box, cudaStream_t st)
{
  auto kern = k_angular_fused<NT, K1, DIMP, ORTHO, SH>;
  if (p->fused_smem > 48 * 1024)
    B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->fused_smem));
  kern<<<grid_for(p->n, BLK), BLK, p->fused_smem, st>>>(
    p->view, p->nb.plane0.p, p->nb.plane1.p, p->nb.planez.p, box, p->arev.p);
  B2_LAUNCHED();
  return B200MD_OK;
}

template <int K1, class SH>
int launch_fused_shape(const b200md_nep* p, const B2Box& box, cudaStream_t st)
{
  if (p->model.nt == 1)
    return box.ortho ? launch_fused_inst<1, K1, FUSED_DIMP, true, SH>(p, box, st)
                     : launch_fused_inst<1, K1, FUSED_DIMP, false, SH>(p, box, st);
  return box.ortho ? launch_fused_inst<2, K1, FUSED_DIMP, true, SH>(p, box, st)
                   : launch_fused_inst<2, K1, FUSED_DIMP, false, SH>(p, box, st);
}

// the one hidden-layer width k_angular_fused is instantiated for (FUSED_DIMP, see nep_setup), on the angular
// shape p->fused_shape (fused_shape_of)
template <int K1>
int launch_angular_fused(const b200md_nep* p, const B2Box& box, cudaStream_t st)
{
  switch (p->fused_shape) {
    case FUSED_SHAPE_4B: return launch_fused_shape<K1, B2AngShape<5, 5, true, false>>(p, box, st);
    case FUSED_SHAPE_3B: return launch_fused_shape<K1, B2AngShape<5, 5, false, false>>(p, box, st);
    default: return launch_fused_shape<K1, B2AngShapeRT>(p, box, st);
  }
}

// k_mlp's weights of every type in shared memory (STAGE = true) while they fit 96 KB
size_t mlp_weight_bytes(const b200md_nep* p)
{
  return (size_t)p->model.nt * p->model.nneu * (p->model.DIMP + 2) * sizeof(float);
}

bool mlp_weights_staged(const b200md_nep* p) { return mlp_weight_bytes(p) <= 96 * 1024; }

template <int DIMP>
int launch_mlp(const b200md_nep* p, cudaStream_t st)
{
  const size_t bytes = mlp_weight_bytes(p);
  if (mlp_weights_staged(p)) {
    auto kern = k_mlp<DIMP, true>;
    if (bytes > 48 * 1024)
      B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    kern<<<grid_for(p->n, MLP_BLK), MLP_BLK, bytes, st>>>(p->view);
  } else {
    k_mlp<DIMP, false><<<grid_for(p->n, MLP_BLK), MLP_BLK, 0, st>>>(p->view);
  }
  B2_LAUNCHED();
  return B200MD_OK;
}

#define B2_TRY(expr)          \
  do {                        \
    const int rc_ = (expr);   \
    if (rc_ != B200MD_OK)     \
      return rc_;             \
  } while (0)

// stage ids reported by b200md_nep_profile_read / b200md_nep_stage_name
enum { ST_NEIGHBOR, ST_DESC_R, ST_DESC_A, ST_MLP, ST_FORCE_A, ST_FORCE_FINAL, ST_ANG_FUSED, ST_COUNT };
const char* const STAGE_NAMES[ST_COUNT] = {
  "neighbor_update", "k_desc_radial", "k_desc_angular", "k_mlp", "k_force_angular",
  "k_force_final", "k_angular_fused"};

// descriptor pass, hidden layer (+ U table) and angular force pass as separate kernels: models that do
// not fit k_angular_fused, many types, and B200MD_NEP_MLP=simt / tc
int angular_stages(b200md_nep* p, const B2Box& box, cudaStream_t st)
{
  const int n = p->n;
  StageProfiler& pf = p->prof;
  pf.begin(st, ST_DESC_A);
  switch (p->model.K1A) {
    case 9: B2_TRY(launch_angular<9>(p, box, st, false)); break;
    case 13: B2_TRY(launch_angular<13>(p, box, st, false)); break;
    default: B2_TRY(launch_angular<17>(p, box, st, false)); break;
  }
  pf.end(st, ST_DESC_A);
  pf.begin(st, ST_MLP);
  if (p->use_tc) {
    const size_t bytes = b2_tc_smem_bytes(p->model.tc_img_floats, p->model.HN, p->model.DK, p->model.DN,
                                          p->view.N3 ? p->model.K3 : 0);
    if (bytes > 48 * 1024)
      B2_CUDA(cudaFuncSetAttribute(
        k_mlp_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    // persistent CTAs: as many as fit per SM, each walking tiles
    int per_sm = 1;
    B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_mlp_tc, 128, bytes));
    per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
    const int tiles = p->nb.max_tiles();
    int ctas = tiles < p->num_sms * per_sm ? tiles : p->num_sms * per_sm;
    if (p->tc_ctas_cap > 0 && ctas > p->tc_ctas_cap)
      ctas = p->tc_ctas_cap; // every tile is still computed by one CTA with the same arithmetic
    p->tc_ctas_last = ctas;
    k_mlp_tc<<<ctas, 128, bytes, st>>>(p->view);
    B2_LAUNCHED();
  } else
  switch (p->model.DIMP) {
    case 16: B2_TRY(launch_mlp<16>(p, st)); break;
    case 32: B2_TRY(launch_mlp<32>(p, st)); break;
    case 48: B2_TRY(launch_mlp<48>(p, st)); break;
    case 64: B2_TRY(launch_mlp<64>(p, st)); break;
    case 80: B2_TRY(launch_mlp<80>(p, st)); break;
    case 96: B2_TRY(launch_mlp<96>(p, st)); break;
    case 112: B2_TRY(launch_mlp<112>(p, st)); break;
    default: B2_TRY(launch_mlp<128>(p, st)); break;
  }
  if (!(p->use_tc && p->view.N3)) { // otherwise k_mlp_tc produced the U table as its third GEMM
    switch (p->model.K1R) {
      case 9: k_utable<9><<<grid_for(n, BLK), BLK, 0, st>>>(p->view); break;
      case 13: k_utable<13><<<grid_for(n, BLK), BLK, 0, st>>>(p->view); break;
      default: k_utable<17><<<grid_for(n, BLK), BLK, 0, st>>>(p->view); break;
    }
    B2_LAUNCHED();
  }
  pf.end(st, ST_MLP);
  pf.begin(st, ST_FORCE_A);
  switch (p->model.K1A) {
    case 9: B2_TRY(launch_angular<9>(p, box, st, true)); break;
    case 13: B2_TRY(launch_angular<13>(p, box, st, true)); break;
    default: B2_TRY(launch_angular<17>(p, box, st, true)); break;
  }
  pf.end(st, ST_FORCE_A);
  return B200MD_OK;
}

int nep_pipeline(
  b200md_nep* p, const B2Box& box, cudaStream_t st, double* d_pe, double* d_force, double* d_virial)
{
  StageProfiler& pf = p->prof;
  p->tc_ctas_last = 0;
  pf.begin(st, ST_DESC_R);
  switch (p->model.K1R) {
    case 9: B2_TRY(dispatch_desc_radial<9>(p, box, st)); break;
    case 13: B2_TRY(dispatch_desc_radial<13>(p, box, st)); break;
    default: B2_TRY(dispatch_desc_radial<17>(p, box, st)); break;
  }
  pf.end(st, ST_DESC_R);
  if (p->ang_fused) {
    pf.begin(st, ST_ANG_FUSED);
    switch (p->model.K1A) {
      case 9: B2_TRY(launch_angular_fused<9>(p, box, st)); break;
      case 13: B2_TRY(launch_angular_fused<13>(p, box, st)); break;
      default: B2_TRY(launch_angular_fused<17>(p, box, st)); break;
    }
    pf.end(st, ST_ANG_FUSED);
  } else {
    B2_TRY(angular_stages(p, box, st));
  }
  pf.begin(st, ST_FORCE_FINAL);
  switch (p->model.K1R) {
    case 9: B2_TRY(dispatch_force_final<9>(p, box, st, d_pe, d_force, d_virial)); break;
    case 13: B2_TRY(dispatch_force_final<13>(p, box, st, d_pe, d_force, d_virial)); break;
    default: B2_TRY(dispatch_force_final<17>(p, box, st, d_pe, d_force, d_virial)); break;
  }
  pf.end(st, ST_FORCE_FINAL);
  return B200MD_OK;
}

int nep_setup(b200md_nep* p, int num_atoms)
{
  NepModel& m = p->model;
  p->n = num_atoms;
  const size_t N = (size_t)num_atoms;
  B2_TRY(upload(p->rc_r, m.rc_r));
  B2_TRY(upload(p->rcinv_r, m.rcinv_r));
  B2_TRY(upload(p->rc2_r, m.rc2_r));
  B2_TRY(upload(p->rc_a, m.rc_a));
  B2_TRY(upload(p->rcinv_a, m.rcinv_a));
  B2_TRY(upload(p->rc2_a, m.rc2_a));
  B2_TRY(upload(p->c_r, m.c_r));
  B2_TRY(upload(p->c_a, m.c_a));
  B2_TRY(upload(p->c_a4, m.c_a4));
  B2_TRY(upload(p->c_r4, m.c_r4));
  B2_TRY(upload(p->w0p, m.w0p));
  B2_TRY(upload(p->b0, m.b0));
  B2_TRY(upload(p->w1, m.w1));
  B2_TRY(upload(p->bias, m.bias));
  B2_TRY(upload(p->q_scaler, m.q_scaler));
  B2_TRY(upload(p->zbl_para, m.zbl_para));
  B2_TRY(upload(p->zbl_z, m.atomic_numbers));
  std::vector<float> cov(COVALENT_RADIUS, COVALENT_RADIUS + 94);
  B2_TRY(upload(p->cov_radius, cov));

  // Neighbor::initialize: skin-list capacity MN*((rc+skin)/rc)^3, neighbor.cu:824-829
  const double rc = m.rc_radial_max;
  const double rs = rc + 1.0;
  const int mn_skin = (int)(m.MN_radial * rs * rs * rs / (rc * rc * rc));
  // radial passes: thread per atom by default.  B200MD_NEP_TEAM=1 selects the lane-team kernels
  // for one- and two-type models: they cut the L1 gather wavefronts ~3x but cost ~30% more
  // instructions and are slower.
  const char* team_env = std::getenv("B200MD_NEP_TEAM");
  const bool team = m.nt <= 2 && team_env && std::strcmp(team_env, "1") == 0;
  p->nb.skin_row_major = team;
  if (const char* v = std::getenv("B200MD_NEP_VARIANT"))
    p->variant = std::atoi(v);
  // fused split pays when few skin candidates fail the radial test: (rc+skin)^3 / rc^3 small
  p->fuse_split = rs * rs * rs / (rc * rc * rc) < 1.45;
  B2_TRY(p->nb.init(num_atoms, rc, mn_skin));
  // one- and two-type models: the plane-based radial kernels (B200MD_NEP_RADIAL=v1 keeps the
  // round-1 kernels for A/B runs)
  const char* rad_env = std::getenv("B200MD_NEP_RADIAL");
  p->radial_v2 = m.nt <= 2 && !team && !(rad_env && std::strcmp(rad_env, "v1") == 0) &&
                 (double)num_atoms * (mn_skin + 2) < 4.0e9; // 32-bit list offsets in those kernels
  if (const char* v = std::getenv("B200MD_NEP_SLOTMAP"))
    p->slot_map = std::atoi(v) != 0;
  if (const char* v = std::getenv("B200MD_NEP_RADREG"))
    p->rad_reg = std::atoi(v) != 0;
  if (const char* v = std::getenv("B200MD_NEP_CSTAGE"))
    p->ang_cstage = std::atoi(v) != 0;
  p->nb.tag_types = p->radial_v2; // skin entries carry the neighbour type (b2_nep_radial.cuh)
  // Hidden layer and angular stages.  B200MD_NEP_MLP unset: k_angular_fused where the model fits its budget
  // (FUSED_DIMP, FUSED_MAX_SMEM; DESIGN.md 3.2); then the SIMT layer is also the hidden layer of the
  // generic kernels (B200MD_NEP_RADIAL=v1), which keeps the two paths bit-identical.  Otherwise the
  // tensor cores unless the shapes do not fit them.  B200MD_NEP_MLP=simt / =tc select the SIMT / the
  // tensor-core layer between separate angular kernels.
  const char* mlp_env = std::getenv("B200MD_NEP_MLP");
  const bool mlp_simt = mlp_env && std::strcmp(mlp_env, "simt") == 0;
  p->fused_smem = b2_fused_smem_bytes(m.nt, m.na1, m.K1A, m.nneu, m.DIMP);
  const bool fused_fits = m.nt <= 2 && !mlp_env && m.DIMP == FUSED_DIMP &&
                          p->fused_smem <= FUSED_MAX_SMEM;
  p->ang_fused = fused_fits && p->radial_v2;
  p->fused_shape = p->ang_fused ? fused_shape_of(m) : FUSED_SHAPE_NONE;
  p->use_tc = m.tc_ok && !mlp_simt && !fused_fits;
  if (p->radial_v2)
    B2_TRY(p->nb.enable_planes());
  {
    const char* e = std::getenv("B200MD_NEP_SCHED");
    p->sched = p->radial_v2 && !(e && e[0] == '0');
    if (p->sched)
      B2_TRY(p->nb.enable_schedule());
  }
  const int pitch_r = (m.MN_radial + 7) / 8 * 8;
  // B200MD_NEP_REVSLOT=1 (many types with the neighbour split as its own kernel): direct reverse slots
  // for the angular pair reduction instead of a binary search per pair: k_force_final gets faster on
  // UNEP-v1, but the extra stores slow k_split down by more, so it stays an opt-in.
  {
    const char* e = std::getenv("B200MD_NEP_REVSLOT");
    p->rev_slot = m.nt > 2 && !team && !p->fuse_split && e && e[0] == '1';
    if (p->rev_slot) {
      B2_TRY(p->nb.enable_reverse());
      B2_CUDA(p->aslot.reserve(N * (size_t)mn_skin));
      B2_CUDA(p->nla_rs.reserve(N * (size_t)m.MN_angular));
      B2_CUDA(cudaMemset(p->aslot.p, 0xff, sizeof(int) * N * (size_t)mn_skin));
      B2_CUDA(cudaMemset(p->nla_rs.p, 0, sizeof(int) * N * (size_t)m.MN_angular));
    }
  }

  B2_CUDA(p->nn_r.reserve(N));
  B2_CUDA(p->nl_r.reserve(N * (size_t)pitch_r));
  B2_CUDA(p->nn_a.reserve(N));
  B2_CUDA(p->nl_a.reserve(N * m.MN_angular));
  B2_CUDA(p->q.reserve(N * m.dim));
  if (!p->ang_fused) { // k_angular_fused keeps s and dU/dq on chip
    B2_CUDA(p->sfx.reserve(N * m.na1 * B2_NABC));
    B2_CUDA(p->FpR.reserve(N * m.nr1));
    B2_CUDA(p->FpA.reserve(N * m.dim_angular));
  }
  B2_CUDA(p->U.reserve(N * m.UST));
  B2_CUDA(p->f12.reserve(N * (p->radial_v2 ? 4 : 3) * m.MN_angular)); // few types: float4 entries
  if (p->radial_v2)
    B2_CUDA(p->arev.reserve(N * m.MN_angular));
  B2_CUDA(p->acc.reserve(N)); // site energies from the MLP pass

  B2NepView& P = p->view;
  std::memset(&P, 0, sizeof P);
  P.nt = m.nt;
  P.nr1 = m.nr1;
  P.na1 = m.na1;
  P.kr1 = m.kr1;
  P.ka1 = m.ka1;
  P.K1R = m.K1R;
  P.K1A = m.K1A;
  P.KP = m.KP;
  P.UST = m.UST;
  P.has222 = m.has222;
  P.has1111 = m.has1111;
  P.num_L = m.num_L;
  P.dim = m.dim;
  P.dim_ang = m.dim_angular;
  P.nneu = m.nneu;
  P.DIMP = m.DIMP;
  P.zbl_enabled = m.zbl_enabled;
  P.zbl_flexible = m.zbl_flexible;
  P.zbl_typewise = m.zbl_typewise;
  P.zbl_rc_inner = m.zbl_rc_inner;
  P.zbl_rc_outer = m.zbl_rc_outer;
  P.zbl_typewise_factor = m.zbl_typewise_factor;
  P.rc_r = p->rc_r.p;
  P.rcinv_r = p->rcinv_r.p;
  P.rc2_r = p->rc2_r.p;
  P.rc_a = p->rc_a.p;
  P.rcinv_a = p->rcinv_a.p;
  P.rc2_a = p->rc2_a.p;
  P.c_r = p->c_r.p;
  P.c_a = p->c_a.p;
  {
    // B200MD_NEP_CVEC=0: scalar coefficient loads in the radial contraction (A/B switch; results are
    // bit-identical).  The angular kernels always use the padded rows.
    const char* e = getenv("B200MD_NEP_CVEC");
    const bool cvec = !(e && e[0] == '0');
    P.c_a4 = reinterpret_cast<const float4*>(p->c_a4.p);
    P.c_r4 = cvec ? reinterpret_cast<const float4*>(p->c_r4.p) : nullptr;
    P.nqr = m.nqr;
    if (const char* d = getenv("B200MD_DEBUG_SKIP")) {
      P.debug_skip = atoi(d);
      if (P.debug_skip)
        fprintf(stderr, "libb200md: B200MD_DEBUG_SKIP=%d -- parts of the NEP force are SWITCHED OFF "
                        "(kernel timing only, results are wrong)\n", P.debug_skip);
    }
  }
  P.w0p = p->w0p.p;
  P.b0 = p->b0.p;
  P.w1 = p->w1.p;
  P.bias = p->bias.p;
  P.q_scaler = p->q_scaler.p;
  P.zbl_z = p->zbl_z.p;
  P.zbl_para = p->zbl_para.p;
  P.cov_radius = p->cov_radius.p;
  P.n = num_atoms;
  P.mn_r = m.MN_radial;
  P.mn_a = m.MN_angular;
  P.atoms = p->nb.atoms.p;
  P.perm = p->nb.perm.p;
  P.nn_skin = p->nb.nn_skin.p;
  P.nl_skin = p->nb.nl_skin.p;
  P.rskin = p->rev_slot ? p->nb.rskin.p : nullptr;
  P.aslot = p->rev_slot ? p->aslot.p : nullptr;
  P.nla_rs = p->rev_slot ? p->nla_rs.p : nullptr;
  P.nn_r = p->nn_r.p;
  P.nl_r = p->nl_r.p;
  P.nn_a = p->nn_a.p;
  P.nl_a = p->nl_a.p;
  P.q = p->q.p;
  P.sfx = p->ang_fused ? nullptr : p->sfx.p;
  P.FpR = p->ang_fused ? nullptr : p->FpR.p;
  P.FpA = p->ang_fused ? nullptr : p->FpA.p;
  P.U = p->U.p;
  P.f12 = p->f12.p;
  P.acc = p->acc.p;
  P.flags = p->nb.flags.p;
  P.seg_order = p->sched ? p->nb.seg_order.p : nullptr;
  P.team = team ? 1 : 0;
  P.u_planes = p->radial_v2 ? 2 : (team ? 1 : 0);
  P.pitch_r = pitch_r;
  {
    const B2NeighborView nv = p->nb.view();
    P.skin_si = nv.skin_si;
    P.skin_sk = nv.skin_sk;
  }
  if (p->use_tc) {
    int dev = 0;
    B2_CUDA(cudaGetDevice(&dev));
    B2_CUDA(cudaDeviceGetAttribute(&p->num_sms, cudaDevAttrMultiProcessorCount, dev));
    // B200MD_NEP_TC_CTAS=k (tests): cap the persistent CTAs so that each walks many tiles
    if (const char* e = std::getenv("B200MD_NEP_TC_CTAS"))
      p->tc_ctas_cap = std::atoi(e) > 0 ? std::atoi(e) : 0;
    B2_TRY(p->nb.enable_type_tiles(m.nt));
    B2_TRY(upload(p->tc_img, m.tc_img));
    P.tc_img = p->tc_img.p;
    P.tc_img_floats = m.tc_img_floats;
    P.HN = m.HN;
    P.DK = m.DK;
    P.DN = m.DN;
    P.K3 = m.K3;
    // the U table as a third GEMM of the same kernel (AoS rows or float4 planes, see epilogue 3)
    const char* u_env = std::getenv("B200MD_NEP_UTABLE");
    P.N3 = (m.tc3_ok && !(u_env && std::strcmp(u_env, "simt") == 0)) ? m.N3 : 0;
    P.tile_atom = p->nb.tile_atom.p;
    { // tile-major q and dU/dq: zeroed once so that padding rows / columns hold finite values
      const size_t floats = (size_t)p->nb.max_tiles() * 128 * m.DK;
      B2_CUDA(p->qt.reserve(floats));
      B2_CUDA(p->fpt.reserve(floats));
      B2_CUDA(cudaMemset(p->qt.p, 0, sizeof(float) * floats));
      B2_CUDA(cudaMemset(p->fpt.p, 0, sizeof(float) * floats));
      P.qt = p->qt.p;
      P.fpt = p->fpt.p;
      P.DKT = m.DK;
      P.tile_slot = p->nb.tile_slot.p;
    }
    P.tile_type = p->nb.tile_type.p;
    P.tile_meta = p->nb.tile_meta.p;
  }

  // shared-memory budgets
  // (k_force_angular2: one padded row of b2_ang_ws4(na1) float4s per thread)
  const size_t ang_row = p->radial_v2 ? b2_ang_ws4(m.na1) * sizeof(float4) : m.na1 * B2_NABC * sizeof(float);
  p->ang_block = BLK;
  p->ang_smem = ang_row * p->ang_block;
  while (p->ang_smem > 200 * 1024 && p->ang_block > 32) {
    p->ang_block /= 2;
    p->ang_smem = ang_row * p->ang_block;
  }
  // Radial descriptor of a many-type model: per-type accumulators in shared memory while two blocks of
  // them fit an SM, else (NEP89: 89 species) the per-pair contraction, which needs no such storage.
  // B200MD_NEP_RADDIRECT=1 forces the latter for any model with more than two types (tests, A/B).
  p->rad_smem = (size_t)m.nt * m.K1R * BLK * sizeof(float);
  p->rad_direct = false;
  if (m.nt > 2) {
    const char* e = std::getenv("B200MD_NEP_RADDIRECT");
    const bool forced = e && e[0] == '1';
    if (forced || p->rad_smem > 96 * 1024) {
      if (m.nqr > B2_NQMAX) {
        set_error("n_max_radial above 19 is not supported for models with this many atom types");
        return B200MD_ERR_ARG;
      }
      p->rad_direct = true;
      p->rad_smem = 0;
      P.c_r4 = reinterpret_cast<const float4*>(p->c_r4.p); // regardless of B200MD_NEP_CVEC
    }
  }
  // 3..16 types: register accumulators (B200MD_NEP_RADREG=1) when NT*K1 fits the register file; the
  // default keeps the accumulators in shared memory
  {
    const int nt = m.nt;
    const int ntb = !p->rad_reg ? 0 : nt <= 4 ? 4 : nt <= 8 ? 8 : nt <= 16 ? 16 : 0;
    p->rad_nt = p->rad_direct ? -1 : ntb * m.K1R <= 160 ? ntb : 0;
  }
  B2_CUDA(cudaDeviceSynchronize());
  return B200MD_OK;
}

// type tiles of the last list rebuild (synchronises; 0 without tiles)
int nep_tile_count(const b200md_nep* p)
{
  if (!p->use_tc || !p->nb.have_grid)
    return 0;
  int ntile = 0;
  if (cudaDeviceSynchronize() != cudaSuccess ||
      cudaMemcpy(&ntile, p->nb.tile_meta.p, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess)
    return -1;
  return ntile;
}

} // namespace

extern "C" {

int b200md_nep_create(const char* path, int num_atoms, b200md_nep** out)
{
  if (!path || !out || num_atoms <= 0) {
    set_error("b200md_nep_create: bad argument");
    return B200MD_ERR_ARG;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_error("b200md_nep_create: no CUDA device (libb200md has no CPU fallback)");
    return B200MD_ERR_CUDA;
  }
  b200md_nep* p = new (std::nothrow) b200md_nep;
  if (!p) {
    set_error("out of host memory");
    return B200MD_ERR_ARG;
  }
  const std::string err = p->model.load(path);
  if (!err.empty()) {
    set_error(err);
    const bool io = err.rfind("Failed to open", 0) == 0;
    delete p;
    return io ? B200MD_ERR_IO : B200MD_ERR_ARG;
  }
  const int rc = nep_setup(p, num_atoms);
  if (rc != B200MD_OK) {
    delete p;
    return rc;
  }
  *out = p;
  return B200MD_OK;
}

void b200md_nep_destroy(b200md_nep* p) { delete p; }

int b200md_nep_info(const b200md_nep* p, int what)
{
  switch (what) {
    case 0: return p->model.nt;
    case 1: return p->model.dim;
    case 2: return p->model.nneu;
    case 3: return p->model.MN_radial;
    case 4: return p->model.MN_angular;
    case 5: return p->model.zbl_enabled ? 1 : 0;
    case 6: {
      int bits = 0, rebuilds = 0;
      const_cast<b200md_nep*>(p)->nb.check(0, &bits, &rebuilds);
      return rebuilds;
    }
    case 7: return p->sched ? p->nb.num_segments() : 0;
    case 8: return nep_tile_count(p);
    case 9: return p->tc_ctas_last;
    case 10: return p->fused_shape;
    case 11: return p->ang_fused ? 0 : p->ang_block;
    case 12: { // mirrors dispatch_desc_radial
      const int nt = p->model.nt;
      if (p->view.team)
        return 200 + nt;
      if (p->radial_v2)
        return 100 + nt;
      return nt <= 2 ? nt : p->rad_nt;
    }
    case 13:
      if (p->view.team || p->radial_v2)
        return -1;
      return (p->model.nt <= 2 || p->fuse_split) ? 1 : 0;
    case 14:
      if (p->ang_fused)
        return 0;
      return (p->use_tc && p->view.N3) ? 1 : 2;
    case 15:
      if (p->radial_v2)
        return -1;
      return ang_coeff_staged(p) ? 1 : 0;
    case 16: return p->rev_slot ? 1 : 0;
    case 17: return (p->ang_fused || p->use_tc) ? 0 : p->model.DIMP;
    case 18:
      if (p->ang_fused || p->use_tc)
        return -1;
      return mlp_weights_staged(p) ? 1 : 0;
    default: return -1;
  }
}

double b200md_nep_rc(const b200md_nep* p) { return p->model.rc_radial_max; }

const char* b200md_nep_symbol(const b200md_nep* p, int t)
{
  return (t >= 0 && t < p->model.nt) ? p->model.symbols[t].c_str() : "";
}

int b200md_nep_compute(
  b200md_nep* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  B2Box box = make_box(h, pbc);
  p->view.overwrite = p->overwrite;
  p->view.n_own = p->n_own;
  p->view.use_active = p->use_active;
  for (int d = 0; d < 3; ++d) {
    p->view.act_lo[d] = p->act_lo[d];
    p->view.act_hi[d] = p->act_hi[d];
  }
  // Small periodic box (a periodic thickness <= 2.5*(rc+skin); the reference switches to explicit
  // images at 2.5*rc, nep.cu:1304-1312, nep_small_box.cuh): evaluate the smallest supercell that
  // the cell-list path accepts and keep the first replica.  Every atom of that replica sees each
  // periodic image of its neighbours as a distinct atom, exactly the reference's pair set.
  int reps[3] = {1, 1, 1};
  const double need = 2.5 * (p->nb.rc + p->nb.skin);
  for (int d = 0; d < 3; ++d)
    if (box.pbc[d] && box.thickness[d] <= need)
      reps[d] = (int)std::floor(need / box.thickness[d]) + 1;
  const long long R = (long long)reps[0] * reps[1] * reps[2];
  p->rep_n = 0;
  if (R > 1) {
    if (R * n > 50000000LL) {
      set_error("small-box supercell would exceed 5e7 atoms");
      return B200MD_ERR_SMALL_BOX;
    }
    const int nR = (int)(R * n);
    if (nR > p->nb.capacity) { // first small-box call (or a shrinking box): grow the scratch
      B2_CUDA(cudaStreamSynchronize(st));
      B2_TRY(nep_setup(p, nR));
      p->view.overwrite = p->overwrite;
      p->view.n_own = p->n_own; // supercell indices below n_own all lie in the first replica
    }
    // The active region is in the caller's coordinates, and the image atoms of the supercell need
    // their descriptors: a small box ignores it.
    p->view.use_active = 0;
    B2_CUDA(p->rep_type.reserve(nR));
    B2_CUDA(p->rep_pos.reserve(3 * (size_t)nR));
    B2_CUDA(p->rep_out.reserve(13 * (size_t)nR));
    k_replicate<<<grid_for(nR, BLK), BLK, 0, st>>>(
      n, reps[0], reps[1], reps[2], box, d_type, d_position, p->rep_type.p, p->rep_pos.p);
    B2_LAUNCHED();
    B2_CUDA(cudaMemsetAsync(p->rep_out.p, 0, sizeof(double) * 13 * (size_t)nR, st));
    double hs[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        hs[3 * r + c] = h[3 * r + c] * reps[c]; // scale lattice vector c (a column)
    box = make_box(hs, pbc);
    p->prof.next_step();
    p->prof.begin(st, ST_NEIGHBOR);
    B2_TRY(p->nb.update(box, p->rep_type.p, p->rep_pos.p, nR, st));
    p->n = nR;
    p->view.n = nR;
    if (!p->view.team)
      p->view.skin_sk = (size_t)nR;
    p->rep_n = n;
    p->prof.end(st, ST_NEIGHBOR);
    double* acc = p->rep_out.p;
    B2_TRY(nep_pipeline(p, box, st, acc, acc + nR, acc + 4 * (size_t)nR));
    k_fold_replica<<<grid_for(n, BLK), BLK, 0, st>>>(
      n, (size_t)nR, acc, d_potential, d_force, d_virial, p->overwrite, p->n_own);
    B2_LAUNCHED();
    return B200MD_OK;
  }
  p->prof.next_step();
  p->prof.begin(st, ST_NEIGHBOR);
  B2_TRY(p->nb.update(box, d_type, d_position, n, st));
  p->n = n; // n may be anything up to the capacity given at construction (domain decomposition)
  p->view.n = n;
  if (!p->view.team)
    p->view.skin_sk = (size_t)n; // column-major skin list: entry stride = current atom count
  p->prof.end(st, ST_NEIGHBOR);
  B2_TRY(nep_pipeline(p, box, st, d_potential, d_force, d_virial));
  return B200MD_OK;
}

int b200md_nep_compute_host(
  b200md_nep* p, int n, const double h[9], const int pbc[3], const int* type,
  const double* position, double* potential, double* force, double* virial)
{
  const size_t N = (size_t)n;
  B2_CUDA(p->h_type.reserve(N));
  B2_CUDA(p->h_pos.reserve(3 * N));
  B2_CUDA(p->h_out.reserve(13 * N));
  cudaStream_t st = 0;
  B2_CUDA(cudaMemcpyAsync(p->h_type.p, type, sizeof(int) * N, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(p->h_pos.p, position, sizeof(double) * 3 * N, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemsetAsync(p->h_out.p, 0, sizeof(double) * 13 * N, st));
  double* d_pe = p->h_out.p;
  double* d_f = p->h_out.p + N;
  double* d_v = p->h_out.p + 4 * N;
  B2_TRY(b200md_nep_compute(p, n, h, pbc, p->h_type.p, p->h_pos.p, d_pe, d_f, d_v, st));
  B2_CUDA(cudaMemcpyAsync(potential, d_pe, sizeof(double) * N, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(force, d_f, sizeof(double) * 3 * N, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaMemcpyAsync(virial, d_v, sizeof(double) * 9 * N, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return b200md_nep_check(p, st);
}

int b200md_nep_export_neighbors(
  b200md_nep* p, int mn_r, int* d_NN_r, int* d_NL_r, int mn_a, int* d_NN_a, int* d_NL_a,
  void* stream)
{
  cudaStream_t st = (cudaStream_t)stream;
  const int n = p->n;
  if (d_NN_r && d_NL_r) {
    k_export_list<<<grid_for(n, 128), 128, 0, st>>>(
      n, p->rep_n ? p->rep_n : n, p->nb.perm.p, p->nn_r.p, p->nl_r.p,
      p->view.team ? (size_t)p->view.pitch_r : 1,
      p->view.team ? 1 : (size_t)n, mn_r, d_NN_r, d_NL_r, p->nb.flags.p,
      p->radial_v2 ? B2_TAG_MASK : -1);
    B2_LAUNCHED();
  }
  if (d_NN_a && d_NL_a) {
    k_export_list<<<grid_for(n, 128), 128, 0, st>>>(
      n, p->rep_n ? p->rep_n : n, p->nb.perm.p, p->nn_a.p, p->nl_a.p, 1, (size_t)n, mn_a, d_NN_a,
      d_NL_a, p->nb.flags.p, p->radial_v2 ? B2_TAG_MASK : -1);
    B2_LAUNCHED();
  }
  return B200MD_OK;
}

int b200md_nep_set_owned(b200md_nep* p, int n_owned)
{
  if (n_owned < 0) {
    set_error("b200md_nep_set_owned: negative count");
    return B200MD_ERR_ARG;
  }
  p->n_own = n_owned;
  return B200MD_OK;
}

int b200md_nep_set_accumulate(b200md_nep* p, int accumulate)
{
  p->overwrite = accumulate ? 0 : 1;
  return B200MD_OK;
}

int b200md_nep_set_active_region(b200md_nep* p, const double lo[3], const double hi[3])
{
  if (!lo || !hi) {
    p->use_active = 0;
    return B200MD_OK;
  }
  p->use_active = 1;
  for (int d = 0; d < 3; ++d) {
    p->act_lo[d] = lo[d];
    p->act_hi[d] = hi[d];
  }
  return B200MD_OK;
}

int b200md_nep_export_descriptors(b200md_nep* p, float* d_q, void* stream)
{
  k_export_q<<<grid_for(p->n, 128), 128, 0, (cudaStream_t)stream>>>(
    p->view, p->rep_n ? p->rep_n : p->n, d_q);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_nep_export_schedule(
  b200md_nep* p, int dims[6], int* d_seg_order, int* d_cell_start, void* stream)
{
  if (!p->sched || !p->nb.have_grid) {
    set_error("b200md_nep_export_schedule: no schedule (identity schedule, or no compute call yet)");
    return B200MD_ERR_ARG;
  }
  const B2Grid& g = p->nb.grid;
  const B2Bricks br = b2_make_bricks(g, p->nb.n);
  for (int d = 0; d < 3; ++d)
    dims[d] = g.nb[d];
  dims[3] = br.bx;
  dims[4] = br.by;
  dims[5] = br.bz;
  cudaStream_t st = (cudaStream_t)stream;
  if (d_seg_order)
    B2_CUDA(cudaMemcpyAsync(d_seg_order, p->nb.seg_order.p, sizeof(int) * p->nb.num_segments(),
                            cudaMemcpyDeviceToDevice, st));
  if (d_cell_start)
    B2_CUDA(cudaMemcpyAsync(d_cell_start, p->nb.cell_start.p, sizeof(int) * ((size_t)g.ncell + 1),
                            cudaMemcpyDeviceToDevice, st));
  return B200MD_OK;
}

int b200md_nep_export_tiles(b200md_nep* p, int* d_slot, int* d_tile_type, void* stream)
{
  const int ntile = nep_tile_count(p);
  if (ntile <= 0) {
    set_error("b200md_nep_export_tiles: no type tiles (SIMT hidden layer, or no compute call yet)");
    return B200MD_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (d_slot) {
    k_export_tile_slot<<<grid_for(p->n, 128), 128, 0, st>>>(
      p->n, p->rep_n ? p->rep_n : p->n, p->nb.perm.p, p->nb.tile_slot.p, d_slot);
    B2_LAUNCHED();
  }
  if (d_tile_type)
    B2_CUDA(cudaMemcpyAsync(d_tile_type, p->nb.tile_type.p, sizeof(int) * ntile, cudaMemcpyDeviceToDevice, st));
  return B200MD_OK;
}

int b200md_nep_export_mlp(b200md_nep* p, float* d_fp, float* d_u, void* stream)
{
  if (p->ang_fused) {
    set_error("b200md_nep_export_mlp: k_angular_fused keeps dU/dq and the U table on chip");
    return B200MD_ERR_ARG;
  }
  k_export_mlp<<<grid_for(p->n, 128), 128, 0, (cudaStream_t)stream>>>(
    p->view, p->rep_n ? p->rep_n : p->n, d_fp, d_u);
  B2_LAUNCHED();
  return B200MD_OK;
}

int b200md_nep_profile(b200md_nep* p, int enable)
{
  p->prof.enable(enable != 0);
  return B200MD_OK;
}

int b200md_nep_profile_read(b200md_nep* p, int max_stages, float* ms_sum, int* counts)
{
  float ms[StageProfiler::MAX_STAGES];
  int cn[StageProfiler::MAX_STAGES];
  p->prof.read(ms, cn);
  const int m = max_stages < ST_COUNT ? max_stages : ST_COUNT;
  for (int k = 0; k < m; ++k) {
    ms_sum[k] = ms[k];
    counts[k] = cn[k];
  }
  return m;
}

const char* b200md_nep_stage_name(int stage)
{
  return (stage >= 0 && stage < ST_COUNT) ? STAGE_NAMES[stage] : "";
}

/* mean neighbour counts of the last compute (skin, radial, angular) -- inputs of the
 * algorithmic-bytes formula in DESIGN.md */
int b200md_nep_mean_neighbors(b200md_nep* p, double out3[3])
{
  const size_t N = (size_t)p->n;
  std::vector<int> a(N), b(N), c(N);
  B2_CUDA(cudaDeviceSynchronize());
  B2_CUDA(cudaMemcpy(a.data(), p->nb.nn_skin.p, sizeof(int) * N, cudaMemcpyDeviceToHost));
  B2_CUDA(cudaMemcpy(b.data(), p->nn_r.p, sizeof(int) * N, cudaMemcpyDeviceToHost));
  B2_CUDA(cudaMemcpy(c.data(), p->nn_a.p, sizeof(int) * N, cudaMemcpyDeviceToHost));
  double s[3] = {0, 0, 0};
  for (size_t i = 0; i < N; ++i) {
    s[0] += a[i];
    s[1] += b[i];
    s[2] += c[i];
  }
  for (int k = 0; k < 3; ++k)
    out3[k] = s[k] / (double)N;
  return B200MD_OK;
}

int b200md_nep_invalidate(b200md_nep* p, int n_new, void* stream)
{
  B2_TRY(p->nb.invalidate(n_new, (cudaStream_t)stream));
  p->n = n_new;
  p->view.n = n_new;
  return B200MD_OK;
}

int b200md_nep_check(b200md_nep* p, void* stream)
{
  int bits = 0, rebuilds = 0;
  B2_TRY(p->nb.check((cudaStream_t)stream, &bits, &rebuilds));
  if (bits) {
    char buf[256];
    snprintf(
      buf, sizeof buf,
      "neighbour capacity exceeded on the device (bits=%d: 1 skin list, 2 radial MN, 4 angular MN)",
      bits);
    set_error(buf);
    return B200MD_ERR_OVERFLOW;
  }
  return B200MD_OK;
}

} // extern "C"

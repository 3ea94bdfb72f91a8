/*
 * b200md_mgpu.h -- C-ABI of libb200md_mgpu.so: spatial-domain sharding of the MD hot path over
 * several GPUs, host side in C++, device side CUDA + NCCL.
 *
 * Replaces NEP_MULTIGPU::compute (src/force/nep_multigpu.cu:1416-1803) and the single-GPU
 * integration around it: there GPU 0 owns all atoms, scatters positions / gathers forces through
 * blocking peer copies every step, rebuilds every list every step and integrates everything itself.
 * Here the box is cut into a Px x Py x Pz grid of BLOCKS (slabs = P x 1 x 1); every rank owns the
 * atoms of one block, integrates them where they live, and receives only the FP64 POSITIONS of the
 * ghost atoms within `halo` of its faces, by a staged (x, then y, then z) ncclSend/ncclRecv exchange
 * per force evaluation.  As in the reference (nep_multigpu.cuh:42-53) the halo of a many-body
 * potential is two cutoffs wide, so descriptors of the first ghost layer are recomputed locally and no
 * force travels back.  Migration and the rebuild of the ghost lists are device-side (flag kernels +
 * CUB compaction + packed NCCL messages) and happen only when some atom has moved further than
 * 0.7 * skin / 2 since the last one.  Thermo is an 8-double ncclAllReduce; thermostat state is
 * replicated.
 *
 * One GROUP = the domains hosted by this process:
 *   - distributed: one process per GPU (torchrun / mpirun style), exactly one domain per group,
 *     nccl_id = the 128 bytes of an ncclUniqueId shared by all ranks (b200md_mgpu_unique_id);
 *   - local: nccl_id = NULL and the group hosts ALL Px*Py*Pz domains on the current device, run in
 *     lock step with device-to-device copies instead of NCCL -- the same kernels, lists and
 *     ordering, testable on one GPU.
 * Functions return 0 or a B200MD_ERR_* code (b200md.h); b200md_mgpu_last_error() describes it.
 */
#ifndef B200MD_MGPU_H
#define B200MD_MGPU_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200md_mgpu b200md_mgpu;

typedef struct {
  double h[9];         /* global box, Box::cpu_h[0..8]; must be orthogonal */
  int pbc[3];          /* decomposed directions must be periodic */
  int grid[3];         /* Px, Py, Pz; world size = Px*Py*Pz */
  int rank;            /* distributed mode: this process's rank in [0, world) */
  const char* potential_file; /* nep*, lj, tersoff_1989, eam_zhou_2004 / eam_dai_2006 */
  double skin;         /* ghost-list skin in A (>= 1); migration when an atom moved 0.7*skin/2 */
  /* ensemble: 0 nve, 1 nvt_ber, 2 nvt_nhc, 4 nvt_bdp (the reference's type codes) */
  int ensemble;
  double temperature, temperature_coupling, time_step; /* time_step in natural units */
  unsigned bdp_seed;
  double capacity_factor; /* local arrays hold capacity_factor * (initial local atoms) + 1024 */
  int use_cuda_graph;     /* 1: replay each step as one CUDA graph (captured after migrations) */
} b200md_mgpu_config;

const char* b200md_mgpu_last_error(void);
/* fills 128 bytes with a fresh ncclUniqueId (call on rank 0, broadcast to the others) */
int b200md_mgpu_unique_id(char out128[128]);

int b200md_mgpu_create(const b200md_mgpu_config* cfg, const char* nccl_id128, b200md_mgpu** out);
void b200md_mgpu_destroy(b200md_mgpu* g);

/* Every rank passes the same GLOBAL host arrays (type[n], position[3n] SoA, mass[n], velocity[3n]
 * SoA or NULL); each domain keeps what it owns, then ghosts are exchanged and forces evaluated. */
int b200md_mgpu_distribute(
  b200md_mgpu* g, int n_global, const int* type, const double* position, const double* mass,
  const double* velocity);

/* nsteps velocity-Verlet steps (Run::perform_a_run's loop body, run.cu:259-295), migration
 * included.  Asynchronous apart from the displacement check every `check_every` steps. */
int b200md_mgpu_run(b200md_mgpu* g, int nsteps, int check_every);

/* the same, bracketed by CUDA events on the module's stream: *ms_out = device time of the nsteps
 * (synchronises before and after) */
int b200md_mgpu_run_timed(b200md_mgpu* g, int nsteps, int check_every, double* ms_out);

/* global thermo[0..7] = T, U, sxx, syy, szz, sxy, sxz, syz (synchronises) */
int b200md_mgpu_thermo(b200md_mgpu* g, double out8[8]);
/* global heat current jx_in, jx_out, jy_in, jy_out, jz (compute_heat.cu:32-90 summed, hac.cu:51,106) */
int b200md_mgpu_heat_current(b200md_mgpu* g, double out5[5]);

/* HNEMD thermal conductivity (Fan et al., PRB 99, 064308 (2019)) inside the step, which becomes
 * VV1 -> halo -> potential -> drive -> VV2 -> thermostat -> heat row (Run::perform_a_run's order):
 *   drive     compute_hnemd's branch of Force::compute, src/force/force.cu:857-897: every block adds
 *             W_i^T fe to the forces of its owned atoms (the per-atom add of b200md_hnemd_drive, bit for
 *             bit), the blocks' totals of the new forces are summed (a 3-double ncclAllReduce; local
 *             mode: in block order) and every owned atom loses total / N;
 *   heat row  HNEMD::process, src/measure/hnemd_kappa.cu:82-106: every block sums the heat current of
 *             its owned atoms into a device row whose index lives on the device, so one captured graph
 *             serves every step; the blocks' rows are summed only by b200md_mgpu_hnemd_take.
 * b200md_mgpu_hnemd_set: call after b200md_mgpu_distribute (which switches HNEMD off).  fe[3] in 1/A;
 *   fe = 0 switches HNEMD off (Force::finalize).  Re-evaluates the forces at the current positions,
 *   driven when HNEMD is on, as the reference does before a run's loop (run.cu:217-248), discards the
 *   captured step and starts a new series.  Refuses output_interval < 1, max_intervals < 1 and a
 *   non-finite fe.  A b200md_mgpu_run that would leave more than max_intervals whole intervals untaken
 *   returns B200MD_ERR_OVERFLOW before it launches anything.
 * b200md_mgpu_hnemd_take: the output branch of HNEMD::process, hnemd_kappa.cu:108-131 (synchronises;
 *   the only HNEMD call that does).  *n_intervals = the intervals completed since the last take; for
 *   each, in order, kappa[5 j + k] (W/mK, k = xx_in xx_out yy_in yy_out zz; the factor of
 *   b200md_hnemd_take with the volume Lx Ly Lz) and, if rows != NULL, its output_interval global heat
 *   sums rows[(j * output_interval + m) * 5 + k].  kappa holds 5 * max_intervals doubles, rows
 *   5 * output_interval * max_intervals.  The steps of an unfinished interval carry over. */
int b200md_mgpu_hnemd_set(b200md_mgpu* g, int output_interval, const double fe[3], int max_intervals);
int b200md_mgpu_hnemd_take(
  b200md_mgpu* g, double temperature, int* n_intervals, double* kappa, double* rows);

/* counters: what = 0 local domains, 1 owned atoms of domain k, 2 local (owned+ghost) atoms of
 * domain k, 3 migrations so far, 4 neighbour rebuilds of domain k, 5 global rank of domain k,
 * 6 kernels launched per step (this module's + libb200md's, counted on the last eager step) */
long long b200md_mgpu_info(b200md_mgpu* g, int what, int k);
/* owned atoms of local domain k in GLOBAL coordinates: id[n], position[3n], velocity[3n],
 * force[3n], potential[n], virial[9n] (host arrays; any may be NULL) */
int b200md_mgpu_get_owned(
  b200md_mgpu* g, int k, long long* id, double* position, double* velocity, double* force,
  double* potential, double* virial);
/* the LOCAL system of domain k as the potential sees it: type[n_loc], position[3*n_loc] in the local
 * frame (owned atoms first), local box h[9] and pbc[3] (host arrays; any may be NULL) */
int b200md_mgpu_get_local(
  b200md_mgpu* g, int k, int* type, double* position, double h_out[9], int pbc_out[3]);
/* per-phase device time of the last b200md_mgpu_run when profiling was on (ms per step):
 * 0 vv1+wrap, 1 halo, 2 force, 3 vv2+thermo; returns the number of phases written */
int b200md_mgpu_profile(b200md_mgpu* g, int enable, double* ms_out, int max_out);
/* latched device-side neighbour-capacity errors of every local domain */
int b200md_mgpu_check(b200md_mgpu* g);

#ifdef __cplusplus
}
#endif
#endif

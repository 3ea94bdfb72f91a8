/*
 * b200md.h -- C-ABI of libb200md.so: the Hopper-native (sm_90a) MD hot path that drops in
 * behind GPUMD's Potential / Ensemble plugin surface.
 *
 * Every entry point states the reference interface it replaces (paths relative to the GPUMD
 * tree, commit d98135d).  Conventions on this boundary are GPUMD's own:
 *   - all `d_*` pointers are DEVICE pointers owned by the caller (GPUMD's GPU_Vector<T>);
 *     the library owns only its scratch (cell lists, neighbour lists, descriptor buffers);
 *   - per-atom arrays are SoA: position[3N] = x[N],y[N],z[N] (src/model/atom.cuh:21-52),
 *     virial[9N] = xx,yy,zz,xy,xz,yz,yx,zx,zy blocks of N (src/force/force.cu:859-861);
 *   - h[9] is Box::cpu_h[0..8] (src/model/box.cuh:18-35): row-major, lattice vectors as columns;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream, which is what
 *     every reference kernel uses, SURVEY.md 8b);
 *   - functions return 0 on success, non-zero on error; b200md_last_error() describes it.
 *     (The reference prints and exit(1)s, src/utilities/error.cuh:22-62; the C++ adapter in
 *     gpumd_b200/host does exactly that with these codes.)
 *   - work is enqueued asynchronously; capacity overflows detected on the device are latched
 *     and reported by b200md_*_check(), which synchronises the stream.
 * There is no CPU fallback anywhere behind this interface.
 */
#ifndef B200MD_H
#define B200MD_H

#ifdef __cplusplus
extern "C" {
#endif

#define B200MD_OK 0
#define B200MD_ERR_ARG 1       /* bad argument / unsupported model */
#define B200MD_ERR_IO 2        /* cannot read potential file */
#define B200MD_ERR_CUDA 3      /* CUDA runtime error */
#define B200MD_ERR_SMALL_BOX 4 /* periodic thickness <= 2.5*(rc+1): reference's small-box path */
#define B200MD_ERR_OVERFLOW 5  /* neighbour / cell capacity exceeded on the device */
#define B200MD_ERR_NOT_CONVERGED 6 /* an iterative solver reached its iteration cap */

const char* b200md_last_error(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
long long b200md_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * NEP potential.  Replaces class NEP : Potential (src/force/nep.cuh:27-184):
 *   b200md_nep_create  <- NEP::NEP(const char* file_potential, const int num_atoms), nep.cu:100-395
 *   b200md_nep_compute <- NEP::compute(Box&, type, position, potential, force, virial),
 *                         nep.cu:1356-1389 -> compute_large_box nep.cu:978-1138
 *                         (outputs are ACCUMULATED with += exactly like nep.cu:653,755-770)
 * ------------------------------------------------------------------------------------------ */
typedef struct b200md_nep b200md_nep;

int b200md_nep_create(const char* nep_txt_path, int num_atoms, b200md_nep** out);
void b200md_nep_destroy(b200md_nep* p);

/* what: 0 num_types, 1 descriptor dim, 2 neurons, 3 MN_radial (enlarged), 4 MN_angular
 * (enlarged), 5 zbl enabled, 6 number of neighbour-list rebuilds so far, 7 segments of the warp
 * schedule (0: identity schedule, see b200md_nep_export_schedule), 8 type tiles of the last list rebuild
 * (0: no tiles, the SIMT hidden layer), 9 CTAs of the last launch of the tensor-core hidden layer (0: the
 * last compute did not run it), 10 angular shape of k_angular_fused (0: the separate angular kernels run,
 * 1: the run-time-shape instance, 2: n_max 4 4 with l_max 4 2 0 compiled in, 3: the same with l_max 4 0 0).
 * The kernel instances the handle runs:
 *   11 threads per block of the angular force kernel (128, 64 or 32; 0: k_angular_fused runs instead)
 *   12 radial descriptor kernel: for three or more types NT of k_desc_radial<NT, K1, SPLIT> (-1 per-pair
 *      contraction, 0 accumulators in shared memory, 4 / 8 / 16 accumulators in registers); for one or two
 *      types 100 + types (the plane-based kernels), 200 + types (the lane-team kernels) or the number of
 *      types (the generic thread-per-atom instance)
 *   13 SPLIT of that k_desc_radial instance (1: the neighbour split is fused into it, 0: k_split runs
 *      before it; -1: the one- and two-type kernels, which have no split)
 *   14 the U table comes from the tensor-core hidden layer's third GEMM (1), from k_utable (2), or is not
 *      stored (0: k_angular_fused)
 *   15 k_desc_angular reads its coefficient table from shared memory (1) or global memory (0); -1: the
 *      one- and two-type angular kernels run instead
 *   16 direct reverse slots in the angular pair reduction (1: B200MD_NEP_REVSLOT=1 is in effect)
 *   17 DIMP of the SIMT hidden layer k_mlp<DIMP, STAGE> (0: the tensor-core layer or k_angular_fused)
 *   18 STAGE of that k_mlp instance (1: weights in shared memory, 0: in global memory; -1: it does not run)
 * 6 and 8 synchronise the device. */
int b200md_nep_info(const b200md_nep* p, int what);
double b200md_nep_rc(const b200md_nep* p); /* Potential::rc, src/force/potential.cuh:32 */
/* atomic symbol of type t (species -> type index mapping, src/model/read_xyz.cu:349-361) */
const char* b200md_nep_symbol(const b200md_nep* p, int t);

int b200md_nep_compute(
  b200md_nep* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream);

/* Same call with HOST buffers (pageable or pinned): copies type/position to the device, runs the
 * path, and OVERWRITES the host arrays potential[n], force[3n], virial[9n] with the result
 * (synchronous).  This is the end-to-end entry bench.py times. */
int b200md_nep_compute_host(
  b200md_nep* p, int n, const double h[9], const int pbc[3], const int* type,
  const double* position, double* potential, double* force, double* virial);

/* Parity hook: the radial / angular neighbour sets of the LAST compute call, mapped back to the
 * caller's atom indices, ascending, row-major NL[i*mn + k] -- the quantity the reference builds
 * in find_neighbor_list_large_box (nep.cu:436-486).  Device pointers. */
int b200md_nep_export_neighbors(
  b200md_nep* p, int mn_r, int* d_NN_r, int* d_NL_r, int mn_a, int* d_NN_a, int* d_NL_a,
  void* stream);
/* Row-major rows NL[i*mn + k] -> the reference's column-major layout NL[k*n + i]
 * (NEP::get_NL_radial_ptr, nep.cuh:100-101 / potential.cuh:66-77).  Device pointers. */
int b200md_transpose_int(int n, int mn, const int* d_row_major, int* d_column_major, void* stream);
/* Parity hook: scaled descriptors q[d*N + i] (caller order) of the last compute call. */
int b200md_nep_export_descriptors(b200md_nep* p, float* d_q, void* stream);

/* Parity hook: the warp schedule of the one- and two-species kernels as of the last list rebuild.  A segment
 * is 32 consecutive cell-sorted atoms; warp w evaluates segment seg_order[w].  dims = cells per direction
 * (3), cells per brick (3); d_seg_order[b200md_nep_info(p, 7)] and d_cell_start[cells + 1] (first sorted
 * atom of every cell, x fastest) are device pointers, each may be null.  Error when the handle runs the
 * identity schedule (B200MD_NEP_SCHED=0, or a model with more than two species). */
int b200md_nep_export_schedule(
  b200md_nep* p, int dims[6], int* d_seg_order, int* d_cell_start, void* stream);

/* Parity hook: the type tiles of the tensor-core hidden layer as of the last list rebuild.  Atoms are
 * bucketed by species in ascending order, each bucket padded to a multiple of 128 slots; d_slot[n] gets the
 * slot of every caller-order atom (tile = slot / 128), d_tile_type[b200md_nep_info(p, 8)] the species of
 * every tile.  Device pointers, each may be null.  Error when the handle has no tiles. */
int b200md_nep_export_tiles(b200md_nep* p, int* d_slot, int* d_tile_type, void* stream);
/* Parity hook: the hidden layer's output of the last compute call, in caller order whatever the storage:
 * d_fp[d*n + i] = dU/dq_d times q_scaler[d] (as the force kernels read it, d < descriptor dim) and
 * d_u[(t2*K + k)*n + i] = sum_m dU/dq_m c_radial(t_i, t2, m, k), the radial U table (K = basis_size_radial + 1
 * padded to 9, 13 or 17; zero beyond the model's basis).  Device pointers, each may be null.  Error on the
 * fused one- and two-species kernel, where neither reaches memory. */
int b200md_nep_export_mlp(b200md_nep* p, float* d_fp, float* d_u, void* stream);

/* synchronise and report latched device-side errors (B200MD_ERR_OVERFLOW) */
int b200md_nep_check(b200md_nep* p, void* stream);

/* Measurement hooks (no reference counterpart; the reference has no tracing, SURVEY.md 5).
 * b200md_nep_profile(p,1) makes every following b200md_nep_compute record CUDA events around each
 * stage on the launching stream (up to 256 calls); b200md_nep_profile_read synchronises and returns
 * the number of stages, filling ms_sum[stage] (total milliseconds) and counts[stage] (samples).
 * b200md_nep_mean_neighbors: mean skin / radial / angular list lengths of the last call. */
int b200md_nep_profile(b200md_nep* p, int enable);
int b200md_nep_profile_read(b200md_nep* p, int max_stages, float* ms_sum, int* counts);
const char* b200md_nep_stage_name(int stage);
int b200md_nep_mean_neighbors(b200md_nep* p, double out3[3]);

/* ------------------------------------------------------------------------------------------
 * LJ potential.  Replaces class LJ : Potential (src/force/lj.cuh:31-49):
 *   b200md_lj_create  <- LJ::LJ(FILE*, int num_types, int num_atoms), lj.cu:28-59
 *                        (the file is the whole potential file, first line "lj Nt sym...")
 *   b200md_lj_compute <- LJ::compute, lj.cu:184-219
 * ------------------------------------------------------------------------------------------ */
typedef struct b200md_lj b200md_lj;
int b200md_lj_create(const char* lj_txt_path, int num_atoms, b200md_lj** out);
void b200md_lj_destroy(b200md_lj* p);
double b200md_lj_rc(const b200md_lj* p);
int b200md_lj_info(const b200md_lj* p, int what); /* 0 num_types, 6 rebuild count */
const char* b200md_lj_symbol(const b200md_lj* p, int t);
int b200md_lj_compute(
  b200md_lj* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream);
int b200md_lj_check(b200md_lj* p, void* stream);
int b200md_lj_invalidate(b200md_lj* p, int n_new, void* stream); /* see b200md_nep_invalidate */

/* ------------------------------------------------------------------------------------------
 * Tersoff-1989 potential, FP64.  Replaces class Tersoff1989 : Potential
 * (src/force/tersoff1989.cuh, tersoff1989.cu:31-586):
 *   b200md_tersoff_create  <- Tersoff1989::Tersoff1989(FILE*, int num_types, int num_atoms), :31-150
 *                             (whole potential file: "tersoff_1989 Nt sym..." + 11 numbers per type
 *                             [+ chi]); 1 or 2 types
 *   b200md_tersoff_compute <- Tersoff1989::compute, :508-586 (local list + step1 + step2 +
 *                             find_properties_many_body, potential.cu:35-134)
 * b200md_compute_heat      <- compute_heat / gpu_compute_heat, src/measure/compute_heat.cu:32-90:
 *                             d_heat[5 * heat_stride] = jx_in, jx_out, jy_in, jy_out, jz per atom
 * ------------------------------------------------------------------------------------------ */
typedef struct b200md_tersoff b200md_tersoff;
int b200md_tersoff_create(const char* path, int num_atoms, b200md_tersoff** out);
void b200md_tersoff_destroy(b200md_tersoff* p);
double b200md_tersoff_rc(const b200md_tersoff* p);
int b200md_tersoff_info(const b200md_tersoff* p, int what); /* 0 num_types, 6 rebuild count */
const char* b200md_tersoff_symbol(const b200md_tersoff* p, int t);
int b200md_tersoff_compute(
  b200md_tersoff* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream);
int b200md_tersoff_invalidate(b200md_tersoff* p, int n_new, void* stream);
int b200md_tersoff_check(b200md_tersoff* p, void* stream);
int b200md_compute_heat(
  int n, int stride, const double* d_virial, const double* d_velocity, double* d_heat,
  int heat_stride, void* stream);

/* ------------------------------------------------------------------------------------------
 * Analytic EAM potentials.  Replaces class EAM : Potential (src/force/eam.cuh:20-90, eam.cu:28-580)
 * for `eam_zhou_2004` (1..18 types) and `eam_dai_2006` (1 type):
 *   b200md_eam_create  <- EAM::EAM(FILE*, char* name, int num_types, int num_atoms), eam.cu:28-44
 *   b200md_eam_compute <- EAM::compute, eam.cu:478-580 (step1 density/embedding, step2 forces)
 * ------------------------------------------------------------------------------------------ */
typedef struct b200md_eam b200md_eam;
int b200md_eam_create(const char* path, int num_atoms, b200md_eam** out);
void b200md_eam_destroy(b200md_eam* p);
double b200md_eam_rc(const b200md_eam* p);
int b200md_eam_info(const b200md_eam* p, int what); /* 0 num_types, 6 rebuild count */
const char* b200md_eam_symbol(const b200md_eam* p, int t);
int b200md_eam_compute(
  b200md_eam* p, int n, const double h[9], const int pbc[3], const int* d_type,
  const double* d_position, double* d_potential, double* d_force, double* d_virial, void* stream);
int b200md_eam_invalidate(b200md_eam* p, int n_new, void* stream);
int b200md_eam_check(b200md_eam* p, void* stream);

/* ------------------------------------------------------------------------------------------
 * Force::compute pre-steps (src/force/force.cu:771-801):
 *   b200md_apply_pbc        <- gpu_apply_pbc, force.cu:424-459
 *   b200md_zero_properties  <- initialize_properties, force.cu:314-333
 * ------------------------------------------------------------------------------------------ */
int b200md_apply_pbc(int n, const double h[9], const int pbc[3], double* d_position, void* stream);
int b200md_zero_properties(
  int n, double* d_potential, double* d_force, double* d_virial, void* stream);

/* ------------------------------------------------------------------------------------------
 * Integrator kernels behind Ensemble::compute1 / compute2 (src/integrate/ensemble.cuh:26-157):
 *   b200md_velocity_verlet <- Ensemble::velocity_verlet / gpu_velocity_verlet,
 *                             ensemble.cu:176-214,348-397 (the variant without groups)
 *   b200md_velocity_verlet_groups <- the variant with `fix` / `move` groups, ensemble.cu:111-174,
 *                             369-391: d_group_label = Group::label of the fixed grouping method
 *                             (device, n ints), fixed_group / move_group = -1 when unused,
 *                             move_velocity in natural units.  Atoms of either group keep zero
 *                             velocity; pass n_temperature = n - |fixed| - |move| to
 *                             b200md_find_thermo (ensemble.cu:645-651).
 *   b200md_find_thermo     <- Ensemble::find_thermo / gpu_find_thermo_instant_temperature,
 *                             ensemble.cu:434-673: d_thermo[0..7] = T,U,sxx,syy,szz,sxy,sxz,syz
 *   b200md_scale_velocity  <- Ensemble::scale_velocity_global, ensemble.cu:676-698
 * time_step is in GPUMD natural units (fs / 10.18051, src/utilities/common.cuh:26).
 * d_scratch for find_thermo: at least b200md_thermo_scratch_bytes(n) bytes of device memory.
 * ------------------------------------------------------------------------------------------ */
int b200md_velocity_verlet(
  int is_step1, int n, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, void* stream);
int b200md_velocity_verlet_groups(
  int is_step1, int n, int stride, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, const int* d_group_label, int fixed_group,
  int move_group, const double move_velocity[3], void* stream);
long long b200md_thermo_scratch_bytes(int n);
int b200md_find_thermo(
  int n, int n_temperature, double volume, const double* d_mass, const double* d_potential,
  const double* d_velocity, const double* d_virial, double* d_thermo8, void* d_scratch,
  void* stream);
int b200md_scale_velocity(int n, double factor, double* d_velocity, void* stream);

/* NVT thermostats (global velocity scaling).  `stride` as in the *_strided calls below (= n for a
 * single domain); d_thermo[0] must hold the instantaneous GLOBAL temperature (b200md_find_thermo,
 * all-reduced over ranks when sharded).  temperature_coupling = tau_T / time_step as in run.in.
 *   b200md_berendsen_temperature <- gpu_berendsen_temperature, src/integrate/ensemble_ber.cu:70-86
 *                                   (Ensemble_BER::compute2, :195-233)
 *   b200md_nhc_*                 <- Ensemble_NHC (src/integrate/ensemble_nhc.cu:31-50, 101-237):
 *                                   one call = find chain factor from d_thermo[0] + scale velocities,
 *                                   i.e. the thermostat half of integrate_nvt_nhc_1 / _2.  The chain
 *                                   is integrated on the device: no D2H copy per half step.
 *   b200md_bdp_*                 <- Ensemble_BDP, NVT branch (src/integrate/ensemble_bdp.cu:69-101,
 *                                   svr_utilities.cuh:27-135): stochastic velocity rescaling after
 *                                   the second half step.  The generator (std::mt19937 semantics)
 *                                   lives on the device; seed 12345678 reproduces the reference's
 *                                   -DDEBUG stream (ensemble_bdp.cu:31-32).  n_global counts the atoms
 *                                   that are integrated, N - N_fixed - N_move: ndeg = 3*n_global
 *                                   (ensemble_bdp.cu:87-95) must fit an int, as in the reference. */
int b200md_berendsen_temperature(
  int n, int stride, double temperature, double temperature_coupling, const double* d_thermo,
  double* d_velocity, void* stream);
typedef struct b200md_nhc b200md_nhc;
int b200md_nhc_create(
  long long n_global, double temperature, double temperature_coupling, double time_step,
  b200md_nhc** out);
void b200md_nhc_destroy(b200md_nhc* p);
int b200md_nhc_half_step(
  b200md_nhc* p, int n, int stride, double time_step, const double* d_thermo, double* d_velocity,
  void* stream);
typedef struct b200md_bdp b200md_bdp;
int b200md_bdp_create(
  long long n_global, double temperature, double temperature_coupling, unsigned seed,
  b200md_bdp** out);
void b200md_bdp_destroy(b200md_bdp* p);
int b200md_bdp_step(
  b200md_bdp* p, int n, int stride, const double* d_thermo, double* d_velocity, void* stream);

/* Heat-current autocorrelation, SURVEY.md 8f rank 4.  Replaces HAC::preprocess / process /
 * postprocess (src/measure/hac.cu:32-280):
 *   b200md_hac_create  <- preprocess: Nd = number_of_steps / sample_interval records of 5 components
 *   b200md_hac_sample  <- process: call every step; on (step+1) % sample_interval == 0 it runs
 *                         compute_heat (compute_heat.cu:32-90) and sums jx_in jx_out jy_in jy_out jz
 *   b200md_hac_finish  <- postprocess: hac[nc + Nc*k] (gpu_find_hac, :111-170) and the running thermal
 *                         conductivity rtc[nc + Nc*k] in W/mK (find_rtc, :173-181; factor dt/2/(kB T^2 V)
 *                         * 1.573769e5); host output arrays of 5*Nc doubles; time_step in natural units
 *   b200md_hac_series  <- the recorded heat-current series [nd + Nd*k] (5*Nd doubles, host) */
typedef struct b200md_hac b200md_hac;
int b200md_hac_create(int number_of_steps, int sample_interval, int Nc, b200md_hac** out);
void b200md_hac_destroy(b200md_hac* p);
int b200md_hac_sample(
  b200md_hac* p, int step, int n, int stride, const double* d_virial, const double* d_velocity,
  void* stream);
int b200md_hac_finish(
  b200md_hac* p, double time_step, double temperature, double volume, double* hac_out,
  double* rtc_out, void* stream);
int b200md_hac_series(b200md_hac* p, double* out, void* stream);

/* Homogeneous non-equilibrium MD (HNEMD) thermal conductivity, the rest of SURVEY.md 8f rank 4.
 *   b200md_hnemd_drive   <- Force::compute's compute_hnemd_ branch, src/force/force.cu:857-897 with
 *                           gpu_add_driving_force / gpu_sum_force / gpu_correct_force (:228-312):
 *                           f_i += W_i^T fe (virial map 0 3 4 / 6 1 5 / 7 8 2), then f_i -= sum_j f_j / n.
 *                           The per-atom add is the reference's bit for bit; only the order of the
 *                           total-force sum differs (fixed, so deterministic).  fe[3] (host) in 1/A;
 *                           d_scratch: b200md_hnemd_drive_scratch_bytes(n) bytes of device memory,
 *                           zeroed before the first call (no allocation per step; the reference
 *                           allocates ftot at every step, force.cu:880)
 *   b200md_hnemd_create  <- HNEMD::parse / preprocess, hnemd_kappa.cu:37-50, 149-184 (fe[3] host)
 *   b200md_hnemd_sample  <- HNEMD::process, :82-106: call every step; the heat current of all atoms
 *                           (compute_heat.cu:32-90) is summed straight into row step % output_interval
 *                           of a device buffer, without the 5N per-atom array
 *   b200md_hnemd_take    <- the output branch of HNEMD::process, :108-131: copies the finished interval
 *                           to the host (the only copy) and writes kappa5[k] = sum of the rows *
 *                           1.573769e5 / output_interval / (volume * temperature * |fe|) in W/mK, k =
 *                           xx_in xx_out yy_in yy_out zz; rows (may be NULL) gets the 5*output_interval
 *                           heat sums [m*5 + k] */
long long b200md_hnemd_drive_scratch_bytes(int n);
int b200md_hnemd_drive(
  int n, int stride, const double fe[3], const double* d_virial, double* d_force, void* d_scratch,
  void* stream);
typedef struct b200md_hnemd b200md_hnemd;
int b200md_hnemd_create(int output_interval, const double fe[3], b200md_hnemd** out);
void b200md_hnemd_destroy(b200md_hnemd* p);
int b200md_hnemd_sample(
  b200md_hnemd* p, int step, int n, int stride, const double* d_virial, const double* d_velocity,
  void* stream);
int b200md_hnemd_take(
  b200md_hnemd* p, double volume, double temperature, double* kappa5, double* rows, void* stream);

/* The same drive, heat sums and kappa for a system held in several arrays (libb200md_mgpu's blocks),
 * whose force total is combined by the caller and whose sampled step lives on the device:
 *   b200md_hnemd_drive_add      f_i += W_i^T fe for i < n (the per-atom add of b200md_hnemd_drive) and
 *                               the total of the new forces into d_ftot[3] (device); n = 0 is one
 *                               thread block that writes a zero total.  d_scratch as for
 *                               b200md_hnemd_drive (b200md_hnemd_drive_scratch_bytes(n), ticket zeroed)
 *   b200md_hnemd_drive_correct  f_i -= d_ftot[.] * one_over_n for i < n (gpu_correct_force with the
 *                               caller's 1.0 / N); n = 0 launches nothing.  b200md_hnemd_drive is
 *                               _add then _correct with 1.0 / n.
 *   b200md_hnemd_heat_row       the heat-current sum of atoms [0, n) (as b200md_hnemd_sample) into row
 *                               *d_row of d_rows[n_rows][5]; the kernel then sets *d_row = (*d_row + 1)
 *                               % n_rows on the device, so one captured launch serves every step.
 *                               d_scratch: b200md_hnemd_heat_row_scratch_bytes(n) bytes, zeroed before
 *                               the first call; n = 0 writes a zero row
 *   b200md_hnemd_kappa          kappa5 of one interval from its host rows[output_interval * 5], the
 *                               formula of b200md_hnemd_take */
int b200md_hnemd_drive_add(
  int n, int stride, const double fe[3], const double* d_virial, double* d_force, void* d_scratch,
  double* d_ftot, void* stream);
int b200md_hnemd_drive_correct(
  int n, int stride, double one_over_n, const double* d_ftot, double* d_force, void* stream);
long long b200md_hnemd_heat_row_scratch_bytes(int n);
int b200md_hnemd_heat_row(
  int n, int stride, const double* d_virial, const double* d_velocity, double* d_rows, int n_rows,
  unsigned int* d_row, void* d_scratch, void* stream);
int b200md_hnemd_kappa(
  int output_interval, double volume, double temperature, const double fe[3], const double* rows,
  double* kappa5);

/* Spectral heat current (SHC), on the time-correlation engine of DOS, SDC and MSD (b2_correlate.cu,
 * below).  Replaces SHC::parse / preprocess / process / postprocess (src/measure/shc.cu:34-542):
 *   b200md_shc_create  <- parse (:466-542) + preprocess (:34-79).  Output groups: num_groups sizes and
 *                         (host) contents, the atom indices of group 0, then group 1, ... (concatenated
 *                         in Group::find_contents order, group.cu:58-70).  contents = NULL: one group,
 *                         the atoms 0 .. group_sizes[0]-1 (no grouping).  `group m -1` passes groups
 *                         1 .. number-1 of method m.  Checks 1 <= sample_interval <= 50, 100 <= Nc <=
 *                         1000, direction 0..2, and that number_of_steps gives at least one time origin.
 *                         B200MD_ERR_CUDA, naming the size, when the device ring does not fit.
 *   b200md_shc_sample  <- process (:162-310): call every step.  Every sample_interval steps the virial
 *                         row of `direction` and the velocities of the groups go into a device ring;
 *                         the correlation is deferred and computed for blocks of time origins
 *   b200md_shc_finish  <- average_k + find_shc (:312-396), FP64 on the host: ki / ko [num_groups *
 *                         (2Nc-1)] (Hann-windowed, A eV/ps) and shc_i / shc_o [num_groups * num_omega]
 *                         (A eV), host arrays; time_step in natural units, max_omega in THz rad */
typedef struct b200md_shc b200md_shc;
int b200md_shc_create(
  int Nc, int sample_interval, int direction, int number_of_steps, int num_groups,
  const int* group_sizes, const int* contents, b200md_shc** out);
void b200md_shc_destroy(b200md_shc* p);
int b200md_shc_sample(
  b200md_shc* p, int step, int n, int stride, const double* d_virial, const double* d_velocity,
  void* stream);
int b200md_shc_finish(
  b200md_shc* p, double time_step, int num_omega, double max_omega, double* ki, double* ko,
  double* shc_i, double* shc_o, void* stream);

/* Time correlations of a per-atom 3-vector over Nc lags, on one engine with SHC above (b2_correlate.cu):
 *   b200md_dos_*  <- DOS (mass-weighted velocity autocorrelation, phonon DOS), src/measure/dos.cu:39-503
 *   b200md_sdc_*  <- SDC (velocity autocorrelation, self-diffusion coefficient), src/measure/sdc.cu:34-338
 *   b200md_msd_*  <- MSD (mean-square displacement of unwrapped positions), src/measure/msd.cu:52-542
 * _create  <- parse + preprocess (dos.cu:153-336, sdc.cu:132-155,300-338, msd.cu:205-267,481-542).
 *            Output groups as in b200md_shc_create: num_groups sizes and (host) contents concatenated
 *            in Group::find_contents order; contents = NULL: one group, the atoms 0 .. group_sizes[0]-1.
 *            `compute_dos ... group m -1` and `compute_msd ... all_groups m` pass every group of method m.
 *            time_step in natural units.  B200MD_ERR_ARG when Nc < 1 or sample_interval < 1, for the
 *            reference's checks (DOS: omega_max > 0, num_dos_points >= 1, the Nyquist check of
 *            dos.cu:286-288; MSD: Nc <= number_of_steps / sample_interval, msd.cu:217-219), and -- a
 *            deliberate divergence for DOS and SDC, where the reference divides by zero -- for a run that
 *            gives no time origin (number_of_steps / sample_interval < Nc).  B200MD_ERR_CUDA, naming the
 *            size, when the device ring of Nc + B - 1 frames does not fit.  DOS gathers the masses of the
 *            groups' atoms from d_mass[n] once, here (dos.cu:326-336).
 * _sample  <- process (dos.cu:220-245, sdc.cu:157-224, msd.cu:269-362): call every step with the
 *            velocities (DOS, SDC) or the unwrapped positions (MSD), [3][stride] SoA.  Every
 *            sample_interval steps the groups' vectors go into a device ring; from sample Nc - 1 on each
 *            sample is a time origin, correlated in deferred blocks with all Nc lags.  Asynchronous.
 * _finish  <- postprocess, FP64 on the host in the reference's order of operations; flushes the pending
 *            origins and synchronises.  Outputs are host arrays [group][component x y z][row]:
 *            DOS: mvac [g][3][Nc] normalised by its lag-0 value per group (dos.cu:414-427; 0 / 0 for an
 *                 empty group, as the reference) and dos [g][3][num_dos_points] after the Hann window and
 *                 cosine transform (dos.cu:450-481), in 1/THz per group of size N_g;
 *            SDC: vac [g][3][Nc] in A^2/ps^2 (scaled by 1 / (N_g origins)) and its running trapezoid
 *                 integral sdc [g][3][Nc] in A^2/ps (sdc.cu:239-285);
 *            MSD: msd [g][3][Nc] in A^2 and the finite-difference sdc [g][3][Nc] in A^2/ps, rows of zeros
 *                 for an empty group (msd.cu:369-445).  It may be called during the run (save_every): it
 *                 then covers every origin sampled so far.
 *            B200MD_ERR_ARG when no time origin has been sampled yet.
 * b200md_unwrap_begin / _end <- Integrate::compute1, integrate.cu:347-374: call _begin before the
 *            ensemble's first half step (copies d_position[3][n] to d_position_old) and _end after it
 *            (d_unwrapped += d_position - d_position_old).  Wrapping into the box happens later, in the
 *            force evaluation; a box scaling in the second half step does not reach d_unwrapped. */
typedef struct b200md_dos b200md_dos;
typedef struct b200md_sdc b200md_sdc;
typedef struct b200md_msd b200md_msd;
int b200md_dos_create(
  int Nc, int sample_interval, int number_of_steps, double time_step, double omega_max, int num_dos_points,
  int num_groups, const int* group_sizes, const int* contents, int n, const double* d_mass, b200md_dos** out);
void b200md_dos_destroy(b200md_dos* p);
int b200md_dos_sample(b200md_dos* p, int step, int n, int stride, const double* d_velocity, void* stream);
int b200md_dos_finish(b200md_dos* p, double* mvac, double* dos, void* stream);
int b200md_sdc_create(
  int Nc, int sample_interval, int number_of_steps, double time_step, int num_groups,
  const int* group_sizes, const int* contents, b200md_sdc** out);
void b200md_sdc_destroy(b200md_sdc* p);
int b200md_sdc_sample(b200md_sdc* p, int step, int n, int stride, const double* d_velocity, void* stream);
int b200md_sdc_finish(b200md_sdc* p, double* vac, double* sdc, void* stream);
int b200md_msd_create(
  int Nc, int sample_interval, int number_of_steps, double time_step, int num_groups,
  const int* group_sizes, const int* contents, b200md_msd** out);
void b200md_msd_destroy(b200md_msd* p);
int b200md_msd_sample(b200md_msd* p, int step, int n, int stride, const double* d_unwrapped, void* stream);
int b200md_msd_finish(b200md_msd* p, double* msd, double* sdc, void* stream);
int b200md_unwrap_begin(int n, const double* d_position, double* d_position_old, void* stream);
int b200md_unwrap_end(
  int n, const double* d_position, const double* d_position_old, double* d_unwrapped, void* stream);

/* Radial distribution function (b2_rdf.cu).  Replaces RDF::parse / preprocess / process / postprocess
 * (src/measure/rdf.cu:128-333, rdf.cuh:27-41):
 *   b200md_rdf_create   <- parse (:264-333) + preprocess (:163-176).  num_types species, the types with at
 *                          least one atom in ascending type id (type_index[], < 94), with num_atoms[] atoms
 *                          each, n atoms in all (the sum).  dr = rc / num_bins.  B200MD_ERR_ARG, with the
 *                          reference's message, for rc <= 0, num_bins <= 20 or > 500.  The box-thickness
 *                          check (:283-292) needs the box: a sample in a box with fewer than 5 cells of rc / 2
 *                          in a periodic direction returns B200MD_ERR_SMALL_BOX.
 *   b200md_rdf_sample   <- process (:178-202) + find_rdf (:128-161): one sample at these positions, with the
 *                          volume of box_h[9] (row-major, lattice vectors as columns); d_pos [3][n] SoA.  Each
 *                          unordered pair within rc is counted once into 64-bit integer bins and the sample
 *                          is folded into the FP64 accumulator on the device.  Asynchronous.
 *   b200md_rdf_finish   <- postprocess (:204-251): out[num_bins][1 + num_types (num_types + 1) / 2] = the
 *                          accumulated total and partial (a, b), a <= b, RDFs divided by num_repeats
 *                          (number_of_steps / interval; must be >= 1).  Synchronises; the only copy. */
typedef struct b200md_rdf b200md_rdf;
int b200md_rdf_create(
  double rc, int num_bins, int num_types, const int* type_index, const int* num_atoms, int n, b200md_rdf** out);
void b200md_rdf_destroy(b200md_rdf* p);
int b200md_rdf_sample(
  b200md_rdf* p, const double* box_h, const int* pbc, const int* d_type, const double* d_pos, int n, void* stream);
int b200md_rdf_finish(b200md_rdf* p, int num_repeats, double* out, void* stream);

/* Direct NEMD: heat source / sink baths and group averages.
 *   b200md_heat_bath_create  <- the heat branches of the Ensemble_LAN / _NHC / _BDP constructors
 *                               (ensemble_lan.cu:43-85, ensemble_nhc.cu:52-91, ensemble_bdp.cu:50-62).
 *                               kind 0 heat_lan (type 22), 1 heat_nhc (21), 2 heat_bdp (23).  Groups of
 *                               grouping method 0: num_groups sizes and (host) contents in
 *                               Group::find_contents order; source / sink are group ids.  The source
 *                               bath is at T + dT, the sink at T - dT.  Tc = tau_T / time_step.
 *                               heat_lan: cuRAND XORWOW states curand_init(seed_source, m, 0) for the m-th
 *                               source atom and curand_init(seed_sink, m, 0) for the m-th sink atom (the
 *                               reference passes its first and second rand(), ensemble_lan.cu:78-81);
 *                               heat_bdp: ONE std::mt19937 stream seeded with (unsigned)seed_source
 *                               (12345678 = the reference's -DDEBUG seed), source drawn before sink;
 *                               heat_nhc: two chains with Q[0] scaled by 3 |group|; seeds unused.
 *   b200md_heat_bath_half    <- integrate_heat_lan_half (ensemble_lan.cu:128-195; kick, no momentum
 *                               correction), integrate_heat_nhc_1 / _2 (ensemble_nhc.cu:239-326) and
 *                               integrate_heat_bdp_2 (ensemble_bdp.cu:103-149, after_vv2 only; a call with
 *                               after_vv2 = 0 does nothing).  Call it before velocity-Verlet step 1
 *                               (after_vv2 = 0) and after step 2 (after_vv2 = 1).  Asynchronous: the
 *                               group sums, chains, generator and the energy transferred stay on the
 *                               device.  No thermo is computed (the reference leaves it stale).
 *   b200md_heat_bath_energy  <- Ensemble::energy_transferred[2] (eV, source then sink); synchronises
 *   b200md_heat_bath_state   <- test hook, synchronises: out[44] = chain[2][12] (eta, v_eta, Q of the
 *                               source / sink chains), stat[2][5] (sum m, sum m v_xyz, sum m v^2 per group
 *                               before the last rescaling), vc[2][3], factor[2], energy[2]
 *   b200md_group_compute_*   <- Compute (compute.cu:31-660).  what_mask: B200MD_COMPUTE_* bits; the
 *                               columns come in the reference's fixed order (temperature, potential,
 *                               force x3, virial x9 as xx xy xz yx yy yz zx zy zz, jp x3, jk x3,
 *                               momentum x3), each a block of num_groups values.  _sample adds one sample
 *                               (call it on the sampling steps only) into a device running sum with a
 *                               fixed-order segmented reduction; _take (synchronises) writes the
 *                               columns * num_groups averages over num_samples samples (temperature also
 *                               divided by the group size, compute.cu:540-561) and resets the sum. */
#define B200MD_COMPUTE_TEMPERATURE 1
#define B200MD_COMPUTE_POTENTIAL 2
#define B200MD_COMPUTE_FORCE 4
#define B200MD_COMPUTE_VIRIAL 8
#define B200MD_COMPUTE_JP 16
#define B200MD_COMPUTE_JK 32
#define B200MD_COMPUTE_MOMENTUM 64
#define B200MD_COMPUTE_ALL 127
typedef struct b200md_heat_bath b200md_heat_bath;
int b200md_heat_bath_create(
  int kind, int n, int num_groups, const int* group_sizes, const int* contents, int source, int sink,
  double T, double Tc, double dT, double time_step, unsigned long long seed_source,
  unsigned long long seed_sink, b200md_heat_bath** out);
void b200md_heat_bath_destroy(b200md_heat_bath* p);
int b200md_heat_bath_half(
  b200md_heat_bath* p, int after_vv2, int n, int stride, const double* d_mass, double* d_velocity,
  void* stream);
int b200md_heat_bath_energy(b200md_heat_bath* p, double out2[2], void* stream);
int b200md_heat_bath_state(b200md_heat_bath* p, double* out44, void* stream);
typedef struct b200md_group_compute b200md_group_compute;
int b200md_group_compute_create(
  int n, int num_groups, const int* group_sizes, const int* contents, unsigned what_mask,
  b200md_group_compute** out);
void b200md_group_compute_destroy(b200md_group_compute* p);
int b200md_group_compute_columns(const b200md_group_compute* p); /* -1 for a null handle */
int b200md_group_compute_sample(
  b200md_group_compute* p, int n, int stride, const double* d_mass, const double* d_potential,
  const double* d_force, const double* d_virial, const double* d_velocity, void* stream);
int b200md_group_compute_take(b200md_group_compute* p, int num_samples, double* out, void* stream);

/* Langevin thermostats and the Berendsen barostat (SURVEY.md 8f rank 3):
 *   b200md_langevin_*         <- curand states + gpu_langevin + momentum correction,
 *                                src/integrate/langevin_utilities.cuh:26-127; one apply() = one
 *                                Ensemble_LAN::integrate_nvt_lan_half (ensemble_lan.cu:92-124, c1 =
 *                                exp(-0.5/Tc)) or Ensemble_BAO::integrate_nvt_lan (ensemble_bao.cu:91-120,
 *                                c1 = exp(-1/Tc)); c2 = sqrt((1-c1^2) k_B T).  cuRAND XORWOW,
 *                                curand_init(seed, atom, 0): seed 1804289383 (glibc's first rand())
 *                                reproduces the stream of the reference's -DDEBUG build when model.xyz
 *                                carries the velocities.
 *   b200md_baoab_operator     <- gpu_operator_A (which = 0) / gpu_operator_B (which = 1),
 *                                ensemble_bao.cu:190-300; d_group_label may be NULL (fixed_group -1)
 *   b200md_berendsen_pressure <- Ensemble_BER::compute2, NPT branch (ensemble_ber.cu:88-172,237-285):
 *                                num_components 1 (isotropic), 3 (orthogonal, optional deform) or 6
 *                                (triclinic, Voigt order); target_pressure / pressure_coupling in
 *                                natural units as integrate.cu:1150-1153 leaves them; h[9] (HOST) is
 *                                updated in place, positions are scaled on the device.  Reads
 *                                d_thermo[2..7] back, i.e. synchronises the stream, as the reference. */
typedef struct b200md_langevin b200md_langevin;
int b200md_langevin_create(int n, unsigned long long seed, b200md_langevin** out);
void b200md_langevin_destroy(b200md_langevin* p);
int b200md_langevin_apply(
  b200md_langevin* p, int n, int stride, double c1, double c2, const double* d_mass,
  double* d_velocity, void* stream);
int b200md_baoab_operator(
  int which, int n, int stride, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, const int* d_group_label, int fixed_group, void* stream);
int b200md_berendsen_pressure(
  int n, int stride, int num_components, const double target_pressure[6],
  const double pressure_coupling[6], const int deform[3], const double deform_rate[3],
  const int pbc[3], double h[9], const double* d_thermo, double* d_position, void* stream);

/* ------------------------------------------------------------------------------------------
 * Spatial-domain sharding (replaces the hub-and-spoke scatter/gather of NEP_MULTIGPU,
 * src/force/nep_multigpu.cu:1249-1310,1552-1582,1764-1802).  A rank keeps ONE set of local SoA
 * arrays of length `stride` = owned + ghost atoms; the first n entries are owned.  The *_strided
 * variants act on the owned part in place; b200md_halo_pack gathers the positions a neighbour
 * domain needs (out[d*m + k] = position[d*stride + index[k]] + shift[d]) into a send buffer for
 * ncclSend/Recv.  Thermo: call b200md_find_thermo_strided with the GLOBAL n_temperature and
 * volume; the 8 outputs are then additive over ranks (ncclAllReduce SUM).
 * b200md_nep_invalidate: the caller changed the local atom set/order (migration): drop the cell
 * order and lists; n_new <= the num_atoms given at creation.
 * ------------------------------------------------------------------------------------------ */
int b200md_apply_pbc_strided(
  int n, int stride, const double h[9], const int pbc[3], double* d_position, void* stream);
int b200md_velocity_verlet_strided(
  int is_step1, int n, int stride, double time_step, const double* d_mass, double* d_position,
  double* d_velocity, const double* d_force, void* stream);
int b200md_find_thermo_strided(
  int n, int stride, int n_temperature, double volume, const double* d_mass,
  const double* d_potential, const double* d_velocity, const double* d_virial, double* d_thermo8,
  void* d_scratch, void* stream);
int b200md_halo_pack(
  int m, const int* d_index, int stride, const double* d_position, const double shift[3],
  double* d_out, void* stream);
int b200md_nep_invalidate(b200md_nep* p, int n_new, void* stream);
/* Only the atoms with caller index < n_owned receive energy / force / virial from the following
 * b200md_nep_compute calls (0 = all atoms, the default): in a spatial domain the rest are ghosts,
 * whose results the owner rank computes and the local rank would discard
 * (cf. nep_multigpu.cu:1764-1802, which copies back the owned range only). */
int b200md_nep_set_owned(b200md_nep* p, int n_owned);
/* accumulate = 1 (default): outputs are ADDED to the caller's arrays, the contract of Potential::compute
 * (nep.cu:653,755-770; Force::compute zeroes them first, force.cu:794-801).  accumulate = 0: they are
 * OVERWRITTEN, so a driver with a single potential can drop its zeroing pass and the final kernel its
 * read-modify-write (208 bytes per atom and step).  The setting, like set_owned and
 * set_active_region, holds for every later call on the handle, small boxes (supercell path) and
 * changes of the atom count included. */
int b200md_nep_set_accumulate(b200md_nep* p, int accumulate);
/* Atoms whose position (in the coordinates passed to b200md_nep_compute) lies outside [lo, hi) get
 * EMPTY radial / angular neighbour sets from the following calls: no descriptor, dU/dq or partial-
 * force work is spent on them, they only serve as neighbours of the others.  A spatial domain sets
 * this to its owned region grown by rc + skin: ghosts further away cannot be a neighbour of an owned
 * atom, so nothing an owned atom's force depends on is skipped (the reference recomputes descriptors
 * for its whole ghost layer, nep_multigpu.cu:1476-1545).  lo = hi = NULL switches it off.  A small
 * periodic box (supercell path of b200md_nep_compute) ignores the region: the image atoms of its
 * supercell lie outside the caller's coordinates and need their descriptors. */
int b200md_nep_set_active_region(b200md_nep* p, const double lo[3], const double hi[3]);

/* ------------------------------------------------------------------------------------------
 * Energy minimization.  Replaces Minimize::parse_minimize's minimizers (src/minimize/minimize.cu:32-156):
 *   b200md_minimizer_create     <- Minimizer_SD / Minimizer_FIRE / Minimizer_FIRE_Box_Change constructors
 *                                  (minimizer.cuh:27-50, minimizer_fire.cuh:24-45,
 *                                  minimizer_fire_box_change.cuh:24-53).  method 0 sd, 1 fire; box_change
 *                                  and hydrostatic (0 / 1) for fire only.  The handle owns the FIRE velocity
 *                                  (zero at creation), the control record and the reduction scratch; nothing
 *                                  is allocated after creation.
 *   b200md_minimizer_sd_begin   <- the start of Minimizer_SD::compute (minimizer_sd.cu:77-118): call after the
 *                                  first force evaluation of (d_position, d_force, d_potential).  Reduces f_max
 *                                  and sum U, then writes the trial positions x + F step / f_max to
 *                                  d_position_trial (the atoms of label fixed_group keep x; fixed_group -1 and
 *                                  d_group_label NULL: none).  The caller evaluates the force at the trial
 *                                  positions into d_force_trial / d_potential_trial (the reference's _temp
 *                                  vectors, minimizer.cuh:38-40; caller-owned, 3n / 3n / n doubles).
 *   b200md_minimizer_sd_step    <- the rest of one SD iteration (minimizer_sd.cu:122-137): sum U_trial; uphill
 *                                  (U_trial > U) -> step *= 0.2, else the trial x, F, U are copied over the
 *                                  caller's on the device and step *= 1.2; then f_max and sum U of the new
 *                                  state and the next trial positions.
 *   b200md_minimizer_fire_step  <- one iteration of Minimizer_FIRE::compute (minimizer_fire.cu:108-180) or
 *                                  Minimizer_FIRE_Box_Change::compute (minimizer_fire_box_change.cu:239-406),
 *                                  after the caller's force evaluation: f_max, sum U, P = v.F, |F|, |v| (and the
 *                                  virial box force) in one reduction, the FIRE control step on the device, and
 *                                  one update pass over the atoms (nothing moves once converged).  Box change:
 *                                  h[9] (HOST) is updated in place to h + dEps h, as b200md_berendsen_pressure
 *                                  does, and L = cbrt(volume) is taken from h at the first call.
 * Each call writes the handle's record (B200MD_MIN_RECORD doubles) to `record` (host, may be NULL for the SD
 * calls): the only device-to-host copy of an iteration, which synchronises the stream.
 *   b200md_minimizer_velocity    the FIRE velocity, device double[3n] (SoA)
 *   b200md_minimizer_set_record  test hook: overwrite the record (the control state dt, alpha, N_neg, step,
 *                                v_box and, when > 0, L)
 * ------------------------------------------------------------------------------------------ */
#define B200MD_MIN_FMAX 0      /* sqrt(max F_i^2) over the atom force components of the current state */
#define B200MD_MIN_U 1         /* sum U of the current state (eV) */
#define B200MD_MIN_CONVERGED 2 /* 1: f_max < tol (box change: and the stress below 1e-4 GPa) */
#define B200MD_MIN_DT 3        /* FIRE time step (natural units) after the control step */
#define B200MD_MIN_ALPHA 4
#define B200MD_MIN_NNEG 5      /* FIRE's count of P > 0 iterations since the last uphill one */
#define B200MD_MIN_P 6         /* v.F before the control step (box change: over the 3N + 9 entries) */
#define B200MD_MIN_FMOD 7      /* |F| (generalized for box change) */
#define B200MD_MIN_VMOD 8      /* |v| after the possible zeroing, before the kick */
#define B200MD_MIN_UPHILL 9    /* FIRE: P <= 0 branch taken; SD: the trial was rejected */
#define B200MD_MIN_PRESSURE 10 /* box change: trace of the stress / 3 (GPa) */
#define B200MD_MIN_STRESS 11   /* box change: max |stress component| (hydrostatic: |pressure|), GPa */
#define B200MD_MIN_STEP 12     /* SD position step (starts at 0.1) */
#define B200MD_MIN_UTRIAL 13   /* SD: sum U at the trial positions */
#define B200MD_MIN_USMALLER 14 /* SD: the lower of sum U and sum U_trial of the last decision */
#define B200MD_MIN_SCALE 15    /* FIRE: alpha |v| / |F|; SD: step / f_max */
#define B200MD_MIN_LSCALE 16   /* box change: L = cbrt(V0) */
#define B200MD_MIN_DEPS 17     /* box change: dEps[9] = v_box dt / L, row-major */
#define B200MD_MIN_VBOX 26     /* box change: v_box[9] */
#define B200MD_MIN_FBOX 35     /* box change: the box force[9] = virial / L (hydrostatic: trace / 3) */
#define B200MD_MIN_RECORD 44
typedef struct b200md_minimizer b200md_minimizer;
int b200md_minimizer_create(
  int method, int n, double force_tolerance, int number_of_steps, int box_change, int hydrostatic,
  b200md_minimizer** out);
void b200md_minimizer_destroy(b200md_minimizer* p);
double* b200md_minimizer_velocity(b200md_minimizer* p);
int b200md_minimizer_set_record(b200md_minimizer* p, const double* record, void* stream);
int b200md_minimizer_sd_begin(
  b200md_minimizer* p, int n, double* d_position, double* d_force, double* d_potential,
  double* d_position_trial, const double* d_force_trial, const double* d_potential_trial,
  const int* d_group_label, int fixed_group, double* record, void* stream);
int b200md_minimizer_sd_step(
  b200md_minimizer* p, int n, double* d_position, double* d_force, double* d_potential,
  double* d_position_trial, const double* d_force_trial, const double* d_potential_trial,
  const int* d_group_label, int fixed_group, double* record, void* stream);
int b200md_minimizer_fire_step(
  b200md_minimizer* p, int n, double h[9], double* d_position, const double* d_force,
  const double* d_potential, const double* d_virial, double* record, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Harmonic phonons.  Replaces Hessian::compute (src/phonon/hessian.cu:65-81):
 *   b200md_phonon_create     <- Hessian::initialize's allocations (hessian.cu:200-253): n atoms, num_basis
 *                               basis atoms (atoms 0 .. num_basis-1; atom n has the label n % num_basis),
 *                               num_kpoints Cartesian k-points kpoints[3 * num_kpoints] (1 / A), the
 *                               displacement d (A).  1 <= num_basis <= B200MD_PHONON_MAX_BASIS.
 *   b200md_phonon_begin      <- the start of Hessian::find_H (hessian.cu:272-302): saves the positions and the
 *                               num_basis masses, computes r12 = x[n2] - x[n1] under the minimum image of
 *                               box (h, pbc) for every basis atom n1 and atom n2 and the mask r12^2 <= cutoff^2
 *                               (Hessian::is_too_far, hessian.cu:255-270), then displaces the position for the
 *                               first force call.
 *   b200md_phonon_step       <- find_H12 (src/force/force_constant.cu:80-133), one step per force call
 *                               call = 0 .. 6 num_basis - 1, made with the positions the previous step left.
 *                               Call j displaces basis atom j / 6 along a = (j % 6) / 2 by -d (j even) or +d
 *                               (j odd); one kernel keeps F(-) or writes H[n1][n2][a*3+b] =
 *                               (F_n2^b(-) - F_n2^b(+)) / 2d (0 beyond the cutoff), then sets the position for
 *                               the next call from the saved copy.  After the last call the positions are the
 *                               saved ones, bit for bit.  No host synchronisation.
 *   b200md_phonon_dynamical  <- the D(k) sums of find_dispersion (hessian.cu:391-419); with one k-point those
 *                               of find_D (hessian.cu:431-458): real, no phase.  D is column-major per k-point
 *                               (entry (row, col) at k * dim^2 + col * dim + row, dim = 3 num_basis).
 *   b200md_phonon_eig        <- eig_hermitian_Jacobi_batch / eig_hermitian_QR (hessian.cu:347-374): the
 *                               eigenvalues of every D(k) from its lower triangle, ascending; with one k-point
 *                               eigenvectors_symmetric_Jacobi (hessian.cu:460-492): eigenvalues and
 *                               eigenvectors of the real D.  Natural units (eV / A^2 / amu).  Synchronises the
 *                               stream and returns B200MD_ERR_NOT_CONVERGED when a matrix is not diagonal after
 *                               the solver's sweep cap.
 *   b200md_phonon_read       copies one array to host memory and synchronises the stream.  what:
 *                               B200MD_PHONON_H  H [num_basis][n][9];
 *                               B200MD_PHONON_D_REAL, _D_IMAG  D [num_kpoints][dim][dim], column-major per k-point
 *                                 (the imaginary part for num_kpoints > 1 only);
 *                               B200MD_PHONON_W  eigenvalues [num_kpoints][dim];
 *                               B200MD_PHONON_V  eigenvectors [dim][dim], column-major, as columns
 *                                 (num_kpoints == 1 only).
 *   b200md_jacobi_eig        the eigensolver on `batch` column-major dim x dim matrices (lower triangle
 *                            read): hermitian 1 -> eigenvalues d_w[batch][dim] of re + i im; hermitian 0 ->
 *                            eigenvalues of re and, when d_v is given, eigenvectors d_v[batch][dim][dim].
 *                            d_info[batch] (device) gets the sweeps each matrix took, or -1 when it was not
 *                            diagonal after the sweep cap.  One CTA per matrix, cyclic Jacobi in shared memory;
 *                            1 <= dim <= 96.  Asynchronous.
 * ------------------------------------------------------------------------------------------- */
#define B200MD_PHONON_MAX_BASIS 32
typedef struct b200md_phonon b200md_phonon;
int b200md_phonon_create(
  int n, int num_basis, int num_kpoints, const double* kpoints, double displacement, b200md_phonon** out);
void b200md_phonon_destroy(b200md_phonon* p);
int b200md_phonon_begin(
  b200md_phonon* p, int n, const double h[9], const int pbc[3], double cutoff, double* d_position,
  const double* d_mass, void* stream);
int b200md_phonon_step(b200md_phonon* p, int call, double* d_position, const double* d_force, void* stream);
int b200md_phonon_dynamical(b200md_phonon* p, void* stream);
int b200md_phonon_eig(b200md_phonon* p, void* stream);
#define B200MD_PHONON_H 0
#define B200MD_PHONON_D_REAL 1
#define B200MD_PHONON_D_IMAG 2
#define B200MD_PHONON_W 3
#define B200MD_PHONON_V 4
int b200md_phonon_read(b200md_phonon* p, int what, double* host, void* stream);
int b200md_jacobi_eig(
  int dim, int batch, int hermitian, const double* d_re, const double* d_im, double* d_w, double* d_v,
  int* d_info, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Tensor-core self-test (no reference counterpart): one CTA computes D[128 x N] = A[128 x K] .
 * B[N x K]^T on the tensor cores (one warpgroup, wgmma.mma_async tf32, 3xTF32 split, FP32
 * register accumulators) exactly as the NEP hidden-layer kernel issues it.  Row-major device
 * arrays; 16 <= N <= 256, N % 16 == 0, K % 8 == 0; layout 0 / 1 = the two shared-memory operand
 * arrangements of b2_tc.cuh (1 is the hidden layer's).  Used by tests/ to validate the descriptor
 * and accumulator-fragment plumbing against a host GEMM.
 * ------------------------------------------------------------------------------------------- */
int b200md_tc_selftest(
  int layout, int N, int K, const float* d_A, const float* d_B, float* d_D, void* stream);

#ifdef __cplusplus
}
#endif
#endif

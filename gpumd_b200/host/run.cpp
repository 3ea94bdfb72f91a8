// run.cpp -- standalone driver `b200md`: reads GPUMD's own input files from the current directory
// (run.in keyword script, model.xyz extended XYZ, potential file) and runs the hot path through the
// adapter classes, writing thermo.out in the reference's format.
//
// Mirrors, for the keywords of the hot path only:
//   Run::Run / execute_run_in / parse_one_keyword   src/main_gpumd/run.cu:144-209, 343-575
//   Run::perform_a_run (the MD loop)                src/main_gpumd/run.cu:211-341
//   initialize_position (model.xyz)                 src/model/read_xyz.cu:145-425, 482-557
//   Velocity::initialize                            src/main_gpumd/velocity.cu:55-75, 312-347
//   Dump_Thermo                                     src/measure/dump_thermo.cu:57-129
//   Dump_XYZ (extended XYZ)                         src/measure/dump_xyz.cu:68-437
//   Dump_Restart (restart.xyz)                      src/measure/dump_restart.cu:66-140
//   Replicate                                       src/main_gpumd/replicate.cu:20-111
// Keywords: replicate <na nb nc>, potential, velocity <T> [seed <s>], ensemble nve |
// nvt_ber|nvt_nhc|nvt_bdp T T tau, time_step <fs>, dump_thermo <n>, dump_xyz <n> <file> [precision
// single|double] [mass velocity force potential virial], dump_restart <n>, compute_hac, compute_hnemd,
// compute_shc, ensemble heat_lan|heat_nhc|heat_bdp T Tc dT source sink, compute, compute_dos,
// compute_sdc, compute_msd, run <n>.  Anything else is an input error (exit 1), as in the reference.
#include "ensemble.h"
#include "force.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>

static const double K_B = 8.617343e-5;                     // common.cuh:21
static const double TIME_UNIT_CONVERSION = 1.018051e+1;    // common.cuh:26
static const double PRESSURE_UNIT_CONVERSION = 1.602177e+2; // common.cuh:25

#include "element_mass.h" // the reference's full MASS_TABLE (read_xyz.cu:36-142)

static bool element_mass(const std::string& symbol, double* mass)
{
  for (int k = 0; k < NUM_ELEMENT_MASS; ++k)
    if (symbol == ELEMENT_MASS[k].symbol) {
      *mass = ELEMENT_MASS[k].mass;
      return true;
    }
  return false;
}

[[noreturn]] static void input_error(const std::string& msg)
{
  fprintf(stderr, "Input Error:\n    %s\n", msg.c_str());
  exit(1);
}

// is_valid_int / is_valid_real, src/utilities/read_file.cu: the whole token must be the number
static bool valid_int(const std::string& s, int* v)
{
  char* end = nullptr;
  const long x = std::strtol(s.c_str(), &end, 10);
  if (s.empty() || *end != '\0' || x < -2147483647L || x > 2147483647L)
    return false;
  *v = (int)x;
  return true;
}

static bool valid_real(const std::string& s, double* v)
{
  char* end = nullptr;
  const double x = std::strtod(s.c_str(), &end);
  if (s.empty() || *end != '\0')
    return false;
  *v = x;
  return true;
}

static std::string lower(std::string s)
{
  std::transform(s.begin(), s.end(), s.begin(), ::tolower);
  return s;
}

// value of key="..." or key=token on the comment line (case-insensitive key), "" if absent
static std::string header_value(const std::string& line, const std::string& key)
{
  const std::string low = lower(line);
  size_t p = low.find(key + "=");
  if (p == std::string::npos)
    return "";
  p += key.size() + 1;
  if (p < line.size() && line[p] == '"') {
    const size_t q = line.find('"', p + 1);
    return line.substr(p + 1, q - p - 1);
  }
  const size_t q = line.find_first_of(" \t", p);
  return line.substr(p, q == std::string::npos ? std::string::npos : q - p);
}

struct Model {
  Box box;
  Atom atom;
  std::vector<Group> group; // one entry per grouping method of model.xyz (group:I:k)
  bool has_velocity = false;
};

static void read_model(const char* path, Model& m)
{
  std::ifstream in(path);
  if (!in.is_open())
    input_error("Failed to open model.xyz.");
  std::string line;
  std::getline(in, line);
  const int N = std::atoi(line.c_str());
  if (N < 1)
    input_error("Number of atoms should be positive.");
  std::getline(in, line);
  std::string lat = header_value(line, "lattice");
  if (lat.empty())
    input_error("'lattice' is missing in the second line of model.xyz.");
  {
    std::istringstream ss(lat);
    double a[9];
    for (double& v : a)
      ss >> v;
    // stored transposed: lattice vectors become the columns of cpu_h (read_xyz.cu:203-219)
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        m.box.cpu_h[r * 3 + c] = a[c * 3 + r];
  }
  const std::string pbc = header_value(line, "pbc");
  if (!pbc.empty()) {
    std::istringstream ss(pbc);
    std::string t[3];
    ss >> t[0] >> t[1] >> t[2];
    m.box.pbc_x = (t[0] == "T" || t[0] == "t");
    m.box.pbc_y = (t[1] == "T" || t[1] == "t");
    m.box.pbc_z = (t[2] == "T" || t[2] == "t");
  }
  // properties=species:S:1:pos:R:3[:mass:R:1][:vel:R:3] -> column offsets
  std::string props = lower(header_value(line, "properties"));
  if (props.empty())
    props = "species:s:1:pos:r:3";
  int off_species = -1, off_pos = -1, off_mass = -1, off_vel = -1, off_group = -1, num_group = 0, col = 0;
  {
    std::istringstream ss(props);
    std::string name, kind, width;
    while (std::getline(ss, name, ':') && std::getline(ss, kind, ':') && std::getline(ss, width, ':')) {
      const int w = std::atoi(width.c_str());
      if (name == "species")
        off_species = col;
      else if (name == "pos")
        off_pos = col;
      else if (name == "mass")
        off_mass = col;
      else if (name == "vel")
        off_vel = col;
      else if (name == "group") { // group:I:k = k grouping methods (read_xyz.cu:271-287)
        off_group = col;
        num_group = w;
      }
      col += w;
    }
  }
  if (off_species < 0 || off_pos < 0)
    input_error("'species' or 'pos' is missing in properties.");
  Atom& a = m.atom;
  a.number_of_atoms = N;
  a.cpu_atom_symbol.resize(N);
  a.cpu_mass.resize(N);
  a.cpu_position_per_atom.resize((size_t)3 * N);
  a.cpu_velocity_per_atom.assign((size_t)3 * N, 0.0);
  m.has_velocity = off_vel >= 0;
  m.group.resize(num_group);
  for (Group& g : m.group)
    g.cpu_label.assign(N, 0);
  for (int n = 0; n < N; ++n) {
    if (!std::getline(in, line))
      input_error("model.xyz ended early.");
    std::istringstream ss(line);
    std::vector<std::string> tok;
    std::string w;
    while (ss >> w)
      tok.push_back(w);
    if ((int)tok.size() < col)
      input_error("Number of items in an atom line is too small.");
    a.cpu_atom_symbol[n] = tok[off_species];
    for (int d = 0; d < 3; ++d)
      a.cpu_position_per_atom[n + (size_t)N * d] = std::atof(tok[off_pos + d].c_str());
    if (off_mass >= 0) {
      a.cpu_mass[n] = std::atof(tok[off_mass].c_str());
    } else {
      if (!element_mass(tok[off_species], &a.cpu_mass[n]))
        input_error("Atom symbol " + tok[off_species] + " is not in the mass table.");
    }
    if (off_vel >= 0)
      for (int d = 0; d < 3; ++d) // A/fs -> natural units (read_xyz.cu:380-387)
        a.cpu_velocity_per_atom[n + (size_t)N * d] =
          std::atof(tok[off_vel + d].c_str()) * TIME_UNIT_CONVERSION;
    for (int g = 0; g < num_group; ++g) { // read_xyz.cu:389-398
      const int label = std::atoi(tok[off_group + g].c_str());
      if (label < 0 || label >= N)
        input_error("Group label should >= 0 and < N.");
      m.group[g].cpu_label[n] = label;
      if (label + 1 > m.group[g].number)
        m.group[g].number = label + 1;
    }
  }
  for (Group& g : m.group) {
    g.cpu_size.assign(g.number, 0);
    for (int n = 0; n < N; ++n)
      g.cpu_size[g.cpu_label[n]]++;
    g.cpu_size_sum.assign(g.number, 0);
    for (int k = 1; k < g.number; ++k)
      g.cpu_size_sum[k] = g.cpu_size_sum[k - 1] + g.cpu_size[k - 1];
    g.contents.assign(N, 0);
    std::vector<int> fill(g.cpu_size_sum);
    for (int n = 0; n < N; ++n)
      g.contents[fill[g.cpu_label[n]]++] = n;
    g.label.resize(N);
    g.label.copy_from_host(g.cpu_label.data());
  }
}

// Velocity::initialize (velocity.cu:55-75, 312-347): uniform random velocities from rand().  Like the
// reference's -DDEBUG build (main_common.cu:30-35: no srand, a release build seeds from the clock)
// this driver never seeds the stream unless `seed` is given, so `velocity T` is reproducible.  Then
// Velocity::correct_velocity (:77-270: zero linear momentum, then remove the rigid rotation
// w = I^-1 L about the centre of mass unless the inertia tensor is singular), then scale to T (:38-53).
static void initialize_velocity(Atom& a, double temperature, bool use_seed, int seed)
{
  const int N = a.number_of_atoms;
  double* vx = a.cpu_velocity_per_atom.data();
  double* vy = vx + N;
  double* vz = vy + N;
  const double* x = a.cpu_position_per_atom.data();
  const double* y = x + N;
  const double* z = y + N;
  const double* m = a.cpu_mass.data();
  for (int n = 0; n < N; ++n) {
    if (use_seed)
      srand((unsigned)seed + n * 3);
    vx[n] = -1.0 + (rand() * 2.0) / RAND_MAX;
    if (use_seed)
      srand((unsigned)seed + n * 3 + 1);
    vy[n] = -1.0 + (rand() * 2.0) / RAND_MAX;
    if (use_seed)
      srand((unsigned)seed + n * 3 + 2);
    vz[n] = -1.0 + (rand() * 2.0) / RAND_MAX;
  }
  // linear momentum
  double p[3] = {0, 0, 0}, mt = 0;
  for (int n = 0; n < N; ++n) {
    mt += m[n];
    p[0] += m[n] * vx[n];
    p[1] += m[n] * vy[n];
    p[2] += m[n] * vz[n];
  }
  for (int n = 0; n < N; ++n) {
    vx[n] -= p[0] / mt;
    vy[n] -= p[1] / mt;
    vz[n] -= p[2] / mt;
  }
  // angular momentum about the centre of mass
  double r0[3] = {0, 0, 0};
  for (int n = 0; n < N; ++n) {
    r0[0] += x[n] * m[n];
    r0[1] += y[n] * m[n];
    r0[2] += z[n] * m[n];
  }
  for (double& c : r0)
    c /= mt;
  double L[3] = {0, 0, 0}, I[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (int n = 0; n < N; ++n) {
    const double dx = x[n] - r0[0], dy = y[n] - r0[1], dz = z[n] - r0[2];
    L[0] += m[n] * (dy * vz[n] - dz * vy[n]);
    L[1] += m[n] * (dz * vx[n] - dx * vz[n]);
    L[2] += m[n] * (dx * vy[n] - dy * vx[n]);
    I[0][0] += m[n] * (dy * dy + dz * dz);
    I[1][1] += m[n] * (dx * dx + dz * dz);
    I[2][2] += m[n] * (dx * dx + dy * dy);
    I[0][1] -= m[n] * dx * dy;
    I[1][2] -= m[n] * dy * dz;
    I[0][2] -= m[n] * dx * dz;
  }
  I[1][0] = I[0][1];
  I[2][1] = I[1][2];
  I[2][0] = I[0][2];
  const double det = I[0][0] * I[1][1] * I[2][2] + I[0][1] * I[1][2] * I[2][0] +
                     I[0][2] * I[1][0] * I[2][1] - I[0][0] * I[1][2] * I[2][1] -
                     I[0][1] * I[1][0] * I[2][2] - I[2][0] * I[1][1] * I[0][2];
  if (!(det > -1.0e-10 && det < 1.0e-10)) {
    double inv[3][3];
    inv[0][0] = I[1][1] * I[2][2] - I[1][2] * I[2][1];
    inv[0][1] = -(I[0][1] * I[2][2] - I[0][2] * I[2][1]);
    inv[0][2] = I[0][1] * I[1][2] - I[0][2] * I[1][1];
    inv[1][0] = -(I[1][0] * I[2][2] - I[1][2] * I[2][0]);
    inv[1][1] = I[0][0] * I[2][2] - I[0][2] * I[2][0];
    inv[1][2] = -(I[0][0] * I[1][2] - I[0][2] * I[1][0]);
    inv[2][0] = I[1][0] * I[2][1] - I[1][1] * I[2][0];
    inv[2][1] = -(I[0][0] * I[2][1] - I[0][1] * I[2][0]);
    inv[2][2] = I[0][0] * I[1][1] - I[0][1] * I[1][0];
    double w[3];
    for (int r = 0; r < 3; ++r)
      w[r] = (inv[r][0] / det) * L[0] + (inv[r][1] / det) * L[1] + (inv[r][2] / det) * L[2];
    for (int n = 0; n < N; ++n) { // v_i -= w x dr_i
      const double dx = x[n] - r0[0], dy = y[n] - r0[1], dz = z[n] - r0[2];
      vx[n] -= w[1] * dz - w[2] * dy;
      vy[n] -= w[2] * dx - w[0] * dz;
      vz[n] -= w[0] * dy - w[1] * dx;
    }
  }
  // scale to the target temperature
  double ke2 = 0;
  for (int n = 0; n < N; ++n)
    ke2 += m[n] * (vx[n] * vx[n] + vy[n] * vy[n] + vz[n] * vz[n]);
  const double factor = std::sqrt(temperature / (ke2 / (3.0 * K_B * N)));
  for (size_t k = 0; k < (size_t)3 * N; ++k)
    vx[k] *= factor;
}

class Run
{
public:
  Run()
  {
    read_model("model.xyz", model_);
    printf("Number of atoms is %d.\n", model_.atom.number_of_atoms);
    execute_run_in();
  }

private:
  Model model_;
  Force force_;
  std::unique_ptr<Ensemble> ensemble_;
  // what the `ensemble` keyword asked for; the object itself is built at `run` from the time step
  // and atom count in force THEN, and rebuilt for every run (Integrate::initialize, integrate.cu:76-280)
  struct EnsembleSpec {
    // 0 nve, 1 nvt_ber, 2 nvt_nhc, 3 nvt_lan, 4 nvt_bdp, 5 nvt_bao, 11 npt_ber, 21 heat_nhc, 22 heat_lan,
    // 23 heat_bdp
    int type = -1;
    double T = 0.0, Tc = 0.0;
    double dT = 0.0;             // heat_*: the source is at T + dT, the sink at T - dT
    int source = -1, sink = -1; // heat_*: group ids of grouping method 0
    // npt_ber: natural units, as integrate.cu:1150-1153 leaves them
    double target_p[6] = {0, 0, 0, 0, 0, 0}, p_coupling[6] = {0, 0, 0, 0, 0, 0};
    int num_p = 0;
    bool has_seed = false;
    unsigned seed = 0;
  } ensemble_spec_;
  GPU_Vector<double> thermo_;
  // `fix [method] group` / `move [method] group vx vy vz` (integrate.cu:1362-1470); both are reset
  // after every run like the reference's Integrate::finalize (integrate.cu:284-290)
  int fixed_group_ = -1, move_group_ = -1, fixed_method_ = 0, move_method_ = 0;
  double move_velocity_[3] = {0.0, 0.0, 0.0};
  double time_step_ = 1.0 / TIME_UNIT_CONVERSION;
  int dump_thermo_ = 0;
  int dump_restart_ = 0;
  // dump_xyz: interval, file, "%.9g" / "%.17g", optional per-atom columns (dump_xyz.cu:68-150)
  struct XyzDump {
    int interval = 0;
    std::string file;
    bool separated = false;
    int precision = 2;
    bool mass = false, velocity = false, force = false, potential = false, virial = false;
  } dump_xyz_;
  // compute_hac sample_interval Nc output_interval (measure/hac.cu:262-300); reset after each run
  double hac_temperature_ = 300.0; // the temperature of the last thermostatted ensemble line (run.cu passes
                                   // integrate.temperature2 to the measurements; an nve line leaves it)
  struct HacSpec {
    int interval = 0, Nc = 0, output_interval = 1;
  } hac_spec_;
  // compute_hnemd output_interval fe_x fe_y fe_z (hnemd_kappa.cu:142-184); reset after each run
  // (HNEMD::postprocess, Force::finalize)
  struct HnemdSpec {
    int output_interval = 0; // 0: off
    double fe[3] = {0.0, 0.0, 0.0};
  } hnemd_spec_;
  // compute grouping_method sample_interval output_interval quantities... (compute.cu:595-660); reset
  // after each run (Compute::postprocess, :69-88)
  struct ComputeSpec {
    int grouping_method = 0, sample_interval = 0, output_interval = 0; // sample_interval 0: off
    unsigned mask = 0;
  } compute_spec_;
  // compute_dos / compute_sdc / compute_msd / compute_shc (dos.cu:153-202, sdc.cu:300-338,
  // msd.cu:481-541, shc.cu:466-542); reset after each run (the postprocess of each).  sample_interval 0:
  // off; group_method -1: the whole system
  struct CorrSpec {
    int sample_interval = 0, Nc = 0, group_method = -1, group_id = -1;
    double omega_max = 0.0; // DOS, SHC (max_omega)
    int num_dos_points = -1; // DOS; -1: Nc
    bool all_groups = false; // MSD
    int save_every = -1;     // MSD
    int direction = 0, num_omega = 0; // SHC
  } dos_spec_, sdc_spec_, msd_spec_, shc_spec_;
  // atom.unwrapped_position of the reference: tracked from the first run with compute_msd on, in every
  // later run too (msd.cu:471-477, integrate.cu:347-374)
  GPU_Vector<double> unwrapped_, position_old_;
  double global_time_ = 0.0; // natural units, as Run::global_time (run.cu:316)
  bool state_on_gpu_ = false;
  bool has_potential_ = false;
  long global_step_ = 0;

  void upload_state()
  {
    Atom& a = model_.atom;
    const int N = a.number_of_atoms;
    a.type.resize(N);
    a.type.copy_from_host(a.cpu_type.data());
    a.mass.resize(N);
    a.mass.copy_from_host(a.cpu_mass.data());
    a.position_per_atom.resize((size_t)3 * N);
    a.position_per_atom.copy_from_host(a.cpu_position_per_atom.data());
    a.velocity_per_atom.resize((size_t)3 * N);
    a.velocity_per_atom.copy_from_host(a.cpu_velocity_per_atom.data());
    a.force_per_atom.resize((size_t)3 * N, 0.0);
    a.virial_per_atom.resize((size_t)9 * N, 0.0);
    a.potential_per_atom.resize(N, 0.0);
    thermo_.resize(12, 0.0);
    state_on_gpu_ = true;
  }

  void execute_run_in()
  {
    std::ifstream in("run.in");
    if (!in.is_open())
      input_error("Failed to open run.in.");
    std::string line;
    while (std::getline(in, line)) {
      const size_t hash = line.find('#');
      if (hash != std::string::npos)
        line = line.substr(0, hash);
      std::istringstream ss(line);
      std::vector<std::string> tok;
      std::string w;
      while (ss >> w)
        tok.push_back(w);
      if (!tok.empty())
        parse_one_keyword(tok);
    }
  }

  void parse_one_keyword(const std::vector<std::string>& t)
  {
    Atom& a = model_.atom;
    if (t[0] == "potential") {
      if (t.size() != 2)
        input_error("potential should have 1 parameter.");
      force_.parse_potential(t[1].c_str(), a.number_of_atoms);
      a.cpu_type.resize(a.number_of_atoms);
      for (int n = 0; n < a.number_of_atoms; ++n) {
        const int ty = force_.potentials[0]->type_of(a.cpu_atom_symbol[n]);
        if (ty < 0)
          input_error("There is atom in model.xyz that is not allowed in the used potential.");
        a.cpu_type[n] = ty;
      }
      has_potential_ = true;
    } else if (t[0] == "velocity") {
      if (t.size() != 2 && t.size() != 4)
        input_error("velocity should have 1 or 3 parameters.");
      if (!model_.has_velocity) {
        const bool use_seed = t.size() == 4 && t[2] == "seed";
        if (state_on_gpu_) // a later run: start from where the atoms are now
          a.position_per_atom.copy_to_host(a.cpu_position_per_atom.data());
        initialize_velocity(a, std::atof(t[1].c_str()), use_seed, use_seed ? std::atoi(t[3].c_str()) : 0);
        if (state_on_gpu_)
          a.velocity_per_atom.copy_from_host(a.cpu_velocity_per_atom.data());
      }
    } else if (t[0] == "ensemble") {
      // Integrate::parse_ensemble, integrate.cu:406-432,569-600: nvt_* take T1 T2 tau_T/dt
      EnsembleSpec e;
      if (t.size() == 2 && t[1] == "nve") {
        e.type = 0;
      } else if ((t.size() == 5 || (t.size() == 7 && t[1] == "nvt_bdp" && t[5] == "seed")) &&
                 (t[1] == "nvt_ber" || t[1] == "nvt_nhc" || t[1] == "nvt_bdp")) {
        const double T1 = std::atof(t[2].c_str()), T2 = std::atof(t[3].c_str());
        e.T = T1;
        e.Tc = std::atof(t[4].c_str());
        if (T1 <= 0.0 || T2 <= 0.0)
          input_error("Temperatures should > 0.");
        if (T1 != T2)
          input_error("temperature ramps are not supported by the b200md backend.");
        if (e.Tc < 1.0)
          input_error("Temperature coupling should >= 1.");
        e.type = t[1] == "nvt_ber" ? 1 : (t[1] == "nvt_bdp" ? 4 : 2);
        if (t.size() == 7) { // extension: `nvt_bdp T T tau seed S` fixes the noise stream
          e.has_seed = true;
          e.seed = (unsigned)std::strtoul(t[6].c_str(), nullptr, 10);
        }
      } else if (t.size() == 5 && (t[1] == "nvt_lan" || t[1] == "nvt_bao")) {
        e.T = std::atof(t[2].c_str());
        e.Tc = std::atof(t[4].c_str());
        if (e.T <= 0.0 || std::atof(t[3].c_str()) != e.T)
          input_error("Temperatures should > 0 and equal (no ramps in the b200md backend).");
        if (e.Tc < 1.0)
          input_error("Temperature coupling should >= 1.");
        e.type = t[1] == "nvt_lan" ? 3 : 5;
      } else if (t[1] == "npt_ber" && (t.size() == 8 || t.size() == 12 || t.size() == 18)) {
        // npt_ber T1 T2 Tc p(1|3|6, GPa) C(1|3|6 elastic moduli, GPa) tau_p  (integrate.cu:630-700)
        e.T = std::atof(t[2].c_str());
        e.Tc = std::atof(t[4].c_str());
        if (e.T <= 0.0 || std::atof(t[3].c_str()) != e.T)
          input_error("Temperatures should > 0 and equal (no ramps in the b200md backend).");
        if (e.Tc < 1.0)
          input_error("Temperature coupling should >= 1.");
        e.num_p = t.size() == 8 ? 1 : (t.size() == 12 ? 3 : 6);
        const Box& b = model_.box;
        const bool tri = b.cpu_h[1] != 0 || b.cpu_h[2] != 0 || b.cpu_h[3] != 0 || b.cpu_h[5] != 0 ||
                         b.cpu_h[6] != 0 || b.cpu_h[7] != 0;
        if (e.num_p < 6 && tri)
          input_error("Cannot use triclinic box with only 1 or 3 target pressure components.");
        if (e.num_p != 3 && !(b.pbc_x && b.pbc_y && b.pbc_z))
          input_error("Cannot use isotropic / 6-component pressure with a non-periodic direction.");
        double modulus[6] = {1, 1, 1, 1, 1, 1};
        for (int k = 0; k < e.num_p; ++k) {
          e.target_p[k] = std::atof(t[5 + k].c_str());
          modulus[k] = std::atof(t[5 + e.num_p + k].c_str());
          if (modulus[k] <= 0)
            input_error("elastic modulus should > 0.");
        }
        const double tau_p = std::atof(t[5 + 2 * e.num_p].c_str());
        if (tau_p < 1)
          input_error("Pressure coupling should >= 1.");
        for (int k = 0; k < 6; ++k) {
          e.p_coupling[k] = modulus[k] > 2.0e3 ? 0.0 : 1.0 / (tau_p * 3.0 * modulus[k]);
          e.target_p[k] /= PRESSURE_UNIT_CONVERSION;
          e.p_coupling[k] *= PRESSURE_UNIT_CONVERSION;
        }
        e.type = 11;
      } else if (t[1] == "heat_nhc" || t[1] == "heat_lan" || t[1] == "heat_bdp") {
        parse_heat(t, e);
      } else {
        input_error("supported by the b200md backend: ensemble nve | nvt_ber|nvt_nhc|nvt_bdp|nvt_lan|"
                    "nvt_bao T T tau | npt_ber T T tau p.. C.. tau_p | heat_lan|heat_nhc|heat_bdp T Tc dT "
                    "source sink");
      }
      ensemble_spec_ = e;
      if (e.type != 0)
        hac_temperature_ = e.T;
    } else if (t[0] == "fix") {
      // fix group_id | fix grouping_method group_id
      if (t.size() != 2 && t.size() != 3)
        input_error("Keyword fix should have 1 or 2 parameters.");
      fixed_method_ = t.size() == 3 ? std::atoi(t[1].c_str()) : 0;
      fixed_group_ = std::atoi(t[t.size() - 1].c_str());
      if (fixed_method_ < 0 || fixed_method_ >= (int)model_.group.size())
        input_error("Grouping method for fix is out of range (does model.xyz have a group column?).");
      if (fixed_group_ < 0 || fixed_group_ >= model_.group[fixed_method_].number)
        input_error("Group ID for fix is out of range.");
      printf("Group %d in grouping method %d will be fixed.\n", fixed_group_, fixed_method_);
    } else if (t[0] == "move") {
      // move group_id vx vy vz | move grouping_method group_id vx vy vz   (velocities in A/fs)
      if (t.size() != 5 && t.size() != 6)
        input_error("Keyword move should have 4 or 5 parameters.");
      const size_t o = t.size() - 4;
      move_method_ = t.size() == 6 ? std::atoi(t[1].c_str()) : 0;
      move_group_ = std::atoi(t[o].c_str());
      if (move_method_ < 0 || move_method_ >= (int)model_.group.size())
        input_error("Grouping method for move is out of range.");
      if (move_group_ < 0 || move_group_ >= model_.group[move_method_].number)
        input_error("Group ID for move is out of range.");
      for (int d = 0; d < 3; ++d)
        move_velocity_[d] = std::atof(t[o + 1 + d].c_str()) * TIME_UNIT_CONVERSION;
      printf("Group %d in grouping method %d will move at (%g, %g, %g) A/fs.\n", move_group_,
             move_method_, move_velocity_[0] / TIME_UNIT_CONVERSION,
             move_velocity_[1] / TIME_UNIT_CONVERSION, move_velocity_[2] / TIME_UNIT_CONVERSION);
    } else if (t[0] == "time_step") {
      if (t.size() < 2)
        input_error("time_step should have at least 1 parameter.");
      time_step_ = std::atof(t[1].c_str()) / TIME_UNIT_CONVERSION; // run.cu:657
    } else if (t[0] == "dump_thermo") {
      if (t.size() != 2 || std::atoi(t[1].c_str()) <= 0)
        input_error("dump_thermo should have 1 positive parameter (the interval).");
      dump_thermo_ = std::atoi(t[1].c_str());
    } else if (t[0] == "compute_hac") {
      if (t.size() != 4)
        input_error("compute_hac should have 3 parameters.");
      hac_spec_.interval = std::atoi(t[1].c_str());
      hac_spec_.Nc = std::atoi(t[2].c_str());
      hac_spec_.output_interval = std::atoi(t[3].c_str());
      if (hac_spec_.interval <= 0 || hac_spec_.Nc <= 0 || hac_spec_.output_interval <= 0)
        input_error("compute_hac parameters should be positive integers.");
      printf("Compute HAC.\n    sample interval is %d.\n    Nc is %d\n    output_interval is %d\n",
             hac_spec_.interval, hac_spec_.Nc, hac_spec_.output_interval);
    } else if (t[0] == "compute") {
      parse_compute(t);
    } else if (t[0] == "compute_hnemd") {
      parse_compute_hnemd(t);
    } else if (t[0] == "compute_shc") {
      parse_compute_shc(t);
    } else if (t[0] == "compute_dos") {
      parse_compute_dos(t);
    } else if (t[0] == "compute_sdc") {
      parse_compute_sdc(t);
    } else if (t[0] == "compute_msd") {
      parse_compute_msd(t);
    } else if (t[0] == "dump_restart") {
      if (t.size() != 2 || std::atoi(t[1].c_str()) <= 0)
        input_error("dump_restart should have 1 positive parameter (the interval).");
      dump_restart_ = std::atoi(t[1].c_str());
    } else if (t[0] == "dump_xyz") {
      parse_dump_xyz(t);
    } else if (t[0] == "replicate") {
      if (state_on_gpu_ || has_potential_)
        input_error("replicate must come before 'potential' (run.cu:356-358).");
      replicate(t);
    } else if (t[0] == "run") {
      if (t.size() != 2 || std::atoi(t[1].c_str()) < 0)
        input_error("run should have 1 parameter (the number of steps).");
      perform_a_run(std::atoi(t[1].c_str()));
      fixed_group_ = move_group_ = -1;
      fixed_method_ = move_method_ = 0;
      hac_spec_ = HacSpec();
      hnemd_spec_ = HnemdSpec();
      compute_spec_ = ComputeSpec();
      dos_spec_ = sdc_spec_ = msd_spec_ = shc_spec_ = CorrSpec();
      force_.finalize();
      dump_thermo_ = 0; // non-propagating keywords are reset after each run (run.cu:329-340)
      dump_restart_ = 0;
      dump_xyz_ = XyzDump();
    } else {
      input_error("'" + t[0] + "' is not a keyword supported by the b200md backend.");
    }
  }

  // Integrate::parse_ensemble, heat branch (integrate.cu:479-493,716-768)
  void parse_heat(const std::vector<std::string>& t, EnsembleSpec& e)
  {
    e.type = t[1] == "heat_nhc" ? 21 : (t[1] == "heat_lan" ? 22 : 23);
    if (t.size() != 7)
      input_error("ensemble " + t[1] + " should have 5 parameters.");
    if (!valid_real(t[2], &e.T))
      input_error("Temperature should be a number.");
    if (e.T <= 0.0)
      input_error("Temperature should > 0.");
    if (!valid_real(t[3], &e.Tc))
      input_error("Temperature coupling should be a number.");
    if (e.Tc < 1.0)
      input_error("Temperature coupling should >= 1.");
    if (!valid_real(t[4], &e.dT))
      input_error("Temperature difference should be a number.");
    if (e.dT >= e.T || e.dT <= -e.T)
      input_error("|Temperature difference| is too large.");
    if (!valid_int(t[5], &e.source))
      input_error("Group ID for heat source should be an integer.");
    if (!valid_int(t[6], &e.sink))
      input_error("Group ID for heat sink should be an integer.");
    if (model_.group.size() < 1)
      input_error("Cannot heat/cold without grouping method.");
    if (e.source == e.sink)
      input_error("Source and sink cannot be the same group.");
    if (e.source < 0)
      input_error("Group ID for heat source should >= 0.");
    if (e.source >= model_.group[0].number)
      input_error("Group ID for heat source should < #groups.");
    if (e.sink < 0)
      input_error("Group ID for heat sink should >= 0.");
    if (e.sink >= model_.group[0].number)
      input_error("Group ID for heat sink should < #groups.");
    printf("Use %s heating/cooling: T = %g K, Tc = %g, dT = %g K, source %d, sink %d.\n", t[1].c_str(), e.T,
           e.Tc, e.dT, e.source, e.sink);
  }

  // Compute::parse, compute.cu:595-660
  void parse_compute(const std::vector<std::string>& t)
  {
    printf("Compute space and/or time average of:\n");
    if (t.size() < 5)
      input_error("compute should have at least 4 parameters.");
    ComputeSpec c;
    if (!valid_int(t[1], &c.grouping_method))
      input_error("grouping method of compute should be integer.");
    if (c.grouping_method < 0)
      input_error("grouping method should >= 0.");
    if (c.grouping_method >= (int)model_.group.size())
      input_error("grouping method exceeds the bound.");
    if (!valid_int(t[2], &c.sample_interval))
      input_error("sampling interval of compute should be integer.");
    if (c.sample_interval <= 0)
      input_error("sampling interval of compute should > 0.");
    if (!valid_int(t[3], &c.output_interval))
      input_error("output interval of compute should be integer.");
    if (c.output_interval <= 0)
      input_error("output interval of compute should > 0.");
    static const char* names[7] = {"temperature", "potential", "force", "virial", "jp", "jk", "momentum"};
    for (size_t k = 4; k < t.size(); ++k) {
      int q = 0;
      while (q < 7 && t[k] != names[q])
        ++q;
      if (q == 7)
        input_error("Invalid property for compute.");
      c.mask |= 1u << q;
      printf("    %s\n", names[q]);
    }
    printf("    using grouping method %d.\n", c.grouping_method);
    printf("    with sampling interval %d.\n", c.sample_interval);
    printf("    and output interval %d.\n", c.output_interval);
    compute_spec_ = c;
  }

  // Compute::output_results, compute.cu:540-561: the averages, then (with temperature) the energy
  // transferred to the source and sink baths.  A non-heat ensemble prints 0 for both (the reference
  // prints its never-initialised energy_transferred there).
  void write_compute(b200md_group_compute* cp, int num_values)
  {
    std::vector<double> v(num_values);
    if (b200md_group_compute_take(cp, compute_spec_.output_interval, v.data(), nullptr) != B200MD_OK)
      b2h_fail("compute");
    FILE* fc = fopen("compute.out", "a");
    if (!fc)
      input_error("Failed to open compute.out.");
    for (double x : v)
      fprintf(fc, "%15.6e", x);
    if (compute_spec_.mask & B200MD_COMPUTE_TEMPERATURE) {
      double e[2] = {0.0, 0.0};
      if (auto* heat = dynamic_cast<Ensemble_HEAT_B200*>(ensemble_.get())) {
        heat->read_energy_transferred();
        e[0] = heat->b2_energy_transferred[0];
        e[1] = heat->b2_energy_transferred[1];
      }
      fprintf(fc, "%15.6e%15.6e", e[0], e[1]);
    }
    fprintf(fc, "\n");
    fclose(fc);
  }

  void parse_compute_hnemd(const std::vector<std::string>& t)
  {
    printf("Compute thermal conductivity using the HNEMD method.\n");
    if (t.size() != 5)
      input_error("compute_hnemd should have 4 parameters.");
    HnemdSpec h;
    if (!valid_int(t[1], &h.output_interval))
      input_error("output_interval for HNEMD should be an integer number.");
    if (h.output_interval < 1)
      input_error("output_interval for HNEMD should be larger than 0.");
    const char* names[3] = {"fe_x", "fe_y", "fe_z"};
    for (int d = 0; d < 3; ++d)
      if (!valid_real(t[2 + d], &h.fe[d]))
        input_error(std::string(names[d]) + " for HNEMD should be a real number.");
    if (hnemd_spec_.output_interval > 0) // Force::set_hnemd_parameters, force.cu:344-346
      input_error("Cannot have more than one HNEMD method within one run.");
    printf("    output_interval = %d\n    fe = (%g, %g, %g) /A\n", h.output_interval, h.fe[0], h.fe[1],
           h.fe[2]);
    hnemd_spec_ = h;
    force_.set_hnemd(h.fe); // already in force for the evaluation before the loop (run.cu:217-248)
  }

  void parse_compute_shc(const std::vector<std::string>& t)
  {
    printf("Compute SHC.\n");
    if (t.size() != 6 && t.size() != 9)
      input_error("compute_shc should have 5 or 8 parameters.");
    CorrSpec c;
    if (!valid_int(t[1], &c.sample_interval))
      input_error("Sampling interval for SHC should be an integer.");
    if (c.sample_interval < 1)
      input_error("Sampling interval for SHC should >= 1.");
    if (c.sample_interval > 50)
      input_error("Sampling interval for SHC should <= 50 (trust me).");
    if (!valid_int(t[2], &c.Nc))
      input_error("Nc for SHC should be an integer.");
    if (c.Nc < 100)
      input_error("Nc for SHC should >= 100 (trust me).");
    if (c.Nc > 1000)
      input_error("Nc for SHC should <= 1000 (trust me).");
    if (!valid_int(t[3], &c.direction))
      input_error("direction for SHC should be an integer.");
    if (c.direction < 0 || c.direction > 2)
      input_error("Transport direction should be x or y or z.");
    if (!valid_int(t[4], &c.num_omega))
      input_error("num_omega for SHC should be an integer.");
    if (c.num_omega < 0)
      input_error("num_omega for SHC should >= 0.");
    if (!valid_real(t[5], &c.omega_max))
      input_error("max_omega for SHC should be a number.");
    if (c.omega_max <= 0)
      input_error("max_omega for SHC should > 0.");
    for (size_t k = 6; k < t.size(); k++) {
      if (t[k] != "group")
        input_error("Unrecognized argument in compute_shc.");
      parse_group(t, true, k, c);
      if (c.group_id < -1)
        input_error("group ID should >= -1 for computing SHC.");
      if (c.group_id == -1 && model_.group[c.group_method].number < 2)
        input_error("compute_shc with group ID -1 needs a grouping method with at least two groups.");
    }
    printf("    sampling interval %d, Nc %d, direction %d, num_omega %d, max_omega %g\n",
           c.sample_interval, c.Nc, c.direction, c.num_omega, c.omega_max);
    shc_spec_ = c;
  }

  // SHC::postprocess, shc.cu:398-464: header, then per output group 2Nc-1 correlation rows and
  // num_omega spectrum rows
  void write_shc(b200md_shc* shc, int num_groups)
  {
    const CorrSpec& c = shc_spec_;
    const int Nk = 2 * c.Nc - 1;
    std::vector<double> ki((size_t)num_groups * Nk), ko(ki.size());
    std::vector<double> si((size_t)num_groups * c.num_omega + 1), so(si.size());
    if (b200md_shc_finish(shc, time_step_, c.num_omega, c.omega_max, ki.data(), ko.data(), si.data(),
                          so.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_shc");
    const double dt_in_ps = time_step_ * c.sample_interval * TIME_UNIT_CONVERSION / 1000.0;
    const double d_omega = c.omega_max / c.num_omega;
    FILE* fid = fopen("shc.out", "a");
    if (!fid)
      input_error("Failed to open shc.out.");
    fprintf(fid, "# compute_shc %d %d %d %d %g", c.sample_interval, c.Nc, c.direction, c.num_omega,
            c.omega_max);
    if (c.group_method >= 0)
      fprintf(fid, " group %d %d", c.group_method, c.group_id);
    fprintf(fid, "\n# format_version 1\n# num_atoms %d\n", model_.atom.number_of_atoms);
    const double* h = model_.box.cpu_h;
    fprintf(fid, "# cell %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e\n", h[0], h[3], h[6],
            h[1], h[4], h[7], h[2], h[5], h[8]);
    fprintf(fid, "# dt_output %.10e ps\n", dt_in_ps);
    fprintf(fid, "# num_correlation_rows %d\n", Nk);
    fprintf(fid, "# num_frequency_rows %d\n", c.num_omega);
    if (c.group_method >= 0 && c.group_id == -1)
      fprintf(fid, "# num_output_groups %d\n", num_groups);
    fprintf(fid, "# columns_correlation time_ps ki ko\n");
    fprintf(fid, "# columns_shc omega_THz shc_i shc_o\n");
    for (int g = 0; g < num_groups; ++g) {
      for (int nc = 0; nc < Nk; ++nc) // ki, ko in A eV/ps
        fprintf(fid, "%g %g %g\n", (nc + 1 - c.Nc) * dt_in_ps, ki[(size_t)g * Nk + nc],
                ko[(size_t)g * Nk + nc]);
      for (int nw = 0; nw < c.num_omega; ++nw) // shc_i, shc_o in A eV = A eV/ps/THz
        fprintf(fid, "%g %g %g\n", (nw + 1) * d_omega, si[(size_t)g * c.num_omega + nw],
                so[(size_t)g * c.num_omega + nw]);
    }
    fclose(fid);
  }

  // the sample interval and Nc that all three correlation keywords start with
  void parse_interval_nc(const std::vector<std::string>& t, CorrSpec& c)
  {
    if (!valid_int(t[1], &c.sample_interval))
      input_error("sample interval should be an integer.");
    if (c.sample_interval <= 0)
      input_error("sample interval should be positive.");
    printf("    sample interval is %d.\n", c.sample_interval);
    if (!valid_int(t[2], &c.Nc))
      input_error("number of correlation steps should be an integer.");
    if (c.Nc <= 0)
      input_error("number of correlation steps should be positive.");
    printf("    number of correlation steps is %d.\n", c.Nc);
  }

  // parse_group, src/measure/parse_utilities.cu:27-62
  void parse_group(const std::vector<std::string>& t, bool allow_all_groups, size_t& k, CorrSpec& c)
  {
    if (k + 3 > t.size())
      input_error("Not enough arguments for option 'group'.");
    if (!valid_int(t[k + 1], &c.group_method))
      input_error("Grouping method should be an integer.");
    if (c.group_method < 0)
      input_error("Grouping method should >= 0.");
    if (c.group_method >= (int)model_.group.size())
      input_error("Grouping method should < number of grouping methods.");
    if (!valid_int(t[k + 2], &c.group_id))
      input_error("Group ID should be an integer.");
    if (c.group_id >= model_.group[c.group_method].number)
      input_error("Group ID should < number of groups.");
    if (c.group_id < 0 && !allow_all_groups)
      input_error("group ID should >= 0.");
    printf("    grouping method is %d and group ID is %d.\n", c.group_method, c.group_id);
    k += 2;
  }

  // DOS::parse, dos.cu:153-202
  void parse_compute_dos(const std::vector<std::string>& t)
  {
    printf("Compute phonon DOS.\n");
    if (t.size() < 4)
      input_error("compute_dos should have at least 3 parameters.");
    if (t.size() > 9)
      input_error("compute_dos has too many parameters.");
    CorrSpec c;
    parse_interval_nc(t, c);
    if (!valid_real(t[3], &c.omega_max))
      input_error("maximal angular frequency should be a number.");
    if (c.omega_max <= 0)
      input_error("maximal angular frequency should be positive.");
    printf("    maximal angular frequency is %g THz.\n", c.omega_max);
    for (size_t k = 4; k < t.size(); k++) {
      if (t[k] == "group") {
        parse_group(t, true, k, c);
      } else if (t[k] == "num_dos_points") {
        if (k + 2 > t.size())
          input_error("Not enough arguments for option 'num_dos_points'.");
        if (!valid_int(t[k + 1], &c.num_dos_points))
          input_error("number of DOS points should be an integer.");
        if (c.num_dos_points < 1)
          input_error("number of DOS points must be > 0.");
        k += 1;
        printf("    num_dos_points is %d.\n", c.num_dos_points);
      } else {
        input_error("Unrecognized argument in compute_dos.");
      }
    }
    dos_spec_ = c;
  }

  // SDC::parse, sdc.cu:300-338
  void parse_compute_sdc(const std::vector<std::string>& t)
  {
    printf("Compute self diffusion coefficient (SDC).\n");
    if (t.size() < 3)
      input_error("compute_sdc should have at least 2 parameters.");
    if (t.size() > 6)
      input_error("compute_sdc has too many parameters.");
    CorrSpec c;
    parse_interval_nc(t, c);
    for (size_t k = 3; k < t.size(); k++) {
      if (t[k] == "group")
        parse_group(t, false, k, c);
      else
        input_error("Unrecognized argument in compute_sdc.");
    }
    sdc_spec_ = c;
  }

  // MSD::parse, msd.cu:481-541.  all_groups reads the method after the keyword (the reference reads
  // param[4], which is that position in the documented form `compute_msd <i> <Nc> all_groups <m>`)
  void parse_compute_msd(const std::vector<std::string>& t)
  {
    printf("Compute mean square displacement (MSD).\n");
    if (t.size() < 3)
      input_error("compute_msd should have at least 2 parameters.");
    if (t.size() > 8)
      input_error("compute_msd has too many parameters.");
    CorrSpec c;
    parse_interval_nc(t, c);
    for (size_t k = 3; k < t.size(); k++) {
      if (t[k] == "group") {
        parse_group(t, false, k, c);
      } else if (t[k] == "all_groups") {
        c.all_groups = true;
        if (k + 2 > t.size() || !valid_int(t[k + 1], &c.group_method))
          input_error("Grouping method should be an integer.");
        if (c.group_method < 0)
          input_error("Grouping method should >= 0.");
        if (c.group_method >= (int)model_.group.size())
          input_error("Grouping method should < number of grouping methods.");
        printf("    will compute MSD for all groups in grouping %d.\n", c.group_method);
        k += 1;
      } else if (t[k] == "save_every") {
        if (k + 2 > t.size() || !valid_int(t[k + 1], &c.save_every))
          input_error("save_every should be an integer.");
        printf("    will save a copy of the MSD every %d steps.\n", c.save_every);
        k += 1;
      } else {
        input_error("Unrecognized argument in compute_msd.");
      }
    }
    if (c.all_groups && c.group_method >= 0 && c.group_id >= 0)
      input_error("Cannot compute MSD over a single group and all groups at the same time");
    msd_spec_ = c;
  }

  // the output groups of a correlation keyword as (sizes, contents): the whole system, one group, or
  // every group of the method (`group m -1` for DOS, `all_groups m` for MSD), or for SHC's `group m -1`
  // every group except 0 (shc.cu:204-205)
  const int* corr_groups(const CorrSpec& c, std::vector<int>& sizes, bool except_group_0 = false) const
  {
    sizes.assign(1, model_.atom.number_of_atoms);
    if (c.group_method < 0)
      return nullptr; // the whole system in atom order
    const Group& g = model_.group[c.group_method];
    if (c.all_groups || c.group_id < 0) {
      const int first = except_group_0 ? 1 : 0;
      sizes.assign(g.cpu_size.begin() + first, g.cpu_size.end());
      return g.contents.data() + g.cpu_size_sum[first]; // the groups are contiguous there
    }
    sizes.assign(1, g.cpu_size[c.group_id]);
    return g.contents.data() + g.cpu_size_sum[c.group_id];
  }

  // DOS::output_vac / output_dos, dos.cu:429-448,483-503: appended, no header, group after group
  void write_dos(b200md_dos* dos, int num_groups)
  {
    const CorrSpec& c = dos_spec_;
    const int Nc = c.Nc, nw = c.num_dos_points;
    std::vector<double> mvac((size_t)num_groups * 3 * Nc), d((size_t)num_groups * 3 * nw);
    if (b200md_dos_finish(dos, mvac.data(), d.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_dos");
    const double dt_in_ps = time_step_ * c.sample_interval * TIME_UNIT_CONVERSION / 1000.0;
    FILE* fid = fopen("mvac.out", "a");
    if (!fid)
      input_error("Failed to open mvac.out.");
    for (int g = 0; g < num_groups; ++g) {
      const double* v = mvac.data() + (size_t)g * 3 * Nc;
      for (int nc = 0; nc < Nc; nc++)
        fprintf(fid, "%g %g %g %g\n", nc * dt_in_ps, v[nc], v[Nc + nc], v[2 * Nc + nc]);
    }
    fclose(fid);
    const double d_omega = c.omega_max / nw;
    fid = fopen("dos.out", "a");
    if (!fid)
      input_error("Failed to open dos.out.");
    for (int g = 0; g < num_groups; ++g) {
      const double* v = d.data() + (size_t)g * 3 * nw;
      for (int k = 0; k < nw; k++)
        fprintf(fid, "%g %g %g %g\n", d_omega + d_omega * k, v[k], v[nw + k], v[2 * nw + k]);
    }
    fclose(fid);
  }

  // SDC::postprocess, sdc.cu:259-285 (the cell at the end of the run)
  void write_sdc(b200md_sdc* sdc, int num_atoms)
  {
    const CorrSpec& c = sdc_spec_;
    const int Nc = c.Nc;
    std::vector<double> vac((size_t)3 * Nc), s((size_t)3 * Nc);
    if (b200md_sdc_finish(sdc, vac.data(), s.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_sdc");
    const double dt_in_ps = time_step_ * c.sample_interval * TIME_UNIT_CONVERSION / 1000.0;
    FILE* fid = fopen("sdc.out", "a");
    if (!fid)
      input_error("Failed to open sdc.out.");
    fprintf(fid, "# compute_sdc %d %d", c.sample_interval, Nc);
    if (c.group_method >= 0)
      fprintf(fid, " group %d %d", c.group_method, c.group_id);
    fprintf(fid, "\n# format_version 1\n# num_atoms %d\n", num_atoms);
    const double* h = model_.box.cpu_h;
    fprintf(fid, "# cell %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e\n", h[0], h[3], h[6], h[1], h[4],
            h[7], h[2], h[5], h[8]);
    fprintf(fid, "# dt_output %.10e ps\n", dt_in_ps);
    fprintf(fid, "# columns time_ps vacx vacy vacz sdcx sdcy sdcz\n");
    for (int nc = 0; nc < Nc; nc++)
      fprintf(fid, "%g %g %g %g %g %g %g\n", nc * dt_in_ps, vac[nc], vac[Nc + nc], vac[2 * Nc + nc], s[nc],
              s[Nc + nc], s[2 * Nc + nc]);
    fclose(fid);
  }

  // MSD::write, msd.cu:365-449; h: the cell at the start of the run (msd.cu:254-255)
  void write_msd(b200md_msd* msd, const char* filename, const std::vector<int>& sizes, int num_atoms,
                 const double* h)
  {
    const CorrSpec& c = msd_spec_;
    const int Nc = c.Nc, ng = (int)sizes.size();
    std::vector<double> m((size_t)ng * 3 * Nc), s(m.size());
    if (b200md_msd_finish(msd, m.data(), s.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_msd");
    const double dt_in_ps = time_step_ * c.sample_interval * TIME_UNIT_CONVERSION / 1000.0;
    FILE* fid = fopen(filename, "a");
    if (!fid)
      input_error(std::string("Failed to open ") + filename + ".");
    fprintf(fid, "# compute_msd %d %d", c.sample_interval, Nc);
    if (c.all_groups)
      fprintf(fid, " all_groups %d", c.group_method);
    else if (c.group_method >= 0)
      fprintf(fid, " group %d %d", c.group_method, c.group_id);
    if (c.save_every > 0)
      fprintf(fid, " save_every %d", c.save_every);
    fprintf(fid, "\n# format_version 1\n# num_atoms %d\n# num_groups %d\n# num_atoms_per_group", num_atoms, ng);
    for (int g = 0; g < ng; ++g)
      fprintf(fid, " %d", sizes[g]);
    fprintf(fid, "\n# cell %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e\n", h[0], h[3], h[6], h[1], h[4],
            h[7], h[2], h[5], h[8]);
    fprintf(fid, "# dt_output %.10e ps\n", dt_in_ps);
    fprintf(fid, "# columns time_ps");
    if (!c.all_groups)
      fprintf(fid, " msdx msdy msdz sdcx sdcy sdcz");
    else
      for (int g = 0; g < ng; ++g)
        fprintf(fid, " msdx_%d msdy_%d msdz_%d sdcx_%d sdcy_%d sdcz_%d", g, g, g, g, g, g);
    fprintf(fid, "\n");
    for (int nc = 0; nc < Nc; nc++) {
      fprintf(fid, "%g", nc * dt_in_ps);
      for (int g = 0; g < ng; g++) {
        const double* a = m.data() + (size_t)g * 3 * Nc;
        const double* b = s.data() + (size_t)g * 3 * Nc;
        fprintf(fid, "% g %g %g %g %g %g", a[nc], a[Nc + nc], a[2 * Nc + nc], b[nc], b[Nc + nc], b[2 * Nc + nc]);
      }
      fprintf(fid, "\n");
    }
    fclose(fid);
  }

  // the temperature the measurements use: run.cu passes integrate.temperature2, which an nve line
  // leaves at the last thermostatted value
  double measure_temperature() const
  {
    return ensemble_spec_.type == 0 ? hac_temperature_ : ensemble_spec_.T;
  }

  // Replicate: copies ordered a-slowest, c-fastest, atoms innermost; box columns scaled
  void replicate(const std::vector<std::string>& t)
  {
    if (t.size() != 4)
      input_error("Replicate should have 3 parameters: number of replications in a, b and c directions.");
    int r[3];
    for (int d = 0; d < 3; ++d) {
      r[d] = std::atoi(t[1 + d].c_str());
      if (r[d] < 1)
        input_error("Number of replications should be a positive integer.");
    }
    Atom& a = model_.atom;
    Box& box = model_.box;
    const int n = a.number_of_atoms, N = n * r[0] * r[1] * r[2];
    std::vector<std::string> sym(N);
    std::vector<double> mass(N), pos((size_t)3 * N), vel((size_t)3 * N);
    int cur = 0;
    for (int i = 0; i < r[0]; ++i)
      for (int j = 0; j < r[1]; ++j)
        for (int k = 0; k < r[2]; ++k)
          for (int m = 0; m < n; ++m, ++cur) {
            sym[cur] = a.cpu_atom_symbol[m];
            mass[cur] = a.cpu_mass[m];
            for (int d = 0; d < 3; ++d) {
              pos[cur + (size_t)d * N] = a.cpu_position_per_atom[m + (size_t)d * n] +
                                         i * box.cpu_h[d * 3] + j * box.cpu_h[d * 3 + 1] +
                                         k * box.cpu_h[d * 3 + 2];
              vel[cur + (size_t)d * N] = a.cpu_velocity_per_atom[m + (size_t)d * n];
            }
          }
    for (int e = 0; e < 9; ++e)
      box.cpu_h[e] *= r[e % 3];
    a.number_of_atoms = N;
    a.cpu_atom_symbol.swap(sym);
    a.cpu_mass.swap(mass);
    a.cpu_position_per_atom.swap(pos);
    a.cpu_velocity_per_atom.swap(vel);
    printf("Replicate cell by %d * %d * %d.\nNumber of atoms is %d.\n", r[0], r[1], r[2], N);
  }

  void parse_dump_xyz(const std::vector<std::string>& t)
  {
    if (t.size() < 3)
      input_error("dump_xyz should have at least 2 parameters.");
    XyzDump d;
    d.interval = std::atoi(t[1].c_str());
    if (d.interval <= 0)
      input_error("dump interval should > 0.");
    d.file = t[2];
    if (d.file.back() == '*') {
      d.separated = true;
      d.file.pop_back();
    }
    for (size_t m = 3; m < t.size(); ++m) {
      if (t[m] == "precision") {
        if (m + 1 >= t.size() || (t[m + 1] != "single" && t[m + 1] != "double"))
          input_error("Invalid precision.");
        d.precision = t[++m] == "single" ? 1 : 2;
      } else if (t[m] == "mass") {
        d.mass = true;
      } else if (t[m] == "velocity") {
        d.velocity = true;
      } else if (t[m] == "force") {
        d.force = true;
      } else if (t[m] == "potential") {
        d.potential = true;
      } else if (t[m] == "virial") {
        d.virial = true;
      } else {
        input_error("Unrecognized argument in dump_xyz (supported: precision, mass, velocity, force, "
                    "potential, virial).");
      }
    }
    dump_xyz_ = d;
  }

  // one frame of extended XYZ: header keys and value formats of dump_xyz.cu:197-437
  void write_xyz_frame(int step)
  {
    const XyzDump& d = dump_xyz_;
    Atom& a = model_.atom;
    const Box& box = model_.box;
    const int N = a.number_of_atoms;
    const char* fmt = d.precision == 1 ? " %.9g" : " %.17g";
    std::vector<double> pos((size_t)3 * N), vel, frc, pe, vir((size_t)9 * N);
    a.position_per_atom.copy_to_host(pos.data());
    a.virial_per_atom.copy_to_host(vir.data());
    if (d.velocity) {
      vel.resize((size_t)3 * N);
      a.velocity_per_atom.copy_to_host(vel.data());
    }
    if (d.force) {
      frc.resize((size_t)3 * N);
      a.force_per_atom.copy_to_host(frc.data());
    }
    if (d.potential) {
      pe.resize(N);
      a.potential_per_atom.copy_to_host(pe.data());
    }
    double th[8];
    thermo_.copy_to_host(th, 8);
    const std::string name = d.separated ? d.file + std::to_string(step + 1) : d.file;
    FILE* fid = fopen(name.c_str(), d.separated ? "w" : "a");
    if (!fid)
      input_error("Failed to open " + name + ".");
    auto tensor = [&](const char* key, const double* v9) {
      fprintf(fid, " %s=\"", key);
      for (int k = 0; k < 9; ++k)
        fprintf(fid, k == 0 ? fmt + 1 : fmt, v9[k]);
      fprintf(fid, "\"");
    };
    fprintf(fid, "%d\n", N);
    fprintf(fid, "Time=%.8f", global_time_ * TIME_UNIT_CONVERSION);
    fprintf(fid, " pbc=\"%c %c %c\"", box.pbc_x ? 'T' : 'F', box.pbc_y ? 'T' : 'F', box.pbc_z ? 'T' : 'F');
    const double* h = box.cpu_h;
    const double lattice[9] = {h[0], h[3], h[6], h[1], h[4], h[7], h[2], h[5], h[8]};
    tensor("Lattice", lattice);
    fprintf(fid, " energy=");
    fprintf(fid, fmt + 1, th[1]);
    double tv[6] = {0, 0, 0, 0, 0, 0}; // totals of xx yy zz xy xz yz
    for (int c = 0; c < 6; ++c)
      for (int n = 0; n < N; ++n)
        tv[c] += vir[(size_t)c * N + n];
    const double virial[9] = {tv[0], tv[3], tv[4], tv[3], tv[1], tv[5], tv[4], tv[5], tv[2]};
    tensor("virial", virial);
    const double stress[9] = {th[2], th[5], th[6], th[5], th[3], th[7], th[6], th[7], th[4]};
    tensor("stress", stress);
    fprintf(fid, " Properties=species:S:1:pos:R:3");
    if (d.mass)
      fprintf(fid, ":mass:R:1");
    if (d.velocity)
      fprintf(fid, ":vel:R:3");
    if (d.force)
      fprintf(fid, ":forces:R:3");
    if (d.potential)
      fprintf(fid, ":energy_atom:R:1");
    if (d.virial)
      fprintf(fid, ":virial:R:9");
    fprintf(fid, "\n");
    const int vidx[9] = {0, 3, 4, 6, 1, 5, 7, 8, 2}; // GPUMD component order -> row-major 3x3
    for (int n = 0; n < N; ++n) {
      fprintf(fid, "%s", a.cpu_atom_symbol[n].c_str());
      for (int k = 0; k < 3; ++k)
        fprintf(fid, fmt, pos[n + (size_t)N * k]);
      if (d.mass)
        fprintf(fid, fmt, a.cpu_mass[n]);
      if (d.velocity)
        for (int k = 0; k < 3; ++k)
          fprintf(fid, fmt, vel[n + (size_t)N * k] / TIME_UNIT_CONVERSION);
      if (d.force)
        for (int k = 0; k < 3; ++k)
          fprintf(fid, fmt, frc[n + (size_t)N * k]);
      if (d.potential)
        fprintf(fid, fmt, pe[n]);
      if (d.virial)
        for (int k = 0; k < 9; ++k)
          fprintf(fid, fmt, vir[n + (size_t)N * vidx[k]]);
      fprintf(fid, "\n");
    }
    fclose(fid);
  }

  // restart.xyz: the model.xyz the next run can start from (dump_restart.cu:83-139)
  void write_restart()
  {
    Atom& a = model_.atom;
    const Box& box = model_.box;
    const int N = a.number_of_atoms;
    std::vector<double> pos((size_t)3 * N), vel((size_t)3 * N);
    a.position_per_atom.copy_to_host(pos.data());
    a.velocity_per_atom.copy_to_host(vel.data());
    FILE* fid = fopen("restart.xyz", "w");
    if (!fid)
      input_error("Failed to open restart.xyz.");
    const double* h = box.cpu_h;
    fprintf(fid, "%d\n", N);
    fprintf(fid, "pbc=\"%c %c %c\" ", box.pbc_x ? 'T' : 'F', box.pbc_y ? 'T' : 'F', box.pbc_z ? 'T' : 'F');
    fprintf(fid, "Lattice=\"%g %g %g %g %g %g %g %g %g\" ", h[0], h[3], h[6], h[1], h[4], h[7], h[2],
            h[5], h[8]);
    fprintf(fid, "Properties=species:S:1:pos:R:3:mass:R:1:vel:R:3\n");
    for (int n = 0; n < N; ++n)
      fprintf(fid, "%s %g %g %g %g %g %g %g \n", a.cpu_atom_symbol[n].c_str(), pos[n],
              pos[n + (size_t)N], pos[n + 2 * (size_t)N], a.cpu_mass[n],
              vel[n] / TIME_UNIT_CONVERSION, vel[n + (size_t)N] / TIME_UNIT_CONVERSION,
              vel[n + 2 * (size_t)N] / TIME_UNIT_CONVERSION);
    fclose(fid);
  }

  void write_thermo(FILE* fid)
  {
    // dump_thermo.cu:73-129: T, K, U, then sxx syy szz syz sxz sxy in GPa, then the box
    double th[8];
    thermo_.copy_to_host(th, 8);
    // the kinetic energy counts every atom but those of the fixed group (dump_thermo.cu:90-101)
    int N = model_.atom.number_of_atoms;
    if (fixed_group_ >= 0)
      N -= model_.group[fixed_method_].cpu_size[fixed_group_];
    const double* h = model_.box.cpu_h;
    fprintf(fid, "%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e", th[0],
            1.5 * N * K_B * th[0], th[1], th[2] * PRESSURE_UNIT_CONVERSION,
            th[3] * PRESSURE_UNIT_CONVERSION, th[4] * PRESSURE_UNIT_CONVERSION,
            th[7] * PRESSURE_UNIT_CONVERSION, th[6] * PRESSURE_UNIT_CONVERSION,
            th[5] * PRESSURE_UNIT_CONVERSION);
    fprintf(fid, "%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e\n", h[0], h[3], h[6],
            h[1], h[4], h[7], h[2], h[5], h[8]);
  }

  void perform_a_run(int number_of_steps)
  {
    if (!has_potential_ || ensemble_spec_.type < 0)
      input_error("'potential' and 'ensemble' must precede 'run'.");
    Atom& a = model_.atom;
    { // Integrate::initialize: a fresh ensemble object per run, from the CURRENT time step
      const EnsembleSpec& e = ensemble_spec_;
      if (move_group_ >= 0) { // integrate.cu:59-73
        if (fixed_group_ < 0)
          input_error("It is not allowed to have moving group but no fixed group.");
        if (fixed_method_ != move_method_)
          input_error("The fixed and moving groups must use the same grouping method.");
        if (move_group_ == fixed_group_)
          input_error("The fixed and moving groups cannot be the same.");
        if (e.type != 1 && e.type != 2 && e.type != 4 && e.type != 22)
          input_error("It is only allowed to use nvt_ber, nvt_nhc, or nvt_bdp with a moving group.");
      }
      const int N = a.number_of_atoms;
      if (e.type == 0) {
        ensemble_.reset(new Ensemble_NVE_B200(0));
      } else if (e.type == 1) {
        ensemble_.reset(new Ensemble_BER_B200(1, move_group_, move_velocity_, e.T, e.Tc));
      } else if (e.type == 4) {
        // the reference seeds std::mt19937 with 12345678 under -DDEBUG and from the clock otherwise
        // (ensemble_bdp.cu:31-37); B200MD_DEBUG_SEED=1 selects the former for trajectory parity
        unsigned seed = e.seed;
        if (!e.has_seed)
          seed = std::getenv("B200MD_DEBUG_SEED")
                   ? 12345678u
                   : (unsigned)std::chrono::system_clock::now().time_since_epoch().count();
        ensemble_.reset(new Ensemble_BDP_B200(4, move_group_, move_velocity_, N, e.T, e.Tc, seed));
      } else if (e.type == 3) {
        ensemble_.reset(new Ensemble_LAN_B200(3, N, e.T, e.Tc, (unsigned long long)rand())); // ensemble_lan.cu:39
      } else if (e.type == 5) {
        ensemble_.reset(new Ensemble_BAO_B200(5, N, e.T, e.Tc, (unsigned long long)rand())); // ensemble_bao.cu:39
      } else if (e.type >= 21 && e.type <= 23) { // integrate.cu:158-199
        const Group& g0 = model_.group[0];
        if (e.type == 22) {
          const unsigned long long seed_source = (unsigned long long)rand(); // ensemble_lan.cu:78-81
          const unsigned long long seed_sink = (unsigned long long)rand();
          ensemble_.reset(new Ensemble_HEAT_LAN_B200(22, move_group_, move_velocity_, N, g0.cpu_size,
                                                     g0.contents.data(), e.source, e.sink, e.T, e.Tc, e.dT,
                                                     seed_source, seed_sink));
        } else if (e.type == 21) {
          ensemble_.reset(new Ensemble_HEAT_NHC_B200(21, N, g0.cpu_size, g0.contents.data(), e.source, e.sink,
                                                     e.T, e.Tc, e.dT, time_step_));
        } else { // the B200MD_DEBUG_SEED rule of nvt_bdp (ensemble_bdp.cu:31-37)
          const unsigned seed = std::getenv("B200MD_DEBUG_SEED")
                                  ? 12345678u
                                  : (unsigned)std::chrono::system_clock::now().time_since_epoch().count();
          ensemble_.reset(new Ensemble_HEAT_BDP_B200(23, N, g0.cpu_size, g0.contents.data(), e.source, e.sink,
                                                     e.T, e.Tc, e.dT, seed));
        }
      } else if (e.type == 11) {
        const double no_rate[3] = {0, 0, 0};
        ensemble_.reset(new Ensemble_BER_B200(11, e.T, e.Tc, e.target_p, e.num_p, e.p_coupling, 0, 0, 0, no_rate));
      } else {
        ensemble_.reset(new Ensemble_NHC_B200(2, move_group_, move_velocity_, N, e.T, e.Tc, time_step_));
      }
      ensemble_->fixed_group = fixed_group_; // integrate.cu:279-281
      ensemble_->fixed_grouping_method = fixed_method_;
      ensemble_->move_grouping_method = move_method_;
    }
    if (!state_on_gpu_)
      upload_state();
    FILE* fid = nullptr;
    if (dump_thermo_ > 0) {
      fid = fopen("thermo.out", "a");
      fprintf(fid, "# dump_thermo %d\n# format_version 1\n# num_atoms %d\n# dt_output %.10e fs\n",
              dump_thermo_, a.number_of_atoms, time_step_ * dump_thermo_ * TIME_UNIT_CONVERSION);
      fprintf(fid, "# columns T KE PE sxx syy szz syz sxz sxy ax ay az bx by bz cx cy cz\n");
    }
    // the first force evaluation is outside the timed loop, as in run.cu:217-248
    force_.compute(model_.box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom,
                   a.virial_per_atom);
    force_.potentials[0]->check();
    b200md_hac* hac = nullptr;
    if (hac_spec_.interval > 0) {
      if (b200md_hac_create(number_of_steps, hac_spec_.interval, hac_spec_.Nc, &hac) != B200MD_OK)
        input_error(std::string("compute_hac: ") + b200md_last_error());
    }
    b200md_hnemd* hnemd = nullptr;
    if (hnemd_spec_.output_interval > 0 &&
        b200md_hnemd_create(hnemd_spec_.output_interval, hnemd_spec_.fe, &hnemd) != B200MD_OK)
      b2h_fail("compute_hnemd");
    b200md_shc* shc = nullptr;
    int shc_groups = 1;
    if (shc_spec_.sample_interval > 0) {
      const CorrSpec& c = shc_spec_;
      std::vector<int> sizes;
      const int* contents = corr_groups(c, sizes, true);
      shc_groups = (int)sizes.size();
      const int rc = b200md_shc_create(c.Nc, c.sample_interval, c.direction, number_of_steps, shc_groups,
                                       sizes.data(), contents, &shc);
      if (rc == B200MD_ERR_ARG)
        input_error(std::string("compute_shc: ") + b200md_last_error());
      if (rc != B200MD_OK)
        b2h_fail("compute_shc");
    }
    b200md_group_compute* cp = nullptr;
    int compute_values = 0;
    if (compute_spec_.sample_interval > 0) { // Compute::preprocess, compute.cu:31-67
      const Group& g = model_.group[compute_spec_.grouping_method];
      if (b200md_group_compute_create(a.number_of_atoms, g.number, g.cpu_size.data(), g.contents.data(),
                                      compute_spec_.mask, &cp) != B200MD_OK)
        b2h_fail("compute");
      compute_values = b200md_group_compute_columns(cp) * g.number;
    }
    // DOS::preprocess, SDC::preprocess, MSD::preprocess (dos.cu:204-218, sdc.cu:132-155, msd.cu:205-267)
    const int N = a.number_of_atoms;
    b200md_dos* dos = nullptr;
    std::vector<int> dos_sizes, sdc_sizes, msd_sizes;
    if (dos_spec_.sample_interval > 0) {
      CorrSpec& c = dos_spec_;
      if (c.num_dos_points < 0)
        c.num_dos_points = c.Nc;
      const int* contents = corr_groups(c, dos_sizes);
      const int rc = b200md_dos_create(c.Nc, c.sample_interval, number_of_steps, time_step_, c.omega_max,
                                       c.num_dos_points, (int)dos_sizes.size(), dos_sizes.data(), contents, N,
                                       a.mass.data(), &dos);
      if (rc == B200MD_ERR_ARG)
        input_error(std::string("compute_dos: ") + b200md_last_error());
      if (rc != B200MD_OK)
        b2h_fail("compute_dos");
    }
    b200md_sdc* sdc = nullptr;
    if (sdc_spec_.sample_interval > 0) {
      const CorrSpec& c = sdc_spec_;
      const int* contents = corr_groups(c, sdc_sizes);
      const int rc = b200md_sdc_create(c.Nc, c.sample_interval, number_of_steps, time_step_,
                                       (int)sdc_sizes.size(), sdc_sizes.data(), contents, &sdc);
      if (rc == B200MD_ERR_ARG)
        input_error(std::string("compute_sdc: ") + b200md_last_error());
      if (rc != B200MD_OK)
        b2h_fail("compute_sdc");
    }
    b200md_msd* msd = nullptr;
    double msd_h[9];
    if (msd_spec_.sample_interval > 0) {
      const CorrSpec& c = msd_spec_;
      const int* contents = corr_groups(c, msd_sizes);
      const int rc = b200md_msd_create(c.Nc, c.sample_interval, number_of_steps, time_step_,
                                       (int)msd_sizes.size(), msd_sizes.data(), contents, &msd);
      if (rc == B200MD_ERR_ARG)
        input_error(std::string("compute_msd: ") + b200md_last_error());
      if (rc != B200MD_OK)
        b2h_fail("compute_msd");
      std::copy(model_.box.cpu_h, model_.box.cpu_h + 9, msd_h);
      if (unwrapped_.size() < (size_t)3 * N) { // the first run with compute_msd (msd.cu:471-477)
        unwrapped_.resize((size_t)3 * N);
        position_old_.resize((size_t)3 * N);
        B2H_CHECK(cudaMemcpy(unwrapped_.data(), a.position_per_atom.data(), sizeof(double) * 3 * N,
                             cudaMemcpyDeviceToDevice));
      }
    }
    const bool unwrap = unwrapped_.size() > 0;
    const int msd_num_atoms = msd_spec_.group_method >= 0 && !msd_spec_.all_groups ? msd_sizes[0] : N;
    printf("Run %d steps.\n", number_of_steps);
    const auto t0 = std::chrono::high_resolution_clock::now();
    for (int step = 0; step < number_of_steps; ++step) {
      if (unwrap && b200md_unwrap_begin(N, a.position_per_atom.data(), position_old_.data(), nullptr) != B200MD_OK)
        b2h_fail("unwrapped positions");
      ensemble_->compute1(time_step_, model_.group, model_.box, a, thermo_);
      if (unwrap && b200md_unwrap_end(N, a.position_per_atom.data(), position_old_.data(), unwrapped_.data(),
                                      nullptr) != B200MD_OK)
        b2h_fail("unwrapped positions");
      force_.compute(model_.box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom,
                     a.virial_per_atom);
      ensemble_->compute2(time_step_, model_.group, model_.box, a, thermo_);
      if (hac && b200md_hac_sample(hac, step, a.number_of_atoms, a.number_of_atoms,
                                   a.virial_per_atom.data(), a.velocity_per_atom.data(), nullptr) != B200MD_OK)
        b2h_fail("compute_hac");
      if (hnemd) {
        if (b200md_hnemd_sample(hnemd, step, a.number_of_atoms, a.number_of_atoms, a.virial_per_atom.data(),
                                a.velocity_per_atom.data(), nullptr) != B200MD_OK)
          b2h_fail("compute_hnemd");
        if ((step + 1) % hnemd_spec_.output_interval == 0) { // hnemd_kappa.cu:108-131
          force_.potentials[0]->check();
          double kappa[5];
          if (b200md_hnemd_take(hnemd, model_.box.get_volume(), measure_temperature(), kappa, nullptr,
                                nullptr) != B200MD_OK)
            b2h_fail("compute_hnemd");
          FILE* fk = fopen("kappa.out", "a");
          if (!fk)
            input_error("Failed to open kappa.out.");
          for (int k = 0; k < 5; ++k)
            fprintf(fk, "%25.15f", kappa[k]);
          fprintf(fk, "\n");
          fclose(fk);
        }
      }
      if (cp && (step + 1) % compute_spec_.sample_interval == 0) { // Compute::process, compute.cu:351-538
        if (b200md_group_compute_sample(cp, a.number_of_atoms, a.number_of_atoms, a.mass.data(),
                                        a.potential_per_atom.data(), a.force_per_atom.data(),
                                        a.virial_per_atom.data(), a.velocity_per_atom.data(),
                                        nullptr) != B200MD_OK)
          b2h_fail("compute");
        if (((step + 1) / compute_spec_.sample_interval) % compute_spec_.output_interval == 0) {
          force_.potentials[0]->check();
          write_compute(cp, compute_values);
        }
      }
      if (shc && b200md_shc_sample(shc, step, a.number_of_atoms, a.number_of_atoms, a.virial_per_atom.data(),
                                   a.velocity_per_atom.data(), nullptr) != B200MD_OK)
        b2h_fail("compute_shc");
      if (dos && b200md_dos_sample(dos, step, N, N, a.velocity_per_atom.data(), nullptr) != B200MD_OK)
        b2h_fail("compute_dos");
      if (sdc && b200md_sdc_sample(sdc, step, N, N, a.velocity_per_atom.data(), nullptr) != B200MD_OK)
        b2h_fail("compute_sdc");
      if (msd) {
        if (b200md_msd_sample(msd, step, N, N, unwrapped_.data(), nullptr) != B200MD_OK)
          b2h_fail("compute_msd");
        const CorrSpec& c = msd_spec_; // a copy every save_every steps, on time origins (msd.cu:355-360)
        if (c.save_every > 0 && (step + 1) % c.sample_interval == 0 && step / c.sample_interval >= c.Nc - 1 &&
            (step + 1) % c.save_every == 0)
          write_msd(msd, ("msd_step" + std::to_string(step + 1) + ".out").c_str(), msd_sizes, msd_num_atoms,
                    msd_h);
      }
      ++global_step_;
      global_time_ += time_step_;
      const bool out_thermo = fid && (step + 1) % dump_thermo_ == 0;
      const bool out_xyz = dump_xyz_.interval > 0 && (step + 1) % dump_xyz_.interval == 0;
      const bool out_restart = dump_restart_ > 0 && (step + 1) % dump_restart_ == 0;
      if (out_thermo || out_xyz || out_restart)
        force_.potentials[0]->check(); // nothing computed from a truncated list reaches a file
      if (out_thermo)
        write_thermo(fid);
      if (out_xyz)
        write_xyz_frame(step);
      if (out_restart)
        write_restart();
    }
    B2H_CHECK(cudaDeviceSynchronize());
    force_.potentials[0]->check();
    const auto t1 = std::chrono::high_resolution_clock::now();
    const double sec = std::chrono::duration<double>(t1 - t0).count();
    printf("Time used for this run = %g second.\n", sec);
    printf("Speed of this run = %g atom*step/second.\n", a.number_of_atoms * (double)number_of_steps / sec);
    if (fid)
      fclose(fid);
    if (hac) { // HAC::postprocess, hac.cu:186-258: hac.out = t(ps), 5 hac averages, 5 rtc averages
      const int Nc = hac_spec_.Nc, oi = hac_spec_.output_interval;
      std::vector<double> h((size_t)5 * Nc), r((size_t)5 * Nc);
      if (b200md_hac_finish(hac, time_step_, measure_temperature(), model_.box.get_volume(), h.data(),
                            r.data(), nullptr) != B200MD_OK)
        b2h_fail("compute_hac");
      const double dt_in_ps = time_step_ * hac_spec_.interval * TIME_UNIT_CONVERSION / 1000.0;
      FILE* fh = fopen("hac.out", "a");
      for (int nd = 0; nd < Nc / oi; ++nd) {
        const int nc = nd * oi;
        fprintf(fh, "%25.15e", (nc + oi * 0.5) * dt_in_ps);
        for (int pass = 0; pass < 2; ++pass)
          for (int k = 0; k < 5; ++k) {
            double ave = 0.0;
            for (int m = 0; m < oi; ++m)
              ave += (pass == 0 ? h : r)[(size_t)Nc * k + nc + m];
            fprintf(fh, "%25.15e", ave / oi);
          }
        fprintf(fh, "\n");
      }
      fclose(fh);
      b200md_hac_destroy(hac);
    }
    if (hnemd)
      b200md_hnemd_destroy(hnemd);
    if (cp)
      b200md_group_compute_destroy(cp);
    if (shc) {
      write_shc(shc, shc_groups);
      b200md_shc_destroy(shc);
    }
    if (dos) {
      write_dos(dos, (int)dos_sizes.size());
      b200md_dos_destroy(dos);
    }
    if (sdc) {
      write_sdc(sdc, sdc_sizes[0]);
      b200md_sdc_destroy(sdc);
    }
    if (msd) {
      write_msd(msd, "msd.out", msd_sizes, msd_num_atoms, msd_h);
      b200md_msd_destroy(msd);
    }
  }
};

int main()
{
  printf("b200md: Hopper-native MD hot path behind GPUMD's Potential/Ensemble surface.\n");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    fprintf(stderr, "Error:\n    no CUDA device found; b200md has no CPU fallback.\n");
    return 1;
  }
  Run run;
  printf("Finished running b200md.\n");
  return 0;
}

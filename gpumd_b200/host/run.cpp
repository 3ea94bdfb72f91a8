// run.cpp -- standalone driver `b200md`: reads GPUMD's own input files from the current directory
// (run.in keyword script, model.xyz extended XYZ, potential file) and runs the hot path through the
// adapter classes, writing thermo.out in the reference's format.
//
// Mirrors, for the keywords of the hot path only:
//   Run::Run / execute_run_in / parse_one_keyword   src/main_gpumd/run.cu:144-209, 343-575
//   Run::perform_a_run (the MD loop)                src/main_gpumd/run.cu:211-341
//   initialize_position (model.xyz)                 src/model/read_xyz.cu:145-425, 482-557
//   Velocity::initialize                            src/main_gpumd/velocity.cu:55-75, 312-347
//   Replicate                                       src/main_gpumd/replicate.cu:20-111
// Keywords here: replicate <na nb nc>, potential, velocity <T> [seed <s>], ensemble nve |
// nvt_ber|nvt_nhc|nvt_bdp|nvt_lan|nvt_bao T T tau | npt_ber | heat_lan|heat_nhc|heat_bdp T Tc dT source
// sink, fix, move, time_step <fs>, minimize sd|fire tol steps [box_change [hydrostatic]],
// compute_phonon <displacement>, run <n>.  The measurement and dump keywords (dump_thermo, dump_xyz,
// dump_restart, compute, compute_hac, compute_hnemd, compute_shc, compute_dos, compute_sdc,
// compute_msd) are one Property each in measure.cpp, held by Measure as the reference's Measure holds
// its properties.  Anything else is an input error (exit 1), as in the reference.
#include "ensemble.h"
#include "force.h"
#include "measure.h"
#include "minimize.h"
#include "phonon.h"
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <fstream>
#include <memory>
#include <sstream>

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
  // the temperature the measurements use: run.cu passes integrate.temperature2, the temperature of the
  // last thermostatted ensemble line (an nve line leaves it)
  double temperature_ = 300.0;
  // atom.unwrapped_position of the reference: tracked from the first run with compute_msd on, in every
  // later run too (msd.cu:471-477, integrate.cu:347-374)
  GPU_Vector<double> unwrapped_, position_old_;
  double global_time_ = 0.0; // natural units, as Run::global_time (run.cu:316)
  bool state_on_gpu_ = false;
  bool has_potential_ = false;
  // the product of the factors of every `replicate` line, wherever it stands (compute_phonon's cell)
  int replicate_[3] = {1, 1, 1};
  bool has_replicate_ = false;
  Measure measure_;
  const MeasureContext ctx_{model_,       force_,   ensemble_,    time_step_,    global_time_,
                            temperature_, thermo_,  fixed_group_, fixed_method_, unwrapped_};

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
    if (measure_.parse(ctx_, t))
      return;
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
        temperature_ = e.T;
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
    } else if (t[0] == "replicate") {
      if (state_on_gpu_ || has_potential_)
        input_error("replicate must come before 'potential' (run.cu:356-358).");
      replicate(t);
    } else if (t[0] == "minimize") {
      minimize(t);
    } else if (t[0] == "compute_phonon") {
      compute_phonon(t);
    } else if (t[0] == "run") {
      if (t.size() != 2 || std::atoi(t[1].c_str()) < 0)
        input_error("run should have 1 parameter (the number of steps).");
      perform_a_run(std::atoi(t[1].c_str()));
      fixed_group_ = move_group_ = -1;
      fixed_method_ = move_method_ = 0;
      measure_.finalize();
      force_.finalize();
    } else {
      input_error("'" + t[0] + "' is not a keyword supported by the b200md backend.");
    }
  }

  // Minimize::parse_minimize (minimize.cu:32-156), run at parse time with the current `fix` group
  // (run.cu:359-369); FIRE ignores the group, as the reference
  void minimize(const std::vector<std::string>& t)
  {
    if (!has_potential_)
      input_error("'potential' must precede 'minimize'.");
    const int num_param = (int)t.size();
    int method = 0, steps = 0, box_change = 0, hydrostatic = 0;
    double tol = 0.0;
    if (num_param >= 2 && t[1] == "sd") {
      if (num_param != 4)
        input_error("minimize sd should have 2 parameters.");
    } else if (num_param >= 2 && t[1] == "fire") {
      method = 1;
      if (!(num_param >= 4 && num_param <= 6))
        input_error("minimize fire should have 2 to 4 parameters.");
    } else {
      input_error("Invalid minimizer.");
    }
    if (!valid_real(t[2], &tol))
      input_error("Force tolerance should be a number.");
    if (!valid_int(t[3], &steps))
      input_error("Number of steps should be an integer.");
    if (steps <= 0)
      input_error("Number of steps should > 0.");
    if (num_param >= 5) {
      if (!valid_int(t[4], &box_change))
        input_error("Box_change should be an integer.");
      if (!(box_change == 0 || box_change == 1))
        input_error("Box_change should be 1 or 0.");
    }
    if (num_param >= 6) {
      if (!valid_int(t[5], &hydrostatic))
        input_error("Hydrostatic_strain should be an integer.");
      if (!(hydrostatic == 0 || hydrostatic == 1))
        input_error("Hydrostatic_strain should be 1 or 0.");
    }
    printf("\nStart to do an energy minimization.\n");
    if (method == 0)
      printf("    using the steepest descent method.\n");
    else
      printf("    using the fast inertial relaxation engine (FIRE) method.\n");
    if (box_change) {
      printf("    with variable box.\n");
      if (hydrostatic)
        printf("    with hydrostatic pressure.\n");
    } else {
      printf("    with fixed box.\n");
    }
    printf("    with a force tolerance of %g eV/A.\n", tol);
    printf("    for maximally %d steps.\n", steps);
    if (!state_on_gpu_)
      upload_state();
    Atom& a = model_.atom;
    const int* label = (method == 0 && fixed_group_ >= 0) ? model_.group[fixed_method_].label.data() : nullptr;
    Minimizer_B200 minimizer(method, a.number_of_atoms, steps, tol, box_change, hydrostatic);
    minimizer.compute(force_, model_.box, a, label, method == 0 ? fixed_group_ : -1);
    force_.potentials[0]->check();
  }

  // run.cu:370-373: Hessian::parse + Hessian::compute at parse time, on the current positions and box
  void compute_phonon(const std::vector<std::string>& t)
  {
    Hessian_B200 hessian;
    hessian.parse(t);
    if (!has_potential_)
      input_error("'potential' must precede 'compute_phonon'.");
    if (!has_replicate_)
      input_error("replicate keyword not found in run.in file.");
    if (!state_on_gpu_)
      upload_state();
    hessian.compute(force_, model_.box, model_.atom, replicate_);
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
    for (int d = 0; d < 3; ++d)
      replicate_[d] *= r[d];
    has_replicate_ = true;
  }

  // Integrate::initialize: a fresh ensemble object per run, from the CURRENT time step
  void build_ensemble()
  {
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
    const int N = model_.atom.number_of_atoms;
    if (e.type == 0) {
      ensemble_.reset(new Ensemble_NVE_B200(0));
    } else if (e.type == 1) {
      ensemble_.reset(new Ensemble_BER_B200(1, move_group_, move_velocity_, e.T, e.Tc));
    } else if (e.type == 4) {
      // the thermostat's degrees of freedom are ndeg = 3 (N - N_fixed - N_move) (ensemble_bdp.cu:87-95,
      // counted by Ensemble_BDP_B200 at its first step): at least one atom must be integrated
      int n_integrated = N;
      if (fixed_group_ >= 0)
        n_integrated -= model_.group[fixed_method_].cpu_size[fixed_group_];
      if (move_group_ >= 0)
        n_integrated -= model_.group[move_method_].cpu_size[move_group_];
      if (n_integrated < 1)
        input_error("nvt_bdp needs at least one atom outside the fixed and moving groups.");
      ensemble_.reset(new Ensemble_BDP_B200(4, move_group_, move_velocity_, e.T, e.Tc,
                                            e.has_seed ? e.seed : bdp_seed()));
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
      } else {
        ensemble_.reset(new Ensemble_HEAT_BDP_B200(23, N, g0.cpu_size, g0.contents.data(), e.source, e.sink,
                                                   e.T, e.Tc, e.dT, bdp_seed()));
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

  // the MT19937 seed of nvt_bdp and heat_bdp: the reference uses 12345678 under -DDEBUG and the clock
  // otherwise (ensemble_bdp.cu:31-37); B200MD_DEBUG_SEED=1 selects the former for trajectory parity
  static unsigned bdp_seed()
  {
    return std::getenv("B200MD_DEBUG_SEED") ? 12345678u
                                            : (unsigned)std::chrono::system_clock::now().time_since_epoch().count();
  }

  void perform_a_run(int number_of_steps)
  {
    if (!has_potential_ || ensemble_spec_.type < 0)
      input_error("'potential' and 'ensemble' must precede 'run'.");
    build_ensemble();
    if (!state_on_gpu_)
      upload_state();
    Atom& a = model_.atom;
    const int N = a.number_of_atoms;
    // the first force evaluation is outside the timed loop, as in run.cu:217-248
    force_.compute(model_.box, a.position_per_atom, a.type, a.potential_per_atom, a.force_per_atom,
                   a.virial_per_atom);
    force_.potentials[0]->check();
    measure_.preprocess(ctx_, number_of_steps);
    const bool unwrap = unwrapped_.size() > 0; // once a measurement has started tracking them
    position_old_.resize(unwrapped_.size());
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
      global_time_ += time_step_;
      measure_.process(ctx_, step);
    }
    B2H_CHECK(cudaDeviceSynchronize());
    force_.potentials[0]->check();
    const auto t1 = std::chrono::high_resolution_clock::now();
    const double sec = std::chrono::duration<double>(t1 - t0).count();
    printf("Time used for this run = %g second.\n", sec);
    printf("Speed of this run = %g atom*step/second.\n", N * (double)number_of_steps / sec);
    measure_.postprocess(ctx_);
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

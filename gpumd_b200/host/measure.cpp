// measure.cpp -- one Property per measurement and dump keyword of the driver: each parses its keyword
// line, creates its libb200md handle after the first force evaluation of a run, samples after every
// step and writes its files in the reference's formats (src/measure/*.cu).
#include "measure.h"
#include <algorithm>

namespace
{

// a create call's status: a rejected argument is an input error, anything else a library failure
void check_create(const char* keyword, int rc)
{
  if (rc == B200MD_ERR_ARG)
    input_error(std::string(keyword) + ": " + b200md_last_error());
  if (rc != B200MD_OK)
    b2h_fail(keyword);
}

FILE* open_output(const std::string& name, const char* mode)
{
  FILE* fid = fopen(name.c_str(), mode);
  if (!fid)
    input_error("Failed to open " + name + ".");
  return fid;
}

// the time between two rows of a correlation, in ps
double dt_in_ps(const MeasureContext& ctx, int sample_interval)
{
  return ctx.time_step * sample_interval * TIME_UNIT_CONVERSION / 1000.0;
}

// the cell and output-interval lines of the shc.out, sdc.out and msd*.out headers
void write_cell_header(FILE* fid, const double* h, double dt)
{
  fprintf(fid, "# cell %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e %.10e\n", h[0], h[3], h[6], h[1], h[4],
          h[7], h[2], h[5], h[8]);
  fprintf(fid, "# dt_output %.10e ps\n", dt);
}

// the sampling and output groups of a correlation keyword; group_method -1: the whole system
struct CorrSpec {
  int sample_interval = 0, Nc = 0, group_method = -1, group_id = -1;
  bool all_groups = false; // MSD's `all_groups m`
};

// the sample interval and Nc that DOS, SDC and MSD start with
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
void parse_group(const MeasureContext& ctx, const std::vector<std::string>& t, bool allow_all_groups, size_t& k,
                 CorrSpec& c)
{
  if (k + 3 > t.size())
    input_error("Not enough arguments for option 'group'.");
  if (!valid_int(t[k + 1], &c.group_method))
    input_error("Grouping method should be an integer.");
  if (c.group_method < 0)
    input_error("Grouping method should >= 0.");
  if (c.group_method >= (int)ctx.model.group.size())
    input_error("Grouping method should < number of grouping methods.");
  if (!valid_int(t[k + 2], &c.group_id))
    input_error("Group ID should be an integer.");
  if (c.group_id >= ctx.model.group[c.group_method].number)
    input_error("Group ID should < number of groups.");
  if (c.group_id < 0 && !allow_all_groups)
    input_error("group ID should >= 0.");
  printf("    grouping method is %d and group ID is %d.\n", c.group_method, c.group_id);
  k += 2;
}

// the output groups of a correlation keyword as (sizes, contents): the whole system, one group, or
// every group of the method (`group m -1` for DOS, `all_groups m` for MSD), or for SHC's `group m -1`
// every group except 0 (shc.cu:204-205)
const int* corr_groups(const MeasureContext& ctx, const CorrSpec& c, std::vector<int>& sizes,
                       bool except_group_0 = false)
{
  sizes.assign(1, ctx.model.atom.number_of_atoms);
  if (c.group_method < 0)
    return nullptr; // the whole system in atom order
  const Group& g = ctx.model.group[c.group_method];
  if (c.all_groups || c.group_id < 0) {
    const int first = except_group_0 ? 1 : 0;
    sizes.assign(g.cpu_size.begin() + first, g.cpu_size.end());
    return g.contents.data() + g.cpu_size_sum[first]; // the groups are contiguous there
  }
  sizes.assign(1, g.cpu_size[c.group_id]);
  return g.contents.data() + g.cpu_size_sum[c.group_id];
}

// compute_hac sample_interval Nc output_interval (hac.cu:262-300)
class ComputeHac : public Property
{
public:
  ComputeHac(const MeasureContext&, const std::vector<std::string>& t)
  {
    if (t.size() != 4)
      input_error("compute_hac should have 3 parameters.");
    interval_ = std::atoi(t[1].c_str());
    Nc_ = std::atoi(t[2].c_str());
    output_interval_ = std::atoi(t[3].c_str());
    if (interval_ <= 0 || Nc_ <= 0 || output_interval_ <= 0)
      input_error("compute_hac parameters should be positive integers.");
    printf("Compute HAC.\n    sample interval is %d.\n    Nc is %d\n    output_interval is %d\n", interval_, Nc_,
           output_interval_);
  }
  ~ComputeHac() override { b200md_hac_destroy(hac_); }
  void preprocess(const MeasureContext&, int number_of_steps) override
  {
    check_create("compute_hac", b200md_hac_create(number_of_steps, interval_, Nc_, &hac_));
  }
  void process(const MeasureContext& ctx, int step) override
  {
    Atom& a = ctx.model.atom;
    if (b200md_hac_sample(hac_, step, a.number_of_atoms, a.number_of_atoms, a.virial_per_atom.data(),
                          a.velocity_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_hac");
  }
  // HAC::postprocess, hac.cu:186-258: hac.out = t(ps), 5 hac averages, 5 rtc averages
  void postprocess(const MeasureContext& ctx) override
  {
    const int Nc = Nc_, oi = output_interval_;
    std::vector<double> h((size_t)5 * Nc), r((size_t)5 * Nc);
    if (b200md_hac_finish(hac_, ctx.time_step, ctx.temperature, ctx.model.box.get_volume(), h.data(), r.data(),
                          nullptr) != B200MD_OK)
      b2h_fail("compute_hac");
    const double dt = dt_in_ps(ctx, interval_);
    FILE* fid = open_output("hac.out", "a");
    for (int nd = 0; nd < Nc / oi; ++nd) {
      const int nc = nd * oi;
      fprintf(fid, "%25.15e", (nc + oi * 0.5) * dt);
      for (int pass = 0; pass < 2; ++pass)
        for (int k = 0; k < 5; ++k) {
          double ave = 0.0;
          for (int m = 0; m < oi; ++m)
            ave += (pass == 0 ? h : r)[(size_t)Nc * k + nc + m];
          fprintf(fid, "%25.15e", ave / oi);
        }
      fprintf(fid, "\n");
    }
    fclose(fid);
  }

private:
  int interval_ = 0, Nc_ = 0, output_interval_ = 1;
  b200md_hac* hac_ = nullptr;
};

// compute_hnemd output_interval fe_x fe_y fe_z (hnemd_kappa.cu:142-184).  The driving force is in
// force already for the evaluation before the loop (run.cu:217-248); Force::finalize ends it.
class ComputeHnemd : public Property
{
public:
  ComputeHnemd(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute thermal conductivity using the HNEMD method.\n");
    if (t.size() != 5)
      input_error("compute_hnemd should have 4 parameters.");
    if (!valid_int(t[1], &output_interval_))
      input_error("output_interval for HNEMD should be an integer number.");
    if (output_interval_ < 1)
      input_error("output_interval for HNEMD should be larger than 0.");
    const char* names[3] = {"fe_x", "fe_y", "fe_z"};
    for (int d = 0; d < 3; ++d)
      if (!valid_real(t[2 + d], &fe_[d]))
        input_error(std::string(names[d]) + " for HNEMD should be a real number.");
    if (ctx.force.hnemd_on()) // Force::set_hnemd_parameters, force.cu:344-346
      input_error("Cannot have more than one HNEMD method within one run.");
    printf("    output_interval = %d\n    fe = (%g, %g, %g) /A\n", output_interval_, fe_[0], fe_[1], fe_[2]);
    ctx.force.set_hnemd(fe_);
  }
  ~ComputeHnemd() override { b200md_hnemd_destroy(hnemd_); }
  void preprocess(const MeasureContext&, int) override
  {
    check_create("compute_hnemd", b200md_hnemd_create(output_interval_, fe_, &hnemd_));
  }
  bool writes_at(int step) const override { return (step + 1) % output_interval_ == 0; }
  void process(const MeasureContext& ctx, int step) override
  {
    Atom& a = ctx.model.atom;
    if (b200md_hnemd_sample(hnemd_, step, a.number_of_atoms, a.number_of_atoms, a.virial_per_atom.data(),
                            a.velocity_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_hnemd");
    if (!writes_at(step))
      return;
    double kappa[5]; // hnemd_kappa.cu:108-131
    if (b200md_hnemd_take(hnemd_, ctx.model.box.get_volume(), ctx.temperature, kappa, nullptr, nullptr) !=
        B200MD_OK)
      b2h_fail("compute_hnemd");
    FILE* fid = open_output("kappa.out", "a");
    for (int k = 0; k < 5; ++k)
      fprintf(fid, "%25.15f", kappa[k]);
    fprintf(fid, "\n");
    fclose(fid);
  }

private:
  int output_interval_ = 0;
  double fe_[3] = {0.0, 0.0, 0.0};
  b200md_hnemd* hnemd_ = nullptr;
};

// compute grouping_method sample_interval output_interval quantities... (Compute::parse, compute.cu:595-660)
class Compute : public Property
{
public:
  Compute(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute space and/or time average of:\n");
    if (t.size() < 5)
      input_error("compute should have at least 4 parameters.");
    if (!valid_int(t[1], &grouping_method_))
      input_error("grouping method of compute should be integer.");
    if (grouping_method_ < 0)
      input_error("grouping method should >= 0.");
    if (grouping_method_ >= (int)ctx.model.group.size())
      input_error("grouping method exceeds the bound.");
    if (!valid_int(t[2], &sample_interval_))
      input_error("sampling interval of compute should be integer.");
    if (sample_interval_ <= 0)
      input_error("sampling interval of compute should > 0.");
    if (!valid_int(t[3], &output_interval_))
      input_error("output interval of compute should be integer.");
    if (output_interval_ <= 0)
      input_error("output interval of compute should > 0.");
    static const char* names[7] = {"temperature", "potential", "force", "virial", "jp", "jk", "momentum"};
    for (size_t k = 4; k < t.size(); ++k) {
      int q = 0;
      while (q < 7 && t[k] != names[q])
        ++q;
      if (q == 7)
        input_error("Invalid property for compute.");
      mask_ |= 1u << q;
      printf("    %s\n", names[q]);
    }
    printf("    using grouping method %d.\n", grouping_method_);
    printf("    with sampling interval %d.\n", sample_interval_);
    printf("    and output interval %d.\n", output_interval_);
  }
  ~Compute() override { b200md_group_compute_destroy(cp_); }
  void preprocess(const MeasureContext& ctx, int) override // Compute::preprocess, compute.cu:31-67
  {
    const Group& g = ctx.model.group[grouping_method_];
    check_create("compute", b200md_group_compute_create(ctx.model.atom.number_of_atoms, g.number,
                                                        g.cpu_size.data(), g.contents.data(), mask_, &cp_));
    num_values_ = b200md_group_compute_columns(cp_) * g.number;
  }
  bool writes_at(int step) const override
  {
    return (step + 1) % sample_interval_ == 0 && ((step + 1) / sample_interval_) % output_interval_ == 0;
  }
  void process(const MeasureContext& ctx, int step) override // Compute::process, compute.cu:351-538
  {
    if ((step + 1) % sample_interval_ != 0)
      return;
    Atom& a = ctx.model.atom;
    if (b200md_group_compute_sample(cp_, a.number_of_atoms, a.number_of_atoms, a.mass.data(),
                                    a.potential_per_atom.data(), a.force_per_atom.data(), a.virial_per_atom.data(),
                                    a.velocity_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("compute");
    if (writes_at(step))
      write(ctx);
  }

private:
  // Compute::output_results, compute.cu:540-561: the averages, then (with temperature) the energy
  // transferred to the source and sink baths.  A non-heat ensemble prints 0 for both (the reference
  // prints its never-initialised energy_transferred there).
  void write(const MeasureContext& ctx)
  {
    std::vector<double> v(num_values_);
    if (b200md_group_compute_take(cp_, output_interval_, v.data(), nullptr) != B200MD_OK)
      b2h_fail("compute");
    FILE* fid = open_output("compute.out", "a");
    for (double x : v)
      fprintf(fid, "%15.6e", x);
    if (mask_ & B200MD_COMPUTE_TEMPERATURE) {
      double e[2] = {0.0, 0.0};
      if (auto* heat = dynamic_cast<Ensemble_HEAT_B200*>(ctx.ensemble.get())) {
        heat->read_energy_transferred();
        e[0] = heat->b2_energy_transferred[0];
        e[1] = heat->b2_energy_transferred[1];
      }
      fprintf(fid, "%15.6e%15.6e", e[0], e[1]);
    }
    fprintf(fid, "\n");
    fclose(fid);
  }
  int grouping_method_ = 0, sample_interval_ = 0, output_interval_ = 0, num_values_ = 0;
  unsigned mask_ = 0;
  b200md_group_compute* cp_ = nullptr;
};

// compute_shc sample_interval Nc direction num_omega max_omega [group m id] (shc.cu:466-542)
class ComputeShc : public Property
{
public:
  ComputeShc(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute SHC.\n");
    if (t.size() != 6 && t.size() != 9)
      input_error("compute_shc should have 5 or 8 parameters.");
    if (!valid_int(t[1], &c_.sample_interval))
      input_error("Sampling interval for SHC should be an integer.");
    if (c_.sample_interval < 1)
      input_error("Sampling interval for SHC should >= 1.");
    if (c_.sample_interval > 50)
      input_error("Sampling interval for SHC should <= 50 (trust me).");
    if (!valid_int(t[2], &c_.Nc))
      input_error("Nc for SHC should be an integer.");
    if (c_.Nc < 100)
      input_error("Nc for SHC should >= 100 (trust me).");
    if (c_.Nc > 1000)
      input_error("Nc for SHC should <= 1000 (trust me).");
    if (!valid_int(t[3], &direction_))
      input_error("direction for SHC should be an integer.");
    if (direction_ < 0 || direction_ > 2)
      input_error("Transport direction should be x or y or z.");
    if (!valid_int(t[4], &num_omega_))
      input_error("num_omega for SHC should be an integer.");
    if (num_omega_ < 0)
      input_error("num_omega for SHC should >= 0.");
    if (!valid_real(t[5], &omega_max_))
      input_error("max_omega for SHC should be a number.");
    if (omega_max_ <= 0)
      input_error("max_omega for SHC should > 0.");
    for (size_t k = 6; k < t.size(); k++) {
      if (t[k] != "group")
        input_error("Unrecognized argument in compute_shc.");
      parse_group(ctx, t, true, k, c_);
      if (c_.group_id < -1)
        input_error("group ID should >= -1 for computing SHC.");
      if (c_.group_id == -1 && ctx.model.group[c_.group_method].number < 2)
        input_error("compute_shc with group ID -1 needs a grouping method with at least two groups.");
    }
    printf("    sampling interval %d, Nc %d, direction %d, num_omega %d, max_omega %g\n", c_.sample_interval, c_.Nc,
           direction_, num_omega_, omega_max_);
  }
  ~ComputeShc() override { b200md_shc_destroy(shc_); }
  void preprocess(const MeasureContext& ctx, int number_of_steps) override
  {
    std::vector<int> sizes;
    const int* contents = corr_groups(ctx, c_, sizes, true);
    num_groups_ = (int)sizes.size();
    check_create("compute_shc", b200md_shc_create(c_.Nc, c_.sample_interval, direction_, number_of_steps,
                                                  num_groups_, sizes.data(), contents, &shc_));
  }
  void process(const MeasureContext& ctx, int step) override
  {
    Atom& a = ctx.model.atom;
    if (b200md_shc_sample(shc_, step, a.number_of_atoms, a.number_of_atoms, a.virial_per_atom.data(),
                          a.velocity_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_shc");
  }
  // SHC::postprocess, shc.cu:398-464: header, then per output group 2Nc-1 correlation rows and
  // num_omega spectrum rows (the cell at the end of the run)
  void postprocess(const MeasureContext& ctx) override
  {
    const int Nc = c_.Nc, Nk = 2 * Nc - 1, ng = num_groups_;
    std::vector<double> ki((size_t)ng * Nk), ko(ki.size());
    std::vector<double> si((size_t)ng * num_omega_ + 1), so(si.size());
    if (b200md_shc_finish(shc_, ctx.time_step, num_omega_, omega_max_, ki.data(), ko.data(), si.data(), so.data(),
                          nullptr) != B200MD_OK)
      b2h_fail("compute_shc");
    const double dt = dt_in_ps(ctx, c_.sample_interval);
    const double d_omega = omega_max_ / num_omega_;
    FILE* fid = open_output("shc.out", "a");
    fprintf(fid, "# compute_shc %d %d %d %d %g", c_.sample_interval, Nc, direction_, num_omega_, omega_max_);
    if (c_.group_method >= 0)
      fprintf(fid, " group %d %d", c_.group_method, c_.group_id);
    fprintf(fid, "\n# format_version 1\n# num_atoms %d\n", ctx.model.atom.number_of_atoms);
    write_cell_header(fid, ctx.model.box.cpu_h, dt);
    fprintf(fid, "# num_correlation_rows %d\n", Nk);
    fprintf(fid, "# num_frequency_rows %d\n", num_omega_);
    if (c_.group_method >= 0 && c_.group_id == -1)
      fprintf(fid, "# num_output_groups %d\n", ng);
    fprintf(fid, "# columns_correlation time_ps ki ko\n");
    fprintf(fid, "# columns_shc omega_THz shc_i shc_o\n");
    for (int g = 0; g < ng; ++g) {
      for (int nc = 0; nc < Nk; ++nc) // ki, ko in A eV/ps
        fprintf(fid, "%g %g %g\n", (nc + 1 - Nc) * dt, ki[(size_t)g * Nk + nc], ko[(size_t)g * Nk + nc]);
      for (int nw = 0; nw < num_omega_; ++nw) // shc_i, shc_o in A eV = A eV/ps/THz
        fprintf(fid, "%g %g %g\n", (nw + 1) * d_omega, si[(size_t)g * num_omega_ + nw],
                so[(size_t)g * num_omega_ + nw]);
    }
    fclose(fid);
  }

private:
  CorrSpec c_;
  int direction_ = 0, num_omega_ = 0, num_groups_ = 1;
  double omega_max_ = 0.0;
  b200md_shc* shc_ = nullptr;
};

// compute_dos sample_interval Nc omega_max [group m id] [num_dos_points n] (DOS::parse, dos.cu:153-202)
class ComputeDos : public Property
{
public:
  ComputeDos(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute phonon DOS.\n");
    if (t.size() < 4)
      input_error("compute_dos should have at least 3 parameters.");
    if (t.size() > 9)
      input_error("compute_dos has too many parameters.");
    parse_interval_nc(t, c_);
    if (!valid_real(t[3], &omega_max_))
      input_error("maximal angular frequency should be a number.");
    if (omega_max_ <= 0)
      input_error("maximal angular frequency should be positive.");
    printf("    maximal angular frequency is %g THz.\n", omega_max_);
    num_dos_points_ = c_.Nc;
    for (size_t k = 4; k < t.size(); k++) {
      if (t[k] == "group") {
        parse_group(ctx, t, true, k, c_);
      } else if (t[k] == "num_dos_points") {
        if (k + 2 > t.size())
          input_error("Not enough arguments for option 'num_dos_points'.");
        if (!valid_int(t[k + 1], &num_dos_points_))
          input_error("number of DOS points should be an integer.");
        if (num_dos_points_ < 1)
          input_error("number of DOS points must be > 0.");
        k += 1;
        printf("    num_dos_points is %d.\n", num_dos_points_);
      } else {
        input_error("Unrecognized argument in compute_dos.");
      }
    }
  }
  ~ComputeDos() override { b200md_dos_destroy(dos_); }
  void preprocess(const MeasureContext& ctx, int number_of_steps) override // dos.cu:204-218
  {
    std::vector<int> sizes;
    const int* contents = corr_groups(ctx, c_, sizes);
    num_groups_ = (int)sizes.size();
    Atom& a = ctx.model.atom;
    check_create("compute_dos", b200md_dos_create(c_.Nc, c_.sample_interval, number_of_steps, ctx.time_step,
                                                  omega_max_, num_dos_points_, num_groups_, sizes.data(), contents,
                                                  a.number_of_atoms, a.mass.data(), &dos_));
  }
  void process(const MeasureContext& ctx, int step) override
  {
    const int N = ctx.model.atom.number_of_atoms;
    if (b200md_dos_sample(dos_, step, N, N, ctx.model.atom.velocity_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_dos");
  }
  // DOS::output_vac / output_dos, dos.cu:429-448,483-503: appended, no header, group after group
  void postprocess(const MeasureContext& ctx) override
  {
    const int Nc = c_.Nc, nw = num_dos_points_;
    std::vector<double> mvac((size_t)num_groups_ * 3 * Nc), d((size_t)num_groups_ * 3 * nw);
    if (b200md_dos_finish(dos_, mvac.data(), d.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_dos");
    const double dt = dt_in_ps(ctx, c_.sample_interval);
    FILE* fid = open_output("mvac.out", "a");
    for (int g = 0; g < num_groups_; ++g) {
      const double* v = mvac.data() + (size_t)g * 3 * Nc;
      for (int nc = 0; nc < Nc; nc++)
        fprintf(fid, "%g %g %g %g\n", nc * dt, v[nc], v[Nc + nc], v[2 * Nc + nc]);
    }
    fclose(fid);
    const double d_omega = omega_max_ / nw;
    fid = open_output("dos.out", "a");
    for (int g = 0; g < num_groups_; ++g) {
      const double* v = d.data() + (size_t)g * 3 * nw;
      for (int k = 0; k < nw; k++)
        fprintf(fid, "%g %g %g %g\n", d_omega + d_omega * k, v[k], v[nw + k], v[2 * nw + k]);
    }
    fclose(fid);
  }

private:
  CorrSpec c_;
  double omega_max_ = 0.0;
  int num_dos_points_ = 0, num_groups_ = 1;
  b200md_dos* dos_ = nullptr;
};

// compute_sdc sample_interval Nc [group m id] (SDC::parse, sdc.cu:300-338)
class ComputeSdc : public Property
{
public:
  ComputeSdc(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute self diffusion coefficient (SDC).\n");
    if (t.size() < 3)
      input_error("compute_sdc should have at least 2 parameters.");
    if (t.size() > 6)
      input_error("compute_sdc has too many parameters.");
    parse_interval_nc(t, c_);
    for (size_t k = 3; k < t.size(); k++) {
      if (t[k] == "group")
        parse_group(ctx, t, false, k, c_);
      else
        input_error("Unrecognized argument in compute_sdc.");
    }
  }
  ~ComputeSdc() override { b200md_sdc_destroy(sdc_); }
  void preprocess(const MeasureContext& ctx, int number_of_steps) override // sdc.cu:132-155
  {
    std::vector<int> sizes;
    const int* contents = corr_groups(ctx, c_, sizes);
    num_atoms_ = sizes[0];
    check_create("compute_sdc", b200md_sdc_create(c_.Nc, c_.sample_interval, number_of_steps, ctx.time_step,
                                                  (int)sizes.size(), sizes.data(), contents, &sdc_));
  }
  void process(const MeasureContext& ctx, int step) override
  {
    const int N = ctx.model.atom.number_of_atoms;
    if (b200md_sdc_sample(sdc_, step, N, N, ctx.model.atom.velocity_per_atom.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_sdc");
  }
  // SDC::postprocess, sdc.cu:259-285 (the cell at the end of the run)
  void postprocess(const MeasureContext& ctx) override
  {
    const int Nc = c_.Nc;
    std::vector<double> vac((size_t)3 * Nc), s((size_t)3 * Nc);
    if (b200md_sdc_finish(sdc_, vac.data(), s.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_sdc");
    const double dt = dt_in_ps(ctx, c_.sample_interval);
    FILE* fid = open_output("sdc.out", "a");
    fprintf(fid, "# compute_sdc %d %d", c_.sample_interval, Nc);
    if (c_.group_method >= 0)
      fprintf(fid, " group %d %d", c_.group_method, c_.group_id);
    fprintf(fid, "\n# format_version 1\n# num_atoms %d\n", num_atoms_);
    write_cell_header(fid, ctx.model.box.cpu_h, dt);
    fprintf(fid, "# columns time_ps vacx vacy vacz sdcx sdcy sdcz\n");
    for (int nc = 0; nc < Nc; nc++)
      fprintf(fid, "%g %g %g %g %g %g %g\n", nc * dt, vac[nc], vac[Nc + nc], vac[2 * Nc + nc], s[nc], s[Nc + nc],
              s[2 * Nc + nc]);
    fclose(fid);
  }

private:
  CorrSpec c_;
  int num_atoms_ = 0;
  b200md_sdc* sdc_ = nullptr;
};

// compute_msd sample_interval Nc [group m id | all_groups m] [save_every n] (MSD::parse, msd.cu:481-541).
// all_groups reads the method after the keyword (the reference reads param[4], which is that position
// in the documented form `compute_msd <i> <Nc> all_groups <m>`)
class ComputeMsd : public Property
{
public:
  ComputeMsd(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute mean square displacement (MSD).\n");
    if (t.size() < 3)
      input_error("compute_msd should have at least 2 parameters.");
    if (t.size() > 8)
      input_error("compute_msd has too many parameters.");
    parse_interval_nc(t, c_);
    for (size_t k = 3; k < t.size(); k++) {
      if (t[k] == "group") {
        parse_group(ctx, t, false, k, c_);
      } else if (t[k] == "all_groups") {
        c_.all_groups = true;
        if (k + 2 > t.size() || !valid_int(t[k + 1], &c_.group_method))
          input_error("Grouping method should be an integer.");
        if (c_.group_method < 0)
          input_error("Grouping method should >= 0.");
        if (c_.group_method >= (int)ctx.model.group.size())
          input_error("Grouping method should < number of grouping methods.");
        printf("    will compute MSD for all groups in grouping %d.\n", c_.group_method);
        k += 1;
      } else if (t[k] == "save_every") {
        if (k + 2 > t.size() || !valid_int(t[k + 1], &save_every_))
          input_error("save_every should be an integer.");
        printf("    will save a copy of the MSD every %d steps.\n", save_every_);
        k += 1;
      } else {
        input_error("Unrecognized argument in compute_msd.");
      }
    }
    if (c_.all_groups && c_.group_method >= 0 && c_.group_id >= 0)
      input_error("Cannot compute MSD over a single group and all groups at the same time");
  }
  ~ComputeMsd() override { b200md_msd_destroy(msd_); }
  void preprocess(const MeasureContext& ctx, int number_of_steps) override // msd.cu:205-267
  {
    const Atom& a = ctx.model.atom;
    const int N = a.number_of_atoms;
    const int* contents = corr_groups(ctx, c_, sizes_);
    check_create("compute_msd", b200md_msd_create(c_.Nc, c_.sample_interval, number_of_steps, ctx.time_step,
                                                  (int)sizes_.size(), sizes_.data(), contents, &msd_));
    std::copy(ctx.model.box.cpu_h, ctx.model.box.cpu_h + 9, h_); // the cell at the start of the run
    num_atoms_ = c_.group_method >= 0 && !c_.all_groups ? sizes_[0] : N;
    if (ctx.unwrapped.size() < (size_t)3 * N) { // the first run with compute_msd (msd.cu:471-477)
      ctx.unwrapped.resize((size_t)3 * N);
      B2H_CHECK(cudaMemcpy(ctx.unwrapped.data(), a.position_per_atom.data(), sizeof(double) * 3 * N,
                           cudaMemcpyDeviceToDevice));
    }
  }
  void process(const MeasureContext& ctx, int step) override
  {
    const int N = ctx.model.atom.number_of_atoms;
    if (b200md_msd_sample(msd_, step, N, N, ctx.unwrapped.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_msd");
    // a copy every save_every steps, on time origins (msd.cu:355-360)
    if (save_every_ > 0 && (step + 1) % c_.sample_interval == 0 && step / c_.sample_interval >= c_.Nc - 1 &&
        (step + 1) % save_every_ == 0)
      write(ctx, "msd_step" + std::to_string(step + 1) + ".out");
  }
  void postprocess(const MeasureContext& ctx) override { write(ctx, "msd.out"); }

private:
  // MSD::write, msd.cu:365-449
  void write(const MeasureContext& ctx, const std::string& filename)
  {
    const int Nc = c_.Nc, ng = (int)sizes_.size();
    std::vector<double> m((size_t)ng * 3 * Nc), s(m.size());
    if (b200md_msd_finish(msd_, m.data(), s.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_msd");
    const double dt = dt_in_ps(ctx, c_.sample_interval);
    FILE* fid = open_output(filename, "a");
    fprintf(fid, "# compute_msd %d %d", c_.sample_interval, Nc);
    if (c_.all_groups)
      fprintf(fid, " all_groups %d", c_.group_method);
    else if (c_.group_method >= 0)
      fprintf(fid, " group %d %d", c_.group_method, c_.group_id);
    if (save_every_ > 0)
      fprintf(fid, " save_every %d", save_every_);
    fprintf(fid, "\n# format_version 1\n# num_atoms %d\n# num_groups %d\n# num_atoms_per_group", num_atoms_, ng);
    for (int g = 0; g < ng; ++g)
      fprintf(fid, " %d", sizes_[g]);
    fprintf(fid, "\n");
    write_cell_header(fid, h_, dt);
    fprintf(fid, "# columns time_ps");
    if (!c_.all_groups)
      fprintf(fid, " msdx msdy msdz sdcx sdcy sdcz");
    else
      for (int g = 0; g < ng; ++g)
        fprintf(fid, " msdx_%d msdy_%d msdz_%d sdcx_%d sdcy_%d sdcz_%d", g, g, g, g, g, g);
    fprintf(fid, "\n");
    for (int nc = 0; nc < Nc; nc++) {
      fprintf(fid, "%g", nc * dt);
      for (int g = 0; g < ng; g++) {
        const double* a = m.data() + (size_t)g * 3 * Nc;
        const double* b = s.data() + (size_t)g * 3 * Nc;
        fprintf(fid, "% g %g %g %g %g %g", a[nc], a[Nc + nc], a[2 * Nc + nc], b[nc], b[Nc + nc], b[2 * Nc + nc]);
      }
      fprintf(fid, "\n");
    }
    fclose(fid);
  }
  CorrSpec c_;
  int save_every_ = -1, num_atoms_ = 0;
  std::vector<int> sizes_;
  double h_[9];
  b200md_msd* msd_ = nullptr;
};

// compute_rdf rc num_bins interval (RDF::parse, rdf.cu:264-333).  The species are the types with at least
// one atom, in type-id order.  One deliberate difference: a run shorter than one interval is refused,
// where the reference divides by num_repeats = 0
class ComputeRdf : public Property
{
public:
  ComputeRdf(const MeasureContext& ctx, const std::vector<std::string>& t)
  {
    printf("Compute radial distribution function (RDF).\n");
    if (t.size() != 4)
      input_error("compute_rdf should have 3 parameters.");
    if (!valid_real(t[1], &rc_))
      input_error("radial cutoff should be a number.");
    if (rc_ <= 0)
      input_error("radial cutoff should be positive.");
    const Box& box = ctx.model.box;
    const double volume = box.get_volume();
    for (int d = 0; d < 3; ++d) { // every direction, open ones included (rdf.cu:283-292)
      if (rc_ > volume / area(box, d) / 2.5)
        input_error("The box has a thickness < 2.5 RDF radial cutoffs in a periodic direction.\n"
                    "                Please increase the periodic direction(s).");
    }
    printf("    radial cutoff %g.\n", rc_);
    if (!valid_int(t[2], &num_bins_))
      input_error("number of bins should be an integer.");
    if (num_bins_ <= 20)
      input_error("A larger nbins is recommended.");
    if (num_bins_ > 500)
      input_error("A smaller nbins is recommended.");
    printf("    radial cutoff will be divided into %d bins.\n", num_bins_);
    if (!valid_int(t[3], &interval_))
      input_error("interval step per sample should be an integer.");
    if (interval_ <= 0)
      input_error("interval step per sample should be positive.");
    printf("    RDF sample interval is %d step.\n", interval_);
    const Atom& a = ctx.model.atom;
    std::vector<int> size;
    for (int n = 0; n < a.number_of_atoms; ++n) {
      if (a.cpu_type[n] >= (int)size.size())
        size.resize(a.cpu_type[n] + 1, 0);
      ++size[a.cpu_type[n]];
    }
    for (int ty = 0; ty < (int)size.size(); ++ty) {
      if (size[ty] != 0) {
        type_index_.push_back(ty);
        num_atoms_.push_back(size[ty]);
      }
    }
    const int T = (int)type_index_.size();
    printf("    There are %d atom types in model.xyz.\n", T);
    for (int k = 0; k < T; ++k)
      printf("        Type %d has %d atoms.\n", type_index_[k], num_atoms_[k]);
    printf("    Will calculate one total RDF and %d partial RDFs.\n", T * (T + 1) / 2);
  }
  ~ComputeRdf() override { b200md_rdf_destroy(rdf_); }
  void preprocess(const MeasureContext& ctx, int number_of_steps) override // rdf.cu:163-176
  {
    num_repeats_ = number_of_steps / interval_;
    if (num_repeats_ < 1)
      input_error("compute_rdf: the run has fewer steps than one sample interval.");
    b200md_rdf_destroy(rdf_);
    rdf_ = nullptr;
    check_create("compute_rdf", b200md_rdf_create(rc_, num_bins_, (int)type_index_.size(), type_index_.data(),
                                                  num_atoms_.data(), ctx.model.atom.number_of_atoms, &rdf_));
  }
  void process(const MeasureContext& ctx, int step) override // rdf.cu:178-202
  {
    if ((step + 1) % interval_ != 0)
      return;
    const Box& box = ctx.model.box;
    int pbc[3];
    box.pbc(pbc);
    const Atom& a = ctx.model.atom;
    if (b200md_rdf_sample(rdf_, box.cpu_h, pbc, a.type.data(), a.position_per_atom.data(), a.number_of_atoms,
                          nullptr) != B200MD_OK)
      b2h_fail("compute_rdf");
  }
  // RDF::postprocess, rdf.cu:204-251: appended to rdf.out
  void postprocess(const MeasureContext& ctx) override
  {
    const int T = (int)type_index_.size(), R = 1 + T * (T + 1) / 2;
    std::vector<double> g((size_t)num_bins_ * R);
    if (b200md_rdf_finish(rdf_, num_repeats_, g.data(), nullptr) != B200MD_OK)
      b2h_fail("compute_rdf");
    const Atom& a = ctx.model.atom;
    std::vector<std::string> symbol(T);
    for (int k = 0; k < T; ++k) {
      for (int n = 0; n < a.number_of_atoms; ++n) {
        if (a.cpu_type[n] == type_index_[k]) {
          symbol[k] = a.cpu_atom_symbol[n];
          break;
        }
      }
    }
    FILE* fid = open_output("rdf.out", "a");
    fprintf(fid, "#radius total");
    for (int p = 0; p < T; p++)
      for (int q = p; q < T; q++)
        fprintf(fid, " %s-%s", symbol[p].c_str(), symbol[q].c_str());
    fprintf(fid, "\n");
    const double dr = rc_ / num_bins_;
    for (int bin = 0; bin < num_bins_; bin++) {
      fprintf(fid, "%.5f", bin * dr + dr / 2);
      for (int k = 0; k < R; ++k)
        fprintf(fid, " %.5f", g[(size_t)bin * R + k]);
      fprintf(fid, "\n");
    }
    fclose(fid);
  }

private:
  // Box::get_area, box.cu:34-48
  static double area(const Box& box, int d)
  {
    const double* h = box.cpu_h;
    const double col[3][3] = {{h[0], h[3], h[6]}, {h[1], h[4], h[7]}, {h[2], h[5], h[8]}};
    const double* u = col[(d + 1) % 3];
    const double* w = col[(d + 2) % 3];
    const double s1 = u[1] * w[2] - u[2] * w[1];
    const double s2 = u[2] * w[0] - u[0] * w[2];
    const double s3 = u[0] * w[1] - u[1] * w[0];
    return sqrt(s1 * s1 + s2 * s2 + s3 * s3);
  }
  double rc_ = 0.0;
  int num_bins_ = 0, interval_ = 0, num_repeats_ = 0;
  std::vector<int> type_index_, num_atoms_;
  b200md_rdf* rdf_ = nullptr;
};

// dump_thermo interval: T, K, U, then sxx syy szz syz sxz sxy in GPa, then the box (dump_thermo.cu:73-129)
class DumpThermo : public Property
{
public:
  DumpThermo(const MeasureContext&, const std::vector<std::string>& t)
  {
    if (t.size() != 2 || std::atoi(t[1].c_str()) <= 0)
      input_error("dump_thermo should have 1 positive parameter (the interval).");
    interval_ = std::atoi(t[1].c_str());
  }
  void preprocess(const MeasureContext& ctx, int) override
  {
    fid_ = fopen("thermo.out", "a");
    fprintf(fid_, "# dump_thermo %d\n# format_version 1\n# num_atoms %d\n# dt_output %.10e fs\n", interval_,
            ctx.model.atom.number_of_atoms, ctx.time_step * interval_ * TIME_UNIT_CONVERSION);
    fprintf(fid_, "# columns T KE PE sxx syy szz syz sxz sxy ax ay az bx by bz cx cy cz\n");
  }
  bool writes_at(int step) const override { return (step + 1) % interval_ == 0; }
  void process(const MeasureContext& ctx, int step) override
  {
    if (!writes_at(step))
      return;
    double th[8];
    ctx.thermo.copy_to_host(th, 8);
    // the kinetic energy counts every atom but those of the fixed group (dump_thermo.cu:90-101)
    int N = ctx.model.atom.number_of_atoms;
    if (ctx.fixed_group >= 0)
      N -= ctx.model.group[ctx.fixed_method].cpu_size[ctx.fixed_group];
    const double* h = ctx.model.box.cpu_h;
    fprintf(fid_, "%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e", th[0], 1.5 * N * K_B * th[0],
            th[1], th[2] * PRESSURE_UNIT_CONVERSION, th[3] * PRESSURE_UNIT_CONVERSION,
            th[4] * PRESSURE_UNIT_CONVERSION, th[7] * PRESSURE_UNIT_CONVERSION, th[6] * PRESSURE_UNIT_CONVERSION,
            th[5] * PRESSURE_UNIT_CONVERSION);
    fprintf(fid_, "%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e%20.10e\n", h[0], h[3], h[6], h[1], h[4],
            h[7], h[2], h[5], h[8]);
  }
  void postprocess(const MeasureContext&) override
  {
    fclose(fid_);
    fid_ = nullptr;
  }

private:
  int interval_ = 0;
  FILE* fid_ = nullptr;
};

// dump_xyz interval file [precision single|double] [mass velocity force potential virial]: one frame of
// extended XYZ, header keys and value formats of dump_xyz.cu:68-437
class DumpXyz : public Property
{
public:
  DumpXyz(const MeasureContext&, const std::vector<std::string>& t)
  {
    if (t.size() < 3)
      input_error("dump_xyz should have at least 2 parameters.");
    interval_ = std::atoi(t[1].c_str());
    if (interval_ <= 0)
      input_error("dump interval should > 0.");
    file_ = t[2];
    if (file_.back() == '*') {
      separated_ = true;
      file_.pop_back();
    }
    for (size_t m = 3; m < t.size(); ++m) {
      if (t[m] == "precision") {
        if (m + 1 >= t.size() || (t[m + 1] != "single" && t[m + 1] != "double"))
          input_error("Invalid precision.");
        precision_ = t[++m] == "single" ? 1 : 2;
      } else if (t[m] == "mass") {
        mass_ = true;
      } else if (t[m] == "velocity") {
        velocity_ = true;
      } else if (t[m] == "force") {
        force_ = true;
      } else if (t[m] == "potential") {
        potential_ = true;
      } else if (t[m] == "virial") {
        virial_ = true;
      } else {
        input_error("Unrecognized argument in dump_xyz (supported: precision, mass, velocity, force, "
                    "potential, virial).");
      }
    }
  }
  bool writes_at(int step) const override { return (step + 1) % interval_ == 0; }
  void process(const MeasureContext& ctx, int step) override
  {
    if (!writes_at(step))
      return;
    Atom& a = ctx.model.atom;
    const Box& box = ctx.model.box;
    const int N = a.number_of_atoms;
    const char* fmt = precision_ == 1 ? " %.9g" : " %.17g";
    std::vector<double> pos((size_t)3 * N), vel, frc, pe, vir((size_t)9 * N);
    a.position_per_atom.copy_to_host(pos.data());
    a.virial_per_atom.copy_to_host(vir.data());
    if (velocity_) {
      vel.resize((size_t)3 * N);
      a.velocity_per_atom.copy_to_host(vel.data());
    }
    if (force_) {
      frc.resize((size_t)3 * N);
      a.force_per_atom.copy_to_host(frc.data());
    }
    if (potential_) {
      pe.resize(N);
      a.potential_per_atom.copy_to_host(pe.data());
    }
    double th[8];
    ctx.thermo.copy_to_host(th, 8);
    const std::string name = separated_ ? file_ + std::to_string(step + 1) : file_;
    FILE* fid = open_output(name, separated_ ? "w" : "a");
    auto tensor = [&](const char* key, const double* v9) {
      fprintf(fid, " %s=\"", key);
      for (int k = 0; k < 9; ++k)
        fprintf(fid, k == 0 ? fmt + 1 : fmt, v9[k]);
      fprintf(fid, "\"");
    };
    fprintf(fid, "%d\n", N);
    fprintf(fid, "Time=%.8f", ctx.global_time * TIME_UNIT_CONVERSION);
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
    if (mass_)
      fprintf(fid, ":mass:R:1");
    if (velocity_)
      fprintf(fid, ":vel:R:3");
    if (force_)
      fprintf(fid, ":forces:R:3");
    if (potential_)
      fprintf(fid, ":energy_atom:R:1");
    if (virial_)
      fprintf(fid, ":virial:R:9");
    fprintf(fid, "\n");
    const int vidx[9] = {0, 3, 4, 6, 1, 5, 7, 8, 2}; // GPUMD component order -> row-major 3x3
    for (int n = 0; n < N; ++n) {
      fprintf(fid, "%s", a.cpu_atom_symbol[n].c_str());
      for (int k = 0; k < 3; ++k)
        fprintf(fid, fmt, pos[n + (size_t)N * k]);
      if (mass_)
        fprintf(fid, fmt, a.cpu_mass[n]);
      if (velocity_)
        for (int k = 0; k < 3; ++k)
          fprintf(fid, fmt, vel[n + (size_t)N * k] / TIME_UNIT_CONVERSION);
      if (force_)
        for (int k = 0; k < 3; ++k)
          fprintf(fid, fmt, frc[n + (size_t)N * k]);
      if (potential_)
        fprintf(fid, fmt, pe[n]);
      if (virial_)
        for (int k = 0; k < 9; ++k)
          fprintf(fid, fmt, vir[n + (size_t)N * vidx[k]]);
      fprintf(fid, "\n");
    }
    fclose(fid);
  }

private:
  int interval_ = 0;
  std::string file_;
  bool separated_ = false;
  int precision_ = 2; // 1: "%.9g", 2: "%.17g"
  bool mass_ = false, velocity_ = false, force_ = false, potential_ = false, virial_ = false;
};

// dump_restart interval: restart.xyz, the model.xyz the next run can start from (dump_restart.cu:83-139)
class DumpRestart : public Property
{
public:
  DumpRestart(const MeasureContext&, const std::vector<std::string>& t)
  {
    if (t.size() != 2 || std::atoi(t[1].c_str()) <= 0)
      input_error("dump_restart should have 1 positive parameter (the interval).");
    interval_ = std::atoi(t[1].c_str());
  }
  bool writes_at(int step) const override { return (step + 1) % interval_ == 0; }
  void process(const MeasureContext& ctx, int step) override
  {
    if (!writes_at(step))
      return;
    const Atom& a = ctx.model.atom;
    const Box& box = ctx.model.box;
    const int N = a.number_of_atoms;
    std::vector<double> pos((size_t)3 * N), vel((size_t)3 * N);
    a.position_per_atom.copy_to_host(pos.data());
    a.velocity_per_atom.copy_to_host(vel.data());
    FILE* fid = open_output("restart.xyz", "w");
    const double* h = box.cpu_h;
    fprintf(fid, "%d\n", N);
    fprintf(fid, "pbc=\"%c %c %c\" ", box.pbc_x ? 'T' : 'F', box.pbc_y ? 'T' : 'F', box.pbc_z ? 'T' : 'F');
    fprintf(fid, "Lattice=\"%g %g %g %g %g %g %g %g %g\" ", h[0], h[3], h[6], h[1], h[4], h[7], h[2], h[5], h[8]);
    fprintf(fid, "Properties=species:S:1:pos:R:3:mass:R:1:vel:R:3\n");
    for (int n = 0; n < N; ++n)
      fprintf(fid, "%s %g %g %g %g %g %g %g \n", a.cpu_atom_symbol[n].c_str(), pos[n], pos[n + (size_t)N],
              pos[n + 2 * (size_t)N], a.cpu_mass[n], vel[n] / TIME_UNIT_CONVERSION,
              vel[n + (size_t)N] / TIME_UNIT_CONVERSION, vel[n + 2 * (size_t)N] / TIME_UNIT_CONVERSION);
    fclose(fid);
  }

private:
  int interval_ = 0;
};

template <class P>
std::unique_ptr<Property> make(const MeasureContext& ctx, const std::vector<std::string>& t)
{
  return std::make_unique<P>(ctx, t);
}

// every keyword, in the order its property samples within a step
const struct {
  const char* keyword;
  std::unique_ptr<Property> (*make)(const MeasureContext&, const std::vector<std::string>&);
} KEYWORDS[] = {
  {"compute_hac", make<ComputeHac>},   {"compute_hnemd", make<ComputeHnemd>}, {"compute", make<Compute>},
  {"compute_shc", make<ComputeShc>},   {"compute_dos", make<ComputeDos>},     {"compute_sdc", make<ComputeSdc>},
  {"compute_msd", make<ComputeMsd>},   {"compute_rdf", make<ComputeRdf>},     {"dump_thermo", make<DumpThermo>},
  {"dump_xyz", make<DumpXyz>},         {"dump_restart", make<DumpRestart>},
};
const size_t NUM_KEYWORDS = sizeof(KEYWORDS) / sizeof(KEYWORDS[0]);

} // namespace

Measure::Measure() : properties_(NUM_KEYWORDS) {}

bool Measure::parse(const MeasureContext& ctx, const std::vector<std::string>& tokens)
{
  for (size_t k = 0; k < NUM_KEYWORDS; ++k)
    if (tokens[0] == KEYWORDS[k].keyword) {
      properties_[k] = KEYWORDS[k].make(ctx, tokens);
      return true;
    }
  return false;
}

void Measure::preprocess(const MeasureContext& ctx, int number_of_steps)
{
  for (auto& p : properties_)
    if (p)
      p->preprocess(ctx, number_of_steps);
}

void Measure::process(const MeasureContext& ctx, int step)
{
  // nothing computed from a truncated neighbour list reaches a file: one check before the first
  // property that writes in this step
  for (auto& p : properties_)
    if (p && p->writes_at(step)) {
      ctx.force.potentials[0]->check();
      break;
    }
  for (auto& p : properties_)
    if (p)
      p->process(ctx, step);
}

void Measure::postprocess(const MeasureContext& ctx)
{
  for (auto& p : properties_)
    if (p)
      p->postprocess(ctx);
}

void Measure::finalize()
{
  for (auto& p : properties_)
    p.reset();
}

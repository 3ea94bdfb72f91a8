// measure.h -- the driver's measurement and dump keywords behind one Property interface, held by
// Measure (the shape of the reference's src/measure/property.cuh and measure.cuh).
#pragma once
#include "driver.h"
#include "ensemble.h"
#include "force.h"
#include <memory>
#include <string>
#include <vector>

// what the properties read from the driver; references into its state, so one context serves every run
struct MeasureContext {
  Model& model;
  Force& force;
  const std::unique_ptr<Ensemble>& ensemble; // the current run's (heat-bath energies of `compute`)
  const double& time_step;
  const double& global_time;
  const double& temperature; // the temperature of the last thermostatted ensemble line
  GPU_Vector<double>& thermo;
  const int& fixed_group;
  const int& fixed_method;
  GPU_Vector<double>& unwrapped; // unwrapped positions; empty until the first run with compute_msd
};

// one keyword: parsed by the constructor, then preprocess before a run, process after every step
// and postprocess after the run.  The destructor releases its libb200md handle.
class Property
{
public:
  virtual ~Property() = default;
  virtual void preprocess(const MeasureContext&, int /*number_of_steps*/) {}
  virtual void process(const MeasureContext& ctx, int step) = 0;
  virtual void postprocess(const MeasureContext&) {}
  // true when process() writes a file from this step's forces, which Measure checks first
  virtual bool writes_at(int /*step*/) const { return false; }
};

class Measure
{
public:
  Measure();
  // false for a keyword that is not a measurement; a repeated keyword replaces the earlier one
  bool parse(const MeasureContext& ctx, const std::vector<std::string>& tokens);
  void preprocess(const MeasureContext& ctx, int number_of_steps);
  void process(const MeasureContext& ctx, int step);
  void postprocess(const MeasureContext& ctx);
  void finalize(); // every measurement and dump keyword holds for one run only (run.cu:329-340)

private:
  std::vector<std::unique_ptr<Property>> properties_; // one slot per keyword, in sampling order
};

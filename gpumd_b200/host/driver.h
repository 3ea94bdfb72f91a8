// driver.h -- what the standalone driver's run.cpp and measure.cpp share: the reference's unit
// constants, its input-error convention and number checks, and the model read from model.xyz.
#pragma once
#include "model.h"
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

static const double K_B = 8.617343e-5;                     // common.cuh:21
static const double TIME_UNIT_CONVERSION = 1.018051e+1;    // common.cuh:26
static const double PRESSURE_UNIT_CONVERSION = 1.602177e+2; // common.cuh:25

struct Model {
  Box box;
  Atom atom;
  std::vector<Group> group; // one entry per grouping method of model.xyz (group:I:k)
  bool has_velocity = false;
};

[[noreturn]] inline void input_error(const std::string& msg)
{
  fprintf(stderr, "Input Error:\n    %s\n", msg.c_str());
  exit(1);
}

// is_valid_int / is_valid_real, src/utilities/read_file.cu: the whole token must be the number
inline bool valid_int(const std::string& s, int* v)
{
  char* end = nullptr;
  const long x = std::strtol(s.c_str(), &end, 10);
  if (s.empty() || *end != '\0' || x < -2147483647L || x > 2147483647L)
    return false;
  *v = (int)x;
  return true;
}

inline bool valid_real(const std::string& s, double* v)
{
  char* end = nullptr;
  const double x = std::strtod(s.c_str(), &end);
  if (s.empty() || *end != '\0')
    return false;
  *v = x;
  return true;
}

/* oracle/rdf_oracle.c -- TEST-ONLY brute-force restatement of the radial distribution function
 * (src/measure/rdf.cu:37-125, 163-251 of GPUMD).  Every ordered pair n1 != n2 is evaluated with the
 * reference's FP64 expressions; fma() stands where nvcc contracts them (read from the PTX of rdf.cu:
 * a*x + b*y + c*z = fma(c,z, fma(a,x, b*y)) and d2 = fma(z,z, fma(x,x, y*y))), and the bin loop over
 * every bin is the reference's, literally.  Build: gcc -O2 -std=c11 -ffp-contract=off -fPIC -shared
 * (tests/rdf_support.py does it); nothing of the product links it. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

static const double RDF_PI = 3.14159265358979323846; /* rdf.cu:55 */

typedef struct {
  double h[18];
  int pbc[3];
  int ortho;
} Box;

/* Box::get_inverse / set_is_orthogonal (box.cu:58-117) */
static void make_box(const double* h9, const int* pbc, Box* b)
{
  double* h = b->h;
  for (int d = 0; d < 9; ++d)
    h[d] = h9[d];
  h[9] = h[4] * h[8] - h[5] * h[7];
  h[10] = h[2] * h[7] - h[1] * h[8];
  h[11] = h[1] * h[5] - h[2] * h[4];
  h[12] = h[5] * h[6] - h[3] * h[8];
  h[13] = h[0] * h[8] - h[2] * h[6];
  h[14] = h[2] * h[3] - h[0] * h[5];
  h[15] = h[3] * h[7] - h[4] * h[6];
  h[16] = h[1] * h[6] - h[0] * h[7];
  h[17] = h[0] * h[4] - h[1] * h[3];
  const double det = h[0] * (h[4] * h[8] - h[5] * h[7]) + h[1] * (h[5] * h[6] - h[3] * h[8]) +
                     h[2] * (h[3] * h[7] - h[4] * h[6]);
  for (int d = 9; d < 18; ++d)
    h[d] /= det;
  for (int d = 0; d < 3; ++d)
    b->pbc[d] = pbc[d];
  b->ortho = h[1] == 0 && h[2] == 0 && h[3] == 0 && h[5] == 0 && h[6] == 0 && h[7] == 0;
}

/* Box::get_volume, box.cu:50-57 */
double rdf_oracle_volume(const double* h)
{
  const double v = h[0] * (h[4] * h[8] - h[5] * h[7]) + h[1] * (h[5] * h[6] - h[3] * h[8]) +
                   h[2] * (h[3] * h[7] - h[4] * h[6]);
  return fabs(v);
}

/* apply_mic (double), box.cuh:37-82 */
static void mic(const Box* b, double* x, double* y, double* z)
{
  const double* h = b->h;
  if (b->ortho) {
    if (b->pbc[0] == 1) {
      if (*x < -h[0] * 0.5)
        *x += h[0];
      else if (*x > +h[0] * 0.5)
        *x -= h[0];
    }
    if (b->pbc[1] == 1) {
      if (*y < -h[4] * 0.5)
        *y += h[4];
      else if (*y > +h[4] * 0.5)
        *y -= h[4];
    }
    if (b->pbc[2] == 1) {
      if (*z < -h[8] * 0.5)
        *z += h[8];
      else if (*z > +h[8] * 0.5)
        *z -= h[8];
    }
  } else {
    double sx = fma(h[11], *z, fma(h[9], *x, h[10] * *y));
    double sy = fma(h[14], *z, fma(h[12], *x, h[13] * *y));
    double sz = fma(h[17], *z, fma(h[15], *x, h[16] * *y));
    if (b->pbc[0] == 1)
      sx -= nearbyint(sx);
    if (b->pbc[1] == 1)
      sy -= nearbyint(sy);
    if (b->pbc[2] == 1)
      sz -= nearbyint(sz);
    *x = fma(h[2], sz, fma(h[0], sx, h[1] * sy));
    *y = fma(h[5], sz, fma(h[3], sx, h[4] * sy));
    *z = fma(h[8], sz, fma(h[6], sx, h[7] * sy));
  }
}

static double pair_d2(const Box* b, const double* pos, int n, int n1, int n2)
{
  double x12 = pos[n2] - pos[n1];
  double y12 = pos[n + n2] - pos[n + n1];
  double z12 = pos[2 * n + n2] - pos[2 * n + n1];
  mic(b, &x12, &y12, &z12);
  return fma(z12, z12, fma(x12, x12, y12 * y12));
}

/* counts[num_bins][1 + T (T + 1) / 2] of ORDERED pairs: column 0 every pair, column 1 + (a, b) for a <= b
 * the pairs with n1 of type_index[a] and n2 of type_index[b] (rdf.cu:90-118).  pos [3][n] SoA. */
void rdf_oracle_counts(int n, const double* h9, const int* pbc, const int* type, const double* pos, double rc,
                       int num_bins, int num_types, const int* type_index, long long* counts)
{
  Box b;
  make_box(h9, pbc, &b);
  const int R = 1 + num_types * (num_types + 1) / 2;
  const double dr = rc / num_bins, rc_square = rc * rc;
  memset(counts, 0, sizeof(long long) * (size_t)num_bins * R);
  for (int n1 = 0; n1 < n; ++n1) {
    for (int n2 = 0; n2 < n; ++n2) {
      if (n1 == n2)
        continue;
      const double d2 = pair_d2(&b, pos, n, n1, n2);
      if (d2 > rc_square)
        continue;
      for (int w = 0; w < num_bins; w++) {
        const double r_low = (w * dr) * (w * dr);
        const double r_up = ((w + 1) * dr) * ((w + 1) * dr);
        if (d2 > r_low && d2 <= r_up) {
          counts[(size_t)w * R + 0] += 1;
          int count = 1;
          for (int a = 0; a < num_types; ++a) {
            for (int c = a; c < num_types; ++c) {
              if (type[n1] == type_index[a] && type[n2] == type_index[c])
                counts[(size_t)w * R + count] += 1;
              ++count;
            }
          }
        }
      }
    }
  }
}

/* The unordered pairs n1 < n2 by the same rule, u[pair (a <= b)][num_bins] with the species of the two
 * atoms sorted; returns the number of pairs whose d2 differs bitwise between n1 -> n2 and n2 -> n1. */
long long rdf_oracle_unordered(int n, const double* h9, const int* pbc, const int* type, const double* pos,
                               double rc, int num_bins, int num_types, const int* type_index, long long* u)
{
  Box b;
  make_box(h9, pbc, &b);
  const int P = num_types * (num_types + 1) / 2;
  const double dr = rc / num_bins, rc_square = rc * rc;
  long long asymmetric = 0;
  memset(u, 0, sizeof(long long) * (size_t)num_bins * P);
  for (int n1 = 0; n1 < n; ++n1) {
    int s1 = -1;
    for (int a = 0; a < num_types; ++a)
      if (type[n1] == type_index[a])
        s1 = a;
    for (int n2 = n1 + 1; n2 < n; ++n2) {
      const double d2 = pair_d2(&b, pos, n, n1, n2);
      const double d2r = pair_d2(&b, pos, n, n2, n1);
      if (memcmp(&d2, &d2r, sizeof(double)) != 0)
        ++asymmetric;
      if (d2 > rc_square)
        continue;
      int s2 = -1;
      for (int a = 0; a < num_types; ++a)
        if (type[n2] == type_index[a])
          s2 = a;
      const int lo = s1 < s2 ? s1 : s2, hi = s1 < s2 ? s2 : s1;
      const int pair = lo * (2 * num_types - lo + 1) / 2 + (hi - lo);
      for (int w = 0; w < num_bins; w++) {
        const double r_low = (w * dr) * (w * dr);
        const double r_up = ((w + 1) * dr) * ((w + 1) * dr);
        if (d2 > r_low && d2 <= r_up)
          u[(size_t)pair * num_bins + w] += 1;
      }
    }
  }
  return asymmetric;
}

/* f[num_bins][R]: what one ordered pair adds in rdf.cu:102-112 at volume V: 1 / (N (N / V) dV) for the
 * total and 1 / (N_a (N_b / V) dV) for (a, b), dV = r_mid^2 * 4 * pi * dr */
void rdf_oracle_factors(double volume, int n, double rc, int num_bins, int num_types, const int* num_atoms,
                        double* f)
{
  const int R = 1 + num_types * (num_types + 1) / 2;
  const double dr = rc / num_bins;
  const double density_global = n / volume;
  for (int w = 0; w < num_bins; w++) {
    const double r_mid_sqaure = ((w + 0.5) * dr) * ((w + 0.5) * dr);
    const double dV = r_mid_sqaure * 4 * RDF_PI * dr;
    f[(size_t)w * R] = 1 / (n * density_global * dV);
    int count = 1;
    for (int a = 0; a < num_types; ++a)
      for (int b = a; b < num_types; ++b)
        f[(size_t)w * R + count++] = 1 / (num_atoms[a] * (num_atoms[b] / volume) * dV);
  }
}

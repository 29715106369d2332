// solve_file.h -- the --system mode shared by solve_split_sim.cu and solve_long_sim.cu: one Toeplitz system read from
// a file (int32 n, then a and b as n complex doubles each) through the simulation's solve; the output file gets an
// int32 verdict and the n complex double weights.  tests/test_wh_conditioning_cpu.py writes and reads these files.
#pragma once

#include <complex>
#include <cstdio>
#include <vector>

template <class Solve>
static int solve_file(const char *tag, Solve solve, const char *in, const char *out) {
  typedef std::complex<long double> cld;
  FILE *f = fopen(in, "rb");
  if (!f) return 2;
  int n = 0;
  std::vector<double> buf;
  bool read = fread(&n, sizeof n, 1, f) == 1 && n >= 1;
  if (read) {
    buf.resize((size_t)4 * n);
    read = fread(buf.data(), sizeof(double), buf.size(), f) == buf.size();
  }
  fclose(f);
  if (!read) return 2;
  std::vector<cld> a(n), b(n), w;
  for (int i = 0; i < n; i++) {
    a[i] = cld(buf[2 * i], buf[2 * i + 1]);
    b[i] = cld(buf[2 * n + 2 * i], buf[2 * n + 2 * i + 1]);
  }
  const int ok = solve(a, b, w);
  for (int i = 0; i < n; i++) { buf[2 * i] = (double)w[i].real(); buf[2 * i + 1] = (double)w[i].imag(); }
  FILE *g = fopen(out, "wb");
  if (!g) return 2;
  const bool written = fwrite(&ok, sizeof ok, 1, g) == 1 &&
                       fwrite(buf.data(), sizeof(double), 2 * (size_t)n, g) == 2 * (size_t)n;
  if (fclose(g) != 0 || !written) return 2;
  printf("%s SYSTEM %d taps ok=%d\n", tag, n, ok);
  return 0;
}

"""The pass kernel replaces `r / w` (plan.go:679) and `x / P` (plan.go:642,650) by the
divisor's correctly rounded reciprocal plus one FMA-residual correction
(assign_pass.cuh: div_exact).  This test runs the same sequence on the CPU (C, real
fma(), no contraction) against true IEEE division on adversarial operands: exact
multiples +- a few ulps, half-way quotients, planner-shaped values, integer divisors from
3 to 2^31 - 1 (node weights are int32), dividends of both signs (counts go negative under
negative partition weights).  Zero mismatches allowed.  CPU only."""
import os
import subprocess
import tempfile

SRC = r'''
#include <math.h>
#include <stdio.h>
#include <stdint.h>
#include <string.h>
static uint64_t s = 0x9E3779B97F4A7C15ull;
static uint64_t rnd(void) { s += 0x9E3779B97F4A7C15ull; uint64_t z = s; z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
static double div_exact(double a, double b, double y) { double q = a * y; double e = fma(-b, q, a); return fma(e, y, q); }
int main(void) {
  long bad = 0, n = 0;
  for (long it = 0; it < 40000000L; ++it) {
    uint64_t a = rnd(), b = rnd(), c = rnd();
    double w = (it & 1) ? (double)(3 + (b % 5000))
             : (c & 1) ? (double)(2000000000ull + (b % 147483648ull)) : (double)(3 + (b % 2000000000ull));
    if ((c & 0xff0) == 0) w = 2147483647.0;
    double r;
    int mode = a & 3;
    if (mode == 0) { uint64_t m = (a >> 8) & ((1ull << 52) - 1); int e = (int)((a >> 60) % 70) - 40; r = ldexp(1.0 + (double)m / 4503599627370496.0, e); }
    else if (mode == 1) { uint64_t m = (a >> 8) & ((1ull << 52) - 1); double q = ldexp(1.0 + (double)m / 4503599627370496.0, (int)((b >> 40) % 30) - 10);
      r = w * q; int64_t d = (int64_t)((b >> 20) % 7) - 3; uint64_t bits; memcpy(&bits, &r, 8); bits += d; memcpy(&r, &bits, 8); }
    else if (mode == 2) { r = (double)((a >> 10) % 5000000) + (double)((b >> 8) % 4000) * 1e-6 + (double)((a >> 33) % 100000) * 1e-9; }
    else { uint64_t m = (a >> 8) & ((1ull << 52) - 1); double q = 1.0 + (double)m / 4503599627370496.0; double h = q + ldexp(1.0, -53);
      r = (double)((long double)h * (long double)w); }
    if (!(r > 0)) continue;
    if (c & 2) r = -r;
    double y = 1.0 / w;
    n++;
    if (div_exact(r, w, y) != r / w) bad++;
    if (div_exact(r, 1.0, 1.0) != r) bad++;
  }
  printf("%ld %ld\n", n, bad);
  return 0;
}
'''


def test_markstein_division_equals_true_division():
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "t.c")
        open(c, "w").write(SRC)
        exe = os.path.join(d, "t")
        subprocess.run(["gcc", "-O2", "-mfma", "-ffp-contract=off", c, "-o", exe, "-lm"], check=True)
        n, bad = map(int, subprocess.run([exe], stdout=subprocess.PIPE, text=True, check=True).stdout.split())
    assert n > 30000000 and bad == 0

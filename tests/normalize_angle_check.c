/* util::normalize_angle (lesson4 UtilFunctions.h:36-48) is fmod(fmod(a, 2pi) + 2pi, 2pi) in double.  hector_grid.cuh takes
 * a shortcut for |a| < 2pi (no remainder loop); this program checks the shortcut against the C library's fmod, bit for
 * bit, on pseudo-random floats of every magnitude below 50 and on the edge cases.  argv[1] = number of samples. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static double shortcut(double d, double two_pi) {
  if (fabs(d) < two_pi) {
    const double x = d + two_pi;
    return x >= two_pi ? x - two_pi : x;
  }
  return fmod(fmod(d, two_pi) + two_pi, two_pi);
}

int main(int argc, char **argv) {
  const double two_pi = 2.0f * 3.14159265358979323846;
  const unsigned long long want = argc > 1 ? strtoull(argv[1], 0, 10) : 10000000ull;
  unsigned long long bad = 0, n = 0;
  uint32_t s = 12345;
  for (unsigned long long k = 0; n < want; k++) {
    s = s * 1664525u + 1013904223u;
    uint32_t bits = s;
    if (k % 4 == 0) bits = (s & 0x807fffffu) | ((uint32_t)(100 + (s >> 9) % 31) << 23);  /* exponents 2^-27 .. 2^3 */
    float e2;
    memcpy(&e2, &bits, 4);
    if (!(fabsf(e2) < 50.0f)) continue;
    n++;
    const double ref = fmod(fmod((double)e2, two_pi) + two_pi, two_pi), got = shortcut((double)e2, two_pi);
    if (memcmp(&ref, &got, 8)) bad++;
  }
  const float sp[] = {0.0f, -0.0f, 6.2831853f, -6.2831853f, 6.283185f, 6.2831855f, -6.2831855f, 1e-30f, -1e-30f, 3.1415927f, -3.1415927f, 12.566371f, -12.566371f};
  for (unsigned i = 0; i < sizeof(sp) / sizeof(sp[0]); i++) {
    const double ref = fmod(fmod((double)sp[i], two_pi) + two_pi, two_pi), got = shortcut((double)sp[i], two_pi);
    if (memcmp(&ref, &got, 8)) bad++;
    n++;
  }
  printf("{\"inputs\": %llu, \"mismatches\": %llu}\n", n, bad);
  return 0;
}

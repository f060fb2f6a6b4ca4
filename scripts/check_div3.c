/* Checks div3_rn (viettts_b200/csrc/tc_conv.cu) against the IEEE division s / 3.0f for all 2^32 float inputs.
 *
 *     cc -O2 -mfma -ffp-contract=off -fopenmp scripts/check_div3.c -o /tmp/check_div3 -lm && /tmp/check_div3
 *
 * Needs a CPU with fused multiply-add (fmaf is then one correctly rounded operation, as __fmaf_rn is on the GPU) and
 * no flush-to-zero.  NaN inputs are skipped.  Prints the inputs where the two differ and exits 1 if there are any. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

static float div3_rn(float s) {
  const float y = 0x1.555556p-2f;
  const float q0 = s * y;
  const float q1 = fmaf(fmaf(-q0, 3.0f, s), y, q0);
  return (s == 0.f || fabsf(s) == INFINITY) ? s : q1;
}

int main(void) {
  long long bad = 0;
#pragma omp parallel for reduction(+ : bad) schedule(static)
  for (long long i = 0; i < (1LL << 32); ++i) {
    const uint32_t u = (uint32_t)i;
    float s;
    memcpy(&s, &u, 4);
    if (isnan(s)) continue;
    volatile float three = 3.0f;
    const float ref = s / three, alt = div3_rn(s);
    uint32_t a, b;
    memcpy(&a, &ref, 4);
    memcpy(&b, &alt, 4);
    if (a != b) {
      ++bad;
      printf("%08x: s / 3 = %a, div3_rn = %a\n", u, ref, alt);
    }
  }
  printf("%lld of 2^32 inputs differ\n", bad);
  return bad != 0;
}

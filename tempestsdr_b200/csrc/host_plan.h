/* host_plan.h -- data-independent host-side planning (plain C, compiled by gcc with -ffp-contract=off).
 * The functions are part of the public C-ABI and are declared in include/tsdrgpu.h:
 *   tsdrgpu_plan_resample, tsdrgpu_geometry, tsdrgpu_gauss_taps. */
#ifndef TSDRGPU_HOST_PLAN_H_
#define TSDRGPU_HOST_PLAN_H_
#include "../../include/tsdrgpu.h"
#ifdef __cplusplus
extern "C" {
#endif
/* internal: 1 when a mode and its parameters are in tsdrgpu.h's ranges (contrast, denoise, stack and deblur ignore them when off), else 0 */
int autogain_ok(int mode, int ppm);
int contrast_ok(int mode, int clip_centi, int tx, int ty);
int denoise_ok(int mode, int h_milli, int r, int p);
int stack_ok(int mode, int depth, int rx, int ry);
int deblur_ok(int mode, int sigma_centi, int iterations);
int superband_ok(const tsdrgpu_superband_t *s);
#ifdef __cplusplus
}
#endif
#endif

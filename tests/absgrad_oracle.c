/*
 * absgrad_oracle.c — CPU oracle of the absolute-gradient densification statistic (DGR_RASTER_ABS_GRAD).  TEST INFRASTRUCTURE ONLY.
 *
 * Built on the rasterizer's C oracle: oracle/dgr_oracle.c is included unchanged (its forward state is the input), and
 * absgrad_oracle_impl.h adds dgr_oracle_absgrad_f32 / _f64.  tests/absgrad_oracle.py compiles this file into a temporary directory.
 */
#include "../oracle/dgr_oracle.c"

#define REAL float
#define SUF f32
#define CAT_(a, b) a##_##b              /* (the oracle's header undefines its own at its end) */
#define CAT(a, b) CAT_(a, b)
#define FN(name) CAT(name, SUF)
#include "absgrad_oracle_impl.h"
#undef REAL
#undef SUF

#define REAL double
#define SUF f64
#include "absgrad_oracle_impl.h"
#undef REAL
#undef SUF

/*
 * contrib_oracle.c — CPU oracle of the blending-weight statistics (DGR_RASTER_CONTRIB).  TEST INFRASTRUCTURE ONLY.
 *
 * Built on the rasterizer's C oracle: oracle/dgr_oracle.c is included unchanged (its forward state is the input), and
 * contrib_oracle_impl.h adds dgr_oracle_contrib_f32 / _f64.  tests/contrib_oracle.py compiles this file into a temporary directory.
 */
#include "../oracle/dgr_oracle.c"

#define REAL float
#define SUF f32
#define CAT_(a, b) a##_##b              /* (the oracle's header undefines its own at its end) */
#define CAT(a, b) CAT_(a, b)
#define FN(name) CAT(name, SUF)
#include "contrib_oracle_impl.h"
#undef REAL
#undef SUF

#define REAL double
#define SUF f64
#include "contrib_oracle_impl.h"
#undef REAL
#undef SUF

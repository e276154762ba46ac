// bwd_fast_lsmr.cu -- the LSMR variants of the kernels of bwd_fast.cu (diffcp's mode = "lsmr"), compiled as a translation unit of their
// own: next to them the LSQR kernels would compile to other code (the non-inlined helpers both call would have two callers).
#define BC_LSMR 1
#include "bwd_fast.cu"

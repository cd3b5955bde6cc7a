// sim_step_defer.cu — the deferred instantiations of the fused step kernel (go1_step_kernel<SELF, true>, user reward terms,
// DESIGN.md §4), in a translation unit of their own: the step kernels compiled in sim_step.cu and sim_step_self.cu keep their code.
#define GO1_STEP_DEFERRED_TU
#include "sim_step.cu"

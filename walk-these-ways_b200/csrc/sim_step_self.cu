// sim_step_self.cu — the self-collision instantiation of the fused step kernel (go1_step_kernel<true>, DESIGN.md §3), in a
// translation unit of its own: compiled next to the default instantiation, it changed the code generated for that one.
#define GO1_STEP_SELF_COLLISION_TU
#include "sim_step.cu"

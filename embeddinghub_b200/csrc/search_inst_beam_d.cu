// K2b instantiations (see beam_impl.cuh): dpad 3072, 4096, fp32 rows and the bf16 shadow
#include "beam_impl.cuh"
namespace ehb {
template struct BeamShape<3072, float>;
template struct BeamShape<3072, __nv_bfloat16>;
template struct BeamShape<4096, float>;
template struct BeamShape<4096, __nv_bfloat16>;
}  // namespace ehb

// K2b instantiations (see beam_impl.cuh): dpad 384 .. 768, fp32 rows and the bf16 shadow
#include "beam_impl.cuh"
namespace ehb {
template struct BeamShape<384, float>;
template struct BeamShape<384, __nv_bfloat16>;
template struct BeamShape<512, float>;
template struct BeamShape<512, __nv_bfloat16>;
template struct BeamShape<768, float>;
template struct BeamShape<768, __nv_bfloat16>;
}  // namespace ehb

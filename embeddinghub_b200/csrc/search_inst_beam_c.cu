// K2b instantiations (see beam_impl.cuh): dpad 1024 .. 2048, fp32 rows and the bf16 shadow
#include "beam_impl.cuh"
namespace ehb {
template struct BeamShape<1024, float>;
template struct BeamShape<1024, __nv_bfloat16>;
template struct BeamShape<1536, float>;
template struct BeamShape<1536, __nv_bfloat16>;
template struct BeamShape<2048, float>;
template struct BeamShape<2048, __nv_bfloat16>;
}  // namespace ehb

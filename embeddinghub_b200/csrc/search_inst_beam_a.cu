// K2b instantiations (see beam_impl.cuh): dpad 32 .. 256, fp32 rows and the bf16 shadow
#include "beam_impl.cuh"
namespace ehb {
template struct BeamShape<32, float>;
template struct BeamShape<32, __nv_bfloat16>;
template struct BeamShape<64, float>;
template struct BeamShape<64, __nv_bfloat16>;
template struct BeamShape<128, float>;
template struct BeamShape<128, __nv_bfloat16>;
template struct BeamShape<256, float>;
template struct BeamShape<256, __nv_bfloat16>;
}  // namespace ehb

// K5 wide-form instantiations (ef_construction 257 .. 4096; see build_beam_impl.cuh): dpad 384 .. 768
#include "build_beam_impl.cuh"
namespace ehb {
template struct BuildBeamShape<384>;
template struct BuildBeamShape<512>;
template struct BuildBeamShape<768>;
}  // namespace ehb

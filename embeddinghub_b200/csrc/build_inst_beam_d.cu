// K5 wide-form instantiations (ef_construction 257 .. 4096; see build_beam_impl.cuh): dpad 3072, 4096
#include "build_beam_impl.cuh"
namespace ehb {
template struct BuildBeamShape<3072>;
template struct BuildBeamShape<4096>;
}  // namespace ehb

// K5 wide-form instantiations (ef_construction 257 .. 4096; see build_beam_impl.cuh): dpad 1024 .. 2048
#include "build_beam_impl.cuh"
namespace ehb {
template struct BuildBeamShape<1024>;
template struct BuildBeamShape<1536>;
template struct BuildBeamShape<2048>;
}  // namespace ehb

// K5 wide-form instantiations (ef_construction 257 .. 4096; see build_beam_impl.cuh): dpad 32 .. 256
#include "build_beam_impl.cuh"
namespace ehb {
template struct BuildBeamShape<32>;
template struct BuildBeamShape<64>;
template struct BuildBeamShape<128>;
template struct BuildBeamShape<256>;
}  // namespace ehb

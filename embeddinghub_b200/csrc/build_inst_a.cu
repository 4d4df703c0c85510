// K5 instantiations for dpad 32 .. 128 (see build_impl.cuh)
#include "build_impl.cuh"
namespace ehb {
template struct BuildShape<32>;
template struct BuildShape<64>;
template struct BuildShape<128>;
}  // namespace ehb

// K5 instantiations for dpad 512 .. 768 (see build_impl.cuh)
#include "build_impl.cuh"
namespace ehb {
template struct BuildShape<512>;
template struct BuildShape<768>;
}  // namespace ehb

// K5 instantiations for dpad 1024 .. 2048 (see build_impl.cuh)
#include "build_impl.cuh"
namespace ehb {
template struct BuildShape<1024>;
template struct BuildShape<1536>;
template struct BuildShape<2048>;
}  // namespace ehb

// K5 instantiations for dpad 256 .. 384 (see build_impl.cuh)
#include "build_impl.cuh"
namespace ehb {
template struct BuildShape<256>;
template struct BuildShape<384>;
}  // namespace ehb

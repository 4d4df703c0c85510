// K5 instantiations for the wide rows, dpad 3072 .. 4096 (see build_impl.cuh)
#include "build_impl.cuh"
namespace ehb {
template struct BuildShape<3072>;
template struct BuildShape<4096>;
}  // namespace ehb

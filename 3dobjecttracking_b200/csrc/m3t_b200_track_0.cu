// k_track instantiations, group 0 of 4 (see m3t_b200_track_variants.h)
#define M3TB_TRACK_TU 1
#include "m3t_b200_kernels.cuh"
#include "m3t_b200_track_variants.h"

namespace m3tb {
#define M3TB_INSTANTIATE(T_, K_, L_, O_) template __global__ void k_track<T_, K_, L_, O_>(const __grid_constant__ TrackArgs);
M3TB_TRACK_GROUP_0(M3TB_INSTANTIATE)
#undef M3TB_INSTANTIATE
}  // namespace m3tb

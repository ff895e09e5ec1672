// tw_voxel_math.cuh - std::min / std::max with the reference's argument order, for the voxel headers (tw_voxel_fill.cuh, tw_voxel_mc.cuh) and the
// translation units that include them. Internal linkage, as everything in those headers.
#pragma once

namespace {
__device__ __forceinline__ float smin(float a, float b) {return (b < a) ? b : a;} // std::min
__device__ __forceinline__ float smax(float a, float b) {return (a < b) ? b : a;} // std::max
} // namespace

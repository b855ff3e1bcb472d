// sorted_ranges.cuh -- the run of every key in a sorted key array: the block -> Gaussian lists of mesh.cu's opacity
// field and the vertex -> face lists of mesh_common.cuh.
#pragma once
#include <cstdint>

namespace dgs {
namespace {

// ranges[k] = [first, last + 1) of the run of key k in the sorted keys (untouched for a key that does not occur)
__global__ void ranges_kernel(int n, const uint32_t* __restrict__ keys, uint2* __restrict__ ranges) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = keys[i];
  if (i == 0 || keys[i - 1] != k) ranges[k].x = i;
  if (i == n - 1 || keys[i + 1] != k) ranges[k].y = i + 1;
}

}  // namespace
}  // namespace dgs

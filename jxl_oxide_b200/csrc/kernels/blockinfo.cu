// Varblock placement as a launch of its own, for the HfMetadata streams that carry Modular transforms: their
// (dct_select, hf_mul) lists are only final after the inverse transforms, so the stream's warp cannot place them. Every
// other HfMetadata stream places its varblocks inside the stream kernel (modular_stream.cu); both run placement.cuh.
#include "placement.cuh"

namespace jxlb {

namespace {

__global__ void __launch_bounds__(32) place_varblocks_kernel(const DevPlacement* __restrict__ jobs, int* __restrict__ status) {
  __shared__ PlaceShared s;
  const int err = place_varblocks(PlaceWarp{threadIdx.x}, s, jobs[blockIdx.x]);
  if (threadIdx.x == 0) status[blockIdx.x] = err;
}

}  // namespace

void launch_place_varblocks(const DevPlacement* jobs, int num_jobs, int* status, cudaStream_t stream) {
  if (num_jobs <= 0) return;
  place_varblocks_kernel<<<num_jobs, 32, 0, stream>>>(jobs, status);
}

}  // namespace jxlb

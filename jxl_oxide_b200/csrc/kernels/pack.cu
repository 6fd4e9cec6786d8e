// Frame packer: the stored f32 planes of a decoded frame -> the sample buffers the reference's Render hands out
// (ImageStream::write_to_buffer, Render::image_all_channels, Render::image_planar; crates/jxl-oxide/src/{lib.rs,fb.rs}).
// The per-sample rules are in pack.cuh; this file only decides which thread handles which sample and where the channel
// and spot tables are read from.
//
// A CTA of 32 x 8 threads packs a 32 x 32 tile of output samples. For orientations 1..4 an output row is a stored row
// (possibly mirrored), so a warp reads one stored row segment per channel, and each thread writes all channels of its
// sample. For 5..8 an output row is a stored column: a warp would read 32 different rows. The tile then goes through
// shared memory one channel at a time: the warps read stored rows into it and write output rows out of it, both coalesced.
//
// Tables of up to kPackParamEntries entries travel in the kernel's parameter block, so that every plane pointer and stride
// is a constant-bank load; longer tables are read from device memory.
#include "kernels.h"
#include "pack.cuh"

namespace jxlb {

namespace {

constexpr uint32_t kTile = 32, kRows = 8;

struct PackParams {
  DevPackSpec spec;
  const DevPackChannel* d_channels;  // device tables, read when the tables do not fit below
  const DevPackSpot* d_spots;
  DevPackChannel channels[kPackParamEntries];
  DevPackSpot spots[kPackParamEntries];
};

template <bool kTablesInParams>
__global__ void __launch_bounds__(kTile* kRows) pack_kernel(const __grid_constant__ PackParams params, void* out) {
  __shared__ float tile[kTile][kTile + 1];
  const DevPackSpec& p = params.spec;
  const DevPackChannel* __restrict__ channels = kTablesInParams ? params.channels : params.d_channels;
  const DevPackSpot* __restrict__ spots = kTablesInParams ? params.spots : params.d_spots;
  const uint32_t ow = p.orientation >= 5 ? p.height : p.width, oh = p.orientation >= 5 ? p.width : p.height;
  const uint32_t ox0 = blockIdx.x * kTile, oy0 = blockIdx.y * kTile;
  const uint32_t tx = threadIdx.x, ty = threadIdx.y;
  if (p.orientation < 5) {  // a thread writes all channels of its samples: one run of num_channels in interleaved output
    for (uint32_t j = ty; j < kTile; j += kRows) {
      const uint32_t x = ox0 + tx, y = oy0 + j;
      if (x >= ow || y >= oh) continue;
      uint32_t sx, sy;
      pack_source_xy(p.orientation, ow, oh, x, y, &sx, &sy);
      for (uint32_t c = 0; c < p.num_channels; ++c)
        pack_store(out, pack_index(p, ow, oh, c, x, y), p.sample_type, pack_sample(p, channels, spots, c, sx, sy));
    }
    return;
  }
  for (uint32_t c = 0; c < p.num_channels; ++c) {
    // transposed: tile[a][b] holds output sample (ox0 + a, oy0 + b); lanes run along b, i.e. along a stored row
    for (uint32_t a = ty; a < kTile; a += kRows) {
      const uint32_t x = ox0 + a, y = oy0 + tx;
      if (x >= ow || y >= oh) continue;
      uint32_t sx, sy;
      pack_source_xy(p.orientation, ow, oh, x, y, &sx, &sy);
      tile[a][tx] = pack_sample(p, channels, spots, c, sx, sy);
    }
    __syncthreads();
    for (uint32_t b = ty; b < kTile; b += kRows) {
      const uint32_t x = ox0 + tx, y = oy0 + b;
      if (x < ow && y < oh) pack_store(out, pack_index(p, ow, oh, c, x, y), p.sample_type, tile[tx][b]);
    }
    __syncthreads();
  }
}

}  // namespace

void launch_pack(const DevPackSpec& p, const DevPackChannel* channels, const DevPackSpot* spots, const DevPackChannel* d_channels,
                 const DevPackSpot* d_spots, void* out, cudaStream_t stream) {
  if (!p.width || !p.height || !p.num_channels) return;
  const uint32_t ow = p.orientation >= 5 ? p.height : p.width, oh = p.orientation >= 5 ? p.width : p.height;
  const dim3 grid((ow + kTile - 1) / kTile, (oh + kTile - 1) / kTile);
  PackParams params = {};
  params.spec = p;
  params.d_channels = d_channels;
  params.d_spots = d_spots;
  if (p.num_channels <= kPackParamEntries && p.num_spots <= kPackParamEntries) {
    for (uint32_t c = 0; c < p.num_channels; ++c) params.channels[c] = channels[c];
    for (uint32_t s = 0; s < p.num_spots; ++s) params.spots[s] = spots[s];
    pack_kernel<true><<<grid, dim3(kTile, kRows), 0, stream>>>(params, out);
  } else {
    pack_kernel<false><<<grid, dim3(kTile, kRows), 0, stream>>>(params, out);
  }
}

}  // namespace jxlb

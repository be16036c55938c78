// The block-per-centre frame of the wide voxel kernels (voxel_wide.cu, firstorder.cu): a window of up to 3375 positions
// staged in shared memory and its levels compacted by the whole block.
#pragma once
#include "vox_features.cuh"

namespace rb {

// Block-wide compact_levels: lidx[p] and val[k] exactly as compact_levels gives them for the window w[0..wn), the number
// of levels to s_n (returned).  fq: shared scratch of wn ints (each position's first occurrence of its level).  Every
// thread of the block calls it; it starts after and ends with a barrier.
__device__ __forceinline__ int block_compact_levels(const uint16_t* w, int wn, int* val, uint16_t* lidx, int* fq,
                                                    int& s_n) {
  for (int p = threadIdx.x; p < wn; p += blockDim.x) {
    const uint16_t g = w[p];
    int q = -1;
    if (g) for (q = 0; w[q] != g; q++) {}
    fq[p] = q;
  }
  __syncthreads();
  // the first occurrences, in position order, are the classes of compact_levels in its order
  if (threadIdx.x == 0) {
    int k = 0;
    for (int p = 0; p < wn; p++)
      if (fq[p] == p) { val[k] = w[p]; lidx[p] = (uint16_t)k++; }
    s_n = k;
  }
  __syncthreads();
  for (int p = threadIdx.x; p < wn; p += blockDim.x)
    if (fq[p] != p) lidx[p] = fq[p] < 0 ? NOLEV : lidx[fq[p]];
  __syncthreads();
  return s_n;
}

// position p of a (2rz+1) x (2ry+1) x (2rx+1) window as its offsets from the centre, in load_window's scan order
struct WindowOffset {
  int dz, dy, dx;
  __device__ __forceinline__ WindowOffset(int p, int rz, int ry, int rx) {
    const int wy = 2 * ry + 1, wx = 2 * rx + 1;
    dz = p / (wy * wx) - rz;
    dy = (p / wx) % wy - ry;
    dx = p % wx - rx;
  }
};

}  // namespace rb

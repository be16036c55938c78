// The frame the radius-1 voxel kernels share: a chunk voxel's coordinates, its 3x3x3 window, the copy of a table block
// into shared memory, and the full/deferred tile loop of the kernels with a full-window body.
// tests/host_emul/solve_kernel_emul.cpp compiles this header for the CPU (through glcm_kernels.cuh) with __device__,
// __shared__ and __syncthreads defined as macros.
#pragma once
#include <type_traits>

#include "vox_features.cuh"

namespace rb {

// voxel t of the chunk of planes starting at z0 (a contiguous level volume: plane = sz = Y * X, sy = X)
struct ChunkVoxel {
  int z, y, x, rem;    // rem = y * X + x
  long long vi;        // index in the level volume
  long long oi;        // index in the output maps, whose plane 0 is out_z0
};

// !live: a stand-in for a thread without a voxel, decoded as t = 0.  Par: VoxParams, or any parameter block with the
// volume's Z, Y, X and element strides sz, sy (first order's FoParams)
template <typename Par>
RB_HD ChunkVoxel chunk_voxel(const Par& P, long long plane, int z0, int out_z0, long long t, bool live = true) {
  ChunkVoxel v;
  v.z = z0 + (int)((live ? t : 0) / plane);
  v.rem = (int)((live ? t : 0) % plane);
  v.y = v.rem / P.X;
  v.x = v.rem % P.X;
  v.vi = (long long)v.z * P.sz + (long long)v.y * P.sy + v.x;
  v.oi = (long long)(v.z - out_z0) * plane + v.rem;
  return v;
}

// The one place the map type of the texture voxel kernels is decided: every map element is stored through here.  OutT
// is double (the reference's map type) or float.  Every value is computed in double and rounded once, here: the float
// conversion is round-to-nearest-even, as __double2float_rn, and keeps NaN.
template <typename OutT>
RB_HD void store_map(OutT* p, double v) { *p = (OutT)v; }

// whether the voxel is a centre: centers[] if given, else a non-zero level (a read, so callers gate it with
// `live && ...` where the thread may have no voxel)
template <typename L>
RB_HD bool chunk_center(const L* lev, const uint8_t* centers, long long plane, const ChunkVoxel& v) {
  return centers ? centers[(long long)v.z * plane + v.rem] != 0 : lev[v.vi] != 0;
}

// the 27 window levels of voxel (z, y, x) with volume index vi to w[p * ws], p in z, y, x order: zeros outside the
// volume, all zeros unless `gate`.  Returns whether the window is full (gate and no zero level).  Par as chunk_voxel.
template <typename W, typename L, typename Par>
RB_HD bool load_window27(const L* lev, const Par& P, int z, int y, int x, long long vi, bool gate, W* w,
                         int ws) {
  bool full = gate;
  int p = 0;
#pragma unroll
  for (int dz = -1; dz <= 1; dz++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dx = -1; dx <= 1; dx++, p++) {
        const int zz = z + dz, yy = y + dy, xx = x + dx;
        const bool in = gate && zz >= 0 && zz < P.Z && yy >= 0 && yy < P.Y && xx >= 0 && xx < P.X;
        const W l = in ? (W)lev[vi + (long long)dz * P.sz + (long long)dy * P.sy + dx] : (W)0;
        full &= l != 0;
        w[p * ws] = l;
      }
  return full;
}

// a block's copy of a table block (a whole number of 32-bit words) into shared memory, NT threads striding (0:
// blockDim.x); the caller's next barrier publishes it
template <int NT = 0, typename T>
__device__ __forceinline__ void copy_tables_to_shared(T& dst, const T* __restrict__ src) {
  const uint32_t* s = reinterpret_cast<const uint32_t*>(src);
  uint32_t* d = reinterpret_cast<uint32_t*>(&dst);
  if constexpr (NT > 0) {
    for (int i = threadIdx.x; i < (int)(sizeof(T) / 4); i += NT) d[i] = s[i];
  } else {
    for (int i = threadIdx.x; i < (int)(sizeof(T) / 4); i += blockDim.x) d[i] = s[i];
  }
}

// Block-uniform tiles of NT consecutive chunk voxels, t in [0, total).  full(t, live, defer_it) handles the tile's voxel
// of this thread (live: t < total): a centre with a full window runs the full-window body (no validity logic, no
// barriers), a voxel that is not a centre stores init_value, and any other centre (the volume's faces, the ROI's border
// and holes) calls defer_it(), which appends t to the block's list `defer` (2 * NT entries, ndefer of them in use: 0
// and published by a barrier on entry).  The block runs general(entry, live) over that list, NT at a time, whenever NT
// are waiting and once at the end.  Every thread of the block calls it, so a general body may hold block barriers;
// entry() is the thread's list entry, to be read only if live.  Each body has one call site, so a warp never holds both
// for one tile.  A voxel's result depends only on its window, not on the tile or the order it is run in: slab and
// whole-volume maps are bit-identical.
template <int NT, typename Idx, typename Full, typename General>
__device__ __forceinline__ void full_window_tiles(long long total, Idx* defer, unsigned& ndefer, Full full,
                                                  General general) {
  const int tid = threadIdx.x;
  const long long ntiles = (total + NT - 1) / NT;
  // one pass per tile and a last pass with no tile
  for (long long tile = blockIdx.x;; tile += gridDim.x) {
    const bool more = tile < ntiles;                                 // block-uniform
    if (more) {
      const long long t = tile * NT + tid;
      full(t, t < total, [&] { defer[atomicAdd(&ndefer, 1u)] = (Idx)t; });
    }
    __syncthreads();
    const unsigned nd = ndefer;
    __syncthreads();
    // the general body over the last `count` list entries
    const unsigned count = more ? (nd >= NT ? NT : 0) : nd;
    if (count) {
      if (tid == 0) ndefer = nd - count;
      general([&]() -> Idx& { return defer[nd - count + tid]; }, (unsigned)tid < count);
      __syncthreads();                                               // every entry read before the list grows again
    }
    if (!more) break;
  }
}

}  // namespace rb

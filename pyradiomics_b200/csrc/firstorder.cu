// Voxel-based first-order feature maps.  Two kernels:
//   firstorder_kernel<WCAP>  any window (r <= 3, clipped radii, 16-bit levels): one thread per centre voxel, grid-stride,
//                            gathers its window of raw intensities + discretised levels and evaluates
//                            firstorder_voxel<> (firstorder.cuh)
//   firstorder_tiles_kernel  kernelRadius 1 on every axis with 8-bit levels: the full/deferred tiles of full_window_tiles
//                            (voxel_tiles.cuh).  A centre whose 27 window voxels are all in the volume, in the kernel
//                            mask, non-zero in level and not NaN runs firstorder_full_body; every other centre is drained
//                            through the generic gather + firstorder_voxel<27>.  Both give the same bits.
#include "common.cuh"
#include "firstorder.cuh"
#include "pixel.cuh"
#include "voxel_tiles.cuh"

namespace rb {

struct FoParams {
  int Z, Y, X;
  long long sz, sy;    // element strides of the (contiguous) image, mask and level volumes
  int rz, ry, rx, z0, z1, out_z0, dtype, level_bytes;
  double shift, voxel_volume, init_value;
};

// the generic window of centre (z, y, x): the intensities of the in-volume, in-mask voxels and every position's level
// (0 = not in the kernel), then firstorder_voxel<WCAP>
template <int WCAP>
__device__ __forceinline__ void firstorder_generic(const void* __restrict__ img, const uint8_t* __restrict__ mask,
                                                   const void* __restrict__ lev, const FoParams& P, int z, int y, int x,
                                                   double* f) {
  double xs[WCAP];
  uint16_t w[WCAP];
  int n = 0, wn = 0;
  for (int dz = -P.rz; dz <= P.rz; dz++)
    for (int dy = -P.ry; dy <= P.ry; dy++)
      for (int dx = -P.rx; dx <= P.rx; dx++, wn++) {
        const int zz = z + dz, yy = y + dy, xx = x + dx;
        w[wn] = 0;
        if (zz < 0 || zz >= P.Z || yy < 0 || yy >= P.Y || xx < 0 || xx >= P.X) continue;
        const long long j = (long long)zz * P.sz + (long long)yy * P.sy + xx;
        if (mask && !mask[j]) continue;
        xs[n++] = load_f64(img, P.dtype, j);
        w[wn] = P.level_bytes == 1 ? (uint16_t)((const uint8_t*)lev)[j] : ((const uint16_t*)lev)[j];
      }
  firstorder_voxel<WCAP>(xs, n, w, wn, P.shift, P.voxel_volume, f);
}

// whether chunk voxel v gets maps: centers[] if given, else the kernel mask (everything when NULL)
__device__ __forceinline__ bool firstorder_center(const uint8_t* __restrict__ mask, const uint8_t* __restrict__ centers,
                                                  const ChunkVoxel& v) {
  return centers ? centers[v.vi] != 0 : (mask ? mask[v.vi] != 0 : true);
}

template <int WCAP>
__global__ void __launch_bounds__(128)
firstorder_kernel(const void* __restrict__ img, const uint8_t* __restrict__ mask, const uint8_t* __restrict__ centers,
                  const void* __restrict__ lev, FoParams P, double* __restrict__ out, long long fstride) {
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(P.z1 - P.z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, t);
    if (!firstorder_center(mask, centers, v)) {
#pragma unroll
      for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = P.init_value;
      continue;
    }
    double f[FIRSTORDER_NF];
    firstorder_generic<WCAP>(img, mask, lev, P, v.z, v.y, v.x, f);
#pragma unroll
    for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = f[k];
  }
}

// the 27 intensities of a window whose positions are all inside the volume, to xv in window order; whether all are in
// the kernel mask (or it is NULL) and none is NaN
template <typename T>
__device__ __forceinline__ bool firstorder_load27(const T* __restrict__ img, const uint8_t* __restrict__ mask,
                                                  const FoParams& P, long long vi, double* xv) {
  bool ok = true;
  int p = 0;
#pragma unroll
  for (int dz = -1; dz <= 1; dz++)
#pragma unroll
    for (int dy = -1; dy <= 1; dy++)
#pragma unroll
      for (int dx = -1; dx <= 1; dx++, p++) {
        const long long j = vi + (long long)dz * P.sz + (long long)dy * P.sy + dx;
        if (mask) ok &= mask[j] != 0;
        xv[p] = (double)img[j];
        ok &= xv[p] == xv[p];
      }
  return ok;
}

__device__ __forceinline__ bool firstorder_load27(const void* img, const uint8_t* mask, const FoParams& P, long long vi,
                                                  double* xv) {
  switch (P.dtype) {
    case RB_DT_INT16: return firstorder_load27((const int16_t*)img, mask, P, vi, xv);
    case RB_DT_INT32: return firstorder_load27((const int32_t*)img, mask, P, vi, xv);
    case RB_DT_FLOAT32: return firstorder_load27((const float*)img, mask, P, vi, xv);
    case RB_DT_FLOAT64: return firstorder_load27((const double*)img, mask, P, vi, xv);
    case RB_DT_UINT8: return firstorder_load27((const uint8_t*)img, mask, P, vi, xv);
    case RB_DT_UINT16: return firstorder_load27((const uint16_t*)img, mask, P, vi, xv);
    default: return firstorder_load27((const long long*)img, mask, P, vi, xv);
  }
}

// 128 threads, 4 blocks per SM (<= 128 registers); the sorted windows live in shared memory, [rank][thread]
constexpr int FO_NT = 128;
template <int NT>
__global__ void __launch_bounds__(NT, 4)
firstorder_tiles_kernel(const void* __restrict__ img, const uint8_t* __restrict__ mask,
                        const uint8_t* __restrict__ centers, const uint8_t* __restrict__ lev,
                        const __grid_constant__ FoParams P, double* __restrict__ out, long long fstride) {
  __shared__ double scr[27 * NT];
  __shared__ long long defer[2 * NT];                              // chunk indices of the centres left to the generic body
  __shared__ unsigned ndefer;
  const int tid = threadIdx.x;
  if (tid == 0) ndefer = 0;
  __syncthreads();
  const long long plane = (long long)P.Y * P.X;
  full_window_tiles<NT>((long long)(P.z1 - P.z0) * plane, defer, ndefer,
    [&](long long t, bool live, auto defer_it) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, t);
      if (!firstorder_center(mask, centers, v)) {
#pragma unroll
        for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = P.init_value;
        return;
      }
      int wl[27];
      double xv[27];
      if (load_window27(lev, P, v.z, v.y, v.x, v.vi, true, wl, 1) && firstorder_load27(img, mask, P, v.vi, xv)) {
        double f[FIRSTORDER_NF];
        firstorder_full_body(xv, wl, P.shift, P.voxel_volume, scr + tid, NT, f);
#pragma unroll
        for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = f[k];
      } else {
        defer_it();
      }
    },
    [&](auto entry, bool live) {
      if (!live) return;
      const ChunkVoxel v = chunk_voxel(P, plane, P.z0, P.out_z0, entry());
      double f[FIRSTORDER_NF];
      firstorder_generic<27>(img, mask, lev, P, v.z, v.y, v.x, f);
#pragma unroll
      for (int k = 0; k < FIRSTORDER_NF; k++) out[k * fstride + v.oi] = f[k];
    });
}

static FoParams fo_params(int dtype, int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift,
                          double voxel_volume, double init_value, int z0, int z1, int out_z0) {
  return FoParams{Z, Y, X, (long long)Y * X, X, rz, ry, rx, z0, z1, out_z0, dtype, level_bytes, shift, voxel_volume,
                  init_value};
}

bool firstorder_fast_applicable(int level_bytes, int rz, int ry, int rx) {
  return level_bytes == 1 && rz == 1 && ry == 1 && rx == 1;
}

int firstorder_fast_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                           int Z, int Y, int X, double shift, double voxel_volume, double init_value, double* out,
                           long long fstride, int z0, int z1, int out_z0, cudaStream_t st) {
  const FoParams P = fo_params(dtype, 1, Z, Y, X, 1, 1, 1, shift, voxel_volume, init_value, z0, z1, out_z0);
  const long long total = (long long)(z1 - z0) * Y * X;
  if (total <= 0) return RB_OK;
  int grid = 0;
  RB_CUDA(resident_grid(firstorder_tiles_kernel<FO_NT>, FO_NT, 0, total, grid));
  firstorder_tiles_kernel<FO_NT><<<grid, FO_NT, 0, st>>>(img, mask, centers, (const uint8_t*)lev, P, out, fstride);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

int firstorder_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                      int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift, double voxel_volume,
                      double init_value, double* out, long long fstride, int z0, int z1, int out_z0, cudaStream_t st) {
  const FoParams P = fo_params(dtype, level_bytes, Z, Y, X, rz, ry, rx, shift, voxel_volume, init_value, z0, z1, out_z0);
  const long long total = (long long)(z1 - z0) * Y * X;
  if (total <= 0) return RB_OK;
  const int grid = grid_for(total, 128, 32);
  const int wcap = (2 * rz + 1) * (2 * ry + 1) * (2 * rx + 1);
  if (wcap <= 27) firstorder_kernel<27><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else if (wcap <= 125) firstorder_kernel<125><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else if (wcap <= 343) firstorder_kernel<343><<<grid, 128, 0, st>>>(img, mask, centers, lev, P, out, fstride);
  else return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb

// Fused voxel-based feature-map kernels, generic path: one thread per centre voxel evaluates a
// whole texture class over its kernel window with the per-voxel math of vox_features.cuh and
// writes the feature maps with coalesced stores (consecutive threads = consecutive x).  Handles
// any kernelRadius <= 3, distances subset {1,2,3}, force2D, asymmetric / weighted GLCM, uint8 or
// uint16 levels, float64 or float32 maps (store_map).  The r=1 fast path lives in voxel_fast.cu.
#include "common.cuh"
#include "vox_features.cuh"
#include "voxel_tiles.cuh"

namespace rb {

template <typename T, int WCAP, int CLS, bool WEIGHTED, typename OutT>
__global__ void __launch_bounds__(128)
voxel_features_kernel(const T* __restrict__ lev, const uint8_t* __restrict__ centers,
                      const __grid_constant__ VoxParams P, OutT* __restrict__ out, long long fstride,
                      int z0, int z1, int out_z0, int* __restrict__ status) {
  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t);
    const bool is_center = chunk_center(lev, centers, plane, v);
    constexpr int NF = CLS == C_GLCM ? GLCM_NF : CLS == C_GLRLM ? GLRLM_NF : CLS == C_GLSZM ? GLSZM_NF
                       : CLS == C_GLDM ? GLDM_NF : NGTDM_NF;
    if (!is_center) {
#pragma unroll
      for (int k = 0; k < NF; k++) store_map(out + k * fstride + v.oi, P.init_value);
      continue;
    }
    uint16_t w[WCAP];
    load_window<T>(lev, P, v.z, v.y, v.x, w);
    double f[NF];
    int st = 0;
    if (CLS == C_GLCM) glcm_voxel<WCAP, WEIGHTED>(w, P, f, &st);
    else if (CLS == C_GLRLM) glrlm_voxel<WCAP, WEIGHTED>(w, P, f);
    else if (CLS == C_GLSZM) glszm_voxel<WCAP>(w, P, f);
    else if (CLS == C_GLDM) gldm_voxel<WCAP>(w, P, f);
    else ngtdm_voxel<WCAP>(w, P, f);
#pragma unroll
    for (int k = 0; k < NF; k++) store_map(out + k * fstride + v.oi, f[k]);
    if (st && status) atomicOr(status, st);
  }
}

// which GLCM angles have at least one co-occurrence in at least one kernel window
template <typename T>
__global__ void __launch_bounds__(256)
glcm_alive_kernel(const T* __restrict__ lev, const uint8_t* __restrict__ centers,
                  const __grid_constant__ VoxParams P, uint32_t* __restrict__ alive) {
  __shared__ uint32_t s_alive[(NW_MAX + 31) / 32];
  if (threadIdx.x < (NW_MAX + 31) / 32) s_alive[threadIdx.x] = 0;
  __syncthreads();
  const long long plane = (long long)P.Y * P.X, total = (long long)P.Z * plane;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / P.X, x = rem % P.X;
    const bool is_center = centers ? centers[t] != 0 : lev[(long long)z * P.sz + (long long)y * P.sy + x] != 0;
    if (!is_center) continue;
    for (int a = 0; a < P.na; a++) {
      if (s_alive[a >> 5] >> (a & 31) & 1u) continue;
      const int az = P.ang[a][0], ay = P.ang[a][1], ax = P.ang[a][2];
      bool found = false;
      for (int dz = -P.rz; dz <= P.rz && !found; dz++)
        for (int dy = -P.ry; dy <= P.ry && !found; dy++)
          for (int dx = -P.rx; dx <= P.rx && !found; dx++) {
            if (dz + az < -P.rz || dz + az > P.rz || dy + ay < -P.ry || dy + ay > P.ry || dx + ax < -P.rx || dx + ax > P.rx) continue;
            const int z1 = z + dz, y1 = y + dy, x1 = x + dx, z2 = z1 + az, y2 = y1 + ay, x2 = x1 + ax;
            if (z1 < 0 || z1 >= P.Z || y1 < 0 || y1 >= P.Y || x1 < 0 || x1 >= P.X) continue;
            if (z2 < 0 || z2 >= P.Z || y2 < 0 || y2 >= P.Y || x2 < 0 || x2 >= P.X) continue;
            if (lev[(long long)z1 * P.sz + (long long)y1 * P.sy + x1] && lev[(long long)z2 * P.sz + (long long)y2 * P.sy + x2]) found = true;
          }
      if (found) atomicOr(&s_alive[a >> 5], 1u << (a & 31));
    }
  }
  __syncthreads();
  if (threadIdx.x < (NW_MAX + 31) / 32 && s_alive[threadIdx.x]) atomicOr(&alive[threadIdx.x], s_alive[threadIdx.x]);
}

template <typename TO>
__global__ void __launch_bounds__(256)
pack_levels_kernel(const int32_t* __restrict__ image, const uint8_t* __restrict__ mask, long long n, int Ng,
                   TO* __restrict__ lev, uint32_t* __restrict__ presence, int* __restrict__ status) {
  bool bad = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    TO v = 0;
    if (mask[i]) {
      const int g = image[i];
      if (g <= 0 || g > Ng) bad = true;
      else { v = (TO)g; if (presence) atomicAdd(&presence[g - 1], 1u); }
    }
    lev[i] = v;
  }
  if (bad && status) atomicOr(status, 1);
}

int voxel_features_generic(const VoxLaunch& A) {
  const long long total = (long long)(A.z1 - A.z0) * A.P.Y * A.P.X;
  return with_level_type(A.level_bytes, [&](auto lt) -> int {
    return with_window_class(window_capacity(A.P), [&](auto wcap) -> int {
      return with_map_type(A.out_f32, [&](auto ot) -> int {
        using T = decltype(lt);
        using OutT = decltype(ot);
        constexpr int WCAP = decltype(wcap)::value;
        if (total <= 0) return RB_OK;
        auto launch = [&](auto kernel) -> int {
          kernel<<<grid_for(total, 128, 64), 128, 0, A.st>>>((const T*)A.lev, A.centers, A.P, (OutT*)A.out, A.fstride,
                                                             A.z0, A.z1, A.out_z0, A.status);
          RB_LAUNCH_CHECK();
          return RB_OK;
        };
        const bool wgt = A.P.weighted != 0;
        switch (A.cls) {
          case C_GLCM: return wgt ? launch(voxel_features_kernel<T, WCAP, C_GLCM, true, OutT>)
                                  : launch(voxel_features_kernel<T, WCAP, C_GLCM, false, OutT>);
          case C_GLRLM: return wgt ? launch(voxel_features_kernel<T, WCAP, C_GLRLM, true, OutT>)
                                   : launch(voxel_features_kernel<T, WCAP, C_GLRLM, false, OutT>);
          case C_GLSZM: return launch(voxel_features_kernel<T, WCAP, C_GLSZM, false, OutT>);
          case C_GLDM: return launch(voxel_features_kernel<T, WCAP, C_GLDM, false, OutT>);
          case C_NGTDM: return launch(voxel_features_kernel<T, WCAP, C_NGTDM, false, OutT>);
          default: return fail(RB_ERR_ARG, "unknown texture class %d", A.cls);
        }
      });
    });
  });
}

int glcm_alive_angles(const void* lev, int level_bytes, const uint8_t* centers, const VoxParams& P, uint32_t* alive,
                      cudaStream_t st) {
  const long long total = (long long)P.Z * P.Y * P.X;
  const int grid = grid_for(total, 256, 8);
  return with_level_type(level_bytes, [&](auto lt) -> int {
    using T = decltype(lt);
    glcm_alive_kernel<T><<<grid, 256, 0, st>>>((const T*)lev, centers, P, alive);
    RB_LAUNCH_CHECK();
    return RB_OK;
  });
}

int pack_levels(const int32_t* image, const uint8_t* mask, long long n, int Ng, void* lev, uint32_t* presence,
                int* status, cudaStream_t st) {
  if (Ng < 1 || Ng > 65535) return fail(RB_ERR_UNSUPPORTED, "Ng=%d outside 1..65535", Ng);
  const int grid = grid_for(n, 256, 16);
  if (Ng <= 255) pack_levels_kernel<uint8_t><<<grid, 256, 0, st>>>(image, mask, n, Ng, (uint8_t*)lev, presence, status);
  else pack_levels_kernel<uint16_t><<<grid, 256, 0, st>>>(image, mask, n, Ng, (uint16_t*)lev, presence, status);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb

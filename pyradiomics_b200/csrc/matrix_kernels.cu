// Texture-MATRIX builders of the cMatrices API surface (what reference radiomics/src/cmatrices.c computes) from host
// image + mask: prepare() uploads and packs the levels (range check), then
//
//   segment mode : segment_matrices / segment_glrlm / segment_glszm (segment_kernels.cu), on the default stream.
//   voxel batch  : one thread per listed voxel writes its private dense matrix (no atomics, reference
//                  radiomics/src/_cmatrices.c:203-207 etc.); this is the API-compatibility path -- the product's
//                  voxel-based features never materialise these (see voxel_kernels.cu / voxel_fast.cu).
// GLSZM is two-phase in both modes: phase one leaves its zones in a GlszmHandle, glszm_fill turns them into the matrix.
#include "common.cuh"
#include "host_common.hpp"
#include "vox_features.cuh"

namespace rb {

// u32 counts -> float64 (segment_kernels.cu)
__global__ void u32_to_f64_kernel(const unsigned* __restrict__ hist, long long n, double* __restrict__ out);

// GLSZM (segment) phase two: the (gray, size) pairs of segment_glszm -> u32 histogram [Ng][max_region]
__global__ void __launch_bounds__(256)
zones_fill_kernel(const int* __restrict__ zones, unsigned nzones, int Ng, int max_region, unsigned* __restrict__ hist,
                  int* __restrict__ status) {
  for (unsigned k = blockIdx.x * blockDim.x + threadIdx.x; k < nzones; k += gridDim.x * blockDim.x) {
    const int g = zones[2 * (size_t)k], s = zones[2 * (size_t)k + 1];
    if (g < 1 || g > Ng || s > max_region) { atomicOr(status, 1); continue; }
    atomicAdd(&hist[(size_t)(g - 1) * max_region + (s - 1)], 1u);
  }
}

// ------------------------------------------------------------------------------- voxel batches
struct BatchGeom {
  int Z, Y, X, rz, ry, rx, nvox;
};

template <typename T, int WCAP>
__device__ __forceinline__ void batch_window(const T* __restrict__ lev, const BatchGeom& G, const int* __restrict__ voxels,
                                             int v, uint16_t* w, VoxParams& P) {
  P.Z = G.Z; P.Y = G.Y; P.X = G.X; P.sy = G.X; P.sz = (long long)G.X * G.Y; P.rz = G.rz; P.ry = G.ry; P.rx = G.rx;
  load_window<T>(lev, P, voxels[v], voxels[G.nvox + v], voxels[2 * G.nvox + v], w);
}

// MODE 0 glcm, 1 gldm, 2 ngtdm, 3 glrlm.  A GLRLM run longer than Nr sets bit 1 of *status and is not counted: its
// flat index would fall in the next gray level's row, or past the voxel's matrix at the top level.
template <typename T, int WCAP, int MODE>
__global__ void __launch_bounds__(128)
batch_matrix_kernel(const T* __restrict__ lev, BatchGeom G, const int* __restrict__ voxels,
                    const __grid_constant__ AngleSet A, int Ng, int Nr, int alpha, double* __restrict__ out,
                    int* __restrict__ status) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= G.nvox) return;
  uint16_t w[WCAP];
  VoxParams P;
  batch_window<T, WCAP>(lev, G, voxels, v, w, P);
  const WinGeom W(P);
  if (MODE == 0) {
    double* o = out + (size_t)v * Ng * Ng * A.na;
    for (int z = 0; z < W.wz; z++) for (int y = 0; y < W.wy; y++) for (int x = 0; x < W.wx; x++) {
      const int gi = w[W.idx(z, y, x)];
      if (!gi) continue;
      for (int a = 0; a < A.na; a++) {
        const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
        if (!W.inside(z2, y2, x2)) continue;
        const int gj = w[W.idx(z2, y2, x2)];
        if (gj) o[((size_t)(gi - 1) * Ng + (gj - 1)) * A.na + a] += 1.0;
      }
    }
  } else if (MODE == 1 || MODE == 2) {
    const int ncol = 2 * A.na + 1;
    double* o = out + (size_t)v * Ng * (MODE == 1 ? ncol : 3);
    if (MODE == 2) for (int g = 0; g < Ng; g++) o[g * 3 + 2] = g + 1;
    for (int z = 0; z < W.wz; z++) for (int y = 0; y < W.wy; y++) for (int x = 0; x < W.wx; x++) {
      const int gi = w[W.idx(z, y, x)];
      if (!gi) continue;
      int dep = 0; double cnt = 0, sum = 0;
      for (int a = 0; a < A.na; a++) {
        const int z2 = z + A.a[a][0], y2 = y + A.a[a][1], x2 = x + A.a[a][2];
        if (!W.inside(z2, y2, x2)) continue;
        const int gj = w[W.idx(z2, y2, x2)];
        if (!gj) continue;
        int d = gi - gj;
        if (d < 0) d = -d;
        if (d <= alpha) dep++;
        cnt += 1; sum += gj;
      }
      if (MODE == 1) o[(size_t)(gi - 1) * ncol + dep] += 1.0;
      else { o[(gi - 1) * 3] += 1.0; o[(gi - 1) * 3 + 1] += cnt == 0 ? 0.0 : fabs((double)gi - sum / cnt); }
    }
  } else {
    double* o = out + (size_t)v * Ng * Nr * A.na;
    bool too_long = false;
    for (int a = 0; a < A.na; a++) {
      const int az = A.a[a][0], ay = A.a[a][1], ax = A.a[a][2];
      const auto count = [&](int gl, int rl) {
        if (rl < Nr) o[((size_t)(gl - 1) * Nr + rl) * A.na + a] += 1.0;
        else too_long = true;
      };
      bool multi = false;
      for (int z = 0; z < W.wz; z++) for (int y = 0; y < W.wy; y++) for (int x = 0; x < W.wx; x++) {
        if (W.inside(z - az, y - ay, x - ax)) continue;
        int cz = z, cy = y, cx = x, gl = 0, rl = 0, elements = 0;
        while (W.inside(cz, cy, cx)) {
          const int g = w[W.idx(cz, cy, cx)];
          if (g) {
            elements++;
            if (!gl) { gl = g; rl = 0; }
            else if (g == gl) rl++;
            else { count(gl, rl); gl = g; rl = 0; }
          } else if (gl) { count(gl, rl); gl = 0; rl = 0; }
          cz += az; cy += ay; cx += ax;
        }
        if (gl) count(gl, rl);
        if (elements > 1) multi = true;
      }
      if (!multi) for (int g = 0; g < Ng; g++) o[((size_t)g * Nr) * A.na + a] = 0.0;
    }
    if (too_long) atomicOr(status, 2);
  }
}

// GLSZM per listed voxel: zone list (gray,size) pairs, count per voxel, global max size
template <typename T, int WCAP>
__global__ void __launch_bounds__(128)
batch_glszm_zones_kernel(const T* __restrict__ lev, BatchGeom G, const int* __restrict__ voxels,
                         const __grid_constant__ AngleSet A, int* __restrict__ zones /*[nvox][2*WCAP]*/,
                         int* __restrict__ nz, unsigned* __restrict__ max_region) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= G.nvox) return;
  uint16_t w[WCAP], stack[WCAP];
  VoxParams P;
  batch_window<T, WCAP>(lev, G, voxels, v, w, P);
  const WinGeom W(P);
  int* zo = zones + (size_t)v * 2 * WCAP;
  int count = 0; unsigned mx = 0;
  for (int s = 0; s < W.n; s++) {
    const uint16_t gl = w[s];
    if (!gl) continue;
    int top = 0, region = 0;
    stack[top++] = (uint16_t)s; w[s] = 0;
    while (top) {
      const int k = stack[--top];
      region++;
      const int kz = k / (W.wy * W.wx), ky = (k / W.wx) % W.wy, kx = k % W.wx;
      for (int a = 0; a < A.na; a++) {
        const int z = kz + A.a[a][0], y = ky + A.a[a][1], x = kx + A.a[a][2];
        if (!W.inside(z, y, x)) continue;
        const int j = W.idx(z, y, x);
        if (w[j] == gl) { stack[top++] = (uint16_t)j; w[j] = 0; }
      }
    }
    zo[2 * count] = gl; zo[2 * count + 1] = region; count++;
    if ((unsigned)region > mx) mx = region;
  }
  nz[v] = count;
  atomicMax(max_region, mx);
}
__global__ void __launch_bounds__(128)
batch_glszm_fill_kernel(const int* __restrict__ zones, const int* __restrict__ nz, int nvox, int wcap, int Ng,
                        int max_region, double* __restrict__ out, int* __restrict__ status) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvox) return;
  const int* zo = zones + (size_t)v * 2 * wcap;
  for (int k = 0; k < nz[v]; k++) {
    const int g = zo[2 * k], s = zo[2 * k + 1];
    if (g < 1 || g > Ng || s > max_region) { atomicOr(status, 1); continue; }
    out[((size_t)v * Ng + (g - 1)) * max_region + (s - 1)] += 1.0;
  }
}

// =============================================================================== host drivers
int pack_levels(const int32_t* image, const uint8_t* mask, long long n, int Ng, void* lev, uint32_t* presence,
                int* status, cudaStream_t st);

// Host image + mask -> packed levels in `lev` (1 byte per voxel when Ng <= 255, else 2) on the default stream; a gray
// level outside 1..Ng inside the mask sets bit 0 of *status_dev (zeroed by the caller).
int upload_levels(const int32_t* image, const uint8_t* mask, long long n, int Ng, DevBuf& lev, int* status_dev) {
  DevBuf dimg, dmsk;
  RB_CUDA(dimg.alloc(n * 4));
  RB_CUDA(dmsk.alloc(n));
  RB_CUDA(lev.alloc(n * (Ng <= 255 ? 1 : 2)));
  RB_CUDA(cudaMemcpyAsync(dimg.p, image, n * 4, cudaMemcpyHostToDevice, 0));
  RB_CUDA(cudaMemcpyAsync(dmsk.p, mask, n, cudaMemcpyHostToDevice, 0));
  const int rc = pack_levels(dimg.as<int32_t>(), dmsk.as<uint8_t>(), n, Ng, lev.p, nullptr, status_dev, 0);
  if (rc) return rc;
  RB_CUDA(cudaStreamSynchronize(0));     // dimg / dmsk go out of scope
  return RB_OK;
}

struct Prepared {
  SegmentGeometry G;
  int nd, f2, lb;
  DevBuf lev, status, vox;
};

// common front end of the host-pointer API: segment geometry (angles_out, may be NULL, gets the offsets), upload + pack
// (range check), optional voxel list upload
static int prepare(const int32_t* image, const uint8_t* mask, const int* size, int nd, const int* distances, int ndist,
                   bool bidirectional, int Ng, int force2D, int force2Ddimension, const int* voxels, int nvox,
                   int kernelRadius, int* angles_out, Prepared& R) {
  if (!image || !mask || !size || (nd != 2 && nd != 3)) return fail(RB_ERR_ARG, "image/mask must be 2-D or 3-D");
  if (voxels && kernelRadius <= 0) return fail(RB_ERR_ARG, "Expecting kernelRadius > 0");
  int rc = segment_geometry(size, nd, distances, ndist, bidirectional, force2D, force2Ddimension, Ng, NA_MAX, angles_out,
                            R.G);
  if (rc) return rc;
  R.nd = nd;
  R.f2 = force2D ? force2Ddimension + (3 - nd) : -1;
  R.lb = Ng <= 255 ? 1 : 2;
  RB_CUDA(R.status.alloc(4));
  RB_CUDA(cudaMemsetAsync(R.status.p, 0, 4, 0));
  rc = upload_levels(image, mask, R.G.n, Ng, R.lev, R.status.as<int>());
  if (rc) return rc;
  if (voxels) {
    if (nvox < 1) return fail(RB_ERR_ARG, "empty voxel list");
    std::vector<int> v3((size_t)3 * nvox, 0);
    for (int d = 0; d < nd; d++) memcpy(&v3[(size_t)(d + 3 - nd) * nvox], voxels + (size_t)d * nvox, sizeof(int) * nvox);
    for (int d = 0; d < nd; d++)
      for (int v = 0; v < nvox; v++) {
        int c = voxels[(size_t)d * nvox + v];
        if (c < 0 || c >= size[d]) return fail(RB_ERR_ARG, "voxel index out of range");
      }
    RB_CUDA(R.vox.alloc(sizeof(int) * 3 * (size_t)nvox));
    RB_CUDA(cudaMemcpyAsync(R.vox.p, v3.data(), sizeof(int) * 3 * (size_t)nvox, cudaMemcpyHostToDevice, 0));
    RB_CUDA(cudaStreamSynchronize(0));   // v3 is a temporary
  }
  return RB_OK;
}

static int check_status(const Prepared& R, const char* what) {
  int st = 0;
  RB_CUDA(cudaMemcpy(&st, R.status.p, sizeof st, cudaMemcpyDeviceToHost));
  if (st & 1) return fail(RB_ERR_LEVEL_RANGE, "Calculation of %s Failed: gray level outside 1..Ng inside the mask", what);
  if (st & 2) return fail(RB_ERR_LEVEL_RANGE, "Calculation of %s Failed: run longer than Nr", what);
  return RB_OK;
}

static BatchGeom batch_geom(const Prepared& R, int kernelRadius, int nvox) {
  BatchGeom G;
  G.Z = R.G.Z; G.Y = R.G.Y; G.X = R.G.X; G.nvox = nvox;
  G.rz = (R.f2 == 0 || R.nd == 2) ? 0 : kernelRadius;
  G.ry = R.f2 == 1 ? 0 : kernelRadius;
  G.rx = R.f2 == 2 ? 0 : kernelRadius;
  return G;
}

template <typename T, int MODE>
static int launch_batch(const Prepared& R, const BatchGeom& G, int Ng, int Nr, int alpha, double* out) {
  const int cap = (2 * G.rz + 1) * (2 * G.ry + 1) * (2 * G.rx + 1);
  const int grid = (G.nvox + 127) / 128;
  const T* lev = R.lev.as<const T>();
  const int* vox = R.vox.as<const int>();
  int* st = R.status.as<int>();
  if (cap <= 27) batch_matrix_kernel<T, 27, MODE><<<grid, 128>>>(lev, G, vox, R.G.A, Ng, Nr, alpha, out, st);
  else if (cap <= 125) batch_matrix_kernel<T, 125, MODE><<<grid, 128>>>(lev, G, vox, R.G.A, Ng, Nr, alpha, out, st);
  else if (cap <= 343) batch_matrix_kernel<T, 343, MODE><<<grid, 128>>>(lev, G, vox, R.G.A, Ng, Nr, alpha, out, st);
  else return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  RB_LAUNCH_CHECK();
  return RB_OK;
}

// one driver for GLCM (mode 0) / GLDM (1) / NGTDM (2) / GLRLM (3) from host image + mask
int calculate_matrix_host(int mode, const int32_t* image, const uint8_t* mask, const int* size, int nd,
                          const int* distances, int ndist, int Ng, int Nr, int alpha, int force2D, int force2Ddimension,
                          int kernelRadius, const int* voxels, int nvox, double* out_host, int* angles_out) {
  static const char* names[] = {"GLCM", "GLDM", "NGTDM", "GLRLM"};
  Prepared R;
  const int one[1] = {1};
  const bool bidir = mode == 1 || mode == 2;
  int rc = prepare(image, mask, size, nd, mode == 3 ? one : distances, mode == 3 ? 1 : ndist, bidir, Ng, force2D,
                   force2Ddimension, voxels, nvox, kernelRadius, angles_out, R);
  if (rc) return rc;
  if (!voxels) {
    rc = mode == 3 ? segment_glrlm(R.lev.p, R.lb, size, nd, Ng, Nr, force2D, force2Ddimension, out_host, angles_out, 0)
                   : segment_matrices(R.lev.p, R.lb, size, nd, distances, ndist, Ng, alpha, force2D, force2Ddimension,
                                      mode == 0 ? out_host : nullptr, mode == 1 ? out_host : nullptr,
                                      mode == 2 ? out_host : nullptr, angles_out, 0);
    return rc ? rc : check_status(R, names[mode]);
  }
  const int na = R.G.A.na;
  size_t per = mode == 0 ? (size_t)Ng * Ng * na : mode == 1 ? (size_t)Ng * (2 * na + 1) : mode == 2 ? (size_t)Ng * 3
                                                                                            : (size_t)Ng * Nr * na;
  if (mode == 3 && Nr < 1) return fail(RB_ERR_ARG, "Nr must be >= 1");
  DevBuf dout;
  RB_CUDA(dout.alloc(sizeof(double) * per * nvox));
  RB_CUDA(cudaMemsetAsync(dout.p, 0, sizeof(double) * per * nvox, 0));
  double* out = dout.as<double>();
  BatchGeom G = batch_geom(R, kernelRadius, nvox);
#define RB_B(MODE) (R.lb == 1 ? launch_batch<uint8_t, MODE>(R, G, Ng, Nr, alpha, out) : launch_batch<uint16_t, MODE>(R, G, Ng, Nr, alpha, out))
  rc = mode == 0 ? RB_B(0) : mode == 1 ? RB_B(1) : mode == 2 ? RB_B(2) : RB_B(3);
#undef RB_B
  if (rc) return rc;
  rc = check_status(R, names[mode]);
  if (rc) return rc;
  RB_CUDA(cudaMemcpy(out_host, out, sizeof(double) * per * nvox, cudaMemcpyDeviceToHost));
  return RB_OK;
}

// ---- GLSZM two-phase --------------------------------------------------------------------
// phase one from host image + mask: the whole ROI (segment mode) or one zone list per listed voxel
int glszm_zones_host(const int32_t* image, const uint8_t* mask, const int* size, int nd, int Ng, int force2D,
                     int force2Ddimension, int kernelRadius, const int* voxels, int nvox, int* max_region_out,
                     void** handle_out) {
  Prepared R;
  const int one[1] = {1};
  int rc = prepare(image, mask, size, nd, one, 1, true, Ng, force2D, force2Ddimension, voxels, nvox, kernelRadius, nullptr, R);
  if (rc) return rc;
  rc = check_status(R, "GLSZM");
  if (rc) return rc;
  if (!voxels) return segment_glszm(R.lev.p, R.lb, size, nd, Ng, force2D, force2Ddimension, max_region_out, handle_out, 0);
  BatchGeom G = batch_geom(R, kernelRadius, nvox);
  const int cap = (2 * G.rz + 1) * (2 * G.ry + 1) * (2 * G.rx + 1);
  const int wcap = cap <= 27 ? 27 : cap <= 125 ? 125 : 343;
  if (cap > 343) return fail(RB_ERR_UNSUPPORTED, "kernelRadius > 3 is outside the implemented envelope");
  std::unique_ptr<GlszmHandle> H(new GlszmHandle);   // handed to the caller only on success
  H->batch = true; H->nvox = nvox; H->wcap = wcap;
  RB_CUDA(H->zones.alloc(sizeof(int) * 2 * (size_t)wcap * nvox));
  RB_CUDA(H->nz.alloc(sizeof(int) * (size_t)nvox));
  DevBuf mx;
  RB_CUDA(mx.alloc(4));
  RB_CUDA(cudaMemsetAsync(mx.p, 0, 4, 0));
  const int grid = (nvox + 127) / 128;
  const int* vox = R.vox.as<const int>();
#define RB_Z(T, W) batch_glszm_zones_kernel<T, W><<<grid, 128>>>(R.lev.as<const T>(), G, vox, R.G.A, H->zones.as<int>(), H->nz.as<int>(), mx.as<unsigned>())
  if (R.lb == 1) { if (wcap == 27) RB_Z(uint8_t, 27); else if (wcap == 125) RB_Z(uint8_t, 125); else RB_Z(uint8_t, 343); }
  else { if (wcap == 27) RB_Z(uint16_t, 27); else if (wcap == 125) RB_Z(uint16_t, 125); else RB_Z(uint16_t, 343); }
#undef RB_Z
  RB_LAUNCH_CHECK();
  unsigned max_region = 0;
  RB_CUDA(cudaMemcpy(&max_region, mx.p, 4, cudaMemcpyDeviceToHost));
  *max_region_out = (int)max_region;
  *handle_out = H.release();
  return RB_OK;
}

// phase two on the handle's stream; consumes the handle on every path
int glszm_fill(void* handle, int Ng, int max_region, double* out_host) {
  std::unique_ptr<GlszmHandle> H((GlszmHandle*)handle);
  if (!H) return fail(RB_ERR_ARG, "null GLSZM handle");
  if (max_region < 1) max_region = 1;
  const cudaStream_t st = H->st;
  const size_t per = (size_t)Ng * max_region, tot = per * H->nvox;
  DevBuf dout, status, hist;
  RB_CUDA(dout.alloc(tot * 8));
  RB_CUDA(status.alloc(4));
  RB_CUDA(cudaMemsetAsync(dout.p, 0, tot * 8, st));
  RB_CUDA(cudaMemsetAsync(status.p, 0, 4, st));
  if (H->batch) {
    batch_glszm_fill_kernel<<<(H->nvox + 127) / 128, 128, 0, st>>>(H->zones.as<const int>(), H->nz.as<const int>(), H->nvox,
                                                                  H->wcap, Ng, max_region, dout.as<double>(), status.as<int>());
  } else {
    RB_CUDA(hist.alloc(per * 4));
    RB_CUDA(cudaMemsetAsync(hist.p, 0, per * 4, st));
    if (H->nzones) zones_fill_kernel<<<grid_for(H->nzones, 256, 8), 256, 0, st>>>(H->zones.as<const int>(), H->nzones, Ng, max_region, hist.as<unsigned>(), status.as<int>());
    u32_to_f64_kernel<<<grid_for((long long)per, 256, 8), 256, 0, st>>>(hist.as<unsigned>(), (long long)per, dout.as<double>());
  }
  RB_LAUNCH_CHECK();
  int stv = 0;
  RB_CUDA(cudaMemcpyAsync(&stv, status.p, 4, cudaMemcpyDeviceToHost, st));
  RB_CUDA(cudaStreamSynchronize(st));
  if (stv) return fail(RB_ERR_LEVEL_RANGE, "Error filling GLSZM.");
  RB_CUDA(cudaMemcpyAsync(out_host, dout.p, tot * 8, cudaMemcpyDeviceToHost, st));
  RB_CUDA(cudaStreamSynchronize(st));
  return RB_OK;
}

}  // namespace rb

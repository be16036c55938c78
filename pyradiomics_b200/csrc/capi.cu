// extern "C" surface of libb200radiomics.so (declared in include/b200radiomics.h).
#include <stdarg.h>
#include <stdlib.h>

#include <vector>

#include "common.cuh"
#include "host_common.hpp"
#include "pixel.cuh"

namespace rb {

std::string& last_error_ref() {
  static thread_local std::string s;
  return s;
}
int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  last_error_ref() = buf;
  return code;
}

// the voxel kernels' launch functions: `out` holds float maps when out_f32, else double
int voxel_features_generic(int cls, const void* lev, int level_bytes, const uint8_t* centers, const VoxParams& P,
                           void* out, bool out_f32, long long fstride, int z0, int z1, int out_z0, int* status,
                           cudaStream_t st);
int glcm_alive_angles(const void* lev, int level_bytes, const uint8_t* centers, const VoxParams& P, uint32_t* alive,
                      cudaStream_t st);
int pack_levels(const int32_t* image, const uint8_t* mask, long long n, int Ng, void* lev, uint32_t* presence,
                int* status, cudaStream_t st);
int glcm_release_queues();
int voxel_features_wide(int cls, const void* lev, int level_bytes, const uint8_t* centers, const VoxParams& P, void* out,
                        bool out_f32, long long fstride, int z0, int z1, int out_z0, int* status, cudaStream_t st);
int wide_release_workspace();
int voxel_fast_launch(int cls, const void* lev, const uint8_t* centers, const VoxParams& P, void* out, bool out_f32,
                      long long fstride, int z0, int z1, int out_z0, cudaStream_t st);

// B200_RADIOMICS_FORCE_GENERIC=1 routes everything through the generic kernels (used by the
// tests to cross-check the fast paths on the GPU)
static bool force_generic() {
  const char* e = getenv("B200_RADIOMICS_FORCE_GENERIC");
  return e && e[0] == '1';
}
// B200_RADIOMICS_FORCE_WIDE=1 sends every window, fast-path ones included, to the wide kernels (window_path): the tests
// compare them with the generic kernels bit for bit
static bool force_wide() {
  const char* e = getenv("B200_RADIOMICS_FORCE_WIDE");
  return e && e[0] == '1';
}

int calculate_matrix_host(int mode, const int32_t* image, const uint8_t* mask, const int* size, int nd,
                          const int* distances, int ndist, int Ng, int Nr, int alpha, int force2D, int force2Ddimension,
                          int kernelRadius, const int* voxels, int nvox, double* out_host, int* angles_out);
int upload_levels(const int32_t* image, const uint8_t* mask, long long n, int Ng, DevBuf& lev, int* status_dev);
int glszm_zones_host(const int32_t* image, const uint8_t* mask, const int* size, int nd, int Ng, int force2D,
                     int force2Ddimension, int kernelRadius, const int* voxels, int nvox, int* max_region_out,
                     void** handle_out);
int glszm_fill(void* handle, int Ng, int max_region, double* out_host);

// the arguments every rb_segment_*_dev entry point checks before it touches the device
static int check_segment_levels(const void* levels_dev, int level_bytes, const int* size, int nd, int Ng) {
  if (!levels_dev || !size || (nd != 2 && nd != 3)) return fail(RB_ERR_ARG, "levels / size");
  if (level_bytes != rb_level_bytes(Ng)) return fail(RB_ERR_ARG, "level_bytes does not match Ng");
  return RB_OK;
}

int minmax_launch(const void* img, int dt, const uint8_t* mask, long long n, long long* keys, cudaStream_t st);
int shape_coefficients_dev(const uint8_t* mask_dev, int Z, int Y, int X, long long sz, long long sy, long long sx,
                           const double* spacing, double* out7, cudaStream_t st);
int shape_moments_dev(const uint8_t* mask_dev, int Z, int Y, int X, unsigned long long* out10, cudaStream_t st);
int shape2d_coefficients_dev(const uint8_t* mask_dev, int Y, int X, long long sy, long long sx, const double* spacing, double* out4,
                             cudaStream_t st);
int digitize_launch(const void* img, int dt, const uint8_t* mask, long long n, const double* edges, int ne, int32_t* out,
                    cudaStream_t st);
int pointwise_image_launch(const void* img, int dt, long long n, int kind, double c, double* out, cudaStream_t st);
int gradient_magnitude_launch(const void* img, int dt, int Z, int Y, int X, const double* w_zyx, double* out, cudaStream_t st);
int roi_moments_launch(const void* img, int dt, const uint8_t* mask, long long n, int passes, void* scratch, double* res,
                       cudaStream_t st);
int normalize_launch(const void* img, int dt, long long n, double mean, double sigma, int clamp, double outliers,
                     double scale, double* out, cudaStream_t st);
int resegment_launch(const void* img, int dt, const uint8_t* mask, long long n, double lo, double hi, int two,
                     uint8_t* out, unsigned long long* counts, cudaStream_t st);
int swt_axis_launch(const double* in, int Z, int Y, int X, int axis, const double* lo, const double* hi, int F,
                    double* out_lo, double* out_hi, cudaStream_t st);
int recursive_gauss_launch(const void* in, int in_is_f32, int Z, int Y, int X, int axis, const double* coef20, float* out,
                           double* scratch, double scale, int accumulate, cudaStream_t st);
int swt3d_launch(const double* in, int Z, int Y, int X, const double* lo, const double* hi, int F, double* out,
                 long long band_stride, int z_begin, int z_end, cudaStream_t st);
int bspline_prefilter_launch(double* coeffs, int Z, int Y, int X, cudaStream_t st, bool exact_init);
int resample_launch(const void* src, int src_dt, const int* in_size, void* dst, int dst_dt, const int* out_size, const double* start,
                    const double* step, int interp, double default_value, cudaStream_t st);

int lbp3d_launch(const void* img, int img_dt, int sample_dt, const uint8_t* roi, int Z, int Y, int X, const double* vertices,
                 int nv, const double* harmonics, int levels, double* coeff_scratch, double* out, cudaStream_t st);
int lbp2d_launch(const void* img, int dt, int Z, int Y, int X, int axis, int P, const double* rp, const double* cp, int method,
                 int out_dt, void* out, cudaStream_t st);

int firstorder_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                      int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift, double voxel_volume,
                      double init_value, double* out, long long fstride, int z0, int z1, int out_z0, cudaStream_t st);
int firstorder_wide_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                           int level_bytes, int Z, int Y, int X, int rz, int ry, int rx, double shift, double voxel_volume,
                           double init_value, double* out, long long fstride, int z0, int z1, int out_z0, cudaStream_t st);
int firstorder_fast_launch(const void* img, int dtype, const uint8_t* mask, const uint8_t* centers, const void* lev,
                           int Z, int Y, int X, double shift, double voxel_volume, double init_value, double* out,
                           long long fstride, int z0, int z1, int out_z0, cudaStream_t st);
int firstorder_segment(const void* img, int dtype, const uint8_t* roi, const void* lev, int level_bytes, long long n,
                       double shift, double voxel_volume, double* out18_host, cudaStream_t st);
static const char* kFirstOrderNames[] = {"10Percentile", "90Percentile", "Energy", "Entropy", "InterquartileRange", "Kurtosis",
  "Maximum", "MeanAbsoluteDeviation", "Mean", "Median", "Minimum", "Range", "RobustMeanAbsoluteDeviation", "RootMeanSquared",
  "Skewness", "TotalEnergy", "Uniformity", "Variance"};

static const char* kGlcmNames[] = {"Autocorrelation", "ClusterProminence", "ClusterShade", "ClusterTendency", "Contrast",
  "Correlation", "DifferenceAverage", "DifferenceEntropy", "DifferenceVariance", "Id", "Idm", "Idmn", "Idn", "Imc1", "Imc2",
  "InverseVariance", "JointAverage", "JointEnergy", "JointEntropy", "MCC", "MaximumProbability", "SumAverage", "SumEntropy",
  "SumSquares"};
static const char* kGlrlmNames[] = {"GrayLevelNonUniformity", "GrayLevelNonUniformityNormalized", "GrayLevelVariance",
  "HighGrayLevelRunEmphasis", "LongRunEmphasis", "LongRunHighGrayLevelEmphasis", "LongRunLowGrayLevelEmphasis",
  "LowGrayLevelRunEmphasis", "RunEntropy", "RunLengthNonUniformity", "RunLengthNonUniformityNormalized", "RunPercentage",
  "RunVariance", "ShortRunEmphasis", "ShortRunHighGrayLevelEmphasis", "ShortRunLowGrayLevelEmphasis"};
static const char* kGlszmNames[] = {"GrayLevelNonUniformity", "GrayLevelNonUniformityNormalized", "GrayLevelVariance",
  "HighGrayLevelZoneEmphasis", "LargeAreaEmphasis", "LargeAreaHighGrayLevelEmphasis", "LargeAreaLowGrayLevelEmphasis",
  "LowGrayLevelZoneEmphasis", "SizeZoneNonUniformity", "SizeZoneNonUniformityNormalized", "SmallAreaEmphasis",
  "SmallAreaHighGrayLevelEmphasis", "SmallAreaLowGrayLevelEmphasis", "ZoneEntropy", "ZonePercentage", "ZoneVariance"};
static const char* kGldmNames[] = {"DependenceEntropy", "DependenceNonUniformity", "DependenceNonUniformityNormalized",
  "DependenceVariance", "GrayLevelNonUniformity", "GrayLevelVariance", "HighGrayLevelEmphasis", "LargeDependenceEmphasis",
  "LargeDependenceHighGrayLevelEmphasis", "LargeDependenceLowGrayLevelEmphasis", "LowGrayLevelEmphasis",
  "SmallDependenceEmphasis", "SmallDependenceHighGrayLevelEmphasis", "SmallDependenceLowGrayLevelEmphasis"};
static const char* kNgtdmNames[] = {"Busyness", "Coarseness", "Complexity", "Contrast", "Strength"};
static const char** kNames[5] = {kGlcmNames, kGlrlmNames, kGlszmNames, kGldmNames, kNgtdmNames};

// RB_ERR_ARG unless every code is an rb_dtype.  Each entry point that takes pixel types runs it before any CUDA call.
static int check_dtypes(std::initializer_list<int> codes) {
  for (int dt : codes)
    if (!dtype_valid(dt)) return fail(RB_ERR_ARG, "unknown dtype code %d", dt);
  return RB_OK;
}

__global__ void maps_to_f32_kernel(const double* __restrict__ src, long long sp, float* __restrict__ dst, long long dp,
                                   long long width, long long height) {
  const long long total = width * height;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / width, c = i - r * width;
    dst[r * dp + c] = (float)src[r * sp + c];
  }
}

}  // namespace rb

using namespace rb;

extern "C" {

const char* rb_last_error(void) { return last_error_ref().c_str(); }
const char* rb_version(void) { return "b200radiomics 0.1 (sm_90a)"; }

int rb_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) return fail(RB_ERR_CUDA, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  return n;
}

int rb_release_device_caches(void) {
  const int rc = glcm_release_queues();
  const int rc2 = wide_release_workspace();
  return rc ? rc : rc2;
}

int rb_num_features(int cls) { return (cls < 0 || cls > 4) ? RB_ERR_ARG : kNumFeatures[cls]; }

const char* rb_feature_name(int cls, int idx) {
  if (cls < 0 || cls > 4 || idx < 0 || idx >= kNumFeatures[cls]) return NULL;
  return kNames[cls][idx];
}

int rb_generate_angles(const int* size, int nd, const int* distances, int ndist, int bidirectional, int force2D,
                       int force2Ddimension, int* angles, int max_angles) {
  if (!size || !distances || nd < 1 || nd > 3 || ndist < 1) return fail(RB_ERR_ARG, "bad size/distances");
  std::vector<int> out;
  int na = generate_angles(size, nd, distances, ndist, bidirectional != 0, force2D ? force2Ddimension : -1, out);
  if (na <= 0) return fail(RB_ERR_ARG, "Error getting angle count.");
  if (na > max_angles) return -1000 - na;
  memcpy(angles, out.data(), sizeof(int) * (size_t)na * nd);
  return na;
}

int rb_level_bytes(int Ng) { return Ng <= 255 ? 1 : 2; }

int rb_pack_levels_dev(const int32_t* image_dev, const uint8_t* mask_dev, long long nvoxels, int Ng, void* levels_dev,
                       uint32_t* presence_dev, int* status_dev, void* stream) {
  return pack_levels(image_dev, mask_dev, nvoxels, Ng, levels_dev, presence_dev, status_dev, (cudaStream_t)stream);
}

int rb_glcm_alive_angles_dev(const void* levels_dev, int level_bytes, const uint8_t* centers_dev, int Z, int Y, int X,
                             const rb_voxel_settings* settings, uint32_t* alive_dev, void* stream) {
  VoxParams P;
  if (fill_vox_params(C_GLCM, Z, Y, X, *settings, P)) return fail(RB_ERR_ARG, "bad voxel settings");
  return glcm_alive_angles(levels_dev, level_bytes, centers_dev, P, alive_dev, (cudaStream_t)stream);
}

int rb_voxel_features_dev(int cls, const void* levels_dev, int level_bytes, const uint8_t* centers_dev, int Z, int Y,
                          int X, int z0, int z1, const rb_voxel_settings* settings, const uint32_t* alive_host,
                          void* out_dev, int out_is_f32, long long out_feature_stride, int out_z0, int* status_dev,
                          void* stream) {
  if (cls < 0 || cls > 4) return fail(RB_ERR_ARG, "unknown texture class %d", cls);
  if (z0 < 0 || z1 > Z || z0 > z1) return fail(RB_ERR_ARG, "bad z range");
  VoxParams P;
  if (fill_vox_params(cls, Z, Y, X, *settings, P)) return fail(RB_ERR_ARG, "bad voxel settings");
  if (alive_host && cls == C_GLCM) memcpy(P.alive, alive_host, sizeof P.alive);
  const bool f32 = out_is_f32 != 0, wide = force_wide();
  if (!force_generic() && !wide && voxel_fast_path(cls, level_bytes, P))
    return voxel_fast_launch(cls, levels_dev, centers_dev, P, out_dev, f32, out_feature_stride, z0, z1, out_z0,
                             (cudaStream_t)stream);
  switch (window_path(window_capacity(P), wide)) {
    case WP_GENERIC:
      return voxel_features_generic(cls, levels_dev, level_bytes, centers_dev, P, out_dev, f32, out_feature_stride, z0,
                                    z1, out_z0, status_dev, (cudaStream_t)stream);
    case WP_WIDE:
      return voxel_features_wide(cls, levels_dev, level_bytes, centers_dev, P, out_dev, f32, out_feature_stride, z0, z1,
                                 out_z0, status_dev, (cudaStream_t)stream);
    default:
      return fail(RB_ERR_UNSUPPORTED, "a kernel window of %d positions is outside the implemented envelope (at most %d: "
                  "kernelRadius <= 7 in 3-D)", window_capacity(P), WIDE_WCAP_MAX);
  }
}

int rb_memcpy2d_async(void* dst, unsigned long long dpitch, const void* src, unsigned long long spitch,
                      unsigned long long width, unsigned long long height, int kind, void* stream) {
  const cudaMemcpyKind k = kind == 1 ? cudaMemcpyHostToDevice : kind == 2 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  if (kind < 1 || kind > 3) return fail(RB_ERR_ARG, "rb_memcpy2d_async: kind must be 1, 2 or 3");
  if (!width || !height) return RB_OK;
  RB_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width, height, k, (cudaStream_t)stream));
  return RB_OK;
}

int rb_maps_to_f32_dev(const double* src_dev, long long src_pitch, float* dst_dev, long long dst_pitch, long long width,
                       long long height, void* stream) {
  if (width <= 0 || height <= 0) return RB_OK;
  maps_to_f32_kernel<<<grid_for(width * height, 256, 16), 256, 0, (cudaStream_t)stream>>>(src_dev, src_pitch, dst_dev,
                                                                                          dst_pitch, width, height);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

int rb_voxel_features_host(int cls, const int32_t* image, const uint8_t* mask, int Z, int Y, int X,
                           const rb_voxel_settings* settings, double* maps) {
  if (cls < 0 || cls > 4) return fail(RB_ERR_ARG, "unknown texture class %d", cls);
  const long long n = (long long)Z * Y * X;
  const int nf = kNumFeatures[cls];
  const int lb = rb_level_bytes(settings->Ng);
  DevBuf lev, out, status, alive_dev;
  RB_CUDA(out.alloc(sizeof(double) * n * nf));
  RB_CUDA(status.alloc(2 * sizeof(int)));
  RB_CUDA(alive_dev.alloc(RB_ALIVE_WORDS * 4));
  RB_CUDA(cudaMemsetAsync(status.p, 0, 2 * sizeof(int), 0));
  RB_CUDA(cudaMemsetAsync(alive_dev.p, 0, RB_ALIVE_WORDS * 4, 0));
  int rc = upload_levels(image, mask, n, settings->Ng, lev, status.as<int>());
  if (rc) return rc;
  uint32_t alive[RB_ALIVE_WORDS];
  if (cls == RB_GLCM) {
    rc = rb_glcm_alive_angles_dev(lev.p, lb, NULL, Z, Y, X, settings, alive_dev.as<uint32_t>(), 0);
    if (rc) return rc;
    RB_CUDA(cudaMemcpy(alive, alive_dev.p, sizeof alive, cudaMemcpyDeviceToHost));
  }
  rc = rb_voxel_features_dev(cls, lev.p, lb, NULL, Z, Y, X, 0, Z, settings, cls == RB_GLCM ? alive : NULL, out.p, 0, n, 0,
                             status.as<int>() + 1, 0);
  if (rc) return rc;
  int st[2] = {0, 0};
  RB_CUDA(cudaMemcpy(st, status.p, sizeof st, cudaMemcpyDeviceToHost));
  if (st[0] & 1) return fail(RB_ERR_LEVEL_RANGE, "gray level outside 1..Ng inside the mask");
  if (st[1] & 2) return fail(RB_ERR_UNSUPPORTED, "weighted GLCM entry list overflow");
  RB_CUDA(cudaMemcpy(maps, out.p, sizeof(double) * n * nf, cudaMemcpyDeviceToHost));
  return RB_OK;
}

int rb_calculate_glcm(const int32_t* image, const uint8_t* mask, const int* size, int nd, const int* distances, int ndist,
                      int Ng, int force2D, int force2Ddimension, int kernelRadius, const int* voxels, int nvox,
                      double* glcm, int* angles) {
  return calculate_matrix_host(0, image, mask, size, nd, distances, ndist, Ng, 0, 0, force2D, force2Ddimension,
                               kernelRadius, voxels, nvox, glcm, angles);
}
int rb_calculate_glrlm(const int32_t* image, const uint8_t* mask, const int* size, int nd, int Ng, int Nr, int force2D,
                       int force2Ddimension, int kernelRadius, const int* voxels, int nvox, double* glrlm, int* angles) {
  return calculate_matrix_host(3, image, mask, size, nd, NULL, 0, Ng, Nr, 0, force2D, force2Ddimension, kernelRadius,
                               voxels, nvox, glrlm, angles);
}
int rb_calculate_gldm(const int32_t* image, const uint8_t* mask, const int* size, int nd, const int* distances, int ndist,
                      int Ng, int alpha, int force2D, int force2Ddimension, int kernelRadius, const int* voxels, int nvox,
                      double* gldm) {
  return calculate_matrix_host(1, image, mask, size, nd, distances, ndist, Ng, 0, alpha, force2D, force2Ddimension,
                               kernelRadius, voxels, nvox, gldm, NULL);
}
int rb_calculate_ngtdm(const int32_t* image, const uint8_t* mask, const int* size, int nd, const int* distances,
                       int ndist, int Ng, int force2D, int force2Ddimension, int kernelRadius, const int* voxels,
                       int nvox, double* ngtdm) {
  return calculate_matrix_host(2, image, mask, size, nd, distances, ndist, Ng, 0, 0, force2D, force2Ddimension,
                               kernelRadius, voxels, nvox, ngtdm, NULL);
}
// ---- segment-mode matrices from a device-resident packed level volume (no host round trip of the image)
int rb_segment_texture_dev(const void* levels_dev, int level_bytes, const int* size, int nd, const int* distances, int ndist,
                           int Ng, int alpha, int force2D, int force2Ddimension, double* glcm, double* gldm, double* ngtdm,
                           int* angles, void* stream) {
  if (int rc = check_segment_levels(levels_dev, level_bytes, size, nd, Ng)) return rc;
  return segment_matrices(levels_dev, level_bytes, size, nd, distances, ndist, Ng, alpha, force2D, force2Ddimension, glcm,
                          gldm, ngtdm, angles, (cudaStream_t)stream);
}
int rb_segment_glrlm_dev(const void* levels_dev, int level_bytes, const int* size, int nd, int Ng, int Nr, int force2D,
                         int force2Ddimension, double* glrlm, int* angles, void* stream) {
  if (int rc = check_segment_levels(levels_dev, level_bytes, size, nd, Ng)) return rc;
  return segment_glrlm(levels_dev, level_bytes, size, nd, Ng, Nr, force2D, force2Ddimension, glrlm, angles,
                       (cudaStream_t)stream);
}
int rb_segment_glszm_dev(const void* levels_dev, int level_bytes, const int* size, int nd, int Ng, int force2D,
                         int force2Ddimension, int* max_region, void** handle, void* stream) {
  if (int rc = check_segment_levels(levels_dev, level_bytes, size, nd, Ng)) return rc;
  return segment_glszm(levels_dev, level_bytes, size, nd, Ng, force2D, force2Ddimension, max_region, handle,
                       (cudaStream_t)stream);
}

int rb_calculate_glszm(const int32_t* image, const uint8_t* mask, const int* size, int nd, int Ng, int force2D,
                       int force2Ddimension, int kernelRadius, const int* voxels, int nvox, int* max_region,
                       void** handle) {
  if (!max_region || !handle) return fail(RB_ERR_ARG, "null output pointer");
  return glszm_zones_host(image, mask, size, nd, Ng, force2D, force2Ddimension, kernelRadius, voxels, nvox, max_region,
                          handle);
}
int rb_fill_glszm(void* handle, int Ng, int max_region, double* glszm) { return glszm_fill(handle, Ng, max_region, glszm); }
void rb_glszm_release(void* handle) { delete (GlszmHandle*)handle; }

int rb_minmax_dev(const void* image_dev, int dtype, const uint8_t* mask_dev, long long nvoxels, long long* keys_dev,
                  void* stream) {
  if (int rc = check_dtypes({dtype})) return rc;
  return minmax_launch(image_dev, dtype, mask_dev, nvoxels, keys_dev, (cudaStream_t)stream);
}
int rb_digitize_dev(const void* image_dev, int dtype, const uint8_t* mask_dev, long long nvoxels, const double* edges_dev,
                    int nedges, int32_t* out_dev, void* stream) {
  if (int rc = check_dtypes({dtype})) return rc;
  if (nedges < 1) return fail(RB_ERR_ARG, "need at least one bin edge");
  return digitize_launch(image_dev, dtype, mask_dev, nvoxels, edges_dev, nedges, out_dev, (cudaStream_t)stream);
}
// getSquareImage / getSquareRootImage / getLogarithmImage / getExponentialImage, radiomics/imageoperations.py:973-1073
int rb_pointwise_image_dev(const void* img_dev, int dtype, long long nvoxels, int kind, double c, double* out_dev,
                           void* stream) {
  if (!img_dev || !out_dev) return fail(RB_ERR_ARG, "pointwise image: null argument");
  if (int rc = check_dtypes({dtype})) return rc;
  if (kind < RB_PW_SQUARE || kind > RB_PW_EXPONENTIAL) return fail(RB_ERR_ARG, "pointwise image: unknown kind %d", kind);
  if (nvoxels < 1) return fail(RB_ERR_ARG, "pointwise image: %lld voxels", nvoxels);
  return pointwise_image_launch(img_dev, dtype, nvoxels, kind, c, out_dev, (cudaStream_t)stream);
}
// getGradientImage (sitk.GradientMagnitudeImageFilter), radiomics/imageoperations.py:1076-1091
int rb_gradient_magnitude_dev(const void* img_dev, int dtype, int Z, int Y, int X, const double* weights_zyx,
                              double* out_dev, void* stream) {
  if (!img_dev || !weights_zyx || !out_dev) return fail(RB_ERR_ARG, "gradient magnitude: null argument");
  if (int rc = check_dtypes({dtype})) return rc;
  if (Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "gradient magnitude: empty volume %d x %d x %d", Z, Y, X);
  return gradient_magnitude_launch(img_dev, dtype, Z, Y, X, weights_zyx, out_dev, (cudaStream_t)stream);
}
// sitk.Normalize's statistics (radiomics/imageoperations.py:638) and resegmentMask's np.max / np.mean / np.std of the
// ROI (radiomics/imageoperations.py:699, 704-705)
int rb_roi_moments_dev(const void* img_dev, int dtype, const uint8_t* mask_dev, long long nvoxels, int passes,
                       void* scratch_dev, double* out_dev, void* stream) {
  if (!img_dev || !scratch_dev || !out_dev) return fail(RB_ERR_ARG, "roi moments: null argument");
  if (int rc = check_dtypes({dtype})) return rc;
  if (nvoxels < 1) return fail(RB_ERR_ARG, "roi moments: %lld voxels", nvoxels);
  if (passes != 1 && passes != 2) return fail(RB_ERR_ARG, "roi moments: passes must be 1 or 2, got %d", passes);
  return roi_moments_launch(img_dev, dtype, mask_dev, nvoxels, passes, scratch_dev, out_dev, (cudaStream_t)stream);
}
// normalizeImage (sitk.Normalize, removeOutliers, normalizeScale), radiomics/imageoperations.py:615-654
int rb_normalize_dev(const void* img_dev, int dtype, long long nvoxels, double mean, double sigma, int remove_outliers,
                     double outliers, double scale, double* out_dev, void* stream) {
  if (!img_dev || !out_dev) return fail(RB_ERR_ARG, "normalize: null argument");
  if (int rc = check_dtypes({dtype})) return rc;
  if (nvoxels < 1) return fail(RB_ERR_ARG, "normalize: %lld voxels", nvoxels);
  return normalize_launch(img_dev, dtype, nvoxels, mean, sigma, remove_outliers != 0, outliers, scale, out_dev,
                          (cudaStream_t)stream);
}
// resegmentMask's thresholding, radiomics/imageoperations.py:713-724
int rb_resegment_dev(const void* img_dev, int dtype, const uint8_t* mask_dev, long long nvoxels, double lower,
                     double upper, int nthresholds, uint8_t* out_dev, unsigned long long* counts_dev, void* stream) {
  if (!img_dev || !mask_dev || !out_dev || !counts_dev) return fail(RB_ERR_ARG, "resegment: null argument");
  if (int rc = check_dtypes({dtype})) return rc;
  if (nvoxels < 1) return fail(RB_ERR_ARG, "resegment: %lld voxels", nvoxels);
  if (nthresholds != 1 && nthresholds != 2) return fail(RB_ERR_ARG, "resegment: %d thresholds (1 or 2)", nthresholds);
  return resegment_launch(img_dev, dtype, mask_dev, nvoxels, lower, upper, nthresholds == 2, out_dev, counts_dev,
                          (cudaStream_t)stream);
}
int rb_swt_axis_dev(const double* in_dev, int Z, int Y, int X, int axis, const double* dec_lo, const double* dec_hi,
                    int flen, double* out_lo_dev, double* out_hi_dev, void* stream) {
  if (axis < 0 || axis > 2) return fail(RB_ERR_ARG, "axis must be 0..2");
  return swt_axis_launch(in_dev, Z, Y, X, axis, dec_lo, dec_hi, flen, out_lo_dev, out_hi_dev, (cudaStream_t)stream);
}
int rb_bspline_prefilter_dev(double* coeffs_dev, int Z, int Y, int X, void* stream) {
  return bspline_prefilter_launch(coeffs_dev, Z, Y, X, (cudaStream_t)stream, false);
}
int rb_resample_dev(const void* src_dev, int src_dtype, const int* in_size_zyx, void* dst_dev, int dst_dtype, const int* out_size_zyx,
                    const double* start_zyx, const double* step_zyx, int interpolator, double default_value, void* stream) {
  if (!src_dev || !dst_dev || !in_size_zyx || !out_size_zyx || !start_zyx || !step_zyx) return fail(RB_ERR_ARG, "null argument");
  if (int rc = check_dtypes({src_dtype, dst_dtype})) return rc;
  return resample_launch(src_dev, src_dtype, in_size_zyx, dst_dev, dst_dtype, out_size_zyx, start_zyx, step_zyx, interpolator,
                         default_value, (cudaStream_t)stream);
}

int rb_lbp3d_dev(const void* img_dev, int img_dtype, int sample_dtype, const uint8_t* roi_u8_dev, int Z, int Y, int X,
                 const double* vertices_host, int nv, const double* harmonics_host, int levels, double* coeff_scratch_dev,
                 double* out_dev, void* stream) {
  if (int rc = check_dtypes({img_dtype, sample_dtype})) return rc;
  return lbp3d_launch(img_dev, img_dtype, sample_dtype, roi_u8_dev, Z, Y, X, vertices_host, nv, harmonics_host, levels,
                      coeff_scratch_dev, out_dev, (cudaStream_t)stream);
}
int rb_lbp2d_dev(const void* img_dev, int dtype, int Z, int Y, int X, int axis, int P, const double* rp_host,
                 const double* cp_host, int method, double* out_dev, void* stream) {
  if (int rc = check_dtypes({dtype})) return rc;
  return lbp2d_launch(img_dev, dtype, Z, Y, X, axis, P, rp_host, cp_host, method, RB_DT_FLOAT64, out_dev, (cudaStream_t)stream);
}
int rb_lbp2d_cast_dev(const void* img_dev, int image_type, int Z, int Y, int X, int axis, int P, const double* rp_host,
                      const double* cp_host, int method, void* out_dev, void* stream) {
  if (int rc = check_dtypes({image_type})) return rc;
  return lbp2d_launch(img_dev, image_type, Z, Y, X, axis, P, rp_host, cp_host, method, image_type, out_dev, (cudaStream_t)stream);
}

int rb_swt3d_dev(const double* in_dev, int Z, int Y, int X, const double* dec_lo, const double* dec_hi, int flen,
                 double* out_dev, long long band_stride, int z_begin, int z_end, void* stream) {
  return swt3d_launch(in_dev, Z, Y, X, dec_lo, dec_hi, flen, out_dev, band_stride, z_begin, z_end, (cudaStream_t)stream);
}

int rb_recursive_gaussian_axis_dev(const void* in_dev, int in_is_f32, int Z, int Y, int X, int axis, const double* coef20,
                                   float* out_dev, double* scratch_dev, double scale, int accumulate, void* stream) {
  if (axis < 0 || axis > 2) return fail(RB_ERR_ARG, "axis must be 0..2");
  return recursive_gauss_launch(in_dev, in_is_f32, Z, Y, X, axis, coef20, out_dev, scratch_dev, scale, accumulate,
                                (cudaStream_t)stream);
}

int rb_shape_coefficients_dev(const uint8_t* mask_dev, int Z, int Y, int X, const double* spacing_zyx, double* out7,
                              void* stream) {
  if (!mask_dev || !spacing_zyx || !out7 || Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "shape: bad arguments");
  return shape_coefficients_dev(mask_dev, Z, Y, X, (long long)Y * X, X, 1, spacing_zyx, out7, (cudaStream_t)stream);
}
int rb_shape_moments_dev(const uint8_t* mask_dev, int Z, int Y, int X, unsigned long long* out10, void* stream) {
  if (!mask_dev || !out10 || Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "shape: bad arguments");
  return shape_moments_dev(mask_dev, Z, Y, X, out10, (cudaStream_t)stream);
}
int rb_calculate_coefficients(const char* mask, const int* size, const int* strides, const double* spacing,
                              double* surfaceArea, double* volume, double* diameters) {
  if (!mask || !size || !strides || !spacing || !surfaceArea || !volume || !diameters) return fail(RB_ERR_ARG, "shape: null argument");
  const int Z = size[0], Y = size[1], X = size[2];
  if (Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "shape: bad size");
  const size_t n = (size_t)Z * Y * X;
  std::vector<uint8_t> packed(n);
  for (int z = 0; z < Z; z++)
    for (int y = 0; y < Y; y++)
      for (int x = 0; x < X; x++)
        packed[((size_t)z * Y + y) * X + x] = mask[(long long)z * strides[0] + (long long)y * strides[1] + (long long)x * strides[2]] != 0;
  DevBuf d;
  RB_CUDA(d.alloc(n));
  cudaError_t e = cudaMemcpy(d.p, packed.data(), n, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return fail(RB_ERR_CUDA, "shape: %s", cudaGetErrorString(e));
  double out7[7];
  const int rc = shape_coefficients_dev(d.as<uint8_t>(), Z, Y, X, (long long)Y * X, X, 1, spacing, out7, 0);
  if (rc) return rc;
  *surfaceArea = out7[0]; *volume = out7[1];
  for (int q = 0; q < 4; q++) diameters[q] = out7[2 + q];
  return RB_OK;
}

int rb_calculate_coefficients2D(const char* mask, const int* size, const int* strides, const double* spacing, double* perimeter,
                                double* surface, double* diameter) {
  if (!mask || !size || !strides || !spacing || !perimeter || !surface || !diameter) return fail(RB_ERR_ARG, "null argument");
  const int Y = size[0], X = size[1];
  if (Y < 1 || X < 1) return fail(RB_ERR_ARG, "empty mask");
  // gather the (possibly strided) host mask into a contiguous byte image, then one upload
  std::vector<uint8_t> h((size_t)Y * X);
  for (int y = 0; y < Y; y++)
    for (int x = 0; x < X; x++) h[(size_t)y * X + x] = mask[(long long)y * strides[0] + (long long)x * strides[1]] != 0;
  DevBuf d;
  RB_CUDA(d.alloc(h.size()));
  cudaError_t e = cudaMemcpy(d.p, h.data(), h.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return fail(RB_ERR_CUDA, "shape2D upload: %s", cudaGetErrorString(e));
  double out4[4];
  const int rc = shape2d_coefficients_dev(d.as<uint8_t>(), Y, X, X, 1, spacing, out4, 0);
  if (rc) return rc;
  *perimeter = out4[0]; *surface = out4[1]; *diameter = out4[2];
  return RB_OK;
}

int rb_firstorder_num_features(void) { return 18; }
const char* rb_firstorder_feature_name(int idx) { return (idx < 0 || idx >= 18) ? NULL : kFirstOrderNames[idx]; }
int rb_firstorder_voxel_dev(const void* image_dev, int dtype, const uint8_t* mask_dev, const uint8_t* centers_dev,
                            const void* levels_dev, int level_bytes, int Z, int Y, int X, int rz, int ry, int rx,
                            double voxelArrayShift, double voxel_volume, double initValue, double* out_dev,
                            long long out_feature_stride, int z0, int z1, int out_z0, void* stream) {
  if (int rc = check_dtypes({dtype})) return rc;
  if (level_bytes != 1 && level_bytes != 2) return fail(RB_ERR_ARG, "level_bytes must be 1 or 2");
  if (rz < 0 || ry < 0 || rx < 0 || z0 < 0 || z1 > Z || z0 > z1) return fail(RB_ERR_ARG, "bad window / z range");
  const bool wide = force_wide();
  if (!force_generic() && !wide && firstorder_fast_path(level_bytes, rz, ry, rx))
    return firstorder_fast_launch(image_dev, dtype, mask_dev, centers_dev, levels_dev, Z, Y, X, voxelArrayShift,
                                  voxel_volume, initValue, out_dev, out_feature_stride, z0, z1, out_z0, (cudaStream_t)stream);
  const int cap = (2 * rz + 1) * (2 * ry + 1) * (2 * rx + 1);
  switch (window_path(cap, wide)) {
    case WP_GENERIC:
      return firstorder_launch(image_dev, dtype, mask_dev, centers_dev, levels_dev, level_bytes, Z, Y, X, rz, ry, rx,
                               voxelArrayShift, voxel_volume, initValue, out_dev, out_feature_stride, z0, z1, out_z0,
                               (cudaStream_t)stream);
    case WP_WIDE:
      return firstorder_wide_launch(image_dev, dtype, mask_dev, centers_dev, levels_dev, level_bytes, Z, Y, X, rz, ry, rx,
                                    voxelArrayShift, voxel_volume, initValue, out_dev, out_feature_stride, z0, z1, out_z0,
                                    (cudaStream_t)stream);
    default:
      return fail(RB_ERR_UNSUPPORTED, "a kernel window of %d positions is outside the implemented envelope (at most %d: "
                  "kernelRadius <= 7 in 3-D)", cap, WIDE_WCAP_MAX);
  }
}

int rb_firstorder_segment_dev(const void* image_dev, int image_type, const uint8_t* roi_dev, const void* levels_dev,
                              int level_bytes, int Z, int Y, int X, double voxelArrayShift, double voxel_volume,
                              double* out18, void* stream) {
  if (int rc = check_dtypes({image_type})) return rc;
  if (level_bytes != 1 && level_bytes != 2) return fail(RB_ERR_ARG, "level_bytes must be 1 or 2");
  if (!image_dev || !roi_dev || !levels_dev || !out18) return fail(RB_ERR_ARG, "first order: null argument");
  if (Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "first order: the ROI is empty");
  return firstorder_segment(image_dev, image_type, roi_dev, levels_dev, level_bytes, (long long)Z * Y * X, voxelArrayShift,
                            voxel_volume, out18, (cudaStream_t)stream);
}

}  // extern "C"

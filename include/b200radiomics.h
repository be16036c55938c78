/* b200radiomics -- C ABI of the H100-native (sm_90a) texture-matrix engine (libb200radiomics.so).
 *
 * Drop-in boundary for the hot path of AIM-Harvard/pyradiomics (SURVEY.md section 8b): the C
 * functions of reference radiomics/src/cmatrices.h:1-8 and the per-voxel driver loops of
 * reference radiomics/src/_cmatrices.c (set_bb + `for v < Nvox` at :203-207, :355-377, :550-569,
 * :699-717, :848-867), plus fused entry points that go from the quantised volume straight to the
 * per-voxel feature maps (what radiomics/{glcm,glrlm,glszm,gldm,ngtdm}.py compute from the dense
 * matrices in voxel-based mode).  Plain pointers and sizes only; no torch / numpy types.
 *
 * Conventions
 *   - volumes are C-contiguous (z,y,x); 2-D images are passed with nd == 2 (y,x).
 *   - `*_host` entry points take HOST pointers and do their own transfers; `*_dev` entry points
 *     take DEVICE pointers plus a `cudaStream_t` passed as `void *stream` (NULL = default stream)
 *     and are asynchronous with respect to the host unless stated otherwise.
 *   - every function returns RB_OK (0) or a negative rb_status; rb_last_error() gives the text.
 *   - gray levels inside the mask must lie in 1..Ng; anything else gives RB_ERR_LEVEL_RANGE, the
 *     analogue of the reference's IndexError("Calculation of <M> Failed.")
 *     (radiomics/src/_cmatrices.c:219,372,566,714,864).
 *   - there is no CPU fallback: without a usable CUDA device every compute entry point fails with
 *     RB_ERR_CUDA.
 */
#ifndef B200RADIOMICS_H
#define B200RADIOMICS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  RB_OK = 0,
  RB_ERR_CUDA = -1,         /* CUDA runtime error / no device                       */
  RB_ERR_LEVEL_RANGE = -2,  /* gray level <= 0 or > Ng inside the mask (IndexError)   */
  RB_ERR_ARG = -3,          /* bad argument (reference: ValueError / RuntimeError)    */
  RB_ERR_NOMEM = -4,        /* allocation failure (reference: MemoryError)            */
  RB_ERR_UNSUPPORTED = -5   /* outside the implemented envelope (see DESIGN.md)        */
} rb_status;

typedef enum { RB_GLCM = 0, RB_GLRLM = 1, RB_GLSZM = 2, RB_GLDM = 3, RB_NGTDM = 4 } rb_class;

/* weightingNorm of reference radiomics/glcm.py:105-108, glrlm.py:80-82 */
typedef enum { RB_W_NONE = 0, RB_W_INFINITY = 1, RB_W_EUCLIDEAN = 2, RB_W_MANHATTAN = 3, RB_W_NO_WEIGHTING = 4 } rb_weighting;

/* Hot-path settings (the kwargs of the reference feature classes, SURVEY.md section 5). */
typedef struct {
  int kernelRadius;        /* voxel-based kernel radius, >= 1                         */
  int force2D;             /* 0/1                                                     */
  int force2Ddimension;    /* 0 = z, 1 = y, 2 = x                                     */
  int ndist;               /* number of entries used in distances[] (GLCM/GLDM/NGTDM) */
  int distances[8];
  int symmetricalGLCM;     /* 0/1                                                     */
  int weighting;           /* rb_weighting (GLCM, GLRLM)                              */
  double spacing_zyx[3];   /* voxel spacing, only used for weighting                  */
  int gldm_a;              /* GLDM alpha                                              */
  double initValue;        /* value of non-computed voxels in the feature maps        */
  int Ng;                  /* max gray level in the ROI (coefficients["Ng"])          */
  int n_roi_levels;        /* number of distinct gray levels in the ROI               */
} rb_voxel_settings;

/* ---- bookkeeping -------------------------------------------------------------------------- */
const char *rb_last_error(void);
const char *rb_version(void);
int rb_device_count(void);          /* >= 0, or RB_ERR_CUDA                                   */
int rb_num_features(int cls);       /* 24 / 16 / 16 / 14 / 5                                  */
/* The fused GLCM path keeps one eigen-task queue per (device, stream) it ran on (grown on demand, up to 1.15 GB), and the
 * kernels for windows of 344+ positions one workspace per (device, stream), so that repeated calls do not reallocate;
 * this frees those of the current device.  It waits for the calls that are enqueueing on them, synchronises the device,
 * then frees; a later call allocates again.
 * Threading contract of the library:
 *   - every `*_dev` voxel entry point (rb_pack_levels_dev, rb_glcm_alive_angles_dev, rb_voxel_features_dev,
 *     rb_firstorder_voxel_dev, rb_memcpy2d_async, rb_maps_to_f32_dev) issues its launches, memsets and copies on the
 *     given stream only;
 *   - concurrent calls are safe from any number of host threads, on the same stream or on different ones: a call holds
 *     its stream's queue or workspace from taking it until its last launch on it is enqueued, so calls on one stream
 *     enqueue one after the other and run in that order;
 *   - rb_release_device_caches may be called at any time, from any thread. */
int rb_release_device_caches(void);
/* name of feature `idx` of class `cls` (the reference's get<Name>FeatureValue names, in the
 * alphabetical order in which the reference enumerates them, radiomics/base.py:163-179). */
const char *rb_feature_name(int cls, int idx);

/* ---- neighbour offsets: replaces get_angle_count + build_angles (cmatrices.c:756-892) and
 *      cmatrices_generate_angles (_cmatrices.c:882-924).  `angles` receives Na x nd ints; returns
 *      Na (> 0), RB_ERR_ARG for an invalid distance / no angle, or the required count negated
 *      minus 1000 if max_angles is too small. */
int rb_generate_angles(const int *size, int nd, const int *distances, int ndist, int bidirectional,
                       int force2D, int force2Ddimension, int *angles, int max_angles);

/* ---- quantised volume on the device --------------------------------------------------------
 * Fold image (int32 gray levels) and mask into the engine's compact level volume: level where
 * mask != 0, 0 elsewhere; 1 byte per voxel when Ng <= 255, else 2.  Also validates 1..Ng and
 * histograms the levels (presence[g-1] += 1, presence has Ng uint32 entries, may be NULL).
 * status_dev (device int, zero-initialised by the caller, may be NULL) gets bit 0 set on a range
 * violation.  Replaces the int32/bool coercion of try_parse_arrays (_cmatrices.c:1023-1085). */
int rb_level_bytes(int Ng);  /* 1 or 2 */
int rb_pack_levels_dev(const int32_t *image_dev, const uint8_t *mask_dev, long long nvoxels, int Ng,
                       void *levels_dev, uint32_t *presence_dev, int *status_dev, void *stream);

/* ---- fused voxel-based feature maps (the headline path) ------------------------------------
 * For every voxel (z,y,x) with z0 <= z < z1 of a (Z,Y,X) level volume: if it is a centre voxel
 * (centers_dev[i] != 0, or levels != 0 when centers_dev is NULL) compute all features of class
 * `cls` over its (2r+1)^3 kernel window and store them; otherwise store settings->initValue.
 * Feature f of voxel (z,y,x) goes to
 *     out[f * out_feature_stride + ((z - out_z0) * Y + y) * X + x]
 * as float64 (out_is_f32 == 0, the reference's map dtype, base.py:205-209) or float32 (out_is_f32 != 0; every path:
 * fast, generic, wide, weighted / asymmetric GLCM, force2D, 16-bit levels).  out_feature_stride and
 * out_z0 count elements of that type.  Features are computed in float64 either way and a float32 map holds each value
 * rounded to nearest once (NaN stays NaN), so it equals the float64 map converted to float32 bit for bit.
 * Angles that are empty for every voxel of the ROI are "deleted" like in the reference
 * (glcm.py:187-196); rb_glcm_alive_angles_dev computes that set (32-bit words, bit a = angle a,
 * RB_ALIVE_WORDS words, zero-initialised by the caller) and alive_dev may be NULL to keep all.
 * Windows of up to 343 positions run one thread per centre, 344 to 3375 (kernelRadius 4 to 7 in 3-D) one block per
 * centre with the same results; a larger window returns RB_ERR_UNSUPPORTED.
 * status_dev: bit 0 = MCC eigen-problem larger than the in-kernel solver (value set to NaN),
 *             bit 1 = weighted GLCM entry overflow (or, on a window of 344+ positions, more levels than Ng allows). */
#define RB_ALIVE_WORDS 6
int rb_glcm_alive_angles_dev(const void *levels_dev, int level_bytes, const uint8_t *centers_dev,
                             int Z, int Y, int X, const rb_voxel_settings *settings,
                             uint32_t *alive_dev, void *stream);
int rb_voxel_features_dev(int cls, const void *levels_dev, int level_bytes, const uint8_t *centers_dev,
                          int Z, int Y, int X, int z0, int z1, const rb_voxel_settings *settings,
                          const uint32_t *alive_host, void *out_dev, int out_is_f32,
                          long long out_feature_stride, int out_z0, int *status_dev, void *stream);

/* Output assembly (reference radiomics/base.py:205-209,232-234: the maps a voxel-based class returns are
 * full-size float64 host arrays).  The fused kernels leave [F][Z][Y][X] maps on the device; these two helpers move a
 * z-chunk of SEVERAL maps with one strided DMA instead of one copy per map:
 * rb_memcpy2d_async: `height` rows of `width` bytes, row pitches in bytes; kind 1 = host->device, 2 = device->host,
 *   3 = device->device (cudaMemcpy2DAsync on `stream`; host memory should be page-locked for a true async copy).
 * rb_maps_to_f32_dev: rows of `width` float64 elements -> float32 (element pitches), the opt-in compact map type
 *   (half the PCIe bytes; the tolerance of the path is 1e-5 relative, float32 carries 6e-8) for maps computed in
 *   float64, such as first order's; the texture classes write float32 maps directly (out_is_f32). */
int rb_memcpy2d_async(void *dst, unsigned long long dpitch, const void *src, unsigned long long spitch,
                      unsigned long long width, unsigned long long height, int kind, void *stream);
int rb_maps_to_f32_dev(const double *src_dev, long long src_pitch, float *dst_dev, long long dst_pitch,
                       long long width, long long height, void *stream);

/* Host-buffer convenience (what a ctypes/cgo caller with NumPy-like arrays uses; e2e path):
 * image int32 + mask bytes (nonzero = ROI; levels must already be discretised, 1..Ng) in, float64
 * maps out: maps[f][z][y][x], f < rb_num_features(cls).  Synchronous. */
int rb_voxel_features_host(int cls, const int32_t *image, const uint8_t *mask, int Z, int Y, int X,
                           const rb_voxel_settings *settings, double *maps);

/* ---- texture matrices: drop-ins for reference radiomics/src/cmatrices.h:1-8 plus the binding's
 *      per-voxel driver (_cmatrices.c: calculate_glcm :84-233, glszm :235-430, glrlm :432-581,
 *      ngtdm :583-730, gldm :732-880).  HOST pointers; synchronous.
 *      image: int32 gray levels, mask: bytes (nonzero = ROI), size[nd] with nd = 2 or 3.
 *      voxels == NULL  -> segment-based: one matrix over the whole array (nvox ignored).
 *      voxels != NULL  -> int32 [nd][nvox] centre coordinates + kernelRadius > 0: one dense matrix
 *                         per listed voxel over its clipped (2r+1)^nd box (force2D collapses one
 *                         dimension), exactly the layout the reference returns:
 *        glcm  [nvox][Ng][Ng][Na]        Na = unidirectional angles of `distances`
 *        glrlm [nvox][Ng][Nr][Na]        Na = unidirectional distance-1 angles
 *        gldm  [nvox][Ng][2*Na+1]        Na = BIdirectional angles of `distances` (_cmatrices.c:790)
 *        ngtdm [nvox][Ng][3]             columns n_i, s_i, i
 *      Use rb_generate_angles first to learn Na; `angles` (may be NULL) receives Na x nd ints.
 *      A GLRLM run longer than Nr, in either mode, gives RB_ERR_LEVEL_RANGE. */
int rb_calculate_glcm(const int32_t *image, const uint8_t *mask, const int *size, int nd,
                      const int *distances, int ndist, int Ng, int force2D, int force2Ddimension,
                      int kernelRadius, const int *voxels, int nvox, double *glcm, int *angles);
int rb_calculate_glrlm(const int32_t *image, const uint8_t *mask, const int *size, int nd, int Ng, int Nr,
                       int force2D, int force2Ddimension, int kernelRadius, const int *voxels, int nvox,
                       double *glrlm, int *angles);
int rb_calculate_gldm(const int32_t *image, const uint8_t *mask, const int *size, int nd,
                      const int *distances, int ndist, int Ng, int alpha, int force2D, int force2Ddimension,
                      int kernelRadius, const int *voxels, int nvox, double *gldm);
int rb_calculate_ngtdm(const int32_t *image, const uint8_t *mask, const int *size, int nd,
                       const int *distances, int ndist, int Ng, int force2D, int force2Ddimension,
                       int kernelRadius, const int *voxels, int nvox, double *ngtdm);
/* GLSZM is two-phase like the reference (calculate_glszm finds the zones and the largest zone,
 * fill_glszm histograms them into [nvox][Ng][max_region]): rb_calculate_glszm returns an opaque
 * handle and *max_region (0 when there is no zone; allocate with max(1, max_region));
 * rb_fill_glszm writes the matrix and frees the handle; rb_glszm_release frees it unused. */
int rb_calculate_glszm(const int32_t *image, const uint8_t *mask, const int *size, int nd, int Ng,
                       int force2D, int force2Ddimension, int kernelRadius, const int *voxels, int nvox,
                       int *max_region, void **handle);
int rb_fill_glszm(void *handle, int Ng, int max_region, double *glszm);
void rb_glszm_release(void *handle);

/* Segment-based matrices straight from a DEVICE-resident packed level volume (rb_pack_levels_dev) -- what the plugin
 * classes call once the image has been discretised on the GPU, instead of shipping it back to the host for the entry
 * points above.  Same matrices / layouts / angle order; results in HOST float64 buffers.  Every launch and copy runs on
 * `stream`, so the levels may still be in flight on it; each call returns once `stream` has reached its results.
 * rb_segment_texture_dev builds GLCM, GLDM and NGTDM in ONE pass over the volume (NULL = not wanted): a CTA stages a box
 *   of the level volume in shared memory -- through TMA (cp.async.bulk.tensor.3d with hardware zero-fill outside the
 *   volume) when the row pitch is a multiple of 16 bytes, else by cooperative loads -- and accumulates the three
 *   matrices in shared-memory histograms (reference radiomics/src/cmatrices.c:4-92, 660-754, 543-658).  `distances`
 *   drives all three (the GLCM uses the unidirectional half of the offsets).
 * rb_segment_glrlm_dev: every run END walks back to the start of its run (cmatrices.c:299-541).
 * rb_segment_glszm_dev: phase one of GLSZM as rb_calculate_glszm (finish with rb_fill_glszm / rb_glszm_release); the
 *   handle keeps `stream`, and rb_fill_glszm runs on it too. */
int rb_segment_texture_dev(const void *levels_dev, int level_bytes, const int *size, int nd, const int *distances,
                           int ndist, int Ng, int alpha, int force2D, int force2Ddimension, double *glcm, double *gldm,
                           double *ngtdm, int *angles, void *stream);
int rb_segment_glrlm_dev(const void *levels_dev, int level_bytes, const int *size, int nd, int Ng, int Nr, int force2D,
                         int force2Ddimension, double *glrlm, int *angles, void *stream);
int rb_segment_glszm_dev(const void *levels_dev, int level_bytes, const int *size, int nd, int Ng, int force2D,
                         int force2Ddimension, int *max_region, void **handle, void *stream);

/* ---- gray-level discretisation and pre-filters (device pointers, asynchronous) --------------
 * Pixel types: every `dtype` argument is an rb_dtype code; any other value gives RB_ERR_ARG. */
typedef enum {
  RB_DT_INT16 = 0, RB_DT_INT32 = 1, RB_DT_FLOAT32 = 2, RB_DT_FLOAT64 = 3, RB_DT_UINT8 = 4, RB_DT_UINT16 = 5, RB_DT_INT64 = 6
} rb_dtype;
/* rb_minmax_dev: ROI minimum / maximum (mask_dev may be NULL = all voxels) as order-preserving
 *   int64 keys in keys_dev[0..1], the voxel count in keys_dev[2] and the count of NaN voxels in
 *   keys_dev[3] (NaN voxels are counted in [2] but take no part in the minimum / maximum);
 *   initialise keys_dev to {INT64_MAX, INT64_MIN, 0, 0}; decode a key k with
 *   bits = k >= 0 ? k : k ^ INT64_MAX.
 *   Replaces the Python-level min()/max() of getBinEdges (radiomics/imageoperations.py:128-129).
 * rb_digitize_dev: out[i] = number of edges <= image[i] inside the mask, 0 outside: np.digitize
 *   on the masked voxels as binImage does (radiomics/imageoperations.py:156-174); comparisons are
 *   made in float64 against the caller's edges, so bins are bit-identical to NumPy's. */
int rb_minmax_dev(const void *image_dev, int dtype, const uint8_t *mask_dev, long long nvoxels,
                  long long *keys_dev, void *stream);
int rb_digitize_dev(const void *image_dev, int dtype, const uint8_t *mask_dev, long long nvoxels,
                    const double *edges_dev, int nedges, int32_t *out_dev, void *stream);
/* One axis (0 = z, 1 = y, 2 = x) of the level-1 stationary wavelet transform with periodic
 * extension (pywt.swtn(level=1) as called at radiomics/imageoperations.py:935): float64 in, the
 * low-pass and high-pass outputs in out_lo_dev / out_hi_dev.  dec_lo / dec_hi are HOST arrays of
 * `flen` decomposition taps.  Odd lengths behave like the reference's wrap-pad-then-crop. */
int rb_swt_axis_dev(const double *in_dev, int Z, int Y, int X, int axis, const double *dec_lo,
                    const double *dec_hi, int flen, double *out_lo_dev, double *out_hi_dev, void *stream);
/* All three axes at once for a 3-D volume: the 8 sub-bands of one level in a single pass (input staged through shared
 * memory plane by plane, a ring of xy-filtered planes feeds the z filter).  Periodic extension in all axes -- wrap-pad odd
 * sizes first, as the reference does (radiomics/imageoperations.py:914-919).  Sub-band b = bx + 2*by + 4*bz (bit set =
 * high-pass 'd' along that axis; pywt's key is the letters in x,y,z order because the reference passes axes=(2,1,0),
 * imageoperations.py:871,935) is written to out_dev[b * band_stride + voxel].  flen in {2, 4, 6, 8}.
 * Only planes [z_begin, z_end) are produced (out plane 0 = input plane z_begin): a multi-GPU caller passes its z-slab
 * with (flen-1-flen/2) halo planes below and flen/2 above, exchanged ring-closed between the ranks, and asks for the
 * interior -- the z wrap-around is then never taken; 0, Z = the whole (periodic) volume. */
int rb_swt3d_dev(const double *in_dev, int Z, int Y, int X, const double *dec_lo, const double *dec_hi, int flen,
                 double *out_dev, long long band_stride, int z_begin, int z_end, void *stream);
/* One axis of a 4th-order recursive (IIR) Gaussian / Gaussian-derivative filter, causal +
 * anti-causal, the building block of ITK's LaplacianRecursiveGaussianImageFilter used at
 * radiomics/imageoperations.py:824-830.  coef20 (HOST) = N0..N3, D1..D4, M1..M4, BN1..4, BM1..4;
 * input float32 (in_is_f32) or float64, output float32 = (causal + anticausal) * scale, added to
 * out_dev when accumulate != 0.  scratch_dev: float64 buffer with as many elements as the volume. */
int rb_recursive_gaussian_axis_dev(const void *in_dev, int in_is_f32, int Z, int Y, int X, int axis,
                                   const double *coef20, float *out_dev, double *scratch_dev, double scale,
                                   int accumulate, void *stream);

/* ---- resampling onto the extraction grid (SURVEY.md section 8f rank 4; reference radiomics/imageoperations.py:448-612:
 *      sitk.ResampleImageFilter, sitkBSpline for the image, sitkNearestNeighbor for the mask, axis-aligned grids).
 * rb_bspline_prefilter_dev: in-place cubic B-spline coefficients of a float64 volume (ITK BSplineDecompositionImageFilter:
 *   pole sqrt(3)-2, mirror boundaries, x then y then z).
 * rb_resample_dev: dst[o] = interpolate(src, start + o * step) for every output voxel o (z,y,x); `interpolator` 0 = nearest
 *   neighbour, 1 = linear, 3 = cubic B-spline (src = the float64 coefficients); `default_value` outside the input buffer
 *   (continuous index outside [-0.5, size-0.5)); the result is clamped to the range of dst_dtype and TRUNCATED like ITK's
 *   cast.  dtype codes as rb_minmax_dev. */
int rb_bspline_prefilter_dev(double *coeffs_dev, int Z, int Y, int X, void *stream);
int rb_resample_dev(const void *src_dev, int src_dtype, const int *in_size_zyx, void *dst_dev, int dst_dtype,
                    const int *out_size_zyx, const double *start_zyx, const double *step_zyx, int interpolator,
                    double default_value, void *stream);

/* ---- 3-D local binary pattern image type (reference radiomics/imageoperations.py:1169-1314, getLBP3DImage).
 * For every voxel with roi_u8_dev != 0: the cubic B-spline samples of the image at the Nv sphere vertices
 *   (scipy.ndimage.map_coordinates(order=3): SciPy's exact mirror prefilter, 0 where a coordinate leaves [0, n-1]), cast
 *   to `sample_dtype`; their Fisher kurtosis; the sign bits sample >= centre; the spherical-harmonic level maps
 *   Re(sqrt(sum_v (sum_m c_nm Y_nm(v))^2)) with c_nm = sum_v bit_v Y_nm(v), n < levels.
 * img_dtype: dtype code (as rb_minmax_dev) of the data at img_dev; sample_dtype: the dtype the samples are cast to, the
 *   image's original one (a uint16 image stored as int32 passes 1 and 5).
 * vertices_host: [nv][3] (z, y, x) offsets in voxels; harmonics_host: [nv][levels (levels + 1) / 2][re, im], entry
 *   n (n + 1) / 2 + m = Y_n^m(vertex) for 0 <= m <= n (negative m follow from Y_n^-m = (-1)^m conj(Y_n^m)).
 * coeff_scratch_dev: Z*Y*X float64; out_dev: float64 [levels + 1][Z][Y][X], the level maps then the kurtosis, 0 outside
 *   the ROI.  nv <= 162 and levels <= 4, else RB_ERR_UNSUPPORTED. */
int rb_lbp3d_dev(const void *img_dev, int img_dtype, int sample_dtype, const uint8_t *roi_u8_dev, int Z, int Y, int X,
                 const double *vertices_host, int nv, const double *harmonics_host, int levels,
                 double *coeff_scratch_dev, double *out_dev, void *stream);

/* ---- 2-D local binary pattern image type (reference radiomics/imageoperations.py:1094-1166, getLBP2DImage ->
 *      skimage.feature.local_binary_pattern), every slice of a (Z, Y, X) volume in one call.
 * The slices are cut along `axis` as the reference's swapaxes(0, axis) does: axis 0 -> rows y, cols x; axis 1 -> rows z,
 *   cols x; axis 2 -> rows y, cols z.  A 2-D image is passed as Z = 1, axis 0.
 * For pixel (r, c) of a slice and k = 0..P-1 (rp_host / cp_host: P HOST doubles, round(-R sin(2 pi k / P), 5) and
 *   round(R cos(2 pi k / P), 5)):
 *   t_k = bilinear sample at (r + rp[k], c + cp[k]): minr = floor, maxr = ceil, dr = r - minr (columns alike),
 *         top = (1 - dc) tl + dc tr, bottom = (1 - dc) bl + dc br, t_k = (1 - dr) top + dr bottom, every operation rounded
 *         on its own (no FMA); a corner outside the slice reads 0;
 *   s_k = (t_k - centre >= 0);
 *   RB_LBP2D_DEFAULT      sum_k s_k 2^k
 *   RB_LBP2D_ROR          the minimum over the P right rotations (v >> 1) | ((v & 1) << (P - 1)) of DEFAULT
 *   RB_LBP2D_UNIFORM      changes = #{k < P - 1: s_k != s_k+1} (not circular); sum_k s_k if changes <= 2, else P + 1
 *   RB_LBP2D_NRI_UNIFORM  changes > 2: P (P - 1) + 2; no ones: 0; all ones: P (P - 1) + 1; else 1 + (n_ones - 1) P + rot,
 *                         rot = n_ones - first_zero if s_0 = 1, else P - first_one
 *   RB_LBP2D_VAR          sum += t, sq += t t over k, v = (sq - sum sum / P) / P; v if v != 0, else NaN
 * out_dev: float64 (Z, Y, X), the input's layout.  img dtype codes as rb_minmax_dev.  1 <= P <= 31 (the library's int32
 *   weights overflow beyond), else RB_ERR_UNSUPPORTED; an unknown method or axis is RB_ERR_ARG. */
enum { RB_LBP2D_DEFAULT = 0, RB_LBP2D_ROR = 1, RB_LBP2D_UNIFORM = 2, RB_LBP2D_NRI_UNIFORM = 3, RB_LBP2D_VAR = 4 };
int rb_lbp2d_dev(const void *img_dev, int dtype, int Z, int Y, int X, int axis, int P, const double *rp_host,
                 const double *cp_host, int method, double *out_dev, void *stream);
/* rb_lbp2d_cast_dev: the same codes stored in the image's own pixel type, as the reference's per-slice assignment
 *   im_arr[idx, ...] = local_binary_pattern(...) stores them (NumPy's unsafe float64 -> image_type cast): out_dev has the
 *   input's rb_dtype (`image_type`) and layout, and no float64 volume is made.  The cast (csrc/lbp2d.cuh, numpy_cast):
 *   float64 unchanged; float32 rounded to nearest (+-inf beyond its range); int32 trunc(v) if it fits, else INT32_MIN (NaN
 *   and +-inf too); int16 / uint16 / uint8 the low bits of that int32; int64 trunc(v) if it fits, else INT64_MIN.
 *   Argument checks as rb_lbp2d_dev. */
int rb_lbp2d_cast_dev(const void *img_dev, int image_type, int Z, int Y, int X, int axis, int P, const double *rp_host,
                      const double *cp_host, int method, void *out_dev, void *stream);

/* ---- per-voxel image types (reference radiomics/imageoperations.py:973-1073, getSquareImage, getSquareRootImage,
 *      getLogarithmImage, getExponentialImage).  out_dev[i] = f(x), x = img_dev[i] as float64, for i < nvoxels:
 *   RB_PW_SQUARE       (c x)^2                                   c = 1 / sqrt(M)                  (:989-991)
 *   RB_PW_SQUAREROOT   x > 0: sqrt(x c), x < 0: -sqrt(-x c), else x   c = M                        (:1014-1017)
 *   RB_PW_LOGARITHM    (x > 0: log(x + 1), x < 0: -log(-(x - 1)), else x) * c
 *                                                                c = M / log(M + 1)               (:1041-1045)
 *   RB_PW_EXPONENTIAL  exp(c x)                                  c = log(M) / M                   (:1067-1069)
 * with M = max|x| over the whole image (rb_minmax_dev with mask_dev = NULL: max(-min, max)).  The caller computes `c`
 * (the reference's NumPy scalar arithmetic); the products and sqrt are correctly rounded, log / exp are CUDA's (<= 1 ulp).
 * dtype codes as rb_minmax_dev. */
enum { RB_PW_SQUARE = 0, RB_PW_SQUAREROOT = 1, RB_PW_LOGARITHM = 2, RB_PW_EXPONENTIAL = 3 };
int rb_pointwise_image_dev(const void *img_dev, int dtype, long long nvoxels, int kind, double c, double *out_dev,
                           void *stream);
/* Gradient magnitude image type (reference radiomics/imageoperations.py:1076-1091, getGradientImage ->
 * sitk.GradientMagnitudeImageFilter): per axis i in x, y, z order g_i = (-0.5 w_i f[-1] + 0 f[0]) + 0.5 w_i f[+1],
 * neighbours outside the volume clamped to the edge (zero-flux Neumann), out = sqrt(((0 + gx^2) + gy^2) + gz^2), float64,
 * every step rounded separately (no FMA).  weights_zyx (HOST, 3 doubles) = 1 / spacing (UseImageSpacing) or ones.  A 2-D
 * image is passed as Z = 1. */
int rb_gradient_magnitude_dev(const void *img_dev, int dtype, int Z, int Y, int X, const double *weights_zyx,
                              double *out_dev, void *stream);

/* ---- normalisation and resegmentation (reference radiomics/imageoperations.py:615-742, normalizeImage and
 *      resegmentMask).  dtype codes as rb_minmax_dev.
 * rb_roi_moments_dev: over the voxels with mask_dev[i] != 0 (mask_dev NULL = every voxel), in float64:
 *   out_dev[0] count, [1] NaN count, [2] sum, [3] maximum (NaN if any voxel is NaN, as np.max), and with passes == 2
 *   [4] sum of (x - mean)^2, mean = [2] / [0] (passes == 1 leaves [4] NaN).  Replaces sitk.Normalize's statistics
 *   (:638, over the whole image) and the np.max / np.mean / np.std of the ROI (:699, :704-705).  The partial sums go
 *   to scratch_dev (RB_MOMENTS_SCRATCH_BYTES) from a grid that depends on nvoxels only, and one block adds them in a
 *   fixed order: the result is bit-identical from run to run and card to card.
 * rb_normalize_dev: out_dev[i] = ((x - mean) * (1 / sigma)), clamped to [-outliers, outliers] when remove_outliers
 *   (NaN stays NaN), then * scale, float64, every step rounded separately (:638-652: ITK's ShiftScale form).
 * rb_resegment_dev: out_dev[i] = 1 if mask_dev[i] != 0 and lower <= x (and x <= upper when nthresholds == 2), else 0
 *   (:713-722).  lower / upper must already be rounded to the dtype NumPy compares in (float32 for a float32 image).
 *   counts_dev[0] = ROI voxels, counts_dev[1] = kept voxels. */
enum { RB_MOMENTS_SCRATCH_BYTES = 40960 };
int rb_roi_moments_dev(const void *img_dev, int dtype, const uint8_t *mask_dev, long long nvoxels, int passes,
                       void *scratch_dev, double *out_dev, void *stream);
int rb_normalize_dev(const void *img_dev, int dtype, long long nvoxels, double mean, double sigma, int remove_outliers,
                     double outliers, double scale, double *out_dev, void *stream);
int rb_resegment_dev(const void *img_dev, int dtype, const uint8_t *mask_dev, long long nvoxels, double lower,
                     double upper, int nthresholds, uint8_t *out_dev, unsigned long long *counts_dev, void *stream);

/* ---- segment-mode shape coefficients (SURVEY.md section 8f rank 4) ------------------------------
 * rb_calculate_coefficients replaces calculate_coefficients (radiomics/src/cshape.h:1-2, binding
 *   radiomics/src/_cshape.c:75-113): HOST mask (non-zero = ROI) of `size` = {Z, Y, X} with element
 *   `strides`, `spacing` = {z, y, x}; marching-cubes surface area and volume of the ROI mesh and the
 *   four maximum diameters (equal-z "Slice", equal-y "Column", equal-x "Row", 3-D) over its vertices.
 *   The diameters are bit-identical to the reference's; area / volume differ by summation order only.
 * rb_shape_coefficients_dev: the same for a contiguous uint8 mask already on the device; out7 (HOST) =
 *   {area, volume, d_slice, d_column, d_row, d_3D, number of mesh vertices}.  Synchronises `stream`.
 * rb_shape_moments_dev: exact integer moments {N, z, y, x, zz, zy, zx, yy, yx, xx} of the ROI voxel
 *   indices (the covariance of shape.py:86-95 is formed from them on the host). */
int rb_calculate_coefficients(const char *mask, const int *size, const int *strides, const double *spacing,
                              double *surfaceArea, double *volume, double *diameters);
int rb_shape_coefficients_dev(const uint8_t *mask_dev, int Z, int Y, int X, const double *spacing_zyx,
                              double *out7, void *stream);
int rb_shape_moments_dev(const uint8_t *mask_dev, int Z, int Y, int X, unsigned long long *out10, void *stream);
/* rb_calculate_coefficients2D replaces calculate_coefficients2D (radiomics/src/cshape.h, cshape.c:420-595, binding
 *   radiomics/src/_cshape.c:33-39 used by radiomics/shape2D.py:99): HOST mask of `size` = {Y, X} with element `strides`,
 *   `spacing` = {y, x}: marching-squares perimeter and surface of the ROI outline and the maximum diameter over its
 *   vertices (bit-identical to the reference's; perimeter / surface differ by summation order only). */
int rb_calculate_coefficients2D(const char *mask, const int *size, const int *strides, const double *spacing,
                                double *perimeter, double *surface, double *diameter);

/* ---- voxel-based first-order feature maps (SURVEY.md section 8f: the next plugin after the five
 *      texture classes; reference radiomics/firstorder.py:40-474).  For every centre voxel of planes
 *      [z0,z1): the 18 first-order features over its kernel window (radii rz,ry,rx per dimension: the
 *      reference limits each to ROI-bbox size - 1 and to 0 in the force2D dimension), written like
 *      rb_voxel_features_dev.  image_dev: raw intensities (dtype codes as rb_minmax_dev);
 *      mask_dev: voxels that belong to kernels (NULL = all); centers_dev: voxels to compute (NULL =
 *      mask); levels_dev: discretised levels (rb_pack_levels_dev) for Entropy / Uniformity.
 *      Feature order = rb_firstorder_feature_name(0..17). */
int rb_firstorder_num_features(void);
const char *rb_firstorder_feature_name(int idx);
int rb_firstorder_voxel_dev(const void *image_dev, int dtype, const uint8_t *mask_dev, const uint8_t *centers_dev,
                            const void *levels_dev, int level_bytes, int Z, int Y, int X, int rz, int ry, int rx,
                            double voxelArrayShift, double voxel_volume, double initValue, double *out_dev,
                            long long out_feature_stride, int z0, int z1, int out_z0, void *stream);

/* ---- segment-based first order: replaces the targetVoxelArray path of RadiomicsFirstOrder (reference
 *      radiomics/firstorder.py:40-60 and the get*FeatureValue methods :62-474), which sorts, takes percentiles and
 *      moments of the ROI vector and histograms its discretised levels on the host.
 *   image_dev: raw or derived intensities (image_type an rb_dtype code; read as float64, like NumPy's astype(np.float64));
 *   roi_dev: uint8 ROI mask (non-zero = in the ROI); levels_dev: the packed levels of rb_pack_levels_dev (level_bytes 1
 *   or 2) for Entropy / Uniformity; all contiguous [Z][Y][X] (a 2-D image is Z = 1).  out18 (HOST) = the 18 features in
 *   rb_firstorder_feature_name order.  Every launch runs on `stream`; the host is synchronised once, at the end.
 *   The order statistics (Minimum, Maximum, Range, 10/90Percentile, InterquartileRange, Median) are exact: a radix select
 *   on the float64 keys, interpolated like NumPy 2.x np.percentile (method "linear") and np.median, with -0.0 taken as
 *   +0.0.  The sums are deterministic (block partials in a fixed order, no floating-point atomics), so repeated calls
 *   give the same bits; they differ from NumPy's pairwise sums by summation order only.
 *   Z, Y or X < 1 returns RB_ERR_ARG before any launch.  Whether the ROI holds a voxel is only known on the device: a
 *   ROI without voxels runs the launches (each returns at once) and returns RB_ERR_ARG after the synchronisation;
 *   voxel.firstorder_segment checks the ROI first and raises ValueError before any launch.
 *   Intensities must be finite: voxel.discretize rejects a ROI with NaN or +-inf before this is called. */
int rb_firstorder_segment_dev(const void *image_dev, int image_type, const uint8_t *roi_dev, const void *levels_dev,
                              int level_bytes, int Z, int Y, int X, double voxelArrayShift, double voxel_volume,
                              double *out18, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RADIOMICS_H */

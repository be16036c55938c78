// Pre-filter and discretisation kernels feeding the texture path (SURVEY.md section 8a: a14-a16):
//   * gray-level discretisation: ROI min/max reduction + np.digitize-exact binning
//     (reference radiomics/imageoperations.py:67-174)
//   * level-1 stationary wavelet transform, periodic, one axis per pass, low+high band per pass
//     (reference radiomics/imageoperations.py:899-970 -> pywt.swtn(level=1), PyWavelets >= 1.6)
//   * Laplacian of Gaussian by recursive (IIR) Gaussian filtering, one line per thread
//     (reference radiomics/imageoperations.py:756-836 -> ITK LaplacianRecursiveGaussianImageFilter)
//   * the square / squareroot / logarithm / exponential image types, one pass per voxel, and the gradient
//     magnitude (reference radiomics/imageoperations.py:973-1091 -> ITK GradientMagnitudeImageFilter)
//   * normalisation and resegmentation: a deterministic two-pass float64 ROI reduction, the normalisation pass and
//     the threshold pass (reference radiomics/imageoperations.py:615-742)
// All are HBM-streaming kernels: every thread handles consecutive x so loads/stores coalesce; the
// wavelet pass reads its 6 taps through L1 (neighbouring threads share them).
#include "common.cuh"
#include "pixel.cuh"

namespace rb {

// order-preserving map double <-> signed 64-bit, so atomicMin/atomicMax work on doubles
__device__ __forceinline__ long long f64_key(double v) {
  long long b = __double_as_longlong(v);
  return b >= 0 ? b : b ^ 0x7FFFFFFFFFFFFFFFll;
}

__global__ void __launch_bounds__(256)
minmax_kernel(const void* __restrict__ img, int dt, const uint8_t* __restrict__ mask, long long n,
              long long* __restrict__ keys /* [0]=min key, [1]=max key, [2]=count, [3]=NaN count */) {
  double lo = 1.0 / 0.0, hi = -1.0 / 0.0;
  long long cnt = 0, nans = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (mask && !mask[i]) continue;
    const double v = load_f64(img, dt, i);
    lo = v < lo ? v : lo; hi = v > hi ? v : hi; cnt++;      // NaN compares false: counted, not in min / max
    nans += v != v;
  }
  for (int o = 16; o; o >>= 1) {
    const double l2 = __shfl_xor_sync(0xffffffffu, lo, o), h2 = __shfl_xor_sync(0xffffffffu, hi, o);
    lo = l2 < lo ? l2 : lo; hi = h2 > hi ? h2 : hi;
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    nans += __shfl_xor_sync(0xffffffffu, nans, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicMin(&keys[0], f64_key(lo));
    atomicMax(&keys[1], f64_key(hi));
    atomicAdd((unsigned long long*)&keys[2], (unsigned long long)cnt);
    if (nans) atomicAdd((unsigned long long*)&keys[3], (unsigned long long)nans);
  }
}

// ---- per-voxel image types (reference radiomics/imageoperations.py:973-1073).  The scalar `c` comes from the host,
// where it is computed by the reference's own NumPy expression from M = max|x|.  Every product and sum is an explicit
// _rn intrinsic, so no FMA contraction can make a voxel differ from NumPy's; sqrt is correctly rounded, log / exp <= 1 ulp.
template <int KIND>
__global__ void __launch_bounds__(256)
pointwise_image_kernel(const void* __restrict__ img, int dt, long long n, double c, double* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double x = load_f64(img, dt, i);
    double r;
    if (KIND == RB_PW_SQUARE) {
      const double t = __dmul_rn(c, x);
      r = __dmul_rn(t, t);
    } else if (KIND == RB_PW_SQUAREROOT) {            // 0 and NaN stay as they are
      r = x > 0 ? sqrt(__dmul_rn(x, c)) : x < 0 ? -sqrt(__dmul_rn(-x, c)) : x;
    } else if (KIND == RB_PW_LOGARITHM) {
      r = __dmul_rn(x > 0 ? log(__dadd_rn(x, 1.0)) : x < 0 ? -log(-__dadd_rn(x, -1.0)) : x, c);
    } else {
      r = exp(__dmul_rn(c, x));
    }
    out[i] = r;
  }
}

// ---- gradient magnitude (ITK GradientMagnitudeImageFilter as called at imageoperations.py:1089-1090): per axis the
// central-difference inner product ((-0.5 w) f[-1] + 0 f[0]) + (0.5 w) f[+1] in ITK's order, neighbours clamped to the
// edge (zero-flux Neumann), then sqrt(((0 + gx^2) + gy^2) + gz^2).  The 0 * f[0] term is kept so that inf / NaN spread
// as they do in ITK.  A thread owns one (y, x) column and marches GRAD_ZCHUNK planes along z, keeping f[z-1], f[z],
// f[z+1] in registers: one new load from HBM per voxel, the four in-plane neighbours were loaded by the neighbouring
// threads in the previous step and come from L1.
constexpr int GRAD_TX = 128, GRAD_ZCHUNK = 32;

__device__ __forceinline__ double central_diff(double fm, double f0, double fp, double w) {
  return __dadd_rn(__dadd_rn(__dmul_rn(-0.5 * w, fm), __dmul_rn(0.0, f0)), __dmul_rn(0.5 * w, fp));
}

__global__ void __launch_bounds__(GRAD_TX)
gradient_magnitude_kernel(const void* __restrict__ img, int dt, int Z, int Y, int X, double wz, double wy, double wx,
                          double* __restrict__ out) {
  const int tiles_x = (X + GRAD_TX - 1) / GRAD_TX;
  const int y = blockIdx.x / tiles_x, x = (blockIdx.x % tiles_x) * GRAD_TX + threadIdx.x;
  if (x >= X) return;
  const int z0 = blockIdx.y * GRAD_ZCHUNK, z1 = min(z0 + GRAD_ZCHUNK, Z);
  const long long plane = (long long)Y * X;
  const int dxm = x > 0 ? -1 : 0, dxp = x < X - 1 ? 1 : 0;
  const int dym = y > 0 ? -X : 0, dyp = y < Y - 1 ? X : 0;
  long long i = (long long)z0 * plane + (long long)y * X + x;
  double f0 = load_f64(img, dt, i);
  double fm = z0 > 0 ? load_f64(img, dt, i - plane) : f0;
  for (int z = z0; z < z1; z++, i += plane) {
    const double fp = z < Z - 1 ? load_f64(img, dt, i + plane) : f0;
    const double gx = central_diff(load_f64(img, dt, i + dxm), f0, load_f64(img, dt, i + dxp), wx);
    const double gy = central_diff(load_f64(img, dt, i + dym), f0, load_f64(img, dt, i + dyp), wy);
    const double gz = central_diff(fm, f0, fp, wz);
    out[i] = sqrt(__dadd_rn(__dadd_rn(__dadd_rn(0.0, __dmul_rn(gx, gx)), __dmul_rn(gy, gy)), __dmul_rn(gz, gz)));
    fm = f0;
    f0 = fp;
  }
}

// ---- normalisation and resegmentation (reference radiomics/imageoperations.py:615-742).
// roi_moments: count, NaN count, sum, max (pass 1) and sum of (x - mean)^2 (pass 2) of the image or of its mask != 0
// voxels, in float64.  The grid is fixed (MOM_GRID blocks at most, fewer only for small images), every block writes its
// partial to scratch and one block adds the partials up in index order, so the result is the same bit pattern on every
// run and every card.  Pass 2 reads the mean from pass 1's result in device memory: the host does not wait in between.
constexpr int MOM_THREADS = 256, MOM_GRID = 1024;
static_assert(RB_MOMENTS_SCRATCH_BYTES >= MOM_GRID * (2 * sizeof(long long) + 3 * sizeof(double)), "moments scratch");

struct MomAcc {
  long long n, nnan;
  double sum, max;
};

// np.max: a NaN anywhere makes the maximum NaN
__device__ __forceinline__ double nan_max(double a, double b) { return (b > a || b != b) ? b : a; }

__device__ __forceinline__ MomAcc mom_combine(MomAcc a, const MomAcc& b) {
  a.n += b.n;
  a.nnan += b.nnan;
  a.sum = __dadd_rn(a.sum, b.sum);
  a.max = nan_max(a.max, b.max);
  return a;
}

// fixed-shape block reduction (shuffle tree per warp, then warp 0 over the warp results): the same order on every run
__device__ MomAcc mom_block_reduce(MomAcc v) {
  __shared__ MomAcc s_w[MOM_THREADS / 32];
  for (int o = 16; o; o >>= 1) {
    MomAcc u;
    u.n = __shfl_down_sync(0xffffffffu, v.n, o);
    u.nnan = __shfl_down_sync(0xffffffffu, v.nnan, o);
    u.sum = __shfl_down_sync(0xffffffffu, v.sum, o);
    u.max = __shfl_down_sync(0xffffffffu, v.max, o);
    v = mom_combine(v, u);
  }
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    v = threadIdx.x < MOM_THREADS / 32 ? s_w[threadIdx.x] : MomAcc{0, 0, 0.0, -1.0 / 0.0};
    for (int o = 16; o; o >>= 1) {
      MomAcc u;
      u.n = __shfl_down_sync(0xffffffffu, v.n, o);
      u.nnan = __shfl_down_sync(0xffffffffu, v.nnan, o);
      u.sum = __shfl_down_sync(0xffffffffu, v.sum, o);
      u.max = __shfl_down_sync(0xffffffffu, v.max, o);
      v = mom_combine(v, u);
    }
  }
  return v;                                               // valid in thread 0
}

// PASS 1: n, nnan, sum, max into part[blockIdx.x].  PASS 2: sum of (x - mean)^2 into part[blockIdx.x].sum, the mean
// being res[2] / res[0] of pass 1.
template <int PASS>
__global__ void __launch_bounds__(MOM_THREADS)
roi_moments_kernel(const void* __restrict__ img, int dt, const uint8_t* __restrict__ mask, long long n,
                   const double* __restrict__ res, MomAcc* __restrict__ part) {
  MomAcc a{0, 0, 0.0, -1.0 / 0.0};
  const double mu = PASS == 2 ? __ddiv_rn(res[2], res[0]) : 0.0;
  for (long long i = (long long)blockIdx.x * MOM_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * MOM_THREADS) {
    if (mask && !mask[i]) continue;
    const double x = load_f64(img, dt, i);
    if (PASS == 1) {
      a.n++;
      a.nnan += x != x;
      a.sum = __dadd_rn(a.sum, x);
      a.max = nan_max(a.max, x);
    } else {
      const double d = __dsub_rn(x, mu);
      a.sum = __dadd_rn(a.sum, __dmul_rn(d, d));
    }
  }
  a = mom_block_reduce(a);
  if (threadIdx.x == 0) part[blockIdx.x] = a;
}

// one block: the `nparts` partials in index order -> res[0..3] (PASS 1: n, nnan, sum, max) or res[4] (PASS 2)
template <int PASS>
__global__ void __launch_bounds__(MOM_THREADS)
roi_moments_final_kernel(const MomAcc* __restrict__ part, int nparts, double* __restrict__ res) {
  MomAcc a{0, 0, 0.0, -1.0 / 0.0};
  for (int k = threadIdx.x; k < nparts; k += MOM_THREADS) a = mom_combine(a, part[k]);
  a = mom_block_reduce(a);
  if (threadIdx.x != 0) return;
  if (PASS == 1) {
    res[0] = (double)a.n;
    res[1] = (double)a.nnan;
    res[2] = a.sum;
    res[3] = a.max;
  } else {
    res[4] = a.sum;
  }
}

// sitk.Normalize (ITK ShiftScale: shift -mean, then scale 1/sigma), the optional clamp to +-outliers and `*= scale`
// (imageoperations.py:638-652).  Plain comparisons in the clamp keep NaN as NaN, like NumPy's masked assignment; every
// step is rounded on its own (no FMA).
__global__ void __launch_bounds__(256)
normalize_kernel(const void* __restrict__ img, int dt, long long n, double mean, double inv_sigma, int clamp,
                 double outliers, double scale, double* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double v = __dmul_rn(__dsub_rn(load_f64(img, dt, i), mean), inv_sigma);
    if (clamp) {
      if (v > outliers) v = outliers;
      if (v < -outliers) v = -outliers;
    }
    out[i] = __dmul_rn(v, scale);
  }
}

// resegmentMask's thresholds (imageoperations.py:713-722): out[i] = mask[i] && lo <= x (&& x <= hi when two).  The
// thresholds arrive rounded to the dtype NumPy compares in, so the float64 comparison gives NumPy's answer.
// counts[0] += ROI voxels, counts[1] += kept voxels (integer sums: the same whatever the order).
__global__ void __launch_bounds__(256)
resegment_kernel(const void* __restrict__ img, int dt, const uint8_t* __restrict__ mask, long long n, double lo,
                 double hi, int two, uint8_t* __restrict__ out, unsigned long long* __restrict__ counts) {
  unsigned long long roi = 0, kept = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    uint8_t k = 0;
    if (mask[i]) {
      const double x = load_f64(img, dt, i);
      k = x >= lo && (!two || x <= hi);
      roi++;
      kept += k;
    }
    out[i] = k;
  }
  for (int o = 16; o; o >>= 1) {
    roi += __shfl_xor_sync(0xffffffffu, roi, o);
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
  }
  if ((threadIdx.x & 31) == 0 && roi) {
    atomicAdd(&counts[0], roi);
    atomicAdd(&counts[1], kept);
  }
}

// out[i] = #{k : edges[k] <= x}  (np.digitize with increasing bins, right=False), 0 outside the mask
__global__ void __launch_bounds__(256)
digitize_kernel(const void* __restrict__ img, int dt, const uint8_t* __restrict__ mask, long long n,
                const double* __restrict__ edges, int ne, int32_t* __restrict__ out) {
  extern __shared__ double s_edges[];
  const bool use_s = ne <= 4096;
  if (use_s) { for (int k = threadIdx.x; k < ne; k += blockDim.x) s_edges[k] = edges[k]; __syncthreads(); }
  const double* e = use_s ? s_edges : edges;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int32_t b = 0;
    if (!mask || mask[i]) {
      const double x = load_f64(img, dt, i);
      int lo = 0, hi = ne;
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (e[mid] <= x) lo = mid + 1; else hi = mid; }
      b = lo;
    }
    out[i] = b;
  }
}

// ---- stationary wavelet, one axis: lo/hi[n] = sum_j f[j] * x[(n + F/2 - j) mod Np], Np = N
// rounded up to even; the pad sample (index N when N is odd) is a copy of x[0] ("wrap" padding,
// imageoperations.py:914-919) and the padded output sample is never stored (cropped, :947-951).
struct SwtFilters { int F; double lo[24], hi[24]; };

__global__ void __launch_bounds__(256)
swt_axis_kernel(const double* __restrict__ in, int Z, int Y, int X, int axis, const __grid_constant__ SwtFilters W,
                double* __restrict__ out_lo, double* __restrict__ out_hi) {
  const long long n = (long long)Z * Y * X, plane = (long long)Y * X;
  const int N = axis == 0 ? Z : axis == 1 ? Y : X;
  const int Np = N + (N & 1);
  const long long stride = axis == 0 ? plane : axis == 1 ? X : 1;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(t / plane), rem = (int)(t % plane), y = rem / X, x = rem % X;
    const int c = axis == 0 ? z : axis == 1 ? y : x;
    const long long base = t - (long long)c * stride;
    double a = 0, d = 0;
    for (int j = 0; j < W.F; j++) {
      int k = (c + W.F / 2 - j) % Np;
      if (k < 0) k += Np;
      if (k >= N) k = 0;                       // the wrap-padding sample
      const double v = in[base + (long long)k * stride];
      a += W.lo[j] * v; d += W.hi[j] * v;
    }
    out_lo[t] = a; out_hi[t] = d;
  }
}

// ---- recursive Gaussian (Deriche 4th order, as used by ITK's RecursiveGaussianImageFilter), one
// line per thread along `axis`; causal + anti-causal passes summed.  Coefficients are computed on
// the host (rg_coefficients).  `scratch` holds the causal pass (same shape as the volume).
struct RGCoef { double N0, N1, N2, N3, D1, D2, D3, D4, M1, M2, M3, M4, BN1, BN2, BN3, BN4, BM1, BM2, BM3, BM4; };

template <typename TIn>
__global__ void __launch_bounds__(128)
recursive_gauss_axis_kernel(const TIn* __restrict__ in, int Z, int Y, int X, int axis, const __grid_constant__ RGCoef C,
                            float* __restrict__ out, double* __restrict__ scratch, double scale, int accumulate) {
  const int N = axis == 0 ? Z : axis == 1 ? Y : X;
  const long long plane = (long long)Y * X;
  const long long stride = axis == 0 ? plane : axis == 1 ? X : 1;
  const long long nlines = (long long)Z * Y * X / N;
  for (long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x; l < nlines; l += (long long)gridDim.x * blockDim.x) {
    long long base;
    if (axis == 2) base = l * X;
    else if (axis == 1) { const long long z = l / X, x = l % X; base = z * plane + x; }
    else base = l;
    // causal pass; boundary: the edge value is assumed to extend to infinity
    const double v0 = (double)in[base];
    double x1 = v0, x2 = v0, x3 = v0;
    const double sN = C.N0 + C.N1 + C.N2 + C.N3, sD = 1.0 + C.D1 + C.D2 + C.D3 + C.D4;
    double y1 = v0 * sN / sD, y2 = y1, y3 = y1, y4 = y1;
    for (int i = 0; i < N; i++) {
      const double xi = (double)in[base + (long long)i * stride];
      const double y = C.N0 * xi + C.N1 * x1 + C.N2 * x2 + C.N3 * x3 - C.D1 * y1 - C.D2 * y2 - C.D3 * y3 - C.D4 * y4;
      scratch[base + (long long)i * stride] = y;
      x3 = x2; x2 = x1; x1 = xi; y4 = y3; y3 = y2; y2 = y1; y1 = y;
    }
    // anti-causal pass
    const double vN = (double)in[base + (long long)(N - 1) * stride];
    double a1 = vN, a2 = vN, a3 = vN, a4 = vN;
    const double sM = C.M1 + C.M2 + C.M3 + C.M4;
    double b1 = vN * sM / sD, b2 = b1, b3 = b1, b4 = b1;
    for (int i = N - 1; i >= 0; i--) {
      const double xi = (double)in[base + (long long)i * stride];
      const double y = C.M1 * a1 + C.M2 * a2 + C.M3 * a3 + C.M4 * a4 - C.D1 * b1 - C.D2 * b2 - C.D3 * b3 - C.D4 * b4;
      const long long o = base + (long long)i * stride;
      const float r = (float)((scratch[o] + y) * scale);
      out[o] = accumulate ? out[o] + r : r;
      a4 = a3; a3 = a2; a2 = a1; a1 = xi; b4 = b3; b3 = b2; b2 = b1; b1 = y;
    }
  }
}

// ---- fused level-1 3-D stationary wavelet transform (all 8 sub-bands in ONE pass over the volume) ----------------
// A CTA owns a TY x TX tile of the (y,x) plane and marches along z.  Per plane: the input tile with its F-1 halo
// columns / rows is staged in shared memory (periodic indices), filtered along x (lo + hi), then along y -> the four
// xy-bands of that plane, which go into a ring of F planes in shared memory; the z filter then reads the ring and
// writes the 8 sub-bands of one output plane with coalesced 256-byte rows.  HBM traffic: the input once (x 1.7 for the
// xy halo) + the 8 outputs once = ~78 B/voxel against 168 B/voxel for seven separate axis passes (ideal 72).
// Periodic in all three axes (callers wrap-pad odd sizes first, like the reference: imageoperations.py:914-919).
// Sub-band b = bx + 2*by + 4*bz (bit set = high-pass along that axis) goes to out[b * band_stride + voxel].
constexpr int SWT_TY = 8, SWT_TX = 32;
template <int F>
__global__ void __launch_bounds__(SWT_TY * SWT_TX)
swt3d_kernel(const double* __restrict__ in, int Z, int Y, int X, const __grid_constant__ SwtFilters W,
             double* __restrict__ out, long long band_stride, int z_begin, int z_end) {
  constexpr int TY = SWT_TY, TX = SWT_TX, H = F - 1, NT = TY * TX;
  constexpr int LOWER = F - 1 - F / 2;                 // taps reach from n - LOWER to n + F/2
  extern __shared__ double swt_smem[];
  double* const tile = swt_smem;                                         // input plane tile with halo [(TY+H)][(TX+H)]
  double (*const xf)[(TY + H) * TX] = reinterpret_cast<double (*)[(TY + H) * TX]>(swt_smem + (TY + H) * (TX + H));   // x-filtered (lo, hi)
  double (*const ring)[4][NT] = reinterpret_cast<double (*)[4][NT]>(swt_smem + (TY + H) * (TX + H) + 2 * (TY + H) * TX);
  // ring: xy-bands of the last F planes [slot][bx + 2*by][ty*TX + tx]
  const int tx = threadIdx.x % TX, ty = threadIdx.x / TX, tid = threadIdx.x;
  const int tiles_x = (X + TX - 1) / TX;
  const int x0 = (blockIdx.x % tiles_x) * TX, y0 = (blockIdx.x / tiles_x) * TY;
  const long long plane = (long long)Y * X;
  auto wrap = [](int i, int n) { i %= n; return i < 0 ? i + n : i; };
  // xy-filter plane zp (periodic) into ring slot `slot`
  auto stage = [&](int zp, int slot) {
    const double* src = in + (long long)wrap(zp, Z) * plane;
    for (int i = tid; i < (TY + H) * (TX + H); i += NT) {
      const int r = i / (TX + H), c = i % (TX + H);
      tile[i] = src[(long long)wrap(y0 + r - LOWER, Y) * X + wrap(x0 + c - LOWER, X)];
    }
    __syncthreads();
    for (int i = tid; i < (TY + H) * TX; i += NT) {
      const int r = i / TX, c = i % TX;
      double a = 0, d = 0;
#pragma unroll
      for (int j = 0; j < F; j++) {                      // out[n] = sum_j f[j] x[n + F/2 - j]; tile column of x is c + LOWER
        const double v = tile[r * (TX + H) + c + LOWER + F / 2 - j];
        a += W.lo[j] * v; d += W.hi[j] * v;
      }
      xf[0][i] = a; xf[1][i] = d;
    }
    __syncthreads();
    double ll = 0, lh = 0, hl = 0, hh = 0;             // first letter = x band, second = y band
#pragma unroll
    for (int j = 0; j < F; j++) {
      const int r = ty + LOWER + F / 2 - j;
      const double va = xf[0][r * TX + tx], vd = xf[1][r * TX + tx];
      ll += W.lo[j] * va; lh += W.hi[j] * va; hl += W.lo[j] * vd; hh += W.hi[j] * vd;
    }
    ring[slot][0][tid] = ll; ring[slot][1][tid] = hl; ring[slot][2][tid] = lh; ring[slot][3][tid] = hh;   // index bx + 2*by
  };
  // output planes [z_begin, z_end) of the input volume (a multi-GPU caller passes its slab plus halo planes and asks for
  // the interior: no z wrap-around is then ever taken); out plane index = z - z_begin
  for (int zp = z_begin - LOWER; zp < z_begin + F / 2; zp++) stage(zp, wrap(zp, F));   // planes z-LOWER .. z+F/2-1 of the first z
  const bool inside = (y0 + ty) < Y && (x0 + tx) < X;
  for (int z = z_begin; z < z_end; z++) {
    stage(z + F / 2, wrap(z + F / 2, F));
    __syncthreads();
    double o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int j = 0; j < F; j++) {
      const int slot = wrap(z + F / 2 - j, F);
#pragma unroll
      for (int b = 0; b < 4; b++) {
        const double v = ring[slot][b][tid];
        o[b] += W.lo[j] * v; o[b + 4] += W.hi[j] * v;
      }
    }
    if (inside) {
      const long long vi = (long long)(z - z_begin) * plane + (long long)(y0 + ty) * X + (x0 + tx);
#pragma unroll
      for (int b = 0; b < 8; b++) out[b * band_stride + vi] = o[b];
    }
    __syncthreads();                                   // the ring slot of plane z-LOWER is overwritten next
  }
}

// ---- recursive Gaussian along x with coalesced access: a warp owns 32 consecutive lines (= rows of one plane) and walks
// them in 32-column tiles staged through shared memory (read: each row segment is 32 consecutive elements; the
// per-thread recursion then reads a column of the transposed tile), causal then anti-causal, the causal results
// parked in the `scratch` volume in the same tiled, coalesced way.  (Round 1: one line per thread -> lanes X elements
// apart, every load its own 32-byte sector.)
template <typename TIn>
__global__ void __launch_bounds__(128)
recursive_gauss_x_kernel(const TIn* __restrict__ in, long long nlines, int X, const __grid_constant__ RGCoef C,
                         float* __restrict__ out, double* __restrict__ scratch, double scale, int accumulate) {
  __shared__ double tile[4][32][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long nwarps = (long long)gridDim.x * 4;
  const double sN = C.N0 + C.N1 + C.N2 + C.N3, sD = 1.0 + C.D1 + C.D2 + C.D3 + C.D4, sM = C.M1 + C.M2 + C.M3 + C.M4;
  for (long long l0 = ((long long)blockIdx.x * 4 + w) * 32; l0 < nlines; l0 += nwarps * 32) {
    const long long myline = l0 + lane;
    const bool live = myline < nlines;
    const long long mybase = (live ? myline : l0) * X;
    const double v0 = (double)in[mybase];
    double x1 = v0, x2 = v0, x3 = v0;
    double y1 = v0 * sN / sD, y2 = y1, y3 = y1, y4 = y1;
    for (int c0 = 0; c0 < X; c0 += 32) {
      // load: row r of the tile = 32 consecutive elements of line l0 + r
      for (int r = 0; r < 32; r++) {
        const long long ln = l0 + r;
        tile[w][r][lane] = (ln < nlines && c0 + lane < X) ? (double)in[ln * X + c0 + lane] : 0.0;
      }
      __syncwarp();
      const int nc = X - c0 < 32 ? X - c0 : 32;
      for (int c = 0; c < nc; c++) {
        const double xi = tile[w][lane][c];
        const double y = C.N0 * xi + C.N1 * x1 + C.N2 * x2 + C.N3 * x3 - C.D1 * y1 - C.D2 * y2 - C.D3 * y3 - C.D4 * y4;
        tile[w][lane][c] = y;
        x3 = x2; x2 = x1; x1 = xi; y4 = y3; y3 = y2; y2 = y1; y1 = y;
      }
      __syncwarp();
      for (int r = 0; r < 32; r++) {
        const long long ln = l0 + r;
        if (ln < nlines && c0 + lane < X) scratch[ln * X + c0 + lane] = tile[w][r][lane];
      }
      __syncwarp();
    }
    const double vN = (double)in[mybase + X - 1];
    double a1 = vN, a2 = vN, a3 = vN, a4 = vN;
    double b1 = vN * sM / sD, b2 = b1, b3 = b1, b4 = b1;
    for (int c0 = (X - 1) / 32 * 32; c0 >= 0; c0 -= 32) {
      for (int r = 0; r < 32; r++) {
        const long long ln = l0 + r;
        tile[w][r][lane] = (ln < nlines && c0 + lane < X) ? (double)in[ln * X + c0 + lane] : 0.0;
      }
      __syncwarp();
      const int nc = X - c0 < 32 ? X - c0 : 32;
      for (int c = nc - 1; c >= 0; c--) {
        const double xi = tile[w][lane][c];
        const double y = C.M1 * a1 + C.M2 * a2 + C.M3 * a3 + C.M4 * a4 - C.D1 * b1 - C.D2 * b2 - C.D3 * b3 - C.D4 * b4;
        tile[w][lane][c] = y;
        a4 = a3; a3 = a2; a2 = a1; a1 = xi; b4 = b3; b3 = b2; b2 = b1; b1 = y;
      }
      __syncwarp();
      for (int r = 0; r < 32; r++) {
        const long long ln = l0 + r;
        if (ln < nlines && c0 + lane < X) {
          const long long o = ln * X + c0 + lane;
          const float res = (float)((scratch[o] + tile[w][r][lane]) * scale);
          out[o] = accumulate ? out[o] + res : res;
        }
      }
      __syncwarp();
    }
  }
}

int minmax_launch(const void* img, int dt, const uint8_t* mask, long long n, long long* keys, cudaStream_t st) {
  minmax_kernel<<<grid_for(n, 256, 8), 256, 0, st>>>(img, dt, mask, n, keys);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int pointwise_image_launch(const void* img, int dt, long long n, int kind, double c, double* out, cudaStream_t st) {
  const int grid = grid_for(n, 256, 8);
  switch (kind) {
    case RB_PW_SQUARE: pointwise_image_kernel<RB_PW_SQUARE><<<grid, 256, 0, st>>>(img, dt, n, c, out); break;
    case RB_PW_SQUAREROOT: pointwise_image_kernel<RB_PW_SQUAREROOT><<<grid, 256, 0, st>>>(img, dt, n, c, out); break;
    case RB_PW_LOGARITHM: pointwise_image_kernel<RB_PW_LOGARITHM><<<grid, 256, 0, st>>>(img, dt, n, c, out); break;
    case RB_PW_EXPONENTIAL: pointwise_image_kernel<RB_PW_EXPONENTIAL><<<grid, 256, 0, st>>>(img, dt, n, c, out); break;
    default: return fail(RB_ERR_ARG, "pointwise image: unknown kind %d", kind);
  }
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int gradient_magnitude_launch(const void* img, int dt, int Z, int Y, int X, const double* w_zyx, double* out, cudaStream_t st) {
  const long long columns = (long long)((X + GRAD_TX - 1) / GRAD_TX) * Y;
  if (columns > 0x7fffffffLL) return fail(RB_ERR_UNSUPPORTED, "gradient magnitude: %d x %d plane too large", Y, X);
  const dim3 grid((unsigned)columns, (unsigned)((Z + GRAD_ZCHUNK - 1) / GRAD_ZCHUNK));
  gradient_magnitude_kernel<<<grid, GRAD_TX, 0, st>>>(img, dt, Z, Y, X, w_zyx[0], w_zyx[1], w_zyx[2], out);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int roi_moments_launch(const void* img, int dt, const uint8_t* mask, long long n, int passes, void* scratch, double* res,
                       cudaStream_t st) {
  const long long need = (n + MOM_THREADS - 1) / MOM_THREADS;
  const int grid = (int)(need < MOM_GRID ? need : MOM_GRID);      // depends on n only, never on the card
  MomAcc* part = (MomAcc*)scratch;
  roi_moments_kernel<1><<<grid, MOM_THREADS, 0, st>>>(img, dt, mask, n, res, part);
  roi_moments_final_kernel<1><<<1, MOM_THREADS, 0, st>>>(part, grid, res);
  if (passes == 2) {
    roi_moments_kernel<2><<<grid, MOM_THREADS, 0, st>>>(img, dt, mask, n, res, part);
    roi_moments_final_kernel<2><<<1, MOM_THREADS, 0, st>>>(part, grid, res);
  } else {
    RB_CUDA(cudaMemsetAsync(res + 4, 0xff, sizeof(double), st));   // NaN: no second pass
  }
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int normalize_launch(const void* img, int dt, long long n, double mean, double sigma, int clamp, double outliers,
                     double scale, double* out, cudaStream_t st) {
  normalize_kernel<<<grid_for(n, 256, 8), 256, 0, st>>>(img, dt, n, mean, 1.0 / sigma, clamp, outliers, scale, out);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int resegment_launch(const void* img, int dt, const uint8_t* mask, long long n, double lo, double hi, int two,
                     uint8_t* out, unsigned long long* counts, cudaStream_t st) {
  RB_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(unsigned long long), st));
  resegment_kernel<<<grid_for(n, 256, 8), 256, 0, st>>>(img, dt, mask, n, lo, hi, two, out, counts);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int digitize_launch(const void* img, int dt, const uint8_t* mask, long long n, const double* edges, int ne, int32_t* out,
                    cudaStream_t st) {
  const size_t sh = ne <= 4096 ? sizeof(double) * ne : 0;
  digitize_kernel<<<grid_for(n, 256, 8), 256, sh, st>>>(img, dt, mask, n, edges, ne, out);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int swt_axis_launch(const double* in, int Z, int Y, int X, int axis, const double* lo, const double* hi, int F,
                    double* out_lo, double* out_hi, cudaStream_t st) {
  if (F < 2 || F > 24) return fail(RB_ERR_UNSUPPORTED, "wavelet filter length %d outside 2..24", F);
  SwtFilters W;
  W.F = F;
  for (int j = 0; j < F; j++) { W.lo[j] = lo[j]; W.hi[j] = hi[j]; }
  swt_axis_kernel<<<grid_for((long long)Z * Y * X, 256, 8), 256, 0, st>>>(in, Z, Y, X, axis, W, out_lo, out_hi);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int swt3d_launch(const double* in, int Z, int Y, int X, const double* lo, const double* hi, int F, double* out,
                 long long band_stride, int z_begin, int z_end, cudaStream_t st) {
  if (z_begin < 0 || z_end > Z || z_begin > z_end) return fail(RB_ERR_ARG, "fused 3-D SWT: bad plane range [%d, %d) of %d", z_begin, z_end, Z);
  if (z_begin == z_end) return RB_OK;
  if (F != 2 && F != 4 && F != 6 && F != 8) return fail(RB_ERR_UNSUPPORTED, "fused 3-D SWT: filter length %d (2, 4, 6 or 8)", F);
  if (Z < 1 || Y < 1 || X < 1) return fail(RB_ERR_ARG, "empty volume");
  SwtFilters W;
  W.F = F;
  for (int j = 0; j < F; j++) { W.lo[j] = lo[j]; W.hi[j] = hi[j]; }
  const int grid = ((X + SWT_TX - 1) / SWT_TX) * ((Y + SWT_TY - 1) / SWT_TY);
  const int H = F - 1, NT = SWT_TY * SWT_TX;
  const int smem = (int)sizeof(double) * ((SWT_TY + H) * (SWT_TX + H) + 2 * (SWT_TY + H) * SWT_TX + F * 4 * NT);
  RB_CUDA(set_max_dynamic_smem(swt3d_kernel<6>, 64 * 1024));
  RB_CUDA(set_max_dynamic_smem(swt3d_kernel<8>, 96 * 1024));
  if (F == 2) swt3d_kernel<2><<<grid, NT, smem, st>>>(in, Z, Y, X, W, out, band_stride, z_begin, z_end);
  else if (F == 4) swt3d_kernel<4><<<grid, NT, smem, st>>>(in, Z, Y, X, W, out, band_stride, z_begin, z_end);
  else if (F == 6) swt3d_kernel<6><<<grid, NT, smem, st>>>(in, Z, Y, X, W, out, band_stride, z_begin, z_end);
  else swt3d_kernel<8><<<grid, NT, smem, st>>>(in, Z, Y, X, W, out, band_stride, z_begin, z_end);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int recursive_gauss_launch(const void* in, int in_is_f32, int Z, int Y, int X, int axis, const double* coef20, float* out,
                           double* scratch, double scale, int accumulate, cudaStream_t st) {
  RGCoef C;
  memcpy(&C, coef20, sizeof C);
  const int N = axis == 0 ? Z : axis == 1 ? Y : X;
  const long long nlines = (long long)Z * Y * X / N;
  if (axis == 2) {                              // x: lines are contiguous -> tile-transposed kernel, 32 lines per warp
    const int gx = grid_for((nlines + 31) / 32, 4, 16);
    if (in_is_f32) recursive_gauss_x_kernel<float><<<gx, 128, 0, st>>>((const float*)in, nlines, X, C, out, scratch, scale, accumulate);
    else recursive_gauss_x_kernel<double><<<gx, 128, 0, st>>>((const double*)in, nlines, X, C, out, scratch, scale, accumulate);
    RB_LAUNCH_CHECK();
    return RB_OK;
  }
  const int grid = grid_for(nlines, 128, 8);
  if (in_is_f32) recursive_gauss_axis_kernel<float><<<grid, 128, 0, st>>>((const float*)in, Z, Y, X, axis, C, out, scratch, scale, accumulate);
  else recursive_gauss_axis_kernel<double><<<grid, 128, 0, st>>>((const double*)in, Z, Y, X, axis, C, out, scratch, scale, accumulate);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb

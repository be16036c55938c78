// Pre-filter and discretisation kernels feeding the texture path (SURVEY.md section 8a: a14-a16):
//   * gray-level discretisation: ROI min/max reduction + np.digitize-exact binning
//     (reference radiomics/imageoperations.py:67-174)
//   * level-1 stationary wavelet transform, periodic, one axis per pass, low+high band per pass
//     (reference radiomics/imageoperations.py:899-970 -> pywt.swtn(level=1), PyWavelets >= 1.6)
//   * Laplacian of Gaussian by recursive (IIR) Gaussian filtering, one line per thread
//     (reference radiomics/imageoperations.py:756-836 -> ITK LaplacianRecursiveGaussianImageFilter)
// All are HBM-streaming kernels: every thread handles consecutive x so loads/stores coalesce; the
// wavelet pass reads its 6 taps through L1 (neighbouring threads share them).
#include "common.cuh"

namespace rb {

enum DType { DT_I16 = 0, DT_I32 = 1, DT_F32 = 2, DT_F64 = 3, DT_U8 = 4, DT_U16 = 5, DT_I64 = 6 };

template <typename T> __device__ __forceinline__ double as_f64(const void* p, long long i) { return (double)((const T*)p)[i]; }
__device__ __forceinline__ double load_any(const void* p, int dt, long long i) {
  switch (dt) {
    case DT_I16: return as_f64<int16_t>(p, i);
    case DT_I32: return as_f64<int32_t>(p, i);
    case DT_F32: return as_f64<float>(p, i);
    case DT_F64: return as_f64<double>(p, i);
    case DT_U8: return as_f64<uint8_t>(p, i);
    case DT_U16: return as_f64<uint16_t>(p, i);
    default: return as_f64<long long>(p, i);
  }
}

// order-preserving map double <-> signed 64-bit, so atomicMin/atomicMax work on doubles
__device__ __forceinline__ long long f64_key(double v) {
  long long b = __double_as_longlong(v);
  return b >= 0 ? b : b ^ 0x7FFFFFFFFFFFFFFFll;
}

__global__ void __launch_bounds__(256)
minmax_kernel(const void* __restrict__ img, int dt, const uint8_t* __restrict__ mask, long long n,
              long long* __restrict__ keys /* [0]=min key, [1]=max key, [2]=count */) {
  double lo = 1.0 / 0.0, hi = -1.0 / 0.0;
  long long cnt = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (mask && !mask[i]) continue;
    const double v = load_any(img, dt, i);
    lo = v < lo ? v : lo; hi = v > hi ? v : hi; cnt++;
  }
  for (int o = 16; o; o >>= 1) {
    const double l2 = __shfl_xor_sync(0xffffffffu, lo, o), h2 = __shfl_xor_sync(0xffffffffu, hi, o);
    lo = l2 < lo ? l2 : lo; hi = h2 > hi ? h2 : hi;
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicMin(&keys[0], f64_key(lo));
    atomicMax(&keys[1], f64_key(hi));
    atomicAdd((unsigned long long*)&keys[2], (unsigned long long)cnt);
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
      const double x = load_any(img, dt, i);
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

static int grid_n(long long n, int block, int per_sm) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long need = (n + block - 1) / block, cap = (long long)sms * per_sm;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

int minmax_launch(const void* img, int dt, const uint8_t* mask, long long n, long long* keys, cudaStream_t st) {
  minmax_kernel<<<grid_n(n, 256, 8), 256, 0, st>>>(img, dt, mask, n, keys);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int digitize_launch(const void* img, int dt, const uint8_t* mask, long long n, const double* edges, int ne, int32_t* out,
                    cudaStream_t st) {
  const size_t sh = ne <= 4096 ? sizeof(double) * ne : 0;
  digitize_kernel<<<grid_n(n, 256, 8), 256, sh, st>>>(img, dt, mask, n, edges, ne, out);
  RB_LAUNCH_CHECK();
  return RB_OK;
}
int swt_axis_launch(const double* in, int Z, int Y, int X, int axis, const double* lo, const double* hi, int F,
                    double* out_lo, double* out_hi, cudaStream_t st) {
  if (F < 2 || F > 24) return fail(RB_ERR_UNSUPPORTED, "wavelet filter length %d outside 2..24", F);
  SwtFilters W;
  W.F = F;
  for (int j = 0; j < F; j++) { W.lo[j] = lo[j]; W.hi[j] = hi[j]; }
  swt_axis_kernel<<<grid_n((long long)Z * Y * X, 256, 8), 256, 0, st>>>(in, Z, Y, X, axis, W, out_lo, out_hi);
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
  static bool attr[64] = {false};
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr[dev & 63]) {
    RB_CUDA(cudaFuncSetAttribute(swt3d_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    RB_CUDA(cudaFuncSetAttribute(swt3d_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr[dev & 63] = true;
  }
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
    const int gx = grid_n((nlines + 31) / 32, 4, 16);
    if (in_is_f32) recursive_gauss_x_kernel<float><<<gx, 128, 0, st>>>((const float*)in, nlines, X, C, out, scratch, scale, accumulate);
    else recursive_gauss_x_kernel<double><<<gx, 128, 0, st>>>((const double*)in, nlines, X, C, out, scratch, scale, accumulate);
    RB_LAUNCH_CHECK();
    return RB_OK;
  }
  const int grid = grid_n(nlines, 128, 8);
  if (in_is_f32) recursive_gauss_axis_kernel<float><<<grid, 128, 0, st>>>((const float*)in, Z, Y, X, axis, C, out, scratch, scale, accumulate);
  else recursive_gauss_axis_kernel<double><<<grid, 128, 0, st>>>((const double*)in, Z, Y, X, axis, C, out, scratch, scale, accumulate);
  RB_LAUNCH_CHECK();
  return RB_OK;
}

}  // namespace rb

// Segment-based first order (rb_firstorder_segment_dev): the 18 features of one ROI, reduced on the device.
//   pass 1     grid-stride over the volume: ROI count, min / max as order-preserving keys, sum x, sum (x + shift)^2 and
//              the histogram of the packed levels (integer atomics; shared memory for 8-bit levels)
//   select     exact order statistics by radix select on the 64-bit keys: 8 passes of 8-bit digits, one digit histogram
//              per still-distinct prefix of the (at most 10) ranks the percentiles and the median need; a one-thread
//              kernel picks each digit, so the host never waits in between
//   pass 3     with the mean, p10 and p90 on the device: sum |d|, d^2, d^3, d^4 (d = x - mean), and sum x and the count
//              over the closed [p10, p90] range (RobustMeanAbsoluteDeviation)
//   pass 4     sum |x - mean_kept| over that range
//   finish     one block sums Entropy / Uniformity over the level bins, then one thread applies the formulas of the
//              reference's firstorder.py
// Every floating-point sum is a per-thread sum in grid-stride order, a fixed shared-memory tree per block and the block
// partials added in index order by one thread: no floating-point atomics, so repeated runs are bit-identical.
#include <stdint.h>

#include "common.cuh"
#include "pixel.cuh"

namespace rb {

namespace {

constexpr int SEG_NT = 256;
constexpr int SEG_MAXR = 10;          // ranks: floor and ceil of the 10th, 25th, 75th, 90th percentiles, the median pair
constexpr int SEG_NS = 6;             // floating-point sums per block partial
constexpr int SEG_NU = 4;             // integer fields per block partial

struct Partial {
  double s[SEG_NS];
  unsigned long long u[SEG_NU];
};

struct SegState {
  unsigned long long n, kmin, kmax;
  double sum, energy, mean;
  // radix select
  int nr, ng;
  unsigned long long rank[SEG_MAXR];      // rank still to find below the target's prefix
  unsigned long long prefix[SEG_MAXR];    // digits picked so far
  int group[SEG_MAXR];                    // index of the target's prefix among the distinct prefixes
  unsigned long long gprefix[SEG_MAXR];
  unsigned long long hist[SEG_MAXR][256];
  unsigned long long want[SEG_MAXR];      // global rank of each target
  double val[SEG_MAXR];                   // the selected order statistics
  double p10, p25, p75, p90, median;
  // pass 3 / 4
  double sabs, s2, s3, s4, mean_kept;
  unsigned long long nkept;
};

// order-preserving key of a float64 (larger value, larger key); -0.0 is keyed as +0.0
__device__ __forceinline__ unsigned long long f64_key(double x) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(__dadd_rn(x, 0.0));
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_f64(unsigned long long k) {
  return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// NumPy 2.x np.percentile(x, q) (method "linear") of the sorted x from its two neighbouring order statistics a = x[lo],
// b = x[lo + 1]: _lerp(a, b, t), t = (n - 1) * q - lo, evaluated b - (b - a)(1 - t) when t >= 0.5
__device__ __forceinline__ double numpy_lerp(double a, double b, double t) {
  const double diff = __dsub_rn(b, a);
  return t >= 0.5 ? __dsub_rn(b, __dmul_rn(diff, __dsub_rn(1.0, t))) : __dadd_rn(a, __dmul_rn(diff, t));
}

// block sum of v[0..NS) / u[0..NU) of every thread in a fixed tree; thread 0 writes the block's partial
template <int NS, int NU>
__device__ void block_partial(double (&v)[NS], unsigned long long (&u)[NU], bool u_is_minmax, Partial* out) {
  __shared__ double sd[SEG_NT];
  __shared__ unsigned long long su[SEG_NT];
  const int t = threadIdx.x;
  for (int k = 0; k < NS; k++) {
    sd[t] = v[k];
    __syncthreads();
    for (int h = SEG_NT / 2; h > 0; h >>= 1) {
      if (t < h) sd[t] = __dadd_rn(sd[t], sd[t + h]);
      __syncthreads();
    }
    if (t == 0) out[blockIdx.x].s[k] = sd[0];
    __syncthreads();
  }
  for (int k = 0; k < NU; k++) {
    su[t] = u[k];
    __syncthreads();
    for (int h = SEG_NT / 2; h > 0; h >>= 1) {
      if (t < h) {
        const unsigned long long a = su[t], b = su[t + h];
        // u_is_minmax: field 1 is a minimum, field 2 a maximum, the others sums
        su[t] = (u_is_minmax && k == 1) ? (a < b ? a : b) : (u_is_minmax && k == 2) ? (a > b ? a : b) : a + b;
      }
      __syncthreads();
    }
    if (t == 0) out[blockIdx.x].u[k] = su[0];
    __syncthreads();
  }
}

struct SegArgs {
  const void* img;
  int dtype;
  const uint8_t* roi;
  const void* lev;
  int level_bytes;
  long long n;
  double shift;
};

__device__ __forceinline__ int level_at(const SegArgs& A, long long i) {
  return A.level_bytes == 1 ? ((const uint8_t*)A.lev)[i] : ((const uint16_t*)A.lev)[i];
}

// pass 1
__global__ void __launch_bounds__(SEG_NT) seg_pass1(SegArgs A, Partial* part, unsigned long long* lhist) {
  __shared__ unsigned int sh[256];
  const bool shared_hist = A.level_bytes == 1;
  if (shared_hist) {
    sh[threadIdx.x] = 0;
    __syncthreads();
  }
  double v[2] = {0.0, 0.0};
  unsigned long long u[3] = {0ull, ~0ull, 0ull};
  for (long long i = (long long)blockIdx.x * SEG_NT + threadIdx.x; i < A.n; i += (long long)gridDim.x * SEG_NT) {
    if (!A.roi[i]) continue;
    const double x = load_f64(A.img, A.dtype, i);
    const unsigned long long k = f64_key(x);
    const double s = __dadd_rn(x, A.shift);
    u[0]++;
    u[1] = k < u[1] ? k : u[1];
    u[2] = k > u[2] ? k : u[2];
    v[0] = __dadd_rn(v[0], x);
    v[1] = __dadd_rn(v[1], __dmul_rn(s, s));
    const int l = level_at(A, i);
    if (shared_hist) atomicAdd(&sh[l], 1u);
    else atomicAdd(&lhist[l], 1ull);
  }
  block_partial<2, 3>(v, u, true, part);
  if (shared_hist && sh[threadIdx.x]) atomicAdd(&lhist[threadIdx.x], (unsigned long long)sh[threadIdx.x]);
}

// one thread: the pass-1 totals, the mean, and the ranks to select
__global__ void seg_plan(const Partial* part, int nblocks, SegState* S) {
  unsigned long long n = 0, kmin = ~0ull, kmax = 0;
  double sum = 0.0, energy = 0.0;
  for (int b = 0; b < nblocks; b++) {
    n += part[b].u[0];
    kmin = part[b].u[1] < kmin ? part[b].u[1] : kmin;
    kmax = part[b].u[2] > kmax ? part[b].u[2] : kmax;
    sum = __dadd_rn(sum, part[b].s[0]);
    energy = __dadd_rn(energy, part[b].s[1]);
  }
  S->n = n; S->kmin = kmin; S->kmax = kmax; S->sum = sum; S->energy = energy;
  S->nr = 0;
  S->ng = 0;
  if (n == 0) return;
  S->mean = __ddiv_rn(sum, (double)n);
  const double qs[4] = {10.0 / 100.0, 25.0 / 100.0, 75.0 / 100.0, 90.0 / 100.0};
  unsigned long long want[SEG_MAXR];
  int nr = 0;
  for (int q = 0; q < 4; q++) {
    const double vi = __dmul_rn((double)(n - 1), qs[q]);
    const unsigned long long lo = (unsigned long long)floor(vi);
    want[nr++] = lo;
    want[nr++] = lo + 1 < n ? lo + 1 : n - 1;
  }
  want[nr++] = (n - 1) / 2;
  want[nr++] = n / 2;
  for (int r = 0; r < nr; r++) {
    S->want[r] = want[r];
    S->rank[r] = want[r];
    S->prefix[r] = 0;
    S->group[r] = 0;
  }
  S->nr = nr;
  S->ng = 1;
  S->gprefix[0] = 0;
}

// one radix pass: the histogram of digit `pass` of the keys whose higher digits equal one of the distinct prefixes
__global__ void __launch_bounds__(SEG_NT) seg_digits(SegArgs A, SegState* S, int pass) {
  __shared__ unsigned int h[SEG_MAXR][256];
  __shared__ unsigned long long gp[SEG_MAXR];
  const int ng = S->ng;
  if (ng == 0) return;
  for (int k = threadIdx.x; k < ng * 256; k += SEG_NT) h[k / 256][k % 256] = 0;
  if (threadIdx.x < ng) gp[threadIdx.x] = S->gprefix[threadIdx.x];
  __syncthreads();
  const int shift = 56 - 8 * pass;
  for (long long i = (long long)blockIdx.x * SEG_NT + threadIdx.x; i < A.n; i += (long long)gridDim.x * SEG_NT) {
    if (!A.roi[i]) continue;
    const unsigned long long k = f64_key(load_f64(A.img, A.dtype, i));
    const unsigned long long hi = pass == 0 ? 0ull : k >> (shift + 8);
    for (int g = 0; g < ng; g++)
      if (gp[g] == hi) {
        atomicAdd(&h[g][(k >> shift) & 255], 1u);
        break;
      }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ng * 256; k += SEG_NT)
    if (h[k / 256][k % 256]) atomicAdd(&S->hist[k / 256][k % 256], (unsigned long long)h[k / 256][k % 256]);
}

// one thread: pick every target's digit of this pass, regroup the prefixes, clear the histograms; after the last pass,
// the order statistics and the percentiles
__global__ void seg_pick(SegState* S, int pass) {
  const int ng = S->ng;
  if (ng == 0) return;
  for (int r = 0; r < S->nr; r++) {
    const int g = S->group[r];
    unsigned long long cum = 0;
    for (int d = 0; d < 256; d++) {
      const unsigned long long c = S->hist[g][d];
      if (S->rank[r] < cum + c) {
        S->prefix[r] = (S->prefix[r] << 8) | (unsigned long long)d;
        S->rank[r] -= cum;
        break;
      }
      cum += c;
    }
  }
  for (int g = 0; g < ng; g++)
    for (int d = 0; d < 256; d++) S->hist[g][d] = 0;
  int ngn = 0;
  for (int r = 0; r < S->nr; r++) {
    int g = 0;
    while (g < ngn && S->gprefix[g] != S->prefix[r]) g++;
    if (g == ngn) S->gprefix[ngn++] = S->prefix[r];
    S->group[r] = g;
  }
  S->ng = ngn;
  if (pass < 7) return;
  for (int r = 0; r < S->nr; r++) S->val[r] = key_f64(S->prefix[r]);
  const double qs[4] = {10.0 / 100.0, 25.0 / 100.0, 75.0 / 100.0, 90.0 / 100.0};
  double p[4];
  for (int q = 0; q < 4; q++) {
    const double vi = __dmul_rn((double)(S->n - 1), qs[q]);
    // NumPy's gamma is vi - floor(vi), also where it clips the upper neighbour (then both neighbours are x[n-1])
    p[q] = numpy_lerp(S->val[2 * q], S->val[2 * q + 1], __dsub_rn(vi, floor(vi)));
  }
  S->p10 = p[0]; S->p25 = p[1]; S->p75 = p[2]; S->p90 = p[3];
  S->median = __ddiv_rn(__dadd_rn(S->val[8], S->val[9]), 2.0);     // np.median: the mean of the middle pair
}

// pass 3
__global__ void __launch_bounds__(SEG_NT) seg_pass3(SegArgs A, const SegState* S, Partial* part) {
  if (S->n == 0) return;
  const double mean = S->mean, p10 = S->p10, p90 = S->p90;
  double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  unsigned long long u[1] = {0ull};
  for (long long i = (long long)blockIdx.x * SEG_NT + threadIdx.x; i < A.n; i += (long long)gridDim.x * SEG_NT) {
    if (!A.roi[i]) continue;
    const double x = load_f64(A.img, A.dtype, i);
    const double d = __dsub_rn(x, mean);
    const double d2 = __dmul_rn(d, d);
    v[0] = __dadd_rn(v[0], fabs(d));
    v[1] = __dadd_rn(v[1], d2);
    v[2] = __dadd_rn(v[2], __dmul_rn(d2, d));
    v[3] = __dadd_rn(v[3], __dmul_rn(d2, d2));
    if (x >= p10 && x <= p90) {
      v[4] = __dadd_rn(v[4], x);
      u[0]++;
    }
  }
  block_partial<5, 1>(v, u, false, part);
}

__global__ void seg_mid(const Partial* part, int nblocks, SegState* S) {
  if (S->n == 0) return;
  double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  unsigned long long nk = 0;
  for (int b = 0; b < nblocks; b++) {
    for (int k = 0; k < 5; k++) s[k] = __dadd_rn(s[k], part[b].s[k]);
    nk += part[b].u[0];
  }
  S->sabs = s[0]; S->s2 = s[1]; S->s3 = s[2]; S->s4 = s[3];
  S->nkept = nk;
  // nk may be 0 (n = 2 with distinct values: p10 > x[0] and p90 < x[1]); mean_kept and RobustMeanAbsoluteDeviation are
  // then 0 / 0 = NaN, as the reference's mean of an empty array
  S->mean_kept = __ddiv_rn(s[4], (double)nk);
}

// pass 4
__global__ void __launch_bounds__(SEG_NT) seg_pass4(SegArgs A, const SegState* S, Partial* part) {
  if (S->n == 0) return;
  const double mk = S->mean_kept, p10 = S->p10, p90 = S->p90;
  double v[1] = {0.0};
  unsigned long long u[1] = {0ull};
  for (long long i = (long long)blockIdx.x * SEG_NT + threadIdx.x; i < A.n; i += (long long)gridDim.x * SEG_NT) {
    if (!A.roi[i]) continue;
    const double x = load_f64(A.img, A.dtype, i);
    if (x >= p10 && x <= p90) v[0] = __dadd_rn(v[0], fabs(__dsub_rn(x, mk)));
  }
  block_partial<1, 1>(v, u, false, part);
}

// one block of SEG_NT threads: Entropy / Uniformity over the level bins (thread t sums bins t, t + SEG_NT, ..., then
// the fixed tree of block_partial), then thread 0 writes the 18 features in rb_firstorder_feature_name order
__global__ void __launch_bounds__(SEG_NT) seg_finish(const Partial* part, int nblocks, const SegState* S,
                                                     const unsigned long long* lhist, int nbins, double voxel_volume,
                                                     Partial* scratch, double* out) {
  if (S->n == 0) return;
  const double n = (double)S->n;
  const double eps = 2.220446049250313e-16;            // np.spacing(1)
  double v[2] = {0.0, 0.0};
  unsigned long long u[1] = {0ull};
  for (int l = threadIdx.x; l < nbins; l += SEG_NT) {
    if (!lhist[l]) continue;
    const double p = __ddiv_rn((double)lhist[l], n);
    v[0] = __dadd_rn(v[0], __dmul_rn(p, log2(__dadd_rn(p, eps))));
    v[1] = __dadd_rn(v[1], __dmul_rn(p, p));
  }
  block_partial<2, 1>(v, u, false, scratch);
  __syncthreads();
  if (threadIdx.x) return;
  const double ent = scratch[0].s[0], uni = scratch[0].s[1];
  double rmad = 0.0;
  for (int b = 0; b < nblocks; b++) rmad = __dadd_rn(rmad, part[b].s[0]);
  const double mn = key_f64(S->kmin), mx = key_f64(S->kmax);
  const double m2 = __ddiv_rn(S->s2, n), m3 = __ddiv_rn(S->s3, n), m4 = __ddiv_rn(S->s4, n);
  const double m2s = m2 == 0.0 ? 1.0 : m2;
  out[0] = S->p10;
  out[1] = S->p90;
  out[2] = S->energy;
  out[3] = -ent;
  out[4] = __dsub_rn(S->p75, S->p25);
  out[5] = __ddiv_rn(m4, __dmul_rn(m2s, m2s));
  out[6] = mx;
  out[7] = __ddiv_rn(S->sabs, n);
  out[8] = S->mean;
  out[9] = S->median;
  out[10] = mn;
  out[11] = __dsub_rn(mx, mn);
  out[12] = __ddiv_rn(rmad, (double)S->nkept);
  out[13] = sqrt(__ddiv_rn(S->energy, n));
  out[14] = __ddiv_rn(m3, pow(m2s, 1.5));
  out[15] = __dmul_rn(S->energy, voxel_volume);
  out[16] = uni;
  out[17] = m2;
}

}  // namespace

int firstorder_segment(const void* img, int dtype, const uint8_t* roi, const void* lev, int level_bytes, long long n,
                       double shift, double voxel_volume, double* out18_host, cudaStream_t st) {
  const int grid = grid_for(n, SEG_NT, 8);
  const int nbins = level_bytes == 1 ? 256 : 65536;
  // one workspace: state | level histogram | block partials
  const size_t off_hist = (sizeof(SegState) + 255) / 256 * 256;
  const size_t off_part = off_hist + sizeof(unsigned long long) * nbins;
  const size_t off_out = off_part + sizeof(Partial) * (grid + 1);      // + the finish block's partial
  DevBuf ws;
  RB_CUDA(ws.alloc(off_out + sizeof(double) * 18));
  char* base = ws.as<char>();
  SegState* S = (SegState*)base;
  unsigned long long* lhist = (unsigned long long*)(base + off_hist);
  Partial* part = (Partial*)(base + off_part);
  double* out = (double*)(base + off_out);
  RB_CUDA(cudaMemsetAsync(base, 0, off_part, st));
  const SegArgs A{img, dtype, roi, lev, level_bytes, n, shift};
  seg_pass1<<<grid, SEG_NT, 0, st>>>(A, part, lhist);
  seg_plan<<<1, 1, 0, st>>>(part, grid, S);
  for (int pass = 0; pass < 8; pass++) {
    seg_digits<<<grid, SEG_NT, 0, st>>>(A, S, pass);
    seg_pick<<<1, 1, 0, st>>>(S, pass);
  }
  seg_pass3<<<grid, SEG_NT, 0, st>>>(A, S, part);
  seg_mid<<<1, 1, 0, st>>>(part, grid, S);
  seg_pass4<<<grid, SEG_NT, 0, st>>>(A, S, part);
  seg_finish<<<1, SEG_NT, 0, st>>>(part, grid, S, lhist, nbins, voxel_volume, part + grid, out);
  RB_LAUNCH_CHECK();
  unsigned long long count = 0;
  cudaError_t e = cudaMemcpyAsync(out18_host, out, sizeof(double) * 18, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&count, &S->n, sizeof count, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) return fail(RB_ERR_CUDA, "firstorder segment: %s", cudaGetErrorString(e));
  if (count == 0) return fail(RB_ERR_ARG, "first order: the ROI is empty");
  return RB_OK;
}

}  // namespace rb

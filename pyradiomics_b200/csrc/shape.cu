// Segment-mode shape coefficients (SURVEY.md section 8f rank 4): the reference's
// cShape.calculate_coefficients (radiomics/src/cshape.c:22-242) as three kernels.
//
//   shape_mesh_kernel      one thread per 2x2x2 cube: corner configuration -> triangles from the
//                          generated table (mc_table.inc, see gen_mc_table.py), surface area and signed
//                          origin volume with the reference's formulas in absolute coordinates;
//                          per-block double reduction + one atomicAdd per block.  The same pass counts /
//                          emits the mesh vertices the reference keeps for the diameters: the three
//                          cube edges meeting at corner (z+1, y+1, x) -- every lattice edge belongs to
//                          exactly one cube, so no vertex is stored twice (cshape.c:94-112).
//   shape_diameter_kernel  all pairs of vertices, tiled through shared memory: the O(V^2) loop of
//                          calculate_meshDiameter (cshape.c:192-242).  Coordinates and squared
//                          distances are formed with exactly the reference's double operations, and a
//                          maximum does not depend on the visiting order, so the four diameters are
//                          bit-identical to the reference's.
//   shape_moments_kernel   exact integer first / second moments of the ROI voxel indices (the
//                          covariance behind the axis-length features, shape.py:86-95).
#include <stdint.h>
#include <string.h>

#include "common.cuh"
#include "mc_table.inc"

namespace rb {

__constant__ signed char c_mc_tri[256][16];
__constant__ signed char c_mc_mid2[12][3];
static bool g_tables_loaded[64] = {false};

static int shape_load_tables() {
  int dev = 0;
  RB_CUDA(cudaGetDevice(&dev));
  if (dev < 64 && g_tables_loaded[dev]) return RB_OK;
  RB_CUDA(cudaMemcpyToSymbol(c_mc_tri, MC_TRI, sizeof(MC_TRI)));
  RB_CUDA(cudaMemcpyToSymbol(c_mc_mid2, MC_EDGE_MID2, sizeof(MC_EDGE_MID2)));
  if (dev < 64) g_tables_loaded[dev] = true;
  return RB_OK;
}

struct ShapeAcc {
  double area, vol6;
  unsigned long long nverts;
};

// verts == nullptr: count only.  Vertex = (2z, 2y, 2x) half-index coordinates.
__global__ void __launch_bounds__(256)
shape_mesh_kernel(const uint8_t* __restrict__ mask, int Z, int Y, int X, long long sz, long long sy, long long sx,
                  double s0, double s1, double s2, ShapeAcc* __restrict__ acc, ushort4* __restrict__ verts,
                  unsigned long long* __restrict__ vcursor) {
  const long long ncubes = (long long)(Z - 1) * (Y - 1) * (X - 1);
  double area = 0, vol6 = 0;
  unsigned nv_local = 0;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < ncubes; t += (long long)gridDim.x * blockDim.x) {
    const int ix = (int)(t % (X - 1));
    const long long r = t / (X - 1);
    const int iy = (int)(r % (Y - 1)), iz = (int)(r / (Y - 1));
    const uint8_t* m = mask + iz * sz + iy * sy + ix * sx;
    unsigned cfg = 0;
#pragma unroll
    for (int c = 0; c < 8; c++)
      cfg |= (unsigned)(m[(c >> 2 & 1) * sz + (c >> 1 & 1) * sy + (c & 1) * sx] != 0) << c;
    // vertices owned by this cube: edges from corner (1,1,0) = bit 6 to (1,1,1) = 7, (1,0,0) = 4, (0,1,0) = 2
    const unsigned own = cfg >> 6 & 1u;
    const bool vx = (cfg >> 7 & 1u) != own, vy = (cfg >> 4 & 1u) != own, vz = (cfg >> 2 & 1u) != own;
    const unsigned nv = (unsigned)vx + vy + vz;
    if (nv) {
      if (verts) {
        unsigned long long at = atomicAdd(vcursor, (unsigned long long)nv);
        if (vx) verts[at++] = make_ushort4((unsigned short)(2 * iz + 2), (unsigned short)(2 * iy + 2), (unsigned short)(2 * ix + 1), 0);
        if (vy) verts[at++] = make_ushort4((unsigned short)(2 * iz + 2), (unsigned short)(2 * iy + 1), (unsigned short)(2 * ix), 0);
        if (vz) verts[at++] = make_ushort4((unsigned short)(2 * iz + 1), (unsigned short)(2 * iy + 2), (unsigned short)(2 * ix), 0);
      } else {
        nv_local += nv;
      }
    }
    if (verts || cfg == 0 || cfg == 255) continue;       // the fill pass only emits vertices
    for (int k = 0; k < 15 && c_mc_tri[cfg][k] >= 0; k += 3) {
      double p[3][3];
#pragma unroll
      for (int v = 0; v < 3; v++) {
        const int e = c_mc_tri[cfg][k + v];
        // (index + offset) * spacing, offset in {0, .5, 1}: the reference's vertex coordinates (cshape.c:125-137)
        p[v][0] = ((double)iz + 0.5 * c_mc_mid2[e][0]) * s0;
        p[v][1] = ((double)iy + 0.5 * c_mc_mid2[e][1]) * s1;
        p[v][2] = ((double)ix + 0.5 * c_mc_mid2[e][2]) * s2;
      }
      double* a = p[0]; double* b = p[1]; double* c = p[2];
      double ab0 = a[1] * b[2] - b[1] * a[2], ab1 = a[2] * b[0] - b[2] * a[0], ab2 = a[0] * b[1] - b[0] * a[1];
      vol6 += ab0 * c[0] + ab1 * c[1] + ab2 * c[2];
#pragma unroll
      for (int d = 0; d < 3; d++) { a[d] -= c[d]; b[d] -= c[d]; }
      ab0 = a[1] * b[2] - b[1] * a[2]; ab1 = a[2] * b[0] - b[2] * a[0]; ab2 = a[0] * b[1] - b[0] * a[1];
      area += 0.5 * sqrt(ab0 * ab0 + ab1 * ab1 + ab2 * ab2);
    }
  }
  if (verts) return;
  // block reduction (fixed tree: deterministic per block; blocks combine by atomicAdd)
  __shared__ double sa[256], sv[256];
  __shared__ unsigned sn[256];
  sa[threadIdx.x] = area; sv[threadIdx.x] = vol6; sn[threadIdx.x] = nv_local;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) { sa[threadIdx.x] += sa[threadIdx.x + h]; sv[threadIdx.x] += sv[threadIdx.x + h]; sn[threadIdx.x] += sn[threadIdx.x + h]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (sa[0] != 0) atomicAdd(&acc->area, sa[0]);
    if (sv[0] != 0) atomicAdd(&acc->vol6, sv[0]);
    if (sn[0]) atomicAdd(&acc->nverts, (unsigned long long)sn[0]);
  }
}

// out[0..3] (as ordered uint64 bit patterns of non-negative doubles): max squared distance among
// pairs with equal z, equal y, equal x coordinate, and among all pairs.
constexpr int DT = 256;
__global__ void __launch_bounds__(DT)
shape_diameter_kernel(const ushort4* __restrict__ verts, long long n, double s0, double s1, double s2,
                      unsigned long long* __restrict__ out) {
  __shared__ ushort4 tile[DT];
  __shared__ double tb[3][DT];
  const long long ntiles = (n + DT - 1) / DT;
  double best[4] = {0, 0, 0, 0};
  for (long long it = blockIdx.x; it < ntiles; it += gridDim.x) {
    const long long i = it * DT + threadIdx.x;
    const bool live = i < n;
    const ushort4 hv = live ? verts[i] : make_ushort4(0, 0, 0, 0);
    // explicit round-to-nearest products / sums: no FMA contraction, so every intermediate equals the
    // reference's (gcc, x86-64, no FMA) and the maxima are bit-identical
    const double a0 = __dmul_rn(0.5 * hv.x, s0), a1 = __dmul_rn(0.5 * hv.y, s1), a2 = __dmul_rn(0.5 * hv.z, s2);
    for (long long jt = 0; jt <= it; jt++) {              // unordered pairs: tiles jt <= it
      __syncthreads();
      const long long j = jt * DT + threadIdx.x;
      const ushort4 w = j < n ? verts[j] : make_ushort4(0xFFFF, 0xFFFF, 0xFFFF, 1);
      tile[threadIdx.x] = w;
      tb[0][threadIdx.x] = __dmul_rn(0.5 * w.x, s0); tb[1][threadIdx.x] = __dmul_rn(0.5 * w.y, s1); tb[2][threadIdx.x] = __dmul_rn(0.5 * w.z, s2);
      __syncthreads();
      if (!live) continue;
      const int kmax = (int)((jt + 1) * DT <= n ? DT : n - jt * DT);
#pragma unroll 4
      for (int k = 0; k < kmax; k++) {
        const ushort4 w2 = tile[k];
        const double d0 = __dsub_rn(a0, tb[0][k]), d1 = __dsub_rn(a1, tb[1][k]), d2 = __dsub_rn(a2, tb[2][k]);
        const double dist = __dadd_rn(__dadd_rn(__dmul_rn(d0, d0), __dmul_rn(d1, d1)), __dmul_rn(d2, d2));
        if (hv.x == w2.x) best[0] = fmax(best[0], dist);
        if (hv.y == w2.y) best[1] = fmax(best[1], dist);
        if (hv.z == w2.z) best[2] = fmax(best[2], dist);
        best[3] = fmax(best[3], dist);
      }
    }
  }
  __shared__ double red[4][DT];
  __syncthreads();
#pragma unroll
  for (int q = 0; q < 4; q++) red[q][threadIdx.x] = best[q];
  __syncthreads();
  for (int h = DT / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h)
#pragma unroll
      for (int q = 0; q < 4; q++) red[q][threadIdx.x] = fmax(red[q][threadIdx.x], red[q][threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x < 4) atomicMax(&out[threadIdx.x], (unsigned long long)__double_as_longlong(red[threadIdx.x][0]));
}

// sums over ROI voxels: {N, z, y, x, zz, zy, zx, yy, yx, xx}
__global__ void __launch_bounds__(256)
shape_moments_kernel(const uint8_t* __restrict__ mask, int Z, int Y, int X, unsigned long long* __restrict__ out) {
  const long long n = (long long)Z * Y * X;
  unsigned long long s[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    if (!mask[t]) continue;
    const unsigned long long x = (unsigned long long)(t % X), y = (unsigned long long)((t / X) % Y), z = (unsigned long long)(t / ((long long)X * Y));
    s[0] += 1; s[1] += z; s[2] += y; s[3] += x;
    s[4] += z * z; s[5] += z * y; s[6] += z * x; s[7] += y * y; s[8] += y * x; s[9] += x * x;
  }
  __shared__ unsigned long long red[256];
  for (int q = 0; q < 10; q++) {
    __syncthreads();
    red[threadIdx.x] = s[q];
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
      if ((int)threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
      __syncthreads();
    }
    if (threadIdx.x == 0 && red[0]) atomicAdd(&out[q], red[0]);
  }
}

// mask_dev: uint8 [Z][Y][X] with element strides (sz, sy, sx).  out7 (host): area, volume, the four
// diameters (equal-z, equal-y, equal-x, 3-D) and the number of mesh vertices.
int shape_coefficients_dev(const uint8_t* mask_dev, int Z, int Y, int X, long long sz, long long sy, long long sx,
                           const double* spacing, double* out7, cudaStream_t st) {
  for (int k = 0; k < 7; k++) out7[k] = 0;
  if (Z < 2 || Y < 2 || X < 2) return RB_OK;             // no cube: the reference's loops do not run
  if (Z > 32767 || Y > 32767 || X > 32767) return fail(RB_ERR_ARG, "shape: dimensions above 32767 are not supported");
  int rc = shape_load_tables();
  if (rc) return rc;
  struct Dev { ShapeAcc acc; unsigned long long cursor; unsigned long long dia[4]; };
  Dev* d = nullptr;
  RB_CUDA(cudaMalloc(&d, sizeof(Dev)));
  cudaMemsetAsync(d, 0, sizeof(Dev), st);
  const long long ncubes = (long long)(Z - 1) * (Y - 1) * (X - 1);
  const int grid = grid_for(ncubes, 256, 8);
  shape_mesh_kernel<<<grid, 256, 0, st>>>(mask_dev, Z, Y, X, sz, sy, sx, spacing[0], spacing[1], spacing[2], &d->acc, nullptr, nullptr);
  Dev h;
  cudaError_t e = cudaMemcpyAsync(&h, d, sizeof(Dev), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { cudaFree(d); return fail(RB_ERR_CUDA, "shape mesh pass: %s", cudaGetErrorString(e)); }
  out7[0] = h.acc.area; out7[1] = h.acc.vol6 / 6; out7[6] = (double)h.acc.nverts;
  if (h.acc.nverts) {
    ushort4* verts = nullptr;
    e = cudaMalloc(&verts, sizeof(ushort4) * h.acc.nverts);
    if (e != cudaSuccess) { cudaFree(d); return fail(RB_ERR_NOMEM, "shape: %llu mesh vertices do not fit", h.acc.nverts); }
    shape_mesh_kernel<<<grid, 256, 0, st>>>(mask_dev, Z, Y, X, sz, sy, sx, spacing[0], spacing[1], spacing[2], &d->acc, verts, &d->cursor);
    const long long nt = ((long long)h.acc.nverts + DT - 1) / DT;
    shape_diameter_kernel<<<grid_for(nt, 1, 8), DT, 0, st>>>(verts, (long long)h.acc.nverts, spacing[0], spacing[1], spacing[2], d->dia);
    e = cudaMemcpyAsync(&h, d, sizeof(Dev), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(verts);
    if (e != cudaSuccess) { cudaFree(d); return fail(RB_ERR_CUDA, "shape diameter pass: %s", cudaGetErrorString(e)); }
    for (int q = 0; q < 4; q++) {
      double v;
      memcpy(&v, &h.dia[q], 8);
      out7[2 + q] = sqrt(v);
    }
  }
  cudaFree(d);
  return RB_OK;
}

int shape_moments_dev(const uint8_t* mask_dev, int Z, int Y, int X, unsigned long long* out10, cudaStream_t st) {
  unsigned long long* d = nullptr;
  RB_CUDA(cudaMalloc(&d, 80));
  cudaMemsetAsync(d, 0, 80, st);
  shape_moments_kernel<<<grid_for((long long)Z * Y * X, 256, 8), 256, 0, st>>>(mask_dev, Z, Y, X, d);
  cudaError_t e = cudaMemcpyAsync(out10, d, 80, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  cudaFree(d);
  if (e != cudaSuccess) return fail(RB_ERR_CUDA, "shape moments: %s", cudaGetErrorString(e));
  return RB_OK;
}

// ---- 2-D shape coefficients (reference radiomics/src/cshape.c:420-595: calculate_coefficients2D + calculate_meshDiameter2D)
// Marching squares with edge-midpoint vertices over every 2x2 neighbourhood of the (zero-padded) mask.  What the reference
// gets from a 16-entry line table is stated geometrically here: a square with 1 or 3 inside corners is cut by ONE corner
// segment (length sqrt((sy/2)^2 + (sx/2)^2), inside area 1/8 or 7/8 of the pixel), two adjacent inside corners by a
// straight segment (length sx or sy, area 1/2), and the two diagonal cases by TWO corner segments that keep the inside
// corners apart (area 2/8; probed on the compiled reference: [[1,0],[0,1]] has surface 1.0).  The signed-triangle sum
// of the reference equals that area by Green's theorem; summing positive per-square areas instead avoids its cancellation.
// Mesh vertices for the diameter = midpoints of the crossed LEFT and BOTTOM square edges (each crossed grid edge once).
struct Shape2DAcc { double perimeter, area8; unsigned long long nverts; };

__global__ void __launch_bounds__(256)
shape2d_kernel(const uint8_t* __restrict__ mask, int Y, int X, long long sy_, long long sx_, double spy, double spx,
               Shape2DAcc* __restrict__ acc, ushort2* __restrict__ verts, unsigned long long* __restrict__ cursor) {
  const long long n = (long long)(Y - 1) * (X - 1);
  const double diag = sqrt(0.25 * spy * spy + 0.25 * spx * spx);
  double per = 0;
  long long a8 = 0;
  unsigned nv = 0;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    const int iy = (int)(t / (X - 1)), ix = (int)(t % (X - 1));
    const bool p0 = mask[iy * sy_ + ix * sx_] != 0, p1 = mask[iy * sy_ + (ix + 1) * sx_] != 0;
    const bool p3 = mask[(iy + 1) * sy_ + ix * sx_] != 0, p2 = mask[(iy + 1) * sy_ + (ix + 1) * sx_] != 0;
    const int cnt = p0 + p1 + p2 + p3;
    if (cnt == 0 || cnt == 4) { if (cnt == 4) a8 += 8; continue; }
    if (cnt == 1) { per += diag; a8 += 1; }
    else if (cnt == 3) { per += diag; a8 += 7; }
    else if (p0 == p2) { per += diag + diag; a8 += 2; }                 // diagonal pair: two separate corner cuts
    else { per += (p0 == p1) ? spx : spy; a8 += 4; }                    // top/bottom rows split: the cut runs along x
    // crossed left edge (p0 | p3) and bottom edge (p3 - p2): stored in half-index units (2*iy+1, 2*ix) / (2*iy+2, 2*ix+1)
    if (verts) {
      if (p0 != p3) verts[atomicAdd(cursor, 1ull)] = make_ushort2((unsigned short)(2 * iy + 1), (unsigned short)(2 * ix));
      if (p3 != p2) verts[atomicAdd(cursor, 1ull)] = make_ushort2((unsigned short)(2 * iy + 2), (unsigned short)(2 * ix + 1));
    } else {
      nv += (p0 != p3) + (p3 != p2);
    }
  }
  __shared__ double rp[256];
  __shared__ long long ra[256];
  __shared__ unsigned rn[256];
  rp[threadIdx.x] = per; ra[threadIdx.x] = a8; rn[threadIdx.x] = nv;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) { rp[threadIdx.x] += rp[threadIdx.x + h]; ra[threadIdx.x] += ra[threadIdx.x + h]; rn[threadIdx.x] += rn[threadIdx.x + h]; }
    __syncthreads();
  }
  if (threadIdx.x == 0 && !verts) {
    if (rp[0] != 0) atomicAdd(&acc->perimeter, rp[0]);
    if (ra[0]) atomicAdd(&acc->area8, (double)ra[0]);            // eighths of a pixel: exact in double
    if (rn[0]) atomicAdd(&acc->nverts, (unsigned long long)rn[0]);
  }
}

// largest squared distance over all vertex pairs; coordinates and products formed exactly like the reference
// ((index + offset) * spacing, difference, square, sum -- no FMA contraction), so the maximum is bit-identical
__global__ void __launch_bounds__(256)
shape2d_diameter_kernel(const ushort2* __restrict__ verts, long long n, double spy, double spx, unsigned long long* __restrict__ best) {
  __shared__ double ty[256], tx[256];
  double mx = 0;
  for (long long i0 = (long long)blockIdx.x * 256; i0 < n; i0 += (long long)gridDim.x * 256) {
    const long long i = i0 + threadIdx.x;
    const bool live = i < n;
    const ushort2 vi = verts[live ? i : 0];
    const double ay = __dmul_rn(0.5 * vi.x, spy), ax = __dmul_rn(0.5 * vi.y, spx);
    for (long long j0 = 0; j0 <= i0; j0 += 256) {
      __syncthreads();
      const long long j = j0 + threadIdx.x;
      const ushort2 vj = verts[j < n ? j : 0];
      ty[threadIdx.x] = __dmul_rn(0.5 * vj.x, spy); tx[threadIdx.x] = __dmul_rn(0.5 * vj.y, spx);
      __syncthreads();
      const int lim = (int)((n - j0) < 256 ? (n - j0) : 256);
      if (live)
        for (int k = 0; k < lim; k++) {
          const double dy = __dsub_rn(ay, ty[k]), dx = __dsub_rn(ax, tx[k]);
          const double d2 = __dadd_rn(__dmul_rn(dy, dy), __dmul_rn(dx, dx));
          mx = d2 > mx ? d2 : mx;
        }
    }
  }
  for (int o = 16; o; o >>= 1) { const double v = __shfl_xor_sync(0xffffffffu, mx, o); mx = v > mx ? v : mx; }
  if ((threadIdx.x & 31) == 0 && mx > 0) atomicMax(best, (unsigned long long)__double_as_longlong(mx));   // positive doubles order like integers
}

// mask_dev: uint8 [Y][X] with element strides (sy, sx) -- already zero-padded by the caller like the reference does
// (shape2D.py:93); out4 (host) = perimeter, surface, maximum diameter, number of mesh vertices
int shape2d_coefficients_dev(const uint8_t* mask_dev, int Y, int X, long long sy, long long sx, const double* spacing, double* out4,
                             cudaStream_t st) {
  for (int k = 0; k < 4; k++) out4[k] = 0;
  if (Y < 2 || X < 2) return RB_OK;
  if (Y > 32767 || X > 32767) return fail(RB_ERR_ARG, "shape2D: dimensions above 32767 are not supported");
  struct Dev { Shape2DAcc acc; unsigned long long cursor, best; };
  Dev* d = nullptr;
  RB_CUDA(cudaMalloc(&d, sizeof(Dev)));
  cudaMemsetAsync(d, 0, sizeof(Dev), st);
  const long long nsq = (long long)(Y - 1) * (X - 1);
  const int grid = grid_for(nsq, 256, 8);
  shape2d_kernel<<<grid, 256, 0, st>>>(mask_dev, Y, X, sy, sx, spacing[0], spacing[1], &d->acc, nullptr, nullptr);
  Dev h;
  cudaError_t e = cudaMemcpyAsync(&h, d, sizeof(Dev), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) { cudaFree(d); return fail(RB_ERR_CUDA, "shape2D pass: %s", cudaGetErrorString(e)); }
  out4[0] = h.acc.perimeter;
  out4[1] = h.acc.area8 * 0.125 * spacing[0] * spacing[1];
  out4[3] = (double)h.acc.nverts;
  if (h.acc.nverts) {
    ushort2* verts = nullptr;
    e = cudaMalloc(&verts, sizeof(ushort2) * h.acc.nverts);
    if (e != cudaSuccess) { cudaFree(d); return fail(RB_ERR_NOMEM, "shape2D: %llu vertices do not fit", h.acc.nverts); }
    shape2d_kernel<<<grid, 256, 0, st>>>(mask_dev, Y, X, sy, sx, spacing[0], spacing[1], &d->acc, verts, &d->cursor);
    const long long nt = ((long long)h.acc.nverts + 255) / 256;
    shape2d_diameter_kernel<<<grid_for(nt, 1, 8), 256, 0, st>>>(verts, (long long)h.acc.nverts, spacing[0], spacing[1], &d->best);
    e = cudaMemcpyAsync(&h, d, sizeof(Dev), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    cudaFree(verts);
    if (e != cudaSuccess) { cudaFree(d); return fail(RB_ERR_CUDA, "shape2D diameter pass: %s", cudaGetErrorString(e)); }
    double v;
    memcpy(&v, &h.best, 8);
    out4[2] = sqrt(v);
  }
  cudaFree(d);
  return RB_OK;
}

}  // namespace rb

// Wide voxel texture kernel: windows of 344 to 3375 positions (kernelRadius 4 to 7 in 3-D, larger force2D / 2-D
// windows), where one thread per centre (voxel_kernels.cu) would need tens of KB of local arrays.  One block owns one
// centre at a time and loops over the chunk's centres:
//   1. the block stages the window's levels in shared memory (load_window's clipped box: 0 outside the volume / ROI);
//   2. block_compact_levels (wide_window.cuh) gives compact_levels' val / lidx;
//   3. the class body runs the generic kernel's own builders and per-matrix functions (vox_features.cuh) on a per-block
//      global workspace instead of local arrays: GLCM and GLRLM one thread per angle, then one thread takes the angle
//      means in angle order as glcm_voxel / glrlm_voxel do; weighted GLCM, GLSZM, GLDM and NGTDM one thread.
// Each entry list is built by the same Entries::add sequence as the generic kernel's, so its entries, their order and
// every floating-point sum are the generic kernel's: the maps are bit-identical wherever both run
// (B200_RADIOMICS_FORCE_WIDE=1 sends windows <= 343 here to show it).
#include "common.cuh"
#include "vox_features.cuh"
#include "voxel_tiles.cuh"
#include "wide_window.cuh"

namespace rb {

constexpr int WIDE_NT = 64;
// > the longest line of any window of <= WIDE_WCAP_MAX positions (57: a 57 x 57 force2D plane)
constexpr int WIDE_RLCAP = 64;
constexpr int WIDE_NJCAP = 32;           // the generic kernel's dense MCC solve (NJCAP for windows over 27 positions)
constexpr long long WIDE_WS_MAX = 1ll << 30;   // workspace bytes per launch; the grid shrinks to stay below

// the sizes of one launch's workspace
struct WideLayout {
  int cls, wn, ncap;   // class, window positions, levels a window can hold (min(wn, Ng))
  int ecap, kcap;      // an angle's / the class body's entry list; GLCM's |i-j| and i+j lists
  int ewcap;           // weighted GLRLM's pooled list
  int slots;           // angle slots per block
  long long slot_bytes, block_bytes;
};

// 8-byte aligned pieces of a byte range; from address 0 it measures
struct Carve {
  uintptr_t p;
  template <typename T>
  __host__ __device__ T* take(long long n) {
    T* r = (T*)p;
    p += (uintptr_t)((n * (long long)sizeof(T) + 7) / 8 * 8);
    return r;
  }
};

// one angle slot: its entry list and the arrays its class's per-matrix function needs
struct WideSlot {
  uint32_t* ekey;
  double* ew;          // int lists use the first 4 bytes of each entry
  GlcmScratch g;       // GLCM
  double *pr, *pg;     // GLRLM
  double* pj;          // GLSZM / GLDM
  uint16_t* stack;     // GLSZM
  double *cnt, *s;     // NGTDM
};

__host__ __device__ inline WideSlot carve_slot(Carve& c, const WideLayout& L) {
  WideSlot S = {};
  S.ekey = c.take<uint32_t>(L.ecap);
  S.ew = c.take<double>(L.ecap);
  if (L.cls == C_GLCM) {
    S.g.px = c.take<double>(L.ncap); S.g.py = c.take<double>(L.ncap);
    S.g.D.key = c.take<uint32_t>(L.kcap); S.g.D.w = c.take<double>(L.kcap); S.g.D.cap = L.kcap;
    S.g.Sm.key = c.take<uint32_t>(L.kcap); S.g.Sm.w = c.take<double>(L.kcap); S.g.Sm.cap = L.kcap;
    S.g.ridx = c.take<uint16_t>(L.ncap); S.g.cidx = c.take<uint16_t>(L.ncap); S.g.parent = c.take<uint16_t>(2 * L.ncap);
    S.g.A = c.take<double>(WIDE_NJCAP * WIDE_NJCAP); S.g.dd = c.take<double>(WIDE_NJCAP); S.g.ee = c.take<double>(WIDE_NJCAP);
  } else if (L.cls == C_GLRLM) {
    S.pr = c.take<double>(WIDE_RLCAP); S.pg = c.take<double>(L.ncap);
  } else if (L.cls == C_GLSZM || L.cls == C_GLDM) {
    S.pj = c.take<double>((L.wn > NA_MAX + 1 ? L.wn : NA_MAX + 1) + 1); S.pg = c.take<double>(L.ncap);
    if (L.cls == C_GLSZM) S.stack = c.take<uint16_t>(L.wn);
  } else {
    S.cnt = c.take<double>(L.ncap); S.s = c.take<double>(L.ncap);
  }
  return S;
}

// the block's own arrays after its slots: every angle's features, ok flag and status bits, weighted GLRLM's pool
struct WideBlock {
  double* res;
  int *ok, *ast;
  uint32_t* ewkey;
  double* eww;
};

__host__ __device__ inline WideBlock carve_block(Carve& c, const WideLayout& L, int na) {
  WideBlock B;
  B.res = c.take<double>((long long)na * GLCM_NF);
  B.ok = c.take<int>(na); B.ast = c.take<int>(na);
  B.ewkey = c.take<uint32_t>(L.ewcap); B.eww = c.take<double>(L.ewcap);
  return B;
}

template <typename W>
__device__ __forceinline__ EntryList<W> slot_list(const WideSlot& S, int cap) {
  EntryList<W> E;
  E.key = S.ekey; E.w = (W*)S.ew; E.cap = cap; E.n = 0; E.overflow = false;
  return E;
}

template <typename T, int CLS, bool WEIGHTED, typename OutT>
__global__ void __launch_bounds__(WIDE_NT)
wide_voxel_kernel(const T* __restrict__ lev, const uint8_t* __restrict__ centers, const __grid_constant__ VoxParams P,
                  const WideLayout L, uint8_t* __restrict__ ws, OutT* __restrict__ out, long long fstride, int z0,
                  int z1, int out_z0, int* __restrict__ status) {
  constexpr int NF = CLS == C_GLCM ? GLCM_NF : CLS == C_GLRLM ? GLRLM_NF : CLS == C_GLSZM ? GLSZM_NF
                     : CLS == C_GLDM ? GLDM_NF : NGTDM_NF;
  extern __shared__ __align__(8) uint8_t smem[];
  const WinGeom G(P);
  const int wn = G.n, tid = threadIdx.x;
  int* val = (int*)smem;
  int* fq = val + wn;
  uint16_t* w = (uint16_t*)(fq + wn);
  uint16_t* lidx = w + wn;
  __shared__ double s_f[GLCM_NF];
  __shared__ int s_n, s_st;

  const uintptr_t base = (uintptr_t)ws + (uintptr_t)blockIdx.x * (uintptr_t)L.block_bytes;
  Carve cs{base + (uintptr_t)tid * (uintptr_t)L.slot_bytes};
  const WideSlot S = carve_slot(cs, L);        // this thread's angle slot (tid < L.slots)
  Carve cb{base + (uintptr_t)L.slots * (uintptr_t)L.slot_bytes};
  const WideBlock B = carve_block(cb, L, P.na);

  const long long plane = (long long)P.Y * P.X;
  const long long total = (long long)(z1 - z0) * plane;
  for (long long t = blockIdx.x; t < total; t += gridDim.x) {        // block-uniform
    const ChunkVoxel v = chunk_voxel(P, plane, z0, out_z0, t);
    if (!chunk_center(lev, centers, plane, v)) {
      if (tid < NF) store_map(out + tid * fstride + v.oi, P.init_value);
      continue;
    }
    for (int p = tid; p < wn; p += WIDE_NT) {
      const WindowOffset o(p, P.rz, P.ry, P.rx);
      const int z = v.z + o.dz, y = v.y + o.dy, x = v.x + o.dx;
      const bool in = z >= 0 && z < P.Z && y >= 0 && y < P.Y && x >= 0 && x < P.X;
      w[p] = in ? (uint16_t)lev[(long long)z * P.sz + (long long)y * P.sy + x] : (uint16_t)0;
    }
    if (tid == 0) s_st = 0;
    __syncthreads();
    const int n = block_compact_levels(w, wn, val, lidx, fq, s_n);
    if (n > L.ncap) {
      // more levels than Ng allows (a level outside 1..Ng): the workspace is sized for Ng
      if (tid < NF) store_map(out + tid * fstride + v.oi, NAN);
      if (tid == 0 && status) atomicOr(status, 2);
      __syncthreads();
      continue;
    }
    if (CLS == C_GLCM && !WEIGHTED) {
      for (int a0 = 0; a0 < P.na; a0 += L.slots) {
        const int a = a0 + tid;
        if (tid < L.slots && a < P.na) {
          Entries<0, int> E;
          static_cast<EntryList<int>&>(E) = slot_list<int>(S, L.ecap);
          E.ws = const_cast<GlcmScratch*>(&S.g);
          glcm_angle_entries(lidx, G, P, a, 1, E);
          int ast = 0;
          B.ok[a] = glcm_angle_features<0, 1, WIDE_NJCAP, int>(E, n, val, P, B.res + a * GLCM_NF, &ast);
          B.ast[a] = ast;
        }
      }
      __syncthreads();
      if (tid == 0) {                        // glcm_voxel's angle mean, in angle order
        double sum[GLCM_NF]; int cnt[GLCM_NF];
        for (int k = 0; k < GLCM_NF; k++) { sum[k] = 0; cnt[k] = 0; }
        bool ja_nan = false, mcc_nan = false;
        int st = 0;
        for (int a = 0; a < P.na; a++) {
          st |= B.ast[a];
          if (B.ast[a] & 1) mcc_nan = true;
          if (!B.ok[a]) { if (P.alive[a >> 5] >> (a & 31) & 1u) ja_nan = true; continue; }
          angle_mean_add<GLCM_NF>(B.res + a * GLCM_NF, sum, cnt);
        }
        for (int k = 0; k < GLCM_NF; k++) s_f[k] = cnt[k] ? sum[k] / cnt[k] : NAN;
        if (ja_nan) s_f[G_JointAverage] = NAN;
        if (mcc_nan) s_f[G_MCC] = NAN;
        s_st = st;
      }
    } else if (CLS == C_GLCM) {
      if (tid == 0) {                        // glcm_voxel's weighted body: every angle pooled into one list
        Entries<0, double> E;
        static_cast<EntryList<double>&>(E) = slot_list<double>(S, L.ecap);
        E.ws = const_cast<GlcmScratch*>(&S.g);
        for (int a = 0; a < P.na; a++) glcm_angle_entries(lidx, G, P, a, P.wgt[a], E);
        double f[GLCM_NF];
        int st = 0;
        bool ok = glcm_angle_features<0, 1, WIDE_NJCAP, double>(E, n, val, P, f, &st);
        if (E.overflow) { ok = false; st |= 2; }
        for (int k = 0; k < GLCM_NF; k++) s_f[k] = ok ? f[k] : NAN;
        s_st = st;
      }
    } else if (CLS == C_GLRLM) {
      for (int a0 = 0; a0 < P.na; a0 += L.slots) {
        const int a = a0 + tid;
        if (tid < L.slots && a < P.na) {
          EntryList<int> E = slot_list<int>(S, L.ecap);
          const bool multi = glrlm_angle_runs(lidx, G, P, a, E);
          if (WEIGHTED) {
            B.ok[a] = multi;
            B.ast[a] = E.n;                  // the list stays in the slot for the pooling below
          } else {
            B.ok[a] = multi && glrlm_angle_features_on<WIDE_RLCAP>(E, n, val, B.res + a * GLCM_NF, S.pr, S.pg);
          }
        }
      }
      __syncthreads();
      if (tid == 0) {
        if (WEIGHTED) {                      // glrlm_voxel's pool: angle by angle, each list in its order
          EntryList<double> EW;
          EW.key = B.ewkey; EW.w = B.eww; EW.cap = L.ewcap; EW.clear();
          for (int a = 0; a < P.na; a++) {
            if (!B.ok[a]) continue;
            Carve ca{base + (uintptr_t)a * (uintptr_t)L.slot_bytes};
            const WideSlot Sa = carve_slot(ca, L);
            const int* wa = (const int*)Sa.ew;
            for (int e = 0; e < B.ast[a]; e++) EW.add(Sa.ekey[e], P.wgt[a] * wa[e]);
          }
          double f[GLRLM_NF];
          const bool ok = glrlm_angle_features_on<WIDE_RLCAP>(EW, n, val, f, S.pr, S.pg);
          for (int k = 0; k < GLRLM_NF; k++) s_f[k] = ok ? f[k] : NAN;
        } else {                             // glrlm_voxel's angle mean
          double sum[GLRLM_NF]; int cnt[GLRLM_NF];
          for (int k = 0; k < GLRLM_NF; k++) { sum[k] = 0; cnt[k] = 0; }
          for (int a = 0; a < P.na; a++)
            if (B.ok[a]) angle_mean_add<GLRLM_NF>(B.res + a * GLCM_NF, sum, cnt);
          for (int k = 0; k < GLRLM_NF; k++) s_f[k] = cnt[k] ? sum[k] / cnt[k] : NAN;
        }
      }
    } else if (tid == 0) {
      if (CLS == C_GLSZM) {
        EntryList<int> E = slot_list<int>(S, L.ecap);
        glszm_zones(lidx, G, P, S.stack, E);
        double f[SIZE_NF];
        size_matrix_features_on(E, n, val, f, wn, S.pj, S.pg);
        for (int k = 0; k < GLSZM_NF; k++) s_f[k] = f[k];
      } else if (CLS == C_GLDM) {
        EntryList<int> E = slot_list<int>(S, L.ecap);
        gldm_entries(lidx, val, G, P, E);
        double f[SIZE_NF];
        size_matrix_features_on(E, n, val, f, NA_MAX + 1, S.pj, S.pg);
        gldm_from_size(f, s_f);
      } else {
        ngtdm_window(lidx, val, n, G, P, S.cnt, S.s, s_f);
      }
    }
    __syncthreads();
    if (tid < NF) store_map(out + tid * fstride + v.oi, s_f[tid]);
    if (tid == 0 && s_st && status) atomicOr(status, s_st);
    __syncthreads();
  }
}

static WideLayout wide_layout(int cls, const VoxParams& P) {
  WideLayout L = {};
  L.cls = cls;
  L.wn = window_capacity(P);
  L.ncap = L.wn < P.Ng ? L.wn : P.Ng;
  const long long pairs = (long long)L.ncap * L.ncap;
  const int wcap = window_class(L.wn);            // the generic kernel's class: its semantic list limits follow it
  if (cls == C_GLCM && P.weighted) {
    L.ecap = wcap <= 27 ? wcap * wcap : 2048;                  // glcm_voxel's ECAP and KCAP: overflow is status bit 1
    L.kcap = L.ecap < 1024 ? L.ecap : 1024;
  } else if (cls == C_GLCM) {
    L.ecap = (int)(2ll * L.wn < pairs ? 2ll * L.wn : pairs);  // every distinct (i, j) of the window: no overflow
    L.kcap = L.ecap < 2 * P.Ng ? L.ecap : 2 * P.Ng;            // every distinct |i - j| and i + j
  } else {
    L.ecap = L.wn;                                             // runs, zones, voxels: at most one entry per position
  }
  L.ewcap = cls == C_GLRLM && P.weighted ? wcap : 0;           // glrlm_voxel's pooled Entries<WCAP>
  L.slots = (cls == C_GLCM && !P.weighted) || cls == C_GLRLM ? (P.na < WIDE_NT ? P.na : WIDE_NT) : 1;
  Carve c{0};
  carve_slot(c, L);
  L.slot_bytes = (long long)c.p;
  Carve b{0};
  carve_block(b, L, P.na);
  L.block_bytes = L.slots * L.slot_bytes + (long long)b.p;
  return L;
}

// one resident wave of blocks (the occupancy at this window's shared memory), at most one block per centre, and no
// more than WIDE_WS_MAX bytes of workspace
template <typename K>
static int wide_grid(K* kernel, int smem, long long total, long long block_bytes, int& grid) {
  int per_sm = 0;
  RB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, WIDE_NT, smem));
  long long g = (long long)sm_count() * (per_sm > 0 ? per_sm : 1);
  if (g > total) g = total;
  const long long by_ws = block_bytes > 0 ? WIDE_WS_MAX / block_bytes : g;
  if (g > by_ws) g = by_ws;
  grid = (int)(g < 1 ? 1 : g);
  return RB_OK;
}

int voxel_features_wide(const VoxLaunch& A) {
  const VoxParams& P = A.P;
  const long long total = (long long)(A.z1 - A.z0) * P.Y * P.X;
  return with_level_type(A.level_bytes, [&](auto lt) -> int {
    return with_map_type(A.out_f32, [&](auto ot) -> int {
      using T = decltype(lt);
      using OutT = decltype(ot);
      if (total <= 0) return RB_OK;
      const WideLayout L = wide_layout(A.cls, P);
      const int smem = 12 * L.wn;
      auto launch = [&](auto kernel) -> int {
        int grid = 0;
        if (int rc = wide_grid(kernel, smem, total, L.block_bytes, grid)) return rc;
        std::unique_lock<std::mutex> lk;    // held until the kernel is enqueued
        StreamScratch* S = stream_scratch(A.st, lk);
        if (!S || !S->grow(S->wide, (size_t)grid * L.block_bytes))
          return fail(RB_ERR_NOMEM, "could not allocate the wide voxel kernel's workspace (%lld bytes)",
                      (long long)grid * L.block_bytes);
        kernel<<<grid, WIDE_NT, smem, A.st>>>((const T*)A.lev, A.centers, P, L, S->wide.as<uint8_t>(), (OutT*)A.out,
                                              A.fstride, A.z0, A.z1, A.out_z0, A.status);
        RB_LAUNCH_CHECK();
        return RB_OK;
      };
      const bool wgt = P.weighted != 0;
      switch (A.cls) {
        case C_GLCM: return wgt ? launch(wide_voxel_kernel<T, C_GLCM, true, OutT>) : launch(wide_voxel_kernel<T, C_GLCM, false, OutT>);
        case C_GLRLM: return wgt ? launch(wide_voxel_kernel<T, C_GLRLM, true, OutT>) : launch(wide_voxel_kernel<T, C_GLRLM, false, OutT>);
        case C_GLSZM: return launch(wide_voxel_kernel<T, C_GLSZM, false, OutT>);
        case C_GLDM: return launch(wide_voxel_kernel<T, C_GLDM, false, OutT>);
        case C_NGTDM: return launch(wide_voxel_kernel<T, C_NGTDM, false, OutT>);
        default: return fail(RB_ERR_ARG, "unknown texture class %d", A.cls);
      }
    });
  });
}

}  // namespace rb

// Host build of the 2-D LBP per-pixel arithmetic (pyradiomics_b200/csrc/lbp2d.cuh) for tests/test_lbp2d_cpu.py: the same
// lbp2d_slice_of / lbp2d_pixel the CUDA kernel runs, over every voxel of a volume in memory order.  Build with
// -ffp-contract=off: the device spells every operation as a separately rounded __d*_rn.
#include "../../pyradiomics_b200/csrc/lbp2d.cuh"

template <int M>
static void run(const void* img, int dt, int Z, int Y, int X, int axis, const rb::Lbp2dOffsets& O, double* out) {
  for (int z = 0; z < Z; z++)
    for (int y = 0; y < Y; y++)
      for (int x = 0; x < X; x++) {
        rb::Lbp2dSlice s;
        int r, c;
        rb::lbp2d_slice_of(img, dt, Z, Y, X, axis, z, y, x, s, r, c);
        out[((long long)z * Y + y) * X + x] = rb::lbp2d_pixel<M>(s, r, c, O);
      }
}

// lbp2d_code of n sign-bit patterns (the integer methods)
extern "C" void lbp2d_codes_emul(int method, int P, const uint32_t* bits, long long n, double* out) {
  for (long long i = 0; i < n; i++) out[i] = rb::lbp2d_code(method, bits[i], P);
}

extern "C" int lbp2d_emul(const void* img, int dt, int Z, int Y, int X, int axis, int P, const double* rp, const double* cp,
                          int method, double* out) {
  if (P < 1 || P > rb::LBP2D_MAX_P) return -5;
  rb::Lbp2dOffsets O;
  O.P = P;
  O.pad_ = 0;
  for (int k = 0; k < rb::LBP2D_MAX_P; k++) {
    O.rp[k] = k < P ? rp[k] : 0.0;
    O.cp[k] = k < P ? cp[k] : 0.0;
  }
  switch (method) {
    case rb::LBP2D_DEFAULT: run<rb::LBP2D_DEFAULT>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_ROR: run<rb::LBP2D_ROR>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_UNIFORM: run<rb::LBP2D_UNIFORM>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_NRI_UNIFORM: run<rb::LBP2D_NRI_UNIFORM>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_VAR: run<rb::LBP2D_VAR>(img, dt, Z, Y, X, axis, O, out); break;
    default: return -3;
  }
  return 0;
}

// Host build of the 2-D LBP store in the image's own dtype (pyradiomics_b200/csrc/lbp2d.cuh: numpy_cast, and the
// lbp2d_pixel -> numpy_cast<T> of lbp2d_kernel<METHOD, T>) for tests/test_lbp2d_pipeline_cpu.py.  Build with
// -ffp-contract=off: the device spells every operation as a separately rounded __d*_rn.
#include "../../pyradiomics_b200/csrc/lbp2d.cuh"

template <typename T>
static void cast_n(const double* v, long long n, void* out) {
  for (long long i = 0; i < n; i++) ((T*)out)[i] = rb::numpy_cast<T>(v[i]);
}

// numpy_cast<T> of n values, T the rb_dtype `dt`
extern "C" int numpy_cast_emul(int dt, const double* v, long long n, void* out) {
  switch (dt) {
    case RB_DT_INT16: cast_n<int16_t>(v, n, out); break;
    case RB_DT_INT32: cast_n<int32_t>(v, n, out); break;
    case RB_DT_FLOAT32: cast_n<float>(v, n, out); break;
    case RB_DT_FLOAT64: cast_n<double>(v, n, out); break;
    case RB_DT_UINT8: cast_n<uint8_t>(v, n, out); break;
    case RB_DT_UINT16: cast_n<uint16_t>(v, n, out); break;
    case RB_DT_INT64: cast_n<int64_t>(v, n, out); break;
    default: return -3;
  }
  return 0;
}

template <int M, typename T>
static void run(const void* img, int dt, int Z, int Y, int X, int axis, const rb::Lbp2dOffsets& O, void* out) {
  for (int z = 0; z < Z; z++)
    for (int y = 0; y < Y; y++)
      for (int x = 0; x < X; x++) {
        rb::Lbp2dSlice s;
        int r, c;
        rb::lbp2d_slice_of(img, dt, Z, Y, X, axis, z, y, x, s, r, c);
        ((T*)out)[((long long)z * Y + y) * X + x] = rb::numpy_cast<T>(rb::lbp2d_pixel<M>(s, r, c, O));
      }
}

template <typename T>
static int run_method(const void* img, int dt, int Z, int Y, int X, int axis, const rb::Lbp2dOffsets& O, int method, void* out) {
  switch (method) {
    case rb::LBP2D_DEFAULT: run<rb::LBP2D_DEFAULT, T>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_ROR: run<rb::LBP2D_ROR, T>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_UNIFORM: run<rb::LBP2D_UNIFORM, T>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_NRI_UNIFORM: run<rb::LBP2D_NRI_UNIFORM, T>(img, dt, Z, Y, X, axis, O, out); break;
    case rb::LBP2D_VAR: run<rb::LBP2D_VAR, T>(img, dt, Z, Y, X, axis, O, out); break;
    default: return -3;
  }
  return 0;
}

// the LBP volume of `img` stored in its own dtype `dt`, what rb_lbp2d_cast_dev writes
extern "C" int lbp2d_cast_emul(const void* img, int dt, int Z, int Y, int X, int axis, int P, const double* rp, const double* cp,
                               int method, void* out) {
  if (P < 1 || P > rb::LBP2D_MAX_P) return -5;
  rb::Lbp2dOffsets O;
  O.P = P;
  O.pad_ = 0;
  for (int k = 0; k < rb::LBP2D_MAX_P; k++) {
    O.rp[k] = k < P ? rp[k] : 0.0;
    O.cp[k] = k < P ? cp[k] : 0.0;
  }
  switch (dt) {
    case RB_DT_INT16: return run_method<int16_t>(img, dt, Z, Y, X, axis, O, method, out);
    case RB_DT_INT32: return run_method<int32_t>(img, dt, Z, Y, X, axis, O, method, out);
    case RB_DT_FLOAT32: return run_method<float>(img, dt, Z, Y, X, axis, O, method, out);
    case RB_DT_FLOAT64: return run_method<double>(img, dt, Z, Y, X, axis, O, method, out);
    case RB_DT_UINT8: return run_method<uint8_t>(img, dt, Z, Y, X, axis, O, method, out);
    case RB_DT_UINT16: return run_method<uint16_t>(img, dt, Z, Y, X, axis, O, method, out);
    case RB_DT_INT64: return run_method<int64_t>(img, dt, Z, Y, X, axis, O, method, out);
    default: return -3;
  }
}

// The pixel types of include/b200radiomics.h (rb_dtype) on the device and in the host builds of the per-voxel headers:
// one loader and one validity check.  Plain C++ without CUDA headers, so that g++ compiles it (tests/host_emul).
#pragma once
#include <stdint.h>

#include "../../include/b200radiomics.h"

#ifndef RB_HD
#ifdef __CUDACC__
#define RB_HD __host__ __device__ __forceinline__
#else
#define RB_HD inline
#endif
#endif

namespace rb {

RB_HD bool dtype_valid(int dt) { return dt >= RB_DT_INT16 && dt <= RB_DT_INT64; }

// element i of an array of pixel type dt, as float64 (dt must be valid: anything else reads int64)
RB_HD double load_f64(const void* p, int dt, long long i) {
  switch (dt) {
    case RB_DT_INT16: return (double)((const int16_t*)p)[i];
    case RB_DT_INT32: return (double)((const int32_t*)p)[i];
    case RB_DT_FLOAT32: return (double)((const float*)p)[i];
    case RB_DT_FLOAT64: return ((const double*)p)[i];
    case RB_DT_UINT8: return (double)((const uint8_t*)p)[i];
    case RB_DT_UINT16: return (double)((const uint16_t*)p)[i];
    default: return (double)((const long long*)p)[i];
  }
}

}  // namespace rb

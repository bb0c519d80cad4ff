// common.cuh — shared helpers for the sm_90a kernels behind include/tio_b200.h
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/tio_b200.h"

namespace tio {

// thread-local error message (tio_last_error)
void set_error(const char* fmt, ...);

// thread-local count of kernels launched (tio_launch_count): every kernel launch in csrc/ is
// followed by launched()
extern thread_local uint64_t g_launches;
inline void launched() { ++g_launches; }

#define TIO_CHECK_ARG(cond, ...)       \
  do {                                 \
    if (!(cond)) {                     \
      ::tio::set_error(__VA_ARGS__);   \
      return 1;                        \
    }                                  \
  } while (0)

#define TIO_CHECK_CUDA(expr)                                              \
  do {                                                                    \
    cudaError_t err__ = (expr);                                           \
    if (err__ != cudaSuccess) {                                           \
      ::tio::set_error("%s failed: %s", #expr, cudaGetErrorString(err__)); \
      return 2;                                                           \
    }                                                                     \
  } while (0)

#define TIO_CHECK_LAUNCH()                                                   \
  do {                                                                       \
    cudaError_t err__ = cudaGetLastError();                                  \
    if (err__ != cudaSuccess) {                                              \
      ::tio::set_error("kernel launch failed: %s", cudaGetErrorString(err__)); \
      return 3;                                                              \
    }                                                                        \
  } while (0)

// switch over the label dtypes of tio_dtype: F(T) for the element type T
#define TIO_LABEL_DISPATCH(dtype, name, F)                          \
  switch (dtype) {                                                  \
    case TIO_F32: F(float); break;                                  \
    case TIO_U8: F(uint8_t); break;                                 \
    case TIO_I8: F(int8_t); break;                                  \
    case TIO_I16: F(int16_t); break;                                \
    case TIO_I32: F(int32_t); break;                                \
    case TIO_I64: F(int64_t); break;                                \
    default: TIO_CHECK_ARG(false, name ": unknown dtype %d", dtype); \
  }

// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe), read once per
// device: the grid caps scale with it
int num_sms();

// ---- align_corners=True linear-upsample index/weights (ATen semantics) -----
// scale = (n_in-1)/(n_out-1) in fp32 (precomputed on the host with the same
// fp32 division), real = scale*o, i0 = floor, i1 = i0 + (i0 < n_in-1),
// l1 = real - i0, l0 = 1 - l1.  When n_in == n_out ATen short-circuits to
// (o, o, 1, 0); the host encodes that as scale = 1 (exact same result:
// real = o, l1 = 0, l0 = 1; v1 weight 0 so i1 is irrelevant bit-wise... except
// 0*v1 must not be NaN/Inf — control grids are finite).
struct LerpAxis {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ LerpAxis lerp_axis(float scale, int n_in, int o) {
  LerpAxis r;
  float real = __fmul_rn(scale, (float)o);
  int a = (int)floorf(real);
  a = min(a, n_in - 1);
  float lam = __fsub_rn(real, (float)a);
  lam = fminf(fmaxf(lam, 0.0f), 1.0f);
  r.i0 = a;
  r.i1 = a + (a < n_in - 1 ? 1 : 0);
  r.l1 = lam;
  r.l0 = __fsub_rn(1.0f, lam);
  return r;
}

// ATen's 2-tap combine as compiled in torch 2.11 CPU: fma(w0, v0, rn(w1*v1)).
__device__ __forceinline__ float lerp2(float w0, float v0, float w1, float v1) {
  return __fmaf_rn(w0, v0, __fmul_rn(w1, v1));
}

}  // namespace tio

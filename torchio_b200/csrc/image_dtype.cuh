// image_dtype.cuh — element types of image volumes (every tio_dtype code) and the conversions the
// reference's `data.float()` ... `.to(dtype)` make on CUDA; shared by interpolate.cu and stats.cu
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"

namespace tio {

// fp16 / bf16 images: 2-byte storage, converted as torch's c10::Half / c10::BFloat16 do on CUDA
struct f16 { unsigned short x; };
struct bf16 { unsigned short x; };

template <typename T>
__device__ __forceinline__ T ld(const T* p) { return __ldg(p); }
template <>
__device__ __forceinline__ f16 ld(const f16* p) { return f16{__ldg(reinterpret_cast<const unsigned short*>(p))}; }
template <>
__device__ __forceinline__ bf16 ld(const bf16* p) { return bf16{__ldg(reinterpret_cast<const unsigned short*>(p))}; }

// `data.float()`: integers and fp64 round to nearest, fp16 / bf16 widen exactly
template <typename T>
__device__ __forceinline__ float to_float(T v) { return (float)v; }
__device__ __forceinline__ float to_float(f16 v) { return __half2float(__ushort_as_half(v.x)); }
__device__ __forceinline__ float to_float(bf16 v) { return __bfloat162float(__ushort_as_bfloat16(v.x)); }

// `.to(dtype)` of an fp32 value, as torch's CUDA cast does it (uint8 goes through int64)
template <typename T>
__device__ __forceinline__ T from_float(float f) {
  if constexpr (std::is_same<T, float>::value) return f;
  else if constexpr (std::is_same<T, uint8_t>::value) return (uint8_t)(long long)f;
  else if constexpr (std::is_same<T, f16>::value) return f16{__half_as_ushort(__float2half(f))};
  else if constexpr (std::is_same<T, bf16>::value) return bf16{__bfloat16_as_ushort(__float2bfloat16(f))};
  else return (T)f;
}

template <typename T>
union Pack {
  uint4 raw;
  T e[16 / sizeof(T)];
};

}  // namespace tio

// the label dtypes plus fp16 / bf16 / fp64 images (computed in fp32, as the reference's data.float())
#define TIO_IMAGE_DISPATCH(dtype, name, F)                          \
  switch (dtype) {                                                  \
    case TIO_F32: F(float); break;                                  \
    case TIO_U8: F(uint8_t); break;                                 \
    case TIO_I8: F(int8_t); break;                                  \
    case TIO_I16: F(int16_t); break;                                \
    case TIO_I32: F(int32_t); break;                                \
    case TIO_I64: F(int64_t); break;                                \
    case TIO_F16: F(f16); break;                                    \
    case TIO_BF16: F(bf16); break;                                  \
    case TIO_F64: F(double); break;                                 \
    default: TIO_CHECK_ARG(false, name ": unknown dtype %d", dtype); \
  }

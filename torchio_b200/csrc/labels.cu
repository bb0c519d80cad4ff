// labels.cu — the materialised form of label_interpolation="label" (SURVEY §8 f-4;
// transforms/spatial/spatial.py:1275-1389 of TorchIO 2.0.0a2).
//
// The fused form (tio_resample, TIO_LABEL_PV) covers the default call.  With antialias=True the
// reference blurs the one-hot channels before it samples them (spatial.py:1367-1368), so the
// channels have to exist: tio_onehot writes them, K3 blurs them, K1 samples them (exact
// coordinates, zero padding), tio_label_argmax folds them back.  Both kernels are single HBM
// streams (n fp32 channels per voxel on one side, one label on the other), 128-bit accesses on
// the fp32 side.
#include <climits>
#include <type_traits>

#include "common.cuh"

namespace tio {

template <typename T> struct LabelTable { typedef int64_t type; };
template <> struct LabelTable<float> { typedef float type; };

// Channel c of a voxel v: `v == (T)labels[c]` (tio_onehot), or, with kClasses, `long(v) == c`
// (tio_onehot_classes): the comparison is made in int64, so a class the dtype cannot hold matches
// nothing, and fp32 values are truncated the way `.long()` converts them on the device.
template <typename T, bool kClasses>
using OneHotKey = typename std::conditional<kClasses, long long, T>::type;

template <typename T, bool kClasses>
__global__ void __launch_bounds__(256)
onehot_kernel(const T* __restrict__ src, int64_t src_stride, int64_t vox,
              const typename LabelTable<T>::type* __restrict__ labels, int n, float* __restrict__ dst) {
  typedef OneHotKey<T, kClasses> Key;
  const int b = blockIdx.y;
  const T* s = src + (int64_t)b * src_stride;
  float* d = dst + (int64_t)b * n * vox;
  auto channel = [&](int c) -> Key {
    if constexpr (kClasses) return (Key)c; else return (T)labels[c];
  };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; t < vox; t += stride) {
    if (t + 4 <= vox && (vox & 3) == 0) {
      const Key v0 = (Key)s[t], v1 = (Key)s[t + 1], v2 = (Key)s[t + 2], v3 = (Key)s[t + 3];
      for (int c = 0; c < n; ++c) {
        const Key lab = channel(c);
        float4 o;
        o.x = v0 == lab ? 1.0f : 0.0f; o.y = v1 == lab ? 1.0f : 0.0f;
        o.z = v2 == lab ? 1.0f : 0.0f; o.w = v3 == lab ? 1.0f : 0.0f;
        *reinterpret_cast<float4*>(d + (int64_t)c * vox + t) = o;
      }
    } else {
      for (int64_t e = t; e < min(t + 4, vox); ++e)
        for (int c = 0; c < n; ++c) d[(int64_t)c * vox + e] = (Key)s[e] == channel(c) ? 1.0f : 0.0f;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
label_argmax_kernel(const float* __restrict__ sampled, int n, int64_t vox,
                    const typename LabelTable<T>::type* __restrict__ labels, float pad, T* __restrict__ dst) {
  const int b = blockIdx.y;
  const float* s = sampled + (int64_t)b * n * vox;
  T* d = dst + (int64_t)b * vox;
  // torch.full_like(resampled, default_pad_label) is built in the labels' dtype: truncation
  const T pad_t = (T)pad;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < vox; t += stride) {
    float best = s[t], total = s[t];
    int arg = 0;
    for (int c = 1; c < n; ++c) {
      const float v = __ldg(s + (int64_t)c * vox + t);
      total = __fadd_rn(total, v);           // sum(dim=1): channels in order
      if (v > best) { best = v; arg = c; }   // argmax: first maximum
    }
    d[t] = (total > 0.5f) ? (T)labels[arg] : pad_t;
  }
}

template <typename T, bool kClasses = false>
static void launch_onehot(const void* src, int B, int64_t src_stride, int64_t vox, const void* labels, int n,
                          float* dst, cudaStream_t st) {
  int64_t blocks = (vox / 4 + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  if (blocks < 1) blocks = 1;
  onehot_kernel<T, kClasses><<<dim3((unsigned)blocks, B), 256, 0, st>>>(
      (const T*)src, src_stride, vox, (const typename LabelTable<T>::type*)labels, n, dst);
  launched();
}

template <typename T>
static void launch_argmax(const float* sampled, int B, int n, int64_t vox, const void* labels, float pad,
                          void* dst, cudaStream_t st) {
  int64_t blocks = (vox + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  if (blocks < 1) blocks = 1;
  label_argmax_kernel<T><<<dim3((unsigned)blocks, B), 256, 0, st>>>(
      sampled, n, vox, (const typename LabelTable<T>::type*)labels, pad, (T*)dst);
  launched();
}

// ---- OneHot (transforms/label/one_hot.py:58-97) -----------------------------------------------

// min and max of long(v) over channel 0 of every element: ranks the classes before any launch of
// onehot_kernel, so an out-of-range class is an error on the host instead of a device assert
__global__ void label_range_init(long long* out) {
  out[0] = LLONG_MAX;
  out[1] = LLONG_MIN;
}

template <typename T>
__global__ void __launch_bounds__(256)
label_range_kernel(const T* __restrict__ src, int64_t src_stride, int64_t vox, long long* __restrict__ out) {
  const T* s = src + (int64_t)blockIdx.y * src_stride;
  long long lo = LLONG_MAX, hi = LLONG_MIN;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < vox; t += (int64_t)gridDim.x * blockDim.x) {
    const long long c = (long long)s[t];
    lo = min(lo, c);
    hi = max(hi, c);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(out, lo);
    atomicMax(out + 1, hi);
  }
}

template <typename T> __device__ __forceinline__ bool is_nan(T) { return false; }
template <> __device__ __forceinline__ bool is_nan<float>(float v) { return v != v; }

// torch.argmax(dim=1): the first maximum, and the first NaN is the maximum.  No early exit at a
// NaN: the channel loads do not depend on the comparisons, so they stay in flight together.
template <typename T>
__device__ __forceinline__ void argmax_step(T v, int c, T& best, int& arg) {
  if (!is_nan(best) && (is_nan(v) || v > best)) {
    best = v;
    arg = c;
  }
}

template <typename T> struct alignas(4 * sizeof(T)) Quad { T v[4]; };

// A thread owns 4 consecutive voxels when `vectorised` (vox % 4 == 0, aligned rows): each channel
// is one 4-element load, and a warp reads 4 * 32 consecutive elements per channel.  One element
// per thread and channel reads at a quarter of the HBM rate: the C rows are vox elements apart.
template <typename T>
__global__ void __launch_bounds__(256)
channel_argmax_kernel(const T* __restrict__ src, int C, int64_t vox, int vectorised, float* __restrict__ dst) {
  const T* s = src + (int64_t)blockIdx.y * C * vox;
  float* d = dst + (int64_t)blockIdx.y * vox;
  const int64_t first = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t quads = vectorised ? vox / 4 : 0;
  for (int64_t q = first; q < quads; q += stride) {
    const Quad<T> x0 = reinterpret_cast<const Quad<T>*>(s)[q];
    T best[4];
    int arg[4] = {0, 0, 0, 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) best[k] = x0.v[k];
#pragma unroll 4
    for (int c = 1; c < C; ++c) {
      const Quad<T> x = reinterpret_cast<const Quad<T>*>(s + (int64_t)c * vox)[q];
#pragma unroll
      for (int k = 0; k < 4; ++k) argmax_step(x.v[k], c, best[k], arg[k]);
    }
    reinterpret_cast<float4*>(d)[q] = make_float4((float)arg[0], (float)arg[1], (float)arg[2], (float)arg[3]);
  }
  for (int64_t t = quads * 4 + first; t < vox; t += stride) {
    T best = s[t];
    int arg = 0;
    for (int c = 1; c < C; ++c) argmax_step(s[(int64_t)c * vox + t], c, best, arg);
    d[t] = (float)arg;
  }
}

static int64_t stream_blocks(int64_t work) {
  int64_t blocks = (work + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  return blocks < 1 ? 1 : blocks;
}

}  // namespace tio

extern "C" int tio_onehot(const void* src, int dtype, int B, int64_t vox, const void* labels, int n,
                          float* dst, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && labels && dst && B > 0 && B <= 65535 && vox > 0 && n > 0, "tio_onehot: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case TIO_F32: launch_onehot<float>(src, B, vox, vox, labels, n, dst, st); break;
    case TIO_U8: launch_onehot<uint8_t>(src, B, vox, vox, labels, n, dst, st); break;
    case TIO_I8: launch_onehot<int8_t>(src, B, vox, vox, labels, n, dst, st); break;
    case TIO_I16: launch_onehot<int16_t>(src, B, vox, vox, labels, n, dst, st); break;
    case TIO_I32: launch_onehot<int32_t>(src, B, vox, vox, labels, n, dst, st); break;
    case TIO_I64: launch_onehot<int64_t>(src, B, vox, vox, labels, n, dst, st); break;
    default: TIO_CHECK_ARG(false, "tio_onehot: unknown dtype %d", dtype);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_label_argmax(const float* sampled, int B, int n, int64_t vox, const void* labels,
                                float pad_label, void* dst, int dtype, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(sampled && labels && dst && B > 0 && B <= 65535 && vox > 0 && n > 0,
                "tio_label_argmax: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case TIO_F32: launch_argmax<float>(sampled, B, n, vox, labels, pad_label, dst, st); break;
    case TIO_U8: launch_argmax<uint8_t>(sampled, B, n, vox, labels, pad_label, dst, st); break;
    case TIO_I8: launch_argmax<int8_t>(sampled, B, n, vox, labels, pad_label, dst, st); break;
    case TIO_I16: launch_argmax<int16_t>(sampled, B, n, vox, labels, pad_label, dst, st); break;
    case TIO_I32: launch_argmax<int32_t>(sampled, B, n, vox, labels, pad_label, dst, st); break;
    case TIO_I64: launch_argmax<int64_t>(sampled, B, n, vox, labels, pad_label, dst, st); break;
    default: TIO_CHECK_ARG(false, "tio_label_argmax: unknown dtype %d", dtype);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}


extern "C" int tio_onehot_classes(const void* src, int dtype, int B, int C, int64_t vox, int num_classes,
                                  float* dst, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst, "tio_onehot_classes: null source or output");
  TIO_CHECK_ARG(B > 0 && B <= 65535 && C > 0 && vox > 0 && num_classes > 0, "tio_onehot_classes: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_ONEHOT_CLASSES(T) launch_onehot<T, true>(src, B, (int64_t)C * vox, vox, nullptr, num_classes, dst, st)
  TIO_LABEL_DISPATCH(dtype, "tio_onehot_classes", TIO_ONEHOT_CLASSES)
#undef TIO_ONEHOT_CLASSES
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_label_range(const void* src, int dtype, int B, int C, int64_t vox, int64_t* range,
                               void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && range, "tio_label_range: null source or output");
  TIO_CHECK_ARG(B > 0 && B <= 65535 && C > 0 && vox > 0, "tio_label_range: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  long long* out = (long long*)range;
  label_range_init<<<1, 1, 0, st>>>(out);
  launched();
  const dim3 grid((unsigned)((stream_blocks(vox) + B - 1) / B), B);
#define TIO_RANGE(T) \
  label_range_kernel<T><<<grid, 256, 0, st>>>((const T*)src, (int64_t)C * vox, vox, out); \
  launched()
  TIO_LABEL_DISPATCH(dtype, "tio_label_range", TIO_RANGE)
#undef TIO_RANGE
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_channel_argmax(const void* src, int dtype, int B, int C, int64_t vox, float* dst,
                                  void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst, "tio_channel_argmax: null source or output");
  TIO_CHECK_ARG(B > 0 && B <= 65535 && C > 0 && vox > 0, "tio_channel_argmax: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  const int vectorised = vox % 4 == 0 && (uintptr_t)src % (4 * 8) == 0 && (uintptr_t)dst % 16 == 0;
  const dim3 grid((unsigned)stream_blocks(vectorised ? vox / 4 : vox), B);
#define TIO_ARGMAX(T) \
  channel_argmax_kernel<T><<<grid, 256, 0, st>>>((const T*)src, C, vox, vectorised, dst); \
  launched()
  TIO_LABEL_DISPATCH(dtype, "tio_channel_argmax", TIO_ARGMAX)
#undef TIO_ARGMAX
  TIO_CHECK_LAUNCH();
  return 0;
}

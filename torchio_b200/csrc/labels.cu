// labels.cu — the materialised form of label_interpolation="label" (SURVEY §8 f-4;
// transforms/spatial/spatial.py:1275-1389 of TorchIO 2.0.0a2).
//
// The fused form (tio_resample, TIO_LABEL_PV) covers the default call.  With antialias=True the
// reference blurs the one-hot channels before it samples them (spatial.py:1367-1368), so the
// channels have to exist: tio_onehot writes them, K3 blurs them, K1 samples them (exact
// coordinates, zero padding), tio_label_argmax folds them back.  Both kernels are single HBM
// streams (n fp32 channels per voxel on one side, one label on the other), 128-bit accesses on
// the fp32 side.
#include "common.cuh"

namespace tio {

template <typename T> struct LabelTable { typedef int64_t type; };
template <> struct LabelTable<float> { typedef float type; };

template <typename T>
__global__ void __launch_bounds__(256)
onehot_kernel(const T* __restrict__ src, int64_t vox, const typename LabelTable<T>::type* __restrict__ labels,
              int n, float* __restrict__ dst) {
  const int b = blockIdx.y;
  const T* s = src + (int64_t)b * vox;
  float* d = dst + (int64_t)b * n * vox;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (int64_t t = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; t < vox; t += stride) {
    if (t + 4 <= vox && (vox & 3) == 0) {
      const T v0 = s[t], v1 = s[t + 1], v2 = s[t + 2], v3 = s[t + 3];
      for (int c = 0; c < n; ++c) {
        const T lab = (T)labels[c];
        float4 o;
        o.x = v0 == lab ? 1.0f : 0.0f; o.y = v1 == lab ? 1.0f : 0.0f;
        o.z = v2 == lab ? 1.0f : 0.0f; o.w = v3 == lab ? 1.0f : 0.0f;
        *reinterpret_cast<float4*>(d + (int64_t)c * vox + t) = o;
      }
    } else {
      for (int64_t e = t; e < min(t + 4, vox); ++e)
        for (int c = 0; c < n; ++c) d[(int64_t)c * vox + e] = s[e] == (T)labels[c] ? 1.0f : 0.0f;
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

template <typename T>
static void launch_onehot(const void* src, int B, int64_t vox, const void* labels, int n, float* dst,
                          cudaStream_t st) {
  int64_t blocks = (vox / 4 + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  if (blocks < 1) blocks = 1;
  onehot_kernel<T><<<dim3((unsigned)blocks, B), 256, 0, st>>>(
      (const T*)src, vox, (const typename LabelTable<T>::type*)labels, n, dst);
}

template <typename T>
static void launch_argmax(const float* sampled, int B, int n, int64_t vox, const void* labels, float pad,
                          void* dst, cudaStream_t st) {
  int64_t blocks = (vox + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  if (blocks < 1) blocks = 1;
  label_argmax_kernel<T><<<dim3((unsigned)blocks, B), 256, 0, st>>>(
      sampled, n, vox, (const typename LabelTable<T>::type*)labels, pad, (T*)dst);
}

}  // namespace tio

extern "C" int tio_onehot(const void* src, int dtype, int B, int64_t vox, const void* labels, int n,
                          float* dst, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && labels && dst && B > 0 && B <= 65535 && vox > 0 && n > 0, "tio_onehot: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  switch (dtype) {
    case TIO_F32: launch_onehot<float>(src, B, vox, labels, n, dst, st); break;
    case TIO_U8: launch_onehot<uint8_t>(src, B, vox, labels, n, dst, st); break;
    case TIO_I8: launch_onehot<int8_t>(src, B, vox, labels, n, dst, st); break;
    case TIO_I16: launch_onehot<int16_t>(src, B, vox, labels, n, dst, st); break;
    case TIO_I32: launch_onehot<int32_t>(src, B, vox, labels, n, dst, st); break;
    case TIO_I64: launch_onehot<int64_t>(src, B, vox, labels, n, dst, st); break;
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

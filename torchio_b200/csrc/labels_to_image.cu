// labels_to_image.cu — LabelsToImage (transforms/intensity/labels_to_image.py:182-290 of TorchIO
// 2.0.0a2) in one pass: read the label, write one fp32 value.
//
// The reference draws one full-volume torch.randn_like per label on the label map's CUDA device
// and keeps, per voxel, only the draw of that voxel's label.  Those draws come from ATen's Philox
// normal kernel (ATen/native/cuda/DistributionTemplates.h): 256-thread blocks, grid_x blocks,
// S = 256 * grid_x; thread t runs curand_init(seed, t, offset) and iteration `it` of its
// grid-stride loop takes one curand_normal4 whose component ii lands on element
// it * 4S + ii * S + t.  Philox is counter-based, so the normal of any element is computed
// directly: component ii of Philox4x32-10 at counter (offset / 4 + it, t), key = seed, through
// curand's Box-Muller.  One thread here handles the four elements of one (t, it) pair — S apart,
// so every load and store of a warp is coalesced — and runs Philox once per distinct drawn label
// among them and Box-Muller once per distinct (label, component pair).
//
// Per voxel of label k (draw k, element b):  out = (((z + 0) * std[b][k]) + mean[b][k]) + 0,
// each step rounded to fp32 on its own: `normal_(0, 1)` stores z * 1 + 0, `* std` and `+ mean`
// are separate kernels, and the running sum starts at +0 (the masked terms of the other labels
// add +-0, which changes nothing).  Voxels whose label is not drawn stay +0.
#include <curand_kernel.h>

#include "common.cuh"
#include "label_lookup.cuh"

namespace tio {

namespace {

constexpr int kThreads = 256;
constexpr int kItersPerBlock = 8;  // grid-stride iterations per block: amortises the table load
constexpr int kMaxLabels = 2048;
constexpr unsigned long long kNotDrawn = ~0ull;

template <typename T>
__global__ void __launch_bounds__(kThreads)
labels_to_image_kernel(const T* __restrict__ labels, int C, uint32_t vox, uint32_t N,
                       const long long* __restrict__ label_values, int n,
                       const float* __restrict__ mean, const float* __restrict__ std,
                       const unsigned long long* __restrict__ draw_offset,
                       unsigned long long seed, uint32_t iters, float* __restrict__ out) {
  // shared: draw offset per slot | sorted label values (wider maps) or a byte -> slot LUT
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* offs = reinterpret_cast<unsigned long long*>(smem);
  long long* values = reinterpret_cast<long long*>(offs + n);
  int* lut = reinterpret_cast<int*>(values + n);
  for (int i = threadIdx.x; i < n; i += kThreads) {
    offs[i] = draw_offset[i];
    values[i] = label_values[i];
  }
  if constexpr (kByteLabels<T>) {
    lut[threadIdx.x] = -1;  // kThreads == 256 entries
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const long long v = label_values[i];
      constexpr bool is_signed = (T)-1 < (T)0;
      const long long lo = is_signed ? -128 : 0, hi = is_signed ? 127 : 255;
      if (v >= lo && v <= hi) lut[(unsigned)(unsigned char)(T)v] = i;
    }
  }
  __syncthreads();

  const uint32_t S = gridDim.x * kThreads;
  const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  const uint32_t it_end = min(iters, (blockIdx.y + 1) * kItersPerBlock);
  for (uint32_t it = blockIdx.y * kItersPerBlock; it < it_end; ++it) {
    int k[4];
    uint32_t b[4];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const uint32_t v = it * 4 * S + ii * S + t;
      k[ii] = -1;
      b[ii] = 0;
      if (v < N) {
        b[ii] = v / vox;
        const uint32_t r = v - b[ii] * vox;
        const int slot = find_slot<T, long long>(labels[((size_t)b[ii] * C) * vox + r], lut, values, n);
        if (slot >= 0 && offs[slot] != kNotDrawn) k[ii] = slot;
      }
    }
    // Philox once per distinct drawn label of the four elements
    uint4 ph[4];
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      ph[ii] = make_uint4(0, 0, 0, 0);
      if (k[ii] < 0) continue;
      bool found = false;
#pragma unroll
      for (int jj = 0; jj < ii; ++jj)
        if (!found && k[jj] == k[ii]) { ph[ii] = ph[jj]; found = true; }
      if (!found) {
        const unsigned long long c = offs[k[ii]] / 4 + it;
        ph[ii] = curand_Philox4x32_10(make_uint4((unsigned)c, (unsigned)(c >> 32), t, 0u), key);
      }
    }
    // curand_normal4: components 0/1 are Box-Muller of words (x, y), 2/3 of (z, w)
    float z[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const int a = 2 * p, c = 2 * p + 1;
      if (k[a] >= 0) {
        const float2 r = p == 0 ? _curand_box_muller(ph[a].x, ph[a].y) : _curand_box_muller(ph[a].z, ph[a].w);
        z[a] = r.x;
        if (k[c] == k[a]) z[c] = r.y;
      }
      if (k[c] >= 0 && k[c] != k[a]) {
        const float2 r = p == 0 ? _curand_box_muller(ph[c].x, ph[c].y) : _curand_box_muller(ph[c].z, ph[c].w);
        z[c] = r.y;
      }
    }
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const uint32_t v = it * 4 * S + ii * S + t;
      if (v >= N) continue;
      float o = 0.0f;
      if (k[ii] >= 0) {
        const int e = b[ii] * n + k[ii];
        const float zn = __fadd_rn(z[ii], 0.0f);
        o = __fadd_rn(__fadd_rn(__fmul_rn(zn, __ldg(std + e)), __ldg(mean + e)), 0.0f);
      }
      out[v] = o;
    }
  }
}

template <typename T>
void launch(const void* labels, int C, uint32_t vox, uint32_t N, const long long* values, int n,
            const float* mean, const float* std, const unsigned long long* offs, unsigned long long seed,
            int grid_x, float* out, cudaStream_t st) {
  const uint32_t S = (uint32_t)grid_x * kThreads;
  const uint32_t iters = (uint32_t)((N - 1) / (4ull * S) + 1);
  const dim3 grid((unsigned)grid_x, (iters + kItersPerBlock - 1) / kItersPerBlock);
  const size_t smem = (size_t)n * 16 + (kByteLabels<T> ? kThreads * sizeof(int) : 0);
  labels_to_image_kernel<T><<<grid, kThreads, smem, st>>>((const T*)labels, C, vox, N, values, n, mean, std,
                                                          offs, seed, iters, out);
  launched();
}

}  // namespace

}  // namespace tio

extern "C" int tio_labels_to_image(const void* labels, int dtype, int C, int B, int64_t vox,
                                   const int64_t* label_values, int n, const float* mean, const float* std,
                                   const uint64_t* draw_offset, uint64_t seed, int grid_x, float* out,
                                   void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(labels && out, "tio_labels_to_image: null labels or output");
  TIO_CHECK_ARG(n >= 0 && n <= kMaxLabels, "tio_labels_to_image: %d labels (at most %d)", n, kMaxLabels);
  TIO_CHECK_ARG(n == 0 || (label_values && mean && std && draw_offset),
                "tio_labels_to_image: null label table");
  TIO_CHECK_ARG(C > 0 && B > 0 && vox > 0, "tio_labels_to_image: bad shape");
  TIO_CHECK_ARG((int64_t)B * vox <= (1ll << 29),
                "tio_labels_to_image: %lld voxels; draws above 2^29 are split into several launches by ATen",
                (long long)B * vox);
  TIO_CHECK_ARG(grid_x > 0 && (int64_t)grid_x * kThreads <= (1ll << 29), "tio_labels_to_image: bad grid_x %d",
                grid_x);
  const uint32_t N = (uint32_t)(B * vox);
  cudaStream_t st = (cudaStream_t)stream;
  const auto* values = (const long long*)label_values;
  const auto* offs = (const unsigned long long*)draw_offset;
  switch (dtype) {
    case TIO_F32: launch<float>(labels, C, (uint32_t)vox, N, values, n, mean, std, offs, seed, grid_x, out, st); break;
    case TIO_U8: launch<uint8_t>(labels, C, (uint32_t)vox, N, values, n, mean, std, offs, seed, grid_x, out, st); break;
    case TIO_I8: launch<int8_t>(labels, C, (uint32_t)vox, N, values, n, mean, std, offs, seed, grid_x, out, st); break;
    case TIO_I16: launch<int16_t>(labels, C, (uint32_t)vox, N, values, n, mean, std, offs, seed, grid_x, out, st); break;
    case TIO_I32: launch<int32_t>(labels, C, (uint32_t)vox, N, values, n, mean, std, offs, seed, grid_x, out, st); break;
    case TIO_I64: launch<int64_t>(labels, C, (uint32_t)vox, N, values, n, mean, std, offs, seed, grid_x, out, st); break;
    default: TIO_CHECK_ARG(false, "tio_labels_to_image: unknown dtype %d", dtype);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

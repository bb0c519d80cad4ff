// motion.cu — Motion of TorchIO 2.0.0a2 (transforms/intensity/motion.py) on the GPU.
//
// The reference takes fftn(x) of every (b, c) row, and for each of N rigid transforms s = 1..N
// replaces the first-axis k-space rows [start_s, end_s) by those of fftn(x_s), x_s the row
// resampled by grid_sample; then ifftn(...).real.  The segments vary only along the first axis I,
// so the FFTs over J and K cancel and each line along I becomes
//   out = Re(ifft_I(sum_s P_s fft_I(x_s))) = ifft_I(sum_s Hs_s fft_I(x_s)),
//   Hs_s(f) = (P_s(f) + P_s(-f mod I)) / 2,
// with P_s the 0/1 indicator of segment s's rows (segment 0: x_0 = x, rows [0, I // (N + 1))).
// Every Hs_s is real and even, so two real lines share one complex FFT, as in ghosting.cu.  The
// resampled copies x_s are computed tile by tile in shared memory and never written to memory.
//
// tio_motion   out of place; per CTA: 2 L columns (j, k) of one (b, c) row, all I points.  Segment 0
//              loads x, segment s >= 1 gathers the 8 trilinear taps of x_s from the row; each is
//              transformed and accumulated with weight Hs_s; one inverse FFT; one write per voxel.
//              A row with a NaN or +-Inf voxel is flagged by the segment-0 loads and a follow-up
//              pass fills it with NaN.  Inactive elements are copied bit for bit.
#include <cmath>

#include "common.cuh"
#include "fft_lines.cuh"
#include "image_dtype.cuh"

namespace tio {

namespace {

constexpr int kThreads = 256;

struct Geometry {
  int C, I, J, K;
  int64_t vox;
};

// ATen's linspace(-1, 1, n)[idx] (affine_grid's base grid with align_corners=True): two-sided, so
// the last point is exactly 1; 0 when n == 1
__device__ __forceinline__ float lin(int idx, int n) {
  if (n <= 1) return 0.0f;
  const float step = __fdiv_rn(2.0f, (float)(n - 1));
  return idx < n / 2 ? __fadd_rn(-1.0f, __fmul_rn(step, (float)idx))
                     : __fsub_rn(1.0f, __fmul_rn(step, (float)(n - idx - 1)));
}

// grid_sample(x, affine_grid(theta), bilinear, zeros, align_corners=True) at the output voxel whose
// base-grid point is (lk, lj, li): affine_grid's frame is (x, y, z) = (K, J, I).  Taps in
// grid_sampler_3d's order (tnw, tne, tsw, tse, bnw, bne, bsw, bse); taps outside the row add 0.
template <typename T>
__device__ __forceinline__ float rigid_sample(const T* __restrict__ x, const float* th, float lk, float lj, float li,
                                              int I, int J, int K) {
  const float gx = fmaf(th[2], li, fmaf(th[1], lj, th[0] * lk)) + th[3];
  const float gy = fmaf(th[6], li, fmaf(th[5], lj, th[4] * lk)) + th[7];
  const float gz = fmaf(th[10], li, fmaf(th[9], lj, th[8] * lk)) + th[11];
  const float ix = (gx + 1.0f) * 0.5f * (float)(K - 1);
  const float iy = (gy + 1.0f) * 0.5f * (float)(J - 1);
  const float iz = (gz + 1.0f) * 0.5f * (float)(I - 1);
  const float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
  const float wx[2] = {fx + 1.0f - ix, ix - fx}, wy[2] = {fy + 1.0f - iy, iy - fy}, wz[2] = {fz + 1.0f - iz, iz - fz};
  float acc = 0.0f;
#pragma unroll
  for (int dz = 0; dz < 2; ++dz) {
    const float z = fz + dz;
    if (!(z >= 0.0f && z <= (float)(I - 1))) continue;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
      const float y = fy + dy;
      if (!(y >= 0.0f && y <= (float)(J - 1))) continue;
      const T* plane = x + ((int64_t)z * J + (int64_t)y) * K;
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        const float xx = fx + dx;
        if (!(xx >= 0.0f && xx <= (float)(K - 1))) continue;
        acc = fmaf(to_float(ld(plane + (int64_t)xx)), wx[dx] * wy[dy] * wz[dz], acc);
      }
    }
  }
  return acc;
}

// Hs_s(f) / (2 I) summed later as conj: the symmetrisation's 1/2 and the inverse FFT's 1/I folded in
__device__ __forceinline__ float segment_weight(int f, int s, int I, int size, int last, float scale) {
  const int fm = f ? I - f : 0;
  const int a = min(f / size, last), b = min(fm / size, last);
  return (float)((a == s) + (b == s)) * scale;
}

// A CTA takes `width` = 2 * lines consecutive (j, k) columns of one (b, c) row (point stride J K
// along I), packed in pairs as the real and imaginary parts of `lines` complex lines: real line c is
// component c & 1 of complex line c >> 1.  Consecutive threads take consecutive columns, so loads,
// gathers and stores of a warp are close in memory.
template <typename T>
__global__ void __launch_bounds__(kThreads)
motion_kernel(const T* __restrict__ in, T* __restrict__ out, Geometry g, int lines, int S, FftPlan plan,
              int segments, const float* __restrict__ theta, const uint8_t* __restrict__ active,
              uint32_t* __restrict__ flags) {
  const int row = blockIdx.y, b = row / g.C;
  const int I = plan.n, width = 2 * lines;
  const int64_t n_cols = (int64_t)g.J * g.K, first = (int64_t)blockIdx.x * width;
  const int cols = (int)(n_cols - first < width ? n_cols - first : width);
  const T* src = in + (int64_t)row * g.vox;
  T* dst = out + (int64_t)row * g.vox;
  if (!active[b]) {  // gated out: the reference's torch.where keeps the input's bits
    for (int e = threadIdx.x; e < I * width; e += blockDim.x) {
      const int c = e % width, t = e / width;
      if (c < cols) dst[t * n_cols + first + c] = src[t * n_cols + first + c];
    }
    return;
  }
  extern __shared__ float2 smem[];
  float2* W = smem;
  float2* buf0 = W + I;
  float2* buf1 = buf0 + lines * S;
  float2* acc = buf1 + lines * S;
  float2* col_lin = acc + lines * S;                         // (lin_K[k], lin_J[j]) of each column
  float* li = reinterpret_cast<float*>(col_lin + width);  // lin_I[i]
  build_table(W, I);
  for (int t = threadIdx.x; t < I; t += blockDim.x) li[t] = lin(t, I);
  for (int c = threadIdx.x; c < width; c += blockDim.x) {
    const int64_t col = first + (c < cols ? c : 0);
    const int j = (int)(col / g.K), k = (int)(col - (int64_t)j * g.K);
    col_lin[c] = make_float2(lin(k, g.K), lin(j, g.J));
  }
  const int size = I / segments, last = segments - 1;
  const float scale = 0.5f / (float)I;

  float* re = reinterpret_cast<float*>(buf0);
  bool bad = false;
  for (int e = threadIdx.x; e < I * width; e += blockDim.x) {
    const int c = e % width, t = e / width;
    const float v = c < cols ? to_float(ld(src + t * n_cols + first + c)) : 0.0f;
    bad |= !isfinite(v);
    re[2 * ((c >> 1) * S + t) + (c & 1)] = v;
  }
  // the reference's 3-D FFT spreads a NaN or an Inf over the whole row: the NaN pass fills it
  if (__syncthreads_or(bad)) {
    if (threadIdx.x == 0) atomicOr(flags + row, 1u);
    return;
  }
  for (int s = 0; s < segments; ++s) {
    if (s > 0) {
      float th[12];
      const float* t_s = theta + ((int64_t)b * last + (s - 1)) * 12;
#pragma unroll
      for (int m = 0; m < 12; ++m) th[m] = __ldg(t_s + m);
      __syncthreads();  // the previous segment's spectrum has been read out of buf0 / buf1
      for (int e = threadIdx.x; e < I * width; e += blockDim.x) {
        const int c = e % width, t = e / width;
        const float2 l = col_lin[c];
        const float v = c < cols ? rigid_sample(src, th, l.x, l.y, li[t], I, g.J, g.K) : 0.0f;
        re[2 * ((c >> 1) * S + t) + (c & 1)] = v;
      }
    }
    const float2* r = fft_lines(buf0, buf1, lines, S, plan, W);
    for (int e = threadIdx.x; e < lines * I; e += blockDim.x) {
      const int line = e / I, f = e - line * I;
      const float h = segment_weight(f, s, I, size, last, scale);
      const float2 v = r[line * S + f];
      const float2 a = s ? acc[line * S + f] : make_float2(0.0f, 0.0f);
      acc[line * S + f] = make_float2(fmaf(h, v.x, a.x), fmaf(-h, v.y, a.y));  // conj(sum Hs_s Y_s / I)
    }
  }
  const float* res = reinterpret_cast<const float*>(fft_lines(acc, buf0, lines, S, plan, W));
  for (int e = threadIdx.x; e < I * width; e += blockDim.x) {
    const int c = e % width, t = e / width;
    if (c < cols) {
      const float v = res[2 * ((c >> 1) * S + t) + (c & 1)];  // out = conj(res): a = Re, b = -Im
      dst[t * n_cols + first + c] = from_float<T>(c & 1 ? -v : v);
    }
  }
}

// rows flagged by motion_kernel become all NaN; every other CTA returns at once (as in ghosting.cu)
template <typename T>
__global__ void __launch_bounds__(kThreads)
nan_rows_kernel(T* data, int64_t vox, const uint32_t* __restrict__ flags) {
  const int row = blockIdx.y;
  if (!flags[row]) return;
  const T nan = from_float<T>(__int_as_float(0x7fffffff));
  T* x = data + (int64_t)row * vox;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < vox; e += (int64_t)gridDim.x * blockDim.x)
    x[e] = nan;
}

// complex lines per CTA: 2048 points per buffer, 1 to 16 lines.  Measured on an H100 80GB HBM3 (700 W
// power limit) on 32 x 1 x 256^3 with N = 2
// (lines 2 / 4 / 8 / 16: 36.1 / 29.0 / 26.1 / 31.2 ms) and 8 x 1 x 128^3 (16 lines best, 1.02 ms
// against 1.15 with 8); the FFT passes' 4096 points are slower here, where the gathers of the moved
// copies want more resident CTAs per SM.
int motion_lines(int I) { return I >= 2048 ? 1 : (2048 / I > kMaxLines ? kMaxLines : 2048 / I); }

size_t motion_smem(int I, int lines) {
  return fft_smem(I, lines) + (size_t)lines * line_stride(I) * sizeof(float2) + 2 * (size_t)lines * sizeof(float2) +
         (size_t)I * sizeof(float);
}

int element_bytes(int dtype) {
  switch (dtype) {
    case TIO_U8: case TIO_I8: return 1;
    case TIO_I16: case TIO_F16: case TIO_BF16: return 2;
    case TIO_I64: case TIO_F64: return 8;
    default: return 4;
  }
}

}  // namespace

}  // namespace tio

extern "C" int tio_motion(const void* in, void* out, int dtype, int B, int C, int I, int J, int K, int segments,
                          const float* theta, const uint8_t* active, uint32_t* flags, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(in && out && theta && active && flags, "tio_motion: null pointer");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "tio_motion: bad shape (%d, %d, %d, %d, %d)", B, C, I, J,
                K);
  TIO_CHECK_ARG((int64_t)B * C <= 65535, "tio_motion: %lld rows (B * C), at most 65535", (long long)B * C);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_motion: unknown dtype %d", dtype);
  TIO_CHECK_ARG(I <= kMaxAxis, "tio_motion: first axis of %d points, at most %d", I, kMaxAxis);
  TIO_CHECK_ARG(segments >= 2 && segments <= I, "tio_motion: %d segments for a first axis of %d points", segments,
                I);
  const int64_t vox = (int64_t)I * J * K, bytes = (int64_t)B * C * vox * element_bytes(dtype);
  const char *a = (const char*)in, *o = (const char*)out;
  TIO_CHECK_ARG(a + bytes <= o || o + bytes <= a, "tio_motion: in and out overlap");
  const int lines = motion_lines(I), width = 2 * lines, S = line_stride(I);
  const int64_t blocks = ((int64_t)J * K + width - 1) / width;
  TIO_CHECK_ARG(blocks < (1ll << 31), "tio_motion: %lld blocks per row", (long long)blocks);
  const Geometry g = {C, I, J, K, vox};
  const int rows = B * C;
  const FftPlan plan = make_plan(I);
  const size_t smem = motion_smem(I, lines);
  const dim3 grid((unsigned)blocks, (unsigned)rows);
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(flags, 0, (size_t)rows * sizeof(uint32_t), st));
#define TIO_MOTION(T)                                                                                                \
  TIO_CHECK_CUDA(cudaFuncSetAttribute(motion_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
  motion_kernel<T><<<grid, kThreads, smem, st>>>((const T*)in, (T*)out, g, lines, S, plan, segments, theta, active, \
                                                 flags);                                                            \
  launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_motion", TIO_MOTION)
#undef TIO_MOTION
  TIO_CHECK_LAUNCH();
  int64_t parts = ((int64_t)num_sms() * 8 + rows - 1) / rows;
  const int64_t useful = (vox + kThreads - 1) / kThreads;
  if (parts > useful) parts = useful;
  const dim3 nan_grid((unsigned)parts, (unsigned)rows);
#define TIO_NAN_ROWS(T) nan_rows_kernel<T><<<nan_grid, kThreads, 0, st>>>((T*)out, vox, flags); launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_motion", TIO_NAN_ROWS)
#undef TIO_NAN_ROWS
  TIO_CHECK_LAUNCH();
  return 0;
}

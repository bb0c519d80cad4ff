// ghosting.cu — Ghosting of TorchIO 2.0.0a2 (transforms/intensity/ghosting.py) on the GPU.
//
// The reference multiplies fftshift(fftn(x)) by a real mask that varies along one axis only and
// inverts the FFT.  The FFTs over the two other axes cancel, so each line along the chosen axis
// becomes
//   out = Re(ifft(H fft(x))) = ifft(Hs fft(x)),   Hs(f) = (H(f) + H(-f mod n)) / 2,
// with H the mask in unshifted order.  Hs is real and even, so two real lines a, b share one
// complex FFT: ifft(Hs fft(a + i b)) = out_a + i out_b.  The inverse runs on the forward engine of
// fft_lines.cuh and its table, as conj(fft(conj(Y))) / n.
//
// tio_ghosting   in place, one read and one write per voxel; a row with a NaN or +-Inf voxel is
//                flagged while its lines load, and a follow-up pass fills only flagged rows with NaN
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

// A CTA filters 2 * lines real lines of the ghosted axis (n points) of one (b, c) row, packed in
// pairs as the real and imaginary parts of `lines` complex lines: real line c is component c & 1
// of complex line c >> 1.  K axis (kContiguous): 2 * lines consecutive K lines.  I and J axes: up to
// 2 * lines consecutive columns, so a warp's loads are consecutive in memory; a column is a
// (j, k) pair on the I axis (point stride J K) and a k at one i on the J axis (point stride K).
template <typename T, bool kContiguous>
__global__ void __launch_bounds__(kThreads)
ghosting_kernel(T* data, Geometry g, int ax, int lines, int S, FftPlan plan, const float* __restrict__ table,
                int n_max, const int32_t* __restrict__ axis, const uint8_t* __restrict__ active,
                uint32_t* __restrict__ flags) {
  const int row = blockIdx.y, b = row / g.C;
  if (!active[b] || axis[b] != ax) return;  // not active or another axis: no byte moves
  const int n = plan.n, width = 2 * lines;
  extern __shared__ float2 smem[];
  float2* W = smem;
  float2* buf0 = W + n;
  float2* buf1 = buf0 + lines * S;
  float* Hs = reinterpret_cast<float*>(buf1 + lines * S);
  build_table(W, n);
  const float* H = table + (int64_t)b * n_max;
  const float scale = 0.5f / (float)n;  // the symmetrisation's 1/2 and the inverse FFT's 1/n
  for (int f = threadIdx.x; f < n; f += blockDim.x) Hs[f] = (H[f] + H[f ? n - f : 0]) * scale;

  T* base = data + (int64_t)row * g.vox;
  int64_t pstride, cstride;
  int cols;
  if (kContiguous) {
    const int64_t n_lines = (int64_t)g.I * g.J, first = (int64_t)blockIdx.x * width;
    cols = (int)(n_lines - first < width ? n_lines - first : width);
    base += first * g.K;
    pstride = 1;
    cstride = g.K;
  } else {
    const int64_t n_cols = ax == 0 ? (int64_t)g.J * g.K : g.K;
    const int64_t tiles = (n_cols + width - 1) / width;
    const int64_t tile = blockIdx.x % tiles, outer = blockIdx.x / tiles;  // outer: i on the J axis, 0 on I
    cols = (int)(n_cols - tile * width < width ? n_cols - tile * width : width);
    base += outer * g.J * g.K + tile * width;
    pstride = ax == 0 ? (int64_t)g.J * g.K : g.K;
    cstride = 1;
  }

  float* re = reinterpret_cast<float*>(buf0);
  bool bad = false;
  for (int e = threadIdx.x; e < n * width; e += blockDim.x) {
    const int c = kContiguous ? e / n : e % width, t = kContiguous ? e - c * n : e / width;
    const float v = c < cols ? to_float(ld(base + t * pstride + c * cstride)) : 0.0f;
    bad |= !isfinite(v);
    re[2 * ((c >> 1) * S + t) + (c & 1)] = v;
  }
  // the reference's 3-D FFT spreads a NaN or an Inf over the whole row: the NaN pass fills it
  if (__syncthreads_or(bad)) {
    if (threadIdx.x == 0) atomicOr(flags + row, 1u);
    return;
  }

  float2* r = fft_lines(buf0, buf1, lines, S, plan, W);
  for (int e = threadIdx.x; e < lines * n; e += blockDim.x) {
    const int line = e / n, f = e - line * n;
    const float2 v = r[line * S + f];
    const float h = Hs[f];
    r[line * S + f] = make_float2(h * v.x, -h * v.y);  // conj(Hs Y / n)
  }
  r = fft_lines(r, r == buf0 ? buf1 : buf0, lines, S, plan, W);  // out = conj(r): a = Re r, b = -Im r

  const float* out = reinterpret_cast<const float*>(r);
  for (int e = threadIdx.x; e < n * width; e += blockDim.x) {
    const int c = kContiguous ? e / n : e % width, t = kContiguous ? e - c * n : e / width;
    if (c < cols) {
      const float v = out[2 * ((c >> 1) * S + t) + (c & 1)];
      base[t * pstride + c * cstride] = from_float<T>(c & 1 ? -v : v);
    }
  }
}

// rows flagged by ghosting_kernel become all NaN; every other CTA returns at once
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

// CTAs of ghosting_kernel along axis a: K lines in groups of `width`; on the I and J axes,
// `width`-column tiles (per i on the J axis)
int64_t ghosting_blocks(int a, int I, int J, int K, int width) {
  if (a == 2) return ((int64_t)I * J + width - 1) / width;
  const int64_t cols = a == 0 ? (int64_t)J * K : K, outer = a == 0 ? 1 : I;
  return outer * ((cols + width - 1) / width);
}

}  // namespace

}  // namespace tio

extern "C" int tio_ghosting(void* data, int dtype, int B, int C, int I, int J, int K, const float* table, int n_max,
                            const int32_t* axis, const uint8_t* active, int axes, uint32_t* flags, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(data && table && axis && active && flags, "tio_ghosting: null pointer");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "tio_ghosting: bad shape (%d, %d, %d, %d, %d)", B, C,
                I, J, K);
  TIO_CHECK_ARG((int64_t)B * C <= 65535, "tio_ghosting: %lld rows (B * C), at most 65535", (long long)B * C);
  TIO_CHECK_ARG(axes > 0 && axes < 8, "tio_ghosting: axes mask %d names an axis outside 0..2", axes);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_ghosting: unknown dtype %d", dtype);
  const int len[3] = {I, J, K};
  for (int a = 0; a < 3; ++a) {
    if (!(axes >> a & 1)) continue;
    TIO_CHECK_ARG(len[a] <= kMaxAxis, "tio_ghosting: axis %d of %d points, at most %d", a, len[a], kMaxAxis);
    TIO_CHECK_ARG(len[a] <= n_max, "tio_ghosting: table rows of %d entries, axis %d has %d points", n_max, a,
                  len[a]);
    const int lines = fft_lines_for(len[a]), width = 2 * lines;
    const int64_t blocks = ghosting_blocks(a, I, J, K, width);
    TIO_CHECK_ARG(blocks < (1ll << 31), "tio_ghosting: %lld blocks along axis %d", (long long)blocks, a);
  }
  const Geometry g = {C, I, J, K, (int64_t)I * J * K};
  const int rows = B * C;
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(flags, 0, (size_t)rows * sizeof(uint32_t), st));
  for (int a = 0; a < 3; ++a) {
    if (!(axes >> a & 1)) continue;
    const int n = len[a], lines = fft_lines_for(n), width = 2 * lines, S = line_stride(n);
    const FftPlan plan = make_plan(n);
    const size_t smem = fft_smem(n, lines) + (size_t)n * sizeof(float);
    const int64_t blocks = ghosting_blocks(a, I, J, K, width);
    const dim3 grid((unsigned)blocks, (unsigned)rows);
#define TIO_GHOST(T)                                                                                                \
  if (a == 2) {                                                                                                     \
    TIO_CHECK_CUDA(cudaFuncSetAttribute(ghosting_kernel<T, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,     \
                                        (int)smem));                                                                \
    ghosting_kernel<T, true><<<grid, kThreads, smem, st>>>((T*)data, g, a, lines, S, plan, table, n_max, axis,    \
                                                           active, flags);                                          \
  } else {                                                                                                          \
    TIO_CHECK_CUDA(cudaFuncSetAttribute(ghosting_kernel<T, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,    \
                                        (int)smem));                                                                \
    ghosting_kernel<T, false><<<grid, kThreads, smem, st>>>((T*)data, g, a, lines, S, plan, table, n_max, axis,   \
                                                            active, flags);                                         \
  }                                                                                                                 \
  launched();
    TIO_IMAGE_DISPATCH(dtype, "tio_ghosting", TIO_GHOST)
#undef TIO_GHOST
    TIO_CHECK_LAUNCH();
  }
  int64_t parts = ((int64_t)num_sms() * 8 + rows - 1) / rows;
  const int64_t useful = (g.vox + kThreads - 1) / kThreads;
  if (parts > useful) parts = useful;
  const dim3 nan_grid((unsigned)parts, (unsigned)rows);
#define TIO_NAN_ROWS(T) nan_rows_kernel<T><<<nan_grid, kThreads, 0, st>>>((T*)data, g.vox, flags); launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_ghosting", TIO_NAN_ROWS)
#undef TIO_NAN_ROWS
  TIO_CHECK_LAUNCH();
  return 0;
}

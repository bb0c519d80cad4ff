// spike.cu — Spike of TorchIO 2.0.0a2 (transforms/intensity/spike.py) on the GPU.
//
// The reference adds peak * intensity at a few points of fftshift(fftn(x)) and inverts the FFT.  A
// point impulse of amplitude a at frequency (u, v, w) is the plane wave (a / N) cos(2 pi (u i / I +
// v j / J + w k / K)) in image space, so the output is x plus a sum of cosines and needs no inverse
// FFT.  Only the amplitude needs the spectrum: for x >= 0 its peak is |F(0)| = sum(x).
//
// tio_spike_stats     per (b, c) row: fp64 sum of float(x), "some value < 0", "some value not finite"
// tio_spectrum_peak   max |F| of the rows that are signed and finite: a forward half-spectrum FFT,
//                     three axis passes over a complex64 workspace, the last one reduces only
// tio_spike           x + A cos(...) in place, per-axis phase tables, integer-reduced phases
#include <cmath>

#include "common.cuh"
#include "fft_lines.cuh"
#include "image_dtype.cuh"

namespace tio {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxParts = 1024;      // stats blocks per row
constexpr int kTableSmem = 96 << 10; // tio_spike keeps its phase tables in smem up to this size
constexpr int kSpikeLanes = 8;       // voxels per lane per work item of tio_spike (32 * 8 along K)

constexpr unsigned kSigned = 1, kNonFinite = 2;

__device__ __forceinline__ bool row_active(const float* intensity, int row, int C) {
  return intensity[row / C] != 0.0f;
}

// ---- stats --------------------------------------------------------------------------------------

// Block `p` of row `blockIdx.y` reduces a contiguous slice; the last block of the row to finish
// (ticket) adds the partials in block order, so the sum does not depend on scheduling.
template <typename T>
__global__ void __launch_bounds__(kThreads)
stats_kernel(const T* __restrict__ src, int C, int64_t vox, const float* __restrict__ intensity,
             double* __restrict__ sum, uint32_t* __restrict__ flags, double* part_sum, uint32_t* part_flags,
             uint32_t* tickets) {
  const int row = blockIdx.y, parts = gridDim.x, p = blockIdx.x;
  if (!row_active(intensity, row, C)) {
    if (p == 0 && threadIdx.x == 0) {
      sum[row] = 0.0;
      flags[row] = 0;
    }
    return;
  }
  const int64_t chunk = (vox + parts - 1) / parts;
  const int64_t lo = (int64_t)p * chunk, hi = lo + chunk < vox ? lo + chunk : vox;
  const T* x = src + (int64_t)row * vox;
  double s = 0.0;
  uint32_t f = 0;
  for (int64_t e = lo + threadIdx.x; e < hi; e += kThreads) {
    const float v = to_float(ld(x + e));
    s += (double)v;
    f |= (v < 0.0f ? kSigned : 0u) | (isfinite(v) ? 0u : kNonFinite);
  }
  __shared__ double s_sum[kThreads / 32];
  __shared__ uint32_t s_flags[kThreads / 32];
  __shared__ bool last;
  for (int o = 16; o; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    f |= __shfl_xor_sync(0xffffffffu, f, o);
  }
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  if (lane == 0) {
    s_sum[warp] = s;
    s_flags[warp] = f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    uint32_t g = 0;
    for (int w = 0; w < kThreads / 32; ++w) {
      t += s_sum[w];
      g |= s_flags[w];
    }
    part_sum[(int64_t)row * parts + p] = t;
    part_flags[(int64_t)row * parts + p] = g;
    __threadfence();
    last = atomicAdd(&tickets[row], 1u) == (unsigned)parts - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x == 0) {
    double t = 0.0;
    uint32_t g = 0;
    const volatile double* ps = part_sum + (int64_t)row * parts;
    const volatile uint32_t* pf = part_flags + (int64_t)row * parts;
    for (int q = 0; q < parts; ++q) {
      t += ps[q];
      g |= pf[q];
    }
    sum[row] = t;
    flags[row] = g;
    tickets[row] = 0;
  }
}

int stats_parts(int rows, int64_t vox) {
  int64_t parts = ((int64_t)num_sms() * 8 + rows - 1) / rows;
  const int64_t useful = (vox + 4 * kThreads - 1) / (4 * kThreads);  // at least 4 voxels per thread
  if (parts > useful) parts = useful;
  if (parts > kMaxParts) parts = kMaxParts;
  return parts < 1 ? 1 : (int)parts;
}

// ---- spectrum peak ------------------------------------------------------------------------------
//
// Lines are transformed by the shared-memory Stockham FFT of fft_lines.cuh.

__device__ __forceinline__ bool needs_fft(const float* intensity, const uint32_t* flags, int row, int C) {
  return row_active(intensity, row, C) && flags[row] == kSigned;
}

struct Geometry {
  int C, I, J, K, Kh;
  int64_t vox;
};

// K pass: real lines x[row][i][j][:] -> bins 0..K/2 of ws[row - row0][i][j][:]
template <typename T>
__global__ void __launch_bounds__(kThreads)
fft_k_kernel(const T* __restrict__ src, Geometry g, int row0, int lines, int S, FftPlan plan,
             const float* __restrict__ intensity, const uint32_t* __restrict__ flags, float2* __restrict__ ws) {
  const int row = row0 + blockIdx.y;
  if (!needs_fft(intensity, flags, row, g.C)) return;
  extern __shared__ float2 smem[];
  float2* W = smem;
  float2* a = W + plan.n;
  float2* b = a + lines * S;
  build_table(W, plan.n);
  const int64_t n_lines = (int64_t)g.I * g.J, first = (int64_t)blockIdx.x * lines;
  const T* x = src + (int64_t)row * g.vox;
  for (int e = threadIdx.x; e < lines * g.K; e += blockDim.x) {
    const int line = e / g.K, k = e - line * g.K;
    const int64_t gl = first + line;
    a[line * S + k] = make_float2(gl < n_lines ? to_float(ld(x + gl * g.K + k)) : 0.0f, 0.0f);
  }
  const float2* r = fft_lines(a, b, lines, S, plan, W);
  float2* out = ws + (int64_t)blockIdx.y * n_lines * g.Kh;
  for (int e = threadIdx.x; e < lines * g.Kh; e += blockDim.x) {
    const int line = e / g.Kh, kb = e - line * g.Kh;
    const int64_t gl = first + line;
    if (gl < n_lines) out[gl * g.Kh + kb] = r[line * S + kb];
  }
}

// J pass (reduce = 0, in place) and I pass (reduce = 1, no write): a CTA takes `lines` consecutive
// kb columns at one i (J pass) or one j (I pass), over the whole transformed axis
__global__ void __launch_bounds__(kThreads)
fft_strided_kernel(Geometry g, int row0, int lines, int S, FftPlan plan, int reduce,
                   const float* __restrict__ intensity, const uint32_t* __restrict__ flags, float2* __restrict__ ws,
                   float* __restrict__ peak) {
  const int row = row0 + blockIdx.y;
  if (!needs_fft(intensity, flags, row, g.C)) return;
  extern __shared__ float2 smem[];
  float2* W = smem;
  float2* a = W + plan.n;
  float2* b = a + lines * S;
  build_table(W, plan.n);
  const int tiles = (g.Kh + lines - 1) / lines;
  const int tile = blockIdx.x % tiles, outer = blockIdx.x / tiles;  // outer: i (J pass) or j (I pass)
  const int kb0 = tile * lines, cols = min(lines, g.Kh - kb0);
  const int n = plan.n;
  float2* base = ws + (int64_t)blockIdx.y * g.I * g.J * g.Kh;
  // element t of the line: (i, j) = (outer, t) in the J pass, (t, outer) in the I pass
  const int64_t line_stride = reduce ? (int64_t)g.J * g.Kh : g.Kh;
  base += (reduce ? (int64_t)outer * g.Kh : (int64_t)outer * g.J * g.Kh) + kb0;
  for (int e = threadIdx.x; e < n * lines; e += blockDim.x) {
    const int t = e / lines, c = e - t * lines;
    a[c * S + t] = c < cols ? base[t * line_stride + c] : make_float2(0.0f, 0.0f);
  }
  const float2* r = fft_lines(a, b, lines, S, plan, W);
  if (!reduce) {
    for (int e = threadIdx.x; e < n * lines; e += blockDim.x) {
      const int t = e / lines, c = e - t * lines;
      if (c < cols) base[t * line_stride + c] = r[c * S + t];
    }
    return;
  }
  float m = 0.0f;
  for (int e = threadIdx.x; e < n * lines; e += blockDim.x) {
    const int t = e / lines, c = e - t * lines;
    if (c < cols) {
      const float2 v = r[c * S + t];
      m = fmaxf(m, fmaf(v.x, v.x, v.y * v.y));
    }
  }
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float s_max[kThreads / 32];
  if (threadIdx.x % 32 == 0) s_max[threadIdx.x / 32] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) m = fmaxf(m, s_max[w]);
    // non-negative floats order as their bits
    atomicMax(reinterpret_cast<int*>(peak + row), __float_as_int(sqrtf(m)));
  }
}

// ---- spike --------------------------------------------------------------------------------------

// tables[b][s] = I + J + K unit phasors exp(2 pi i (f n mod L) / L) of spike s's frequency f on
// each axis (L = I, J, K); zeros for the padding after an element's list
__global__ void spike_tables_kernel(const int4* __restrict__ spikes, int B, int S, int I, int J, int K,
                                    const float* __restrict__ intensity, float2* __restrict__ tables) {
  const int per = I + J + K;
  const int64_t total = (int64_t)B * S * per;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t bs = e / per;
    const int t = (int)(e - bs * per);
    const int b = (int)(bs / S);
    const int4 sp = spikes[bs];
    if (!sp.w || intensity[b] == 0.0f) {
      tables[e] = make_float2(0.0f, 0.0f);
      continue;
    }
    int f, n, L;
    if (t < I) f = sp.x, n = t, L = I;
    else if (t < I + J) f = sp.y, n = t - I, L = J;
    else f = sp.z, n = t - I - J, L = K;
    const long long m = ((long long)f * n) % L;  // 0 <= f < L
    double s, c;
    sincospi(2.0 * (double)m / (double)L, &s, &c);
    tables[e] = make_float2((float)c, (float)s);
  }
}

// A warp takes 256 consecutive voxels of one K line (lane + 32 v, v < 8).  Per spike the lane forms
// q = eI[i] eJ[j] once and adds Re(q eK[k]) for each of its voxels.
template <typename T>
__global__ void __launch_bounds__(kThreads)
spike_kernel(T* data, Geometry g, const int4* __restrict__ spikes, int S, const float* __restrict__ intensity,
             const double* __restrict__ sum, const uint32_t* __restrict__ flags, const float* __restrict__ peak,
             const float2* __restrict__ tables, int tables_in_smem) {
  const int row = blockIdx.y, b = row / g.C;
  const float ratio = intensity[b];
  if (ratio == 0.0f) return;  // not active: no byte moves
  const uint32_t f = flags[row];
  const double amp = f & kSigned ? (double)peak[row] : sum[row];
  const float A = (float)(amp * (double)ratio / ((double)g.I * g.J * g.K));
  const int per = g.I + g.J + g.K;
  const float2* tab = tables + (int64_t)b * S * per;
  extern __shared__ float2 s_tab[];
  if (tables_in_smem) {
    for (int e = threadIdx.x; e < S * per; e += blockDim.x) s_tab[e] = tab[e];
    __syncthreads();
    tab = s_tab;
  }
  int n_spikes = 0;
  while (n_spikes < S && spikes[(int64_t)b * S + n_spikes].w) ++n_spikes;
  const int kblocks = (g.K + 32 * kSpikeLanes - 1) / (32 * kSpikeLanes);
  const int64_t items = (int64_t)g.I * g.J * kblocks;
  const int64_t per_block = (items + gridDim.x - 1) / gridDim.x;
  const int64_t lo = (int64_t)blockIdx.x * per_block, hi = lo + per_block < items ? lo + per_block : items;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  T* x = data + (int64_t)row * g.vox;
  const float nan = __int_as_float(0x7fffffff);
  for (int64_t item = lo + warp; item < hi; item += kThreads / 32) {
    const int64_t line = item / kblocks;
    const int k0 = (int)(item - line * kblocks) * 32 * kSpikeLanes + lane;
    T* p = x + line * g.K;
    if (f & kNonFinite) {  // the reference's FFT spreads a NaN or an Inf over the whole row
#pragma unroll
      for (int v = 0; v < kSpikeLanes; ++v)
        if (k0 + 32 * v < g.K) p[k0 + 32 * v] = from_float<T>(nan);
      continue;
    }
    const int i = (int)(line / g.J), j = (int)(line - (int64_t)i * g.J);
    float in[kSpikeLanes], acc[kSpikeLanes];
#pragma unroll
    for (int v = 0; v < kSpikeLanes; ++v) {
      const int k = k0 + 32 * v;
      in[v] = k < g.K ? to_float(p[k]) : 0.0f;
      acc[v] = 0.0f;
    }
    for (int s = 0; s < n_spikes; ++s) {
      const float2* t = tab + s * per;
      const float2 q = cmul(t[i], t[g.I + j]);
      const float2* tk = t + g.I + g.J;
#pragma unroll
      for (int v = 0; v < kSpikeLanes; ++v) {
        const int k = k0 + 32 * v;
        if (k < g.K) {
          const float2 e = tk[k];
          acc[v] = fmaf(q.x, e.x, fmaf(-q.y, e.y, acc[v]));
        }
      }
    }
#pragma unroll
    for (int v = 0; v < kSpikeLanes; ++v) {
      const int k = k0 + 32 * v;
      if (k < g.K) p[k] = from_float<T>(fmaf(A, acc[v], in[v]));
    }
  }
}

int check_shape(const char* name, int B, int C, int I, int J, int K) {
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "%s: bad shape (%d, %d, %d, %d, %d)", name, B, C, I,
                J, K);
  TIO_CHECK_ARG((int64_t)B * C <= 65535, "%s: %lld rows (B * C), at most 65535", name, (long long)B * C);
  return 0;
}

}  // namespace

}  // namespace tio

extern "C" size_t tio_spike_stats_workspace_bytes(int rows) {
  if (rows <= 0) return 0;
  return (size_t)rows * (tio::kMaxParts * (sizeof(double) + sizeof(uint32_t)) + sizeof(uint32_t));
}

extern "C" int tio_spike_stats(const void* src, int dtype, int B, int C, int64_t vox, const float* intensity,
                               double* sum, uint32_t* flags, void* workspace, size_t workspace_bytes,
                               void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && intensity && sum && flags && workspace, "tio_spike_stats: null pointer");
  TIO_CHECK_ARG(B > 0 && C > 0 && vox > 0, "tio_spike_stats: bad shape (B %d, C %d, %lld voxels)", B, C,
                (long long)vox);
  TIO_CHECK_ARG((int64_t)B * C <= 65535, "tio_spike_stats: %lld rows (B * C), at most 65535", (long long)B * C);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_spike_stats: unknown dtype %d", dtype);
  const int rows = B * C;
  TIO_CHECK_ARG(workspace_bytes >= tio_spike_stats_workspace_bytes(rows), "tio_spike_stats: workspace of %zu bytes, %zu needed",
                workspace_bytes, tio_spike_stats_workspace_bytes(rows));
  cudaStream_t st = (cudaStream_t)stream;
  double* part_sum = (double*)workspace;
  uint32_t* part_flags = (uint32_t*)(part_sum + (size_t)rows * kMaxParts);
  uint32_t* tickets = part_flags + (size_t)rows * kMaxParts;
  TIO_CHECK_CUDA(cudaMemsetAsync(tickets, 0, (size_t)rows * sizeof(uint32_t), st));
  const dim3 grid((unsigned)stats_parts(rows, vox), (unsigned)rows);
#define TIO_STATS(T)                                                                                     \
  stats_kernel<T><<<grid, kThreads, 0, st>>>((const T*)src, C, vox, intensity, sum, flags, part_sum, \
                                             part_flags, tickets);                                   \
  launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_spike_stats", TIO_STATS)
#undef TIO_STATS
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_spectrum_peak(const void* src, int dtype, int B, int C, int I, int J, int K,
                                 const float* intensity, const uint32_t* flags, float* peak, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && intensity && flags && peak && workspace, "tio_spectrum_peak: null pointer");
  if (check_shape("tio_spectrum_peak", B, C, I, J, K)) return 1;
  TIO_CHECK_ARG(I <= kMaxAxis && J <= kMaxAxis && K <= kMaxAxis,
                "tio_spectrum_peak: axis of %d points, at most %d", I > J ? (I > K ? I : K) : (J > K ? J : K), kMaxAxis);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_spectrum_peak: unknown dtype %d", dtype);
  const size_t row_bytes = (size_t)I * J * (K / 2 + 1) * sizeof(float2);
  const int64_t chunk64 = (int64_t)(workspace_bytes / row_bytes);
  TIO_CHECK_ARG(chunk64 >= 1, "tio_spectrum_peak: workspace of %zu bytes, one row needs %zu", workspace_bytes,
                row_bytes);
  const int rows = B * C, chunk = chunk64 < rows ? (int)chunk64 : rows;
  const Geometry g = {C, I, J, K, K / 2 + 1, (int64_t)I * J * K};
  const FftPlan pk = make_plan(K), pj = make_plan(J), pi = make_plan(I);
  const int lk = fft_lines_for(K), lj = fft_lines_for(J), li = fft_lines_for(I);
  const size_t sk = fft_smem(K, lk), sj = fft_smem(J, lj), si = fft_smem(I, li);
  const int64_t k_blocks = ((int64_t)I * J + lk - 1) / lk;
  const int64_t j_blocks = (int64_t)I * ((g.Kh + lj - 1) / lj), i_blocks = (int64_t)J * ((g.Kh + li - 1) / li);
  TIO_CHECK_ARG(k_blocks < (1ll << 31) && j_blocks < (1ll << 31) && i_blocks < (1ll << 31),
                "tio_spectrum_peak: too many lines");
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(peak, 0, (size_t)rows * sizeof(float), st));
  TIO_CHECK_CUDA(cudaFuncSetAttribute(fft_strided_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)(sj > si ? sj : si)));
  float2* ws = (float2*)workspace;
  for (int row0 = 0; row0 < rows; row0 += chunk) {
    const int n = rows - row0 < chunk ? rows - row0 : chunk;
#define TIO_FFT_K(T)                                                                                     \
  TIO_CHECK_CUDA(cudaFuncSetAttribute(fft_k_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sk)); \
  fft_k_kernel<T><<<dim3((unsigned)k_blocks, (unsigned)n), kThreads, sk, st>>>((const T*)src, g, row0, lk,    \
                                                                               line_stride(K), pk, intensity, \
                                                                               flags, ws);                    \
  launched()
    TIO_IMAGE_DISPATCH(dtype, "tio_spectrum_peak", TIO_FFT_K)
#undef TIO_FFT_K
    fft_strided_kernel<<<dim3((unsigned)j_blocks, (unsigned)n), kThreads, sj, st>>>(
        g, row0, lj, line_stride(J), pj, 0, intensity, flags, ws, peak);
    launched();
    fft_strided_kernel<<<dim3((unsigned)i_blocks, (unsigned)n), kThreads, si, st>>>(
        g, row0, li, line_stride(I), pi, 1, intensity, flags, ws, peak);
    launched();
    TIO_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int tio_spike(void* data, int dtype, int B, int C, int I, int J, int K, const int32_t* spikes, int S,
                         const float* intensity, const double* sum, const uint32_t* flags, const float* peak,
                         void* tables, size_t tables_bytes, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(data && spikes && intensity && sum && flags && peak && tables, "tio_spike: null pointer");
  if (check_shape("tio_spike", B, C, I, J, K)) return 1;
  TIO_CHECK_ARG(S > 0, "tio_spike: %d spikes per element", S);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_spike: unknown dtype %d", dtype);
  const size_t need = (size_t)B * S * ((size_t)I + J + K) * sizeof(float2);
  TIO_CHECK_ARG(tables_bytes >= need, "tio_spike: tables of %zu bytes, %zu needed", tables_bytes, need);
  const Geometry g = {C, I, J, K, K / 2 + 1, (int64_t)I * J * K};
  const int64_t kblocks = (K + 32 * kSpikeLanes - 1) / (32 * kSpikeLanes);
  const int64_t items = (int64_t)I * J * kblocks;
  const int rows = B * C;
  int64_t parts = ((int64_t)num_sms() * 8 + rows - 1) / rows;
  const int64_t useful = (items + 4 * (kThreads / 32) - 1) / (4 * (kThreads / 32));  // >= 4 items per warp
  if (parts > useful) parts = useful;
  if (parts < 1) parts = 1;
  const size_t smem = (size_t)S * (I + J + K) * sizeof(float2);
  const int in_smem = smem <= (size_t)kTableSmem;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t table_entries = (int64_t)B * S * (I + J + K);
  spike_tables_kernel<<<(unsigned)((table_entries + kThreads - 1) / kThreads < 4096
                                       ? (table_entries + kThreads - 1) / kThreads
                                       : 4096),
                        kThreads, 0, st>>>((const int4*)spikes, B, S, I, J, K, intensity, (float2*)tables);
  launched();
  const dim3 grid((unsigned)parts, (unsigned)rows);
#define TIO_SPIKE(T)                                                                                        \
  if (in_smem)                                                                                              \
    TIO_CHECK_CUDA(cudaFuncSetAttribute(spike_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
  spike_kernel<T><<<grid, kThreads, in_smem ? smem : 0, st>>>((T*)data, g, (const int4*)spikes, S, intensity, sum, \
                                                              flags, peak, (const float2*)tables, in_smem); \
  launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_spike", TIO_SPIKE)
#undef TIO_SPIKE
  TIO_CHECK_LAUNCH();
  return 0;
}

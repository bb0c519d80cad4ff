// pca.cu — PCA of TorchIO 2.0.0a2 (transforms/intensity/pca.py) on the GPU.
//
// The reference runs torch.pca_lowrank on A = (voxels x channels) fp32 minus its channel means:
// a Gaussian sketch, QRs of tall N x q matrices, an SVD of q x C, then A @ V.  Every step depends
// on A only through products G W with G = A^T A and W a small C x q matrix, so the volume is read
// by three kinds of pass and the C x q algebra between them runs on the host (transforms/pca.py):
//
// tio_pca_mean        per (b, c) fp64 mean of float(x)
// tio_pca_gram_apply  per b, G W_b = sum_v d_v (d_v^T W_b) with d_v = float(x_v) - mean, fp64
// tio_pca_project     y[b, k] = clip(sum_c (x_c - mean_c) coef[b, c, k] + offset), fp32
//
// Both reductions are deterministic: each block reduces a fixed slice in a fixed order into its own
// partial, and the last block of a row or element to finish (ticket) adds the partials in block
// order.  No float atomics, so the same input gives the same bits.
#include <cmath>

#include "common.cuh"
#include "image_dtype.cuh"

namespace tio {

namespace {

constexpr int kThreads = 256;
constexpr int kMaxParts = 1024;              // blocks per mean row or gram element
constexpr int kChunkValues = 4096;           // staged (channel, voxel) values of a gram chunk
constexpr int kMaxTile = 1024;               // voxels per gram tile
constexpr size_t kTBytes = 96 << 10;         // bound of the per-tile t = d^T W table
constexpr size_t kAccSmemBytes = 48 << 10;   // block accumulators live in smem up to this size
constexpr int kMaxComponents = (int)(kTBytes / (2 * sizeof(double)));  // q at a one-voxel tile
constexpr int kProjectGroup = 4;             // components a projecting thread accumulates at once

int pow2_floor(int64_t v) {
  int p = 1;
  while ((int64_t)p * 2 <= v) p *= 2;
  return p;
}

// ---- mean ---------------------------------------------------------------------------------------

template <typename T>
__global__ void __launch_bounds__(kThreads)
mean_kernel(const T* __restrict__ src, int64_t vox, double* __restrict__ mean, double* part,
            uint32_t* tickets) {
  const int64_t row = blockIdx.x;
  const int parts = gridDim.y, p = blockIdx.y;
  const int64_t chunk = (vox + parts - 1) / parts;
  const int64_t lo = (int64_t)p * chunk, hi = lo + chunk < vox ? lo + chunk : vox;
  const T* x = src + row * vox;
  double s = 0.0;
  for (int64_t e = lo + threadIdx.x; e < hi; e += kThreads) s += (double)to_float(ld(x + e));
  __shared__ double s_sum[kThreads / 32];
  __shared__ bool last;
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x % 32 == 0) s_sum[threadIdx.x / 32] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kThreads / 32; ++w) t += s_sum[w];
    part[row * parts + p] = t;
    __threadfence();
    last = atomicAdd(&tickets[row], 1u) == (unsigned)parts - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double t = 0.0;
  const volatile double* ps = part + row * parts;
  for (int q = 0; q < parts; ++q) t += ps[q];
  mean[row] = t / (double)vox;
}

int mean_parts(int64_t rows, int64_t vox) {
  int64_t parts = ((int64_t)num_sms() * 8 + rows - 1) / rows;
  const int64_t useful = (vox + 4 * kThreads - 1) / (4 * kThreads);  // at least 4 voxels per thread
  if (parts > useful) parts = useful;
  if (parts > kMaxParts) parts = kMaxParts;
  return parts < 1 ? 1 : (int)parts;
}

// ---- G W ----------------------------------------------------------------------------------------
//
// A block owns a run of tiles of V voxels of one element.  Per tile, pass 1 streams the channels in
// chunks of CT through shared memory and builds t[k][v] = sum_c d[c][v] W[c][k]; pass 2 streams them
// again (from L2: a tile is at most 16 KiB of fp32 per chunk) and adds acc[c][k] += sum_v d[c][v]
// t[k][v].  In pass 2 each (c, k) pair is summed by S lanes over interleaved voxels and reduced by
// shuffles, so that a few pairs still keep the block busy.  Rows of d and t are padded to V + 1.

struct GramShape {
  int C, q, V, CT, S;
  int64_t vox, tiles_per_block;
  int acc_in_smem;
};

GramShape gram_shape(int B, int C, int q, int64_t vox) {
  GramShape g{};
  g.C = C;
  g.q = q;
  g.vox = vox;
  int V = pow2_floor(kChunkValues / C > 1 ? kChunkValues / C : 1);
  if (V > kMaxTile) V = kMaxTile;
  while (V > 1 && (size_t)q * (V + 1) * sizeof(double) > kTBytes) V /= 2;
  g.V = V;
  g.CT = kChunkValues / V < C ? kChunkValues / V : C;
  const int64_t pairs = (int64_t)g.CT * q;
  int S = pairs >= kThreads ? 1 : pow2_floor(kThreads / pairs);
  g.S = S > 32 ? 32 : S;
  const int64_t tiles = (vox + V - 1) / V;
  int64_t parts = ((int64_t)num_sms() * 4 + B - 1) / B;
  if (parts > tiles) parts = tiles;
  if (parts > kMaxParts) parts = kMaxParts;
  if (parts < 1) parts = 1;
  g.tiles_per_block = (tiles + parts - 1) / parts;
  g.acc_in_smem = (size_t)C * q * sizeof(double) <= kAccSmemBytes;
  return g;
}

int64_t gram_parts(const GramShape& g) {
  const int64_t tiles = (g.vox + g.V - 1) / g.V;
  return (tiles + g.tiles_per_block - 1) / g.tiles_per_block;
}

size_t gram_smem(const GramShape& g) {
  size_t n = (size_t)g.CT * (g.V + 1) + (size_t)g.q * (g.V + 1);
  if (g.acc_in_smem) n += (size_t)g.C * g.q;
  return n * sizeof(double);
}

template <typename T>
__device__ __forceinline__ void stage_chunk(double* d, const T* x, const double* mu, const GramShape& g, int c0,
                                            int nc, int64_t v0, int nv) {
  const int V = g.V;
  for (int e = threadIdx.x; e < g.CT * V; e += kThreads) {
    const int c = e / V, v = e - c * V;
    double value = 0.0;
    if (c < nc && v < nv) value = (double)to_float(ld(x + (int64_t)(c0 + c) * g.vox + v0 + v)) - mu[c0 + c];
    d[c * (V + 1) + v] = value;
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
gram_kernel(const T* __restrict__ src, const double* __restrict__ mean, const double* __restrict__ w_all,
            double* __restrict__ out, double* part, uint32_t* tickets, GramShape g) {
  extern __shared__ double smem[];
  const int b = blockIdx.y, p = blockIdx.x, parts = gridDim.x;
  const int C = g.C, q = g.q, V = g.V, S = g.S;
  const int64_t cq = (int64_t)C * q;
  double* d = smem;                               // [CT][V + 1]
  double* t = d + (size_t)g.CT * (V + 1);         // [q][V + 1]
  double* slot = part + ((int64_t)b * parts + p) * cq;
  double* acc = g.acc_in_smem ? t + (size_t)q * (V + 1) : slot;
  const T* x = src + (int64_t)b * C * g.vox;
  const double* mu = mean + (int64_t)b * C;
  const double* w = w_all + (int64_t)b * cq;
  for (int64_t e = threadIdx.x; e < cq; e += kThreads) acc[e] = 0.0;

  const int groups = kThreads / S, lane = threadIdx.x % S;
  const int64_t tiles = (g.vox + V - 1) / V;
  const int64_t t0 = (int64_t)p * g.tiles_per_block;
  const int64_t t1 = t0 + g.tiles_per_block < tiles ? t0 + g.tiles_per_block : tiles;
  for (int64_t tile = t0; tile < t1; ++tile) {
    const int64_t v0 = tile * V;
    const int nv = g.vox - v0 < V ? (int)(g.vox - v0) : V;
    __syncthreads();  // the previous tile's pass 2 is done with t
    for (int e = threadIdx.x; e < q * V; e += kThreads) t[(e / V) * (V + 1) + e % V] = 0.0;
    // pass 1: t[k][v] = sum_c d[c][v] W[c][k]
    for (int c0 = 0; c0 < C; c0 += g.CT) {
      const int nc = C - c0 < g.CT ? C - c0 : g.CT;
      __syncthreads();
      stage_chunk(d, x, mu, g, c0, nc, v0, nv);
      __syncthreads();
      for (int e = threadIdx.x; e < q * V; e += kThreads) {
        const int k = e / V, v = e - k * V;
        double s = t[k * (V + 1) + v];
        for (int c = 0; c < nc; ++c) s = fma(d[c * (V + 1) + v], __ldg(w + (int64_t)(c0 + c) * q + k), s);
        t[k * (V + 1) + v] = s;
      }
    }
    // pass 2: acc[c][k] += sum_v d[c][v] t[k][v]
    for (int c0 = 0; c0 < C; c0 += g.CT) {
      const int nc = C - c0 < g.CT ? C - c0 : g.CT;
      __syncthreads();
      stage_chunk(d, x, mu, g, c0, nc, v0, nv);
      __syncthreads();
      const int pairs = nc * q;
      const int rounds = (pairs + groups - 1) / groups;
      for (int r = 0; r < rounds; ++r) {
        const int e = r * groups + threadIdx.x / S;
        double s = 0.0;
        int c = 0, k = 0;
        if (e < pairs) {
          c = e / q;
          k = e - c * q;
          const double* dc = d + c * (V + 1);
          const double* tk = t + k * (V + 1);
          for (int v = lane; v < nv; v += S) s = fma(dc[v], tk[v], s);
        }
        for (int o = S / 2; o; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o, S);
        if (e < pairs && lane == 0) acc[(int64_t)(c0 + c) * q + k] += s;
      }
    }
  }
  __syncthreads();
  __shared__ bool last;
  if (g.acc_in_smem)
    for (int64_t e = threadIdx.x; e < cq; e += kThreads) slot[e] = acc[e];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&tickets[b], 1u) == (unsigned)parts - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  const volatile double* pb = part + (int64_t)b * parts * cq;
  for (int64_t e = threadIdx.x; e < cq; e += kThreads) {
    double s = 0.0;
    for (int r = 0; r < parts; ++r) s += pb[r * cq + e];
    out[(int64_t)b * cq + e] = s;
  }
}

// ---- projection ---------------------------------------------------------------------------------

template <typename T>
__global__ void __launch_bounds__(kThreads)
project_kernel(const T* __restrict__ src, int B, int C, int64_t vox, int q, const double* __restrict__ mean,
               const float* __restrict__ coef, float offset, int clip, float* __restrict__ out) {
  const int64_t total = (int64_t)B * vox;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < total; e += (int64_t)gridDim.x * kThreads) {
    const int64_t b = e / vox, v = e - b * vox;
    const T* x = src + b * C * vox + v;
    const double* mu = mean + b * C;
    const float* cf = coef + b * C * q;
    float* y = out + b * q * vox + v;
    for (int k0 = 0; k0 < q; k0 += kProjectGroup) {
      float acc[kProjectGroup] = {0.0f, 0.0f, 0.0f, 0.0f};
      const int nk = q - k0 < kProjectGroup ? q - k0 : kProjectGroup;
#pragma unroll 4
      for (int c = 0; c < C; ++c) {
        const float d = __fsub_rn(to_float(ld(x + (int64_t)c * vox)), (float)mu[c]);
        const float* row = cf + (int64_t)c * q + k0;
#pragma unroll
        for (int j = 0; j < kProjectGroup; ++j)
          if (j < nk) acc[j] = __fmaf_rn(d, __ldg(row + j), acc[j]);
      }
#pragma unroll
      for (int j = 0; j < kProjectGroup; ++j) {
        if (j >= nk) break;
        float r = __fadd_rn(acc[j], offset);
        if (clip) r = r < 0.0f ? 0.0f : (r > 1.0f ? 1.0f : r);  // NaN stays NaN, as torch.clamp
        y[(int64_t)(k0 + j) * vox] = r;
      }
    }
  }
}

int check_common(const char* name, const void* src, int dtype, int B, int C, int64_t vox) {
  TIO_CHECK_ARG(src, "%s: null pointer", name);
  TIO_CHECK_ARG(B > 0 && C > 0 && vox > 0, "%s: bad shape B=%d C=%d vox=%lld", name, B, C, (long long)vox);
  TIO_CHECK_ARG(B <= 65535, "%s: %d elements, at most 65535", name, B);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "%s: unknown dtype %d", name, dtype);
  return 0;
}

size_t mean_workspace(int B, int C, int64_t vox) {
  const int64_t rows = (int64_t)B * C;
  return (size_t)rows * mean_parts(rows, vox) * sizeof(double) + (size_t)rows * sizeof(uint32_t);
}

size_t gram_workspace(int B, int C, int q, int64_t vox) {
  const GramShape g = gram_shape(B, C, q, vox);
  return (size_t)B * gram_parts(g) * C * q * sizeof(double) + (size_t)B * sizeof(uint32_t);
}

}  // namespace

}  // namespace tio

extern "C" size_t tio_pca_workspace_bytes(int B, int C, int q, int64_t vox) {
  using namespace tio;
  if (B <= 0 || C <= 0 || q <= 0 || vox <= 0) return 0;
  const size_t a = mean_workspace(B, C, vox), b = gram_workspace(B, C, q, vox);
  return a > b ? a : b;
}

extern "C" int tio_pca_mean(const void* src, int dtype, int B, int C, int64_t vox, double* mean, void* workspace,
                            size_t workspace_bytes, void* stream) {
  using namespace tio;
  if (check_common("tio_pca_mean", src, dtype, B, C, vox)) return 1;
  TIO_CHECK_ARG(mean && workspace, "tio_pca_mean: null pointer");
  const size_t need = mean_workspace(B, C, vox);
  TIO_CHECK_ARG(workspace_bytes >= need, "tio_pca_mean: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  const int64_t rows = (int64_t)B * C;
  TIO_CHECK_ARG(rows <= 0x7fffffff, "tio_pca_mean: %lld rows (B * C)", (long long)rows);
  const int parts = mean_parts(rows, vox);
  double* part = (double*)workspace;
  uint32_t* tickets = (uint32_t*)(part + rows * parts);
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(tickets, 0, (size_t)rows * sizeof(uint32_t), st));
  const dim3 grid((unsigned)rows, (unsigned)parts);
#define TIO_PCA_MEAN(T)                                                                        \
  mean_kernel<T><<<grid, kThreads, 0, st>>>((const T*)src, vox, mean, part, tickets); \
  launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_pca_mean", TIO_PCA_MEAN)
#undef TIO_PCA_MEAN
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_pca_gram_apply(const void* src, int dtype, int B, int C, int64_t vox, int q, const double* mean,
                                  const double* w, double* out, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  using namespace tio;
  if (check_common("tio_pca_gram_apply", src, dtype, B, C, vox)) return 1;
  TIO_CHECK_ARG(mean && w && out && workspace, "tio_pca_gram_apply: null pointer");
  TIO_CHECK_ARG(q >= 1 && q <= kMaxComponents, "tio_pca_gram_apply: %d columns, 1 to %d supported", q,
                kMaxComponents);
  const size_t need = gram_workspace(B, C, q, vox);
  TIO_CHECK_ARG(workspace_bytes >= need, "tio_pca_gram_apply: workspace of %zu bytes, %zu needed",
                workspace_bytes, need);
  const GramShape g = gram_shape(B, C, q, vox);
  const int64_t parts = gram_parts(g);
  double* part = (double*)workspace;
  uint32_t* tickets = (uint32_t*)(part + (size_t)B * parts * C * q);
  const size_t smem = gram_smem(g);
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(tickets, 0, (size_t)B * sizeof(uint32_t), st));
  const dim3 grid((unsigned)parts, (unsigned)B);
#define TIO_PCA_GRAM(T)                                                                                      \
  TIO_CHECK_CUDA(cudaFuncSetAttribute(gram_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
  gram_kernel<T><<<grid, kThreads, smem, st>>>((const T*)src, mean, w, out, part, tickets, g);              \
  launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_pca_gram_apply", TIO_PCA_GRAM)
#undef TIO_PCA_GRAM
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_pca_project(const void* src, int dtype, int B, int C, int64_t vox, int q, const double* mean,
                               const float* coef, float offset, int clip, float* out, void* stream) {
  using namespace tio;
  if (check_common("tio_pca_project", src, dtype, B, C, vox)) return 1;
  TIO_CHECK_ARG(mean && coef && out, "tio_pca_project: null pointer");
  TIO_CHECK_ARG(q >= 1, "tio_pca_project: %d components", q);
  const int64_t total = (int64_t)B * vox;
  int64_t blocks = (total + kThreads - 1) / kThreads;
  if (blocks > (int64_t)num_sms() * 16) blocks = (int64_t)num_sms() * 16;
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_PCA_PROJECT(T)                                                                                       \
  project_kernel<T><<<(unsigned)blocks, kThreads, 0, st>>>((const T*)src, B, C, vox, q, mean, coef, offset, clip, \
                                                           out);                                                 \
  launched()
  TIO_IMAGE_DISPATCH(dtype, "tio_pca_project", TIO_PCA_PROJECT)
#undef TIO_PCA_PROJECT
  TIO_CHECK_LAUNCH();
  return 0;
}

// stats.cu — data-derived parameters and the affine epilogue of Normalize / Standardize
// (SURVEY §8 f-3; transforms/intensity/normalize.py:104-232,332-366, standardize.py:52-107,
// _statistics.py:11-45 of TorchIO 2.0.0a2).
//
// The reference derives its parameters from batch element 0 on the host:
//   Standardize: values.float().mean() / .std()      (all channels of sample 0, optional mask)
//   Normalize:   two quantiles of the same values via torch.kthvalue + lerp
// and then applies `(x - mean) / std` or `(clamp(x) - in_min) / in_range * out_range + out_min`
// as separate fp32 elementwise ops over the whole batch.
//
//   tio_moments    one pass: count, sum, sum of squares (fp64 accumulators) of the selected voxels
//   tio_quantiles  exact order statistics by a 3-level radix select on the order-preserving
//                  integer image of fp32 (11 + 11 + 10 bits): three streaming passes over the
//                  sample instead of a sort; returns the two neighbours of each quantile and the
//                  interpolation weight, i.e. exactly what kthvalue(lower+1), kthvalue(lower+2)
//                  and `index - lower` give
//   tio_rescale    dst = ((clamp(x, lo, hi) - sub[b]) / div[b]) * mul[b] + add[b], every step
//                  rounded like the reference's separate fp32 ops (bit-exact given equal constants)
// All three are single-pass HBM streams (4 or 8 bytes per voxel), 128-bit loads.
#include "common.cuh"

namespace tio {

__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ---- moments ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
moments_kernel(const float* __restrict__ src, const uint8_t* __restrict__ mask, int64_t n, double* out) {
  double s = 0.0, ss = 0.0;
  long long cnt = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (!mask && ((uintptr_t)src & 15) == 0) {
    const float4* p = reinterpret_cast<const float4*>(src);
    for (int64_t t = t0; t < (n >> 2); t += stride) {
      const float4 v = __ldg(p + t);
      s += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
      ss += ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w);
      cnt += 4;
    }
    for (int64_t t = (n & ~(int64_t)3) + t0; t < n; t += stride) { const double v = src[t]; s += v; ss += v * v; ++cnt; }
  } else {
    for (int64_t t = t0; t < n; t += stride)
      if (!mask || mask[t]) { const double v = src[t]; s += v; ss += v * v; ++cnt; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  __shared__ double ps[8], pss[8];
  __shared__ long long pc[8];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { ps[w] = s; pss[w] = ss; pc[w] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int t = 1; t < 8; ++t) { s += ps[t]; ss += pss[t]; cnt += pc[t]; }
    atomicAdd(out + 0, s);
    atomicAdd(out + 1, ss);
    atomicAdd(out + 2, (double)cnt);
  }
}

// ---- radix select ----------------------------------------------------------------------
constexpr int kMaxQ = 2;        // quantiles per call
constexpr int kTargets = 2 * kMaxQ;  // ranks: lower and upper neighbour of each
struct SelectState {
  long long count;              // selected voxels
  long long rank[kTargets];     // residual rank inside the current prefix
  unsigned prefix[kTargets];    // key bits fixed so far (left aligned per level)
  double weight[kMaxQ];
  int m;                        // quantiles requested
};

template <int LEVEL>  // 0: bits 31..21 (no prefix), 1: bits 20..10, 2: bits 9..0
__global__ void __launch_bounds__(256)
select_hist_kernel(const float* __restrict__ src, const uint8_t* __restrict__ mask, int64_t n,
                   const SelectState* __restrict__ st, unsigned* __restrict__ hist /* [targets][2048] */) {
  constexpr int BINS = LEVEL == 2 ? 1024 : 2048;
  constexpr int T = LEVEL == 0 ? 1 : kTargets;
  __shared__ unsigned h[T * BINS];
  for (int t = threadIdx.x; t < T * BINS; t += blockDim.x) h[t] = 0;
  unsigned pre[kTargets];
  int nt = 1;
  if (LEVEL > 0) {
    nt = 2 * st->m;
#pragma unroll
    for (int t = 0; t < kTargets; ++t) pre[t] = st->prefix[t];
  }
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) {
    if (mask && !mask[t]) continue;
    const uint32_t k = order_key(__ldg(src + t));
    if (LEVEL == 0) {
      atomicAdd(&h[k >> 21], 1u);
    } else {
#pragma unroll
      for (int q = 0; q < kTargets; ++q) {
        if (q >= nt) break;
        if (LEVEL == 1) { if ((k >> 21) == pre[q]) atomicAdd(&h[q * BINS + ((k >> 10) & 2047u)], 1u); }
        else            { if ((k >> 10) == pre[q]) atomicAdd(&h[q * BINS + (k & 1023u)], 1u); }
      }
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < T * BINS; t += blockDim.x)
    if (h[t]) atomicAdd(&hist[t / BINS * 2048 + t % BINS], h[t]);
}

// one warp per target walks the histogram to the bin that holds the target's rank
__global__ void select_init_kernel(SelectState* st, int m) {
  st->count = 0;
  st->m = m;
  for (int t = 0; t < kTargets; ++t) { st->rank[t] = 0; st->prefix[t] = 0; }
  for (int t = 0; t < kMaxQ; ++t) st->weight[t] = 0.0;
}

template <int LEVEL>
__global__ void select_scan_kernel(SelectState* st, unsigned* hist, double q0, double q1, long long n_all, int masked) {
  const double q[kMaxQ] = {q0, q1};
  constexpr int BINS = LEVEL == 2 ? 1024 : 2048;
  const int t = threadIdx.x;  // target
  if (LEVEL == 0 && t == 0) {
    long long c = 0;
    if (masked) for (int b = 0; b < BINS; ++b) c += hist[b];
    else c = n_all;
    st->count = c;
  }
  __syncthreads();
  if (t >= 2 * st->m) return;
  if (LEVEL == 0) {
    // _statistics.py:37-45: index = q * (n - 1); lower = floor(index); weight = index - lower
    const long long c = st->count;
    const double index = q[t >> 1] * (double)(c > 0 ? c - 1 : 0);
    const long long lower = (long long)floor(index);
    st->weight[t >> 1] = index - (double)lower;
    long long r = lower + (t & 1);
    if (r > c - 1) r = c - 1;
    if (r < 0) r = 0;
    st->rank[t] = r;
  }
  const unsigned* h = hist + (LEVEL == 0 ? 0 : t * 2048);
  long long r = st->rank[t];
  int b = 0;
  for (; b < BINS - 1; ++b) {
    const unsigned c = h[b];
    if (r < (long long)c) break;
    r -= c;
  }
  st->rank[t] = r;
  st->prefix[t] = LEVEL == 0 ? (unsigned)b : (LEVEL == 1 ? ((st->prefix[t] << 11) | (unsigned)b)
                                                          : ((st->prefix[t] << 10) | (unsigned)b));
}

__global__ void select_finish_kernel(const SelectState* st, float* values, double* weights, double* count) {
  const int t = threadIdx.x;
  if (t < 2 * st->m) values[t] = key_value(st->prefix[t]);
  if (t < st->m) weights[t] = st->weight[t];
  if (t == 0) *count = (double)st->count;
}

// ---- rescale ---------------------------------------------------------------------------
// flags: 1 clamp, 2 sub, 4 div, 8 mul, 16 add; keep[b] == 0 -> copy the row
template <int V>
__global__ void __launch_bounds__(256)
rescale_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t per_elem, float lo, float hi,
               const float* __restrict__ sub, const float* __restrict__ div, const float* __restrict__ mul,
               const float* __restrict__ add, const uint8_t* __restrict__ keep, int flags) {
  const int b = blockIdx.y;
  const float* x = src + (int64_t)b * per_elem;
  float* y = dst + (int64_t)b * per_elem;
  const bool copy = keep && !keep[b];
  const float fs = sub ? sub[b] : 0.f, fd = div ? div[b] : 1.f, fm = mul ? mul[b] : 1.f, fa = add ? add[b] : 0.f;
  auto f = [&](float v) {
    if (copy) return v;
    if (flags & 1) v = fminf(fmaxf(v, lo), hi);  // Tensor.clamp(min, max)
    if (flags & 2) v = __fsub_rn(v, fs);
    if (flags & 4) v = __fdiv_rn(v, fd);
    if (flags & 8) v = __fmul_rn(v, fm);
    if (flags & 16) v = __fadd_rn(v, fa);
    return v;
  };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (V == 4) {
    const float4* p = reinterpret_cast<const float4*>(x);
    float4* o = reinterpret_cast<float4*>(y);
    for (int64_t t = t0; t < (per_elem >> 2); t += stride) {
      float4 v = __ldg(p + t);
      v.x = f(v.x); v.y = f(v.y); v.z = f(v.z); v.w = f(v.w);
      o[t] = v;
    }
  } else {
    for (int64_t t = t0; t < per_elem; t += stride) y[t] = f(__ldg(x + t));
  }
}

}  // namespace tio

using namespace tio;

extern "C" int tio_moments(const float* src, const uint8_t* mask, int64_t n, double* out3, void* stream) {
  TIO_CHECK_ARG(src && out3 && n > 0, "tio_moments: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(out3, 0, 3 * sizeof(double), st));
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  if (blocks < 1) blocks = 1;
  moments_kernel<<<blocks, 256, 0, st>>>(src, mask, n, out3);
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" size_t tio_quantiles_workspace_bytes(void) {
  return sizeof(SelectState) + (size_t)kTargets * 2048 * sizeof(unsigned) + 64;
}

extern "C" int tio_quantiles(const float* src, const uint8_t* mask, int64_t n, const double* q_host, int m,
                             float* values, double* weights, double* count, void* workspace,
                             size_t workspace_bytes, void* stream) {
  TIO_CHECK_ARG(src && q_host && values && weights && count && workspace, "tio_quantiles: null pointer");
  TIO_CHECK_ARG(n > 0 && m >= 1 && m <= kMaxQ, "tio_quantiles: need n > 0 and 1 <= m <= %d", kMaxQ);
  TIO_CHECK_ARG(workspace_bytes >= tio_quantiles_workspace_bytes() && ((uintptr_t)workspace & 15) == 0,
                "tio_quantiles: workspace too small or misaligned");
  for (int t = 0; t < m; ++t)
    TIO_CHECK_ARG(q_host[t] >= 0.0 && q_host[t] <= 1.0, "Only values 0 <= q <= 1 are supported, but got %g", q_host[t]);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* ws = (unsigned char*)workspace;
  SelectState* state = (SelectState*)ws;
  unsigned* hist = (unsigned*)(ws + ((sizeof(SelectState) + 15) / 16) * 16);
  const double q0 = q_host[0], q1 = m > 1 ? q_host[1] : 0.0;
  select_init_kernel<<<1, 1, 0, st>>>(state, m);
  int blocks = (int)((n + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  const size_t hbytes = (size_t)kTargets * 2048 * sizeof(unsigned);
  TIO_CHECK_CUDA(cudaMemsetAsync(hist, 0, hbytes, st));
  select_hist_kernel<0><<<blocks, 256, 0, st>>>(src, mask, n, state, hist);
  select_scan_kernel<0><<<1, 32, 0, st>>>(state, hist, q0, q1, (long long)n, mask != nullptr);
  TIO_CHECK_CUDA(cudaMemsetAsync(hist, 0, hbytes, st));
  select_hist_kernel<1><<<blocks, 256, 0, st>>>(src, mask, n, state, hist);
  select_scan_kernel<1><<<1, 32, 0, st>>>(state, hist, q0, q1, (long long)n, mask != nullptr);
  TIO_CHECK_CUDA(cudaMemsetAsync(hist, 0, hbytes, st));
  select_hist_kernel<2><<<blocks, 256, 0, st>>>(src, mask, n, state, hist);
  select_scan_kernel<2><<<1, 32, 0, st>>>(state, hist, q0, q1, (long long)n, mask != nullptr);
  select_finish_kernel<<<1, 32, 0, st>>>(state, values, weights, count);
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_rescale(const float* src, float* dst, int B, int64_t per_elem, float lo, float hi,
                           const float* sub, const float* div, const float* mul, const float* add,
                           const uint8_t* keep, int flags, void* stream) {
  TIO_CHECK_ARG(src && dst && B > 0 && per_elem > 0, "tio_rescale: bad arguments");
  TIO_CHECK_ARG((flags & ~31) == 0, "tio_rescale: unknown flag bits %d", flags);
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = ((per_elem & 3) == 0) && (((uintptr_t)src | (uintptr_t)dst) & 15) == 0;
  const int64_t work = vec ? per_elem / 4 : per_elem;
  int bx = (int)((work + 255) / 256);
  const int cap = (num_sms() * 16 + B - 1) / B;
  if (bx > cap) bx = cap < 1 ? 1 : cap;
  TIO_CHECK_ARG(B <= 65535, "tio_rescale: batch too large");
  dim3 grid(bx, B);
  if (vec) rescale_kernel<4><<<grid, 256, 0, st>>>(src, dst, per_elem, lo, hi, sub, div, mul, add, keep, flags);
  else rescale_kernel<1><<<grid, 256, 0, st>>>(src, dst, per_elem, lo, hi, sub, div, mul, add, keep, flags);
  TIO_CHECK_LAUNCH();
  return 0;
}

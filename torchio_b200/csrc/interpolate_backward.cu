// interpolate_backward.cu — the adjoints of tio_interpolate and tio_axis_resample (interpolate.cu)
// for fp32 gradients: Resize and Anisotropy under autograd.
//
// tio_interpolate_backward     grad_in = Aᵀ grad_out for the separable map A of tio_interpolate.
//                              Per axis, a CSR table inverts the forward's taps: for each input
//                              index x, the (output index o, weight) pairs whose tap lands on x, in
//                              ascending o (`tables.interpolate_adjoint_tables`).  One thread per
//                              grad_in voxel sums ((w_i*w_j)*w_k)*g over its three windows, I then J
//                              then K, each ascending: a gather, so no atomics and no memset, and
//                              the order of every sum is fixed by the tables.
// tio_axis_resample_backward   Anisotropy's per-instance path: input plane p of element b sums
//                              (1 - w[o])*g_o over the o with lo[o] = p and w[o]*g_o over those with
//                              hi[o] = p (nearest: g_o over lo[o] = p), in ascending o, from
//                              per-element CSR rows; elements with axis -1 copy g.
//
// Every term the forward reads is kept, zero weights included (the L -> L axes of a trilinear
// pass, the tap pair that collapses onto the last plane): a NaN or Inf in grad_out spreads to the
// inputs that ATen's upsample_trilinear3d_backward / the gather backward spreads it to.  Each term
// is rounded as the reference's backward rounds it (t*h*w*g left to right; g*(1 - w) and g*w), so
// a voxel with one term equals the reference bit for bit.
//
// tio_interpolate_backward follows the forward's layout: a warp takes 128 consecutive K inputs of
// one row, lane l taking l, l + 32, l + 64, l + 96, so stores coalesce and the lanes of one load
// read neighbouring outputs; the I and J window bounds are read once per row.  Reads of grad_out go
// through L1 / L2, which the warps of one CTA and CTAs launched together share as they walk the
// input in order.  tio_axis_resample_backward writes 4 consecutive K inputs per thread with
// 16-byte loads and stores when rows are 16-byte aligned.
#include "common.cuh"

namespace tio {

namespace {

constexpr int kThreads = 256;
constexpr int kLanes = 32, kPerLane = 4, kChunk = kLanes * kPerLane;  // K inputs per warp

__global__ void __launch_bounds__(kThreads)
interpolate_backward_kernel(const float* __restrict__ g, float* __restrict__ grad, int I, int J, int K, int OI,
                            int OJ, int OK, const int* __restrict__ ptr, const int* __restrict__ ent,
                            const float* __restrict__ wt, int chunks) {
  const int chunks_per_row = (K + kChunk - 1) / kChunk;
  const int lane = threadIdx.x % kLanes;
  const int* ptr_i = ptr;
  const int* ptr_j = ptr + I + 1;
  const int* ptr_k = ptr + I + J + 2;
  const int warps = gridDim.x * (kThreads / kLanes);
  // 32-bit chunk and row indices (the entry point checks chunks < 2^31): 64-bit divisions are
  // subroutine calls whose saved registers spill
  for (int w = (blockIdx.x * kThreads + threadIdx.x) / kLanes; w < chunks; w += warps) {
    const int row = w / chunks_per_row;
    const int k_base = (w - row * chunks_per_row) * kChunk + lane;
    const int j = row % J;
    const int vi = row / J;
    const int i = vi % I;
    const int v = vi / I;
    const int i_beg = __ldg(ptr_i + i), i_end = __ldg(ptr_i + i + 1);
    const int j_beg = __ldg(ptr_j + j), j_end = __ldg(ptr_j + j + 1);
    const float* gv = g + (int64_t)v * OI * OJ * OK;
    // the K windows of the lane's 4 inputs, walked side by side (entry t of each in one step) so
    // that 4 independent reads of grad_out are in flight; each input's own sum keeps its order
    int kb[kPerLane], kn[kPerLane], kmax = 0;
    float acc[kPerLane];
#pragma unroll
    for (int q = 0; q < kPerLane; ++q) {
      const int k = k_base + q * kLanes;
      kb[q] = k < K ? __ldg(ptr_k + k) : 0;
      kn[q] = k < K ? __ldg(ptr_k + k + 1) - kb[q] : 0;
      kmax = max(kmax, kn[q]);
      acc[q] = 0.0f;
    }
    for (int a = i_beg; a < i_end; ++a) {
      const int oi = __ldg(ent + a);
      const float wi = __ldg(wt + a);
      for (int c = j_beg; c < j_end; ++c) {
        const float wij = __fmul_rn(wi, __ldg(wt + c));
        const float* gr = gv + ((int64_t)oi * OJ + __ldg(ent + c)) * OK;
        for (int t = 0; t < kmax; ++t) {
#pragma unroll
          for (int q = 0; q < kPerLane; ++q) {
            if (t < kn[q]) {
              const int e = kb[q] + t;
              acc[q] = __fadd_rn(acc[q], __fmul_rn(__fmul_rn(wij, __ldg(wt + e)), __ldg(gr + __ldg(ent + e))));
            }
          }
        }
      }
    }
    float* d = grad + (int64_t)row * K;
#pragma unroll
    for (int q = 0; q < kPerLane; ++q) {
      const int k = k_base + q * kLanes;
      if (k < K) d[k] = acc[q];
    }
  }
}

// the coefficient of entry e = 2*o + (hi tap) of a linear row: (1 - w[o]) or w[o], as the forward
__device__ __forceinline__ float axis_coef(const float* __restrict__ wrow, int e) {
  const float wo = __ldg(wrow + (e >> 1));
  return (e & 1) ? wo : __fsub_rn(1.0f, wo);
}

constexpr int V = 4;  // fp32 K inputs per thread

__global__ void __launch_bounds__(kThreads)
axis_resample_backward_kernel(const float* __restrict__ g, float* __restrict__ grad, int C, int I, int J, int K,
                              const int* __restrict__ axis, const int* __restrict__ ptr,
                              const int* __restrict__ ent, const float* __restrict__ w, int L, int linear,
                              int64_t segments, int vectorised) {
  const int seg_per_row = (K + V - 1) / V;
  for (int64_t s = (int64_t)blockIdx.x * kThreads + threadIdx.x; s < segments; s += (int64_t)gridDim.x * kThreads) {
    const int64_t row = s / seg_per_row;
    const int k0 = (int)(s - row * seg_per_row) * V;
    const int j = (int)(row % J);
    const int64_t bci = row / J;
    const int i = (int)(bci % I);
    const int64_t bc = bci / I;
    const int b = (int)(bc / C);
    const int e = __ldg(axis + b);
    const int64_t vol = bc * I * J * K;
    const int* prow = ptr + (int64_t)b * (L + 1);
    const int* erow = ent + (int64_t)b * 2 * L;
    const float* wrow = w + (int64_t)b * L;
    float* d = grad + row * K + k0;
    float acc[V] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (e == 0 || e == 1) {
      // every term reads a whole grad_out row: (o, j) along I, (i, o) along J
      const int p = e == 0 ? i : j;
      const int end = __ldg(prow + p + 1);
      for (int t = __ldg(prow + p); t < end; ++t) {
        const int code = __ldg(erow + t);
        const int o = code >> 1;
        const float* src = g + vol + (e == 0 ? ((int64_t)o * J + j) : ((int64_t)i * J + o)) * K + k0;
        float x[V];
        if (vectorised) {
          const float4 r = __ldg(reinterpret_cast<const float4*>(src));
          x[0] = r.x, x[1] = r.y, x[2] = r.z, x[3] = r.w;
        } else {
#pragma unroll
          for (int q = 0; q < V; ++q) x[q] = __ldg(src + min(q, K - 1 - k0));
        }
        const float cf = linear ? axis_coef(wrow, code) : 1.0f;
#pragma unroll
        for (int q = 0; q < V; ++q) acc[q] = __fadd_rn(acc[q], linear ? __fmul_rn(x[q], cf) : x[q]);
      }
    } else if (e == 2) {
      const float* src = g + vol + ((int64_t)i * J + j) * K;
#pragma unroll
      for (int q = 0; q < V; ++q) {
        if (k0 + q >= K) break;
        const int end = __ldg(prow + k0 + q + 1);
        for (int t = __ldg(prow + k0 + q); t < end; ++t) {
          const int code = __ldg(erow + t);
          const float x = __ldg(src + (code >> 1));
          acc[q] = __fadd_rn(acc[q], linear ? __fmul_rn(x, axis_coef(wrow, code)) : x);
        }
      }
    } else {
      // element copied by the forward: its gradient passes through
      const float* src = g + row * K + k0;
#pragma unroll
      for (int q = 0; q < V; ++q) acc[q] = __ldg(src + min(q, K - 1 - k0));
    }
    if (vectorised) {
      *reinterpret_cast<float4*>(d) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    } else {
#pragma unroll
      for (int q = 0; q < V; ++q)
        if (k0 + q < K) d[q] = acc[q];
    }
  }
}

unsigned grid_for(int64_t threads) {
  int64_t blocks = (threads + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)num_sms() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

}  // namespace

}  // namespace tio

extern "C" int tio_interpolate_backward(const float* grad_out, float* grad_in, int volumes, int I, int J, int K,
                                        int OI, int OJ, int OK, const int32_t* ptr, const int32_t* ent,
                                        const float* wt, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(grad_out && grad_in && ptr && ent && wt, "tio_interpolate_backward: null gradient or table");
  TIO_CHECK_ARG(volumes >= 0 && I > 0 && J > 0 && K > 0 && OI > 0 && OJ > 0 && OK > 0,
                "tio_interpolate_backward: bad shape");
  TIO_CHECK_ARG((const void*)grad_out != (const void*)grad_in, "tio_interpolate_backward: grad_out and grad_in are aliased");
  if (volumes == 0) return 0;
  const int64_t chunks = (int64_t)volumes * I * J * ((K + kChunk - 1) / kChunk);
  TIO_CHECK_ARG(chunks <= INT32_MAX, "tio_interpolate_backward: %lld warp chunks of 128 K inputs exceed 2^31 - 1",
                (long long)chunks);
  interpolate_backward_kernel<<<grid_for(chunks * kLanes), kThreads, 0, (cudaStream_t)stream>>>(
      grad_out, grad_in, I, J, K, OI, OJ, OK, ptr, ent, wt, (int)chunks);
  launched();
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_axis_resample_backward(const float* grad_out, float* grad_in, int B, int C, int I, int J, int K,
                                          const int32_t* axis, const int32_t* ptr, const int32_t* ent,
                                          const float* w, int L, int linear, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(grad_out && grad_in && axis && ptr && ent, "tio_axis_resample_backward: null gradient or table");
  TIO_CHECK_ARG(!linear || w, "tio_axis_resample_backward: null weights");
  TIO_CHECK_ARG(B >= 0 && C >= 0 && I > 0 && J > 0 && K > 0 && L >= I && L >= J && L >= K,
                "tio_axis_resample_backward: bad shape");
  TIO_CHECK_ARG((const void*)grad_out != (const void*)grad_in, "tio_axis_resample_backward: grad_out and grad_in are aliased");
  if (B == 0 || C == 0) return 0;
  const bool vectorised = K % V == 0 && (uintptr_t)grad_out % 16 == 0 && (uintptr_t)grad_in % 16 == 0;
  const int64_t segments = (int64_t)B * C * I * J * ((K + V - 1) / V);
  axis_resample_backward_kernel<<<grid_for(segments), kThreads, 0, (cudaStream_t)stream>>>(
      grad_out, grad_in, C, I, J, K, axis, ptr, ent, w, L, linear ? 1 : 0, segments, vectorised ? 1 : 0);
  launched();
  TIO_CHECK_LAUNCH();
  return 0;
}

// interpolate.cu — Resize and Anisotropy of TorchIO 2.0.0a2 (transforms/spatial/resize.py,
// anisotropy.py) in one pass each.
//
// tio_interpolate     ATen's upsample_trilinear3d (align_corners=True) / upsample_nearest3d on the
//                     data's fp32 image, from per-axis (i0, i1, l0, l1) tables built on the host.
//                     The 8-tap combine is ATen's nested expression as nvcc compiled it for sm_90
//                     (read from the SASS of libtorch_cuda): every `a*x + b*y` is fma(a, x, rn(b*y))
//                     (lerp2), and every tap is read, zero-weight ones included, so NaN / Inf
//                     neighbours propagate as they do there.  Anisotropy's shared path is one call
//                     with the nearest-down map composed into the up table.
// tio_axis_resample   Anisotropy's per-instance path: one axis per batch element, (lo, hi, w) per
//                     output index along it, combined by nearest copy or by the reference's four
//                     separately rounded fp32 ops; inactive elements are copied bit for bit.
//
// tio_axis_resample writes V = 16 / sizeof(T) consecutive K outputs per thread, with 16-byte loads
// and stores when rows are 16-byte aligned and a scalar path otherwise.  tio_interpolate gives each
// warp 128 consecutive K outputs of one row, lane l taking l, l + 32, l + 64, l + 96: the lanes of
// one load instruction read neighbouring source voxels (8 sectors per warp-wide gather on a 2x
// downsize instead of 32 when a thread owns 4 adjacent outputs) and stores are coalesced.  Taps
// are read through the read-only cache; neighbouring rows and planes of a source are reused from
// L1 / L2 by the warps of one CTA and by CTAs launched together, which walk the output in order.
#include "image_dtype.cuh"

namespace tio {

namespace {

constexpr int kThreads = 256;

struct Taps {
  int i0, i1;
  float l0, l1;
};

// axis table: lo[O], hi[O] in `idx`, l0[O], l1[O] in `lam` (nearest: lo only, lam NULL)
__device__ __forceinline__ Taps taps(const int* __restrict__ idx, const float* __restrict__ lam, int O, int o,
                                     bool linear) {
  Taps t;
  t.i0 = __ldg(idx + o);
  if (linear) {
    t.i1 = __ldg(idx + O + o);
    t.l0 = __ldg(lam + o);
    t.l1 = __ldg(lam + O + o);
  } else {
    t.i1 = t.i0;
    t.l0 = 1.0f;
    t.l1 = 0.0f;
  }
  return t;
}

constexpr int kLanes = 32, kPerLane = 4, kChunk = kLanes * kPerLane;  // K outputs per warp

template <typename T, bool kLinear>
__global__ void __launch_bounds__(kThreads)
interpolate_kernel(const T* __restrict__ src, T* __restrict__ dst, int I, int J, int K, int OI, int OJ, int OK,
                   const int* __restrict__ idx, const float* __restrict__ lam, int64_t chunks) {
  const int chunks_per_row = (OK + kChunk - 1) / kChunk;
  const int lane = threadIdx.x % kLanes;
  const int* idx_i = idx;
  const int* idx_j = idx + 2 * OI;
  const int* idx_k = idx + 2 * (OI + OJ);
  const float* lam_i = lam;
  const float* lam_j = kLinear ? lam + 2 * OI : nullptr;
  const float* lam_k = kLinear ? lam + 2 * (OI + OJ) : nullptr;
  const int64_t warps = (int64_t)gridDim.x * (kThreads / kLanes);
  for (int64_t w = ((int64_t)blockIdx.x * kThreads + threadIdx.x) / kLanes; w < chunks; w += warps) {
    const int64_t row = w / chunks_per_row;
    const int k_base = (int)(w - row * chunks_per_row) * kChunk + lane;
    const int oj = (int)(row % OJ);
    const int64_t vi = row / OJ;
    const int oi = (int)(vi % OI);
    const int64_t v = vi / OI;
    const Taps ti = taps(idx_i, lam_i, OI, oi, kLinear);
    const Taps tj = taps(idx_j, lam_j, OJ, oj, kLinear);
    const T* s00 = src + (((int64_t)v * I + ti.i0) * J + tj.i0) * K;
    const T* s01 = src + (((int64_t)v * I + ti.i0) * J + tj.i1) * K;
    const T* s10 = src + (((int64_t)v * I + ti.i1) * J + tj.i0) * K;
    const T* s11 = src + (((int64_t)v * I + ti.i1) * J + tj.i1) * K;
    T* d = dst + row * OK;
#pragma unroll
    for (int q = 0; q < kPerLane; ++q) {
      const int k = k_base + q * kLanes;
      if (k >= OK) break;
      const Taps tk = taps(idx_k, lam_k, OK, k, kLinear);
      float r;
      if constexpr (kLinear) {
        // t0*(h0*(w0*x000 + w1*x001) + h1*(w0*x010 + w1*x011)) + t1*(h0*(...) + h1*(...))
        const float a0 = lerp2(tk.l0, to_float(ld(s00 + tk.i0)), tk.l1, to_float(ld(s00 + tk.i1)));
        const float a1 = lerp2(tk.l0, to_float(ld(s01 + tk.i0)), tk.l1, to_float(ld(s01 + tk.i1)));
        const float b0 = lerp2(tk.l0, to_float(ld(s10 + tk.i0)), tk.l1, to_float(ld(s10 + tk.i1)));
        const float b1 = lerp2(tk.l0, to_float(ld(s11 + tk.i0)), tk.l1, to_float(ld(s11 + tk.i1)));
        r = lerp2(ti.l0, lerp2(tj.l0, a0, tj.l1, a1), ti.l1, lerp2(tj.l0, b0, tj.l1, b1));
      } else {
        r = to_float(ld(s00 + tk.i0));
      }
      d[k] = from_float<T>(r);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
axis_resample_kernel(const T* __restrict__ src, T* __restrict__ dst, int C, int I, int J, int K,
                     const int* __restrict__ axis, const int* __restrict__ lo, const int* __restrict__ hi,
                     const float* __restrict__ w, int L, int linear, int64_t segments, int vectorised) {
  constexpr int V = 16 / sizeof(T);
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
    T* d = dst + row * K + k0;
    Pack<T> a, c;  // the lo and hi taps of the V outputs
    float wq[V];
    if (e == 0 || e == 1) {
      // the whole row comes from one (lo) and one (hi) source row
      const int o = e == 0 ? i : j;
      const int r_lo = __ldg(lo + (int64_t)b * L + o);
      const int r_hi = linear ? __ldg(hi + (int64_t)b * L + o) : r_lo;
      const float wr = linear ? __ldg(w + (int64_t)b * L + o) : 0.0f;
      const T* p_lo = src + vol + (e == 0 ? ((int64_t)r_lo * J + j) : ((int64_t)i * J + r_lo)) * K + k0;
      const T* p_hi = src + vol + (e == 0 ? ((int64_t)r_hi * J + j) : ((int64_t)i * J + r_hi)) * K + k0;
      if (vectorised) {
        a.raw = __ldg(reinterpret_cast<const uint4*>(p_lo));
        c.raw = linear ? __ldg(reinterpret_cast<const uint4*>(p_hi)) : a.raw;
      } else {
#pragma unroll
        for (int q = 0; q < V; ++q) {
          const int kk = min(q, K - 1 - k0);
          a.e[q] = ld(p_lo + kk);
          c.e[q] = ld(p_hi + kk);
        }
      }
#pragma unroll
      for (int q = 0; q < V; ++q) wq[q] = wr;
    } else if (e == 2) {
      const T* p = src + vol + ((int64_t)i * J + j) * K;
#pragma unroll
      for (int q = 0; q < V; ++q) {
        const int k = min(k0 + q, K - 1);
        const int64_t t = (int64_t)b * L + k;
        a.e[q] = ld(p + __ldg(lo + t));
        c.e[q] = linear ? ld(p + __ldg(hi + t)) : a.e[q];
        wq[q] = linear ? __ldg(w + t) : 0.0f;
      }
    } else {
      // inactive element: the reference's clone, bit for bit
      const T* p = src + row * K + k0;
      if (vectorised) {
        *reinterpret_cast<uint4*>(d) = __ldg(reinterpret_cast<const uint4*>(p));
      } else {
        for (int q = 0; q < V && k0 + q < K; ++q) d[q] = p[q];
      }
      continue;
    }
    Pack<T> out;
#pragma unroll
    for (int q = 0; q < V; ++q) {
      float r = to_float(a.e[q]);
      if (linear) {
        // lower * (1 - w) + upper * w, four separately rounded fp32 ops
        r = __fadd_rn(__fmul_rn(r, __fsub_rn(1.0f, wq[q])), __fmul_rn(to_float(c.e[q]), wq[q]));
      }
      out.e[q] = from_float<T>(r);
    }
    if (vectorised) {
      *reinterpret_cast<uint4*>(d) = out.raw;
    } else {
#pragma unroll
      for (int q = 0; q < V; ++q)
        if (k0 + q < K) d[q] = out.e[q];
    }
  }
}

unsigned grid_for(int64_t segments) {
  int64_t blocks = (segments + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)num_sms() * 16;
  return (unsigned)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

template <typename T>
void launch_interpolate(const void* src, void* dst, int volumes, int I, int J, int K, int OI, int OJ, int OK,
                        const int* idx, const float* lam, int linear, cudaStream_t st) {
  const int64_t chunks = (int64_t)volumes * OI * OJ * ((OK + kChunk - 1) / kChunk);
  const unsigned grid = grid_for(chunks * kLanes);
  if (linear)
    interpolate_kernel<T, true><<<grid, kThreads, 0, st>>>((const T*)src, (T*)dst, I, J, K, OI, OJ, OK, idx, lam,
                                                           chunks);
  else
    interpolate_kernel<T, false><<<grid, kThreads, 0, st>>>((const T*)src, (T*)dst, I, J, K, OI, OJ, OK, idx, lam,
                                                            chunks);
  launched();
}

template <typename T>
void launch_axis_resample(const void* src, void* dst, int B, int C, int I, int J, int K, const int* axis,
                          const int* lo, const int* hi, const float* w, int L, int linear, cudaStream_t st) {
  constexpr int V = 16 / sizeof(T);
  const bool vectorised = K % V == 0 && (uintptr_t)src % 16 == 0 && (uintptr_t)dst % 16 == 0;
  const int64_t segments = (int64_t)B * C * I * J * ((K + V - 1) / V);
  axis_resample_kernel<T><<<grid_for(segments), kThreads, 0, st>>>(
      (const T*)src, (T*)dst, C, I, J, K, axis, lo, hi, w, L, linear, segments, vectorised ? 1 : 0);
  launched();
}

}  // namespace

}  // namespace tio

extern "C" int tio_interpolate(const void* src, void* dst, int dtype, int volumes, int I, int J, int K, int OI,
                               int OJ, int OK, const int32_t* idx, const float* lam, int linear, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst && idx, "tio_interpolate: null source, output or table");
  TIO_CHECK_ARG(!linear || lam, "tio_interpolate: null weights");
  TIO_CHECK_ARG(volumes >= 0 && I > 0 && J > 0 && K > 0 && OI > 0 && OJ > 0 && OK > 0,
                "tio_interpolate: bad shape");
  if (volumes == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_INTERP(T) launch_interpolate<T>(src, dst, volumes, I, J, K, OI, OJ, OK, idx, lam, linear, st)
  TIO_IMAGE_DISPATCH(dtype, "tio_interpolate", TIO_INTERP)
#undef TIO_INTERP
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_axis_resample(const void* src, void* dst, int dtype, int B, int C, int I, int J, int K,
                                 const int32_t* axis, const int32_t* lo, const int32_t* hi, const float* w,
                                 int L, int linear, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst && axis && lo, "tio_axis_resample: null source, output or table");
  TIO_CHECK_ARG(!linear || (hi && w), "tio_axis_resample: null linear table");
  TIO_CHECK_ARG(B >= 0 && C >= 0 && I > 0 && J > 0 && K > 0 && L >= I && L >= J && L >= K,
                "tio_axis_resample: bad shape");
  if (B == 0 || C == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_AXIS(T) launch_axis_resample<T>(src, dst, B, C, I, J, K, axis, lo, hi, w, L, linear, st)
  TIO_IMAGE_DISPATCH(dtype, "tio_axis_resample", TIO_AXIS)
#undef TIO_AXIS
  TIO_CHECK_LAUNCH();
  return 0;
}

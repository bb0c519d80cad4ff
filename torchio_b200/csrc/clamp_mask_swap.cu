// clamp_mask_swap.cu — Clamp, Mask and Swap of TorchIO 2.0.0a2 (transforms/intensity/) on the GPU.
//
// tio_clamp          torch.clamp(min, max) for every image dtype, 16-byte accesses where aligned.
// tio_mask           torch.where(mask.expand_as(x), x, outside): the mask of batch element 0 is read
//                    once per voxel for all B elements; in place it writes only the outside voxels.
// tio_swap_patches   Swap's ordered patch exchanges in place, one launch for the whole batch: each
//                    element's list runs on its own thread-block cluster, cluster.sync() between steps.
#include <cooperative_groups.h>

#include <cmath>
#include <cstring>

#include "common.cuh"
#include "image_dtype.cuh"
#include "label_lookup.cuh"

namespace cg = cooperative_groups;

namespace tio {

namespace {

constexpr int kThreads = 256;

template <typename T, int N>
struct alignas(sizeof(T) * N) Vec {
  T e[N];
};

// ---- clamp --------------------------------------------------------------------------------------
//
// ATen's clamp_scalar / clamp_min_scalar / clamp_max_scalar CUDA kernels: the bounds are converted
// to the result dtype (done by the caller), a NaN element is returned as is, and otherwise
// min(max(v, lo), hi) with ::max / ::min (fmaxf / fminf for floating types; fp16 and bf16 compare
// as the floats they widen to).

template <typename D> struct Compute { typedef D type; };
template <> struct Compute<f16> { typedef float type; };
template <> struct Compute<bf16> { typedef float type; };

template <typename T> __device__ __forceinline__ T dmax(T a, T b) { return a > b ? a : b; }
template <typename T> __device__ __forceinline__ T dmin(T a, T b) { return a < b ? a : b; }
template <> __device__ __forceinline__ float dmax(float a, float b) { return fmaxf(a, b); }
template <> __device__ __forceinline__ float dmin(float a, float b) { return fminf(a, b); }
template <> __device__ __forceinline__ double dmax(double a, double b) { return fmax(a, b); }
template <> __device__ __forceinline__ double dmin(double a, double b) { return fmin(a, b); }

template <typename T> __device__ __forceinline__ bool is_nan(T) { return false; }
template <> __device__ __forceinline__ bool is_nan(float v) { return v != v; }
template <> __device__ __forceinline__ bool is_nan(double v) { return v != v; }

template <typename D> __device__ __forceinline__ typename Compute<D>::type widen(D v) { return v; }
template <> __device__ __forceinline__ float widen(f16 v) { return to_float(v); }
template <> __device__ __forceinline__ float widen(bf16 v) { return to_float(v); }
template <typename D> __device__ __forceinline__ D narrow(typename Compute<D>::type v) { return v; }
template <> __device__ __forceinline__ f16 narrow(float v) { return from_float<f16>(v); }
template <> __device__ __forceinline__ bf16 narrow(float v) { return from_float<bf16>(v); }

// the source element as the result dtype: itself, or an integer promoted to fp32 (round to nearest)
template <typename S, typename D> __device__ __forceinline__ D promote(S v) { return (D)v; }
template <> __device__ __forceinline__ f16 promote(f16 v) { return v; }
template <> __device__ __forceinline__ bf16 promote(bf16 v) { return v; }

// bounds: bit 0 = lo present, bit 1 = hi present, 4 = every output NaN (clamp_out's NaN bound)
template <typename D>
__device__ __forceinline__ D clamp_value(D x, typename Compute<D>::type lo, typename Compute<D>::type hi,
                                         int bounds) {
  typedef typename Compute<D>::type C;
  C v = widen(x);
  if (is_nan(v)) return x;
  if (bounds & 1) v = dmax(v, lo);
  if (bounds & 2) v = dmin(v, hi);
  return narrow<D>(v);
}

template <typename S, typename D>
__global__ void __launch_bounds__(kThreads)
clamp_kernel(const S* src, D* dst, int64_t count, typename Compute<D>::type lo, typename Compute<D>::type hi,
             int bounds, D nan_value, int vectorised) {
  constexpr int kVec = 16 / (sizeof(S) > sizeof(D) ? sizeof(S) : sizeof(D));
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int64_t first = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  auto one = [&](S s) -> D { return bounds & 4 ? nan_value : clamp_value<D>(promote<S, D>(s), lo, hi, bounds); };
  const int64_t n_vec = vectorised ? count / kVec : 0;
  for (int64_t i = first; i < n_vec; i += stride) {
    const Vec<S, kVec> in = reinterpret_cast<const Vec<S, kVec>*>(src)[i];
    Vec<D, kVec> out;
#pragma unroll
    for (int j = 0; j < kVec; ++j) out.e[j] = one(in.e[j]);
    reinterpret_cast<Vec<D, kVec>*>(dst)[i] = out;
  }
  for (int64_t i = n_vec * kVec + first; i < count; i += stride) dst[i] = one(src[i]);
}

int64_t grid_for(int64_t work) {
  int64_t blocks = (work + kThreads - 1) / kThreads;
  if (blocks > (int64_t)num_sms() * 8) blocks = (int64_t)num_sms() * 8;
  return blocks < 1 ? 1 : blocks;
}

template <typename T> T host_value(const void* p) {
  T v;
  memcpy(&v, p, sizeof(T));
  return v;
}
template <typename D> typename Compute<D>::type host_bound(const void* p) { return host_value<D>(p); }
template <> float host_bound<f16>(const void* p) {
  return __half2float(__ushort_as_half(host_value<unsigned short>(p)));
}
template <> float host_bound<bf16>(const void* p) {
  return __bfloat162float(__ushort_as_bfloat16(host_value<unsigned short>(p)));
}
template <typename C> bool host_nan(C v) { return v != v; }

template <typename S, typename D>
void launch_clamp(const void* src, void* dst, int64_t count, const void* lo, const void* hi, cudaStream_t st) {
  typedef typename Compute<D>::type C;
  constexpr int kVec = 16 / (sizeof(S) > sizeof(D) ? sizeof(S) : sizeof(D));
  const C lo_v = lo ? host_bound<D>(lo) : C(0), hi_v = hi ? host_bound<D>(hi) : C(0);
  int bounds = (lo ? 1 : 0) | (hi ? 2 : 0);
  D nan_value{};
  if (lo && hi && (host_nan(lo_v) || host_nan(hi_v))) {
    bounds = 4;
    nan_value = host_nan(lo_v) ? host_value<D>(lo) : host_value<D>(hi);
  }
  const bool vectorised = (uintptr_t)src % (kVec * sizeof(S)) == 0 && (uintptr_t)dst % (kVec * sizeof(D)) == 0;
  clamp_kernel<S, D><<<(unsigned)grid_for(count / kVec + 1), kThreads, 0, st>>>(
      (const S*)src, (D*)dst, count, lo_v, hi_v, bounds, nan_value, vectorised ? 1 : 0);
  launched();
}

// ---- mask ---------------------------------------------------------------------------------------

template <typename M> struct MaskKey { typedef long long type; };
template <> struct MaskKey<float> { typedef float type; };

// one thread per (mask channel, voxel): the mask value is read once and applied to every element
// (and to every image channel when the mask has one channel).  promote = 0: dst is the image
// itself, only outside voxels are written; promote = 1: dst (fp32) = inside ? float(src) : outside.
template <typename M, typename S, typename D>
__global__ void __launch_bounds__(kThreads)
mask_kernel(const M* __restrict__ mask, int mask_channels, const typename MaskKey<M>::type* __restrict__ keys,
            int n_keys, const S* src, D* dst, int B, int C, int64_t vox, D outside) {
  typedef typename MaskKey<M>::type K;
  const int64_t total = (int64_t)mask_channels * vox;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x; e < total; e += stride) {
    const M m = __ldg(mask + e);
    bool inside;
    if (n_keys < 0) {
      inside = m != (M)0;
    } else {
      K key;
      inside = label_key<M, K>(m, key) && sorted_slot(key, keys, n_keys) >= 0;
    }
    if constexpr (std::is_same<S, D>::value) {
      if (inside) continue;
    }
    const int64_t v = e % vox;
    const int c0 = mask_channels == 1 ? 0 : (int)(e / vox), c1 = mask_channels == 1 ? C : c0 + 1;
    for (int b = 0; b < B; ++b) {
      for (int c = c0; c < c1; ++c) {
        const int64_t i = ((int64_t)b * C + c) * vox + v;
        if constexpr (std::is_same<S, D>::value) dst[i] = outside;
        else dst[i] = inside ? (D)src[i] : outside;
      }
    }
  }
}

template <typename M, typename S, typename D>
void launch_mask(const void* mask, int mask_channels, const void* keys, int n_keys, const void* src, void* dst,
                 int B, int C, int64_t vox, const void* outside, cudaStream_t st) {
  mask_kernel<M, S, D><<<(unsigned)grid_for((int64_t)mask_channels * vox), kThreads, 0, st>>>(
      (const M*)mask, mask_channels, (const typename MaskKey<M>::type*)keys, n_keys, (const S*)src, (D*)dst, B,
      C, vox, host_value<D>(outside));
  launched();
}

// in place, the image is never read: the outside value is stored as raw bytes of its width
template <typename M>
int dispatch_mask_in_place(int elem_size, const void* mask, int mask_channels, const void* keys, int n_keys,
                           void* dst, int B, int C, int64_t vox, const void* outside, cudaStream_t st) {
#define TIO_MASK_BYTES(T) launch_mask<M, T, T>(mask, mask_channels, keys, n_keys, dst, dst, B, C, vox, outside, st)
  switch (elem_size) {
    case 1: TIO_MASK_BYTES(uint8_t); break;
    case 2: TIO_MASK_BYTES(uint16_t); break;
    case 4: TIO_MASK_BYTES(uint32_t); break;
    case 8: TIO_MASK_BYTES(unsigned long long); break;
    default: TIO_CHECK_ARG(false, "tio_mask: element size %d", elem_size);
  }
#undef TIO_MASK_BYTES
  return 0;
}

template <typename M>
int dispatch_mask(const void* mask, int mask_channels, const void* keys, int n_keys, const void* src, int dtype,
                  void* dst, int dst_dtype, int B, int C, int64_t vox, const void* outside, cudaStream_t st) {
  if (dtype == dst_dtype) {
    static const int kBytes[] = {4, 1, 1, 2, 4, 8, 2, 2, 8};
    return dispatch_mask_in_place<M>(kBytes[dtype], mask, mask_channels, keys, n_keys, dst, B, C, vox, outside,
                                     st);
  }
#define TIO_MASK_PROMOTE(S) launch_mask<M, S, float>(mask, mask_channels, keys, n_keys, src, dst, B, C, vox, outside, st)
  switch (dtype) {
    case TIO_U8: TIO_MASK_PROMOTE(uint8_t); break;
    case TIO_I8: TIO_MASK_PROMOTE(int8_t); break;
    case TIO_I16: TIO_MASK_PROMOTE(int16_t); break;
    case TIO_I32: TIO_MASK_PROMOTE(int32_t); break;
    case TIO_I64: TIO_MASK_PROMOTE(int64_t); break;
    default: TIO_CHECK_ARG(false, "tio_mask: dtype %d is not promoted to fp32", dtype);
  }
#undef TIO_MASK_PROMOTE
  return 0;
}

// ---- swap ---------------------------------------------------------------------------------------

constexpr int kSwapThreads = 256;
constexpr int kMaxCluster = 8;  // the portable cluster size
constexpr int kSwapInts = 8;    // ai, aj, ak, bi, bj, bk, kind, 0

enum SwapKind { kExchange = 0, kStaged = 1, kNoOp = 2 };
constexpr int kUnroll = 8;  // voxels a thread has in flight per pass

// dst patch voxel offset(o) = src[o] for the thread's offsets o, loads batched ahead of the stores
template <typename T, typename Offset>
__device__ __forceinline__ void copy_out(T* dst, const T* src, int64_t first, int64_t stride, int64_t n,
                                         const Offset& offset) {
  for (int64_t o0 = first; o0 < n; o0 += kUnroll * stride) {
    T v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
      if (o0 + u * stride < n) v[u] = src[o0 + u * stride];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u)
      if (o0 + u * stride < n) dst[offset(o0 + u * stride)] = v[u];
  }
}

// Element `blockIdx.x / cluster size` runs the steps of its list in order.  Each offset o of the
// C * pi * pj * pk patch voxels belongs to one thread of the cluster for every step, so a
// non-overlapping pair is a per-voxel exchange; an overlapping pair stages both patches in the
// element's slice of `stage` (written and read by the same thread), then writes A, then B.
// cluster.sync() (barrier.cluster arrive.release / wait.acquire) orders the steps.
template <typename T>
__global__ void __launch_bounds__(kSwapThreads)
swap_patches_kernel(T* data, int C, int I, int J, int K, int pi, int pj, int pk, const int* __restrict__ list,
                    int steps, int shared, T* stage) {
  cg::cluster_group cluster = cg::this_cluster();
  const int cs = (int)cluster.num_blocks();
  const int element = blockIdx.x / cs;
  const int64_t vol = (int64_t)I * J * K;
  T* base = data + (int64_t)element * C * vol;
  const int* own = list + (shared ? 0 : (int64_t)element * steps * kSwapInts);
  const int plane = pj * pk, patch = pi * plane;
  const int64_t n = (int64_t)C * patch;
  T* st = stage ? stage + (int64_t)element * 2 * n : nullptr;
  const int64_t first = (int64_t)cluster.block_rank() * kSwapThreads + threadIdx.x;
  const int64_t stride = (int64_t)cs * kSwapThreads;
  auto offset = [&](int64_t o) -> int64_t {
    const int c = (int)(o / patch), r = (int)(o - (int64_t)c * patch);
    const int x = r / plane, yz = r - x * plane, y = yz / pk, z = yz - y * pk;
    return c * vol + ((int64_t)x * J + y) * K + z;
  };
  for (int t = 0; t < steps; ++t) {
    const int4 s0 = __ldg(reinterpret_cast<const int4*>(own + (int64_t)t * kSwapInts));
    const int4 s1 = __ldg(reinterpret_cast<const int4*>(own + (int64_t)t * kSwapInts) + 1);
    const int kind = s1.z;
    if (kind == kNoOp) continue;  // uniform across the cluster: no barrier needed
    T* a = base + ((int64_t)s0.x * J + s0.y) * K + s0.z;
    T* b = base + ((int64_t)s0.w * J + s1.x) * K + s1.y;
    // each pass loads kUnroll voxels of a thread before storing any: the loads overlap in flight
    // instead of each store waiting for its own load
    if (kind == kExchange) {
      for (int64_t o0 = first; o0 < n; o0 += kUnroll * stride) {
        int64_t off[kUnroll];
        T va[kUnroll], vb[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const int64_t o = o0 + u * stride;
          off[u] = o < n ? offset(o) : -1;
          if (off[u] >= 0) {
            va[u] = a[off[u]];
            vb[u] = b[off[u]];
          }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          if (off[u] >= 0) {
            a[off[u]] = vb[u];
            b[off[u]] = va[u];
          }
        }
      }
    } else {
      for (int64_t o0 = first; o0 < n; o0 += kUnroll * stride) {
        T va[kUnroll], vb[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const int64_t o = o0 + u * stride;
          if (o < n) {
            const int64_t off = offset(o);
            va[u] = a[off];
            vb[u] = b[off];
          }
        }
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
          const int64_t o = o0 + u * stride;
          if (o < n) {
            st[o] = va[u];
            st[n + o] = vb[u];
          }
        }
      }
      cluster.sync();  // every voxel of both patches is read before any is written
      copy_out(a, st + n, first, stride, n, offset);
      cluster.sync();  // then B, so that B wins where the two overlap
      copy_out(b, st, first, stride, n, offset);
    }
    cluster.sync();
  }
}

template <typename T>
int launch_swap(void* data, int B, int C, int I, int J, int K, int pi, int pj, int pk, const int* list, int steps,
                int shared, void* stage, cudaStream_t st) {
  const int64_t n = (int64_t)C * pi * pj * pk;
  int cs = (int)((n + 4 * kSwapThreads - 1) / (4 * kSwapThreads));  // about four voxels per thread
  cs = cs < 1 ? 1 : (cs > kMaxCluster ? kMaxCluster : cs);
  cudaLaunchConfig_t config = {};
  config.gridDim = dim3((unsigned)(B * cs));
  config.blockDim = dim3(kSwapThreads);
  config.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  config.attrs = attr;
  config.numAttrs = 1;
  TIO_CHECK_CUDA(cudaLaunchKernelEx(&config, swap_patches_kernel<T>, (T*)data, C, I, J, K, pi, pj, pk, list, steps,
                                    shared, (T*)stage));
  launched();
  return 0;
}

}  // namespace

}  // namespace tio

extern "C" int tio_clamp(const void* src, void* dst, int dtype, int dst_dtype, int64_t count, const void* lo,
                         const void* hi, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst, "tio_clamp: null source or output");
  TIO_CHECK_ARG(lo || hi, "tio_clamp: no bound");
  TIO_CHECK_ARG(count >= 0, "tio_clamp: bad count");
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_clamp: unknown dtype %d", dtype);
  TIO_CHECK_ARG(dst_dtype == dtype || (dst_dtype == TIO_F32 && dtype >= TIO_U8 && dtype <= TIO_I64),
                "tio_clamp: dtype %d cannot give dtype %d", dtype, dst_dtype);
  TIO_CHECK_ARG(dst_dtype == dtype || src != dst, "tio_clamp: a promoting clamp cannot run in place");
  if (count == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (dst_dtype != dtype) {
#define TIO_CLAMP_PROMOTE(S) launch_clamp<S, float>(src, dst, count, lo, hi, st)
    TIO_LABEL_DISPATCH(dtype, "tio_clamp", TIO_CLAMP_PROMOTE)
#undef TIO_CLAMP_PROMOTE
  } else {
#define TIO_CLAMP(T) launch_clamp<T, T>(src, dst, count, lo, hi, st)
    TIO_IMAGE_DISPATCH(dtype, "tio_clamp", TIO_CLAMP)
#undef TIO_CLAMP
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_mask(const void* mask, int mask_dtype, int mask_channels, const void* keys, int n_keys,
                        const void* src, int dtype, void* dst, int dst_dtype, int B, int C, int64_t vox,
                        const void* outside, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(mask && dst && outside, "tio_mask: null mask, output or outside value");
  TIO_CHECK_ARG(n_keys <= 0 || keys, "tio_mask: null label table");
  TIO_CHECK_ARG(B >= 0 && C > 0 && vox >= 0 && (mask_channels == 1 || mask_channels == C),
                "tio_mask: bad shape (B %d, C %d, mask channels %d)", B, C, mask_channels);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_mask: unknown dtype %d", dtype);
  if (dst_dtype == dtype) {
    TIO_CHECK_ARG(src == dst || src == nullptr, "tio_mask: without promotion the mask is applied in place");
  } else {
    TIO_CHECK_ARG(dst_dtype == TIO_F32 && dtype >= TIO_U8 && dtype <= TIO_I64,
                  "tio_mask: dtype %d cannot give dtype %d", dtype, dst_dtype);
    TIO_CHECK_ARG(src && src != dst, "tio_mask: a promoting mask reads a separate source");
  }
  if (B == 0 || vox == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = 0;
#define TIO_MASK(M) rc = dispatch_mask<M>(mask, mask_channels, keys, n_keys, src, dtype, dst, dst_dtype, B, C, vox, outside, st)
  TIO_LABEL_DISPATCH(mask_dtype, "tio_mask", TIO_MASK)
#undef TIO_MASK
  if (rc) return rc;
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_swap_patches(void* data, int elem_size, int B, int C, int I, int J, int K, int pi, int pj, int pk,
                                const int32_t* swaps, int lists, int steps, int32_t* swaps_device, void* stage,
                                void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(data && swaps && swaps_device, "tio_swap_patches: null volume or swap list");
  TIO_CHECK_ARG(elem_size == 1 || elem_size == 2 || elem_size == 4 || elem_size == 8,
                "tio_swap_patches: element size %d", elem_size);
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "tio_swap_patches: bad shape");
  TIO_CHECK_ARG(pi > 0 && pj > 0 && pk > 0 && pi <= I && pj <= J && pk <= K,
                "tio_swap_patches: patch (%d, %d, %d) does not fit in (%d, %d, %d)", pi, pj, pk, I, J, K);
  TIO_CHECK_ARG(lists == 1 || lists == B, "tio_swap_patches: %d lists for %d elements", lists, B);
  TIO_CHECK_ARG(steps >= 0, "tio_swap_patches: bad step count");
  TIO_CHECK_ARG((int64_t)B * kMaxCluster <= INT32_MAX, "tio_swap_patches: batch too large");
  const int dims[3] = {I, J, K}, patch[3] = {pi, pj, pk};
  bool staged = false;
  for (int64_t e = 0; e < (int64_t)lists * steps; ++e) {
    const int32_t* s = swaps + e * kSwapInts;
    for (int axis = 0; axis < 3; ++axis) {
      for (int side = 0; side < 2; ++side) {
        const int origin = s[3 * side + axis];
        TIO_CHECK_ARG(origin >= 0 && origin <= dims[axis] - patch[axis],
                      "tio_swap_patches: list %lld step %lld: patch at %d on axis %d does not fit in %d",
                      (long long)(e / (steps ? steps : 1)), (long long)(e % (steps ? steps : 1)), origin, axis,
                      dims[axis]);
      }
    }
    const int kind = s[6];
    TIO_CHECK_ARG(kind == kExchange || kind == kStaged || kind == kNoOp, "tio_swap_patches: step kind %d", kind);
    if (kind == kExchange) {
      bool overlap = true;
      for (int axis = 0; axis < 3; ++axis)
        if (s[axis] + patch[axis] <= s[3 + axis] || s[3 + axis] + patch[axis] <= s[axis]) overlap = false;
      TIO_CHECK_ARG(!overlap, "tio_swap_patches: overlapping pair marked as an exchange");
    }
    staged |= kind == kStaged;
  }
  TIO_CHECK_ARG(!staged || stage, "tio_swap_patches: an overlapping pair needs the staging buffer");
  if (steps == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemcpyAsync(swaps_device, swaps, (size_t)lists * steps * kSwapInts * sizeof(int32_t),
                                 cudaMemcpyHostToDevice, st));
  int rc = 0;
  switch (elem_size) {
    case 1: rc = launch_swap<uint8_t>(data, B, C, I, J, K, pi, pj, pk, swaps_device, steps, lists == 1, stage, st); break;
    case 2: rc = launch_swap<uint16_t>(data, B, C, I, J, K, pi, pj, pk, swaps_device, steps, lists == 1, stage, st); break;
    case 4: rc = launch_swap<uint32_t>(data, B, C, I, J, K, pi, pj, pk, swaps_device, steps, lists == 1, stage, st); break;
    default: rc = launch_swap<unsigned long long>(data, B, C, I, J, K, pi, pj, pk, swaps_device, steps, lists == 1, stage, st);
  }
  if (rc) return rc;
  TIO_CHECK_LAUNCH();
  return 0;
}

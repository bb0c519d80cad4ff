// aggregate.cu — PatchAggregator: stitch a batch of patches back into its output volume.
//
// The reference adds one patch at a time on the host (data/aggregator.py:75-245): a slice
// assignment (crop) or `out[box] += patch`, `counts[box] += 1` (average) or
// `out[box] += patch * window`, `counts[box] += window` (hann), patch after patch, in the patch's
// dtype.  Here one launch adds a whole batch.  It is output-stationary: a CTA owns a tile of the
// bounding box of the batch's destination boxes, keeps (in add order) the boxes that meet its tile,
// and each thread folds every covering patch of its voxels in that order, so each voxel's buffer
// and count are read once and written once, no atomics are needed and the result does not depend
// on scheduling.  The arithmetic is ATen's CPU arithmetic: explicit-rounding intrinsics, fp16 /
// bf16 widened to fp32 and rounded back where ATen rounds, integer adds that wrap.
#include <type_traits>

#include "image_dtype.cuh"

namespace tio {
namespace {

constexpr int kCrop = 0, kAverage = 1, kHann = 2;
constexpr int kTileI = 4, kTileJ = 8, kTileK = 32;  // 256 threads: K across the warp, J across warps
constexpr int kThreads = kTileJ * kTileK;
constexpr int kList = 256;    // boxes a tile keeps per pass; a tile that meets more runs more passes
constexpr int kBoxInts = 10;  // host table row: dst lo[3], dst hi[3], src lo[3], patch row

struct Box {
  int lo[3], hi[3], off[3], p;  // destination [lo, hi); source index = destination + off
};

// ---- ATen's arithmetic in the buffer's dtype ----------------------------------------------------

__device__ __forceinline__ f16 round_f16(float v) { return f16{__half_as_ushort(__float2half_rn(v))}; }
__device__ __forceinline__ bf16 round_bf16(float v) { return bf16{__bfloat16_as_ushort(__float2bfloat16_rn(v))}; }

// `out += patch` and `counts += 1`
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ f16 add(f16 a, f16 b) { return round_f16(__fadd_rn(to_float(a), to_float(b))); }
__device__ __forceinline__ bf16 add(bf16 a, bf16 b) { return round_bf16(__fadd_rn(to_float(a), to_float(b))); }
template <typename T, typename = std::enable_if_t<std::is_integral<T>::value>>
__device__ __forceinline__ T add(T a, T b) {
  using U = std::make_unsigned_t<T>;
  return (T)(U)((U)a + (U)b);  // wraps, as ATen's integer add
}

template <typename T>
__device__ __forceinline__ T one() {
  if constexpr (std::is_same<T, f16>::value) return f16{0x3C00};
  else if constexpr (std::is_same<T, bf16>::value) return bf16{0x3F80};
  else return (T)1;
}

// `out += patch * window`: the product is an fp32 tensor (fp64 for an fp64 patch), the add is
// computed in that type and rounded once to the buffer's dtype
__device__ __forceinline__ float hann_add(float a, float p, float w) { return __fadd_rn(a, __fmul_rn(p, w)); }
__device__ __forceinline__ double hann_add(double a, double p, float w) { return __dadd_rn(a, __dmul_rn(p, (double)w)); }
__device__ __forceinline__ f16 hann_add(f16 a, f16 p, float w) {
  return round_f16(__fadd_rn(to_float(a), __fmul_rn(to_float(p), w)));
}
__device__ __forceinline__ bf16 hann_add(bf16 a, bf16 p, float w) {
  return round_bf16(__fadd_rn(to_float(a), __fmul_rn(to_float(p), w)));
}

// `counts += window`
__device__ __forceinline__ float hann_count(float c, float w) { return __fadd_rn(c, w); }
__device__ __forceinline__ double hann_count(double c, float w) { return __dadd_rn(c, (double)w); }
__device__ __forceinline__ f16 hann_count(f16 c, float w) { return round_f16(__fadd_rn(to_float(c), w)); }
__device__ __forceinline__ bf16 hann_count(bf16 c, float w) { return round_bf16(__fadd_rn(to_float(c), w)); }

__device__ __forceinline__ bool covers(const Box& b, int i, int j, int k) {
  return i >= b.lo[0] && i < b.hi[0] && j >= b.lo[1] && j < b.hi[1] && k >= b.lo[2] && k < b.hi[2];
}

// every voxel of the thread in the tile, over the kept boxes list[0, kept) in add order
template <typename T, int MODE>
__device__ __forceinline__ void fold(const Box* list, int kept, const T* __restrict__ patches, T* __restrict__ out,
                                     T* __restrict__ counts, int C, int J, int K, long long vol, int pi, int pj,
                                     int pk, const float* __restrict__ window, int i0, int i1, int j, int k) {
  for (int i = i0; i < i1; ++i) {
    int first = -1, last = -1;
    for (int e = 0; e < kept; ++e)
      if (covers(list[e], i, j, k)) {
        if (first < 0) first = e;
        last = e;
      }
    if (first < 0) continue;  // no patch of the batch covers this voxel: left untouched
    const long long v = ((long long)i * J + j) * K + k;
    const long long patch_vol = (long long)pi * pj * pk;
    if constexpr (MODE == kCrop) {  // the last covering patch wins
      const Box& b = list[last];
      const long long s = ((long long)(i + b.off[0]) * pj + (j + b.off[1])) * pk + (k + b.off[2]);
      const T* src = patches + (long long)b.p * C * patch_vol + s;
      for (int c = 0; c < C; ++c) out[c * vol + v] = ld(src + c * patch_vol);
    } else {
      T n = counts[v];
      for (int e = first; e <= last; ++e) {
        const Box& b = list[e];
        if (!covers(b, i, j, k)) continue;
        if constexpr (MODE == kAverage) {
          n = add(n, one<T>());
        } else {
          const float w = __fmul_rn(__fmul_rn(__ldg(window + i + b.off[0]), __ldg(window + pi + j + b.off[1])),
                                    __ldg(window + pi + pj + k + b.off[2]));
          n = hann_count(n, w);
        }
      }
      counts[v] = n;
      for (int c = 0; c < C; ++c) {
        T a = out[c * vol + v];
        for (int e = first; e <= last; ++e) {
          const Box& b = list[e];
          if (!covers(b, i, j, k)) continue;
          const int si = i + b.off[0], sj = j + b.off[1], sk = k + b.off[2];
          const T p = ld(patches + ((long long)b.p * C + c) * patch_vol + ((long long)si * pj + sj) * pk + sk);
          if constexpr (MODE == kAverage) {
            a = add(a, p);
          } else {
            const float w = __fmul_rn(__fmul_rn(__ldg(window + si), __ldg(window + pi + sj)),
                                      __ldg(window + pi + pj + sk));
            a = hann_add(a, p, w);
          }
        }
        out[c * vol + v] = a;
      }
    }
  }
}

template <typename T, int MODE>
__global__ void __launch_bounds__(kThreads, 4)  // 64 registers: no spills
aggregate_kernel(const T* __restrict__ patches, T* __restrict__ out, T* __restrict__ counts, int C, int I, int J,
                 int K, int pi, int pj, int pk, const int32_t* __restrict__ boxes, int n, int lo_i, int lo_j,
                 int lo_k, int hi_i, int hi_j, int hi_k, int tiles_j, int tiles_k,
                 const float* __restrict__ window) {
  __shared__ Box list[kList];
  __shared__ int warp_kept[kThreads / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int tile = blockIdx.x;
  const int tk = tile % tiles_k, tj = (tile / tiles_k) % tiles_j, ti = tile / (tiles_k * tiles_j);
  const int i0 = lo_i + ti * kTileI, j0 = lo_j + tj * kTileJ, k0 = lo_k + tk * kTileK;
  const int i1 = min(i0 + kTileI, hi_i), j1 = min(j0 + kTileJ, hi_j), k1 = min(k0 + kTileK, hi_k);
  const int j = j0 + warp, k = k0 + lane;
  const bool mine = j < j1 && k < k1;
  const long long vol = (long long)I * J * K;
  int kept = 0, base = 0;
  for (;;) {
    if (base < n) {
      // each thread tests one box of the next chunk of the table against the tile
      Box b;
      bool meets = false;
      if (base + t < n) {
        const int32_t* r = boxes + (long long)(base + t) * kBoxInts;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          b.lo[a] = __ldg(r + a);
          b.hi[a] = __ldg(r + 3 + a);
          b.off[a] = __ldg(r + 6 + a) - b.lo[a];
        }
        b.p = __ldg(r + 9);
        meets = b.lo[0] < i1 && b.hi[0] > i0 && b.lo[1] < j1 && b.hi[1] > j0 && b.lo[2] < k1 && b.hi[2] > k0;
      }
      const unsigned ballot = __ballot_sync(0xffffffffu, meets);
      if (lane == 0) warp_kept[warp] = __popc(ballot);
      __syncthreads();
      int before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < kThreads / 32; ++w) {
        const int s = warp_kept[w];
        before += w < warp ? s : 0;
        total += s;
      }
      if (kept + total <= kList) {  // keep this chunk's boxes, in table order, after the earlier ones
        if (meets) list[kept + before + __popc(ballot & ((1u << lane) - 1u))] = b;
        kept += total;
        base += kThreads;
        __syncthreads();
        continue;
      }
      // the list is full: apply it, then test this chunk again against an empty list
    }
    if (mine && kept) fold<T, MODE>(list, kept, patches, out, counts, C, J, K, vol, pi, pj, pk, window, i0, i1, j, k);
    if (base >= n) break;
    kept = 0;
    __syncthreads();
  }
}

// ---- get_output: out / counts.clamp(min=1), the single-channel count broadcast over C ----------

__device__ __forceinline__ float divide(float a, float c) { return __fdiv_rn(a, c < 1.0f ? 1.0f : c); }
__device__ __forceinline__ double divide(double a, double c) { return __ddiv_rn(a, c < 1.0 ? 1.0 : c); }
__device__ __forceinline__ f16 divide(f16 a, f16 c) {
  const float n = to_float(c);
  return round_f16(__fdiv_rn(to_float(a), n < 1.0f ? 1.0f : n));
}
__device__ __forceinline__ bf16 divide(bf16 a, bf16 c) {
  const float n = to_float(c);
  return round_bf16(__fdiv_rn(to_float(a), n < 1.0f ? 1.0f : n));
}
template <typename T, typename = std::enable_if_t<std::is_integral<T>::value>>
__device__ __forceinline__ float divide(T a, T c) {  // true division of integers: both cast to fp32
  return __fdiv_rn((float)a, (float)(c < (T)1 ? (T)1 : c));
}

template <typename T>
__global__ void __launch_bounds__(256)
aggregate_finish_kernel(const T* __restrict__ out, const T* __restrict__ counts,
                        decltype(divide(T{}, T{}))* __restrict__ dst, long long vox) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // voxel; blockIdx.y = channel
  if (v >= vox) return;
  const long long e = (long long)blockIdx.y * vox + v;
  dst[e] = divide(ld(out + e), ld(counts + v));
}

template <typename T, int MODE>
void launch_aggregate(const void* patches, void* out, void* counts, int C, int I, int J, int K, int pi, int pj,
                      int pk, const int32_t* boxes, int n, const int lo[3], const int hi[3],
                      const float* window, cudaStream_t st) {
  const int tiles_i = (hi[0] - lo[0] + kTileI - 1) / kTileI;
  const int tiles_j = (hi[1] - lo[1] + kTileJ - 1) / kTileJ;
  const int tiles_k = (hi[2] - lo[2] + kTileK - 1) / kTileK;
  const unsigned blocks = (unsigned)((long long)tiles_i * tiles_j * tiles_k);
  aggregate_kernel<T, MODE><<<blocks, kThreads, 0, st>>>((const T*)patches, (T*)out, (T*)counts, C, I, J, K, pi, pj,
                                                         pk, boxes, n, lo[0], lo[1], lo[2], hi[0], hi[1], hi[2],
                                                         tiles_j, tiles_k, window);
  launched();
}

template <typename T>
void launch_finish(const void* out, const void* counts, void* dst, int C, long long vox, cudaStream_t st) {
  const dim3 grid((unsigned)((vox + 255) / 256), (unsigned)C);
  aggregate_finish_kernel<T><<<grid, 256, 0, st>>>((const T*)out, (const T*)counts,
                                                   (decltype(divide(T{}, T{}))*)dst, vox);
  launched();
}

}  // namespace
}  // namespace tio

using namespace tio;

extern "C" int tio_aggregate_patches(const void* patches, void* out, void* counts, int dtype, int mode, int C,
                                     int I, int J, int K, int B, int pi, int pj, int pk, int n,
                                     const int32_t* boxes, const int32_t* boxes_device, const float* window,
                                     void* stream) {
  TIO_CHECK_ARG(patches && out && boxes && boxes_device, "tio_aggregate_patches: null pointer");
  TIO_CHECK_ARG(mode == kCrop || mode == kAverage || mode == kHann, "tio_aggregate_patches: mode %d not in 0..2",
                mode);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_F64, "tio_aggregate_patches: unknown dtype %d", dtype);
  const bool floating = dtype == TIO_F32 || dtype == TIO_F16 || dtype == TIO_BF16 || dtype == TIO_F64;
  TIO_CHECK_ARG(mode != kHann || floating, "tio_aggregate_patches: hann needs a floating-point dtype, got %d",
                dtype);
  TIO_CHECK_ARG(mode == kCrop || counts, "tio_aggregate_patches: null counts");
  TIO_CHECK_ARG(mode != kHann || window, "tio_aggregate_patches: null window");
  TIO_CHECK_ARG(C > 0 && I > 0 && J > 0 && K > 0 && B > 0 && pi > 0 && pj > 0 && pk > 0 && n > 0 && n <= B,
                "tio_aggregate_patches: bad shape");
  int lo[3] = {I, J, K}, hi[3] = {0, 0, 0};
  const int size[3] = {I, J, K}, patch[3] = {pi, pj, pk};
  for (int e = 0; e < n; ++e) {
    const int32_t* r = boxes + (long long)e * kBoxInts;
    for (int a = 0; a < 3; ++a) {
      TIO_CHECK_ARG(0 <= r[a] && r[a] < r[3 + a] && r[3 + a] <= size[a],
                    "tio_aggregate_patches: box %d is empty or outside the buffer on axis %d", e, a);
      TIO_CHECK_ARG(0 <= r[6 + a] && r[6 + a] + (r[3 + a] - r[a]) <= patch[a],
                    "tio_aggregate_patches: box %d is outside its patch on axis %d", e, a);
      lo[a] = r[a] < lo[a] ? r[a] : lo[a];
      hi[a] = r[3 + a] > hi[a] ? r[3 + a] : hi[a];
    }
    TIO_CHECK_ARG(0 <= r[9] && r[9] < B, "tio_aggregate_patches: box %d names patch %d of %d", e, r[9], B);
  }
  TIO_CHECK_ARG((long long)((hi[0] - lo[0] + kTileI - 1) / kTileI) * ((hi[1] - lo[1] + kTileJ - 1) / kTileJ) *
                        ((hi[2] - lo[2] + kTileK - 1) / kTileK) < (1ll << 31),
                "tio_aggregate_patches: too many tiles");
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_AGGREGATE(T, M) \
  launch_aggregate<T, M>(patches, out, counts, C, I, J, K, pi, pj, pk, boxes_device, n, lo, hi, window, st)
  if (mode == kCrop) {  // bytes moved verbatim; bool goes as TIO_U8
    switch (dtype) {
      case TIO_U8: case TIO_I8: TIO_AGGREGATE(uint8_t, kCrop); break;
      case TIO_I16: case TIO_F16: case TIO_BF16: TIO_AGGREGATE(uint16_t, kCrop); break;
      case TIO_F32: case TIO_I32: TIO_AGGREGATE(uint32_t, kCrop); break;
      default: TIO_AGGREGATE(uint64_t, kCrop); break;
    }
  } else if (mode == kAverage) {
#define TIO_AVERAGE(T) TIO_AGGREGATE(T, kAverage)
    TIO_IMAGE_DISPATCH(dtype, "tio_aggregate_patches", TIO_AVERAGE)
#undef TIO_AVERAGE
  } else {
    switch (dtype) {
      case TIO_F32: TIO_AGGREGATE(float, kHann); break;
      case TIO_F16: TIO_AGGREGATE(f16, kHann); break;
      case TIO_BF16: TIO_AGGREGATE(bf16, kHann); break;
      default: TIO_AGGREGATE(double, kHann); break;
    }
  }
#undef TIO_AGGREGATE
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_aggregate_finish(const void* out, const void* counts, void* dst, int dtype, int C,
                                    int64_t vox, void* stream) {
  TIO_CHECK_ARG(out && counts && dst, "tio_aggregate_finish: null pointer");
  TIO_CHECK_ARG(C > 0 && C <= 65535 && vox > 0 && (vox + 255) / 256 < (1ll << 31), "tio_aggregate_finish: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_FINISH(T) launch_finish<T>(out, counts, dst, C, vox, st)
  TIO_IMAGE_DISPATCH(dtype, "tio_aggregate_finish", TIO_FINISH)
#undef TIO_FINISH
  TIO_CHECK_LAUNCH();
  return 0;
}

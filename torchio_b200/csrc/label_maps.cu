// label_maps.cu — the label-map utilities of TorchIO 2.0.0a2 (transforms/label/) in one pass each.
//
// tio_label_lut      RemapLabels / RemoveLabels / SequentialLabels and the inverses: the reference
//                    runs one compare pass and one masked index_put per table entry; here every
//                    voxel is looked up once (label_lookup.cuh) and written in the map's dtype.
// tio_label_contour  Contour: pad with -1, erode by a 3x3x3 min (max_pool3d of the negation), compare
//                    with the voxel.  A CTA owns a (J, K) tile with a one-voxel halo and marches along
//                    I, keeping the 3x3 (J, K) minimum of the last three planes in registers.
#include "common.cuh"
#include "label_lookup.cuh"

namespace tio {

namespace {

// ---- lookup -------------------------------------------------------------------------------------

constexpr int kLutThreads = 256;
constexpr int kSharedEntries = 2048;  // larger tables are searched in global memory

template <typename T> struct LutKey { typedef long long type; };
template <> struct LutKey<float> { typedef float type; };

template <typename T>
__global__ void __launch_bounds__(kLutThreads)
label_lut_kernel(const T* __restrict__ src, T* __restrict__ dst, int64_t count,
                 const typename LutKey<T>::type* __restrict__ keys, const T* __restrict__ values, int n,
                 int identity, int vectorised) {
  typedef typename LutKey<T>::type K;
  extern __shared__ __align__(16) unsigned char smem[];
  T* lut = reinterpret_cast<T*>(smem);  // 8-bit maps: the output of every byte value
  const K* k_tab = keys;
  const T* v_tab = values;
  if constexpr (kByteLabels<T>) {
    const T v = (T)(unsigned char)threadIdx.x;  // kLutThreads == 256 entries
    const int slot = sorted_slot((K)v, keys, n);
    lut[threadIdx.x] = slot >= 0 ? values[slot] : (identity ? v : (T)0);
    __syncthreads();
  } else if (n <= kSharedEntries) {
    K* sk = reinterpret_cast<K*>(smem);
    T* sv = reinterpret_cast<T*>(sk + n);
    for (int i = threadIdx.x; i < n; i += kLutThreads) {
      sk[i] = keys[i];
      sv[i] = values[i];
    }
    __syncthreads();
    k_tab = sk;
    v_tab = sv;
  }
  auto map = [&](T v) -> T {
    if constexpr (kByteLabels<T>) {
      return lut[(unsigned)(unsigned char)v];
    } else {
      const int slot = find_slot<T, K>(v, nullptr, k_tab, n);
      return slot >= 0 ? v_tab[slot] : (identity ? v : (T)0);
    }
  };
  constexpr int kVec = 16 / sizeof(T);
  union Pack {
    uint4 raw;
    T e[kVec];
  };
  const int64_t stride = (int64_t)gridDim.x * kLutThreads;
  const int64_t first = (int64_t)blockIdx.x * kLutThreads + threadIdx.x;
  const int64_t n_vec = vectorised ? count / kVec : 0;
  for (int64_t i = first; i < n_vec; i += stride) {
    Pack p;
    p.raw = __ldg(reinterpret_cast<const uint4*>(src) + i);
#pragma unroll
    for (int j = 0; j < kVec; ++j) p.e[j] = map(p.e[j]);
    reinterpret_cast<uint4*>(dst)[i] = p.raw;
  }
  for (int64_t i = n_vec * kVec + first; i < count; i += stride) dst[i] = map(src[i]);
}

template <typename T>
void launch_lut(const void* src, void* dst, int64_t count, const void* keys, const void* values, int n,
                int identity, cudaStream_t st) {
  typedef typename LutKey<T>::type K;
  const bool vectorised = ((uintptr_t)src % 16 == 0) && ((uintptr_t)dst % 16 == 0);
  int64_t blocks = (count / (16 / sizeof(T)) + kLutThreads - 1) / kLutThreads;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  if (blocks < 1) blocks = 1;
  size_t smem = 0;
  if (kByteLabels<T>) smem = 256 * sizeof(T);
  else if (n <= kSharedEntries) smem = (size_t)n * (sizeof(K) + sizeof(T));
  label_lut_kernel<T><<<(unsigned)blocks, kLutThreads, smem, st>>>(
      (const T*)src, (T*)dst, count, (const K*)keys, (const T*)values, n, identity, vectorised ? 1 : 0);
  launched();
}

// ---- contour ------------------------------------------------------------------------------------

constexpr int kTileK = 32, kTileJ = 16;  // outputs per CTA: each thread owns 4 consecutive K
constexpr int kHaloK = kTileK + 2, kHaloJ = kTileJ + 2;
constexpr int kContourThreads = (kTileK / 4) * kTileJ;
constexpr int kPlanesPerCta = 64;  // I is cut into runs: two extra planes per run buy parallelism

// min that returns NaN when either operand is NaN (max_pool3d propagates NaN; fminf drops it)
__device__ __forceinline__ float min_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

template <typename T>
__global__ void __launch_bounds__(kContourThreads)
label_contour_kernel(const T* __restrict__ src, float* __restrict__ dst, int I, int J, int K, int tiles_k,
                     int vectorised) {
  __shared__ float plane[2][kHaloJ][kHaloK];
  const int j0 = (blockIdx.x / tiles_k) * kTileJ, k0 = (blockIdx.x % tiles_k) * kTileK;
  const int i_begin = blockIdx.y * kPlanesPerCta, i_end = min(I, i_begin + kPlanesPerCta);
  const size_t vol = (size_t)I * J * K;
  const T* s = src + blockIdx.z * vol;
  float* d = dst + blockIdx.z * vol;
  const int lj = threadIdx.x / (kTileK / 4), lk = (threadIdx.x % (kTileK / 4)) * 4;
  const int j = j0 + lj, k = k0 + lk;

  float m_prev[4], m_cur[4], x_cur[4];  // 3x3 minima of planes p-2, p-1 and the centre of p-1
  for (int p = i_begin - 1; p <= i_end; ++p) {
    // plane p with its halo, float(v), -1 outside the volume (F.pad(value=-1))
    float(*buf)[kHaloK] = plane[(p + 1) & 1];
    for (int e = threadIdx.x; e < kHaloJ * kHaloK; e += kContourThreads) {
      const int r = e / kHaloK, c = e % kHaloK;
      const int jj = j0 - 1 + r, kk = k0 - 1 + c;
      float v = -1.0f;
      if (p >= 0 && p < I && jj >= 0 && jj < J && kk >= 0 && kk < K) v = (float)s[((size_t)p * J + jj) * K + kk];
      buf[r][c] = v;
    }
    __syncthreads();  // the buffer written here was last read two planes ago, before this barrier
    float col[6], m[4], x[4];
#pragma unroll
    for (int c = 0; c < 6; ++c) col[c] = min_nan(min_nan(buf[lj][lk + c], buf[lj + 1][lk + c]), buf[lj + 2][lk + c]);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      m[q] = min_nan(min_nan(col[q], col[q + 1]), col[q + 2]);
      x[q] = buf[lj + 1][lk + 1 + q];
    }
    if (p > i_begin && j < J) {  // plane p - 1 has all three neighbour planes
      float o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) o[q] = min_nan(min_nan(m_prev[q], m_cur[q]), m[q]) != x_cur[q] ? 1.0f : 0.0f;
      float* out = d + ((size_t)(p - 1) * J + j) * K + k;
      if (vectorised && k + 4 <= K) {
        *reinterpret_cast<float4*>(out) = make_float4(o[0], o[1], o[2], o[3]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (k + q < K) out[q] = o[q];
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      m_prev[q] = m_cur[q];
      m_cur[q] = m[q];
      x_cur[q] = x[q];
    }
  }
}

template <typename T>
void launch_contour(const void* src, float* dst, int volumes, int I, int J, int K, cudaStream_t st) {
  const int tiles_k = (K + kTileK - 1) / kTileK, tiles_j = (J + kTileJ - 1) / kTileJ;
  const bool vectorised = K % 4 == 0 && (uintptr_t)dst % 16 == 0;
  const dim3 grid((unsigned)(tiles_k * tiles_j), (unsigned)((I + kPlanesPerCta - 1) / kPlanesPerCta),
                  (unsigned)volumes);
  label_contour_kernel<T><<<grid, kContourThreads, 0, st>>>((const T*)src, dst, I, J, K, tiles_k,
                                                            vectorised ? 1 : 0);
  launched();
}

}  // namespace

}  // namespace tio

extern "C" int tio_label_lut(const void* src, void* dst, int dtype, int64_t count, const void* keys,
                             const void* values, int n, int identity, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst, "tio_label_lut: null source or output");
  TIO_CHECK_ARG(n >= 0 && (n == 0 || (keys && values)), "tio_label_lut: null table");
  TIO_CHECK_ARG(count >= 0, "tio_label_lut: bad count");
  TIO_CHECK_ARG((dtype != TIO_U8 && dtype != TIO_I8) || n <= 256, "tio_label_lut: %d keys for an 8-bit map", n);
  if (count == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_LUT(T) launch_lut<T>(src, dst, count, keys, values, n, identity, st)
  TIO_LABEL_DISPATCH(dtype, "tio_label_lut", TIO_LUT)
#undef TIO_LUT
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_label_contour(const void* src, int dtype, int volumes, int I, int J, int K, float* dst,
                                 void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst, "tio_label_contour: null source or output");
  TIO_CHECK_ARG(volumes > 0 && volumes <= 65535 && I > 0 && J > 0 && K > 0, "tio_label_contour: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_CONTOUR(T) launch_contour<T>(src, dst, volumes, I, J, K, st)
  TIO_LABEL_DISPATCH(dtype, "tio_label_contour", TIO_CONTOUR)
#undef TIO_CONTOUR
  TIO_CHECK_LAUNCH();
  return 0;
}

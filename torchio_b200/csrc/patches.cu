// patches.cu — patch extraction for the Queue path (SURVEY §8 f-2).
//
// The reference cuts patches one at a time as tensor views
// (`image[:, si, sj, sk]`, data/sampler.py:54-67) and later copies each of them
// again in `torch.stack` when a batch is collated (loader.py:15-24,
// data/batch.py:52-58).  On the device one launch gathers all `n` patches of a
// volume into a dense (n, C, pi, pj, pk) block, reading every source byte once.
// Pure data movement: bound by HBM, algorithmic bytes = 2 x patch bytes.
#include "common.cuh"

namespace tio {

// General path: one thread row-group per (patch, channel, i, j) row, threads along k.
template <typename T>
__global__ void __launch_bounds__(256)
crop_patches_kernel(const T* __restrict__ src, T* __restrict__ dst, int C, int I, int J, int K, int n,
                    const int32_t* __restrict__ corners, int pi, int pj, int pk) {
  const int rows_per_block = blockDim.y;
  const long long row = (long long)blockIdx.x * rows_per_block + threadIdx.y;  // over n*C*pi*pj
  const long long total_rows = (long long)n * C * pi * pj;
  if (row >= total_rows) return;
  const int j = (int)(row % pj);
  const int i = (int)((row / pj) % pi);
  const int c = (int)((row / ((long long)pj * pi)) % C);
  const int p = (int)(row / ((long long)pj * pi * C));
  const int ci = corners[3 * p + 0], cj = corners[3 * p + 1], ck = corners[3 * p + 2];
  const T* s = src + (((long long)c * I + (ci + i)) * J + (cj + j)) * K + ck;
  T* d = dst + row * pk;
  for (int k = threadIdx.x; k < pk; k += blockDim.x) d[k] = s[k];
}

// 16 bytes per thread (rows that are multiples of 16 bytes, 16-byte aligned destination): one
// 128-bit store per thread; the source row starts wherever the corner puts it, so it is read
// with one 128-bit load when that address happens to be aligned and element by element
// otherwise (a warp still reads one contiguous 512-byte span either way).
template <typename T>
__global__ void __launch_bounds__(256)
crop_patches_vec_kernel(const T* __restrict__ src, T* __restrict__ dst, int C, int I, int J, int K,
                        long long units, const int32_t* __restrict__ corners, int pi, int pj, int pk) {
  constexpr int V = 16 / (int)sizeof(T);
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over n*C*pi*pj*(pk/V)
  if (u >= units) return;
  const int per_row = pk / V;
  const long long row = u / per_row;
  const int kq = (int)(u - row * per_row) * V;
  const int j = (int)(row % pj);
  const int i = (int)((row / pj) % pi);
  const int c = (int)((row / ((long long)pj * pi)) % C);
  const int p = (int)(row / ((long long)pj * pi * C));
  const int ci = __ldg(corners + 3 * p), cj = __ldg(corners + 3 * p + 1), ck = __ldg(corners + 3 * p + 2);
  const T* s = src + (((long long)c * I + (ci + i)) * J + (cj + j)) * K + ck + kq;
  uint4 v;
  if (((uintptr_t)s & 15) == 0) {
    v = __ldg(reinterpret_cast<const uint4*>(s));
  } else {
    T t[V];
#pragma unroll
    for (int e = 0; e < V; ++e) t[e] = __ldg(s + e);
    memcpy(&v, t, 16);
  }
  *reinterpret_cast<uint4*>(dst + row * pk + kq) = v;
}

template <typename T>
static void launch_crop(const void* src, void* dst, int C, int I, int J, int K, int n,
                        const int32_t* corners, int pi, int pj, int pk, cudaStream_t st) {
  const long long rows = (long long)n * C * pi * pj;
  constexpr int V = 16 / (int)sizeof(T);
  if (pk % V == 0 && ((uintptr_t)dst & 15) == 0) {
    const long long units = rows * (pk / V);
    const unsigned blocks = (unsigned)((units + 255) / 256);
    crop_patches_vec_kernel<T><<<blocks, 256, 0, st>>>((const T*)src, (T*)dst, C, I, J, K, units, corners, pi, pj, pk);
    launched();
    return;
  }
  const int tx = pk >= 128 ? 128 : (pk >= 64 ? 64 : 32);
  dim3 block(tx, 256 / tx);
  const unsigned blocks = (unsigned)((rows + block.y - 1) / block.y);
  crop_patches_kernel<T><<<blocks, block, 0, st>>>((const T*)src, (T*)dst, C, I, J, K, n, corners, pi, pj, pk);
  launched();
}

}  // namespace tio

using namespace tio;

extern "C" int tio_crop_patches(const void* src, void* dst, int elem_bytes, int C, int I, int J,
                                int K, int n, const int32_t* corners, int pi, int pj, int pk,
                                void* stream) {
  TIO_CHECK_ARG(src && dst && corners, "tio_crop_patches: null pointer");
  TIO_CHECK_ARG(C > 0 && I > 0 && J > 0 && K > 0 && n > 0, "tio_crop_patches: bad shape");
  TIO_CHECK_ARG(pi > 0 && pj > 0 && pk > 0 && pi <= I && pj <= J && pk <= K,
                "tio_crop_patches: patch (%d,%d,%d) does not fit the volume (%d,%d,%d)", pi, pj, pk, I, J, K);
  TIO_CHECK_ARG((long long)n * C * pi * pj / 2 < (1ll << 31), "tio_crop_patches: too many rows");
  TIO_CHECK_ARG((long long)n * C * pi * pj * ((pk + 3) / 4) / 256 < (1ll << 31), "tio_crop_patches: too many elements");
  cudaStream_t st = (cudaStream_t)stream;
  switch (elem_bytes) {
    case 1: launch_crop<uint8_t>(src, dst, C, I, J, K, n, corners, pi, pj, pk, st); break;
    case 2: launch_crop<uint16_t>(src, dst, C, I, J, K, n, corners, pi, pj, pk, st); break;
    case 4: launch_crop<uint32_t>(src, dst, C, I, J, K, n, corners, pi, pj, pk, st); break;
    case 8: launch_crop<uint64_t>(src, dst, C, I, J, K, n, corners, pi, pj, pk, st); break;
    default: TIO_CHECK_ARG(false, "tio_crop_patches: element size %d not in {1,2,4,8}", elem_bytes);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

// ---- tio_remap: Flip / Crop / Pad as one index-remap copy (SURVEY §8 f-3) ----------
// out[b,c,oi,oj,ok] = in[b,c, f_i(m_i(oi - off_i)), f_j(...), f_k(...)], where m is the
// padding rule for indices outside [0,n) (constant -> fill value, replicate -> clamp,
// reflect -> mirror without repeating the edge, circular -> wrap) and f reverses the
// axis when the element's flip bit is set.  Replaces torch.flip + torch.where
// (spatial/flip.py:233-263), the crop slicing (crop.py:84-101) and F.pad
// (_padding.py:73-104) on 5-D batches.  Pure data movement: 2 x bytes of the output.
namespace tio {

__device__ __forceinline__ int remap_index(int s, int n, int mode, bool& outside) {
  if ((unsigned)s < (unsigned)n) return s;
  switch (mode) {
    case 1: return s < 0 ? 0 : n - 1;                                  // replicate
    case 2: {                                                          // reflect
      if (n == 1) return 0;
      const int period = 2 * (n - 1);
      int r = s % period;
      if (r < 0) r += period;
      return r < n ? r : period - r;
    }
    case 3: { int r = s % n; return r < 0 ? r + n : r; }               // circular
    default: outside = true; return 0;                                 // constant
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
remap_kernel(const T* __restrict__ src, T* __restrict__ dst, int B, int C, int I, int J, int K, int OI,
             int OJ, int OK, int off_i, int off_j, int off_k, int mode, T fill,
             const uint8_t* __restrict__ flip) {
  const long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y;  // over B*C*OI*OJ
  const long long rows = (long long)B * C * OI * OJ;
  if (row >= rows) return;
  const int oj = (int)(row % OJ);
  const int oi = (int)((row / OJ) % OI);
  const long long bc = row / ((long long)OJ * OI);
  const int b = (int)(bc / C);
  const uint8_t fl = flip ? flip[b] : 0;
  bool outside = false;
  int si = remap_index(oi - off_i, I, mode, outside);
  int sj = remap_index(oj - off_j, J, mode, outside);
  if (fl & 1) si = I - 1 - si;
  if (fl & 2) sj = J - 1 - sj;
  const T* s = src + ((bc * I + si) * J + sj) * K;
  T* d = dst + row * OK;
  for (int ok = threadIdx.x; ok < OK; ok += blockDim.x) {
    bool out_k = outside;
    int sk = remap_index(ok - off_k, K, mode, out_k);
    if (fl & 4) sk = K - 1 - sk;
    d[ok] = out_k ? fill : s[sk];
  }
}

// 16 bytes of an output row per thread (rows that are multiples of 16 bytes, 16-byte aligned
// destination): one 128-bit store; the source elements come with one 128-bit load when the unit
// maps to an in-range, unflipped, aligned run of the source row, element by element otherwise
// (padding, flips along K, unaligned crops).
template <typename T>
__global__ void __launch_bounds__(256)
remap_vec_kernel(const T* __restrict__ src, T* __restrict__ dst, int B, int C, int I, int J, int K, int OI,
                 int OJ, int OK, int off_i, int off_j, int off_k, int mode, T fill,
                 const uint8_t* __restrict__ flip, long long units) {
  constexpr int V = 16 / (int)sizeof(T);
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over B*C*OI*OJ*(OK/V)
  if (u >= units) return;
  const int per_row = OK / V;
  const long long row = u / per_row;
  const int ok0 = (int)(u - row * per_row) * V;
  const int oj = (int)(row % OJ);
  const int oi = (int)((row / OJ) % OI);
  const long long bc = row / ((long long)OJ * OI);
  const int b = (int)(bc / C);
  const uint8_t fl = flip ? __ldg(flip + b) : 0;
  bool outside = false;
  int si = remap_index(oi - off_i, I, mode, outside);
  int sj = remap_index(oj - off_j, J, mode, outside);
  if (fl & 1) si = I - 1 - si;
  if (fl & 2) sj = J - 1 - sj;
  const T* s = src + ((bc * I + si) * J + sj) * K;
  const int sk0 = ok0 - off_k;
  uint4 v;
  const bool whole = !outside && sk0 >= 0 && sk0 + V <= K;  // the unit maps to V in-range source elements
  const int first = (fl & 4) ? K - V - sk0 : sk0;           // ... which start here (mirrored run when flipped)
  if (whole && ((uintptr_t)(s + first) & 15) == 0) {
    v = __ldg(reinterpret_cast<const uint4*>(s + first));
    if (fl & 4) {  // reverse the V elements in registers
      T t[V], r[V];
      memcpy(t, &v, 16);
#pragma unroll
      for (int e = 0; e < V; ++e) r[e] = t[V - 1 - e];
      memcpy(&v, r, 16);
    }
  } else {
    T t[V];
#pragma unroll
    for (int e = 0; e < V; ++e) {
      bool out_k = outside;
      int sk = remap_index(sk0 + e, K, mode, out_k);
      if (fl & 4) sk = K - 1 - sk;
      t[e] = out_k ? fill : __ldg(s + sk);
    }
    memcpy(&v, t, 16);
  }
  *reinterpret_cast<uint4*>(dst + row * OK + ok0) = v;
}

template <typename T>
static void launch_remap(const void* src, void* dst, int B, int C, int I, int J, int K, int OI, int OJ,
                         int OK, int oi, int oj, int ok, int mode, unsigned long long fill_bits,
                         const uint8_t* flip, cudaStream_t st) {
  T fill;
  memcpy(&fill, &fill_bits, sizeof(T));
  const long long rows = (long long)B * C * OI * OJ;
  constexpr int V = 16 / (int)sizeof(T);
  if (OK % V == 0 && ((uintptr_t)dst & 15) == 0 && rows * (OK / V) / 256 < (1ll << 31)) {
    const long long units = rows * (OK / V);
    remap_vec_kernel<T><<<(unsigned)((units + 255) / 256), 256, 0, st>>>(
        (const T*)src, (T*)dst, B, C, I, J, K, OI, OJ, OK, oi, oj, ok, mode, fill, flip, units);
    launched();
    return;
  }
  const int tx = OK >= 128 ? 128 : (OK >= 64 ? 64 : 32);
  dim3 block(tx, 256 / tx);
  const unsigned blocks = (unsigned)((rows + block.y - 1) / block.y);
  remap_kernel<T><<<blocks, block, 0, st>>>((const T*)src, (T*)dst, B, C, I, J, K, OI, OJ, OK, oi, oj, ok,
                                            mode, fill, flip);
  launched();
}

}  // namespace tio

extern "C" int tio_remap(const void* src, void* dst, int elem_bytes, int B, int C, int I, int J, int K,
                         int OI, int OJ, int OK, int off_i, int off_j, int off_k, int mode,
                         const void* fill, const uint8_t* flip, void* stream) {
  TIO_CHECK_ARG(src && dst && src != dst, "tio_remap: null or aliased src/dst");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0 && OI > 0 && OJ > 0 && OK > 0,
                "tio_remap: non-positive shape");
  TIO_CHECK_ARG(mode >= 0 && mode <= 3, "tio_remap: mode %d not in 0..3", mode);
  TIO_CHECK_ARG((long long)B * C * OI * OJ / 2 < (1ll << 31), "tio_remap: too many rows");
  if (mode == 2)
    TIO_CHECK_ARG(off_i < I && off_j < J && off_k < K && OI - I - off_i < I && OJ - J - off_j < J &&
                      OK - K - off_k < K,
                  "tio_remap: reflect padding must be smaller than the axis");
  unsigned long long fill_bits = 0;
  if (fill) memcpy(&fill_bits, fill, (size_t)elem_bytes);
  cudaStream_t st = (cudaStream_t)stream;
  switch (elem_bytes) {
    case 1: launch_remap<uint8_t>(src, dst, B, C, I, J, K, OI, OJ, OK, off_i, off_j, off_k, mode, fill_bits, flip, st); break;
    case 2: launch_remap<uint16_t>(src, dst, B, C, I, J, K, OI, OJ, OK, off_i, off_j, off_k, mode, fill_bits, flip, st); break;
    case 4: launch_remap<uint32_t>(src, dst, B, C, I, J, K, OI, OJ, OK, off_i, off_j, off_k, mode, fill_bits, flip, st); break;
    case 8: launch_remap<uint64_t>(src, dst, B, C, I, J, K, OI, OJ, OK, off_i, off_j, off_k, mode, fill_bits, flip, st); break;
    default: TIO_CHECK_ARG(false, "tio_remap: element size %d not in {1,2,4,8}", elem_bytes);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

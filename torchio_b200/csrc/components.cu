// components.cu — KeepLargestComponent of TorchIO 2.0.0a2 (transforms/label/keep_largest.py) on the GPU:
// connected components of every selected label of every batch element in one union-find.
//
// A voxel "takes part" when it carries a selected label; two neighbouring voxels that both take part
// are connected when their values compare equal (6 face neighbours, or 26).  Each component's root
// is the smallest C-order index (i*J + j)*K + k of its voxels: links only ever go from a larger index
// to a smaller one (min-hooking with atomicMin), so the forest, and every result, is independent of
// the order in which the atomics land.
//
// tio_components       1. per 4 x 8 x 32 tile: union-find in shared memory, global roots written out
//                      2. the backward neighbours that lie in another tile: global union-find
//                      3. every voxel's parent set to its root; component sizes added at the roots
//                         (one atomic per run of a warp's lanes that share a root)
// tio_component_roots  the value of every root, compacted (labels=None on 32/64-bit and fp32 maps:
//                      the caller sorts the distinct values into the slot table)
// tio_keep_largest     4. per (element, label slot) the winner: atomicMax of (size << 32) | ~root,
//                         so the largest component and, among equal sizes, the smallest root
//                      5. in place: a voxel that takes part and whose root is not its slot's winner
//                         gets the background value; no other voxel is written
#include <cstring>

#include "common.cuh"
#include "label_lookup.cuh"

namespace tio {

namespace {

constexpr unsigned kNoRoot = 0xFFFFFFFFu;  // a voxel that takes no part
constexpr int kTI = 4, kTJ = 8, kTK = 32;   // tile: one warp per K row, one thread per (J, K) column
constexpr int kTileVox = kTI * kTJ * kTK;
constexpr int kThreads = kTJ * kTK;
constexpr int kFlatThreads = 256;

enum { kModeKeys = 0, kModeValue = 1, kModeSearch = 2 };
enum { kFlagPresent = 1, kFlagNaN = 2, kFlagInf = 4 };

template <typename T> struct CcKey { typedef long long type; };
template <> struct CcKey<float> { typedef float type; };

// Which voxels take part, and their label slot.
//   kModeKeys    explicit labels: the slot of the value's key in the ascending table (tio_label_lut's
//                keys and comparison rules); 8-bit maps through a 256-entry LUT in shared memory
//   kModeValue   labels=None on 8/16-bit maps: int(v) != background; the slot is the value itself
//   kModeSearch  labels=None on 32/64-bit and fp32 maps: int(v) != background (fp32: only finite
//                integral values, as int() truncates and data == int(v) then matches only v itself);
//                the slot is the value's position in the table of the roots' distinct values
struct Select {
  int mode;
  int n_keys;
  long long background;
  int has_background;  // 0: no value of the map equals the background label
};

template <typename T>
__device__ __forceinline__ bool is_background(T v, const Select& s) {
  if (!s.has_background) return false;
  if constexpr (sizeof(T) == 4 && T(0.5f) != T(0)) {  // fp32: the host checked it is exact
    return v == (float)s.background;
  } else {
    return (long long)v == s.background;
  }
}

template <typename T>
__device__ __forceinline__ bool takes_part(T v, const Select& s, const int* lut,
                                           const typename CcKey<T>::type* keys) {
  typedef typename CcKey<T>::type K;
  if (s.mode == kModeKeys) return find_slot<T, K>(v, lut, keys, s.n_keys) >= 0;
  if constexpr (T(0.5f) != T(0)) {
    if (!isfinite((float)v) || truncf((float)v) != (float)v) return false;
  }
  return !is_background(v, s);
}

// slot of a voxel that takes part
template <typename T>
__device__ __forceinline__ int slot_of(T v, const Select& s, const int* lut, const typename CcKey<T>::type* keys) {
  typedef typename CcKey<T>::type K;
  if (s.mode == kModeValue) {
    if constexpr (sizeof(T) <= 2 && T(0.5f) == T(0)) {
      return (int)v - (T(-1) < T(0) ? -(1 << (8 * sizeof(T) - 1)) : 0);
    }
    return -1;
  }
  if (s.mode == kModeKeys) return find_slot<T, K>(v, lut, keys, s.n_keys);
  return sorted_slot((K)v, keys, s.n_keys);
}

template <typename T>
__device__ __forceinline__ void build_lut(int* lut, const Select& s, const long long* keys) {
  if constexpr (kByteLabels<T>) {
    if (s.mode == kModeKeys) {
      for (int e = threadIdx.x; e < 256; e += blockDim.x) lut[e] = sorted_slot((long long)(T)(unsigned char)e, keys, s.n_keys);
    }
    __syncthreads();
  }
}

// backward neighbours (smaller C-order index): the 3 face ones first, then the other 10 of the 26
__constant__ signed char kBack[13][3] = {
    {-1, 0, 0}, {0, -1, 0}, {0, 0, -1},
    {-1, -1, -1}, {-1, -1, 0}, {-1, -1, 1}, {-1, 0, -1}, {-1, 0, 1}, {-1, 1, -1}, {-1, 1, 0}, {-1, 1, 1},
    {0, -1, -1}, {0, -1, 1}};

// union-find with min-hooking: the larger root is linked under the smaller one; a failed atomicMin
// returns the root's new parent, and the union continues from there
template <typename I>
__device__ __forceinline__ I find_root(const volatile I* parent, I x) {
  I p;
  while ((p = parent[x]) != x) x = p;
  return x;
}

template <typename I>
__device__ __forceinline__ void unite(I* parent, I a, I b) {
  for (;;) {
    a = find_root<I>(parent, a);
    b = find_root<I>(parent, b);
    if (a == b) return;
    if (a < b) {
      const I t = a;
      a = b;
      b = t;
    }
    const I old = atomicMin(parent + a, b);
    if (old == a) return;
    a = old;
  }
}

struct Shape {
  int I, J, K;
  int tiles_j, tiles_k;
  unsigned long long vox;
};

__device__ __forceinline__ void tile_origin(const Shape& sh, int& i0, int& j0, int& k0) {
  const int t = blockIdx.x;
  k0 = (t % sh.tiles_k) * kTK;
  j0 = ((t / sh.tiles_k) % sh.tiles_j) * kTJ;
  i0 = (t / (sh.tiles_k * sh.tiles_j)) * kTI;
}

// 1. one tile: which voxels take part, union-find over the neighbours inside the tile, global roots
template <typename T>
__global__ void __launch_bounds__(kThreads)
cc_local_kernel(const T* __restrict__ src, unsigned* __restrict__ parent, unsigned* __restrict__ count,
                unsigned* __restrict__ flags, Shape sh, Select sel, const typename CcKey<T>::type* __restrict__ keys,
                int neighbours) {
  __shared__ int s_parent[kTileVox];
  __shared__ T s_value[kTileVox];
  __shared__ int lut[kByteLabels<T> ? 256 : 1];
  build_lut<T>(lut, sel, reinterpret_cast<const long long*>(keys));
  int i0, j0, k0;
  tile_origin(sh, i0, j0, k0);
  const unsigned long long base = blockIdx.y * sh.vox;
  const int lj = threadIdx.x / kTK, lk = threadIdx.x % kTK;
  const int j = j0 + lj, k = k0 + lk;
  int present = 0, nan = 0, inf = 0;
#pragma unroll
  for (int li = 0; li < kTI; ++li) {
    const int l = (li * kTJ + lj) * kTK + lk;
    const int i = i0 + li;
    int p = -1;
    T v = T(0);
    if (i < sh.I && j < sh.J && k < sh.K) {
      v = src[base + ((unsigned long long)i * sh.J + j) * sh.K + k];
      if (takes_part<T>(v, sel, lut, keys)) p = l;
      if constexpr (T(0.5f) != T(0)) {
        nan |= v != v;
        inf |= isinf((float)v);
      }
    }
    present |= p >= 0;
    s_parent[l] = p;
    s_value[l] = v;
  }
  __syncthreads();
#pragma unroll
  for (int li = 0; li < kTI; ++li) {
    const int l = (li * kTJ + lj) * kTK + lk;
    if (s_parent[l] < 0) continue;
    const T v = s_value[l];
    for (int q = 0; q < neighbours; ++q) {
      const int ni = li + kBack[q][0], nj = lj + kBack[q][1], nk = lk + kBack[q][2];
      if (ni < 0 || nj < 0 || nj >= kTJ || nk < 0 || nk >= kTK) continue;
      const int n = (ni * kTJ + nj) * kTK + nk;
      if (s_parent[n] >= 0 && s_value[n] == v) unite<int>(s_parent, l, n);
    }
  }
  __syncthreads();
#pragma unroll
  for (int li = 0; li < kTI; ++li) {
    const int l = (li * kTJ + lj) * kTK + lk;
    const int i = i0 + li;
    if (i >= sh.I || j >= sh.J || k >= sh.K) continue;
    const unsigned long long g = base + ((unsigned long long)i * sh.J + j) * sh.K + k;
    unsigned root = kNoRoot;
    if (s_parent[l] >= 0) {
      const int r = find_root<int>(s_parent, l);
      const int ri = i0 + r / (kTJ * kTK), rj = j0 + (r / kTK) % kTJ, rk = k0 + r % kTK;
      root = (unsigned)(((unsigned long long)ri * sh.J + rj) * sh.K + rk);
    }
    parent[g] = root;
    count[g] = 0;
  }
  const int f = (__syncthreads_or(present) ? kFlagPresent : 0) | (__syncthreads_or(nan) ? kFlagNaN : 0) |
                (__syncthreads_or(inf) ? kFlagInf : 0);
  if (threadIdx.x == 0 && f && (*(volatile unsigned*)(flags + blockIdx.y) & f) != (unsigned)f)
    atomicOr(flags + blockIdx.y, (unsigned)f);
}

// 2. the backward neighbours that lie in another tile
template <typename T>
__global__ void __launch_bounds__(kThreads)
cc_merge_kernel(const T* __restrict__ src, unsigned* parent, Shape sh, int neighbours) {
  int i0, j0, k0;
  tile_origin(sh, i0, j0, k0);
  const unsigned long long base = blockIdx.y * sh.vox;
  unsigned* par = parent + base;
  const T* s = src + base;
  const int lj = threadIdx.x / kTK, lk = threadIdx.x % kTK;
  const int j = j0 + lj, k = k0 + lk;
  if (j >= sh.J || k >= sh.K) return;
  for (int li = 0; li < kTI; ++li) {
    const int i = i0 + li;
    if (i >= sh.I) return;
    const unsigned idx = (unsigned)(((unsigned long long)i * sh.J + j) * sh.K + k);
    if (par[idx] == kNoRoot) continue;
    const T v = s[idx];
    for (int q = 0; q < neighbours; ++q) {
      const int ni = li + kBack[q][0], nj = lj + kBack[q][1], nk = lk + kBack[q][2];
      if (ni >= 0 && nj >= 0 && nj < kTJ && nk >= 0 && nk < kTK) continue;  // done by the tile
      const int gi = i0 + ni, gj = j0 + nj, gk = k0 + nk;
      if (gi < 0 || gj < 0 || gj >= sh.J || gk < 0 || gk >= sh.K) continue;
      const unsigned n = (unsigned)(((unsigned long long)gi * sh.J + gj) * sh.K + gk);
      // equal values take part alike, so the neighbour's value decides
      if (s[n] == v) unite<unsigned>(par, idx, n);
    }
  }
}

// 3. parent := root, and the component sizes at the roots
__global__ void __launch_bounds__(kFlatThreads)
cc_compress_kernel(unsigned* parent, unsigned* __restrict__ count, unsigned long long vox) {
  unsigned* par = parent + blockIdx.y * vox;
  unsigned* cnt = count + blockIdx.y * vox;
  const unsigned long long stride = (unsigned long long)gridDim.x * kFlatThreads;
  const int lane = threadIdx.x & 31;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * kFlatThreads + threadIdx.x; idx < vox;
       idx += stride) {
    const unsigned p = par[idx];
    unsigned root = kNoRoot;
    if (p != kNoRoot) {
      root = find_root<unsigned>(par, p);
      if (root != p) par[idx] = root;
    }
    const unsigned peers = __match_any_sync(__activemask(), root);
    if (root != kNoRoot && lane == __ffs(peers) - 1) atomicAdd(cnt + root, (unsigned)__popc(peers));
  }
}

// the value of every root, compacted into `values` (order unspecified)
template <typename T>
__global__ void __launch_bounds__(kFlatThreads)
cc_roots_kernel(const T* __restrict__ src, const unsigned* __restrict__ parent, unsigned long long vox,
                T* __restrict__ values, unsigned* __restrict__ n_values) {
  const unsigned long long base = blockIdx.y * vox;
  const unsigned long long stride = (unsigned long long)gridDim.x * kFlatThreads;
  const int lane = threadIdx.x & 31;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * kFlatThreads + threadIdx.x; idx < vox;
       idx += stride) {
    const bool is_root = parent[base + idx] == (unsigned)idx;
    const unsigned mask = __activemask();
    const unsigned roots = __ballot_sync(mask, is_root);
    if (!roots) continue;
    const int leader = __ffs(roots) - 1;
    unsigned first = 0;
    if (lane == leader) first = atomicAdd(n_values, (unsigned)__popc(roots));
    first = __shfl_sync(mask, first, leader);
    if (is_root) values[first + __popc(roots & ((1u << lane) - 1))] = src[base + idx];
  }
}

// 4. the winner of every (element, slot): the largest size, then the smallest root
template <typename T>
__global__ void __launch_bounds__(kFlatThreads)
cc_winner_kernel(const T* __restrict__ src, const unsigned* __restrict__ parent, const unsigned* __restrict__ count,
                 unsigned long long vox, Select sel, const typename CcKey<T>::type* __restrict__ keys,
                 unsigned long long* winner, int slots) {
  __shared__ int lut[kByteLabels<T> ? 256 : 1];
  build_lut<T>(lut, sel, reinterpret_cast<const long long*>(keys));
  const unsigned long long base = blockIdx.y * vox;
  unsigned long long* win = winner + (unsigned long long)blockIdx.y * slots;
  const unsigned long long stride = (unsigned long long)gridDim.x * kFlatThreads;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * kFlatThreads + threadIdx.x; idx < vox;
       idx += stride) {
    if (parent[base + idx] != (unsigned)idx) continue;
    const int slot = slot_of<T>(src[base + idx], sel, lut, keys);
    if (slot < 0) continue;
    const unsigned long long key = ((unsigned long long)count[base + idx] << 32) | (kNoRoot - (unsigned)idx);
    if (*(volatile unsigned long long*)(win + slot) < key) atomicMax(win + slot, key);
  }
}

// 5. in place: the voxels of every component that did not win become the background value
template <typename T>
__global__ void __launch_bounds__(kFlatThreads)
cc_write_kernel(T* data, const unsigned* __restrict__ parent, unsigned long long vox, Select sel,
                const typename CcKey<T>::type* __restrict__ keys, const unsigned long long* __restrict__ winner,
                int slots, T fill) {
  __shared__ int lut[kByteLabels<T> ? 256 : 1];
  build_lut<T>(lut, sel, reinterpret_cast<const long long*>(keys));
  const unsigned long long base = blockIdx.y * vox;
  const unsigned long long* win = winner + (unsigned long long)blockIdx.y * slots;
  const unsigned long long stride = (unsigned long long)gridDim.x * kFlatThreads;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * kFlatThreads + threadIdx.x; idx < vox;
       idx += stride) {
    const unsigned root = parent[base + idx];
    if (root == kNoRoot) continue;
    const T v = data[base + idx];
    const int slot = slot_of<T>(v, sel, lut, keys);
    if (slot < 0) continue;
    if (root != kNoRoot - (unsigned)win[slot]) data[base + idx] = fill;
  }
}

dim3 flat_grid(unsigned long long vox, int B) {
  unsigned long long blocks = (vox + kFlatThreads - 1) / kFlatThreads;
  const unsigned long long cap = (unsigned long long)num_sms() * 16 / (unsigned long long)B + 1;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return dim3((unsigned)blocks, (unsigned)B);
}

Shape make_shape(int I, int J, int K) {
  Shape sh;
  sh.I = I;
  sh.J = J;
  sh.K = K;
  sh.tiles_j = (J + kTJ - 1) / kTJ;
  sh.tiles_k = (K + kTK - 1) / kTK;
  sh.vox = (unsigned long long)I * J * K;
  return sh;
}

template <typename T>
void launch_components(const void* src, int B, const Shape& sh, const Select& sel, const void* keys, int neighbours,
                       unsigned* parent, unsigned* count, unsigned* flags, cudaStream_t st) {
  typedef typename CcKey<T>::type K;
  const dim3 tiles((unsigned)(((sh.I + kTI - 1) / kTI) * sh.tiles_j * sh.tiles_k), (unsigned)B);
  cc_local_kernel<T><<<tiles, kThreads, 0, st>>>((const T*)src, parent, count, flags, sh, sel, (const K*)keys,
                                                 neighbours);
  launched();
  cc_merge_kernel<T><<<tiles, kThreads, 0, st>>>((const T*)src, parent, sh, neighbours);
  launched();
  cc_compress_kernel<<<flat_grid(sh.vox, B), kFlatThreads, 0, st>>>(parent, count, sh.vox);
  launched();
}

template <typename T>
void launch_roots(const void* src, int B, unsigned long long vox, const unsigned* parent, void* values,
                  unsigned* n_values, cudaStream_t st) {
  cc_roots_kernel<T><<<flat_grid(vox, B), kFlatThreads, 0, st>>>((const T*)src, parent, vox, (T*)values, n_values);
  launched();
}

template <typename T>
void launch_keep(void* data, int B, unsigned long long vox, const Select& sel, const void* keys,
                 const unsigned* parent, const unsigned* count, unsigned long long* winner, int slots,
                 const void* fill, cudaStream_t st) {
  typedef typename CcKey<T>::type K;
  T value;
  memcpy(&value, fill, sizeof(T));
  const dim3 grid = flat_grid(vox, B);
  cc_winner_kernel<T><<<grid, kFlatThreads, 0, st>>>((const T*)data, parent, count, vox, sel, (const K*)keys, winner,
                                                     slots);
  launched();
  cc_write_kernel<T><<<grid, kFlatThreads, 0, st>>>((T*)data, parent, vox, sel, (const K*)keys, winner, slots, value);
  launched();
}

bool select_ok(int dtype, int mode, int n_keys, const void* keys) {
  if (mode == kModeKeys) return n_keys >= 0 && (n_keys == 0 || keys) && ((dtype != TIO_U8 && dtype != TIO_I8) || n_keys <= 256);
  if (mode == kModeValue) return dtype == TIO_U8 || dtype == TIO_I8 || dtype == TIO_I16;
  if (mode == kModeSearch) return n_keys >= 0 && (n_keys == 0 || keys);
  return false;
}

int value_slots(int dtype) { return dtype == TIO_I16 ? 65536 : 256; }

}  // namespace

}  // namespace tio

extern "C" int tio_components(const void* src, int dtype, int B, int I, int J, int K, int mode, const void* keys,
                              int n_keys, int64_t background, int has_background, int fully_connected,
                              uint32_t* parent, uint32_t* count, uint32_t* flags, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && parent && count && flags, "tio_components: null source, parent, count or flags");
  TIO_CHECK_ARG(B >= 0 && B <= 65535 && I >= 0 && J >= 0 && K >= 0, "tio_components: bad shape");
  TIO_CHECK_ARG((unsigned long long)I * J * K < (1ull << 32),
                "tio_components: %d x %d x %d voxels per element: at most 2^32 - 1", I, J, K);
  TIO_CHECK_ARG(select_ok(dtype, mode, n_keys, keys), "tio_components: mode %d with %d keys for dtype %d", mode,
                n_keys, dtype);
  if (B == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(flags, 0, sizeof(uint32_t) * B, st));
  if ((long long)I * J * K == 0) return 0;
  const Shape sh = make_shape(I, J, K);
  TIO_CHECK_ARG((unsigned long long)((I + kTI - 1) / kTI) * sh.tiles_j * sh.tiles_k < (1ull << 31),
                "tio_components: too many tiles");
  Select sel{mode, n_keys, (long long)background, has_background ? 1 : 0};
  const int neighbours = fully_connected ? 13 : 3;
#define TIO_CC(T) launch_components<T>(src, B, sh, sel, keys, neighbours, parent, count, flags, st)
  TIO_LABEL_DISPATCH(dtype, "tio_components", TIO_CC)
#undef TIO_CC
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_component_roots(const void* src, int dtype, int B, int64_t vox, const uint32_t* parent,
                                   void* values, uint32_t* n_values, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && parent && values && n_values, "tio_component_roots: null source, parent or output");
  TIO_CHECK_ARG(B >= 0 && B <= 65535 && vox >= 0 && (unsigned long long)vox < (1ull << 32),
                "tio_component_roots: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(n_values, 0, sizeof(uint32_t), st));
  if (B == 0 || vox == 0) return 0;
#define TIO_ROOTS(T) launch_roots<T>(src, B, (unsigned long long)vox, parent, values, n_values, st)
  TIO_LABEL_DISPATCH(dtype, "tio_component_roots", TIO_ROOTS)
#undef TIO_ROOTS
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_keep_largest(void* data, int dtype, int B, int64_t vox, int mode, const void* keys, int n_keys,
                                int64_t background, int has_background, const uint32_t* parent,
                                const uint32_t* count, uint64_t* winner, const void* fill, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(data && parent && count && winner && fill, "tio_keep_largest: null data, workspace or fill");
  TIO_CHECK_ARG(B >= 0 && B <= 65535 && vox >= 0 && (unsigned long long)vox < (1ull << 32),
                "tio_keep_largest: bad shape");
  TIO_CHECK_ARG(select_ok(dtype, mode, n_keys, keys), "tio_keep_largest: mode %d with %d keys for dtype %d", mode,
                n_keys, dtype);
  if (B == 0 || vox == 0) return 0;
  const int slots = mode == kModeValue ? value_slots(dtype) : n_keys;
  if (slots == 0) return 0;  // nothing takes part
  Select sel{mode, n_keys, (long long)background, has_background ? 1 : 0};
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(winner, 0, sizeof(uint64_t) * (size_t)B * slots, st));
#define TIO_KEEP(T) launch_keep<T>(data, B, (unsigned long long)vox, sel, keys, parent, count, \
                                   (unsigned long long*)winner, slots, fill, st)
  TIO_LABEL_DISPATCH(dtype, "tio_keep_largest", TIO_KEEP)
#undef TIO_KEEP
  TIO_CHECK_LAUNCH();
  return 0;
}

// label_lookup.cuh — label -> table slot, shared by LabelsToImage (labels_to_image.cu) and the
// label-map lookup tables (label_maps.cu).
//
// A table is n strictly ascending keys.  8-bit maps index a 256-entry LUT built from it; wider
// maps binary-search it (in shared memory when it fits, else in global memory: same code).
#pragma once

#include "common.cuh"

namespace tio {

template <typename T> constexpr bool kByteLabels = sizeof(T) == 1;

// The key a voxel value is looked up under; false = it can match no key.
// K = long long: `label == int(l)` — integer maps compare exactly; an fp32 map compares in fp32,
// and since every key came from int() of a voxel value it is exactly representable, so only
// integral values match.
// K = float (fp32 maps keyed by fp32 values): by value, so -0 finds +0 and NaN finds nothing.
template <typename T, typename K>
__device__ __forceinline__ bool label_key(T v, K& key) {
  key = (K)v;
  return true;
}
template <>
__device__ __forceinline__ bool label_key<float, long long>(float v, long long& key) {
  if (!(fabsf(v) < 9.2e18f) || truncf(v) != v) return false;
  key = (long long)v;
  return true;
}

// slot of `key` in the ascending `keys[0..n)`, or -1
template <typename K>
__device__ __forceinline__ int sorted_slot(K key, const K* keys, int n) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (keys[mid] < key) lo = mid + 1; else hi = mid;
  }
  return (lo < n && keys[lo] == key) ? lo : -1;
}

// slot of `v`: the 256-entry `lut` for 8-bit maps, else a search of `keys`
template <typename T, typename K>
__device__ __forceinline__ int find_slot(T v, const int* lut, const K* keys, int n) {
  if constexpr (kByteLabels<T>) {
    return lut[(unsigned)(unsigned char)v];
  } else {
    K key;
    if (!label_key<T, K>(v, key)) return -1;
    return sorted_slot(key, keys, n);
  }
}

}  // namespace tio

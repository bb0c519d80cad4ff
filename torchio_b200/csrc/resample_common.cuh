// resample_common.cuh — types and per-column arithmetic shared by the K1 kernels.
#pragma once
#include "common.cuh"

namespace tio {


template <typename T>
struct ElemTraits;
template <>
struct ElemTraits<float> {
  static __device__ __forceinline__ float to_f32(float v) { return v; }
  static __device__ __forceinline__ float from_f32(float v) { return v; }
};
#define TIO_INT_TRAITS(T)                                                    \
  template <>                                                                \
  struct ElemTraits<T> {                                                     \
    static __device__ __forceinline__ float to_f32(T v) { return (float)v; } \
    static __device__ __forceinline__ T from_f32(float v) {                  \
      return (T)(long long)v; /* Tensor.to(int): truncation */               \
    }                                                                        \
  };
TIO_INT_TRAITS(uint8_t)
TIO_INT_TRAITS(int8_t)
TIO_INT_TRAITS(int16_t)
TIO_INT_TRAITS(int32_t)
TIO_INT_TRAITS(int64_t)

struct ResampleArgs {
  const void* src;
  void* dst;
  const float* mat;      // [B][12]
  const float* cp;       // [B][ni][nj][nk][3] or null
  const uint8_t* flags;  // [B] or null
  const float* fill;     // [C] or null
  // TMA tile launches: batch element of each of the launch's B slots (device), or null = slot b
  // is element b.  A tiered call runs one launch per box edge, each over its own elements.
  const int* elems;
  int B, C, I, J, K, OI, OJ, OK;
  int ni, nj, nk;
  float sc_i, sc_j, sc_k;        // (n-1)/(O-1) upsample scales (fp32)
  float sp_in[3], sp_out[3];     // spacings
  float nm1[3];                  // max(size-1, 1) (normalise)
  float sm1[3];                  // size-1       (ATen un-normalise)
  int affine_first;
  int cp_in_smem;
};

constexpr int TK = 64;   // lanes along K
constexpr int TJ = 4;    // rows along J  -> 256 threads
constexpr int TI = 16;   // planes walked per CTA

// [p,1] @ M^T exactly as the reference's CPU sgemm rounds it: sequential FMA
// chain from the rounded first product (spatial.py:1621-1624).
__device__ __forceinline__ float affine_row(const float* m, float pi, float pj, float pk) {
  float acc = __fmul_rn(pi, m[0]);
  acc = __fmaf_rn(pj, m[1], acc);
  acc = __fmaf_rn(pk, m[2], acc);
  acc = __fmaf_rn(1.0f, m[3], acc);
  return acc;
}

// 2.0*q/nm1 - 1.0 (spatial.py:1646) then ATen's ((g+1)/2)*(size-1).
__device__ __forceinline__ float renormalise(float q, float nm1, float sm1) {
  float g = __fsub_rn(__fdiv_rn(__fmul_rn(2.0f, q), nm1), 1.0f);
  return __fmul_rn(__fmul_rn(__fadd_rn(g, 1.0f), 0.5f), sm1);
}


// label_interpolation="label" for one voxel (spatial.py:1275-1389, C == 1): the sampled value of a
// one-hot channel is the sum, in grid_sample's corner order, of the weights of the corners that
// carry its label (1 * w and + 0 * w are exact), so only the labels of the 8 taps matter.  Labels
// are visited in ascending order (torch.unique's channel order): the largest sum wins, the first
// on ties (argmax), and the sequential channel sum decides in-bounds (> 0.5) vs pad label.
// `active`: bit t set = corner t is inside the volume (out-of-bounds corners are skipped).
template <typename T>
__device__ __forceinline__ T label_pv_pick(const T tap[8], const float w[8], const unsigned active, const T pad) {
  if (active == 0u) return pad;
  // one label on every corner (the inside of a region, i.e. most voxels): its channel is the
  // ordered sum of the active weights, every other channel is exactly 0
  {
    T first = tap[7];
#pragma unroll
    for (int t = 6; t >= 0; --t)  // the lowest active corner (no dynamic register indexing)
      if ((active >> t) & 1u) first = tap[t];
    bool same = true;
    float s = 0.0f;
#pragma unroll
    for (int t = 0; t < 8; ++t)
      if ((active >> t) & 1u) { same = same && (tap[t] == first); s = __fadd_rn(s, w[t]); }
    if (same) return (s > 0.5f) ? first : pad;
  }
  unsigned todo = active;
  float total = 0.0f, best_s = -1.0f;
  T best = (T)0;
  while (todo) {
    T lab = (T)0;
    bool have = false;
#pragma unroll
    for (int t = 0; t < 8; ++t)
      if (((todo >> t) & 1u) && (!have || tap[t] < lab)) { lab = tap[t]; have = true; }
    float s = 0.0f;
#pragma unroll
    for (int t = 0; t < 8; ++t)
      if (((active >> t) & 1u) && tap[t] == lab) { s = __fadd_rn(s, w[t]); todo &= ~(1u << t); }
    total = __fadd_rn(total, s);  // sampled.sum(dim=1): ascending label order
    if (s > best_s) { best_s = s; best = lab; }
  }
  return (total > 0.5f) ? best : pad;
}

// The reference's fp32 input-voxel coordinates q = voxel_grid (spatial.py:1504-1579) of the output
// voxels of one (oj, ok) column, walked along I: the affine row of each axis, with the control-point
// displacement d = lerp_I(lerp_J(lerp_K(cp))) added before (affine_first) or after it.  The two
// inner lerp levels stay in registers across the walk and are recomputed only when the walk enters
// a new control-grid cell.  Shared by K1 and the B-spline pull, so both sample at the same points.
template <bool HAS_CP>
struct ColumnCoords {
  float m[12];
  LerpAxis lj, lk;
  int64_t o00 = 0, o01 = 0, o10 = 0, o11 = 0;  // (j0|j1, k0|k1) offsets in cp, x3
  int plane, cur_i0 = -1, cur_i1 = -1;
  float r_lo[3] = {0.f, 0.f, 0.f}, r_hi[3] = {0.f, 0.f, 0.f};
  float pj, pk;
  bool elastic;

  __device__ __forceinline__ ColumnCoords(const ResampleArgs& a, const int b, const bool elastic_,
                                          const int oj, const int ok)
      : plane(a.nj * a.nk * 3), pj((float)oj), pk((float)ok), elastic(elastic_) {
#pragma unroll
    for (int t = 0; t < 12; ++t) m[t] = a.mat[b * 12 + t];
    if (HAS_CP && elastic) {
      lj = lerp_axis(a.sc_j, a.nj, oj);
      lk = lerp_axis(a.sc_k, a.nk, ok);
      o00 = ((int64_t)lj.i0 * a.nk + lk.i0) * 3;
      o01 = ((int64_t)lj.i0 * a.nk + lk.i1) * 3;
      o10 = ((int64_t)lj.i1 * a.nk + lk.i0) * 3;
      o11 = ((int64_t)lj.i1 * a.nk + lk.i1) * 3;
    }
  }

  // q of output plane oi; `g` is the element's control grid (shared or global memory)
  __device__ __forceinline__ void at(const ResampleArgs& a, const float* g, const int oi, float q[3]) {
    const float pi = (float)oi;
    float d[3] = {0.f, 0.f, 0.f};
    if (HAS_CP && elastic) {
      LerpAxis li = lerp_axis(a.sc_i, a.ni, oi);  // warp-uniform
      if (li.i0 != cur_i0 || li.i1 != cur_i1) {
        const float* p0 = g + (int64_t)li.i0 * plane;
        const float* p1 = g + (int64_t)li.i1 * plane;
#pragma unroll
        for (int ax = 0; ax < 3; ++ax) {
          float a00 = lerp2(lk.l0, p0[o00 + ax], lk.l1, p0[o01 + ax]);
          float a01 = lerp2(lk.l0, p0[o10 + ax], lk.l1, p0[o11 + ax]);
          r_lo[ax] = lerp2(lj.l0, a00, lj.l1, a01);
          float b00 = lerp2(lk.l0, p1[o00 + ax], lk.l1, p1[o01 + ax]);
          float b01 = lerp2(lk.l0, p1[o10 + ax], lk.l1, p1[o11 + ax]);
          r_hi[ax] = lerp2(lj.l0, b00, lj.l1, b01);
        }
        cur_i0 = li.i0;
        cur_i1 = li.i1;
      }
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) d[ax] = lerp2(li.l0, r_lo[ax], li.l1, r_hi[ax]);
    }
    if (!(HAS_CP && elastic)) {
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) q[ax] = affine_row(m + 4 * ax, pi, pj, pk);
    } else if (a.affine_first) {  // spatial.py:1570-1573
#pragma unroll
      for (int ax = 0; ax < 3; ++ax)
        q[ax] = __fadd_rn(affine_row(m + 4 * ax, pi, pj, pk), __fdiv_rn(d[ax], a.sp_in[ax]));
    } else {  // spatial.py:1574-1577
      float e0 = __fadd_rn(pi, __fdiv_rn(d[0], a.sp_out[0]));
      float e1 = __fadd_rn(pj, __fdiv_rn(d[1], a.sp_out[1]));
      float e2 = __fadd_rn(pk, __fdiv_rn(d[2], a.sp_out[2]));
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) q[ax] = affine_row(m + 4 * ax, e0, e1, e2);
    }
  }
};

// General per-thread column: walks output planes [oi0, oi_end) at (oj, ok),
// gathering straight from global memory with exact ATen rounding everywhere
// (bit-exact with oracle/c/tio_oracle.c for every dtype and mode).
template <typename T, int MODE, bool HAS_CP, bool HAS_FILL>
__device__ __forceinline__ void general_column(const ResampleArgs& a, const int b, const bool elastic,
                                               const float* g, const T* __restrict__ src,
                                               T* __restrict__ dst, const int64_t n_in,
                                               const int64_t n_out, const int oi0,
                                               const int oi_end, const int oj, const int ok) {
  ColumnCoords<HAS_CP> coords(a, b, elastic, oj, ok);
  for (int oi = oi0; oi < oi_end; ++oi) {
    float q[3];
    coords.at(a, g, oi, q);
    float u[3];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) u[ax] = renormalise(q[ax], a.nm1[ax], a.sm1[ax]);

    // trilinear corner weights: needed for MODE==linear and for the mask
    float f0 = floorf(u[0]), f1 = floorf(u[1]), f2 = floorf(u[2]);
    // clamp before the int conversion so wild coordinates stay out of bounds
    int c0 = (int)fminf(fmaxf(f0, -2.0f), (float)a.I);
    int c1 = (int)fminf(fmaxf(f1, -2.0f), (float)a.J);
    int c2 = (int)fminf(fmaxf(f2, -2.0f), (float)a.K);
    const bool interior = (c0 >= 0) & (c0 + 1 < a.I) & (c1 >= 0) & (c1 + 1 < a.J) &
                          (c2 >= 0) & (c2 + 1 < a.K);

    float w[8];
    bool inb[8];
    bool need_w = (MODE != TIO_NEAREST) || (HAS_FILL && !interior);
    if (need_w) {
      // ATen: weight_lo = (c+1) - u, weight_hi = u - c  (exact ints as floats)
      float lo0 = __fsub_rn(__fadd_rn(f0, 1.0f), u[0]), hi0 = __fsub_rn(u[0], f0);
      float lo1 = __fsub_rn(__fadd_rn(f1, 1.0f), u[1]), hi1 = __fsub_rn(u[1], f1);
      float lo2 = __fsub_rn(__fadd_rn(f2, 1.0f), u[2]), hi2 = __fsub_rn(u[2], f2);
      float w00 = __fmul_rn(lo0, lo1), w10 = __fmul_rn(hi0, lo1);
      float w01 = __fmul_rn(lo0, hi1), w11 = __fmul_rn(hi0, hi1);
      // order: i fastest, then j, then k  (tnw, tne, tsw, tse, bnw, ...)
      w[0] = __fmul_rn(w00, lo2); w[1] = __fmul_rn(w10, lo2);
      w[2] = __fmul_rn(w01, lo2); w[3] = __fmul_rn(w11, lo2);
      w[4] = __fmul_rn(w00, hi2); w[5] = __fmul_rn(w10, hi2);
      w[6] = __fmul_rn(w01, hi2); w[7] = __fmul_rn(w11, hi2);
    }
    if (!interior) {
      const bool i_lo = (c0 >= 0) & (c0 < a.I), i_hi = (c0 + 1 >= 0) & (c0 + 1 < a.I);
      const bool j_lo = (c1 >= 0) & (c1 < a.J), j_hi = (c1 + 1 >= 0) & (c1 + 1 < a.J);
      const bool k_lo = (c2 >= 0) & (c2 < a.K), k_hi = (c2 + 1 >= 0) & (c2 + 1 < a.K);
      inb[0] = i_lo & j_lo & k_lo; inb[1] = i_hi & j_lo & k_lo;
      inb[2] = i_lo & j_hi & k_lo; inb[3] = i_hi & j_hi & k_lo;
      inb[4] = i_lo & j_lo & k_hi; inb[5] = i_hi & j_lo & k_hi;
      inb[6] = i_lo & j_hi & k_hi; inb[7] = i_hi & j_hi & k_hi;
    }
    bool use_fill = false;
    if (MODE != TIO_LABEL_PV && HAS_FILL && !interior) {
      float msum = 0.0f;
#pragma unroll
      for (int t = 0; t < 8; ++t)
        if (inb[t]) msum = __fadd_rn(msum, w[t]);
      use_fill = !(msum > 0.5f);
    }

    const int64_t o_off = ((int64_t)oi * a.OJ + oj) * a.OK + ok;
    if (MODE == TIO_NEAREST) {
      // round-half-to-even like std::nearbyint; clamp keeps the cvt in range
      int r0 = __float2int_rn(fminf(fmaxf(u[0], -2.0f), (float)a.I + 1.0f));
      int r1 = __float2int_rn(fminf(fmaxf(u[1], -2.0f), (float)a.J + 1.0f));
      int r2 = __float2int_rn(fminf(fmaxf(u[2], -2.0f), (float)a.K + 1.0f));
      const bool ok_in = (r0 >= 0) & (r0 < a.I) & (r1 >= 0) & (r1 < a.J) & (r2 >= 0) & (r2 < a.K);
      const int64_t off = ((int64_t)r0 * a.J + r1) * a.K + r2;
      for (int c = 0; c < a.C; ++c) {
        T v;
        if (HAS_FILL && use_fill) v = ElemTraits<T>::from_f32(a.fill[c]);
        else v = ok_in ? __ldg(src + c * n_in + off) : (T)0;
        dst[c * n_out + o_off] = v;
      }
    } else if (MODE == TIO_LABEL_PV) {
      // partial-volume label resampling: see label_pv_pick
      const int64_t base = ((int64_t)c0 * a.J + c1) * a.K + c2;
      const int64_t sI = (int64_t)a.J * a.K, sJ = a.K;
      T tap[8];
      unsigned todo = 0;
#pragma unroll
      for (int t = 0; t < 8; ++t) {
        const bool act = interior || inb[t];
        tap[t] = act ? __ldg(src + base + (t & 1) * sI + ((t >> 1) & 1) * sJ + ((t >> 2) & 1)) : (T)0;
        todo |= act ? (1u << t) : 0u;
      }
      dst[o_off] = label_pv_pick<T>(tap, w, todo, ElemTraits<T>::from_f32(a.fill[0]));
    } else {
      const int64_t base = ((int64_t)c0 * a.J + c1) * a.K + c2;
      const int64_t sI = (int64_t)a.J * a.K, sJ = a.K;
      for (int c = 0; c < a.C; ++c) {
        const T* s = src + c * n_in;
        float v = 0.0f;
        if (HAS_FILL && use_fill) {
          v = a.fill[c];
        } else if (interior) {
          const T* p = s + base;
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p)), w[0]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + sI)), w[1]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + sJ)), w[2]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + sI + sJ)), w[3]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + 1)), w[4]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + sI + 1)), w[5]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + sJ + 1)), w[6]));
          v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(p + sI + sJ + 1)), w[7]));
        } else {
#pragma unroll
          for (int t = 0; t < 8; ++t)
            if (inb[t]) {
              int64_t off = base + (t & 1) * sI + ((t >> 1) & 1) * sJ + ((t >> 2) & 1);
              v = __fadd_rn(v, __fmul_rn(ElemTraits<T>::to_f32(__ldg(s + off)), w[t]));
            }
        }
        dst[c * n_out + o_off] = ElemTraits<T>::from_f32(v);
      }
    }
  }
}

}  // namespace tio

// resample_tile.cuh — pieces shared by the two K1 tile kernels (resample_tile.cu: exact
// coordinate chain, label maps; resample_fast.cu: relaxed one-fma coordinates for fp32 images):
// tile geometry, the per-tile bounds pre-pass, shared-memory loads, two-lane fp32 arithmetic.
#pragma once
#include <cuda.h>

#include "resample_common.cuh"
#include "tma.cuh"

namespace tio {

constexpr int XT = 16;  // output tile edge
constexpr int kSmallBox = 18;  // second, smaller box of elastic fast-kernel launches
// inner (K) extent of the staged box in elements: BOX plus room for rounding the origin down
// to a 16-byte boundary, itself rounded up so that a box row is a multiple of 16 bytes
// (cuTensorMapEncodeTiled rejects other inner extents: BOX = 22 fp32 needs 28, not 26)
__host__ __device__ constexpr int box_k_extent(int box, int elem_bytes) {
  return (box + 16 / elem_bytes + 16 / elem_bytes - 1) / (16 / elem_bytes) * (16 / elem_bytes);
}
constexpr float kMagic = 12582912.0f;  // 1.5 * 2^23: floor() via round-down add
constexpr int kMagicBits = 0x4B400000;

struct TileArgs {
  float hd[3];   // max(size-1,1)/2      (divisor of the normalise step, exact)
  float rcp[3];  // rn(1/hd)
  float hs[3];   // (size-1)/2           (ATen un-normalise multiplier, exact)
  int sp_in_one, sp_out_one;
  float rsp_in[3], rsp_out[3];  // 1 / spacing (fast kernel: the division folds into column constants)
  unsigned magic_bytes;         // kMagicBits << 2 (mod 2^32), see resample_fast.cu
  // launch-invariant index arithmetic, done once on the host
  long long n_in, n_out;      // voxels per input / output channel
  int tiles_i;                // output tiles along I
  unsigned inv_tiles_i;       // floor(2^32 / tiles_i) + 1: z / tiles_i == umulhi(z, inv) for z < 2^16
};

template <int OFFSET>
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(addr), "n"(OFFSET));
  return v;
}

// nearest mode: one tap of the staged box, moved bit for bit
template <typename T>
__device__ __forceinline__ T lds_elem(uint32_t addr) {
  if (sizeof(T) == 1) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return (T)v;
  } else if (sizeof(T) == 2) {
    uint16_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
    return (T)v;
  } else {
    uint32_t v;
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
    T out;
    memcpy(&out, &v, sizeof(T) < 4 ? sizeof(T) : 4);
    return out;
  }
}

template <bool FASTDIV>
__device__ __forceinline__ float norm_div(float x, float hd, float rcp) {
  if (FASTDIV) {
    const float q0 = __fmul_rn(x, rcp);
    const float e = __fmaf_rn(-q0, hd, x);
    return __fmaf_rn(e, rcp, q0);
  }
  return __fdiv_rn(x, hd);
}

// trilinear displacement (3 components) at one output position, exact ATen order
__device__ __forceinline__ void disp_at(const float* g, const ResampleArgs& a, int oi, int oj,
                                        int ok, float d[3]) {
  const LerpAxis li = lerp_axis(a.sc_i, a.ni, oi);
  const LerpAxis lj = lerp_axis(a.sc_j, a.nj, oj);
  const LerpAxis lk = lerp_axis(a.sc_k, a.nk, ok);
  const int plane = a.nj * a.nk * 3;
  const float* p0 = g + li.i0 * plane;
  const float* p1 = g + li.i1 * plane;
  const int o00 = (lj.i0 * a.nk + lk.i0) * 3, o01 = (lj.i0 * a.nk + lk.i1) * 3;
  const int o10 = (lj.i1 * a.nk + lk.i0) * 3, o11 = (lj.i1 * a.nk + lk.i1) * 3;
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    float a00 = lerp2(lk.l0, p0[o00 + ax], lk.l1, p0[o01 + ax]);
    float a01 = lerp2(lk.l0, p0[o10 + ax], lk.l1, p0[o11 + ax]);
    float b00 = lerp2(lk.l0, p1[o00 + ax], lk.l1, p1[o01 + ax]);
    float b01 = lerp2(lk.l0, p1[o10 + ax], lk.l1, p1[o11 + ax]);
    d[ax] = lerp2(li.l0, lerp2(lj.l0, a00, lj.l1, a01), li.l1, lerp2(lj.l0, b00, lj.l1, b01));
  }
}

// Sample positions along one axis where a piecewise-linear (in `scale*o`)
// function over integers o in [lo, hi] can attain its extrema: both ends and
// the integers adjacent to every breakpoint.  Returns count (<= 8) or -1
// (pts must hold 12 entries).
__device__ __forceinline__ int axis_points(float scale, int lo, int hi, int* pts) {
  int n = 0;
  pts[n++] = lo;
  if (hi > lo) {
    const float rlo = scale * (float)lo, rhi = scale * (float)hi;
    const int c_first = (int)floorf(rlo) + 1, c_last = (int)ceilf(rhi) - 1;
    for (int c = c_first; c <= c_last; ++c) {
      if (n > 6) return -1;
      const int o = (int)floorf((float)c / scale);
      for (int t = o - 1; t <= o + 1; ++t)  // +-1 guards the fp32 division above
        if (t > lo && t < hi && t > pts[n - 1]) pts[n++] = t;
    }
    pts[n++] = hi;
    if (n > 8) return -1;
  }
  return n;
}

// ---------------------------------------------------------------------------
// pre-pass: one warp per output tile bounds the tile's pre-image and records
// (box origin, fit code) so the main kernel can issue its TMA load at once.
//   code 0: does not fit the box -> general path     code 1: fits
//   code 2: pre-image entirely outside the volume    code 3: pass-through element
//   bit 8: every tap in bounds   bit 9: identity matrix   bit 10: elastic element
//   bit 11: the output tile is a full 16^3 (no ragged edge)
//   bit 12: the pre-image also fits the small box (box_s x box_s x bk_s) of the fast kernel
// ---------------------------------------------------------------------------
template <bool HAS_CP>
__global__ void __launch_bounds__(128)
tile_bounds_kernel(const ResampleArgs a, const int box, const int kalign, const int bk, const int box_s,
                   const int bk_s, int4* __restrict__ records) {
  // ONE THREAD per tile: the work of a tile is a short serial chain (index arithmetic, a dozen
  // table loads, interval arithmetic); a warp per tile left 31 lanes idle and made the pass
  // latency-bound (many waves of one-lane warps per SM).
  const int tiles_i = (a.OI + XT - 1) / XT, tiles_j = (a.OJ + XT - 1) / XT, tiles_k = (a.OK + XT - 1) / XT;
  const int64_t n_tiles = (int64_t)a.B * tiles_i * tiles_j * tiles_k;
  const int64_t tile = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tile >= n_tiles) return;
  const unsigned per_b = (unsigned)(tiles_i * tiles_j * tiles_k);
  const int slot = (int)(tile / per_b);
  const int b = a.elems ? a.elems[slot] : slot;
  unsigned rest = (unsigned)(tile - (int64_t)slot * per_b);
  const int tk = (int)(rest % (unsigned)tiles_k);
  rest /= (unsigned)tiles_k;
  const int tj = (int)(rest % (unsigned)tiles_j), ti = (int)(rest / (unsigned)tiles_j);
  const int i0 = ti * XT, j0 = tj * XT, k0 = tk * XT;
  const int i1 = min(i0 + XT, a.OI) - 1, j1 = min(j0 + XT, a.OJ) - 1, k1 = min(k0 + XT, a.OK) - 1;
  const uint8_t fl = a.flags ? a.flags[b] : 0;
  if (fl & TIO_FLAG_PASSTHROUGH) {
    records[tile] = make_int4(0, 0, 0, 3);
    return;
  }
  const bool elastic = HAS_CP && (fl & TIO_FLAG_ELASTIC);
  float dmn[3] = {0.f, 0.f, 0.f}, dmx[3] = {0.f, 0.f, 0.f};
  bool ok_bounds = true;
  if (elastic) {
    const float* g = a.cp + (int64_t)b * a.ni * a.nj * a.nk * 3;
    int pi[12], pj[12], pk[12];
    const int ni_ = axis_points(a.sc_i, i0, i1, pi);
    const int nj_ = axis_points(a.sc_j, j0, j1, pj);
    const int nk_ = axis_points(a.sc_k, k0, k1, pk);
    if (ni_ < 0 || nj_ < 0 || nk_ < 0) {
      ok_bounds = false;
    } else {
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) { dmn[ax] = 3.0e38f; dmx[ax] = -3.0e38f; }
      for (int qi = 0; qi < ni_; ++qi)
        for (int qj = 0; qj < nj_; ++qj)
          for (int qk = 0; qk < nk_; ++qk) {
            float d[3];
            disp_at(g, a, pi[qi], pj[qj], pk[qk], d);
#pragma unroll
            for (int ax = 0; ax < 3; ++ax) { dmn[ax] = fminf(dmn[ax], d[ax]); dmx[ax] = fmaxf(dmx[ax], d[ax]); }
          }
    }
  }
  const float* m = a.mat + b * 12;
  const int dims[3] = {a.I, a.J, a.K};
  const float plo[3] = {(float)i0, (float)j0, (float)k0};
  const float phi[3] = {(float)i1, (float)j1, (float)k1};
  float elo[3], ehi[3], add_lo[3] = {0.f, 0.f, 0.f}, add_hi[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) { elo[ax] = plo[ax]; ehi[ax] = phi[ax]; }
  if (elastic) {
    if (a.affine_first) {
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) { add_lo[ax] = dmn[ax] / a.sp_in[ax]; add_hi[ax] = dmx[ax] / a.sp_in[ax]; }
    } else {
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) { elo[ax] += dmn[ax] / a.sp_out[ax]; ehi[ax] += dmx[ax] / a.sp_out[ax]; }
    }
  }
  bool fits = ok_bounds, interior = true, outside = false;
  bool fits_small = ok_bounds && box_s > 0;  // also fits the small box of the fast kernel (bit 12)
  int ilo[3];
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    float qlo = m[4 * ax + 3], qhi = m[4 * ax + 3];
#pragma unroll
    for (int bx = 0; bx < 3; ++bx) {
      const float v0 = m[4 * ax + bx] * elo[bx], v1 = m[4 * ax + bx] * ehi[bx];
      qlo += fminf(v0, v1);
      qhi += fmaxf(v0, v1);
    }
    qlo += add_lo[ax];
    qhi += add_hi[ax];
    const float margin = 0.02f + 1e-5f * fmaxf(fabsf(qlo), fabsf(qhi));
    qlo -= margin;
    qhi += margin;
    if (dims[ax] == 1) { qlo = 0.0f; qhi = 0.0f; }  // (size-1) == 0 collapses the axis
    if (!(fabsf(qlo) < 1.0e6f && fabsf(qhi) < 1.0e6f)) { fits = false; qlo = 0.f; qhi = 0.f; }
    int lo = (int)floorf(qlo), hi = (int)floorf(qhi) + 1;
    // every corner (floor(u), floor(u)+1) out of bounds on this axis => all padding
    if (hi < 0 || lo > dims[ax] - 1) outside = true;
    if (ax == 2) lo &= ~(kalign - 1);  // TMA: innermost coordinate must be 16-byte aligned
    if (hi - lo + 1 > (ax == 2 ? bk : box)) fits = false;
    if (hi - lo + 1 > (ax == 2 ? bk_s : box_s)) fits_small = false;
    if (lo < 0 || hi > dims[ax] - 1) interior = false;
    ilo[ax] = lo;
  }
  const int code = (ok_bounds && outside) ? 2 : (fits ? 1 : 0);
  const bool ident = m[0] == 1.f && m[1] == 0.f && m[2] == 0.f && m[3] == 0.f && m[4] == 0.f &&
                     m[5] == 1.f && m[6] == 0.f && m[7] == 0.f && m[8] == 0.f && m[9] == 0.f &&
                     m[10] == 1.f && m[11] == 0.f;  // [p,1] @ I^T == p exactly
  const bool full = (i0 + XT <= a.OI) && (j0 + XT <= a.OJ) && (k0 + XT <= a.OK);
  records[tile] = make_int4(ilo[0], ilo[1], ilo[2], code | (interior ? 256 : 0) | (ident ? 512 : 0) |
                                                        (elastic ? 1024 : 0) | (full ? 2048 : 0) |
                                                        ((fits && fits_small) ? 4096 : 0));
}

struct LiEntry {  // per output plane of the tile: I-axis lerp of the control grid
  int off0, off1;  // i0 * plane, i1 * plane (floats)
  float l0, l1;
};
struct __align__(16) LiPair {  // planes (2p, 2p+1) of the tile, weights laid out as two-lane operands
  int off0, off1;    // of plane 2p
  float l0a, l0b;    // l0 of plane 2p, 2p+1
  float l1a, l1b;
  int same_cell;     // both planes lerp between the same two control planes
  int pad;
};

// ---- two-lane fp32 arithmetic ----------------------------------------------------
// Two output planes are walked at once, lane by lane.  sm_90 has no packed fp32x2
// instructions, so each lane is one scalar instruction with an explicit rounding mode
// (the __f*_rn intrinsics are never contracted), rounded exactly like the one-plane path.
struct f2 {
  float lo, hi;
};
__device__ __forceinline__ f2 pack2(float lo, float hi) { return f2{lo, hi}; }
__device__ __forceinline__ f2 bc(float x) { return f2{x, x}; }
__device__ __forceinline__ void unpack2(f2 v, float& lo, float& hi) {
  lo = v.lo;
  hi = v.hi;
}
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) {
  return f2{__fmaf_rn(a.lo, b.lo, c.lo), __fmaf_rn(a.hi, b.hi, c.hi)};
}
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return f2{__fadd_rn(a.lo, b.lo), __fadd_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 sub2(f2 a, f2 b) { return f2{__fsub_rn(a.lo, b.lo), __fsub_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.lo, b.lo), __fmul_rn(a.hi, b.hi)}; }
__device__ __forceinline__ f2 add2_rd(f2 a, f2 b) { return f2{__fadd_rd(a.lo, b.lo), __fadd_rd(a.hi, b.hi)}; }
// affine_row (resample_common.cuh) on two positions at once
__device__ __forceinline__ f2 affine_row2(const float* m, f2 pi, f2 pj, f2 pk) {
  f2 acc = mul2(pi, bc(m[0]));
  acc = fma2(pj, bc(m[1]), acc);
  acc = fma2(pk, bc(m[2]), acc);
  return add2(acc, bc(m[3]));  // fma(1, m3, acc) == rn(m3 + acc)
}
template <bool FASTDIV>
__device__ __forceinline__ f2 norm_div2(f2 x, float hd, float rcp) {
  if (FASTDIV) {
    const f2 q0 = mul2(x, bc(rcp));
    const f2 e = fma2(q0, bc(-hd), x);  // fma(-q0, hd, x): the sign moves to the exact operand
    return fma2(e, bc(rcp), q0);
  }
  float lo, hi;
  unpack2(x, lo, hi);
  return pack2(__fdiv_rn(lo, hd), __fdiv_rn(hi, hd));
}


constexpr int kAuxFloats = 160;  // li table 64 | pair table 64 | mbarrier 2 | kbase 1 | pad 1 | fast kernel 28

}  // namespace tio

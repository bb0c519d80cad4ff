// resample_tile.cu — K1 fast path: fp32, trilinear, TMA-staged input tiles.
//
// One CTA produces a 16 x 16 x 16 output tile.  Warp 0 bounds the tile's
// pre-image in input voxel space (affine corners by interval arithmetic,
// elastic displacement by evaluating the piecewise-trilinear field at the
// tile corners and control-cell crossings, where its extrema lie), and one
// thread issues a single 4-D TMA box load (cp.async.bulk.tensor, zero fill
// outside the volume = grid_sample's padding_mode="zeros").  The innermost box
// coordinate must be a multiple of 16 bytes (probed: other values raise an
// illegal-instruction fault), so the K origin is rounded down to a multiple
// of 4 voxels and the box is BOX x BOX x (BOX+4).  256 threads then
// walk the 16 planes of their (j,k) column reading the 8 taps from shared
// memory.  Tiles whose pre-image does not fit the box fall back to the
// general global-memory column (same results).
//
// Coordinates reproduce the reference's CPU rounding sequence exactly
// (oracle/c/tio_oracle.c); the divide by (size-1)/2 uses the reciprocal +
// two-FMA correction, admitted per divisor only after an exhaustive on-device
// check against __fdiv_rn over every float (see verify_fastdiv).  Tap blending
// uses FMA lerps (<= 1 ulp from the reference's mul+add chain).
#include <cuda.h>

#include <map>
#include <mutex>

#include "resample_tile.cuh"

namespace tio {

// The 16-plane walk of one (j,k) column over the staged box, two planes per step.
// CHECK = the tile touches the volume border and a fill value is set: per-voxel ATen mask.
// EMODE (CTA-uniform, resolved outside the loop):
//   0 no displacement            1 q = p + d (identity matrix, unit spacing)
//   2 q = M p + d (unit spacing) 3 q = M (p + d) (unit spacing)
//   4 displacement with non-unit spacing: plane-at-a-time path only
//   T/MODE: float + TIO_LINEAR (8 taps, separable lerp) or a label type + TIO_NEAREST
//   (round-half-even via a round-to-nearest magic add, one tap moved bit for bit;
//   CHECK is not used with nearest: border tiles with a fill take the general column)
template <int BOX, typename T, int MODE, bool HAS_CP, bool CHECK, bool FASTDIV, int EMODE>
__device__ __forceinline__ void walk_column(
    const ResampleArgs& a, const TileArgs& ta, const T* __restrict__ box,
    const float* __restrict__ cps, const LiEntry* __restrict__ li_tab,
    const LiPair* __restrict__ li_pairs, const float m[12],
    const bool elastic, const bool identity, const uint32_t kbase, const int i0, const int i1,
    const int oj, const int ok, const float fill_c, T* __restrict__ out, const int64_t ostride) {
  constexpr int BK = box_k_extent(BOX, (int)sizeof(T));
  constexpr int C1 = BOX * BK, C2 = BK;
  constexpr int ESH = sizeof(T) == 1 ? 0 : (sizeof(T) == 2 ? 1 : 2);
  const float hd0 = ta.hd[0], hd1 = ta.hd[1], hd2 = ta.hd[2];
  const float rc0 = ta.rcp[0], rc1 = ta.rcp[1], rc2 = ta.rcp[2];
  const float hs0 = ta.hs[0], hs1 = ta.hs[1], hs2 = ta.hs[2];
  const float pj = (float)oj, pk = (float)ok;
  // J/K levels of the nested displacement lerp, cached across the walk
  LerpAxis lj, lk;
  int o00 = 0, o01 = 0, o10 = 0, o11 = 0;
  if (HAS_CP && elastic) {
    lj = lerp_axis(a.sc_j, a.nj, oj);
    lk = lerp_axis(a.sc_k, a.nk, ok);
    o00 = (lj.i0 * a.nk + lk.i0) * 3; o01 = (lj.i0 * a.nk + lk.i1) * 3;
    o10 = (lj.i1 * a.nk + lk.i0) * 3; o11 = (lj.i1 * a.nk + lk.i1) * 3;
  }
  int cur0 = -1, cur1 = -1;
  float r_lo[3] = {0.f, 0.f, 0.f}, r_hi[3] = {0.f, 0.f, 0.f};

  auto refresh = [&](const LiEntry& li) {  // J/K-collapsed control values of the I-cell pair
    if (li.off0 != cur0 || li.off1 != cur1) {
      // control points straight from global memory: a tile touches at most 2x2 (j,k)
      // cells, so these are a few L1-resident sectors per warp, once or twice per walk
      const float* p0 = cps + li.off0;
      const float* p1 = cps + li.off1;
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) {
        float a00 = lerp2(lk.l0, __ldg(p0 + o00 + ax), lk.l1, __ldg(p0 + o01 + ax));
        float a01 = lerp2(lk.l0, __ldg(p0 + o10 + ax), lk.l1, __ldg(p0 + o11 + ax));
        r_lo[ax] = lerp2(lj.l0, a00, lj.l1, a01);
        float b00 = lerp2(lk.l0, __ldg(p1 + o00 + ax), lk.l1, __ldg(p1 + o01 + ax));
        float b01 = lerp2(lk.l0, __ldg(p1 + o10 + ax), lk.l1, __ldg(p1 + o11 + ax));
        r_hi[ax] = lerp2(lj.l0, b00, lj.l1, b01);
      }
      cur0 = li.off0; cur1 = li.off1;
    }
  };
  // exact ATen mask for a voxel with out-of-bounds corners: ordered sum of the in-bounds weights
  auto needs_fill = [&](int c0, int c1, int c2, float u0, float u1, float u2, float f0, float f1,
                        float f2_, float hi0, float hi1, float hi2) -> bool {
    const float lo0 = __fsub_rn(__fadd_rn(f0, 1.0f), u0), lo1 = __fsub_rn(__fadd_rn(f1, 1.0f), u1),
                lo2 = __fsub_rn(__fadd_rn(f2_, 1.0f), u2);
    const float w00 = __fmul_rn(lo0, lo1), w10 = __fmul_rn(hi0, lo1);
    const float w01 = __fmul_rn(lo0, hi1), w11 = __fmul_rn(hi0, hi1);
    const bool il = (unsigned)c0 < (unsigned)a.I, ih = (unsigned)(c0 + 1) < (unsigned)a.I;
    const bool jl = (unsigned)c1 < (unsigned)a.J, jh = (unsigned)(c1 + 1) < (unsigned)a.J;
    const bool kl = (unsigned)c2 < (unsigned)a.K, kh = (unsigned)(c2 + 1) < (unsigned)a.K;
    float msum = 0.0f;
    if (il & jl & kl) msum = __fadd_rn(msum, __fmul_rn(w00, lo2));
    if (ih & jl & kl) msum = __fadd_rn(msum, __fmul_rn(w10, lo2));
    if (il & jh & kl) msum = __fadd_rn(msum, __fmul_rn(w01, lo2));
    if (ih & jh & kl) msum = __fadd_rn(msum, __fmul_rn(w11, lo2));
    if (il & jl & kh) msum = __fadd_rn(msum, __fmul_rn(w00, hi2));
    if (ih & jl & kh) msum = __fadd_rn(msum, __fmul_rn(w10, hi2));
    if (il & jh & kh) msum = __fadd_rn(msum, __fmul_rn(w01, hi2));
    if (ih & jh & kh) msum = __fadd_rn(msum, __fmul_rn(w11, hi2));
    return !(msum > 0.5f);
  };
  auto interior = [&](int c0, int c1, int c2) -> bool {
    return ((unsigned)c0 < (unsigned)(a.I - 1)) & ((unsigned)c1 < (unsigned)(a.J - 1)) &
           ((unsigned)c2 < (unsigned)(a.K - 1));
  };

  // partial-volume label value at exact coordinates (u0, u1, u2): the weights in the reference's
  // order, the 8 label taps from the box, corners outside the volume skipped (CHECK tiles)
  auto label_pv = [&](const float u0, const float u1, const float u2) -> T {
    const float s0 = __fadd_rd(u0, kMagic), s1 = __fadd_rd(u1, kMagic), s2 = __fadd_rd(u2, kMagic);
    const float f0 = __fsub_rn(s0, kMagic), f1 = __fsub_rn(s1, kMagic), f2_ = __fsub_rn(s2, kMagic);
    const float hi0 = __fsub_rn(u0, f0), hi1 = __fsub_rn(u1, f1), hi2 = __fsub_rn(u2, f2_);
    const float lo0 = __fsub_rn(__fadd_rn(f0, 1.0f), u0), lo1 = __fsub_rn(__fadd_rn(f1, 1.0f), u1),
                lo2 = __fsub_rn(__fadd_rn(f2_, 1.0f), u2);
    const float w00 = __fmul_rn(lo0, lo1), w10 = __fmul_rn(hi0, lo1);
    const float w01 = __fmul_rn(lo0, hi1), w11 = __fmul_rn(hi0, hi1);
    float w[8];
    w[0] = __fmul_rn(w00, lo2); w[1] = __fmul_rn(w10, lo2); w[2] = __fmul_rn(w01, lo2); w[3] = __fmul_rn(w11, lo2);
    w[4] = __fmul_rn(w00, hi2); w[5] = __fmul_rn(w10, hi2); w[6] = __fmul_rn(w01, hi2); w[7] = __fmul_rn(w11, hi2);
    const int b0 = __float_as_int(s0), b1 = __float_as_int(s1), b2 = __float_as_int(s2);
    const uint32_t addr = kbase + (((unsigned)b0 * C1 + (unsigned)b1 * C2 + (unsigned)b2) << ESH);
    unsigned active = 0xffu;
    if (CHECK) {
      const int c0 = b0 - kMagicBits, c1 = b1 - kMagicBits, c2 = b2 - kMagicBits;
      if (!interior(c0, c1, c2)) {
        const bool il = (unsigned)c0 < (unsigned)a.I, ih = (unsigned)(c0 + 1) < (unsigned)a.I;
        const bool jl = (unsigned)c1 < (unsigned)a.J, jh = (unsigned)(c1 + 1) < (unsigned)a.J;
        const bool kl = (unsigned)c2 < (unsigned)a.K, kh = (unsigned)(c2 + 1) < (unsigned)a.K;
        active = (il & jl & kl ? 1u : 0u) | (ih & jl & kl ? 2u : 0u) | (il & jh & kl ? 4u : 0u) |
                 (ih & jh & kl ? 8u : 0u) | (il & jl & kh ? 16u : 0u) | (ih & jl & kh ? 32u : 0u) |
                 (il & jh & kh ? 64u : 0u) | (ih & jh & kh ? 128u : 0u);
      }
    }
    T tap[8];
#pragma unroll
    for (int t = 0; t < 8; ++t)  // corner t: +1 in I (bit 0), J (bit 1), K (bit 2)
      tap[t] = lds_elem<T>(addr + ((unsigned)((t & 1) * C1 + ((t >> 1) & 1) * C2 + ((t >> 2) & 1)) << ESH));
    return label_pv_pick<T>(tap, w, active, ElemTraits<T>::from_f32(fill_c));
  };

  // ---- one plane (odd tail, cell changes inside a pair, non-unit spacing) ----
  // (`rel` = plane index within the walk, `pi` = its output coordinate as a float: the loop
  // carries both so that nothing has to be re-derived from blockIdx inside it)
  auto one = [&](const int rel, const float pi, T* __restrict__ dst) {
    float q0, q1, q2;
    if (HAS_CP && elastic) {
      const LiEntry li = li_tab[rel];  // warp-uniform broadcast
      refresh(li);
      float d0 = lerp2(li.l0, r_lo[0], li.l1, r_hi[0]);
      float d1 = lerp2(li.l0, r_lo[1], li.l1, r_hi[1]);
      float d2 = lerp2(li.l0, r_lo[2], li.l1, r_hi[2]);
      if (a.affine_first) {
        if (!ta.sp_in_one) { d0 = __fdiv_rn(d0, a.sp_in[0]); d1 = __fdiv_rn(d1, a.sp_in[1]); d2 = __fdiv_rn(d2, a.sp_in[2]); }
        if (identity) {  // [p,1] @ I^T == p exactly
          q0 = __fadd_rn(pi, d0); q1 = __fadd_rn(pj, d1); q2 = __fadd_rn(pk, d2);
        } else {
          q0 = __fadd_rn(affine_row(m + 0, pi, pj, pk), d0);
          q1 = __fadd_rn(affine_row(m + 4, pi, pj, pk), d1);
          q2 = __fadd_rn(affine_row(m + 8, pi, pj, pk), d2);
        }
      } else {
        if (!ta.sp_out_one) { d0 = __fdiv_rn(d0, a.sp_out[0]); d1 = __fdiv_rn(d1, a.sp_out[1]); d2 = __fdiv_rn(d2, a.sp_out[2]); }
        const float e0 = __fadd_rn(pi, d0), e1 = __fadd_rn(pj, d1), e2 = __fadd_rn(pk, d2);
        q0 = affine_row(m + 0, e0, e1, e2);
        q1 = affine_row(m + 4, e0, e1, e2);
        q2 = affine_row(m + 8, e0, e1, e2);
      }
    } else {
      q0 = affine_row(m + 0, pi, pj, pk);
      q1 = affine_row(m + 4, pi, pj, pk);
      q2 = affine_row(m + 8, pi, pj, pk);
    }
    // 2q/nm1 - 1  ->  ((g+1)/2)*(size-1), as rn(q/hd), -1, +1, *hs (exact rescalings)
    const float u0 = __fmul_rn(__fadd_rn(__fsub_rn(norm_div<FASTDIV>(q0, hd0, rc0), 1.0f), 1.0f), hs0);
    const float u1 = __fmul_rn(__fadd_rn(__fsub_rn(norm_div<FASTDIV>(q1, hd1, rc1), 1.0f), 1.0f), hs1);
    const float u2 = __fmul_rn(__fadd_rn(__fsub_rn(norm_div<FASTDIV>(q2, hd2, rc2), 1.0f), 1.0f), hs2);
    if (MODE == TIO_NEAREST) {
      // nearbyint(u) via round-to-nearest-even magic add; taps outside the volume are the
      // zero halo of the box (grid_sample padding_mode="zeros")
      const int r0 = __float_as_int(__fadd_rn(u0, kMagic)), r1 = __float_as_int(__fadd_rn(u1, kMagic)),
                r2 = __float_as_int(__fadd_rn(u2, kMagic));
      *dst = lds_elem<T>(kbase + (((unsigned)r0 * C1 + (unsigned)r1 * C2 + (unsigned)r2) << ESH));
      return;
    }
    if (MODE == TIO_LABEL_PV) {
      *dst = label_pv(u0, u1, u2);
      return;
    }
    // floor via round-down magic add: the mantissa holds floor(u)
    const float s0 = __fadd_rd(u0, kMagic), s1 = __fadd_rd(u1, kMagic), s2 = __fadd_rd(u2, kMagic);
    const float f0 = __fsub_rn(s0, kMagic), f1 = __fsub_rn(s1, kMagic), f2_ = __fsub_rn(s2, kMagic);
    const float hi0 = __fsub_rn(u0, f0), hi1 = __fsub_rn(u1, f1), hi2 = __fsub_rn(u2, f2_);
    const int b0 = __float_as_int(s0), b1 = __float_as_int(s1), b2 = __float_as_int(s2);
    // byte address of tap (floor i, floor j, floor k): one base register, the other
    // seven taps are compile-time immediates off it
    const uint32_t addr = kbase + (((unsigned)b0 * C1 + (unsigned)b1 * C2 + (unsigned)b2) << 2);
    bool use_fill = false;
    if (CHECK) {
      const int c0 = b0 - kMagicBits, c1 = b1 - kMagicBits, c2 = b2 - kMagicBits;
      if (!interior(c0, c1, c2)) use_fill = needs_fill(c0, c1, c2, u0, u1, u2, f0, f1, f2_, hi0, hi1, hi2);
    }
    // separable lerp K -> J -> I over the zero-padded box (<= 1 ulp from ATen's 8-term
    // weighted sum; the zero halo == skipping out-of-bounds corners)
    const float v000 = lds_f32<0>(addr), v001 = lds_f32<4>(addr);
    const float v010 = lds_f32<4 * C2>(addr), v011 = lds_f32<4 * C2 + 4>(addr);
    const float v100 = lds_f32<4 * C1>(addr), v101 = lds_f32<4 * C1 + 4>(addr);
    const float v110 = lds_f32<4 * (C1 + C2)>(addr), v111 = lds_f32<4 * (C1 + C2) + 4>(addr);
    const float a00 = __fmaf_rn(hi2, v001 - v000, v000);
    const float a01 = __fmaf_rn(hi2, v011 - v010, v010);
    const float a10 = __fmaf_rn(hi2, v101 - v100, v100);
    const float a11 = __fmaf_rn(hi2, v111 - v110, v110);
    const float bb0 = __fmaf_rn(hi1, a01 - a00, a00);
    const float bb1 = __fmaf_rn(hi1, a11 - a10, a10);
    float v = __fmaf_rn(hi0, bb1 - bb0, bb0);
    if (CHECK && use_fill) v = fill_c;
    *dst = ElemTraits<T>::from_f32(v);
  };

  // ---- two planes (oi, oi+1) in packed registers: same operations, lane by lane ----
  const f2 pj2 = bc(pj), pk2 = bc(pk);
  int planes = i1 - i0 + 1;
  // opaque to the optimiser: otherwise the trip count is re-derived from blockIdx (nine
  // instructions) in every iteration instead of living in a register
  asm volatile("" : "+r"(planes));
  f2 pi2 = pack2((float)i0, (float)(i0 + 1));
#pragma unroll 1
  for (int rel = 0; rel < planes; rel += 2, out += 2 * ostride, pi2 = add2(pi2, bc(2.0f))) {
    f2 q0, q1, q2;
    // planes go one at a time (single call site, the scalar body is large) when the pair
    // straddles a control cell, at the odd tail, and for EMODE 4 (spacing divides)
    bool pair_ok = (EMODE != 4) && (rel + 1 < planes);
    LiPair lp;
    if (EMODE != 0 && EMODE != 4) {
      lp = li_pairs[rel >> 1];  // warp-uniform broadcast (two LDS.128)
      pair_ok = pair_ok && lp.same_cell;
    }
    if (!pair_ok) {
      float pa, pb;
      unpack2(pi2, pa, pb);
      const int count = min(2, planes - rel);
#pragma unroll 1
      for (int t = 0; t < count; ++t) one(rel + t, t ? pb : pa, out + t * ostride);
      continue;
    }
    if (EMODE != 0) {
      refresh(LiEntry{lp.off0, lp.off1, lp.l0a, lp.l1a});
      const f2 l0 = pack2(lp.l0a, lp.l0b), l1 = pack2(lp.l1a, lp.l1b);
      const f2 d0 = fma2(l0, bc(r_lo[0]), mul2(l1, bc(r_hi[0])));
      const f2 d1 = fma2(l0, bc(r_lo[1]), mul2(l1, bc(r_hi[1])));
      const f2 d2 = fma2(l0, bc(r_lo[2]), mul2(l1, bc(r_hi[2])));
      if (EMODE == 1) {
        q0 = add2(pi2, d0); q1 = add2(pj2, d1); q2 = add2(pk2, d2);
      } else if (EMODE == 2) {
        q0 = add2(affine_row2(m + 0, pi2, pj2, pk2), d0);
        q1 = add2(affine_row2(m + 4, pi2, pj2, pk2), d1);
        q2 = add2(affine_row2(m + 8, pi2, pj2, pk2), d2);
      } else {
        const f2 e0 = add2(pi2, d0), e1 = add2(pj2, d1), e2 = add2(pk2, d2);
        q0 = affine_row2(m + 0, e0, e1, e2);
        q1 = affine_row2(m + 4, e0, e1, e2);
        q2 = affine_row2(m + 8, e0, e1, e2);
      }
    } else {
      q0 = affine_row2(m + 0, pi2, pj2, pk2);
      q1 = affine_row2(m + 4, pi2, pj2, pk2);
      q2 = affine_row2(m + 8, pi2, pj2, pk2);
    }
    const f2 one2 = bc(1.0f), mone2 = bc(-1.0f), magic2 = bc(kMagic), mmagic2 = bc(-kMagic);
    const f2 u0 = mul2(add2(add2(norm_div2<FASTDIV>(q0, hd0, rc0), mone2), one2), bc(hs0));
    const f2 u1 = mul2(add2(add2(norm_div2<FASTDIV>(q1, hd1, rc1), mone2), one2), bc(hs1));
    const f2 u2 = mul2(add2(add2(norm_div2<FASTDIV>(q2, hd2, rc2), mone2), one2), bc(hs2));
    if (MODE == TIO_NEAREST) {
      // round-to-nearest-even adds on the unpacked lanes: a multiply fused into this add
      // would round exact ties (u = n + 0.5) down instead of to even
      float u0a, u0b, u1a, u1b, u2a, u2b;
      unpack2(u0, u0a, u0b); unpack2(u1, u1a, u1b); unpack2(u2, u2a, u2b);
      const float r0a = __fadd_rn(u0a, kMagic), r0b = __fadd_rn(u0b, kMagic);
      const float r1a = __fadd_rn(u1a, kMagic), r1b = __fadd_rn(u1b, kMagic);
      const float r2a = __fadd_rn(u2a, kMagic), r2b = __fadd_rn(u2b, kMagic);
      const unsigned na = (unsigned)__float_as_int(r0a) * C1 + (unsigned)__float_as_int(r1a) * C2 +
                          (unsigned)__float_as_int(r2a);
      const unsigned nb = (unsigned)__float_as_int(r0b) * C1 + (unsigned)__float_as_int(r1b) * C2 +
                          (unsigned)__float_as_int(r2b);
      out[0] = lds_elem<T>(kbase + (na << ESH));
      out[ostride] = lds_elem<T>(kbase + (nb << ESH));
      continue;
    }
    if (MODE == TIO_LABEL_PV) {
      float u0a, u0b, u1a, u1b, u2a, u2b;
      unpack2(u0, u0a, u0b); unpack2(u1, u1a, u1b); unpack2(u2, u2a, u2b);
      out[0] = label_pv(u0a, u1a, u2a);
      out[ostride] = label_pv(u0b, u1b, u2b);
      continue;
    }
    const f2 s0 = add2_rd(u0, magic2), s1 = add2_rd(u1, magic2), s2 = add2_rd(u2, magic2);
    const f2 f0 = add2(s0, mmagic2), f1 = add2(s1, mmagic2), f2_ = add2(s2, mmagic2);
    const f2 hi0 = sub2(u0, f0), hi1 = sub2(u1, f1), hi2 = sub2(u2, f2_);
    float s0a, s0b, s1a, s1b, s2a, s2b;
    unpack2(s0, s0a, s0b); unpack2(s1, s1a, s1b); unpack2(s2, s2a, s2b);
    const int b0a = __float_as_int(s0a), b1a = __float_as_int(s1a), b2a = __float_as_int(s2a);
    const int b0b = __float_as_int(s0b), b1b = __float_as_int(s1b), b2b = __float_as_int(s2b);
    const uint32_t addr_a = kbase + (((unsigned)b0a * C1 + (unsigned)b1a * C2 + (unsigned)b2a) << 2);
    const uint32_t addr_b = kbase + (((unsigned)b0b * C1 + (unsigned)b1b * C2 + (unsigned)b2b) << 2);
    bool fill_a = false, fill_b = false;
    if (CHECK) {
      const int c0a = b0a - kMagicBits, c1a = b1a - kMagicBits, c2a = b2a - kMagicBits;
      const int c0b = b0b - kMagicBits, c1b = b1b - kMagicBits, c2b = b2b - kMagicBits;
      const bool in_a = interior(c0a, c1a, c2a), in_b = interior(c0b, c1b, c2b);
      if (!(in_a & in_b)) {
        float ua[3], ub[3], fa[3], fb[3], ha[3], hb[3];
        unpack2(u0, ua[0], ub[0]); unpack2(u1, ua[1], ub[1]); unpack2(u2, ua[2], ub[2]);
        unpack2(f0, fa[0], fb[0]); unpack2(f1, fa[1], fb[1]); unpack2(f2_, fa[2], fb[2]);
        unpack2(hi0, ha[0], hb[0]); unpack2(hi1, ha[1], hb[1]); unpack2(hi2, ha[2], hb[2]);
        if (!in_a) fill_a = needs_fill(c0a, c1a, c2a, ua[0], ua[1], ua[2], fa[0], fa[1], fa[2], ha[0], ha[1], ha[2]);
        if (!in_b) fill_b = needs_fill(c0b, c1b, c2b, ub[0], ub[1], ub[2], fb[0], fb[1], fb[2], hb[0], hb[1], hb[2]);
      }
    }
    const f2 v000 = pack2(lds_f32<0>(addr_a), lds_f32<0>(addr_b));
    const f2 v001 = pack2(lds_f32<4>(addr_a), lds_f32<4>(addr_b));
    const f2 v010 = pack2(lds_f32<4 * C2>(addr_a), lds_f32<4 * C2>(addr_b));
    const f2 v011 = pack2(lds_f32<4 * C2 + 4>(addr_a), lds_f32<4 * C2 + 4>(addr_b));
    const f2 v100 = pack2(lds_f32<4 * C1>(addr_a), lds_f32<4 * C1>(addr_b));
    const f2 v101 = pack2(lds_f32<4 * C1 + 4>(addr_a), lds_f32<4 * C1 + 4>(addr_b));
    const f2 v110 = pack2(lds_f32<4 * (C1 + C2)>(addr_a), lds_f32<4 * (C1 + C2)>(addr_b));
    const f2 v111 = pack2(lds_f32<4 * (C1 + C2) + 4>(addr_a), lds_f32<4 * (C1 + C2) + 4>(addr_b));
    const f2 a00 = fma2(hi2, sub2(v001, v000), v000);
    const f2 a01 = fma2(hi2, sub2(v011, v010), v010);
    const f2 a10 = fma2(hi2, sub2(v101, v100), v100);
    const f2 a11 = fma2(hi2, sub2(v111, v110), v110);
    const f2 bb0 = fma2(hi1, sub2(a01, a00), a00);
    const f2 bb1 = fma2(hi1, sub2(a11, a10), a10);
    float va, vb;
    unpack2(fma2(hi0, sub2(bb1, bb0), bb0), va, vb);
    if (CHECK && fill_a) va = fill_c;
    if (CHECK && fill_b) vb = fill_c;
    out[0] = ElemTraits<T>::from_f32(va);
    out[ostride] = ElemTraits<T>::from_f32(vb);
  }
}

template <int BOX, typename T, int MODE, bool HAS_CP, bool HAS_FILL, bool FASTDIV>
__global__ void __launch_bounds__(256, (BOX <= 22 && sizeof(T) == 4) ? 4 : 3)
resample_tile_kernel(const __grid_constant__ CUtensorMap tmap, const ResampleArgs a,
                     const TileArgs ta, const int4* __restrict__ records) {
  constexpr int BK = box_k_extent(BOX, (int)sizeof(T));
  constexpr int NBOX = BOX * BOX * BK;
  constexpr int BOXBYTES = (NBOX * (int)sizeof(T) + 15) / 16 * 16;
  constexpr int ESH = sizeof(T) == 1 ? 0 : (sizeof(T) == 2 ? 1 : 2);
  // layout: [box elements | li table (16 entries) | pair table (8) | mbarrier, kbase]
  extern __shared__ __align__(128) unsigned char smem_raw[];
  T* box = reinterpret_cast<T*>(smem_raw);
  float* aux = reinterpret_cast<float*>(smem_raw + BOXBYTES);
  LiEntry* li_tab = reinterpret_cast<LiEntry*>(aux);                          // [16]  64 floats
  LiPair* li_pairs = reinterpret_cast<LiPair*>(aux + 64);                     // [8]   64 floats
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(aux + 128);  // [+130] = kbase
  const int ncp = HAS_CP ? a.ni * a.nj * a.nk * 3 : 0;

  const int tid = threadIdx.x;
  const int tiles_i = ta.tiles_i;
  const int b = tiles_i == 1 ? (int)blockIdx.z : (int)__umulhi(blockIdx.z, ta.inv_tiles_i);
  const float* cps = HAS_CP ? a.cp + (int64_t)b * ncp : nullptr;  // global; see walk_column::refresh
  const int ti = blockIdx.z - b * tiles_i;
  const int i0 = ti * XT, j0 = blockIdx.y * XT, k0 = blockIdx.x * XT;
  const int i1 = min(i0 + XT, a.OI) - 1;
  // lanes 0-15 / 16-31 of a warp take rows DJ apart: with row pitch BK the two
  // half-warps then hit disjoint banks (DJ * BK == 16 mod 32) for axis-aligned reads
  // BK = 24, 28, 28, 32, 36 -> DJ = 2, 4, 4, (none: 4), 4
  constexpr int DJ = (BOX == 20) ? 2 : 4;
  const int warp = tid >> 5, half = (tid >> 4) & 1;
  const int jrow = (warp % DJ) + (warp / DJ) * (2 * DJ) + half * DJ;
  int oj = j0 + jrow, ok = k0 + (tid & 15);
  // kept in registers across the TMA wait (opaque to the optimiser, which otherwise
  // re-derives them from threadIdx/blockIdx after the barrier)
  asm volatile("" : "+r"(oj), "+r"(ok));
  const bool active = (oj < a.OJ) && (ok < a.OK);
  const int64_t n_in = ta.n_in, n_out = ta.n_out;
  const uint8_t fl = a.flags ? a.flags[b] : 0;
  const T* __restrict__ src = (const T*)a.src + (int64_t)b * a.C * n_in;
  T* __restrict__ dst = (T*)a.dst + (int64_t)b * a.C * n_out;

  if (fl & TIO_FLAG_PASSTHROUGH) {
    if (active)
      for (int c = 0; c < a.C; ++c)
        for (int oi = i0; oi <= i1; ++oi) {
          const int64_t o = ((int64_t)oi * a.OJ + oj) * a.OK + ok;
          dst[c * n_out + o] = src[c * n_in + o];
        }
    return;
  }
  const unsigned tile_id = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;  // < 2^31 (launcher)
  const int4 rec = __ldg(records + tile_id);
  const bool tile_interior = (rec.w & 256) != 0;
  // nearest + fill on a tile that touches the border: the per-voxel mask lives in the general column
  const int fit_code = (MODE == TIO_NEAREST && HAS_FILL && !tile_interior && (rec.w & 255) == 1) ? 0 : (rec.w & 255);
  const bool elastic = HAS_CP && (fl & TIO_FLAG_ELASTIC);

  if (fit_code == 2) {  // pre-image entirely outside the volume
    if (active)
      for (int c = 0; c < a.C; ++c) {
        const T v = HAS_FILL ? ElemTraits<T>::from_f32(a.fill[c]) : (T)0;
        for (int oi = i0; oi <= i1; ++oi)
          dst[c * n_out + ((int64_t)oi * a.OJ + oj) * a.OK + ok] = v;
      }
    return;
  }
  if (tid == 0 && fit_code == 1) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    // first channel's box: in flight while the CTA stages the control grid
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"((uint32_t)(NBOX * sizeof(T)))
                 : "memory");
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(smem_u32(box)),
        "l"((unsigned long long)&tmap), "r"(rec.z), "r"(rec.y), "r"(rec.x), "r"(b * a.C), "r"(smem_u32(bar))
        : "memory");
  }
  if (tid == 32) {
    constexpr int C1 = BOX * BK, C2 = BK;
    const unsigned koff = (unsigned)(kMagicBits + rec.x) * C1 + (unsigned)(kMagicBits + rec.y) * C2 +
                          (unsigned)(kMagicBits + rec.z);
    *reinterpret_cast<uint32_t*>(aux + 130) = smem_u32(box) - (koff << ESH);
  }
  if (elastic) {
    if (tid < XT) {
      const LerpAxis li = lerp_axis(a.sc_i, a.ni, min(i0 + tid, a.OI - 1));
      const int plane = a.nj * a.nk * 3;
      li_tab[tid] = LiEntry{li.i0 * plane, li.i1 * plane, li.l0, li.l1};
    } else if (tid >= 32 && tid < 32 + XT / 2) {
      const int pr = tid - 32;
      const LerpAxis la = lerp_axis(a.sc_i, a.ni, min(i0 + 2 * pr, a.OI - 1));
      const LerpAxis lb = lerp_axis(a.sc_i, a.ni, min(i0 + 2 * pr + 1, a.OI - 1));
      const int plane = a.nj * a.nk * 3;
      li_pairs[pr] = LiPair{la.i0 * plane, la.i1 * plane, la.l0, lb.l0, la.l1, lb.l1,
                            (la.i0 == lb.i0 && la.i1 == lb.i1) ? 1 : 0, 0};
    }
  }
  __syncthreads();  // mbarrier init + control grid + li table visible

  if (fit_code == 0) {  // general global-memory path for this tile (CTA-uniform branch)
    if (active)
      general_column<T, MODE, HAS_CP, HAS_FILL>(a, b, elastic, elastic ? cps : nullptr, src,
                                                          dst, n_in, n_out, i0, i1 + 1, oj, ok);
    return;
  }

  constexpr int C1 = BOX * BK, C2 = BK;
  // wraps; undone by the per-voxel sum.  Read back through shared memory so ptxas sees
  // an opaque value (it otherwise splits off the 0x4B400000*(C1+C2+1) part and re-adds
  // it in front of each of the 8 taps)
  const uint32_t kbase = *reinterpret_cast<volatile uint32_t*>(aux + 130);
  const bool identity = elastic && (rec.w & 512);  // matrix == I (tile_bounds_kernel)
  float m[12];
  if (!identity) {
#pragma unroll
    for (int t = 0; t < 12; ++t) m[t] = a.mat[b * 12 + t];
  } else {
#pragma unroll
    for (int t = 0; t < 12; ++t) m[t] = (t % 5 == 0) ? 1.0f : 0.0f;
  }
  const int64_t ostride = (int64_t)a.OJ * a.OK;
  const bool unit_spacing = a.affine_first ? ta.sp_in_one : ta.sp_out_one;
  const int emode = !elastic ? 0 : (!unit_spacing ? 4 : (!a.affine_first ? 3 : (identity ? 1 : 2)));

  for (int c = 0; c < a.C; ++c) {
    if (c > 0 && tid == 0) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                   "r"((uint32_t)(NBOX * sizeof(T)))
                   : "memory");
      asm volatile(
          "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
          " [%0], [%1, {%2, %3, %4, %5}], [%6];" ::"r"(smem_u32(box)),
          "l"((unsigned long long)&tmap), "r"(rec.z), "r"(rec.y), "r"(rec.x), "r"(b * a.C + c),
          "r"(smem_u32(bar))
          : "memory");
    }
    // wait for the box (phase parity = c & 1): one warp polls the mbarrier, the other
    // seven park on the hardware barrier instead of burning issue slots in a spin loop
    if (tid < 32) {
      const uint32_t parity = (uint32_t)(c & 1);
      uint32_t done;
      do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
      } while (!done);
    }
    __syncthreads();
    if (active) {
      T* out = dst + c * n_out + ((int64_t)i0 * a.OJ + oj) * a.OK + ok;
      const bool chk = HAS_FILL && !tile_interior;
#define TIO_WALK(CHK, EM)                                                                            \
  walk_column<BOX, T, MODE, HAS_CP, CHK, FASTDIV, EM>(a, ta, box, cps, li_tab, li_pairs, m, elastic, identity, \
                                             kbase, i0, i1, oj, ok,                                         \
                                             (chk || MODE == TIO_LABEL_PV) ? a.fill[c] : 0.0f, out, ostride)
      bool walked = false;
      if constexpr ((MODE == TIO_LINEAR || MODE == TIO_LABEL_PV) && HAS_FILL) {
        if (chk) {
          walked = true;
          if (emode == 0) TIO_WALK(true, 0);
          else if (emode == 1) TIO_WALK(true, 1);
          else if (emode == 2) TIO_WALK(true, 2);
          else if (emode == 3) TIO_WALK(true, 3);
          else TIO_WALK(true, 4);
        }
      }
      if (!walked) {
        if (emode == 0) TIO_WALK(false, 0);
        else if (emode == 1) TIO_WALK(false, 1);
        else if (emode == 2) TIO_WALK(false, 2);
        else if (emode == 3) TIO_WALK(false, 3);
        else TIO_WALK(false, 4);
      }
#undef TIO_WALK
    }
    if (c + 1 < a.C) __syncthreads();  // box is reused by the next channel
  }
}


// ---- exhaustive admission test of the reciprocal division --------------------
__global__ void verify_fastdiv_kernel(float d, float r, unsigned long long* bad) {
  const unsigned long long total = 1ull << 32;
  unsigned long long local = 0;
  for (unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned bits = (unsigned)t;
    const unsigned ex = (bits >> 23) & 0xffu;
    // quotients below 2^-25 all normalise to g = -1 exactly, so |x| < 2^-100 cannot
    // change any coordinate; inf/nan never reach the fast path (box-fit test)
    if (ex < 27u || ex > 190u) continue;
    const float x = __uint_as_float(bits);
    const float want = __fdiv_rn(x, d);
    const float q0 = __fmul_rn(x, r);
    const float q = __fmaf_rn(__fmaf_rn(-q0, d, x), r, q0);
    local += (__float_as_uint(q) != __float_as_uint(want));
  }
  if (local) atomicAdd(bad, local);
}

static std::mutex g_fd_mutex;
static std::map<uint32_t, bool> g_fd_cache;

// true iff rn(x*r) + 2-FMA correction == x/d for every float x (r = rn(1/d))
static bool fastdiv_admitted(float d, cudaStream_t st) {
  uint32_t key;
  memcpy(&key, &d, 4);
  {
    std::lock_guard<std::mutex> lock(g_fd_mutex);
    auto it = g_fd_cache.find(key);
    if (it != g_fd_cache.end()) return it->second;
  }
  bool ok = false;
  unsigned long long* bad = nullptr;
  if (cudaMalloc(&bad, 8) == cudaSuccess) {
    cudaMemsetAsync(bad, 0, 8, st);
    verify_fastdiv_kernel<<<num_sms() * 16, 256, 0, st>>>(d, (float)(1.0 / (double)d), bad);
    launched();
    unsigned long long host = 1;
    if (cudaMemcpyAsync(&host, bad, 8, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
        cudaStreamSynchronize(st) == cudaSuccess)
      ok = (host == 0);
    cudaFree(bad);
  }
  std::lock_guard<std::mutex> lock(g_fd_mutex);
  g_fd_cache[key] = ok;
  return ok;
}

template <int BOX, typename T, int MODE, bool HAS_CP, bool FASTDIV>
static void launch_tile(const CUtensorMap& tm, const ResampleArgs& a, const TileArgs& ta, dim3 grid,
                        size_t smem, const int4* records, cudaStream_t st) {
  if (a.fill) {
    cudaFuncSetAttribute(resample_tile_kernel<BOX, T, MODE, HAS_CP, true, FASTDIV>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    resample_tile_kernel<BOX, T, MODE, HAS_CP, true, FASTDIV><<<grid, 256, smem, st>>>(tm, a, ta, records);
  } else {
    cudaFuncSetAttribute(resample_tile_kernel<BOX, T, MODE, HAS_CP, false, FASTDIV>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    resample_tile_kernel<BOX, T, MODE, HAS_CP, false, FASTDIV><<<grid, 256, smem, st>>>(tm, a, ta, records);
  }
  launched();
}

template <int BOX>
static void launch_box(const CUtensorMap& tm, const ResampleArgs& a, const TileArgs& ta, dim3 grid,
                       size_t smem, bool fast, const int4* records, cudaStream_t st) {
  if (a.cp) {
    if (fast) launch_tile<BOX, float, TIO_LINEAR, true, true>(tm, a, ta, grid, smem, records, st);
    else launch_tile<BOX, float, TIO_LINEAR, true, false>(tm, a, ta, grid, smem, records, st);
  } else {
    if (fast) launch_tile<BOX, float, TIO_LINEAR, false, true>(tm, a, ta, grid, smem, records, st);
    else launch_tile<BOX, float, TIO_LINEAR, false, false>(tm, a, ta, grid, smem, records, st);
  }
}

void launch_resample_fast(int box, const CUtensorMap& tm, const CUtensorMap& tm_small, const ResampleArgs& a,
                          const TileArgs& ta, dim3 grid,
                          size_t smem, const int4* records, cudaStream_t st);  // resample_fast.cu

// nearest-neighbour label maps: the admitted-division variants only (else the caller's
// general kernel), boxes 24 and 32
template <typename T>
static void launch_nearest(int box, const CUtensorMap& tm, const ResampleArgs& a, const TileArgs& ta,
                           dim3 grid, size_t smem, const int4* records, cudaStream_t st) {
  if (box == 24) {
    if (a.cp) launch_tile<24, T, TIO_NEAREST, true, true>(tm, a, ta, grid, smem, records, st);
    else launch_tile<24, T, TIO_NEAREST, false, true>(tm, a, ta, grid, smem, records, st);
  } else {
    if (a.cp) launch_tile<32, T, TIO_NEAREST, true, true>(tm, a, ta, grid, smem, records, st);
    else launch_tile<32, T, TIO_NEAREST, false, true>(tm, a, ta, grid, smem, records, st);
  }
}

// partial-volume label maps (TIO_LABEL_PV): same boxes and admitted-division variants as nearest;
// the pad label is always present (HAS_FILL)
template <typename T>
static void launch_label_pv(int box, const CUtensorMap& tm, const ResampleArgs& a, const TileArgs& ta,
                            dim3 grid, size_t smem, const int4* records, cudaStream_t st) {
  if (box == 24) {
    if (a.cp) launch_tile<24, T, TIO_LABEL_PV, true, true>(tm, a, ta, grid, smem, records, st);
    else launch_tile<24, T, TIO_LABEL_PV, false, true>(tm, a, ta, grid, smem, records, st);
  } else {
    if (a.cp) launch_tile<32, T, TIO_LABEL_PV, true, true>(tm, a, ta, grid, smem, records, st);
    else launch_tile<32, T, TIO_LABEL_PV, false, true>(tm, a, ta, grid, smem, records, st);
  }
}

// Returns 0 when launched, 1 when the fast path does not apply (caller falls back),
// >1 on error.
size_t resample_tile_workspace_bytes(int B, int OI, int OJ, int OK) {
  const size_t tiles = (size_t)B * ((OI + XT - 1) / XT) * ((OJ + XT - 1) / XT) * ((OK + XT - 1) / XT);
  return tiles * sizeof(int4);
}

int launch_resample_tile(const ResampleArgs& a, int dtype, int mode, bool exact_coords, int box_hint,
                         const int* runs, int n_runs, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  // fp32 trilinear, or nearest for the 1/2/4-byte label types
  int esize = 0;
  if (mode == TIO_LINEAR) esize = dtype == TIO_F32 ? 4 : 0;
  else esize = dtype == TIO_U8 ? 1 : dtype == TIO_I16 ? 2 : dtype == TIO_I32 ? 4 : 0;
  if (!esize) return 1;
  const int kalign = 16 / esize;
  if (((int64_t)a.K * esize & 15) || ((uintptr_t)a.src & 15)) return 1;   // TMA strides must be 16-byte multiples
  if ((int64_t)a.B * a.C > (1 << 30)) return 1;
  EncodeTiledFn encode = encode_tiled_fn();
  if (!encode) return 1;
  // supported box edges; 0 (auto) = 24
  int box = 24;
  if (box_hint > 0) box = box_hint <= 20 ? 20 : box_hint <= 22 ? 22 : box_hint <= 24 ? 24 : box_hint <= 28 ? 28 : 32;
  if (mode != TIO_LINEAR) box = box <= 24 ? 24 : 32;
  const int tiles_i = (a.OI + XT - 1) / XT;
  if ((int64_t)a.B * tiles_i > 65535 || (a.OJ + XT - 1) / XT > 65535) return 1;

  const cuuint64_t gdim[4] = {(cuuint64_t)a.K, (cuuint64_t)a.J, (cuuint64_t)a.I, (cuuint64_t)a.B * a.C};
  const cuuint64_t gstride[3] = {(cuuint64_t)a.K * esize, (cuuint64_t)a.J * a.K * esize,
                                 (cuuint64_t)a.I * a.J * a.K * esize};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapDataType ttype = mode == TIO_LINEAR ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                    : esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                    : esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                                                 : CU_TENSOR_MAP_DATA_TYPE_INT32;
  // tensor map of a box x box x box_k_extent(box) box
  auto encode_box = [&](CUtensorMap* tm, int edge) {
    const cuuint32_t bdim[4] = {(cuuint32_t)box_k_extent(edge, esize), (cuuint32_t)edge, (cuuint32_t)edge, 1};
    return encode(tm, ttype, 4, const_cast<void*>(a.src), gdim, gstride, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  };

  TileArgs ta;
  bool fast = true;
  for (int t = 0; t < 3; ++t) {
    ta.hd[t] = a.nm1[t] * 0.5f;
    ta.rcp[t] = (float)(1.0 / (double)ta.hd[t]);
    ta.hs[t] = a.sm1[t] * 0.5f;
    fast = fast && fastdiv_admitted(ta.hd[t], st);
  }
  ta.n_in = (long long)a.I * a.J * a.K;
  ta.n_out = (long long)a.OI * a.OJ * a.OK;
  ta.tiles_i = tiles_i;
  ta.inv_tiles_i = (unsigned)((1ull << 32) / (unsigned)tiles_i) + 1u;
  ta.sp_in_one = (a.sp_in[0] == 1.f && a.sp_in[1] == 1.f && a.sp_in[2] == 1.f);
  ta.sp_out_one = (a.sp_out[0] == 1.f && a.sp_out[1] == 1.f && a.sp_out[2] == 1.f);
  ta.magic_bytes = (unsigned)kMagicBits << 2;
  for (int t = 0; t < 3; ++t) {
    ta.rsp_in[t] = (float)(1.0 / (double)a.sp_in[t]);
    ta.rsp_out[t] = (float)(1.0 / (double)a.sp_out[t]);
  }

  const int64_t tiles_per_elem = (int64_t)tiles_i * ((a.OJ + XT - 1) / XT) * ((a.OK + XT - 1) / XT);
  const int64_t n_tiles = (int64_t)a.B * tiles_per_elem;
  if (n_tiles >= (1ll << 31)) return 1;
  // per-tile records live in caller-provided workspace: no allocation, no state kept
  if (!workspace || workspace_bytes < (size_t)n_tiles * sizeof(int4) || ((uintptr_t)workspace & 15)) return 1;
  if (mode != TIO_LINEAR && !fast) return 1;
  // elastic launches of the fast kernel: most tiles need far less than the launch's box (the
  // displacement is smooth, its borders are locked) and load a small box instead
  const bool dual = !exact_coords && mode == TIO_LINEAR && a.cp;  // every edge is > kSmallBox
  CUtensorMap tm_small;
  if (dual && !encode_box(&tm_small, kSmallBox)) return 1;

  // one launch pair (bounds pre-pass, tile kernel) per run of slots sharing a box edge: the
  // caller's runs for a tiered call (a.elems set), else all B elements at `box`
  const int whole[2] = {a.B, box};
  if (!a.elems) { runs = whole; n_runs = 1; }
  CUtensorMap tms[5];
  for (int r = 0; r < n_runs; ++r)
    if (!encode_box(&tms[r], runs[2 * r + 1])) return 1;
  int offset = 0;
  for (int r = 0; r < n_runs; ++r) {
    const int count = runs[2 * r], edge = runs[2 * r + 1];
    const CUtensorMap& tm = tms[r];
    ResampleArgs ar = a;
    ar.B = count;
    ar.elems = a.elems ? a.elems + offset : nullptr;
    int4* records = (int4*)workspace + offset * tiles_per_elem;
    offset += count;
    const dim3 grid((a.OK + XT - 1) / XT, (a.OJ + XT - 1) / XT, (unsigned)(count * tiles_i));
    const int bk = box_k_extent(edge, esize);
    const int box_s = dual ? kSmallBox : 0, bk_s = dual ? box_k_extent(kSmallBox, 4) : 0;
    const unsigned bounds_blocks = (unsigned)((count * tiles_per_elem + 127) / 128);
    if (ar.cp) tile_bounds_kernel<true><<<bounds_blocks, 128, 0, st>>>(ar, edge, kalign, bk, box_s, bk_s, records);
    else tile_bounds_kernel<false><<<bounds_blocks, 128, 0, st>>>(ar, edge, kalign, bk, box_s, bk_s, records);
    launched();
    const size_t smem = ((size_t)edge * edge * bk * esize + 15) / 16 * 16 + kAuxFloats * sizeof(float);
    if (mode == TIO_LABEL_PV) {
      if (dtype == TIO_U8) launch_label_pv<uint8_t>(edge, tm, ar, ta, grid, smem, records, st);
      else if (dtype == TIO_I16) launch_label_pv<int16_t>(edge, tm, ar, ta, grid, smem, records, st);
      else launch_label_pv<int32_t>(edge, tm, ar, ta, grid, smem, records, st);
    } else if (mode == TIO_NEAREST) {
      if (dtype == TIO_U8) launch_nearest<uint8_t>(edge, tm, ar, ta, grid, smem, records, st);
      else if (dtype == TIO_I16) launch_nearest<int16_t>(edge, tm, ar, ta, grid, smem, records, st);
      else launch_nearest<int32_t>(edge, tm, ar, ta, grid, smem, records, st);
    } else if (!exact_coords) {  // fp32 images: one-fma coordinates where no tap can leave the volume
      launch_resample_fast(edge, tm, dual ? tm_small : tm, ar, ta, grid, smem, records, st);
    } else if (edge == 20) launch_box<20>(tm, ar, ta, grid, smem, fast, records, st);
    else if (edge == 22) launch_box<22>(tm, ar, ta, grid, smem, fast, records, st);
    else if (edge == 24) launch_box<24>(tm, ar, ta, grid, smem, fast, records, st);
    else if (edge == 28) launch_box<28>(tm, ar, ta, grid, smem, fast, records, st);
    else launch_box<32>(tm, ar, ta, grid, smem, fast, records, st);
  }
  return 0;
}

}  // namespace tio

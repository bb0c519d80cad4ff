// resample_fast.cu — K1 for fp32 images, trilinear: TMA-staged tiles with one-fma coordinates.
//
// A large share of the exact kernel's (resample_tile.cu) instructions per voxel is the
// reference's fp32 rounding chain (sgemm order, normalise / un-normalise round trip).
//
// For a voxel whose 8 taps all lie inside the volume that chain only reproduces the
// reference's own coordinate noise (<= 1.5e-5 voxel): no fill decision and no zero halo
// depends on it.  This kernel therefore evaluates the same mapping as ONE fma per axis
// and voxel,
//     u(rel) = A + rel * B          rel = plane within the 16-plane tile
// in BOX-RELATIVE coordinates (|u| < 36, ulp 2e-6: closer to the real-valued mapping than
// the reference's chain, whose intermediate terms are volume-sized).  A and B are per
// (j,k)-column constants; the trilinear upsample of the control grid is linear in rel
// inside a control cell, so the elastic displacement (and the spacing divide, and
// M (p + d)) folds into the same two constants, recomputed when the walk enters a new
// cell.  The tile base, where volume-sized terms cancel, is formed once per tile in fp64.
//
// Zero padding comes from the TMA box (out-of-volume taps arrive as zeros).  The fill
// decision of border tiles (mask > 0.5, the mask being the trilinear weight of the in-bounds
// corners) is evaluated from the same coordinates through its separable form; the few voxels
// within 1e-3 of the threshold are recomputed by the exact general column of
// resample_common.cuh, so fill decisions stay bit-exact.  Label maps, nearest interpolation
// and TIO_EXACT_COORDS launches use resample_tile.cu.
#include <type_traits>

#include "resample_tile.cuh"

namespace tio {

// lane -> (row, column) of the 16 x 16 (j,k) face; LK = lanes along k per row
template <int BOX, int LK>
__device__ __forceinline__ void lane_column(int tid, int& jrow, int& kcol) {
  const int warp = tid >> 5, lane = tid & 31;
  if (LK == 16) {
    constexpr int DJ = (BOX == 20) ? 2 : 4;
    const int half = lane >> 4;
    jrow = (warp % DJ) + (warp / DJ) * (2 * DJ) + half * DJ;
    kcol = lane & 15;
  } else if (LK == 8) {
    jrow = (warp >> 1) * 4 + (lane >> 3);
    kcol = (warp & 1) * 8 + (lane & 7);
  } else {
    jrow = (warp >> 2) * 8 + (lane >> 2);
    kcol = (warp & 3) * 4 + (lane & 3);
  }
}

// exact planes [oi0, oi_end) of one column (fill decisions, zero padding): global-memory taps
template <bool HAS_CP, bool HAS_FILL>
__device__ __forceinline__ void exact_planes(const ResampleArgs& a, const TileArgs& ta, int b, bool elastic,
                                          int oi0, int oi_end, int oj, int ok) {
  const int64_t n_in = ta.n_in, n_out = ta.n_out;
  const float* src = (const float*)a.src + (int64_t)b * a.C * n_in;
  float* dst = (float*)a.dst + (int64_t)b * a.C * n_out;
  const float* cps = (HAS_CP && elastic) ? a.cp + (int64_t)b * (a.ni * a.nj * a.nk * 3) : nullptr;
  general_column<float, TIO_LINEAR, HAS_CP, HAS_FILL>(a, b, elastic, cps, src, dst, n_in, n_out, oi0, oi_end, oj, ok);
}

// planes of one column flagged in `planes` (bit rel), runs of consecutive planes at a time
template <bool HAS_CP, bool HAS_FILL>
__device__ __noinline__ void exact_fix(const ResampleArgs& a, const TileArgs& ta, int b, bool elastic, int i0,
                                       unsigned planes, int oj, int ok) {
  while (planes) {
    const int first = __ffs(planes) - 1;
    const int len = __ffs(~(planes >> first)) - 1;  // run of set bits starting at `first`
    exact_planes<HAS_CP, HAS_FILL>(a, ta, b, elastic, i0 + first, i0 + first + len, oj, ok);
    planes &= ~(((1u << len) - 1u) << first);
  }
}

// Tiles the fast walk does not take: pass-through elements, pre-images outside the volume,
// boxes that do not fit, ragged tiles at the end of an axis.
template <bool HAS_CP, bool HAS_FILL>
__device__ __noinline__ void slow_tile(const ResampleArgs& a, const TileArgs& ta, const int4 rec, int b, int i0,
                                       int j0, int k0) {
  const int tid = threadIdx.x;
  const int oj = j0 + (tid >> 4), ok = k0 + (tid & 15);
  if (oj >= a.OJ || ok >= a.OK) return;
  const int i1 = min(i0 + XT, a.OI);
  const int code = rec.w & 255;
  const int64_t n_in = ta.n_in, n_out = ta.n_out;
  const float* src = (const float*)a.src + (int64_t)b * a.C * n_in;
  float* dst = (float*)a.dst + (int64_t)b * a.C * n_out;
  if (code == 3) {  // bit copy (spatial.py:1101-1106)
    for (int c = 0; c < a.C; ++c)
      for (int oi = i0; oi < i1; ++oi) {
        const int64_t o = ((int64_t)oi * a.OJ + oj) * a.OK + ok;
        dst[c * n_out + o] = src[c * n_in + o];
      }
    return;
  }
  if (code == 2) {  // every tap is padding
    for (int c = 0; c < a.C; ++c) {
      const float v = HAS_FILL ? a.fill[c] : 0.0f;
      for (int oi = i0; oi < i1; ++oi) dst[c * n_out + ((int64_t)oi * a.OJ + oj) * a.OK + ok] = v;
    }
    return;
  }
  exact_planes<HAS_CP, HAS_FILL>(a, ta, b, HAS_CP && (rec.w & 1024), i0, i1, oj, ok);
}

// Taps of the upper plane (i + 1) of the previous voxel of the walk and the shared-memory address
// they were read from.  Along the walk the sampling point advances by about one voxel in I and
// by little in J/K, so for most voxels the lower-plane taps ARE the previous voxel's upper-plane
// taps: they stay in registers and the four lower-plane loads run predicated, only for the lanes
// whose cell moved in J/K or skipped a plane: the kernel is bound by the shared-memory data
// pipe (rotated rows step across box rows, so an LDS takes about two wavefronts).
struct Carry {
  float u00, u01, u10, u11;
  uint32_t up;  // address of the (i + 1, j, k) tap the values came from; 0xffffffff = none
};

template <int C2>
__device__ __forceinline__ void lds4_unless(float& v00, float& v01, float& v10, float& v11, const uint32_t addr,
                                            const uint32_t same) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.u32 p, %4, %5;\n\t"
      "@p ld.shared.f32 %0, [%4];\n\t"
      "@p ld.shared.f32 %1, [%4+4];\n\t"
      "@p ld.shared.f32 %2, [%4+%6];\n\t"
      "@p ld.shared.f32 %3, [%4+%7];\n\t"
      "}"
      : "+f"(v00), "+f"(v01), "+f"(v10), "+f"(v11)
      : "r"(addr), "r"(same), "n"(4 * C2), "n"(4 * C2 + 4));
}

// One pair of planes (rel, rel + 1) of a column.  MASKED (border tile with a fill value): the
// reference's mask, the trilinear weight sum of the in-bounds corners, is separable — per axis
// the in-bounds weight is the trapezoid sat(min(u - (lo - 1), (hi + 1) - u)) — so it is
// evaluated from the same coordinates; voxels whose mask is within 1e-3 of the 0.5 threshold
// (coordinate noise moves it by < 1e-4) are flagged and recomputed exactly afterwards.
template <int C1, int C2, bool MASKED, bool REUSE>
__device__ __forceinline__ void pair_step(const f2 rel2, const f2 A0, const f2 A1, const f2 A2, const f2 B0,
                                          const f2 B1, const f2 B2, const uint32_t kb, const float* tz,
                                          const float fill_c, float& va, float& vb, bool& unc_a, bool& unc_b,
                                          Carry& carry) {
  const f2 magic2 = bc(kMagic), mmagic2 = bc(-kMagic);
  const f2 u0 = fma2(rel2, B0, A0), u1 = fma2(rel2, B1, A1), u2 = fma2(rel2, B2, A2);
  const f2 s0 = add2_rd(u0, magic2), s1 = add2_rd(u1, magic2), s2 = add2_rd(u2, magic2);
  const f2 f0 = add2(s0, mmagic2), f1 = add2(s1, mmagic2), f2_ = add2(s2, mmagic2);
  const f2 hi0 = sub2(u0, f0), hi1 = sub2(u1, f1), hi2 = sub2(u2, f2_);
  // magic + (b0 * C1 + b1 * C2 + b2): exact (< 2^24), the mantissa is the element index
  const f2 idx = fma2(f0, bc((float)C1), fma2(f1, bc((float)C2), s2));
  float ia, ib;
  unpack2(idx, ia, ib);
  const uint32_t addr_a = ((uint32_t)__float_as_int(ia) << 2) + kb;
  const uint32_t addr_b = ((uint32_t)__float_as_int(ib) << 2) + kb;
  f2 v000, v001, v010, v011, v100, v101, v110, v111;
  if (REUSE) {
    const float ua00 = lds_f32<4 * C1>(addr_a), ua01 = lds_f32<4 * C1 + 4>(addr_a);
    const float ua10 = lds_f32<4 * (C1 + C2)>(addr_a), ua11 = lds_f32<4 * (C1 + C2) + 4>(addr_a);
    const float ub00 = lds_f32<4 * C1>(addr_b), ub01 = lds_f32<4 * C1 + 4>(addr_b);
    const float ub10 = lds_f32<4 * (C1 + C2)>(addr_b), ub11 = lds_f32<4 * (C1 + C2) + 4>(addr_b);
    float la00 = carry.u00, la01 = carry.u01, la10 = carry.u10, la11 = carry.u11;
    lds4_unless<C2>(la00, la01, la10, la11, addr_a, carry.up);
    float lb00 = ua00, lb01 = ua01, lb10 = ua10, lb11 = ua11;
    lds4_unless<C2>(lb00, lb01, lb10, lb11, addr_b, addr_a + 4u * C1);
    carry.u00 = ub00; carry.u01 = ub01; carry.u10 = ub10; carry.u11 = ub11;
    carry.up = addr_b + 4u * C1;
    v000 = pack2(la00, lb00); v001 = pack2(la01, lb01); v010 = pack2(la10, lb10); v011 = pack2(la11, lb11);
    v100 = pack2(ua00, ub00); v101 = pack2(ua01, ub01); v110 = pack2(ua10, ub10); v111 = pack2(ua11, ub11);
  } else {
    v000 = pack2(lds_f32<0>(addr_a), lds_f32<0>(addr_b));
    v001 = pack2(lds_f32<4>(addr_a), lds_f32<4>(addr_b));
    v010 = pack2(lds_f32<4 * C2>(addr_a), lds_f32<4 * C2>(addr_b));
    v011 = pack2(lds_f32<4 * C2 + 4>(addr_a), lds_f32<4 * C2 + 4>(addr_b));
    v100 = pack2(lds_f32<4 * C1>(addr_a), lds_f32<4 * C1>(addr_b));
    v101 = pack2(lds_f32<4 * C1 + 4>(addr_a), lds_f32<4 * C1 + 4>(addr_b));
    v110 = pack2(lds_f32<4 * (C1 + C2)>(addr_a), lds_f32<4 * (C1 + C2)>(addr_b));
    v111 = pack2(lds_f32<4 * (C1 + C2) + 4>(addr_a), lds_f32<4 * (C1 + C2) + 4>(addr_b));
  }
  const f2 a00 = fma2(hi2, sub2(v001, v000), v000);
  const f2 a01 = fma2(hi2, sub2(v011, v010), v010);
  const f2 a10 = fma2(hi2, sub2(v101, v100), v100);
  const f2 a11 = fma2(hi2, sub2(v111, v110), v110);
  const f2 bb0 = fma2(hi1, sub2(a01, a00), a00);
  const f2 bb1 = fma2(hi1, sub2(a11, a10), a10);
  unpack2(fma2(hi0, sub2(bb1, bb0), bb0), va, vb);
  if (MASKED) {
    float ma = 1.0f, mb = 1.0f;
    const f2 u[3] = {u0, u1, u2};
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
      float pa, pb, qa, qb;
      unpack2(sub2(u[ax], bc(tz[2 * ax])), pa, pb);      // u - (lo - 1)
      unpack2(sub2(bc(tz[2 * ax + 1]), u[ax]), qa, qb);  // (hi + 1) - u
      ma *= __saturatef(fminf(pa, qa));
      mb *= __saturatef(fminf(pb, qb));
    }
    if (!(ma > 0.5f)) va = fill_c;
    if (!(mb > 0.5f)) vb = fill_c;
    unc_a = fabsf(ma - 0.5f) < 1.0e-3f;
    unc_b = fabsf(mb - 0.5f) < 1.0e-3f;
  }
}

// Affine launches keep the upper-plane taps in registers along the walk (Carry); elastic launches
// load all eight taps of every voxel.
template <int BOX, bool HAS_CP, bool HAS_FILL>
__global__ void __launch_bounds__(256, BOX <= 22 ? 4 : 3)
resample_fast_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_s,
                     const __grid_constant__ ResampleArgs a, const __grid_constant__ TileArgs ta,
                     const int4* __restrict__ records) {
  constexpr int BK = box_k_extent(BOX, 4);
  constexpr int NBOX = BOX * BOX * BK;
  constexpr int BOXBYTES = (NBOX * 4 + 15) / 16 * 16;
  constexpr int C1 = BOX * BK, C2 = BK;
  // elastic launches: tiles whose pre-image fits the small box load that instead (bit 12)
  constexpr bool DUAL = HAS_CP && BOX > kSmallBox;
  constexpr int BKS = box_k_extent(kSmallBox, 4);
  constexpr int NBOXS = kSmallBox * kSmallBox * BKS, C1S = kSmallBox * BKS, C2S = BKS;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* aux = reinterpret_cast<float*>(smem_raw + BOXBYTES);
  const uint32_t box_u32 = smem_u32(smem_raw);
  const uint32_t bar = smem_u32(aux + 128);
  float* tbase = aux + 132;                            // [3] tile base coordinate, box relative
  int* cell_tab = reinterpret_cast<int*>(aux + 136);   // [16] control cell of each plane
  unsigned* chg_mask = reinterpret_cast<unsigned*>(aux + 152);

  const int tid = threadIdx.x;
  const int tiles_i = ta.tiles_i;
  const int slot = tiles_i == 1 ? (int)blockIdx.z : (int)__umulhi(blockIdx.z, ta.inv_tiles_i);
  const int ti = blockIdx.z - slot * tiles_i;
  const int b = a.elems ? __ldg(a.elems + slot) : slot;
  const int i0 = ti * XT, j0 = blockIdx.y * XT, k0 = blockIdx.x * XT;
  const unsigned tile_id = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  const int4 rec = __ldg(records + tile_id);
  // fits the box + full 16^3 tile
  if ((rec.w & (255 | 2048)) != (1 | 2048)) {
    slow_tile<HAS_CP, HAS_FILL>(a, ta, rec, b, i0, j0, k0);
    return;
  }
  const bool small = DUAL && (rec.w & 4096);
  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
    mbar_expect_tx(bar, (uint32_t)((small ? NBOXS : NBOX) * 4));
    tma_load_4d(box_u32, small ? &tmap_s : &tmap, rec.z, rec.y, rec.x, b * a.C, bar);
  }
  const bool elastic = HAS_CP && (rec.w & 1024);
  const bool masked = HAS_FILL && !(rec.w & 256);  // some tap of the tile may leave the volume
  const float* __restrict__ mp = a.mat + b * 12;
  if (tid >= 32 && tid < 35) {  // tile base in fp64: the only place where volume-sized terms cancel
    const int ax = tid - 32;
    const double t = (double)mp[4 * ax] * i0 + (double)mp[4 * ax + 1] * j0 + (double)mp[4 * ax + 2] * k0 +
                     (double)mp[4 * ax + 3] - (double)(ax == 0 ? rec.x : (ax == 1 ? rec.y : rec.z));
    tbase[ax] = (float)t;
  }
  if (HAS_CP && elastic && tid >= 64 && tid < 96) {
    const int lane = tid - 64;
    auto cell_of = [&](int rel) { return min((int)floorf(__fmul_rn(a.sc_i, (float)(i0 + rel))), a.ni - 1); };
    if (lane < XT) cell_tab[lane] = cell_of(lane);
    bool chg = false;
    if (lane < XT / 2)
      chg = lane == 0 || cell_of(2 * lane) != cell_of(2 * lane - 2) || cell_of(2 * lane + 1) != cell_of(2 * lane - 1);
    const unsigned mask = __ballot_sync(0xffffffffu, chg);
    if (lane == 0) *chg_mask = mask;
  }
  int jrow, kcol;
  lane_column<BOX, 16>(tid, jrow, kcol);
  // an axis of size 1 collapses to u = 0 whatever the matrix says ((size - 1) == 0 in the
  // reference's un-normalise step)
  const float keep[3] = {a.I > 1 ? 1.0f : 0.0f, a.J > 1 ? 1.0f : 0.0f, a.K > 1 ? 1.0f : 0.0f};
  // J/K levels of the displacement lerp of this column (exact ATen order, as the exact walk)
  LerpAxis lj, lk;
  int o00 = 0, o01 = 0, o10 = 0, o11 = 0;
  const float* cps = nullptr;
  if (HAS_CP && elastic) {
    cps = a.cp + (int64_t)b * (a.ni * a.nj * a.nk * 3);
    lj = lerp_axis(a.sc_j, a.nj, j0 + jrow);
    lk = lerp_axis(a.sc_k, a.nk, k0 + kcol);
    o00 = (lj.i0 * a.nk + lk.i0) * 3; o01 = (lj.i0 * a.nk + lk.i1) * 3;
    o10 = (lj.i1 * a.nk + lk.i0) * 3; o11 = (lj.i1 * a.nk + lk.i1) * 3;
  }
  // column constants without displacement: A = T + m1 * jrow + m2 * kcol, B = m0 (every term < 64)
  const float fj = (float)jrow, fk = (float)kcol;
  float Aaff[3], Baff[3];
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    Aaff[ax] = fmaf(__ldg(mp + 4 * ax + 2), fk, __ldg(mp + 4 * ax + 1) * fj);
    Baff[ax] = __ldg(mp + 4 * ax) * keep[ax];
  }
  // J/K-collapsed control values of the first cell: their global loads overlap the TMA transfer
  int cur_cell = -1;
  float r_lo[3] = {0.f, 0.f, 0.f}, r_hi[3] = {0.f, 0.f, 0.f};
  const int plane = HAS_CP ? a.nj * a.nk * 3 : 0;
  auto collapse = [&](int cell) {
    if (cell == cur_cell) return;
    const float* p0 = cps + cell * plane;
    const float* p1 = cps + min(cell + 1, a.ni - 1) * plane;
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
      float a00 = lerp2(lk.l0, __ldg(p0 + o00 + ax), lk.l1, __ldg(p0 + o01 + ax));
      float a01 = lerp2(lk.l0, __ldg(p0 + o10 + ax), lk.l1, __ldg(p0 + o11 + ax));
      r_lo[ax] = lerp2(lj.l0, a00, lj.l1, a01);
      float b00 = lerp2(lk.l0, __ldg(p1 + o00 + ax), lk.l1, __ldg(p1 + o01 + ax));
      float b01 = lerp2(lk.l0, __ldg(p1 + o10 + ax), lk.l1, __ldg(p1 + o11 + ax));
      r_hi[ax] = lerp2(lj.l0, b00, lj.l1, b01);
    }
    cur_cell = cell;
  };
  if (HAS_CP && elastic) collapse(min((int)floorf(__fmul_rn(a.sc_i, (float)i0)), a.ni - 1));
  if (tid == 0) mbar_wait(bar, 0);
  __syncthreads();
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) Aaff[ax] = (Aaff[ax] + tbase[ax]) * keep[ax];

  f2 A0 = pack2(Aaff[0], Aaff[0]), A1 = pack2(Aaff[1], Aaff[1]), A2 = pack2(Aaff[2], Aaff[2]);
  f2 B0 = pack2(Baff[0], Baff[0]), B1 = pack2(Baff[1], Baff[1]), B2 = pack2(Baff[2], Baff[2]);
  unsigned mask = 0, unsafe = 0;
  if (HAS_CP && elastic) mask = *chg_mask;
  // (A, B) of one plane lane inside control cell `cell`: d(rel) = D0 + rel * D1
  auto cell_constants = [&](int cell, float out_a[3], float out_b[3]) {
    collapse(cell);
    const float t0 = fmaf(a.sc_i, (float)i0, -(float)cell);  // lambda of plane rel = 0 (may be < 0)
    float d0[3], d1[3];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
      const float delta = r_hi[ax] - r_lo[ax];
      const float rs = a.affine_first ? ta.rsp_in[ax] : ta.rsp_out[ax];
      d0[ax] = fmaf(t0, delta, r_lo[ax]) * rs;  // voxels
      d1[ax] = a.sc_i * delta * rs;
    }
    if (a.affine_first) {  // q = M p + d / spacing_in
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) {
        out_a[ax] = (Aaff[ax] + d0[ax]) * keep[ax];
        out_b[ax] = (Baff[ax] + d1[ax]) * keep[ax];
      }
    } else {               // q = M (p + d / spacing_out)
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) {
        const float m0 = __ldg(mp + 4 * ax), m1 = __ldg(mp + 4 * ax + 1), m2 = __ldg(mp + 4 * ax + 2);
        out_a[ax] = fmaf(m2, d0[2], fmaf(m1, d0[1], fmaf(m0, d0[0], Aaff[ax]))) * keep[ax];
        out_b[ax] = fmaf(m2, d1[2], fmaf(m1, d1[1], fmaf(m0, d1[0], Baff[ax]))) * keep[ax];
      }
    }
  };

  const int64_t n_out = ta.n_out;
  const int64_t ostride = (int64_t)a.OJ * a.OK;
  float* __restrict__ out0 = (float*)a.dst + (int64_t)b * a.C * n_out +
                             ((int64_t)i0 * a.OJ + (j0 + jrow)) * a.OK + (k0 + kcol);
  // smem byte address of box element idx = (bits(magic + idx) << 2) + kb   (mod 2^32)
  // (the constant comes from the launch arguments: ptxas folds a literal and then re-adds it in
  // front of each of the 16 taps)
  const uint32_t kb = box_u32 - ta.magic_bytes;
  long long pair_bytes = 2 * ostride * (long long)sizeof(float);  // opaque: no per-iteration 64-bit multiply
  asm volatile("" : "+l"(pair_bytes));
  // trapezoid corners of the in-bounds weight per axis, box relative: lo - 1 and hi + 1
  float tz[6];
  tz[0] = (float)(-rec.x - 1); tz[1] = (float)(a.I - rec.x);
  tz[2] = (float)(-rec.y - 1); tz[3] = (float)(a.J - rec.y);
  tz[4] = (float)(-rec.z - 1); tz[5] = (float)(a.K - rec.z);

  for (int c = 0; c < a.C; ++c) {
    if (c > 0) {
      __syncthreads();  // every thread is done with the previous channel's box
      if (tid == 0) {
        mbar_expect_tx(bar, (uint32_t)((small ? NBOXS : NBOX) * 4));
        tma_load_4d(box_u32, small ? &tmap_s : &tmap, rec.z, rec.y, rec.x, b * a.C + c, bar);
        mbar_wait(bar, (uint32_t)(c & 1));
      }
      __syncthreads();
    }
    char* out_a = reinterpret_cast<char*>(out0 + c * n_out);
    char* out_b = out_a + ostride * (long long)sizeof(float);
    const float fill_c = masked ? a.fill[c] : 0.0f;
    f2 rel2 = pack2(0.0f, 1.0f);
    Carry carry;
    carry.u00 = carry.u01 = carry.u10 = carry.u11 = 0.0f;
    carry.up = 0xffffffffu;  // the box was (re)loaded: nothing to reuse
    // pairs [p, p + count) with the column constants as they are; MASKED resolved outside
    auto run = [&](const int p0, const int count, auto masked_tag, auto small_tag) {
      constexpr bool MASKED = decltype(masked_tag)::value;
      constexpr bool SMALL = decltype(small_tag)::value;
#pragma unroll 2
      for (int q = 0; q < count; ++q) {
        float va, vb;
        bool unc_a = false, unc_b = false;
        pair_step<SMALL ? C1S : C1, SMALL ? C2S : C2, MASKED, !HAS_CP>(rel2, A0, A1, A2, B0, B1, B2, kb, tz, fill_c,
                                                                         va, vb, unc_a, unc_b, carry);
        *reinterpret_cast<float*>(out_a) = va;
        *reinterpret_cast<float*>(out_b) = vb;
        if (MASKED) {
          if (unc_a) unsafe |= 1u << (2 * (p0 + q));
          if (unc_b) unsafe |= 2u << (2 * (p0 + q));
        }
        out_a += pair_bytes; out_b += pair_bytes;
        rel2 = add2(rel2, bc(2.0f));
      }
    };
    if constexpr (HAS_CP) {
      // segments of pairs that share their control cells (CTA-uniform): the cell set-up runs
      // between segments, the walk inside a segment is the plain loop
      int p = 0;
      while (p < XT / 2) {
        if ((mask >> p) & 1u) {
          float aa[3], ab[3], ba[3], bb[3];
          const int cell_a = cell_tab[2 * p], cell_b = cell_tab[2 * p + 1];
          cell_constants(cell_a, aa, ba);
          if (cell_b != cell_a) {
            cell_constants(cell_b, ab, bb);
          } else {
#pragma unroll
            for (int ax = 0; ax < 3; ++ax) { ab[ax] = aa[ax]; bb[ax] = ba[ax]; }
          }
          A0 = pack2(aa[0], ab[0]); A1 = pack2(aa[1], ab[1]); A2 = pack2(aa[2], ab[2]);
          B0 = pack2(ba[0], bb[0]); B1 = pack2(ba[1], bb[1]); B2 = pack2(ba[2], bb[2]);
        }
        const unsigned later = (mask >> (p + 1)) << (p + 1);  // next pair that changes cells
        const int stop = later ? __ffs(later) - 1 : XT / 2;
        if (small) {
          if (masked) run(p, stop - p, std::true_type{}, std::true_type{});
          else run(p, stop - p, std::false_type{}, std::true_type{});
        } else {
          if (masked) run(p, stop - p, std::true_type{}, std::false_type{});
          else run(p, stop - p, std::false_type{}, std::false_type{});
        }
        p = stop;
      }
    } else {
#pragma unroll
      for (int p = 0; p < XT / 2; ++p) {
        float va, vb;
        bool unc_a = false, unc_b = false;
        if (masked)
          pair_step<C1, C2, true, !HAS_CP>(rel2, A0, A1, A2, B0, B1, B2, kb, tz, fill_c, va, vb, unc_a, unc_b, carry);
        else
          pair_step<C1, C2, false, !HAS_CP>(rel2, A0, A1, A2, B0, B1, B2, kb, tz, fill_c, va, vb, unc_a, unc_b, carry);
        *reinterpret_cast<float*>(out_a) = va;
        *reinterpret_cast<float*>(out_b) = vb;
        if (HAS_FILL) {
          if (unc_a) unsafe |= 1u << (2 * p);
          if (unc_b) unsafe |= 2u << (2 * p);
        }
        out_a += pair_bytes; out_b += pair_bytes;
        rel2 = add2(rel2, bc(2.0f));
      }
    }
  }
  // voxels on the fill threshold again, all channels, with the exact chain and global-memory
  // taps: the decision is the reference's bit for bit
  if (HAS_FILL && unsafe) exact_fix<HAS_CP, HAS_FILL>(a, ta, b, elastic, i0, unsafe, j0 + jrow, k0 + kcol);
}

template <int BOX, bool HAS_CP>
static void launch_fast_cp(const CUtensorMap& tm, const CUtensorMap& tms, const ResampleArgs& a, const TileArgs& ta,
                           dim3 grid, size_t smem, const int4* records, cudaStream_t st) {
  if (a.fill) {
    cudaFuncSetAttribute(resample_fast_kernel<BOX, HAS_CP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)smem);
    resample_fast_kernel<BOX, HAS_CP, true><<<grid, 256, smem, st>>>(tm, tms, a, ta, records);
  } else {
    cudaFuncSetAttribute(resample_fast_kernel<BOX, HAS_CP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)smem);
    resample_fast_kernel<BOX, HAS_CP, false><<<grid, 256, smem, st>>>(tm, tms, a, ta, records);
  }
  launched();
}

template <int BOX>
static void launch_fast(const CUtensorMap& tm, const CUtensorMap& tms, const ResampleArgs& a, const TileArgs& ta,
                        dim3 grid, size_t smem, const int4* records, cudaStream_t st) {
  if (a.cp) launch_fast_cp<BOX, true>(tm, tms, a, ta, grid, smem, records, st);
  else launch_fast_cp<BOX, false>(tm, tms, a, ta, grid, smem, records, st);
}

// fp32 + trilinear tiles of the launch prepared by launch_resample_tile (tensor map, tile
// arguments, bounds records)
void launch_resample_fast(int box, const CUtensorMap& tm, const CUtensorMap& tm_small, const ResampleArgs& a,
                          const TileArgs& ta, dim3 grid, size_t smem, const int4* records, cudaStream_t st) {
  if (box == 20) launch_fast<20>(tm, tm_small, a, ta, grid, smem, records, st);
  else if (box == 22) launch_fast<22>(tm, tm_small, a, ta, grid, smem, records, st);
  else if (box == 24) launch_fast<24>(tm, tm_small, a, ta, grid, smem, records, st);
  else if (box == 28) launch_fast<28>(tm, tm_small, a, ta, grid, smem, records, st);
  else launch_fast<32>(tm, tm_small, a, ta, grid, smem, records, st);
}

}  // namespace tio

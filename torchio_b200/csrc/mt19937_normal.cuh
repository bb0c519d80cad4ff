// mt19937_normal.cuh — the normal stage of K4a (mt19937.cu) as a device function: one segment
// of torch's CPU `randn` stream, regenerated from its start state and written as normals.
// `mt_normal_kernel` (mt19937.cu) runs it as one CTA per segment; `pass1_normals_kernel`
// (fused_intensity.cu) runs it in five warpgroups of a CTA whose other two run pass 1 of the
// intensity chain.  There is one copy of the arithmetic, so both give the same bits.
#pragma once

#include "common.cuh"

namespace tio {

constexpr int MT_N = 624, MT_M = 397;

__device__ __forceinline__ uint32_t mt_twist(uint32_t a, uint32_t b, uint32_t c) {
  const uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
  return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

__device__ __forceinline__ uint32_t mt_temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  y ^= y >> 18;
  return y;
}

// sin and cos of theta in [0, 2*pi]: quadrant by Cody-Waite reduction with a two-term pi/2,
// then the single-precision minimax polynomials of Cephes sinf/cosf on |r| <= pi/4 (~1e-7
// absolute).  About half the instructions of libm's sincosf (no large-argument path); against
// torch's CPU stream it is as close as a correctly rounded sin/cos (measured on 2^20 draws:
// max |dz| 2.0e-6 either way, 64 % vs 61 % of the normals bit-identical).
__device__ __forceinline__ void sincos_0_2pi(float theta, float& sn, float& cs) {
  const float t = __fmaf_rn(theta, 0.6366197723675814f, 12582912.0f);  // rint(theta * 2/pi) in the mantissa
  const int j = __float_as_int(t);                                      // low bits = quadrant index 0..4
  const float jf = __fsub_rn(t, 12582912.0f);
  float r = __fmaf_rn(jf, -1.5707962512969971f, theta);
  r = __fmaf_rn(jf, -7.549789415861596e-08f, r);
  const float r2 = __fmul_rn(r, r);
  float ps = __fmaf_rn(r2, -1.9515295891e-4f, 8.3321608736e-3f);
  ps = __fmaf_rn(ps, r2, -1.6666654611e-1f);
  const float s = __fmaf_rn(__fmul_rn(ps, r2), r, r);
  float pc = __fmaf_rn(r2, 2.443315711809948e-5f, -1.388731625493765e-3f);
  pc = __fmaf_rn(pc, r2, 4.166664568298827e-2f);
  const float c = __fmaf_rn(__fmul_rn(pc, r2), r2, __fmaf_rn(r2, -0.5f, 1.0f));
  const bool swap = j & 1;
  const float a = swap ? c : s, b = swap ? s : c;
  sn = (j & 2) ? -a : a;
  cs = ((j + 1) & 2) ? -b : b;
}

// One pair of torch's normal_fill: words a = u[j] and b = u[j+8] of a 16-group ->
// z[j] = r cos th, z[j+8] = r sin th.  The arithmetic fixes every output bit of the
// stream; keep it as it is.
__device__ __forceinline__ void mt_box_muller(uint32_t a, uint32_t b, float& zc, float& zs) {
  const float u1 = (float)(mt_temper(a) & 0xffffffu) * (1.0f / 16777216.0f);
  const float u2 = (float)(mt_temper(b) & 0xffffffu) * (1.0f / 16777216.0f);
  float radius;  // sqrt(-2 log(1 - u1)); MUFU.SQRT (<= 1 ulp) instead of the IEEE sequence
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(radius) : "f"(-2.0f * logf(1.0f - u1)));
  const float theta = (float)(6.283185307179586 * (double)u2);  // 2.0f * pi<double> * u2
  float sn, cs;
  sincos_0_2pi(theta, sn, cs);
  zc = radius * cs;
  zs = radius * sn;
}

// named barriers with immediate ids, so that ptxas reserves only the ones used
template <int ID, int COUNT>
__device__ __forceinline__ void mt_bar_sync() {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(COUNT) : "memory");
}
template <int ID, int COUNT>
__device__ __forceinline__ void mt_bar_arrive() {
  asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(COUNT) : "memory");
}

// Normal stage layout.  MT_THREADS threads emit stream words [q*L, (q+1)*L) of segment q
// intersected with [offset, offset+n) as z[word - offset].  Warp-specialised:
//   producers (8 warps) regenerate the segment's 624-word blocks in the recurrence's three
//     dependency waves (227, 227, 170 words), synchronised among themselves only;
//   consumers (10 warps) temper and transform them.  A consumer thread owns one "item" per
//     round: half of a 16-group (pairs j0..j0+3, j0 = 0 or 4), i.e. four independent
//     Box-Muller chains, read with two LDS.128 and written with two 16-byte stores.
// Blocks pass in rounds of MT_ROUND blocks (= 312 items, one per consumer thread) through a
// ring of two rounds: producers fill one round while consumers drain the other.  Named
// barriers: MT_BAR_PROD among producers, MT_BAR_FULL + r and MT_BAR_EMPTY + r (round buffer
// r) between the two roles.  Producers wait for consumers only when both buffers are full.
constexpr int MT_ROUND = 4;                          // blocks per round
constexpr int MT_RING = 2 * MT_ROUND;                // blocks in shared memory (19.5 KB)
constexpr int MT_ITEMS = MT_ROUND * MT_N / 8;        // 312 items per round
constexpr int MT_PRODUCERS = 256;                    // >= 227 (one wave's width), whole warps
constexpr int MT_CONSUMERS = (MT_ITEMS + 31) / 32 * 32;  // 320
constexpr int MT_THREADS = MT_PRODUCERS + MT_CONSUMERS;  // 576
constexpr int MT_BAR_PROD = 1, MT_BAR_FULL = 2, MT_BAR_EMPTY = 4;  // ids 1..5; none uses barrier 0

// `ring`: MT_RING * MT_N words of shared memory, 16-byte aligned (block b in slot b % MT_RING);
// `tid` in [0, MT_THREADS).  Every barrier is balanced within the call, but the last consumers
// may still read the ring when the producers return: a caller that runs a second segment puts a
// barrier over the MT_THREADS threads between the two.
__device__ __forceinline__ void mt_normal_segment(uint32_t* __restrict__ ring, const int tid,
                                                  const uint32_t* __restrict__ states, const int q,
                                                  unsigned long long L, unsigned long long offset,
                                                  unsigned long long n, float* __restrict__ z) {
  const unsigned long long seg_begin = (unsigned long long)q * L;
  const unsigned long long lo = max(seg_begin, offset);
  const unsigned long long hi = min(seg_begin + L, offset + n);
  if (lo >= hi) return;  // uniform over the MT_THREADS threads
  // positions relative to the segment start fit 32 bits (L <= 2^30); lo_rel and hi_rel are
  // multiples of 16, so each 16-group lies wholly inside or wholly outside the window
  const int lo_rel = (int)(lo - seg_begin), hi_rel = (int)(hi - seg_begin);
  const int rounds = ((hi_rel + MT_N - 1) / MT_N + MT_ROUND - 1) / MT_ROUND;
  if (tid < MT_PRODUCERS) {
    constexpr int W = MT_N - MT_M;  // 227
    // the start window W_{qL} plays block -1
    const uint32_t* w = states + (size_t)q * MT_N;
    uint32_t* start = ring + (MT_RING - 1) * MT_N;
    for (int t = tid; t < MT_N; t += MT_PRODUCERS) start[t] = w[t];
    mt_bar_sync<MT_BAR_PROD, MT_PRODUCERS>();
    for (int r = 0; r < rounds; ++r) {
      if (r >= 2) {  // consumers are done with round r-2
        if (r & 1) mt_bar_sync<MT_BAR_EMPTY + 1, MT_THREADS>();
        else mt_bar_sync<MT_BAR_EMPTY, MT_THREADS>();
      }
      for (int i = 0; i < MT_ROUND; ++i) {
        const int b = r * MT_ROUND + i;
        const uint32_t* cur = ring + ((b + MT_RING - 1) % MT_RING) * MT_N;
        uint32_t* nxt = ring + (b % MT_RING) * MT_N;
        // wave 0: k in [0,227): x[k], x[k+1], x[k+397] all in the previous block
        if (tid < W) nxt[tid] = mt_twist(cur[tid], cur[tid + 1], cur[tid + MT_M]);
        mt_bar_sync<MT_BAR_PROD, MT_PRODUCERS>();
        // wave 1: k in [227,454): x[k+397] = new word k-227
        if (tid < W) nxt[W + tid] = mt_twist(cur[W + tid], cur[W + tid + 1], nxt[tid]);
        mt_bar_sync<MT_BAR_PROD, MT_PRODUCERS>();
        // wave 2: k in [454,624): x[k+397] = new word k-227; x[624] = new word 0
        if (tid < MT_N - 2 * W) {
          const int k = 2 * W + tid;
          const uint32_t c = (k + 1 < MT_N) ? cur[k + 1] : nxt[0];
          nxt[k] = mt_twist(cur[k], c, nxt[k - W]);
        }
        mt_bar_sync<MT_BAR_PROD, MT_PRODUCERS>();
      }
      if (r & 1) mt_bar_arrive<MT_BAR_FULL + 1, MT_THREADS>();
      else mt_bar_arrive<MT_BAR_FULL, MT_THREADS>();
    }
  } else {
    const int c = tid - MT_PRODUCERS;
    const int blk = c / (MT_N / 8), item = c % (MT_N / 8);  // block of the round, item in the block
    const int word = 16 * (item >> 1) + 4 * (item & 1);      // u[j0] of the item's group
    const long long seg_to_z = (long long)seg_begin - (long long)offset;  // < 0 only in the first segment
    // 16-byte stores need z 16-byte aligned (every word offset below is a multiple of 4)
    const bool vec = ((reinterpret_cast<uintptr_t>(z) & 15) == 0);
    for (int r = 0; r < rounds; ++r) {
      if (r & 1) mt_bar_sync<MT_BAR_FULL + 1, MT_THREADS>();
      else mt_bar_sync<MT_BAR_FULL, MT_THREADS>();
      const int b = r * MT_ROUND + blk;
      const int group = b * MT_N + (word & ~15);  // position of the group relative to the segment
      if (c < MT_ITEMS && group >= lo_rel && group < hi_rel) {
        const uint32_t* x = ring + (b % MT_RING) * MT_N + word;
        const uint4 a = *reinterpret_cast<const uint4*>(x);
        const uint4 s = *reinterpret_cast<const uint4*>(x + 8);
        float4 zc, zs;
        mt_box_muller(a.x, s.x, zc.x, zs.x);
        mt_box_muller(a.y, s.y, zc.y, zs.y);
        mt_box_muller(a.z, s.z, zc.z, zs.z);
        mt_box_muller(a.w, s.w, zc.w, zs.w);
        float* zp = z + (seg_to_z + b * MT_N + word);  // >= 0: group >= lo_rel
        if (vec) {
          *reinterpret_cast<float4*>(zp) = zc;
          *reinterpret_cast<float4*>(zp + 8) = zs;
        } else {
          zp[0] = zc.x; zp[1] = zc.y; zp[2] = zc.z; zp[3] = zc.w;
          zp[8] = zs.x; zp[9] = zs.y; zp[10] = zs.z; zp[11] = zs.w;
        }
      }
      if (r + 2 < rounds) {  // producers wait on it
        if (r & 1) mt_bar_arrive<MT_BAR_EMPTY + 1, MT_THREADS>();
        else mt_bar_arrive<MT_BAR_EMPTY, MT_THREADS>();
      }
    }
  }
}

// Host side of the replay up to the normal stage (mt19937.cu): checks the window, then seeds
// and jumps, leaving the start state W_{qL} of every segment q the window [offset, offset+n)
// touches in `workspace` (tio_randn_mt19937_workspace_bytes).  q_lo, q_hi: those segments.
int mt_start_states(uint64_t seed, uint64_t offset, uint64_t n, const void* table, void* workspace,
                    size_t workspace_bytes, cudaStream_t st, const char* who, int* q_lo, int* q_hi);

}  // namespace tio

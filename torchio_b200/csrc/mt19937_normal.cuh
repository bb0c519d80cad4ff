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

// Normal stage layout.  MT_THREADS threads emit the 16-groups of a draw whose first word lies in
// segment q (stream words [q*L, (q+1)*L)).  A draw of n normals at stream word s is torch's
// normal_fill: groups of 16 words [s + 16g, s + 16g + 16) give outputs [16g, 16g + 16) (u[j] and
// u[j+8] pair up); when n % 16 != 0 a tail group of the 16 words [s + n, s + n + 16) then gives
// outputs [n - 16, n), overwriting what the last groups wrote there.  Only outputs [lo, hi) of
// the draw are written, output i to z[i - lo].  A group belongs to the segment holding its first
// word, so the last groups of a segment may read up to 15 words of the next one.
// Warp-specialised:
//   producers (8 warps) regenerate the segment's 624-word blocks in the recurrence's three
//     dependency waves (227, 227, 170 words), synchronised among themselves only;
//   consumers (10 warps) temper and transform them.  A consumer thread owns one "item" per
//     round: half of a 16-group (pairs j0..j0+3, j0 = 0 or 4), i.e. four independent
//     Box-Muller chains, read with two LDS.128 and written with two 16-byte stores where the
//     draw's alignment allows (scalar accesses otherwise).  Each block holds the first words of
//     39 groups; two of the otherwise idle consumers take the tail group.
// Blocks pass in rounds of MT_ROUND blocks (= 312 items, one per consumer thread) through a
// ring of two rounds: producers fill one round while consumers drain the other.  A round's
// blocks are contiguous and followed by the first 16 words of the next block, so a group that
// straddles two blocks, or two rounds, reads consecutive words.  Named barriers: MT_BAR_PROD
// among producers, MT_BAR_FULL + r and MT_BAR_EMPTY + r (round buffer r) between the two roles.
// Producers wait for consumers only when both buffers are full.
constexpr int MT_ROUND = 4;                          // blocks per round
constexpr int MT_RING = 2 * MT_ROUND;                // blocks in the ring
constexpr int MT_ROUND_WORDS = MT_ROUND * MT_N + 16;  // a round's blocks, then the next block's first 16 words
constexpr int MT_RING_WORDS = 2 * MT_ROUND_WORDS;    // 5024 words (19.6 KB)
constexpr int MT_ITEMS = MT_ROUND * MT_N / 8;        // 312 items per round
constexpr int MT_PRODUCERS = 256;                    // >= 227 (one wave's width), whole warps
constexpr int MT_CONSUMERS = (MT_ITEMS + 31) / 32 * 32;  // 320
constexpr int MT_THREADS = MT_PRODUCERS + MT_CONSUMERS;  // 576
constexpr int MT_BAR_PROD = 1, MT_BAR_FULL = 2, MT_BAR_EMPTY = 4;  // ids 1..5; none uses barrier 0
static_assert(MT_CONSUMERS >= MT_ITEMS + 2, "the tail group needs two spare consumers");

// block b >= -1 of the segment (block -1: the start window) in the ring
__device__ __forceinline__ uint32_t* mt_block(uint32_t* ring, int b) {
  const int slot = (b + MT_RING) % MT_RING;
  return ring + (slot / MT_ROUND) * MT_ROUND_WORDS + (slot % MT_ROUND) * MT_N;
}

// segment-relative positions, clamped to a range that keeps every comparison below exact
__device__ __forceinline__ int mt_rel(long long v, unsigned long long L) {
  return (int)min(max(v, -32ll), (long long)L + 32);
}

// `ring`: MT_RING_WORDS words of shared memory, 16-byte aligned; `tid` in [0, MT_THREADS).
// The draw: n >= 16 normals at stream word s, outputs [lo, hi) with lo < hi <= n.
// WINDOW = false compiles the stage for the [0, n) window of an aligned draw only (s and n
// multiples of 16, lo = 0, hi = n, z 16-byte aligned): no group straddles a block, there is no
// tail, and every item takes the 16-byte path, so the consumer loop carries none of the window's
// bounds (pass1_normals_kernel, where this stage is the longer of the two roles).  Every
// barrier is balanced within the call, but the last consumers may still read the ring when the
// producers return: a caller that runs a second segment puts a barrier over the MT_THREADS
// threads between the two.
template <bool WINDOW>
__device__ __forceinline__ void mt_normal_segment(uint32_t* __restrict__ ring, const int tid,
                                                  const uint32_t* __restrict__ states, const int q,
                                                  unsigned long long L, unsigned long long s,
                                                  unsigned long long n, unsigned long long lo,
                                                  unsigned long long hi, float* __restrict__ z) {
  constexpr int RW = MT_ROUND * MT_N;  // stream words per round
  // positions relative to the segment start fit 32 bits (L <= 2^30).  A main group at relative
  // position p writes outputs [p + ofs, p + ofs + 16); the tail's outputs [n - 16, n) sit at
  // relative positions [tail_p - 16, tail_p).  Outputs [lo, hi) are relative [lo_rel, *_hi).
  const long long ofs = (long long)q * L - (long long)s;
  const unsigned long long kept = (n & 15) ? n - 16 : n;  // outputs of main groups the tail leaves
  const int lo_rel = mt_rel((long long)lo - ofs, L);
  const int main_hi = mt_rel((long long)min(hi, kept) - ofs, L);
  const int tail_hi = mt_rel((long long)hi - ofs, L);
  const long long tail_p = (long long)(s + n) - (long long)q * L;
  const bool tail = WINDOW && (n & 15) && hi > n - 16 && tail_p >= 0 && tail_p < (long long)L;
  const int main_end = min(main_hi, (int)L);  // main groups of the segment start below it
  int rounds = (main_end > 0 && main_end + 15 > lo_rel) ? (main_end + RW - 1) / RW : 0;
  if (tail) rounds = max(rounds, (int)tail_p / RW + 1);
  if (rounds == 0) return;  // uniform over the MT_THREADS threads
  if (tid < MT_PRODUCERS) {
    constexpr int W = MT_N - MT_M;  // 227
    const uint32_t* w = states + (size_t)q * MT_N;
    uint32_t* start = mt_block(ring, -1);
    for (int t = tid; t < MT_N; t += MT_PRODUCERS) start[t] = w[t];
    mt_bar_sync<MT_BAR_PROD, MT_PRODUCERS>();
    for (int r = 0; r < rounds; ++r) {
      if (r >= 2) {  // consumers are done with round r-2
        if (r & 1) mt_bar_sync<MT_BAR_EMPTY + 1, MT_THREADS>();
        else mt_bar_sync<MT_BAR_EMPTY, MT_THREADS>();
      }
      for (int i = 0; i < MT_ROUND; ++i) {
        const int b = r * MT_ROUND + i;
        const uint32_t* cur = mt_block(ring, b - 1);
        uint32_t* nxt = mt_block(ring, b);
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
        } else if (WINDOW && i == MT_ROUND - 1 && tid < MT_N - 2 * W + 16) {
          // after the round's last block: word k < 16 of the next block (wave 0 of that block,
          // whose inputs nxt[k], nxt[k+1], nxt[k+397] came from waves 0 and 1)
          const int k = tid - (MT_N - 2 * W);
          nxt[MT_N + k] = mt_twist(nxt[k], nxt[k + 1], nxt[k + MT_M]);
        }
        mt_bar_sync<MT_BAR_PROD, MT_PRODUCERS>();
      }
      if (r & 1) mt_bar_arrive<MT_BAR_FULL + 1, MT_THREADS>();
      else mt_bar_arrive<MT_BAR_FULL, MT_THREADS>();
    }
  } else {
    const int c = tid - MT_PRODUCERS;
    // the item's group: c < MT_ITEMS: block c / 78 of each round, group (c % 78) / 2 of the block,
    // every round; c = MT_ITEMS + h: the tail group, once.  In round r it starts at relative
    // position p = r * RW + at and is the item's iff p lies in [p_min, p_max).  The item's output
    // j (0..3, 8..11) is at relative position p + j + to_out and is written iff that lies in
    // [lo_rel, end), i.e. iff p + j lies in [w_lo, w_hi).
    const int half = 4 * (c & 1);  // j0 of the item (78 items per block: c and item have one parity)
    int at, p_min, p_max, shift, end;
    if (c < MT_ITEMS) {
      at = (c / (MT_N / 8)) * MT_N + (WINDOW ? (int)(s & 15) : 0) + 16 * ((c % (MT_N / 8)) >> 1);
      p_min = lo_rel - 15;
      p_max = main_end;
      shift = 0;
      end = main_hi;
    } else {
      at = (int)tail_p % RW;
      p_min = (tail && c < MT_ITEMS + 2) ? (int)tail_p : 0;
      p_max = (tail && c < MT_ITEMS + 2) ? (int)tail_p + 1 : 0;
      shift = 16;
      end = tail_hi;
    }
    const int to_out = half - shift, w_lo = lo_rel - to_out, w_hi = end - to_out;
    float* const zq = z + (ofs - (long long)lo + to_out);  // the item's output j of p lands at zq[p + j]
    // 16-byte ring loads and z stores where the item's words and outputs allow (RW % 4 == 0: the
    // same in every round)
    const bool ld128 = !WINDOW || ((at + half) & 3) == 0;
    const bool st128 = (reinterpret_cast<uintptr_t>(zq + at) & 15) == 0;
    for (int r = 0; r < rounds; ++r) {
      if (r & 1) mt_bar_sync<MT_BAR_FULL + 1, MT_THREADS>();
      else mt_bar_sync<MT_BAR_FULL, MT_THREADS>();
      const int p = r * RW + at;
      if (p >= p_min && p < p_max) {
        const uint32_t* x = ring + (r & 1) * MT_ROUND_WORDS + at + half;
        uint4 a, b;
        if (ld128) {
          a = *reinterpret_cast<const uint4*>(x);
          b = *reinterpret_cast<const uint4*>(x + 8);
        } else {
          a = make_uint4(x[0], x[1], x[2], x[3]);
          b = make_uint4(x[8], x[9], x[10], x[11]);
        }
        float4 zc, zs;
        mt_box_muller(a.x, b.x, zc.x, zs.x);
        mt_box_muller(a.y, b.y, zc.y, zs.y);
        mt_box_muller(a.z, b.z, zc.z, zs.z);
        mt_box_muller(a.w, b.w, zc.w, zs.w);
        float* zp = zq + p;
        if (!WINDOW || (st128 && p >= w_lo && p + 12 <= w_hi)) {
          *reinterpret_cast<float4*>(zp) = zc;
          *reinterpret_cast<float4*>(zp + 8) = zs;
        } else {
          const float v[8] = {zc.x, zc.y, zc.z, zc.w, zs.x, zs.y, zs.z, zs.w};
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            const int j = (t & 3) + (t & 4) * 2;  // j0 + t, then j0 + 8 + t
            if (p + j >= w_lo && p + j < w_hi) zp[j] = v[t];
          }
        }
      }
      if (r + 2 < rounds) {  // producers wait on it
        if (r & 1) mt_bar_arrive<MT_BAR_EMPTY + 1, MT_THREADS>();
        else mt_bar_arrive<MT_BAR_EMPTY, MT_THREADS>();
      }
    }
  }
}

// Host side of the replay up to the normal stage (mt19937.cu): seeds and jumps, leaving the
// start state W_{qL} of every segment q in [q_lo, q_hi) in `workspace`, the segments that hold
// stream words [first_word, last_word] (the first words of the groups a draw needs).  Checks
// the table's reach and the workspace size ((q_hi + kS1) states).
int mt_start_states(uint64_t seed, uint64_t first_word, uint64_t last_word, const void* table,
                    void* workspace, size_t workspace_bytes, cudaStream_t st, const char* who,
                    int* q_lo, int* q_hi);

}  // namespace tio

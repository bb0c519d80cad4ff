// mt19937.cu — K4a: device replay of torch's CPU `randn` stream.
//
// torch.randn(shape, generator=CPU mt19937(seed)) (the reference's noise source,
// transforms/intensity/noise.py:166-178) for n >= 16 is ATen's normal_fill:
//   u[t]  = (mt19937_word[t] & 0xFFFFFF) * 2^-24                t = 0..n-1
//   per 16-block, j = 0..7:  r = sqrt(-2 log(1 - u[j])),  th = 2*pi*u[j+8]
//                            z[j] = r cos th,  z[j+8] = r sin th
// one sequential stream per call.  Here the stream is cut into segments of
// L = 2^21 words (mt19937_layout.h); segment start states come from jump-ahead
// polynomials (mt19937_jump.cpp): seed -> W_0, coarse jumps W_0 -> W_{m*S2*L}, fine
// jumps -> W_{(S2*m+r)L}; then one CTA per segment regenerates its 624-word blocks
// (three dependency waves of <= 227 words) and emits normals.
//
// Window W_t = (x[t], ..., x[t+623]) of the word recurrence
//   x[k+624] = x[k+397] ^ twist(x[k], x[k+1]);  stream word t = temper(x[624+t]).
#include "common.cuh"
#include "mt19937_layout.h"

namespace tio {

constexpr int MT_N = 624, MT_M = 397, MT_DEG = 19937;
constexpr int MT_SEQ = MT_DEG + MT_N;  // words needed to apply a jump polynomial
constexpr int MT_OFFS = (MT_SEQ + 7) / 4 * 4;  // 16-byte aligned start of the staged offsets

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

// states[q] = W_{q*L}; slot 0 is the seeded state.
__global__ void mt_seed_kernel(uint32_t seed, uint32_t* __restrict__ states) {
  if (threadIdx.x == 0) {
    uint32_t v = seed;
    states[0] = v;
    for (int j = 1; j < MT_N; ++j) {
      v = 1812433253u * (v ^ (v >> 30)) + (uint32_t)j;
      states[j] = v;
    }
  }
}

// dst window = g(F) src window, g given as ascending set-bit positions.
//   coarse level (fine == 0): job i -> m = first + i: W_0 -> W_{m*S2*L}, slot (S2-1)+(m-1)
//   fine level   (fine == 1): job i -> q = first + i, r = q % S2 (r == 0: nothing to do):
//                             W_{(q-r)L} -> W_{qL}, slot r-1
// Each job is split over `parts` CTAs (blockIdx.x = job * parts + part), each taking a
// contiguous slice of the set bits.  With parts > 1 the slices are XORed into a zeroed
// dst with atomicXor: the coarse level has only one job per S2 segments, so without the
// split it would occupy a few SMs while the rest of the GPU waits for it.
struct MtJob { int src, dst, slot; };

__global__ void __launch_bounds__(640)
mt_jump_kernel(uint32_t* __restrict__ states, const uint16_t* __restrict__ polys, int stride,
               int first, int S2, int fine, int parts) {
  extern __shared__ __align__(16) uint32_t seq[];  // MT_SEQ words (+pad), then 2048 staged byte offsets
  uint32_t* offs = seq + MT_OFFS;
  const int job_idx = (int)blockIdx.x / parts, part = (int)blockIdx.x % parts;
  MtJob job;
  if (fine) {
    const int q = first + job_idx, r = q % S2;
    if (r == 0) return;
    job = MtJob{q - r, q, r - 1};
  } else {
    const int m = first + job_idx;
    job = MtJob{0, m * S2, (S2 - 1) + (m - 1)};
  }
  const int tid = threadIdx.x;
  const uint32_t* src = states + (size_t)job.src * MT_N;
  for (int t = tid; t < MT_N; t += blockDim.x) seq[t] = src[t];
  __syncthreads();
  // extend the sequence: 227 new words per dependency wave
  for (int base = 0; base + MT_N < MT_SEQ; base += MT_N - MT_M) {
    const int k = base + tid;
    if (tid < MT_N - MT_M && k + MT_N < MT_SEQ)
      seq[k + MT_N] = mt_twist(seq[k], seq[k + 1], seq[k + MT_M]);
    __syncthreads();
  }
  const uint16_t* p = polys + (size_t)job.slot * stride;
  const uint32_t count = p[0] | ((uint32_t)p[1] << 16);
  const uint32_t t_begin = (uint32_t)((uint64_t)count * part / parts);
  const uint32_t t_end = (uint32_t)((uint64_t)count * (part + 1) / parts);
  // out[tid] = XOR over the polynomial's set bits i of seq[i + tid].  The loop is bound
  // by shared-memory wavefronts (one per warp per term), so everything else is kept off
  // the LSU: offsets arrive four per broadcast LDS.128, pre-scaled to bytes.
  const char* mine = reinterpret_cast<const char*>(seq + (tid < MT_N ? tid : 0));
  uint32_t acc = 0;
  for (uint32_t c0 = t_begin; c0 < t_end; c0 += 2048) {
    const uint32_t chunk = min(2048u, t_end - c0);
    for (uint32_t t = tid; t < chunk; t += blockDim.x) offs[t] = (uint32_t)p[2 + c0 + t] << 2;
    __syncthreads();
    if (tid < MT_N) {
      const uint4* o4 = reinterpret_cast<const uint4*>(offs);
      const uint32_t quads = chunk >> 2;
#pragma unroll 4
      for (uint32_t t = 0; t < quads; ++t) {
        const uint4 o = o4[t];
        acc ^= *reinterpret_cast<const uint32_t*>(mine + o.x) ^ *reinterpret_cast<const uint32_t*>(mine + o.y);
        acc ^= *reinterpret_cast<const uint32_t*>(mine + o.z) ^ *reinterpret_cast<const uint32_t*>(mine + o.w);
      }
      for (uint32_t t = quads << 2; t < chunk; ++t) acc ^= *reinterpret_cast<const uint32_t*>(mine + offs[t]);
    }
    __syncthreads();
  }
  if (tid < MT_N) {
    uint32_t* dst = states + (size_t)job.dst * MT_N + tid;
    if (parts == 1) *dst = acc;
    else atomicXor(dst, acc);
  }
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

// Normal kernel layout.  One CTA per segment q emits stream words [q*L, (q+1)*L)
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
constexpr int MT_BAR_PROD = 1, MT_BAR_FULL = 2, MT_BAR_EMPTY = 4;

__global__ void __launch_bounds__(MT_THREADS, 2)
mt_normal_kernel(const uint32_t* __restrict__ states, int q_first, unsigned long long L,
                 unsigned long long offset, unsigned long long n, float* __restrict__ z) {
  __shared__ __align__(16) uint32_t ring[MT_RING * MT_N];  // block b in slot b % MT_RING
  const int tid = threadIdx.x;
  const int q = q_first + blockIdx.x;
  const unsigned long long seg_begin = (unsigned long long)q * L;
  const unsigned long long lo = max(seg_begin, offset);
  const unsigned long long hi = min(seg_begin + L, offset + n);
  if (lo >= hi) return;  // CTA-uniform
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

}  // namespace tio

using namespace tio;

constexpr uint64_t MT_L = 1ull << tio_mt::kLog2L;

// workspace: the segment start states W_{qL}, q < q_hi
extern "C" size_t tio_randn_mt19937_workspace_bytes(uint64_t offset, uint64_t n) {
  const uint64_t q_hi = (offset + n + MT_L - 1) / MT_L;
  return (size_t)(q_hi + tio_mt::kS1) * MT_N * 4;
}

extern "C" int tio_randn_mt19937(uint64_t seed, uint64_t offset, uint64_t n, float* z,
                                 const void* table, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  TIO_CHECK_ARG(z && table && workspace, "tio_randn_mt19937: null pointer");
  TIO_CHECK_ARG(n >= 16 && (n % 16) == 0 && (offset % 16) == 0,
                "tio_randn_mt19937: n and offset must be multiples of 16 (n >= 16)");
  const int S2 = tio_mt::kS2, S1 = tio_mt::kS1, stride = tio_mt::kStride;
  const uint64_t q_lo = offset / MT_L, q_hi = (offset + n + MT_L - 1) / MT_L;  // segments [q_lo, q_hi)
  TIO_CHECK_ARG(q_hi <= (uint64_t)S1 * S2, "tio_randn_mt19937: stream position beyond %d segments", S1 * S2);
  TIO_CHECK_ARG(workspace_bytes >= tio_randn_mt19937_workspace_bytes(offset, n),
                "tio_randn_mt19937: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  uint32_t* states = (uint32_t*)workspace;
  const uint16_t* polys = (const uint16_t*)((const char*)table + tio_mt::kHeaderBytes);
  mt_seed_kernel<<<1, 32, 0, st>>>((uint32_t)seed, states);
  const size_t jump_smem = (size_t)(MT_OFFS + 2048) * 4;
  cudaFuncSetAttribute(mt_jump_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)jump_smem);
  const int m_lo = (int)(q_lo / S2), m_hi = (int)((q_hi - 1) / S2);
  const int m_first = m_lo > 1 ? m_lo : 1;
  if (m_hi >= m_first) {
    // coarse jobs XOR their slices into zeroed start states W_{m*S2*L}
    constexpr int kCoarseParts = 8;
    const size_t pitch = (size_t)S2 * MT_N * 4;
    cudaMemset2DAsync(states + (size_t)m_first * S2 * MT_N, pitch, 0, MT_N * 4, m_hi - m_first + 1, st);
    mt_jump_kernel<<<(m_hi - m_first + 1) * kCoarseParts, 640, jump_smem, st>>>(states, polys, stride, m_first,
                                                                             S2, 0, kCoarseParts);
  }
  mt_jump_kernel<<<(unsigned)(q_hi - q_lo), 640, jump_smem, st>>>(states, polys, stride, (int)q_lo, S2, 1, 1);
  mt_normal_kernel<<<(unsigned)(q_hi - q_lo), MT_THREADS, 0, st>>>(states, (int)q_lo, MT_L, offset, n, z);
  TIO_CHECK_LAUNCH();
  return 0;
}

// mt19937.cu — K4a: device replay of torch's CPU `randn` stream.
//
// torch.randn(shape, generator=CPU mt19937(seed)) (the reference's noise source,
// transforms/intensity/noise.py:166-178) for n >= 16 is ATen's normal_fill:
//   u[t]  = (mt19937_word[s + t] & 0xFFFFFF) * 2^-24            t = 0..n-1
//   per 16-block, j = 0..7:  r = sqrt(-2 log(1 - u[j])),  th = 2*pi*u[j+8]
//                            z[j] = r cos th,  z[j+8] = r sin th
//   n % 16 != 0: 16 more words u[n..n+16) as one more block, written to z[n-16..n)
// where s is the number of words the generator used before; the calls of one generator
// continue one sequential stream.  A draw may start at any word and only a window of its
// outputs may be wanted (tio_randn_mt19937_window).  Here the stream is cut into segments of
// L = 2^21 words (mt19937_layout.h); segment start states come from jump-ahead
// polynomials (mt19937_jump.cpp): seed -> W_0, coarse jumps W_0 -> W_{m*S2*L}, fine
// jumps -> W_{(S2*m+r)L}; then one CTA per segment regenerates its 624-word blocks
// (three dependency waves of <= 227 words) and emits the normals of the 16-blocks whose
// first word lies in the segment.
//
// Window W_t = (x[t], ..., x[t+623]) of the word recurrence
//   x[k+624] = x[k+397] ^ twist(x[k], x[k+1]);  stream word t = temper(x[624+t]).
#include "common.cuh"
#include "mt19937_layout.h"
#include "mt19937_normal.cuh"

namespace tio {

constexpr int MT_DEG = 19937;
constexpr int MT_SEQ = MT_DEG + MT_N;  // words needed to apply a jump polynomial
constexpr int MT_OFFS = (MT_SEQ + 7) / 4 * 4;  // 16-byte aligned start of the staged offsets

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

// One CTA per segment q (the stage itself: mt19937_normal.cuh)
__global__ void __launch_bounds__(MT_THREADS, 2)
mt_normal_kernel(const uint32_t* __restrict__ states, int q_first, unsigned long long L, unsigned long long s,
                 unsigned long long n, unsigned long long lo, unsigned long long hi, float* __restrict__ z) {
  __shared__ __align__(16) uint32_t ring[MT_RING_WORDS];
  mt_normal_segment<true>(ring, (int)threadIdx.x, states, q_first + (int)blockIdx.x, L, s, n, lo, hi, z);
}

constexpr uint64_t MT_L = 1ull << tio_mt::kLog2L;
constexpr uint64_t MT_MAX_WORDS = (uint64_t)tio_mt::kS1 * tio_mt::kS2 * MT_L;  // the table's reach

int mt_start_states(uint64_t seed, uint64_t first_word, uint64_t last_word, const void* table,
                    void* workspace, size_t workspace_bytes, cudaStream_t st, const char* who, int* q_lo_out,
                    int* q_hi_out) {
  TIO_CHECK_ARG(table && workspace, "%s: null table or workspace", who);
  const int S2 = tio_mt::kS2, S1 = tio_mt::kS1, stride = tio_mt::kStride;
  const uint64_t q_lo = first_word / MT_L, q_hi = last_word / MT_L + 1;  // segments [q_lo, q_hi)
  TIO_CHECK_ARG(q_hi <= (uint64_t)S1 * S2, "%s: stream position beyond %d segments", who, S1 * S2);
  TIO_CHECK_ARG(workspace_bytes >= (size_t)(q_hi + S1) * MT_N * 4, "%s: workspace too small", who);
  uint32_t* states = (uint32_t*)workspace;
  const uint16_t* polys = (const uint16_t*)((const char*)table + tio_mt::kHeaderBytes);
  mt_seed_kernel<<<1, 32, 0, st>>>((uint32_t)seed, states);
  launched();
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
    launched();
  }
  mt_jump_kernel<<<(unsigned)(q_hi - q_lo), 640, jump_smem, st>>>(states, polys, stride, (int)q_lo, S2, 1, 1);
  launched();
  *q_lo_out = (int)q_lo;
  *q_hi_out = (int)q_hi;
  return 0;
}

}  // namespace tio

using namespace tio;

// workspace: the segment start states W_{qL}, q < q_hi
extern "C" size_t tio_randn_mt19937_workspace_bytes(uint64_t offset, uint64_t n) {
  const uint64_t q_hi = (offset + n + MT_L - 1) / MT_L;
  return (size_t)(q_hi + tio_mt::kS1) * MT_N * 4;
}

// q_hi = the segment of the last group's first word, + 1: the tail's s + n, or s + n - 16
extern "C" size_t tio_randn_mt19937_window_workspace_bytes(uint64_t offset, uint64_t n) {
  const uint64_t last = offset + ((n % 16) ? n : n - 16);
  return (size_t)(last / MT_L + 1 + tio_mt::kS1) * MT_N * 4;
}

extern "C" int tio_randn_mt19937_window(uint64_t seed, uint64_t offset, uint64_t n, uint64_t lo, uint64_t hi,
                                        float* z, const void* table, void* workspace, size_t workspace_bytes,
                                        void* stream) {
  const char* who = "tio_randn_mt19937_window";
  TIO_CHECK_ARG(z, "%s: null pointer", who);
  TIO_CHECK_ARG(n >= 16 && lo < hi && hi <= n, "%s: needs n >= 16 and lo < hi <= n", who);
  const uint64_t words = n + ((n % 16) ? 16 : 0);  // the tail group takes 16 more words
  TIO_CHECK_ARG(offset < MT_MAX_WORDS && words <= MT_MAX_WORDS - offset,
                "%s: the draw ends beyond stream word 2^31", who);
  // first words of the first and last groups with outputs in [lo, hi)
  const uint64_t kept = (n % 16) ? n - 16 : n;  // outputs of the 16-groups the tail leaves
  const uint64_t first = lo < kept ? offset + lo / 16 * 16 : offset + n;
  const uint64_t last = hi > kept ? offset + n : offset + (hi - 1) / 16 * 16;
  cudaStream_t st = (cudaStream_t)stream;
  int q_lo, q_hi;
  if (int rc = mt_start_states(seed, first, last, table, workspace, workspace_bytes, st, who, &q_lo, &q_hi))
    return rc;
  mt_normal_kernel<<<(unsigned)(q_hi - q_lo), MT_THREADS, 0, st>>>((const uint32_t*)workspace, q_lo, MT_L, offset,
                                                                   n, lo, hi, z);
  launched();
  TIO_CHECK_LAUNCH();
  return 0;
}

// the [0, n) window of an aligned draw
extern "C" int tio_randn_mt19937(uint64_t seed, uint64_t offset, uint64_t n, float* z,
                                 const void* table, void* workspace, size_t workspace_bytes,
                                 void* stream) {
  TIO_CHECK_ARG(n >= 16 && (n % 16) == 0 && (offset % 16) == 0,
                "tio_randn_mt19937: n and offset must be multiples of 16 (n >= 16)");
  return tio_randn_mt19937_window(seed, offset, n, 0, n, z, table, workspace, workspace_bytes, stream);
}

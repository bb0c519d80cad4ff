// permute.cu — axis permutation with flips of a (B,C,I,J,K) batch in one pass (Reorient, Transpose).
//
// out[b,c,o0,o1,o2] = in[b,c,s] with s[perm_d] = o_d, mirrored (n − 1 − o_d) where bit perm_d of
// flip_bits is set: the reference's torch.flip per flipped axis followed by
// permute(...).contiguous() (spatial/reorient.py:63-91, transpose.py:36-50), up to four copies,
// done as one read and one write of every element.  Bytes move verbatim, so any dtype of 1, 2, 4
// or 8 bytes works.  Two paths:
//   * K stays last (perm = (1,0,2)): every output row is a whole input row, reversed under a K
//     flip; 16 bytes per thread as in remap_vec_kernel.
//   * K moves: a tile transpose through shared memory between K and the input axis `a` that
//     becomes the output's last axis; the third axis `m` is a slab index.
#include "common.cuh"

namespace tio {

// ---- K stays last ---------------------------------------------------------------------------
// Output row (bc, o0, o1) of length K is input row (bc, s_i, s_j) with s_j from o0 and s_i from o1.

template <typename T>
__global__ void __launch_bounds__(256)
permute_ij_vec_kernel(const T* __restrict__ src, T* __restrict__ dst, int I, int J, int K, int flips,
                      long long units) {
  constexpr int V = 16 / (int)sizeof(T);
  const long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // over B*C*J*I*(K/V)
  if (u >= units) return;
  const int per_row = K / V;
  const long long row = u / per_row;
  const int k0 = (int)(u - row * per_row) * V;
  const int o1 = (int)(row % I);
  const int o0 = (int)((row / I) % J);
  const long long bc = row / ((long long)I * J);
  const int si = (flips & 1) ? I - 1 - o1 : o1;
  const int sj = (flips & 2) ? J - 1 - o0 : o0;
  const T* s = src + ((bc * I + si) * J + sj) * K;
  const int first = (flips & 4) ? K - V - k0 : k0;  // the V source elements of this unit start here
  uint4 v;
  if (((uintptr_t)(s + first) & 15) == 0) {
    v = __ldg(reinterpret_cast<const uint4*>(s + first));
    if (flips & 4) {  // reverse the V elements in registers
      T t[V], r[V];
      memcpy(t, &v, 16);
#pragma unroll
      for (int e = 0; e < V; ++e) r[e] = t[V - 1 - e];
      memcpy(&v, r, 16);
    }
  } else {
    T t[V];
#pragma unroll
    for (int e = 0; e < V; ++e) t[e] = __ldg(s + ((flips & 4) ? K - 1 - (k0 + e) : k0 + e));
    memcpy(&v, t, 16);
  }
  *reinterpret_cast<uint4*>(dst + row * K + k0) = v;
}

// rows that are not a multiple of 16 bytes, or an unaligned destination: threads along K
template <typename T>
__global__ void __launch_bounds__(256)
permute_ij_kernel(const T* __restrict__ src, T* __restrict__ dst, int I, int J, int K, int flips, long long rows) {
  const long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y;  // over B*C*J*I
  if (row >= rows) return;
  const int o1 = (int)(row % I);
  const int o0 = (int)((row / I) % J);
  const long long bc = row / ((long long)I * J);
  const int si = (flips & 1) ? I - 1 - o1 : o1;
  const int sj = (flips & 2) ? J - 1 - o0 : o0;
  const T* s = src + ((bc * I + si) * J + sj) * K;
  T* d = dst + row * K;
  for (int k = threadIdx.x; k < K; k += blockDim.x) d[k] = __ldg(s + ((flips & 4) ? K - 1 - k : k));
}

// ---- K moves --------------------------------------------------------------------------------
// One CTA (256 threads) moves a TD x TD tile of (output a, input k) for one (b, c, s_m), TD = 32·P.
// A word W holds P = sizeof(W)/sizeof(T) elements (4 bytes for 1- and 2-byte T, one element
// otherwise), so every warp instruction reads or writes 32 words: 128 contiguous bytes (256 for
// 8-byte T).  Loads: each thread reads one word along k from each of P consecutive rows of a,
// transposes the P x P block in registers and stores P words, one per k, each holding P
// consecutive a.  Shared memory is tile[k][a-word] with the word column XOR-swizzled by k / P,
// so both the stores (one a-word, 32 k-words per warp) and the row reads of the write phase hit
// 32 different banks.  Stores: each warp writes rows of the output along a.  The tile is indexed
// by INPUT k (aligned loads) and OUTPUT a (aligned stores); flips only mirror the other side's
// coordinate.  `word_load`: K % P == 0 and src word-aligned; `word_store`: n_a % P == 0 and dst
// word-aligned; otherwise the same tile moves element by element with bounds checks.
struct TileGeometry {
  int n_a, K, n_m;            // lengths of axis a (the output's last), K, and the slab axis m
  long long in_stride_a;      // input element strides of a and m
  long long in_stride_m;
  long long out_stride_k;     // output element strides of the axes that k and m become
  long long out_stride_m;
  long long slab;             // I*J*K
  int tiles_a, tiles_k;
  int flip_a, flip_k, flip_m;
  int word_load, word_store;
};

template <typename T, typename W>
__global__ void __launch_bounds__(256)
permute_tile_kernel(const T* __restrict__ src, T* __restrict__ dst, TileGeometry g) {
  constexpr int P = (int)(sizeof(W) / sizeof(T));
  constexpr int TD = 32 * P;
  __shared__ W tile[TD][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long t = blockIdx.x;
  const int tk = (int)(t % g.tiles_k);
  t /= g.tiles_k;
  const int ta = (int)(t % g.tiles_a);
  t /= g.tiles_a;
  const int sm = (int)(t % g.n_m);
  const long long bc = t / g.n_m;
  const int k0 = tk * TD, a0 = ta * TD;
  const int om = g.flip_m ? g.n_m - 1 - sm : sm;
  const T* in = src + bc * g.slab + sm * g.in_stride_m;
  T* out = dst + bc * g.slab + om * g.out_stride_m;

  const int k = k0 + lane * P;  // this thread's first k in the load phase
#pragma unroll
  for (int qi = 0; qi < 4; ++qi) {
    const int q = warp + 8 * qi;  // a-word of the tile
    T e[P][P];                    // e[r][c]: output a = a0 + q·P + r, input k = k + c
#pragma unroll
    for (int r = 0; r < P; ++r) {
      const int oa = a0 + q * P + r;
      if (oa < g.n_a && k < g.K) {
        const int sa = g.flip_a ? g.n_a - 1 - oa : oa;
        const T* row = in + sa * g.in_stride_a;
        if (g.word_load) {
          const W w = __ldg(reinterpret_cast<const W*>(row + k));
          memcpy(e[r], &w, sizeof(W));
        } else {
#pragma unroll
          for (int c = 0; c < P; ++c) e[r][c] = k + c < g.K ? __ldg(row + k + c) : T(0);
        }
      } else {
#pragma unroll
        for (int c = 0; c < P; ++c) e[r][c] = T(0);
      }
    }
#pragma unroll
    for (int c = 0; c < P; ++c) {
      T col[P];
#pragma unroll
      for (int r = 0; r < P; ++r) col[r] = e[r][c];
      W w;
      memcpy(&w, col, sizeof(W));
      tile[lane * P + c][q ^ lane] = w;  // row k - k0, swizzled by (k - k0) / P = lane
    }
  }
  __syncthreads();

  const int oa = a0 + lane * P;  // this thread's first output a in the store phase
  if (oa >= g.n_a) return;
  for (int ik = warp; ik < TD; ik += 8) {
    const int kk = k0 + ik;
    if (kk >= g.K) break;
    const int ok = g.flip_k ? g.K - 1 - kk : kk;
    const W w = tile[ik][lane ^ ((ik / P) & 31)];
    T* o = out + ok * g.out_stride_k + oa;
    if (g.word_store) {
      *reinterpret_cast<W*>(o) = w;
    } else {
      T v[P];
      memcpy(v, &w, sizeof(W));
#pragma unroll
      for (int c = 0; c < P; ++c)
        if (oa + c < g.n_a) o[c] = v[c];
    }
  }
}

template <typename T, typename W>
static void launch_tile(const void* src, void* dst, TileGeometry g, long long blocks, cudaStream_t st) {
  constexpr int P = (int)(sizeof(W) / sizeof(T));
  g.word_load = g.word_load && g.K % P == 0 && ((uintptr_t)src % sizeof(W)) == 0;
  g.word_store = g.word_store && g.n_a % P == 0 && ((uintptr_t)dst % sizeof(W)) == 0;
  permute_tile_kernel<T, W><<<(unsigned)blocks, 256, 0, st>>>((const T*)src, (T*)dst, g);
  launched();
}

template <typename T>
static void launch_ij(const void* src, void* dst, int B, int C, int I, int J, int K, int flips, cudaStream_t st) {
  const long long rows = (long long)B * C * I * J;
  constexpr int V = 16 / (int)sizeof(T);
  if (K % V == 0 && ((uintptr_t)dst & 15) == 0) {
    const long long units = rows * (K / V);
    permute_ij_vec_kernel<T><<<(unsigned)((units + 255) / 256), 256, 0, st>>>((const T*)src, (T*)dst, I, J, K,
                                                                              flips, units);
    launched();
    return;
  }
  const int tx = K >= 128 ? 128 : (K >= 64 ? 64 : 32);
  dim3 block(tx, 256 / tx);
  permute_ij_kernel<T><<<(unsigned)((rows + block.y - 1) / block.y), block, 0, st>>>((const T*)src, (T*)dst, I, J,
                                                                                      K, flips, rows);
  launched();
}

static int tile_edge(int elem_bytes) { return elem_bytes < 4 ? 32 * (4 / elem_bytes) : 32; }

}  // namespace tio

using namespace tio;

extern "C" int tio_permute(const void* src, void* dst, int elem_bytes, int B, int C, int I, int J, int K,
                           int perm0, int perm1, int perm2, int flip_bits, void* stream) {
  TIO_CHECK_ARG(src && dst, "tio_permute: null src/dst");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "tio_permute: non-positive shape");
  TIO_CHECK_ARG(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4 || elem_bytes == 8,
                "tio_permute: element size %d not in {1,2,4,8}", elem_bytes);
  const int perm[3] = {perm0, perm1, perm2};
  TIO_CHECK_ARG(perm0 >= 0 && perm0 < 3 && perm1 >= 0 && perm1 < 3 && perm2 >= 0 && perm2 < 3 &&
                    perm0 != perm1 && perm0 != perm2 && perm1 != perm2,
                "tio_permute: (%d, %d, %d) is not a permutation of (0, 1, 2)", perm0, perm1, perm2);
  TIO_CHECK_ARG(flip_bits >= 0 && flip_bits <= 7, "tio_permute: flip_bits %d not in 0..7", flip_bits);
  TIO_CHECK_ARG(!(perm0 == 0 && perm1 == 1 && perm2 == 2),
                "tio_permute: identity permutation (flips alone are tio_remap's; without flips nothing moves)");
  const long long total = (long long)B * C * I * J * K;
  TIO_CHECK_ARG(total <= (1ll << 62) / elem_bytes, "tio_permute: too many elements");
  const uintptr_t s = (uintptr_t)src, d = (uintptr_t)dst, bytes = (uintptr_t)(total * elem_bytes);
  TIO_CHECK_ARG(s + bytes <= d || d + bytes <= s, "tio_permute: src and dst overlap");
  cudaStream_t st = (cudaStream_t)stream;
  const int n[3] = {I, J, K};

  if (perm2 == 2) {  // (1, 0, 2): K stays last
    const long long rows = (long long)B * C * I * J;  // blocks: rows / 2 at most, or 16-byte units / 256
    TIO_CHECK_ARG(rows / 2 < (1ll << 31) && rows * ((K * elem_bytes + 15) / 16) / 256 < (1ll << 31),
                  "tio_permute: too many rows");
    switch (elem_bytes) {
      case 1: launch_ij<uint8_t>(src, dst, B, C, I, J, K, flip_bits, st); break;
      case 2: launch_ij<uint16_t>(src, dst, B, C, I, J, K, flip_bits, st); break;
      case 4: launch_ij<uint32_t>(src, dst, B, C, I, J, K, flip_bits, st); break;
      default: launch_ij<uint64_t>(src, dst, B, C, I, J, K, flip_bits, st); break;
    }
    TIO_CHECK_LAUNCH();
    return 0;
  }

  // K moves: a = the input axis that becomes the output's last, m = the remaining one
  const int a = perm2, m = 3 - a - 2;
  int out_axis[3];  // output axis of each input axis
  for (int dd = 0; dd < 3; ++dd) out_axis[perm[dd]] = dd;
  const long long in_stride[3] = {(long long)J * K, K, 1};
  const long long out_stride[3] = {(long long)n[perm1] * n[perm2], n[perm2], 1};
  TileGeometry g;
  g.n_a = n[a];
  g.K = K;
  g.n_m = n[m];
  g.in_stride_a = in_stride[a];
  g.in_stride_m = in_stride[m];
  g.out_stride_k = out_stride[out_axis[2]];
  g.out_stride_m = out_stride[out_axis[m]];
  g.slab = (long long)I * J * K;
  const int td = tile_edge(elem_bytes);
  g.tiles_a = (n[a] + td - 1) / td;
  g.tiles_k = (K + td - 1) / td;
  g.flip_a = (flip_bits >> a) & 1;
  g.flip_k = (flip_bits >> 2) & 1;
  g.flip_m = (flip_bits >> m) & 1;
  g.word_load = g.word_store = 1;
  const long long blocks = (long long)B * C * n[m] * g.tiles_a * g.tiles_k;
  TIO_CHECK_ARG(blocks < (1ll << 31), "tio_permute: too many tiles");
  switch (elem_bytes) {
    case 1: launch_tile<uint8_t, uint32_t>(src, dst, g, blocks, st); break;
    case 2: launch_tile<uint16_t, uint32_t>(src, dst, g, blocks, st); break;
    case 4: launch_tile<uint32_t, uint32_t>(src, dst, g, blocks, st); break;
    default: launch_tile<uint64_t, uint64_t>(src, dst, g, blocks, st); break;
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

// resample_backward.cu — K1ᵀ: the adjoint of tio_resample with respect to its input image.
//
// Replaces the backward of the reference's sampling, ATen's grid_sampler_3d_backward (one global
// atomic per tap and voxel) through F.grid_sample and torch.where (transforms/spatial/spatial.py:
// 1651-1731, 1764-1857 of TorchIO 2.0.0a2).  Each output voxel sends g * w to each of its in-bounds
// trilinear taps (nearest: g to the rounded voxel); a voxel the forward filled (mask <= 0.5 with a
// fill value) sends nothing; pass-through elements copy g.
//
// Work decomposition: the forward's 16^3 output tiles and the boxes tile_bounds_kernel records for
// them.  A CTA zeroes a shared-memory accumulator of its tile's box, walks the tile's 256 columns
// with shared-memory atomics, and adds the box into grad_in with vector reductions
// (red.global.add.v4.f32), dropping the parts outside the volume and chunks nothing reached.  Tiles
// whose pre-image does not fit the box add straight into grad_in.  The result is not deterministic:
// the order of the additions depends on the schedule.
//
// Coordinates, weights and fill decisions are the exact chain of general_column
// (resample_common.cuh), i.e. the reference's fp32 rounding sequence, in both coordinate modes: the
// fill decisions are the ones either forward mode makes, and the weights are the ones the
// reference's own backward uses.  The forward's one-fma mode moves its weights by its coordinate
// noise (<= ~2e-5 voxel), so it is the adjoint of this kernel to within that noise.
#include "resample_tile.cuh"

namespace tio {

// one tap of the adjoint: into the shared box when the tap lies in it, else into grad_in
struct TapSink {
  float* acc;            // shared accumulator, null = global atomics only
  float* gin;            // grad_in of the (b, c) volume
  int lo_i, lo_j, lo_k;  // box origin in the volume
  int edge, bk;
  int J, K;

  __device__ __forceinline__ void add(int i, int j, int k, float v) const {
    if (acc) {
      const int bi = i - lo_i, bj = j - lo_j, bkk = k - lo_k;
      if ((unsigned)bi < (unsigned)edge && (unsigned)bj < (unsigned)edge && (unsigned)bkk < (unsigned)bk) {
        atomicAdd(acc + (bi * edge + bj) * bk + bkk, v);
        return;
      }
    }
    atomicAdd(gin + ((int64_t)i * J + j) * K + k, v);
  }
};

// Output planes [oi0, oi_end) of column (oj, ok) of element b, channel volume g_out: the adjoint
// of general_column's MODE / HAS_FILL paths, with its coordinate, weight and mask arithmetic.
template <int MODE, bool HAS_CP, bool HAS_FILL>
__device__ __forceinline__ void adjoint_column(const ResampleArgs& a, const int b, const bool elastic, const float* cps,
                                               const float* __restrict__ g_out, const TapSink& sink, const int oi0,
                                               const int oi_end, const int oj, const int ok) {
  ColumnCoords<HAS_CP> coords(a, b, elastic, oj, ok);
  for (int oi = oi0; oi < oi_end; ++oi) {
    float q[3];
    coords.at(a, cps, oi, q);
    const float g = __ldg(g_out + ((int64_t)oi * a.OJ + oj) * a.OK + ok);
    float u[3];
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) u[ax] = renormalise(q[ax], a.nm1[ax], a.sm1[ax]);
    const float f0 = floorf(u[0]), f1 = floorf(u[1]), f2 = floorf(u[2]);
    const int c0 = (int)fminf(fmaxf(f0, -2.0f), (float)a.I);
    const int c1 = (int)fminf(fmaxf(f1, -2.0f), (float)a.J);
    const int c2 = (int)fminf(fmaxf(f2, -2.0f), (float)a.K);
    const bool interior = (c0 >= 0) & (c0 + 1 < a.I) & (c1 >= 0) & (c1 + 1 < a.J) & (c2 >= 0) & (c2 + 1 < a.K);
    float w[8];
    const bool need_w = (MODE != TIO_NEAREST) || (HAS_FILL && !interior);
    if (need_w) {
      const float lo0 = __fsub_rn(__fadd_rn(f0, 1.0f), u[0]), hi0 = __fsub_rn(u[0], f0);
      const float lo1 = __fsub_rn(__fadd_rn(f1, 1.0f), u[1]), hi1 = __fsub_rn(u[1], f1);
      const float lo2 = __fsub_rn(__fadd_rn(f2, 1.0f), u[2]), hi2 = __fsub_rn(u[2], f2);
      const float w00 = __fmul_rn(lo0, lo1), w10 = __fmul_rn(hi0, lo1);
      const float w01 = __fmul_rn(lo0, hi1), w11 = __fmul_rn(hi0, hi1);
      w[0] = __fmul_rn(w00, lo2); w[1] = __fmul_rn(w10, lo2);
      w[2] = __fmul_rn(w01, lo2); w[3] = __fmul_rn(w11, lo2);
      w[4] = __fmul_rn(w00, hi2); w[5] = __fmul_rn(w10, hi2);
      w[6] = __fmul_rn(w01, hi2); w[7] = __fmul_rn(w11, hi2);
    }
    bool inb[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) inb[t] = true;
    if (!interior) {
      const bool i_lo = (c0 >= 0) & (c0 < a.I), i_hi = (c0 + 1 >= 0) & (c0 + 1 < a.I);
      const bool j_lo = (c1 >= 0) & (c1 < a.J), j_hi = (c1 + 1 >= 0) & (c1 + 1 < a.J);
      const bool k_lo = (c2 >= 0) & (c2 < a.K), k_hi = (c2 + 1 >= 0) & (c2 + 1 < a.K);
      inb[0] = i_lo & j_lo & k_lo; inb[1] = i_hi & j_lo & k_lo;
      inb[2] = i_lo & j_hi & k_lo; inb[3] = i_hi & j_hi & k_lo;
      inb[4] = i_lo & j_lo & k_hi; inb[5] = i_hi & j_lo & k_hi;
      inb[6] = i_lo & j_hi & k_hi; inb[7] = i_hi & j_hi & k_hi;
    }
    if (HAS_FILL && !interior) {
      float msum = 0.0f;
#pragma unroll
      for (int t = 0; t < 8; ++t)
        if (inb[t]) msum = __fadd_rn(msum, w[t]);
      if (!(msum > 0.5f)) continue;  // filled: the output does not depend on the input
    }
    if (MODE == TIO_NEAREST) {
      const int r0 = __float2int_rn(fminf(fmaxf(u[0], -2.0f), (float)a.I + 1.0f));
      const int r1 = __float2int_rn(fminf(fmaxf(u[1], -2.0f), (float)a.J + 1.0f));
      const int r2 = __float2int_rn(fminf(fmaxf(u[2], -2.0f), (float)a.K + 1.0f));
      if ((r0 >= 0) & (r0 < a.I) & (r1 >= 0) & (r1 < a.J) & (r2 >= 0) & (r2 < a.K)) sink.add(r0, r1, r2, g);
    } else {
#pragma unroll
      for (int t = 0; t < 8; ++t)
        if (inb[t]) sink.add(c0 + (t & 1), c1 + ((t >> 1) & 1), c2 + ((t >> 2) & 1), __fmul_rn(g, w[t]));
    }
  }
}

__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// One CTA per output tile (grid as the forward's tile kernels), one thread per (j, k) column.
template <int BOX, int MODE, bool HAS_CP, bool HAS_FILL>
__global__ void __launch_bounds__(256)
resample_backward_kernel(const float* __restrict__ grad_out, float* __restrict__ grad_in, const ResampleArgs a,
                         const int4* __restrict__ records, const int vec_ok) {
  constexpr int BK = box_k_extent(BOX, 4);
  constexpr int NBOX = BOX * BOX * BK;
  extern __shared__ __align__(16) float acc[];
  const int tid = threadIdx.x;
  const int tiles_i = (a.OI + XT - 1) / XT;
  const int b = blockIdx.z / tiles_i;
  const int i0 = (blockIdx.z - b * tiles_i) * XT, j0 = blockIdx.y * XT, k0 = blockIdx.x * XT;
  const int4 rec = __ldg(records + ((int64_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x);
  const int code = rec.w & 255;
  const int oj = j0 + (tid >> 4), ok = k0 + (tid & 15);
  const bool col = oj < a.OJ && ok < a.OK;
  const int i1 = min(i0 + XT, a.OI);
  const int64_t n_in = (int64_t)a.I * a.J * a.K, n_out = (int64_t)a.OI * a.OJ * a.OK;
  if (code == 2) return;  // every tap outside the volume: nothing reaches the input
  if (code == 3) {        // pass-through element: grad_in = g (spatial.py:1101-1106)
    if (col)
      for (int c = 0; c < a.C; ++c)
        for (int oi = i0; oi < i1; ++oi) {
          const int64_t o = ((int64_t)oi * a.OJ + oj) * a.OK + ok;
          grad_in[((int64_t)b * a.C + c) * n_in + o] = grad_out[((int64_t)b * a.C + c) * n_out + o];
        }
    return;
  }
  const bool elastic = HAS_CP && (rec.w & 1024);
  const float* cps = elastic ? a.cp + (int64_t)b * a.ni * a.nj * a.nk * 3 : nullptr;
  const bool staged = code == 1;
  for (int c = 0; c < a.C; ++c) {
    const float* g_out = grad_out + ((int64_t)b * a.C + c) * n_out;
    float* gin = grad_in + ((int64_t)b * a.C + c) * n_in;
    TapSink sink{staged ? acc : nullptr, gin, rec.x, rec.y, rec.z, BOX, BK, a.J, a.K};
    if (staged) {
      if (c > 0) __syncthreads();  // the previous channel's flush has read the box
      float4* acc4 = reinterpret_cast<float4*>(acc);
      for (int t = tid; t < NBOX / 4; t += 256) acc4[t] = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
    }
    if (col) adjoint_column<MODE, HAS_CP, HAS_FILL>(a, b, elastic, cps, g_out, sink, i0, i1, oj, ok);
    if (!staged) continue;
    __syncthreads();
    // flush: four K-consecutive voxels per step; chunks nothing reached are skipped
    constexpr int CHUNKS = BK / 4;
    for (int t = tid; t < BOX * BOX * CHUNKS; t += 256) {
      const int row = t / CHUNKS, q = t - row * CHUNKS;
      const int gi = rec.x + row / BOX, gj = rec.y + row % BOX, gk = rec.z + 4 * q;
      if ((unsigned)gi >= (unsigned)a.I || (unsigned)gj >= (unsigned)a.J) continue;
      const float4 v = reinterpret_cast<const float4*>(acc)[t];
      if (v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f) continue;
      float* p = gin + ((int64_t)gi * a.J + gj) * a.K + gk;
      if (vec_ok && gk >= 0 && gk + 3 < a.K) {
        red_add_v4(p, v);
      } else {
        const float e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int s = 0; s < 4; ++s)
          if ((unsigned)(gk + s) < (unsigned)a.K && e[s] != 0.f) atomicAdd(p + s, e[s]);
      }
    }
  }
}

template <int BOX, int MODE, bool HAS_CP>
static void launch_backward_fill(const float* g, float* gin, const ResampleArgs& a, const int4* records, int vec_ok,
                                 dim3 grid, size_t smem, cudaStream_t st) {
  if (a.fill) {
    cudaFuncSetAttribute(resample_backward_kernel<BOX, MODE, HAS_CP, true>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    resample_backward_kernel<BOX, MODE, HAS_CP, true><<<grid, 256, smem, st>>>(g, gin, a, records, vec_ok);
  } else {
    cudaFuncSetAttribute(resample_backward_kernel<BOX, MODE, HAS_CP, false>,
                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    resample_backward_kernel<BOX, MODE, HAS_CP, false><<<grid, 256, smem, st>>>(g, gin, a, records, vec_ok);
  }
  launched();
}

template <int BOX>
static void launch_backward(const float* g, float* gin, const ResampleArgs& a, int mode, const int4* records,
                            int vec_ok, dim3 grid, size_t smem, cudaStream_t st) {
  if (mode == TIO_NEAREST) {
    if (a.cp) launch_backward_fill<BOX, TIO_NEAREST, true>(g, gin, a, records, vec_ok, grid, smem, st);
    else launch_backward_fill<BOX, TIO_NEAREST, false>(g, gin, a, records, vec_ok, grid, smem, st);
  } else {
    if (a.cp) launch_backward_fill<BOX, TIO_LINEAR, true>(g, gin, a, records, vec_ok, grid, smem, st);
    else launch_backward_fill<BOX, TIO_LINEAR, false>(g, gin, a, records, vec_ok, grid, smem, st);
  }
}

}  // namespace tio

extern "C" int tio_resample_backward(const float* grad_out, float* grad_in, int B, int C, int I, int J, int K,
                                     int OI, int OJ, int OK, const float* mat, const float* cp,
                                     const uint8_t* flags, int ni, int nj, int nk, const float* spacing_in,
                                     const float* spacing_out, int affine_first, int mode, const float* fill,
                                     int box_hint, void* workspace, size_t workspace_bytes, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(grad_out && grad_in && mat, "tio_resample_backward: null grad_out/grad_in/mat");
  TIO_CHECK_ARG(grad_out != grad_in, "tio_resample_backward: grad_out and grad_in must not alias");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0 && OI > 0 && OJ > 0 && OK > 0,
                "tio_resample_backward: non-positive shape");
  mode &= ~TIO_EXACT_COORDS;  // one coordinate chain for both forward modes (see the file comment)
  TIO_CHECK_ARG(mode == TIO_NEAREST || mode == TIO_LINEAR, "tio_resample_backward: bad mode %d", mode);
  TIO_CHECK_ARG(spacing_in && spacing_out, "tio_resample_backward: null spacing");
  TIO_CHECK_ARG(!cp || (ni >= 2 && nj >= 2 && nk >= 2), "tio_resample_backward: control grid < 2 per axis");
  const int tiles_i = (OI + XT - 1) / XT;
  TIO_CHECK_ARG((int64_t)B * tiles_i <= 65535 && (OJ + XT - 1) / XT <= 65535,
                "tio_resample_backward: grid too large (B*ceil(OI/16) and ceil(OJ/16) must be <= 65535)");
  const size_t need = tio_resample_workspace_bytes(B, OI, OJ, OK);
  TIO_CHECK_ARG(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 15) == 0,
                "tio_resample_backward: needs a 16-byte aligned workspace of %zu bytes", need);
  ResampleArgs a;
  a.src = nullptr; a.dst = nullptr; a.mat = mat; a.cp = cp; a.flags = flags; a.fill = fill; a.elems = nullptr;
  a.B = B; a.C = C; a.I = I; a.J = J; a.K = K; a.OI = OI; a.OJ = OJ; a.OK = OK;
  a.ni = ni; a.nj = nj; a.nk = nk;
  auto scale = [](int n_in, int n_out) {  // as tio_resample
    if (n_in == n_out) return 1.0f;
    return n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.0f;
  };
  a.sc_i = cp ? scale(ni, OI) : 0.f; a.sc_j = cp ? scale(nj, OJ) : 0.f; a.sc_k = cp ? scale(nk, OK) : 0.f;
  const int dims[3] = {I, J, K};
  for (int t = 0; t < 3; ++t) {
    a.sp_in[t] = spacing_in[t]; a.sp_out[t] = spacing_out[t];
    a.nm1[t] = (float)(dims[t] - 1 > 1 ? dims[t] - 1 : 1);
    a.sm1[t] = (float)(dims[t] - 1);
  }
  a.affine_first = affine_first;
  a.cp_in_smem = 0;
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(grad_in, 0, (size_t)B * C * I * J * K * sizeof(float), st));
  // the forward's box edges: 24 covers its default and the smaller hints, 32 the rest
  const int box = box_hint > 24 ? 32 : 24;
  const int bk = box_k_extent(box, 4);
  int4* records = (int4*)workspace;
  const int64_t n_tiles = (int64_t)B * tiles_i * ((OJ + XT - 1) / XT) * ((OK + XT - 1) / XT);
  const unsigned bounds_blocks = (unsigned)((n_tiles + 127) / 128);
  // K origins rounded down to 4 voxels: box rows line up with 16-byte chunks of grad_in rows
  if (cp) tile_bounds_kernel<true><<<bounds_blocks, 128, 0, st>>>(a, box, 4, bk, 0, 0, records);
  else tile_bounds_kernel<false><<<bounds_blocks, 128, 0, st>>>(a, box, 4, bk, 0, 0, records);
  launched();
  const int vec_ok = (K % 4 == 0) && (((uintptr_t)grad_in & 15) == 0);
  const dim3 grid((OK + XT - 1) / XT, (OJ + XT - 1) / XT, (unsigned)(B * tiles_i));
  const size_t smem = (size_t)box * box * bk * sizeof(float);
  if (box == 24) launch_backward<24>(grad_out, grad_in, a, mode, records, vec_ok, grid, smem, st);
  else launch_backward<32>(grad_out, grad_in, a, mode, records, vec_ok, grid, smem, st);
  TIO_CHECK_LAUNCH();
  return 0;
}

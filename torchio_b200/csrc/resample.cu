// resample.cu — K1: fused affine + elastic displacement + gather + fill.
//
// One pass replaces the reference's grid construction and sampling
// (transforms/spatial/spatial.py:1504-1579, 1651-1731, 1764-1857 of TorchIO
// 2.0.0a2): arange/meshgrid/cat/sgemm, F.interpolate(trilinear), two
// F.grid_sample passes and torch.where.  Coordinate arithmetic reproduces the
// CPU op order of those ATen calls rounding-for-rounding (see
// oracle/c/tio_oracle.c, which is bit-exact against the reference), so
// nearest-neighbour label maps and fill decisions are bit-identical.
//
// Work decomposition: a CTA owns a (TJ x TK) window of output columns and
// walks TI output planes along I.  A thread owns one (j,k) column, so
//   - stores (and, for small rotations, gathers) are coalesced along K;
//   - the displacement field d = lerp_I(lerp_J(lerp_K(cp))) keeps its two
//     inner levels in registers across the I walk (recomputed only when the
//     walk enters a new control-grid cell), i.e. ~6 FMA/voxel instead of 42.
#include "resample_common.cuh"

namespace tio {

template <typename T, int MODE, bool HAS_CP, bool HAS_FILL>
__global__ void __launch_bounds__(TK* TJ)
resample_kernel(const ResampleArgs a) {
  extern __shared__ float smem_cp[];
  const int tiles_i = (a.OI + TI - 1) / TI;
  const int b = blockIdx.z / tiles_i;
  const int oi0 = (blockIdx.z % tiles_i) * TI;
  const int ok = blockIdx.x * TK + threadIdx.x;
  const int oj = blockIdx.y * TJ + threadIdx.y;
  const int64_t n_in = (int64_t)a.I * a.J * a.K;
  const int64_t n_out = (int64_t)a.OI * a.OJ * a.OK;
  const uint8_t fl = a.flags ? a.flags[b] : 0;
  const T* __restrict__ src = (const T*)a.src + (int64_t)b * a.C * n_in;
  T* __restrict__ dst = (T*)a.dst + (int64_t)b * a.C * n_out;
  const int oi_end = min(oi0 + TI, a.OI);

  if (fl & TIO_FLAG_PASSTHROUGH) {  // exact copy (spatial.py:1101-1106)
    if (ok < a.OK && oj < a.OJ)
      for (int c = 0; c < a.C; ++c)
        for (int oi = oi0; oi < oi_end; ++oi) {
          int64_t o = ((int64_t)oi * a.OJ + oj) * a.OK + ok;
          dst[c * n_out + o] = src[c * n_in + o];
        }
    return;
  }

  const bool elastic = HAS_CP && (fl & TIO_FLAG_ELASTIC);
  const float* g = nullptr;
  if (HAS_CP && elastic) {
    const int ncp = a.ni * a.nj * a.nk * 3;
    const float* gsrc = a.cp + (int64_t)b * ncp;
    if (a.cp_in_smem) {
      for (int t = threadIdx.y * TK + threadIdx.x; t < ncp; t += TK * TJ) smem_cp[t] = gsrc[t];
      __syncthreads();
      g = smem_cp;
    } else {
      g = gsrc;
    }
  }
  if (ok >= a.OK || oj >= a.OJ) return;

  general_column<T, MODE, HAS_CP, HAS_FILL>(a, b, elastic, g, src, dst, n_in, n_out, oi0, oi_end,
                                            oj, ok);
}

template <typename T, int MODE, bool HAS_CP>
static int launch_fill(const ResampleArgs& a, dim3 grid, dim3 block, size_t smem, cudaStream_t st) {
  if (a.fill)
    resample_kernel<T, MODE, HAS_CP, true><<<grid, block, smem, st>>>(a);
  else
    resample_kernel<T, MODE, HAS_CP, false><<<grid, block, smem, st>>>(a);
  launched();
  return 0;
}

template <typename T>
static int launch_typed(const ResampleArgs& a, int mode, cudaStream_t st) {
  dim3 block(TK, TJ, 1);
  const int tiles_i = (a.OI + TI - 1) / TI;
  dim3 grid((a.OK + TK - 1) / TK, (a.OJ + TJ - 1) / TJ, (unsigned)(a.B * tiles_i));
  size_t smem = (a.cp && a.cp_in_smem) ? (size_t)a.ni * a.nj * a.nk * 3 * sizeof(float) : 0;
  const bool has_cp = a.cp != nullptr;
#define TIO_SET_SMEM(KERN)                                                              \
  if (smem > 48 * 1024)                                                                 \
    cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (has_cp) {
    TIO_SET_SMEM((resample_kernel<T, TIO_NEAREST, true, true>))
    TIO_SET_SMEM((resample_kernel<T, TIO_NEAREST, true, false>))
    TIO_SET_SMEM((resample_kernel<T, TIO_LINEAR, true, true>))
    TIO_SET_SMEM((resample_kernel<T, TIO_LINEAR, true, false>))
  }
#undef TIO_SET_SMEM
  if (mode == TIO_LABEL_PV) {  // fill[0] is the pad label: always present
    if (has_cp) {
      if (smem > 48 * 1024)
        cudaFuncSetAttribute(resample_kernel<T, TIO_LABEL_PV, true, true>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      resample_kernel<T, TIO_LABEL_PV, true, true><<<grid, block, smem, st>>>(a);
    } else {
      resample_kernel<T, TIO_LABEL_PV, false, true><<<grid, block, smem, st>>>(a);
    }
    launched();
    return 0;
  }
  if (mode == TIO_NEAREST) {
    if (has_cp) return launch_fill<T, TIO_NEAREST, true>(a, grid, block, smem, st);
    return launch_fill<T, TIO_NEAREST, false>(a, grid, block, smem, st);
  }
  if (has_cp) return launch_fill<T, TIO_LINEAR, true>(a, grid, block, smem, st);
  return launch_fill<T, TIO_LINEAR, false>(a, grid, block, smem, st);
}

// ---- min of sample 0 (fill value "minimum") --------------------------------

// torch.amin's order: NaN wins, otherwise the least value (one instruction, as fminf)
__device__ __forceinline__ float min_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// valid for any mix of signs once *addr was initialised to +inf.  Dispatch on the sign bit: -0.0
// takes the unsigned path, where it orders above +0.0 and below every negative.  A NaN is stored
// as 0xffffffff, which wins both paths (the largest unsigned, a negative int) and reads as NaN.
__device__ __forceinline__ void atomic_min_float(float* addr, float v) {
  const unsigned u = v != v ? 0xffffffffu : __float_as_uint(v);
  if (u & 0x80000000u)
    atomicMax((unsigned int*)addr, u);
  else
    atomicMin((int*)addr, (int)u);
}

__global__ void min_init_kernel(float* fill, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) fill[c] = __int_as_float(0x7f800000);
}

template <bool VEC>
__global__ void __launch_bounds__(256) min_kernel(const float* __restrict__ src, int64_t n,
                                                  float* fill) {
  const int c = blockIdx.y;
  const float* base = src + (int64_t)c * n;
  float m = __int_as_float(0x7f800000);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (VEC) {
    const float4* p = (const float4*)base;
    for (int64_t t = t0; t < (n >> 2); t += stride) {
      float4 v = __ldg(p + t);
      m = min_nan(min_nan(m, v.x), min_nan(min_nan(v.y, v.z), v.w));
    }
  } else {
    for (int64_t t = t0; t < n; t += stride) m = min_nan(m, __ldg(base + t));
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) m = min_nan(m, __shfl_xor_sync(0xffffffffu, m, s));
  __shared__ float part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int t = 1; t < 8; ++t) m = min_nan(m, part[t]);
    atomic_min_float(fill + c, m);
  }
}

int launch_resample_tile(const ResampleArgs& a, int dtype, int mode, bool exact_coords, int box_hint,
                         const int* runs, int n_runs, void* workspace, size_t workspace_bytes, cudaStream_t st);
size_t resample_tile_workspace_bytes(int B, int OI, int OJ, int OK);

}  // namespace tio

namespace {

int resample(const void* src, void* dst, int dtype, int B, int C, int I, int J, int K, int OI, int OJ, int OK,
             const float* mat, const float* cp, const uint8_t* flags, int ni, int nj, int nk,
             const float* spacing_in, const float* spacing_out, int affine_first, int mode, const float* fill,
             int box_hint, const int* elems, const int* runs, int n_runs, void* workspace, size_t workspace_bytes,
             void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && dst && mat, "tio_resample: null src/dst/mat");
  TIO_CHECK_ARG(src != dst, "tio_resample: src and dst must not alias");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0 && OI > 0 && OJ > 0 && OK > 0,
                "tio_resample: non-positive shape");
  const bool exact_coords = (mode & TIO_EXACT_COORDS) != 0;
  mode &= ~TIO_EXACT_COORDS;
  TIO_CHECK_ARG(mode == TIO_NEAREST || mode == TIO_LINEAR || mode == TIO_LABEL_PV, "tio_resample: bad mode %d", mode);
  TIO_CHECK_ARG(mode != TIO_LABEL_PV || (C == 1 && fill),
                "tio_resample: TIO_LABEL_PV needs C == 1 and fill[0] = the pad label");
  TIO_CHECK_ARG(spacing_in && spacing_out, "tio_resample: null spacing");
  TIO_CHECK_ARG(!cp || (ni >= 2 && nj >= 2 && nk >= 2), "tio_resample: control grid < 2 per axis");
  TIO_CHECK_ARG((int64_t)B * ((OI + TI - 1) / TI) <= 65535 && (OJ + TJ - 1) / TJ <= 65535,
                "tio_resample: grid too large (B*ceil(OI/16) and ceil(OJ/4) must be <= 65535)");
  ResampleArgs a;
  a.src = src; a.dst = dst; a.mat = mat; a.cp = cp; a.flags = flags; a.fill = fill; a.elems = elems;
  a.B = B; a.C = C; a.I = I; a.J = J; a.K = K; a.OI = OI; a.OJ = OJ; a.OK = OK;
  a.ni = ni; a.nj = nj; a.nk = nk;
  auto scale = [](int n_in, int n_out) {
    if (n_in == n_out) return 1.0f;  // ATen short-circuit == identity weights
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
  a.cp_in_smem = cp && ((size_t)ni * nj * nk * 12 <= 96 * 1024);
  cudaStream_t st = (cudaStream_t)stream;
  if (box_hint >= 0) {  // fp32 trilinear and 1/2/4-byte nearest take the TMA tile path when it applies
    const int rc = launch_resample_tile(a, dtype, mode, exact_coords, box_hint, runs, n_runs, workspace,
                                        workspace_bytes, st);
    if (rc == 0) {
      TIO_CHECK_LAUNCH();
      return 0;
    }
    TIO_CHECK_ARG(rc == 1, "tio_resample: TMA tile path failed (code %d)", rc);
  }
  switch (dtype) {
    case TIO_F32: launch_typed<float>(a, mode, st); break;
    case TIO_U8: launch_typed<uint8_t>(a, mode, st); break;
    case TIO_I8: launch_typed<int8_t>(a, mode, st); break;
    case TIO_I16: launch_typed<int16_t>(a, mode, st); break;
    case TIO_I32: launch_typed<int32_t>(a, mode, st); break;
    case TIO_I64: launch_typed<int64_t>(a, mode, st); break;
    default: TIO_CHECK_ARG(false, "tio_resample: unknown dtype %d", dtype);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

}  // namespace

extern "C" int tio_resample(const void* src, void* dst, int dtype, int B, int C, int I, int J,
                            int K, int OI, int OJ, int OK, const float* mat, const float* cp,
                            const uint8_t* flags, int ni, int nj, int nk,
                            const float* spacing_in, const float* spacing_out,
                            int affine_first, int mode, const float* fill, int box_hint,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return resample(src, dst, dtype, B, C, I, J, K, OI, OJ, OK, mat, cp, flags, ni, nj, nk, spacing_in, spacing_out,
                  affine_first, mode, fill, box_hint, nullptr, nullptr, 0, workspace, workspace_bytes, stream);
}

extern "C" int tio_resample_tiered(const void* src, void* dst, int dtype, int B, int C, int I, int J,
                                   int K, int OI, int OJ, int OK, const float* mat, const float* cp,
                                   const uint8_t* flags, int ni, int nj, int nk,
                                   const float* spacing_in, const float* spacing_out,
                                   int affine_first, int mode, const float* fill, int box_hint,
                                   const int* elems, const int* runs, int n_runs,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(elems && runs && n_runs >= 1 && n_runs <= 5, "tio_resample_tiered: null elems/runs or n_runs %d",
                n_runs);
  TIO_CHECK_ARG(dtype == TIO_F32 && mode == TIO_LINEAR && box_hint >= 0 && workspace,
                "tio_resample_tiered: needs an fp32 image, TIO_LINEAR without TIO_EXACT_COORDS, box_hint >= 0 and"
                " a workspace");
  int total = 0, last = 0;
  for (int r = 0; r < n_runs; ++r) {
    const int count = runs[2 * r], edge = runs[2 * r + 1];
    TIO_CHECK_ARG(count > 0 && edge > last && (edge == 20 || edge == 22 || edge == 24 || edge == 28 || edge == 32),
                  "tio_resample_tiered: run %d: %d elements at edge %d (edges 20/22/24/28/32, ascending)", r, count,
                  edge);
    total += count;
    last = edge;
  }
  TIO_CHECK_ARG(total == B, "tio_resample_tiered: the runs hold %d elements, the batch %d", total, B);
  return resample(src, dst, dtype, B, C, I, J, K, OI, OJ, OK, mat, cp, flags, ni, nj, nk, spacing_in, spacing_out,
                  affine_first, mode, fill, box_hint, elems, runs, n_runs, workspace, workspace_bytes, stream);
}

extern "C" size_t tio_resample_workspace_bytes(int B, int OI, int OJ, int OK) {
  return tio::resample_tile_workspace_bytes(B, OI, OJ, OK);
}

extern "C" int tio_min_sample0(const float* src, int C, int64_t n, float* fill, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && fill && C > 0 && n > 0, "tio_min_sample0: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  min_init_kernel<<<(C + 31) / 32, 32, 0, st>>>(fill, C);
  launched();
  const bool vec = (((uintptr_t)src & 15) == 0) && ((n & 3) == 0);
  int64_t work = vec ? (n >> 2) : n;
  int blocks = (int)((work + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  if (blocks < 1) blocks = 1;
  if (vec)
    min_kernel<true><<<dim3(blocks, C), 256, 0, st>>>(src, n, fill);
  else
    min_kernel<false><<<dim3(blocks, C), 256, 0, st>>>(src, n, fill);
  launched();
  TIO_CHECK_LAUNCH();
  return 0;
}

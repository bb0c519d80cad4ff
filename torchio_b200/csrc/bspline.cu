// bspline.cu — B-spline interpolation of orders 2-7: the reference's
//   interpol.grid_pull(data.float(), voxel_grid, interpolation=order, bound="dct2",
//                      extrapolate=False, prefilter=True)
// (transforms/spatial/spatial.py:1734-1761, 1860-1878 of TorchIO 2.0.0a2) as two kernels.
//
// Prefilter: the interpolating B-spline coefficients c of each (b, c) volume, one in-place pass per
// axis longer than 1.  On every line, per pole z of the sampled B-spline, a causal and an anticausal
// first-order recursion with the initial conditions of the half-sample-symmetric (dct2) extension,
// after the gain prod (1 - z)(1 - 1/z).  A CTA stages up to 32 whole lines in shared memory (one
// thread per line), so every pass reads and writes HBM once and coalesced: the K pass loads 32
// consecutive rows as one contiguous block, the J and I passes load 32 consecutive K columns per
// line element.
//
// Pull: each thread walks an output column along I as K1's general kernel does (ColumnCoords, so
// both sample at the same fp32 coordinates) and sums the (n+1)^3 taps of the coefficients around
// each coordinate, with the B-spline weights and the dct2-folded tap indices computed once per axis.
// Voxels with a coordinate outside (-0.05, n - 1 + 0.05) are 0 (extrapolate=False).
#include "resample_common.cuh"

namespace tio {

constexpr int kLines = 32;                     // threads of a prefilter CTA: at most one line each
constexpr size_t kPrefilterSmem = 200 * 1024;  // the most shared memory a prefilter CTA asks for

struct Poles {
  int n;
  float z[3];
  float gain;
};

// Roots inside the unit circle of the sampled B-spline of each order (Unser, Aldroubi & Eden 1993;
// Thevenaz, Blu & Unser 2000, Table 1); the gain is prod (1 - z)(1 - 1/z).
static Poles poles_of(int order) {
  Poles p{};
  switch (order) {
    case 2: p.n = 1; p.z[0] = (float)(sqrt(8.0) - 3.0); break;
    case 3: p.n = 1; p.z[0] = (float)(sqrt(3.0) - 2.0); break;
    case 4:
      p.n = 2;
      p.z[0] = (float)(sqrt(664.0 - sqrt(438976.0)) + sqrt(304.0) - 19.0);
      p.z[1] = (float)(sqrt(664.0 + sqrt(438976.0)) - sqrt(304.0) - 19.0);
      break;
    case 5:
      p.n = 2;
      p.z[0] = (float)(sqrt(135.0 / 2.0 - sqrt(17745.0 / 4.0)) + sqrt(105.0 / 4.0) - 13.0 / 2.0);
      p.z[1] = (float)(sqrt(135.0 / 2.0 + sqrt(17745.0 / 4.0)) - sqrt(105.0 / 4.0) - 13.0 / 2.0);
      break;
    case 6:
      p.n = 3;
      p.z[0] = -0.48829458930304475513011803888378906211227916123938;
      p.z[1] = -0.081679271076237512597937765737059080653379610398148;
      p.z[2] = -0.0014141518083258177510872439765585925278641690553467;
      break;
    default:
      p.n = 3;
      p.z[0] = -0.53528043079643816554240378168164607183392315234269;
      p.z[1] = -0.12255461519232669051527226435935734360548654942730;
      p.z[2] = -0.0091486948096082769285930216516478534156925639545994;
      break;
  }
  double g = 1.0;
  for (int t = 0; t < p.n; ++t) {
    const double z = (double)p.z[t];
    g *= (1.0 - z) * (1.0 - 1.0 / z);
  }
  p.gain = (float)g;
  return p;
}

// Interpolating coefficients of one line of n > 1 values, in place; element e at s[e * step].
// The causal initial value is the exact sum over the dct2 extension (period 2n) while the line is
// shorter than the pole's decay horizon, and the sum truncated where |z|^i < 2^-24 otherwise.
__device__ __forceinline__ void filter_line(float* s, const int64_t step, const int n, const Poles& p) {
  for (int e = 0; e < n; ++e) s[e * step] *= p.gain;
  for (int t = 0; t < p.n; ++t) {
    const float z = p.z[t];
    const int horizon = (int)ceilf(-24.0f * 0.69314718f / logf(fabsf(z)));
    const float c0 = s[0];
    float acc, zi = z;
    if (n <= horizon) {  // z/(1 - z^2n) * sum_i z^i (c[i] + z^n c[n-1-i]) + c[0]
      const float zn = powf(z, (float)n);
      acc = 0.0f;
      for (int e = 0; e < n; ++e) {
        acc = fmaf(zi, fmaf(zn, s[(n - 1 - e) * step], s[e * step]), acc);
        zi *= z;
      }
      acc = acc / (1.0f - zn * zn);
    } else {  // sum_i z^(i+1) c[i]
      acc = 0.0f;
      for (int e = 0; e < horizon; ++e) {
        acc = fmaf(zi, s[e * step], acc);
        zi *= z;
      }
    }
    float prev = c0 + acc;
    s[0] = prev;
    for (int e = 1; e < n; ++e) {
      prev = fmaf(z, prev, s[e * step]);
      s[e * step] = prev;
    }
    prev = prev * (z / (z - 1.0f));  // anticausal initial value of the half-sample-symmetric extension
    s[(int64_t)(n - 1) * step] = prev;
    for (int e = n - 2; e >= 0; --e) {
      prev = z * (prev - s[e * step]);
      s[e * step] = prev;
    }
  }
}

// One prefilter pass over the lines of length n along one axis, `cta_lines` (<= kLines) lines per
// CTA, one thread each.  `rows`: the K pass, lines are consecutive rows, so a CTA's lines are one
// contiguous block that its threads stride through.  Otherwise line L starts at
// (L / inner) * n * inner + L % inner and steps by `inner` (J pass: inner = K; I pass: inner = J * K),
// so thread l walks line l and the CTA touches consecutive addresses at each step.  Reads T from
// `src` (the K pass; the same memory as `coeff` otherwise, hence no __restrict__: each CTA reads
// its whole tile before it writes, and no other CTA touches it) and writes fp32 `coeff`.
// Passthrough elements are skipped.
template <typename T>
__global__ void __launch_bounds__(kLines)
bspline_prefilter_kernel(const T* src, float* coeff, const uint8_t* flags, const int C,
                         const int64_t lines_per_volume, const int64_t inner, const int n,
                         const bool rows, const int pitch, const int cta_lines, const Poles p) {
  extern __shared__ float tile[];
  const int64_t per_volume = lines_per_volume * n;
  const int64_t tiles_per_volume = (lines_per_volume + cta_lines - 1) / cta_lines;
  const int64_t volume = blockIdx.x / tiles_per_volume;
  if (flags && (flags[volume / C] & TIO_FLAG_PASSTHROUGH)) return;  // copied from the source by the pull
  const int64_t first = (blockIdx.x % tiles_per_volume) * cta_lines;  // first line of this CTA
  const int lines = (int)min((int64_t)cta_lines, lines_per_volume - first);
  const T* s = src + volume * per_volume;
  float* d = coeff + volume * per_volume;
  const int l = threadIdx.x;
  if (rows) {
    const T* sb = s + first * n;
    const int total = lines * n;
    int row = 0, e = l;  // (row, e) of element t = l + k * kLines, stepped without divisions
    while (e >= n) { e -= n; ++row; }
    constexpr int kBatch = 8;  // loads in flight per thread before their shared-memory stores
    for (int t0 = l; t0 < total; t0 += kBatch * kLines) {
      float v[kBatch];
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        const int t = t0 + u * kLines;
        v[u] = t < total ? ElemTraits<T>::to_f32(sb[t]) : 0.0f;
      }
#pragma unroll
      for (int u = 0; u < kBatch; ++u) {
        if (t0 + u * kLines < total) tile[row * pitch + e] = v[u];
        e += kLines;
        while (e >= n) { e -= n; ++row; }
      }
    }
  } else if (l < lines) {
    const int64_t line = first + l;
    const T* sl = s + (line / inner) * n * inner + line % inner;
    for (int e = 0; e < n; ++e) tile[l * pitch + e] = ElemTraits<T>::to_f32(sl[e * inner]);
  }
  __syncthreads();
  if (l < lines) filter_line(tile + l * pitch, 1, n, p);
  __syncthreads();
  if (rows) {
    float* db = d + first * n;
    int row = 0, e = l;
    while (e >= n) { e -= n; ++row; }
    for (int t = l; t < lines * n; t += kLines) {
      db[t] = tile[row * pitch + e];
      e += kLines;
      while (e >= n) { e -= n; ++row; }
    }
  } else if (l < lines) {
    const int64_t line = first + l;
    float* dl = d + (line / inner) * n * inner + line % inner;
    for (int e = 0; e < n; ++e) dl[e * inner] = tile[l * pitch + e];
  }
}

// The n + 1 B-spline weights and dct2-folded tap indices of coordinate x on an axis of size n:
// taps t0 + j, t0 = floor(x - (n-1)/2), weight beta^ORDER(x - t0 - j) by the Cox-de Boor recursion
// on g = x - t0 - (ORDER-1)/2 in [0, 1) (every term non-negative, so no cancellation).
template <int ORDER>
__device__ __forceinline__ void axis_taps(const float x, const int n, float w[ORDER + 1], int idx[ORDER + 1]) {
  const float shift = 0.5f * (float)(ORDER - 1);
  const float f = floorf(x - shift);
  const float g = x - shift - f;
  const int t0 = (int)f;
  w[0] = 1.0f;
#pragma unroll
  for (int k = 1; k <= ORDER; ++k) {
    const float inv = 1.0f / (float)k;
    w[k] = g * w[k - 1] * inv;
#pragma unroll
    for (int j = k - 1; j >= 1; --j) w[j] = ((g + (float)(k - j)) * w[j - 1] + ((float)(j + 1) - g) * w[j]) * inv;
    w[0] = (1.0f - g) * w[0] * inv;
  }
  const int period = 2 * n;
#pragma unroll
  for (int j = 0; j <= ORDER; ++j) {
    int t = (t0 + j) % period;
    t += t < 0 ? period : 0;
    idx[j] = t < n ? t : period - 1 - t;
  }
}

template <typename T, int ORDER, bool HAS_CP>
__global__ void __launch_bounds__(TK* TJ)
bspline_pull_kernel(const ResampleArgs a, const float* __restrict__ coeff) {
  extern __shared__ float smem_cp[];
  const int tiles_i = (a.OI + TI - 1) / TI;
  const int b = blockIdx.z / tiles_i;
  const int oi0 = (blockIdx.z % tiles_i) * TI;
  const int ok = blockIdx.x * TK + threadIdx.x;
  const int oj = blockIdx.y * TJ + threadIdx.y;
  const int64_t n_in = (int64_t)a.I * a.J * a.K;
  const int64_t n_out = (int64_t)a.OI * a.OJ * a.OK;
  const uint8_t fl = a.flags ? a.flags[b] : 0;
  T* __restrict__ dst = (T*)a.dst + (int64_t)b * a.C * n_out;
  const int oi_end = min(oi0 + TI, a.OI);

  if (fl & TIO_FLAG_PASSTHROUGH) {  // exact copy of the source (spatial.py:1101-1106)
    const T* __restrict__ src = (const T*)a.src + (int64_t)b * a.C * n_in;
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

  const float* __restrict__ cf = coeff + (int64_t)b * a.C * n_in;
  ColumnCoords<HAS_CP> coords(a, b, elastic, oj, ok);
  for (int oi = oi0; oi < oi_end; ++oi) {
    float q[3];
    coords.at(a, g, oi, q);
    const int64_t o_off = ((int64_t)oi * a.OJ + oj) * a.OK + ok;
    // extrapolate=False: strictly inside (-0.05, n - 1 + 0.05) on every axis; NaN fails the test
    const bool inside = (q[0] > -0.05f) & (q[0] < (float)(a.I - 1) + 0.05f) & (q[1] > -0.05f) &
                        (q[1] < (float)(a.J - 1) + 0.05f) & (q[2] > -0.05f) & (q[2] < (float)(a.K - 1) + 0.05f);
    if (!inside) {
      for (int c = 0; c < a.C; ++c) dst[c * n_out + o_off] = ElemTraits<T>::from_f32(0.0f);
      continue;
    }
    float wi[ORDER + 1], wj[ORDER + 1], wk[ORDER + 1];
    int ii[ORDER + 1], jj[ORDER + 1], kk[ORDER + 1];
    axis_taps<ORDER>(q[0], a.I, wi, ii);
    axis_taps<ORDER>(q[1], a.J, wj, jj);
    axis_taps<ORDER>(q[2], a.K, wk, kk);
    for (int c = 0; c < a.C; ++c) {
      const float* s = cf + c * n_in;
      float v = 0.0f;
      // the I taps roll through slot 0 (static register indices; a fully unrolled (n+1)^3 sum
      // hoists every load and spills for orders >= 5)
      float wx[ORDER + 1];
      int ix[ORDER + 1];
#pragma unroll
      for (int x = 0; x <= ORDER; ++x) { wx[x] = wi[x]; ix[x] = ii[x]; }
#pragma unroll 1
      for (int x = 0; x <= ORDER; ++x) {
        const float* sx = s + (int64_t)ix[0] * a.J * a.K;
        float vj = 0.0f;
#pragma unroll
        for (int y = 0; y <= ORDER; ++y) {
          const float* sy = sx + (int64_t)jj[y] * a.K;
          float vk = 0.0f;
#pragma unroll
          for (int z = 0; z <= ORDER; ++z) vk = fmaf(wk[z], __ldg(sy + kk[z]), vk);
          vj = fmaf(wj[y], vk, vj);
        }
        v = fmaf(wx[0], vj, v);
#pragma unroll
        for (int t = 0; t < ORDER; ++t) { wx[t] = wx[t + 1]; ix[t] = ix[t + 1]; }
      }
      dst[c * n_out + o_off] = ElemTraits<T>::from_f32(v);
    }
  }
}

// Lines a prefilter CTA stages for lines of `pitch` floats: kLines while they fit in kPrefilterSmem,
// fewer for long axes (0: the axis is too long for even one line)
static int cta_lines_for(int pitch) {
  const int fit = (int)(kPrefilterSmem / ((size_t)pitch * sizeof(float)));
  return fit < kLines ? fit : kLines;
}

template <typename TS>
static void launch_pass(const TS* src, float* coeff, const uint8_t* flags, int64_t volumes, int C, int64_t lines,
                        int64_t inner, int n, bool rows, const Poles& p, cudaStream_t st) {
  const int pitch = n | 1;  // odd: the lines of a CTA fall in different banks
  const int cta_lines = cta_lines_for(pitch);
  const size_t smem = (size_t)cta_lines * pitch * sizeof(float);
  const unsigned grid = (unsigned)(volumes * ((lines + cta_lines - 1) / cta_lines));
  auto kern = bspline_prefilter_kernel<TS>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  kern<<<grid, kLines, smem, st>>>(src, coeff, flags, C, lines, inner, n, rows, pitch, cta_lines, p);
  launched();
}

template <typename T>
static void launch_prefilter(const T* src, float* coeff, const uint8_t* flags, int B, int C, int I, int J,
                             int K, const Poles& p, cudaStream_t st) {
  const int64_t vox = (int64_t)I * J * K, volumes = (int64_t)B * C;
  const int dims[3] = {I, J, K};
  bool first = true;
  for (int axis = 2; axis >= 0; --axis) {  // K first: it reads the source dtype
    const int n = dims[axis];
    if (n < 2) continue;
    const int64_t inner = axis == 2 ? 1 : (axis == 1 ? K : (int64_t)J * K);
    if (first)
      launch_pass<T>(src, coeff, flags, volumes, C, vox / n, inner, n, axis == 2, p, st);
    else
      launch_pass<float>(coeff, coeff, flags, volumes, C, vox / n, inner, n, axis == 2, p, st);
    first = false;
  }
  if (first && (const void*)src != (const void*)coeff) {
    // every axis has length 1: the coefficients are the values; one identity pass converts them
    const Poles identity{0, {0.f, 0.f, 0.f}, 1.0f};
    launch_pass<T>(src, coeff, flags, volumes, C, vox, 1, 1, true, identity, st);
  }
}

template <typename T, int ORDER>
static void launch_pull(const ResampleArgs& a, const float* coeff, cudaStream_t st) {
  dim3 block(TK, TJ, 1);
  const int tiles_i = (a.OI + TI - 1) / TI;
  dim3 grid((a.OK + TK - 1) / TK, (a.OJ + TJ - 1) / TJ, (unsigned)(a.B * tiles_i));
  if (a.cp) {
    const size_t smem = a.cp_in_smem ? (size_t)a.ni * a.nj * a.nk * 3 * sizeof(float) : 0;
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(bspline_pull_kernel<T, ORDER, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)smem);
    bspline_pull_kernel<T, ORDER, true><<<grid, block, smem, st>>>(a, coeff);
  } else {
    bspline_pull_kernel<T, ORDER, false><<<grid, block, 0, st>>>(a, coeff);
  }
  launched();
}

template <typename T>
static void launch_pull_order(const ResampleArgs& a, const float* coeff, int order, cudaStream_t st) {
  switch (order) {
    case 2: launch_pull<T, 2>(a, coeff, st); break;
    case 3: launch_pull<T, 3>(a, coeff, st); break;
    case 4: launch_pull<T, 4>(a, coeff, st); break;
    case 5: launch_pull<T, 5>(a, coeff, st); break;
    case 6: launch_pull<T, 6>(a, coeff, st); break;
    default: launch_pull<T, 7>(a, coeff, st); break;
  }
}

static size_t dtype_size(int dtype) {
  switch (dtype) {
    case TIO_U8: case TIO_I8: return 1;
    case TIO_I16: return 2;
    case TIO_F32: case TIO_I32: return 4;
    default: return 8;
  }
}

// [a, a + na) and [b, b + nb) share a byte
static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + nb && y < x + na;
}

}  // namespace tio

extern "C" int tio_bspline_prefilter(const void* src, int dtype, float* coeff, const uint8_t* flags, int B,
                                     int C, int I, int J, int K, int order, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(src && coeff, "tio_bspline_prefilter: null src/coeff");
  TIO_CHECK_ARG(order >= 2 && order <= 7, "tio_bspline_prefilter: order %d is not 2-7", order);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_I64, "tio_bspline_prefilter: unknown dtype %d", dtype);
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "tio_bspline_prefilter: non-positive shape");
  const int64_t vox = (int64_t)I * J * K;
  TIO_CHECK_ARG(src == (const void*)coeff || !overlaps(src, (size_t)B * C * vox * dtype_size(dtype), coeff,
                                                       (size_t)B * C * vox * sizeof(float)),
                "tio_bspline_prefilter: coeff overlaps src without being it");
  TIO_CHECK_ARG(src != (const void*)coeff || dtype == TIO_F32,
                "tio_bspline_prefilter: coeff may alias src only for TIO_F32");
  const int longest = I > J ? (I > K ? I : K) : (J > K ? J : K);
  TIO_CHECK_ARG(cta_lines_for(longest | 1) >= 1,
                "tio_bspline_prefilter: an axis of %d voxels does not fit the %d KiB a CTA stages (at most %d)",
                longest, (int)(kPrefilterSmem / 1024), (int)(kPrefilterSmem / sizeof(float)) - 1);
  const int dims[3] = {I, J, K};
  for (int t = 0; t < 3; ++t) {
    const int cl = cta_lines_for(dims[t] | 1);
    TIO_CHECK_ARG(dims[t] < 2 || (int64_t)B * C * ((vox / dims[t] + cl - 1) / cl) < (1ll << 31),
                  "tio_bspline_prefilter: grid too large");
  }
  const Poles p = poles_of(order);
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_PREFILTER(T) launch_prefilter<T>((const T*)src, coeff, flags, B, C, I, J, K, p, st)
  TIO_LABEL_DISPATCH(dtype, "tio_bspline_prefilter", TIO_PREFILTER)
#undef TIO_PREFILTER
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_bspline_resample(const float* coeff, const void* src, void* dst, int dtype, int B, int C,
                                    int I, int J, int K, int OI, int OJ, int OK, const float* mat,
                                    const float* cp, const uint8_t* flags, int ni, int nj, int nk,
                                    const float* spacing_in, const float* spacing_out, int affine_first,
                                    int order, void* stream) {
  using namespace tio;
  TIO_CHECK_ARG(coeff && src && dst && mat, "tio_bspline_resample: null coeff/src/dst/mat");
  TIO_CHECK_ARG(order >= 2 && order <= 7, "tio_bspline_resample: order %d is not 2-7", order);
  TIO_CHECK_ARG(dtype >= TIO_F32 && dtype <= TIO_I64, "tio_bspline_resample: unknown dtype %d", dtype);
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0 && OI > 0 && OJ > 0 && OK > 0,
                "tio_bspline_resample: non-positive shape");
  TIO_CHECK_ARG(spacing_in && spacing_out, "tio_bspline_resample: null spacing");
  TIO_CHECK_ARG(!cp || (ni >= 2 && nj >= 2 && nk >= 2), "tio_bspline_resample: control grid < 2 per axis");
  const size_t out_bytes = (size_t)B * C * OI * OJ * OK * dtype_size(dtype);
  TIO_CHECK_ARG(!overlaps(dst, out_bytes, coeff, (size_t)B * C * I * J * K * sizeof(float)),
                "tio_bspline_resample: dst must not alias coeff");
  TIO_CHECK_ARG(!overlaps(dst, out_bytes, src, (size_t)B * C * I * J * K * dtype_size(dtype)),
                "tio_bspline_resample: dst must not alias src");
  TIO_CHECK_ARG((int64_t)B * ((OI + TI - 1) / TI) <= 65535 && (OJ + TJ - 1) / TJ <= 65535,
                "tio_bspline_resample: grid too large (B*ceil(OI/16) and ceil(OJ/4) must be <= 65535)");
  ResampleArgs a{};
  a.src = src; a.dst = dst; a.mat = mat; a.cp = cp; a.flags = flags; a.fill = nullptr;
  a.B = B; a.C = C; a.I = I; a.J = J; a.K = K; a.OI = OI; a.OJ = OJ; a.OK = OK;
  a.ni = ni; a.nj = nj; a.nk = nk;
  auto scale = [](int n_in, int n_out) {  // as tio_resample: ATen's align_corners upsample scale
    if (n_in == n_out) return 1.0f;
    return n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.0f;
  };
  a.sc_i = cp ? scale(ni, OI) : 0.f; a.sc_j = cp ? scale(nj, OJ) : 0.f; a.sc_k = cp ? scale(nk, OK) : 0.f;
  for (int t = 0; t < 3; ++t) { a.sp_in[t] = spacing_in[t]; a.sp_out[t] = spacing_out[t]; }
  a.affine_first = affine_first;
  a.cp_in_smem = cp && ((size_t)ni * nj * nk * 12 <= 96 * 1024);
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_PULL(T) launch_pull_order<T>(a, coeff, order, st)
  TIO_LABEL_DISPATCH(dtype, "tio_bspline_resample", TIO_PULL)
#undef TIO_PULL
  TIO_CHECK_LAUNCH();
  return 0;
}

// stats.cu — data-derived parameters and the affine epilogue of Normalize / Standardize
// (SURVEY §8 f-3; transforms/intensity/normalize.py:104-232,332-366, standardize.py:52-107,
// _statistics.py:11-45 of TorchIO 2.0.0a2).
//
// The reference derives its parameters from batch element 0 on the host:
//   Standardize: values.float().mean() / .std()      (all channels of sample 0, optional mask)
//   Normalize:   two quantiles of the same values via torch.kthvalue + lerp
// and then applies `(x - mean) / std` or `(clamp(x) - in_min) / in_range * out_range + out_min`
// as separate fp32 elementwise ops over the whole batch.
//
//   tio_moments    one pass: count, sum, sum of squares (fp64 accumulators) of the selected voxels
//   tio_quantiles_batched  exact order statistics of every batch element by a 3-level radix select
//                  on the order-preserving integer image of fp32 (11 + 11 + 10 bits): three
//                  streaming passes instead of a sort; returns the two neighbours of each quantile
//                  and the interpolation weight, i.e. exactly what kthvalue(lower+1),
//                  kthvalue(lower+2) and `index - lower` give.  tio_quantiles is its B = 1 case.
//   tio_histogram_tables / tio_histogram_map  HistogramStandardization
//                  (histogram_standardization.py:216-303): the percentile lerp and fp32 map tables
//                  on the device, then the piecewise-linear map in the image's own dtype
//   tio_rescale    dst = ((clamp(x, lo, hi) - sub[b]) / div[b]) * mul[b] + add[b], every step
//                  rounded like the reference's separate fp32 ops (bit-exact given equal constants)
// The select is one HBM read per level, the others single-pass streams; 128-bit loads where aligned.
#include "image_dtype.cuh"

namespace tio {

__device__ __forceinline__ uint32_t order_key(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// ---- moments ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
moments_kernel(const float* __restrict__ src, const uint8_t* __restrict__ mask, int64_t n, double* out) {
  double s = 0.0, ss = 0.0;
  long long cnt = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (!mask && ((uintptr_t)src & 15) == 0) {
    const float4* p = reinterpret_cast<const float4*>(src);
    for (int64_t t = t0; t < (n >> 2); t += stride) {
      const float4 v = __ldg(p + t);
      s += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w);
      ss += ((double)v.x * v.x + (double)v.y * v.y) + ((double)v.z * v.z + (double)v.w * v.w);
      cnt += 4;
    }
    for (int64_t t = (n & ~(int64_t)3) + t0; t < n; t += stride) { const double v = src[t]; s += v; ss += v * v; ++cnt; }
  } else {
    for (int64_t t = t0; t < n; t += stride)
      if (!mask || mask[t]) { const double v = src[t]; s += v; ss += v * v; ++cnt; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  __shared__ double ps[8], pss[8];
  __shared__ long long pc[8];
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { ps[w] = s; pss[w] = ss; pc[w] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int t = 1; t < 8; ++t) { s += ps[t]; ss += pss[t]; cnt += pc[t]; }
    atomicAdd(out + 0, s);
    atomicAdd(out + 1, ss);
    atomicAdd(out + 2, (double)cnt);
  }
}

// ---- radix select ----------------------------------------------------------------------
// Exact order statistics of every batch element at once: three histogram levels over the order
// key (bits 31..21, 20..10, 9..0), one launch per level for the whole batch (element on
// gridDim.y), and a one-block-per-element scan between levels that walks each target rank to its
// bin.  Targets whose key prefixes agree at a level share one histogram ("slot"), so the 26 ranks
// of 13 percentiles cost one histogram per distinct prefix; at most kSlots targets go through a
// round, larger quantile sets take further rounds over levels 1 and 2.
constexpr int kBins0 = 2048, kBins1 = 2048, kBins2 = 1024;
constexpr int kSlots = 26;             // targets (2 ranks per quantile) per round: 26 x 8 KiB of shared histograms
constexpr int kQuantPerRound = kSlots / 2;
constexpr int kSelectThreads = 1024;

struct SelectElem {
  long long count;                 // selected voxels
  long long rank[kSlots];          // residual rank of each target inside its prefix
  unsigned prefix[kSlots];         // key bits fixed so far, right aligned
  unsigned uniq[kSlots];           // distinct prefixes of this level, ascending
  int slot[kSlots];                // index of the target's prefix in `uniq`
  int nuniq, nt;
  int nan;                         // a selected voxel is NaN
};

struct RoundQ {
  double q[kQuantPerRound];
  int first, nq;                   // quantiles [first, first + nq) of the call
};

__host__ __device__ constexpr int select_bins(int level) { return level == 2 ? kBins2 : kBins1; }

// adds `run` to bin `idx` of the shared histograms: consecutive voxels of one thread that fall in
// the same bin (a constant background) cost one atomic
__device__ __forceinline__ void flush_run(unsigned* h, int& last, unsigned& run, int idx) {
  if (idx == last) { ++run; return; }
  if (last >= 0) atomicAdd(h + last, run);
  last = idx;
  run = 1;
}

// LEVEL 0: one 2048-bin histogram per element into hist0[B][2048], NaN flags.  LEVEL 1 / 2: one
// histogram per distinct prefix into hist[B][slots][2048].  The shared table `tab` maps the top 11
// key bits to the range of `uniq` entries that start with them (start << 8 | count, 0 = none).
template <typename T, int LEVEL>
__global__ void __launch_bounds__(kSelectThreads)
select_hist_kernel(const T* __restrict__ src, const uint8_t* __restrict__ mask, int64_t per_elem,
                   SelectElem* __restrict__ st, unsigned* __restrict__ hist, int slots) {
  extern __shared__ unsigned smem[];
  constexpr int BINS = LEVEL == 0 ? kBins0 : select_bins(LEVEL);
  const int b = blockIdx.y;
  SelectElem& e = st[b];
  const int nh = LEVEL == 0 ? 1 : e.nuniq;
  unsigned* h = smem;
  unsigned short* tab = reinterpret_cast<unsigned short*>(smem + (size_t)slots * BINS);
  __shared__ unsigned uniq[kSlots];
  for (int t = threadIdx.x; t < nh * BINS; t += blockDim.x) h[t] = 0;
  if (LEVEL > 0) {
    for (int t = threadIdx.x; t < kBins0; t += blockDim.x) tab[t] = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int u = 0; u < nh; ++u) {
        uniq[u] = e.uniq[u];
        const unsigned top = LEVEL == 1 ? e.uniq[u] : e.uniq[u] >> 11;
        if (tab[top] == 0) tab[top] = (unsigned short)(u << 8);
        tab[top] += 1;
      }
    }
  }
  __syncthreads();

  const T* x = src + (int64_t)b * per_elem;
  const uint8_t* mk = mask ? mask + (int64_t)b * per_elem : nullptr;
  bool nan = false;
  int last = -1;
  unsigned run = 0;
  auto voxel = [&](float f) {
    if (f != f) nan = true;
    const uint32_t k = order_key(f);
    int idx = -1;
    if (LEVEL == 0) {
      idx = (int)(k >> 21);
    } else {
      const unsigned short te = tab[k >> 21];
      if (te) {
        if (LEVEL == 1) {
          idx = (te >> 8) * BINS + (int)((k >> 10) & 2047u);
        } else {
          for (int u = te >> 8, end = (te >> 8) + (te & 255); u < end; ++u)
            if (uniq[u] == (k >> 10)) { idx = u * BINS + (int)(k & 1023u); break; }
        }
      }
    }
    if (idx >= 0) flush_run(h, last, run, idx);
  };
  constexpr int V = 16 / sizeof(T);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t done = 0;
  if (((uintptr_t)x & 15) == 0) {
    const int64_t nv = per_elem / V;
    const uint4* p = reinterpret_cast<const uint4*>(x);
    for (int64_t t = t0; t < nv; t += stride) {
      Pack<T> pk;
      pk.raw = __ldg(p + t);
#pragma unroll
      for (int j = 0; j < V; ++j)
        if (!mk || mk[t * V + j]) voxel(to_float(pk.e[j]));
    }
    done = nv * V;
  }
  for (int64_t t = done + t0; t < per_elem; t += stride)
    if (!mk || mk[t]) voxel(to_float(ld(x + t)));
  if (last >= 0) atomicAdd(h + last, run);
  if (LEVEL == 0 && __syncthreads_or(nan) && threadIdx.x == 0) atomicOr(&e.nan, 1);
  __syncthreads();
  unsigned* g = hist + (size_t)b * (LEVEL == 0 ? 1 : slots) * (size_t)BINS;
  for (int t = threadIdx.x; t < nh * BINS; t += blockDim.x)
    if (h[t]) atomicAdd(g + t, h[t]);
}

__global__ void select_reset_kernel(SelectElem* st) {
  SelectElem& e = st[blockIdx.x];
  e.count = 0;
  e.nan = 0;
}

// one block per element, warp w walks target w through its histogram; then thread 0 collects the
// distinct prefixes of the next level.  At level 0 the round's ranks are set up first:
// index = q * (count - 1), lower = floor(index) (_statistics.py:37-45, numpy's "linear" method),
// targets 2j, 2j + 1 = ranks lower, min(lower + 1, count - 1).  Level 2 writes the results.
template <int LEVEL>
__global__ void __launch_bounds__(kSelectThreads)
select_scan_kernel(SelectElem* st, const unsigned* hist0, const unsigned* hist, int slots, RoundQ rq,
                   int64_t per_elem, int masked, int m, float* values, double* weights, double* count,
                   uint8_t* has_nan) {
  const int b = blockIdx.x;
  SelectElem& e = st[b];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (LEVEL == 0) {
    __shared__ unsigned long long total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    if (masked) {
      unsigned long long c = 0;
      for (int t = threadIdx.x; t < kBins0; t += blockDim.x) c += hist0[(size_t)b * kBins0 + t];
      atomicAdd(&total, c);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const long long c = masked ? (long long)total : (long long)per_elem;
      e.count = c;
      e.nt = 2 * rq.nq;
      for (int t = 0; t < 2 * rq.nq; ++t) {
        const double index = rq.q[t >> 1] * (double)(c > 0 ? c - 1 : 0);
        const long long lower = (long long)floor(index);
        if ((t & 1) == 0) weights[(size_t)b * m + rq.first + (t >> 1)] = index - (double)lower;
        long long r = lower + (t & 1);
        if (r > c - 1) r = c - 1;
        if (r < 0) r = 0;
        e.rank[t] = r;
        e.prefix[t] = 0;
        e.slot[t] = 0;
      }
      if (rq.first == 0) {
        count[b] = (double)c;
        if (has_nan) has_nan[b] = (uint8_t)(e.nan != 0);
      }
    }
    __syncthreads();
  }
  constexpr int BINS = LEVEL == 0 ? kBins0 : select_bins(LEVEL);
  if (w < e.nt) {
    const unsigned* h = LEVEL == 0 ? hist0 + (size_t)b * kBins0
                                   : hist + ((size_t)b * slots + e.slot[w]) * BINS;
    long long r = e.rank[w];
    int bin = BINS - 1;
    for (int c0 = 0; c0 < BINS; c0 += 32) {
      const unsigned v = h[c0 + lane];
      unsigned long long incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
      }
      const unsigned long long tot = __shfl_sync(0xffffffffu, incl, 31);
      if ((unsigned long long)r < tot) {
        const unsigned hit = __ballot_sync(0xffffffffu, (unsigned long long)r < incl);
        const int l = __ffs(hit) - 1;
        const unsigned long long before = __shfl_sync(0xffffffffu, incl - v, l);
        bin = c0 + l;
        r -= (long long)before;
        break;
      }
      r -= (long long)tot;
      if (c0 + 32 >= BINS) r += (long long)__shfl_sync(0xffffffffu, v, 31);  // not found: the last bin
    }
    __syncwarp();
    if (lane == 0) {
      e.rank[w] = r;
      e.prefix[w] = (e.prefix[w] << (LEVEL == 2 ? 10 : 11)) | (unsigned)bin;
      if (LEVEL == 2) values[(size_t)b * 2 * m + 2 * rq.first + w] = key_value(e.prefix[w]);
    }
  }
  if (LEVEL < 2) {
    __syncthreads();
    if (threadIdx.x == 0) {
      int nu = 0;
      for (int t = 0; t < e.nt; ++t) {
        const unsigned p = e.prefix[t];
        int u = 0;
        while (u < nu && e.uniq[u] < p) ++u;
        if (u == nu || e.uniq[u] != p) {
          for (int s = nu; s > u; --s) e.uniq[s] = e.uniq[s - 1];
          e.uniq[u] = p;
          ++nu;
        }
      }
      e.nuniq = nu;
      for (int t = 0; t < e.nt; ++t) {
        int u = 0;
        while (e.uniq[u] != e.prefix[t]) ++u;
        e.slot[t] = u;
      }
    }
  }
}

// ---- histogram standardization ---------------------------------------------------------
// Per element b (one block): np.percentile's "linear" value of each quantile from its two order
// statistics, then the fp32 map tables of _apply_histogram_standardization
// (histogram_standardization.py:283-300), each op rounded as the reference's:
//   pv   = a + d*g  (g < 0.5)  or  b - d*(1 - g),  d = b - a in fp32, the rest in fp64 (numpy's
//          _lerp on an fp32 array); NaN when the element holds a NaN
//   il   = fp32(pv);  din = il[j+1] - il[j], +inf where |din| < fp32(1e-5)
//   s[j] = (lm[j+1] - lm[j]) / din;  c[j] = lm[j] - s[j]*il[j];  edges = il[1 .. m-2]
// tables[b] = {s[0..m-2], c[0..m-2], edges[0..m-3]} (stride 3*(m-1)).
__device__ __forceinline__ float percentile_f32(const float* v, const double* w, bool nan, int j) {
  if (nan) return __int_as_float(0x7fffffff);
  const float a = v[2 * j], b = v[2 * j + 1];
  const double g = w[j], d = (double)__fsub_rn(b, a);
  const double pv = g >= 0.5 ? __dsub_rn((double)b, __dmul_rn(d, __dsub_rn(1.0, g))) : __dadd_rn((double)a, __dmul_rn(d, g));
  return __double2float_rn(pv);
}

__global__ void histogram_tables_kernel(const float* __restrict__ values, const double* __restrict__ weights,
                                        const uint8_t* __restrict__ has_nan, const float* __restrict__ lm, int m,
                                        float* __restrict__ tables) {
  const int b = blockIdx.x;
  const float* v = values + (size_t)b * 2 * m;
  const double* w = weights + (size_t)b * m;
  const bool nan = has_nan && has_nan[b];
  float* s = tables + (size_t)b * 3 * (m - 1);
  float* c = s + (m - 1);
  float* edges = c + (m - 1);
  for (int j = threadIdx.x; j < m - 1; j += blockDim.x) {
    const float il0 = percentile_f32(v, w, nan, j), il1 = percentile_f32(v, w, nan, j + 1);
    float din = __fsub_rn(il1, il0);
    if (fabsf(din) < 1e-5f) din = __int_as_float(0x7f800000);
    const float slope = __fdiv_rn(__fsub_rn(lm[j + 1], lm[j]), din);
    s[j] = slope;
    c[j] = __fsub_rn(lm[j], __fmul_rn(slope, il0));
    if (j > 0) edges[j - 1] = il0;
  }
}

// y = rn(rn(s[bin] * x) + c[bin]), bin = torch.bucketize(x, edges, right=False) as ATen's CUDA
// lower bound computes it (NaN goes past the last edge), stored with torch's cast; src may be dst
template <typename T>
__global__ void __launch_bounds__(256)
histogram_map_kernel(const T* src, T* dst, int64_t per_elem, const float* __restrict__ tables, int m) {
  extern __shared__ float tab[];
  const int b = blockIdx.y;
  const int nseg = m - 1, ne = m - 2;
  for (int t = threadIdx.x; t < 3 * nseg; t += blockDim.x) tab[t] = tables[(size_t)b * 3 * nseg + t];
  __syncthreads();
  const float* s = tab;
  const float* c = tab + nseg;
  const float* edges = tab + 2 * nseg;
  auto f = [&](float x) {
    int lo = 0, hi = ne;
    while (lo < hi) {
      const int mid = lo + ((hi - lo) >> 1);
      if (!(edges[mid] >= x)) lo = mid + 1;
      else hi = mid;
    }
    return __fadd_rn(__fmul_rn(s[lo], x), c[lo]);
  };
  const T* x = src + (int64_t)b * per_elem;
  T* y = dst + (int64_t)b * per_elem;
  constexpr int V = 16 / sizeof(T);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t done = 0;
  if ((((uintptr_t)x | (uintptr_t)y) & 15) == 0) {
    const int64_t nv = per_elem / V;
    for (int64_t t = t0; t < nv; t += stride) {
      Pack<T> pk;
      pk.raw = reinterpret_cast<const uint4*>(x)[t];
#pragma unroll
      for (int j = 0; j < V; ++j) pk.e[j] = from_float<T>(f(to_float(pk.e[j])));
      reinterpret_cast<uint4*>(y)[t] = pk.raw;
    }
    done = nv * V;
  }
  for (int64_t t = done + t0; t < per_elem; t += stride) y[t] = from_float<T>(f(to_float(x[t])));
}

// ---- rescale ---------------------------------------------------------------------------
// flags: 1 clamp, 2 sub, 4 div, 8 mul, 16 add; keep[b] == 0 -> copy the row
template <int V>
__global__ void __launch_bounds__(256)
rescale_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t per_elem, float lo, float hi,
               const float* __restrict__ sub, const float* __restrict__ div, const float* __restrict__ mul,
               const float* __restrict__ add, const uint8_t* __restrict__ keep, int flags) {
  const int b = blockIdx.y;
  const float* x = src + (int64_t)b * per_elem;
  float* y = dst + (int64_t)b * per_elem;
  const bool copy = keep && !keep[b];
  const float fs = sub ? sub[b] : 0.f, fd = div ? div[b] : 1.f, fm = mul ? mul[b] : 1.f, fa = add ? add[b] : 0.f;
  auto f = [&](float v) {
    if (copy) return v;
    if (flags & 1) v = fminf(fmaxf(v, lo), hi);  // Tensor.clamp(min, max)
    if (flags & 2) v = __fsub_rn(v, fs);
    if (flags & 4) v = __fdiv_rn(v, fd);
    if (flags & 8) v = __fmul_rn(v, fm);
    if (flags & 16) v = __fadd_rn(v, fa);
    return v;
  };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (V == 4) {
    const float4* p = reinterpret_cast<const float4*>(x);
    float4* o = reinterpret_cast<float4*>(y);
    for (int64_t t = t0; t < (per_elem >> 2); t += stride) {
      float4 v = __ldg(p + t);
      v.x = f(v.x); v.y = f(v.y); v.z = f(v.z); v.w = f(v.w);
      o[t] = v;
    }
  } else {
    for (int64_t t = t0; t < per_elem; t += stride) y[t] = f(__ldg(x + t));
  }
}

}  // namespace tio

using namespace tio;

extern "C" int tio_moments(const float* src, const uint8_t* mask, int64_t n, double* out3, void* stream) {
  TIO_CHECK_ARG(src && out3 && n > 0, "tio_moments: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  TIO_CHECK_CUDA(cudaMemsetAsync(out3, 0, 3 * sizeof(double), st));
  int blocks = (int)((n / 4 + 255) / 256);
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  if (blocks < 1) blocks = 1;
  moments_kernel<<<blocks, 256, 0, st>>>(src, mask, n, out3);
  TIO_CHECK_LAUNCH();
  return 0;
}

namespace {

struct SelectLayout {
  SelectElem* state;
  unsigned* hist0;  // [B][2048]
  unsigned* hist;   // [B][slots][2048]
  int slots;
  size_t bytes;
};

size_t align16(size_t n) { return (n + 15) / 16 * 16; }

SelectLayout select_layout(void* ws, int B, int m) {
  SelectLayout l;
  l.slots = 2 * m < kSlots ? 2 * m : kSlots;
  unsigned char* p = (unsigned char*)ws;
  const size_t s0 = align16((size_t)B * sizeof(SelectElem));
  const size_t s1 = align16((size_t)B * kBins0 * sizeof(unsigned));
  const size_t s2 = (size_t)B * l.slots * kBins1 * sizeof(unsigned);
  l.state = (SelectElem*)p;
  l.hist0 = (unsigned*)(p + s0);
  l.hist = (unsigned*)(p + s0 + s1);
  l.bytes = s0 + s1 + s2;
  return l;
}

template <typename T, int LEVEL>
int launch_select_hist(const void* src, const uint8_t* mask, int B, int64_t per_elem, const SelectLayout& l,
                       cudaStream_t st) {
  const int bins = LEVEL == 0 ? kBins0 : select_bins(LEVEL);
  const int slots = LEVEL == 0 ? 1 : l.slots;
  const size_t smem = (size_t)slots * bins * sizeof(unsigned) + kBins0 * sizeof(unsigned short);
  auto kernel = select_hist_kernel<T, LEVEL>;
  TIO_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int per_sm = smem > 110 * 1024 ? 1 : 2;  // 2048 threads per SM
  int bx = (num_sms() * per_sm + B - 1) / B;
  const int64_t work = (per_elem + (int64_t)kSelectThreads * (16 / sizeof(T)) - 1) / ((int64_t)kSelectThreads * (16 / sizeof(T)));
  if (bx > work) bx = (int)work;
  if (bx < 1) bx = 1;
  kernel<<<dim3(bx, B), kSelectThreads, smem, st>>>((const T*)src, mask, per_elem, l.state,
                                                   LEVEL == 0 ? l.hist0 : l.hist, l.slots);
  TIO_CHECK_LAUNCH();
  return 0;
}

template <typename T>
int run_select(const void* src, const uint8_t* mask, int B, int64_t per_elem, const double* q_host, int m,
               float* values, double* weights, double* count, uint8_t* has_nan, const SelectLayout& l,
               cudaStream_t st) {
  int rc;
  select_reset_kernel<<<B, 1, 0, st>>>(l.state);
  TIO_CHECK_CUDA(cudaMemsetAsync(l.hist0, 0, (size_t)B * kBins0 * sizeof(unsigned), st));
  if ((rc = launch_select_hist<T, 0>(src, mask, B, per_elem, l, st))) return rc;
  const size_t hbytes = (size_t)B * l.slots * kBins1 * sizeof(unsigned);
  for (int first = 0; first < m; first += kQuantPerRound) {
    RoundQ rq;
    rq.first = first;
    rq.nq = m - first < kQuantPerRound ? m - first : kQuantPerRound;
    for (int j = 0; j < kQuantPerRound; ++j) rq.q[j] = j < rq.nq ? q_host[first + j] : 0.0;
    select_scan_kernel<0><<<B, kSelectThreads, 0, st>>>(l.state, l.hist0, l.hist, l.slots, rq, per_elem,
                                                         mask != nullptr, m, values, weights, count, has_nan);
    TIO_CHECK_CUDA(cudaMemsetAsync(l.hist, 0, hbytes, st));
    if ((rc = launch_select_hist<T, 1>(src, mask, B, per_elem, l, st))) return rc;
    select_scan_kernel<1><<<B, kSelectThreads, 0, st>>>(l.state, l.hist0, l.hist, l.slots, rq, per_elem,
                                                         mask != nullptr, m, values, weights, count, has_nan);
    TIO_CHECK_CUDA(cudaMemsetAsync(l.hist, 0, hbytes, st));
    if ((rc = launch_select_hist<T, 2>(src, mask, B, per_elem, l, st))) return rc;
    select_scan_kernel<2><<<B, kSelectThreads, 0, st>>>(l.state, l.hist0, l.hist, l.slots, rq, per_elem,
                                                         mask != nullptr, m, values, weights, count, has_nan);
    TIO_CHECK_LAUNCH();
  }
  return 0;
}

}  // namespace

extern "C" size_t tio_quantiles_batched_workspace_bytes(int B, int m) {
  if (B < 1 || m < 1) return 0;
  return select_layout(nullptr, B, m).bytes;
}

extern "C" int tio_quantiles_batched(const void* src, int dtype, const uint8_t* mask, int B, int64_t per_elem,
                                     const double* q_host, int m, float* values, double* weights, double* count,
                                     uint8_t* has_nan, void* workspace, size_t workspace_bytes, void* stream) {
  TIO_CHECK_ARG(src && q_host && values && weights && count && workspace, "tio_quantiles_batched: null pointer");
  TIO_CHECK_ARG(B >= 1 && B <= 65535 && per_elem > 0 && per_elem <= (int64_t)UINT32_MAX && m >= 1,
                "tio_quantiles_batched: need 1 <= B <= 65535, 0 < per_elem < 2^32 and m >= 1");
  TIO_CHECK_ARG(workspace_bytes >= tio_quantiles_batched_workspace_bytes(B, m) && ((uintptr_t)workspace & 15) == 0,
                "tio_quantiles_batched: workspace too small or misaligned");
  for (int t = 0; t < m; ++t)
    TIO_CHECK_ARG(q_host[t] >= 0.0 && q_host[t] <= 1.0, "Only values 0 <= q <= 1 are supported, but got %g", q_host[t]);
  const SelectLayout l = select_layout(workspace, B, m);
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_SELECT(T) return run_select<T>(src, mask, B, per_elem, q_host, m, values, weights, count, has_nan, l, st)
  TIO_IMAGE_DISPATCH(dtype, "tio_quantiles_batched", TIO_SELECT)
#undef TIO_SELECT
  return 0;
}

extern "C" size_t tio_quantiles_workspace_bytes(void) { return tio_quantiles_batched_workspace_bytes(1, 2); }

extern "C" int tio_quantiles(const float* src, const uint8_t* mask, int64_t n, const double* q_host, int m,
                             float* values, double* weights, double* count, void* workspace,
                             size_t workspace_bytes, void* stream) {
  TIO_CHECK_ARG(src && q_host && values && weights && count && workspace, "tio_quantiles: null pointer");
  TIO_CHECK_ARG(n > 0 && m >= 1 && m <= 2, "tio_quantiles: need n > 0 and 1 <= m <= %d", 2);
  return tio_quantiles_batched(src, TIO_F32, mask, 1, n, q_host, m, values, weights, count, nullptr, workspace,
                               workspace_bytes, stream);
}

extern "C" int tio_histogram_tables(const float* values, const double* weights, const uint8_t* has_nan,
                                    const float* landmarks, int B, int m, float* tables, void* stream) {
  TIO_CHECK_ARG(values && weights && landmarks && tables, "tio_histogram_tables: null pointer");
  TIO_CHECK_ARG(B >= 1 && m >= 2, "tio_histogram_tables: need B >= 1 and at least 2 landmarks");
  histogram_tables_kernel<<<B, 32, 0, (cudaStream_t)stream>>>(values, weights, has_nan, landmarks, m, tables);
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_histogram_map(const void* src, void* dst, int dtype, int B, int64_t per_elem,
                                 const float* tables, int m, void* stream) {
  TIO_CHECK_ARG(src && dst && tables, "tio_histogram_map: null pointer");
  TIO_CHECK_ARG(B >= 1 && B <= 65535 && per_elem > 0 && m >= 2, "tio_histogram_map: bad sizes");
  const size_t smem = (size_t)3 * (m - 1) * sizeof(float);
  TIO_CHECK_ARG(smem <= 48 * 1024, "tio_histogram_map: %d landmarks do not fit in shared memory", m);
  cudaStream_t st = (cudaStream_t)stream;
#define TIO_MAP(T)                                                                                  \
  {                                                                                                 \
    constexpr int V = 16 / sizeof(T);                                                               \
    int64_t bx = (per_elem + 256 * V - 1) / (256 * V);                                              \
    const int64_t cap = (num_sms() * 8 + B - 1) / B;                                                \
    if (bx > cap) bx = cap;                                                                         \
    histogram_map_kernel<T><<<dim3((unsigned)bx, B), 256, smem, st>>>((const T*)src, (T*)dst, per_elem, \
                                                                      tables, m);                   \
  }
  TIO_IMAGE_DISPATCH(dtype, "tio_histogram_map", TIO_MAP)
#undef TIO_MAP
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_rescale(const float* src, float* dst, int B, int64_t per_elem, float lo, float hi,
                           const float* sub, const float* div, const float* mul, const float* add,
                           const uint8_t* keep, int flags, void* stream) {
  TIO_CHECK_ARG(src && dst && B > 0 && per_elem > 0, "tio_rescale: bad arguments");
  TIO_CHECK_ARG((flags & ~31) == 0, "tio_rescale: unknown flag bits %d", flags);
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = ((per_elem & 3) == 0) && (((uintptr_t)src | (uintptr_t)dst) & 15) == 0;
  const int64_t work = vec ? per_elem / 4 : per_elem;
  int bx = (int)((work + 255) / 256);
  const int cap = (num_sms() * 16 + B - 1) / B;
  if (bx > cap) bx = cap < 1 ? 1 : cap;
  TIO_CHECK_ARG(B <= 65535, "tio_rescale: batch too large");
  dim3 grid(bx, B);
  if (vec) rescale_kernel<4><<<grid, 256, 0, st>>>(src, dst, per_elem, lo, hi, sub, div, mul, add, keep, flags);
  else rescale_kernel<1><<<grid, 256, 0, st>>>(src, dst, per_elem, lo, hi, sub, div, mul, add, keep, flags);
  TIO_CHECK_LAUNCH();
  return 0;
}

// fft_lines.cuh — the shared-memory line FFT of spike.cu and ghosting.cu: a mixed-radix Stockham
// FFT of every length up to 4096 points, several lines per CTA.
//
// Lines of length n are transformed in shared memory (natural order in and out, two buffers).
// Stage with radix R after radices of product ns:
//   for butterfly j: v[r] = in[j + r n/R] * w^(r (j % ns)),  w = exp(-2 pi i / (ns R)),
//                    v = DFT_R(v),  out[(j - j % ns) R + j % ns + r ns] = v[r]
// Every twiddle is W[m] = exp(-2 pi i m / n) of one table, since ns R divides n.  The inverse is
// the same forward transform: ifft(Y) = conj(fft(conj(Y))) / n.
//
// Everything here has internal linkage: each translation unit that includes it gets its own copy.
#pragma once

#include <cstddef>

namespace tio {

namespace {

constexpr int kMaxAxis = 4096;     // longest FFT axis (a line of both buffers + table fits in smem)
constexpr int kLinePoints = 4096;  // complex points per buffer a CTA of the FFT passes holds
constexpr int kMaxLines = 16;      // lines per CTA
constexpr int kMaxStages = 16;

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 mul_minus_i(float2 a) { return make_float2(a.y, -a.x); }

struct FftPlan {
  int n, stages;
  int radix[kMaxStages];
};

__device__ void build_table(float2* W, int n) {
  for (int m = threadIdx.x; m < n; m += blockDim.x) {
    double s, c;
    sincospi(-2.0 * (double)m / (double)n, &s, &c);
    W[m] = make_float2((float)c, (float)s);
  }
}

__device__ __forceinline__ void dft2(float2* v) {
  const float2 a = v[0];
  v[0] = cadd(a, v[1]);
  v[1] = csub(a, v[1]);
}

__device__ __forceinline__ void dft4(float2& x0, float2& x1, float2& x2, float2& x3) {
  const float2 t0 = cadd(x0, x2), t1 = csub(x0, x2), t2 = cadd(x1, x3), t3 = mul_minus_i(csub(x1, x3));
  x0 = cadd(t0, t2);
  x2 = csub(t0, t2);
  x1 = cadd(t1, t3);
  x3 = csub(t1, t3);
}

__device__ __forceinline__ void dft8(float2* v) {
  constexpr float h = 0.70710678118654752f;
  float2 a[4], b[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    a[k] = cadd(v[k], v[k + 4]);
    b[k] = csub(v[k], v[k + 4]);
  }
  b[1] = make_float2(h * (b[1].x + b[1].y), h * (b[1].y - b[1].x));   // * exp(-i pi / 4)
  b[2] = mul_minus_i(b[2]);                                             // * exp(-i pi / 2)
  b[3] = make_float2(h * (b[3].y - b[3].x), -h * (b[3].x + b[3].y));  // * exp(-3 i pi / 4)
  dft4(a[0], a[1], a[2], a[3]);
  dft4(b[0], b[1], b[2], b[3]);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    v[2 * k] = a[k];
    v[2 * k + 1] = b[k];
  }
}

// radix 3, 5, 7: the R-point DFT unrolled in registers, its constants W[(r q mod R) n / R]
template <int R>
__device__ __forceinline__ void dft_odd(float2* v, const float2* W, int n) {
  float2 out[R];
#pragma unroll
  for (int q = 0; q < R; ++q) {
    float2 acc = v[0];
#pragma unroll
    for (int r = 1; r < R; ++r) {
      const float2 w = W[((r * q) % R) * (n / R)];
      acc = cadd(acc, cmul(v[r], w));
    }
    out[q] = acc;
  }
#pragma unroll
  for (int q = 0; q < R; ++q) v[q] = out[q];
}

template <int R>
__device__ void stage_fixed(const float2* in, float2* out, int lines, int n, int S, int ns, const float2* W) {
  const int nb = n / R, step = n / (ns * R);
  for (int g = threadIdx.x; g < lines * nb; g += blockDim.x) {
    const int line = g / nb, j = g - line * nb, k = j % ns;
    const float2* a = in + line * S;
    float2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      v[r] = a[j + r * nb];
      if (r > 0 && k > 0) v[r] = cmul(v[r], W[k * r * step]);
    }
    if constexpr (R == 2) dft2(v);
    else if constexpr (R == 4) dft4(v[0], v[1], v[2], v[3]);
    else if constexpr (R == 8) dft8(v);
    else dft_odd<R>(v, W, n);
    float2* b = out + line * S + (j - k) * R + k;
#pragma unroll
    for (int r = 0; r < R; ++r) b[r * ns] = v[r];
  }
}

// any other prime p: one thread per output, a direct p-point DFT with the twiddle folded in
__device__ void stage_generic(const float2* in, float2* out, int lines, int n, int S, int ns, int p,
                              const float2* W) {
  const int nb = n / p, L = ns * p, step = n / L;
  for (int g = threadIdx.x; g < lines * n; g += blockDim.x) {
    const int line = g / n, o = g - line * n, q = o / nb, j = o - q * nb, k = j % ns;
    const float2* a = in + line * S + j;
    const int e = k + q * ns;  // output exponent: r (k + q ns) over L
    float2 acc = make_float2(0.0f, 0.0f);
    int m = 0;
    for (int r = 0; r < p; ++r) {
      acc = cadd(acc, cmul(a[r * nb], W[m * step]));
      m += e;
      if (m >= L) m -= L;
    }
    out[line * S + (j - k) * p + k + q * ns] = acc;
  }
}

// transforms `lines` lines of a (stride S) in place of a / b; returns the buffer holding the result
__device__ float2* fft_lines(float2* a, float2* b, int lines, int S, const FftPlan& plan, const float2* W) {
  int ns = 1;
  for (int s = 0; s < plan.stages; ++s) {
    __syncthreads();
    const int R = plan.radix[s];
    switch (R) {
      case 2: stage_fixed<2>(a, b, lines, plan.n, S, ns, W); break;
      case 3: stage_fixed<3>(a, b, lines, plan.n, S, ns, W); break;
      case 4: stage_fixed<4>(a, b, lines, plan.n, S, ns, W); break;
      case 5: stage_fixed<5>(a, b, lines, plan.n, S, ns, W); break;
      case 7: stage_fixed<7>(a, b, lines, plan.n, S, ns, W); break;
      case 8: stage_fixed<8>(a, b, lines, plan.n, S, ns, W); break;
      default: stage_generic(a, b, lines, plan.n, S, ns, R, W);
    }
    ns *= R;
    float2* t = a;
    a = b;
    b = t;
  }
  __syncthreads();
  return a;
}

FftPlan make_plan(int n) {
  FftPlan plan = {};
  plan.n = n;
  int rest = n;
  auto take = [&](int r) {
    while (rest % r == 0 && plan.stages < kMaxStages) {
      plan.radix[plan.stages++] = r;
      rest /= r;
    }
  };
  take(8);
  take(4);
  take(2);
  take(3);
  take(5);
  take(7);
  for (int p = 11; rest > 1; p += 2) take(p);
  return plan;
}

int fft_lines_for(int n) {
  const int lines = kLinePoints / n;
  return lines < 1 ? 1 : (lines > kMaxLines ? kMaxLines : lines);
}

int line_stride(int n) { return n % 2 ? n : n + 1; }  // odd: the strided loads hit distinct banks

size_t fft_smem(int n, int lines) { return ((size_t)n + 2 * (size_t)lines * line_stride(n)) * sizeof(float2); }

}  // namespace

}  // namespace tio

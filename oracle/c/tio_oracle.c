/*
 * tio_oracle.c — CPU oracle, part 2: plain-C restatement of the arithmetic.
 *
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.  Linked/loaded only by tests/,
 * __graft_entry__.smoke() and bench.py's CPU-baseline leg.
 *
 * The reference (TorchIO 2.0.0a2 @ 2b019d2) computes this path with PyTorch
 * ATen CPU ops (torch 2.11.0, build 70d99e9; not vendored under
 * /root/reference).  This file restates those ops' published algorithms as
 * scalar fp32 loops, with the operation ORDER of the CPU kernels, so the CUDA
 * kernels can be checked bit-for-bit where the domain is discrete (nearest
 * labels, mask decisions) without importing torch.  Pinned by
 * tests/test_oracle_c.py against the golden vectors produced by the
 * unmodified reference (tests/golden/).
 *
 * Entry points mirror include/tio_b200.h with prefix orc_ and host pointers.
 * Compile with -O2 -ffp-contract=off: every rounding below is intentional.
 *
 * Citations: "spatial.py" = src/torchio/transforms/spatial/spatial.py etc.
 * ATen behaviour restated (names only; no ATen source is available offline):
 *   grid_sampler_3d (CPU, align_corners=True, zeros padding), bilinear/nearest
 *   upsample_trilinear3d (CPU, align_corners=True)
 *   normal_fill / mt19937 (CPU generator)
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { ORC_F32 = 0, ORC_U8, ORC_I8, ORC_I16, ORC_I32, ORC_I64 };

/* ---- helpers ---------------------------------------------------------- */

static inline float load_as_f32(const void* p, int dtype, int64_t idx) {
  switch (dtype) {
    case ORC_F32: return ((const float*)p)[idx];
    case ORC_U8: return (float)((const uint8_t*)p)[idx];
    case ORC_I8: return (float)((const int8_t*)p)[idx];
    case ORC_I16: return (float)((const int16_t*)p)[idx];
    case ORC_I32: return (float)((const int32_t*)p)[idx];
    default: return (float)((const int64_t*)p)[idx];
  }
}

static inline void store_from_f32(void* p, int dtype, int64_t idx, float v) {
  switch (dtype) { /* Tensor.to(int dtype): truncation toward zero */
    case ORC_F32: ((float*)p)[idx] = v; break;
    case ORC_U8: ((uint8_t*)p)[idx] = (uint8_t)(int64_t)v; break;
    case ORC_I8: ((int8_t*)p)[idx] = (int8_t)(int64_t)v; break;
    case ORC_I16: ((int16_t*)p)[idx] = (int16_t)(int64_t)v; break;
    case ORC_I32: ((int32_t*)p)[idx] = (int32_t)(int64_t)v; break;
    default: ((int64_t*)p)[idx] = (int64_t)v; break;
  }
}

static inline size_t dtype_size(int dtype) {
  switch (dtype) {
    case ORC_F32: case ORC_I32: return 4;
    case ORC_U8: case ORC_I8: return 1;
    case ORC_I16: return 2;
    default: return 8;
  }
}

/* Source index + weights of ATen's align_corners=True linear upsampling:
 * scale = (in-1)/(out-1) in fp32, real = scale*o, i0 = floor, i1 = i0 + (i0 <
 * in-1), l1 = real - i0, l0 = 1 - l1.  (F.interpolate call sites:
 * spatial.py:2182-2187, bias_field.py:237-242,333-338.) */
static inline void lerp_setup(int n_in, int n_out, int o, int* i0, int* i1,
                              float* l0, float* l1) {
  if (n_in == n_out) { /* ATen shortcut when sizes match */
    *i0 = *i1 = o; *l0 = 1.0f; *l1 = 0.0f; return;
  }
  float scale = n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.0f;
  float real = scale * (float)o;
  int a = (int)floorf(real);
  if (a > n_in - 1) a = n_in - 1;
  float lam = real - (float)a;
  if (lam < 0.0f) lam = 0.0f;
  if (lam > 1.0f) lam = 1.0f;
  *i0 = a; *i1 = a + (a < n_in - 1 ? 1 : 0);
  *l1 = lam; *l0 = 1.0f - lam;
}

/* ATen's nested 2-tap combine as compiled in the pinned torch build:
 * fma(w0, v0, round(w1*v1)), innermost axis first (probe-verified bit-exact
 * against F.interpolate on this build). */
static inline float lerp2(float w0, float v0, float w1, float v1) {
  return fmaf(w0, v0, w1 * v1);
}

/* trilinear, align_corners=True, of one coarse channel at output (i,j,k) */
static inline float trilerp(const float* g, int nj, int nk, int64_t sc,
                            int i0, int i1, float a0, float a1,
                            int j0, int j1, float b0, float b1,
                            int k0, int k1, float c0, float c1) {
  /* g indexed [(i*nj + j)*nk + k] * sc  (sc = element stride, 3 for the
   * interleaved control grid, 1 for planar bias fields) */
#define G(i, j, k) g[(((int64_t)(i)*nj + (j)) * nk + (k)) * sc]
  float r00 = lerp2(c0, G(i0, j0, k0), c1, G(i0, j0, k1));
  float r01 = lerp2(c0, G(i0, j1, k0), c1, G(i0, j1, k1));
  float r10 = lerp2(c0, G(i1, j0, k0), c1, G(i1, j0, k1));
  float r11 = lerp2(c0, G(i1, j1, k0), c1, G(i1, j1, k1));
#undef G
  float r0 = lerp2(b0, r00, b1, r01);
  float r1 = lerp2(b0, r10, b1, r11);
  return lerp2(a0, r0, a1, r1);
}

/* IEEE fp32 a/b (plain C division is correctly rounded) */
static inline float fdiv(float a, float b) { return a / b; }

/* ---- K1: resample ------------------------------------------------------ */

/* [p,1] @ M^T as the CPU sgemm evaluates it on the pinned build: a
 * sequential fused-multiply-add chain over k = 0..3 starting from the rounded
 * first product (probe-verified bit-exact, spatial.py:1621-1624). */
static inline float affine_row(const float* m, float pi, float pj, float pk) {
  float acc = pi * m[0];
  acc = fmaf(pj, m[1], acc);
  acc = fmaf(pk, m[2], acc);
  acc = fmaf(1.0f, m[3], acc);
  return acc;
}

/* Geometry of one orc_resample / orc_resample_adjoint call, shared by every voxel. */
typedef struct {
  int I, J, K, OI, OJ, OK, ni, nj, nk, affine_first, mode, has_fill;
  const float *spacing_in, *spacing_out;
  float nm1[3], sm1[3];
} orc_geom;

static orc_geom geom_of(int I, int J, int K, int OI, int OJ, int OK, int ni, int nj, int nk,
                        const float* spacing_in, const float* spacing_out, int affine_first,
                        int mode, int has_fill) {
  orc_geom G;
  G.I = I; G.J = J; G.K = K; G.OI = OI; G.OJ = OJ; G.OK = OK;
  G.ni = ni; G.nj = nj; G.nk = nk;
  G.spacing_in = spacing_in; G.spacing_out = spacing_out;
  G.affine_first = affine_first; G.mode = mode; G.has_fill = has_fill;
  /* max(size-1, 1) (spatial.py:1638-1640) */
  G.nm1[0] = (float)(I - 1 > 1 ? I - 1 : 1);
  G.nm1[1] = (float)(J - 1 > 1 ? J - 1 : 1);
  G.nm1[2] = (float)(K - 1 > 1 ? K - 1 : 1);
  /* ATen un-normalise multiplies by (size - 1) without the max() */
  G.sm1[0] = (float)(I - 1); G.sm1[1] = (float)(J - 1); G.sm1[2] = (float)(K - 1);
  return G;
}

/* What output voxel (oi, oj, ok) reads: its 8 trilinear corners (weight, in-bounds bit, offset
 * in the input volume), whether the fill replaces it, and its nearest-mode voxel (-1: outside).
 * The one per-voxel chain of orc_resample and orc_resample_adjoint, so the adjoint's weights and
 * fill decisions are the forward's. */
typedef struct {
  float w8[8];
  int inb[8];
  int64_t off8[8];
  int use_fill;
  int64_t nn_off;
} orc_voxel;

/* Input-voxel coordinates q of output voxel (oi, oj, ok) (spatial.py:1504-1579), before the
 * grid's normalisation: the sampling points of K1 and of the B-spline pull. */
static void voxel_coords(const orc_geom* G, const float* m, const float* g, int oi, int oj, int ok,
                         float q[3]) {
  float p[3] = {(float)oi, (float)oj, (float)ok};
  float d[3] = {0.f, 0.f, 0.f};
  if (g) { /* spatial.py:2171-2189 */
    int i0, i1, j0, j1, k0, k1; float a0, a1, b0, b1, c0, c1;
    lerp_setup(G->ni, G->OI, oi, &i0, &i1, &a0, &a1);
    lerp_setup(G->nj, G->OJ, oj, &j0, &j1, &b0, &b1);
    lerp_setup(G->nk, G->OK, ok, &k0, &k1, &c0, &c1);
    for (int a = 0; a < 3; ++a)
      d[a] = trilerp(g + a, G->nj, G->nk, 3, i0, i1, a0, a1, j0, j1, b0, b1, k0, k1, c0, c1);
  }
  if (!g) {
    for (int a = 0; a < 3; ++a) q[a] = affine_row(m + 4 * a, p[0], p[1], p[2]);
  } else if (G->affine_first) { /* spatial.py:1570-1573 */
    for (int a = 0; a < 3; ++a)
      q[a] = affine_row(m + 4 * a, p[0], p[1], p[2]) + fdiv(d[a], G->spacing_in[a]);
  } else { /* spatial.py:1574-1577 */
    float e[3];
    for (int a = 0; a < 3; ++a) e[a] = p[a] + fdiv(d[a], G->spacing_out[a]);
    for (int a = 0; a < 3; ++a) q[a] = affine_row(m + 4 * a, e[0], e[1], e[2]);
  }
}

static void resample_voxel(const orc_geom* G, const float* m, const float* g, int oi, int oj,
                           int ok, orc_voxel* v) {
  const int I = G->I, J = G->J, K = G->K;
  const int dims[3] = {I, J, K};
  float q[3];
  voxel_coords(G, m, g, oi, oj, ok, q);
  /* normalise (spatial.py:1646) then ATen un-normalise */
  float u[3];
  for (int a = 0; a < 3; ++a) {
    float gn = fdiv(2.0f * q[a], G->nm1[a]) - 1.0f;
    u[a] = ((gn + 1.0f) / 2.0f) * G->sm1[a];
  }
  /* trilinear corner weights (always needed for the mask) */
  float fl0[3], lo[3], hi[3]; int64_t c0[3];
  for (int a = 0; a < 3; ++a) {
    fl0[a] = floorf(u[a]);
    c0[a] = (int64_t)fl0[a];
    lo[a] = (float)(c0[a] + 1) - u[a]; /* weight of corner c0 */
    hi[a] = u[a] - (float)c0[a];       /* weight of corner c0+1 */
  }
  /* ATen order: x(=i) fastest, then y(=j), then z(=k); weight =
   * (wx*wy)*wz; accumulate mul-then-add from 0 over in-bounds corners */
  for (int t = 0; t < 8; ++t) {
    int di = t & 1, dj = (t >> 1) & 1, dk = (t >> 2) & 1;
    float wi = di ? hi[0] : lo[0], wj = dj ? hi[1] : lo[1], wk = dk ? hi[2] : lo[2];
    v->w8[t] = (wi * wj) * wk;
    int64_t ci = c0[0] + di, cj = c0[1] + dj, ck = c0[2] + dk;
    v->inb[t] = ci >= 0 && ci < I && cj >= 0 && cj < J && ck >= 0 && ck < K;
    v->off8[t] = (ci * J + cj) * K + ck;
  }
  v->use_fill = 0;
  if (G->has_fill) {
    float msum = 0.0f;
    for (int t = 0; t < 8; ++t) if (v->inb[t]) msum = msum + 1.0f * v->w8[t];
    v->use_fill = !(msum > 0.5f);
  }
  v->nn_off = -1;
  if (G->mode == 0) { /* nearest: round-half-even */
    int64_t r[3]; int ok_in = 1;
    for (int a = 0; a < 3; ++a) {
      r[a] = (int64_t)nearbyintf(u[a]);
      if (r[a] < 0 || r[a] >= dims[a]) ok_in = 0;
    }
    if (ok_in) v->nn_off = (r[0] * J + r[1]) * K + r[2];
  }
}

int orc_resample(const void* src, void* dst, int dtype,
                 int B, int C, int I, int J, int K,
                 int OI, int OJ, int OK,
                 const float* mat, const float* cp, const uint8_t* flags,
                 int ni, int nj, int nk,
                 const float* spacing_in, const float* spacing_out,
                 int affine_first, int mode, const float* fill) {
  const int64_t n_in = (int64_t)I * J * K, n_out = (int64_t)OI * OJ * OK;
  const size_t es = dtype_size(dtype);
  const orc_geom G = geom_of(I, J, K, OI, OJ, OK, ni, nj, nk, spacing_in, spacing_out,
                             affine_first, mode, fill != NULL);
  for (int b = 0; b < B; ++b) {
    const uint8_t fl = flags ? flags[b] : 0;
    if (fl & 1u) { /* pass-through row: exact copy (spatial.py:1101-1106) */
      memcpy((char*)dst + (size_t)b * C * n_out * es,
             (const char*)src + (size_t)b * C * n_in * es, (size_t)C * n_in * es);
      continue;
    }
    const float* m = mat + (size_t)b * 12;
    const float* g = (cp && (fl & 2u)) ? cp + (size_t)b * ni * nj * nk * 3 : NULL;
    for (int oi = 0; oi < OI; ++oi)
      for (int oj = 0; oj < OJ; ++oj)
        for (int ok = 0; ok < OK; ++ok) {
          orc_voxel vx;
          resample_voxel(&G, m, g, oi, oj, ok, &vx);
          const int64_t o_off = ((int64_t)oi * OJ + oj) * OK + ok;
          for (int c = 0; c < C; ++c) {
            const int64_t ibase = ((int64_t)b * C + c) * n_in;
            const int64_t obase = ((int64_t)b * C + c) * n_out;
            float v;
            if (vx.use_fill) {
              v = fill[c];
            } else if (mode == 0) {
              v = vx.nn_off >= 0 ? load_as_f32(src, dtype, ibase + vx.nn_off) : 0.0f;
            } else {
              v = 0.0f;
              for (int t = 0; t < 8; ++t)
                if (vx.inb[t]) v = v + load_as_f32(src, dtype, ibase + vx.off8[t]) * vx.w8[t];
            }
            store_from_f32(dst, dtype, obase + o_off, v);
          }
        }
  }
  return 0;
}

/* The fp32 coordinates q (B, OI, OJ, OK, 3) at which orc_resample samples each output voxel, in
 * input voxels before the grid's normalisation; pass-through elements get their own voxel's
 * indices (they are copied, not sampled). */
int orc_sampling_coords(float* q, int B, int OI, int OJ, int OK,
                        const float* mat, const float* cp, const uint8_t* flags,
                        int ni, int nj, int nk,
                        const float* spacing_in, const float* spacing_out, int affine_first) {
  /* the coordinates do not depend on the input's shape */
  const orc_geom G = geom_of(1, 1, 1, OI, OJ, OK, ni, nj, nk, spacing_in, spacing_out,
                             affine_first, 1, 0);
  for (int b = 0; b < B; ++b) {
    const uint8_t fl = flags ? flags[b] : 0;
    const float* m = mat + (size_t)b * 12;
    const float* g = (cp && (fl & 2u)) ? cp + (size_t)b * ni * nj * nk * 3 : NULL;
    for (int oi = 0; oi < OI; ++oi)
      for (int oj = 0; oj < OJ; ++oj)
        for (int ok = 0; ok < OK; ++ok) {
          float* out = q + ((((int64_t)b * OI + oi) * OJ + oj) * OK + ok) * 3;
          if (fl & 1u) {
            out[0] = (float)oi; out[1] = (float)oj; out[2] = (float)ok;
          } else {
            voxel_coords(&G, m, g, oi, oj, ok, out);
          }
        }
  }
  return 0;
}

/* Adjoint of orc_resample with respect to its fp32 input, in float64: for every input voxel,
 * grad64 = sum of g * w over the output voxels that read it (g of the fp32 grad_out, w the
 * forward's fp32 weight; product and sum in double), abs64 = sum of |g * w|, and count = the
 * number of terms.  The reference's backward (grid_sampler_3d_backward, then torch.where) adds
 * the same terms in fp32:
 *   - a voxel the forward fills sends nothing (torch.where routes no gradient to it);
 *   - nearest sends g to its rounded voxel when that voxel is inside the volume;
 *   - linear sends g * w to every in-bounds corner, zero weights included, so a NaN or Inf g
 *     reaches them as NaN (NaN * 0 and Inf * 0 are NaN in double as in fp32);
 *   - a pass-through element copies g (the shapes must then be equal).
 * grad64 / abs64 are (B, C, I, J, K) double, count (B, C, I, J, K) int32. */
int orc_resample_adjoint(const float* grad_out, double* grad64, double* abs64, int32_t* count,
                         int B, int C, int I, int J, int K, int OI, int OJ, int OK,
                         const float* mat, const float* cp, const uint8_t* flags,
                         int ni, int nj, int nk,
                         const float* spacing_in, const float* spacing_out,
                         int affine_first, int mode, const float* fill) {
  const int64_t n_in = (int64_t)I * J * K, n_out = (int64_t)OI * OJ * OK;
  const orc_geom G = geom_of(I, J, K, OI, OJ, OK, ni, nj, nk, spacing_in, spacing_out,
                             affine_first, mode, fill != NULL);
  memset(grad64, 0, (size_t)B * C * n_in * sizeof(double));
  memset(abs64, 0, (size_t)B * C * n_in * sizeof(double));
  memset(count, 0, (size_t)B * C * n_in * sizeof(int32_t));
  for (int b = 0; b < B; ++b) {
    const uint8_t fl = flags ? flags[b] : 0;
    if (fl & 1u) {
      if (n_in != n_out) return 1;
      for (int64_t t = 0; t < (int64_t)C * n_in; ++t) {
        const int64_t o = (int64_t)b * C * n_in + t;
        grad64[o] = (double)grad_out[o];
        abs64[o] = fabs((double)grad_out[o]);
        count[o] = 1;
      }
      continue;
    }
    const float* m = mat + (size_t)b * 12;
    const float* g = (cp && (fl & 2u)) ? cp + (size_t)b * ni * nj * nk * 3 : NULL;
    for (int oi = 0; oi < OI; ++oi)
      for (int oj = 0; oj < OJ; ++oj)
        for (int ok = 0; ok < OK; ++ok) {
          orc_voxel vx;
          resample_voxel(&G, m, g, oi, oj, ok, &vx);
          if (vx.use_fill) continue;
          const int64_t o_off = ((int64_t)oi * OJ + oj) * OK + ok;
          for (int c = 0; c < C; ++c) {
            const int64_t ibase = ((int64_t)b * C + c) * n_in;
            const double go = (double)grad_out[((int64_t)b * C + c) * n_out + o_off];
            if (mode == 0) {
              if (vx.nn_off < 0) continue;
              grad64[ibase + vx.nn_off] += go;
              abs64[ibase + vx.nn_off] += fabs(go);
              count[ibase + vx.nn_off] += 1;
              continue;
            }
            for (int t = 0; t < 8; ++t) {
              if (!vx.inb[t]) continue;
              const double p = go * (double)vx.w8[t];
              grad64[ibase + vx.off8[t]] += p;
              abs64[ibase + vx.off8[t]] += fabs(p);
              count[ibase + vx.off8[t]] += 1;
            }
          }
        }
  }
  return 0;
}

int orc_min_sample0(const float* src, int C, int64_t n, float* fill) {
  for (int c = 0; c < C; ++c) {
    float m = src[(int64_t)c * n];
    for (int64_t t = 1; t < n; ++t) {
      float v = src[(int64_t)c * n + t];
      if (v < m || v != v) m = v; /* torch.min propagates NaN */
    }
    fill[c] = m;
  }
  return 0;
}

/* ---- K2: bias field ---------------------------------------------------- */

int orc_bias_field(const float* src, float* dst, int B, int C, int I, int J, int K,
                   const float* coarse, int si, int sj, int sk,
                   const uint8_t* identity, int divide) {
  const int64_t n = (int64_t)I * J * K, ns = (int64_t)si * sj * sk;
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c) {
      const float* x = src + ((int64_t)b * C + c) * n;
      float* y = dst + ((int64_t)b * C + c) * n;
      if (identity && identity[b]) { memmove(y, x, (size_t)n * 4); continue; }
      const float* g = coarse + ((int64_t)b * C + c) * ns;
      for (int i = 0; i < I; ++i) {
        int i0, i1; float a0, a1; lerp_setup(si, I, i, &i0, &i1, &a0, &a1);
        for (int j = 0; j < J; ++j) {
          int j0, j1; float b0, b1; lerp_setup(sj, J, j, &j0, &j1, &b0, &b1);
          for (int k = 0; k < K; ++k) {
            int k0, k1; float c0, c1; lerp_setup(sk, K, k, &k0, &k1, &c0, &c1);
            float f = expf(trilerp(g, sj, sk, 1, i0, i1, a0, a1, j0, j1, b0, b1,
                                   k0, k1, c0, c1));
            int64_t o = ((int64_t)i * J + j) * K + k;
            y[o] = divide ? x[o] / f : x[o] * f;
          }
        }
      }
    }
  return 0;
}

/* ---- K3: blur ---------------------------------------------------------- */

static void blur_axis(const float* x, float* y, int I, int J, int K, int axis,
                      const float* taps, int R, int r) {
  const int dims[3] = {I, J, K};
  const int64_t strides[3] = {(int64_t)J * K, K, 1};
  const int n = dims[axis]; const int64_t s = strides[axis];
  for (int i = 0; i < I; ++i)
    for (int j = 0; j < J; ++j)
      for (int k = 0; k < K; ++k) {
        int pos[3] = {i, j, k};
        int64_t base = ((int64_t)i * J + j) * K + k - (int64_t)pos[axis] * s;
        float acc = 0.0f;
        for (int t = -r; t <= r; ++t) { /* replicate padding = clamp */
          int q = pos[axis] + t; if (q < 0) q = 0; if (q > n - 1) q = n - 1;
          acc = acc + taps[R + t] * x[base + (int64_t)q * s];
        }
        y[((int64_t)i * J + j) * K + k] = acc;
      }
}

int orc_blur(const float* src, float* dst, float* scratch,
             int B, int C, int I, int J, int K,
             const float* taps, const int32_t* radius, int R,
             const uint8_t* identity) {
  const int64_t n = (int64_t)I * J * K; const int W = 2 * R + 1;
  float* tmp[2] = {NULL, NULL};
  tmp[0] = (float*)malloc((size_t)n * 4); tmp[1] = (float*)malloc((size_t)n * 4);
  (void)scratch;
  for (int b = 0; b < B; ++b)
    for (int c = 0; c < C; ++c) {
      const float* x = src + ((int64_t)b * C + c) * n;
      float* y = dst + ((int64_t)b * C + c) * n;
      if (identity && identity[b]) { memcpy(y, x, (size_t)n * 4); continue; }
      const float* cur = x; int flip = 0;
      for (int axis = 0; axis < 3; ++axis) {
        int r = radius[axis * B + b];
        if (r <= 0) continue;
        blur_axis(cur, tmp[flip], I, J, K, axis, taps + ((int64_t)axis * B + b) * W, R, r);
        cur = tmp[flip]; flip ^= 1;
      }
      memcpy(y, cur, (size_t)n * 4);
    }
  free(tmp[0]); free(tmp[1]);
  return 0;
}

/* ---- K4: noise --------------------------------------------------------- */

typedef struct { uint32_t s[624]; int idx; } orc_mt;

static void mt_seed(orc_mt* g, uint32_t seed) {
  g->s[0] = seed;
  for (int j = 1; j < 624; ++j)
    g->s[j] = 1812433253u * (g->s[j - 1] ^ (g->s[j - 1] >> 30)) + (uint32_t)j;
  g->idx = 624;
}

static uint32_t mt_next(orc_mt* g) {
  if (g->idx >= 624) {
    for (int k = 0; k < 624; ++k) {
      uint32_t y = (g->s[k] & 0x80000000u) | (g->s[(k + 1) % 624] & 0x7fffffffu);
      g->s[k] = g->s[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    g->idx = 0;
  }
  uint32_t y = g->s[g->idx++];
  y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
  return y;
}

static inline float mt_uniform24(orc_mt* g) { /* 24-bit mantissa uniform in [0,1) */
  return (float)(mt_next(g) & 0xffffffu) * (1.0f / 16777216.0f);
}

static void box_muller_16(float* d) {
  for (int j = 0; j < 8; ++j) {
    float u1 = 1.0f - d[j], u2 = d[j + 8];
    float radius = sqrtf(-2.0f * logf(u1));
    float theta = 2.0f * 3.14159265358979323846f * u2;
    d[j] = radius * cosf(theta);
    d[j + 8] = radius * sinf(theta);
  }
}

/* torch.randn(n, generator=CPU mt19937(seed)) for n >= 16 (ATen normal_fill):
 * fill with uniforms, Box-Muller per 16-block, and if n % 16 != 0 redo the
 * LAST 16 from fresh uniforms.  Raw words are consumed in flat order;
 * `skip` words are discarded first (a generator shared across calls). */
int orc_randn_mt19937(uint64_t seed, uint64_t skip, uint64_t n, float* z,
                      uint64_t* consumed) {
  orc_mt g; mt_seed(&g, (uint32_t)seed);
  for (uint64_t t = 0; t < skip; ++t) (void)mt_next(&g);
  if (n < 16) return 1; /* scalar path not restated */
  for (uint64_t t = 0; t < n; ++t) z[t] = mt_uniform24(&g);
  for (uint64_t t = 0; t + 15 < n; t += 16) box_muller_16(z + t);
  uint64_t used = n;
  if (n % 16 != 0) {
    float* tail = z + n - 16;
    for (int t = 0; t < 16; ++t) tail[t] = mt_uniform24(&g);
    box_muller_16(tail);
    used += 16;
  }
  if (consumed) *consumed = used;
  return 0;
}

int orc_noise(const float* src, float* dst, int B, int64_t per_elem,
              const float* mean, const float* std, const uint8_t* keep,
              const float* z, const float* z2) {
  for (int b = 0; b < B; ++b)
    for (int64_t t = 0; t < per_elem; ++t) {
      int64_t o = (int64_t)b * per_elem + t;
      float x = src[o];
      if (keep && !keep[b]) { dst[o] = x; continue; }
      float n1 = mean[b] + std[b] * z[o];
      if (z2) {
        float n2 = mean[b] + std[b] * z2[o];
        float s = x + n1;
        dst[o] = sqrtf(s * s + n2 * n2);
      } else {
        dst[o] = x + n1;
      }
    }
  return 0;
}

/* ---- K5: gamma --------------------------------------------------------- */

int orc_gamma(const float* src, float* dst, int B, int64_t per_elem, const float* gamma) {
  for (int b = 0; b < B; ++b)
    for (int64_t t = 0; t < per_elem; ++t) {
      int64_t o = (int64_t)b * per_elem + t;
      float x = src[o];
      float s = (x > 0.0f) ? 1.0f : ((x < 0.0f) ? -1.0f : 0.0f);
      dst[o] = s * powf(fabsf(x), gamma[b]);
    }
  return 0;
}

/* ---- widened rows: index-remap neighbours and patch extraction -----------------
 * Scalar restatements with the signatures of tio_remap / tio_crop_patches
 * (include/tio_b200.h), host pointers.  torch.flip (spatial/flip.py:233-263), the crop
 * slice (crop.py:84-101) and F.pad's constant / replicate / reflect / circular modes
 * (_padding.py:73-104) are one mapping out[o] = in[f(m(o - off))] per spatial axis;
 * PatchSampler._extract_patch (data/sampler.py:54-67) is a sub-block copy. */

static int remap_index(int s, int n, int mode, int* outside) {
  if (s >= 0 && s < n) return s;
  if (mode == 1) return s < 0 ? 0 : n - 1;                 /* replicate */
  if (mode == 2) {                                         /* reflect (edge not repeated) */
    if (n == 1) return 0;
    int period = 2 * (n - 1);
    int r = s % period;
    if (r < 0) r += period;
    return r < n ? r : period - r;
  }
  if (mode == 3) { int r = s % n; return r < 0 ? r + n : r; } /* circular */
  *outside = 1;                                            /* constant */
  return 0;
}

int orc_remap(const void* src, void* dst, int elem_bytes, int B, int C, int I, int J, int K,
              int OI, int OJ, int OK, int off_i, int off_j, int off_k, int mode,
              const void* fill, const uint8_t* flip) {
  const char* s = (const char*)src;
  char* d = (char*)dst;
  for (int b = 0; b < B; ++b) {
    const uint8_t fl = flip ? flip[b] : 0;
    for (int c = 0; c < C; ++c)
      for (int oi = 0; oi < OI; ++oi)
        for (int oj = 0; oj < OJ; ++oj)
          for (int ok = 0; ok < OK; ++ok) {
            int outside = 0;
            int si = remap_index(oi - off_i, I, mode, &outside);
            int sj = remap_index(oj - off_j, J, mode, &outside);
            int sk = remap_index(ok - off_k, K, mode, &outside);
            if (fl & 1) si = I - 1 - si;
            if (fl & 2) sj = J - 1 - sj;
            if (fl & 4) sk = K - 1 - sk;
            int64_t o = ((((int64_t)b * C + c) * OI + oi) * OJ + oj) * OK + ok;
            int64_t i = ((((int64_t)b * C + c) * I + si) * J + sj) * K + sk;
            if (outside) memcpy(d + o * elem_bytes, fill, (size_t)elem_bytes);
            else memcpy(d + o * elem_bytes, s + i * elem_bytes, (size_t)elem_bytes);
          }
  }
  return 0;
}

int orc_crop_patches(const void* src, void* dst, int elem_bytes, int C, int I, int J, int K,
                     int n, const int32_t* corners, int pi, int pj, int pk) {
  const char* s = (const char*)src;
  char* d = (char*)dst;
  for (int p = 0; p < n; ++p)
    for (int c = 0; c < C; ++c)
      for (int i = 0; i < pi; ++i)
        for (int j = 0; j < pj; ++j) {
          int64_t o = ((((int64_t)p * C + c) * pi + i) * pj + j) * pk;
          int64_t q = (((int64_t)c * I + corners[3 * p] + i) * J + corners[3 * p + 1] + j) * K + corners[3 * p + 2];
          memcpy(d + o * elem_bytes, s + q * elem_bytes, (size_t)pk * elem_bytes);
        }
  return 0;
}

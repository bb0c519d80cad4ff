/*
 * components.c — CPU oracle for KeepLargestComponent: connected components restated from the
 * definition in plain C.
 *
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.  Loaded only by tests/ and tools/ through
 * oracle/components.py; torchio_b200 never links it.  Written from the definition (a sequential
 * scan-order union-find), not from the CUDA kernels of torchio_b200/csrc/components.cu, and pinned
 * by tests/test_keep_largest.py against scipy.ndimage.label and the reference's fixtures.
 *
 * Compile with -O2 (no floating-point arithmetic here beyond comparisons).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { ORC_F32 = 0, ORC_U8, ORC_I8, ORC_I16, ORC_I32, ORC_I64 };

static size_t dtype_size(int dtype) {
  switch (dtype) {
    case ORC_F32: case ORC_I32: return 4;
    case ORC_U8: case ORC_I8: return 1;
    case ORC_I16: return 2;
    default: return 8;
  }
}
/* ---- connected components (label/keep_largest.py:63-125) -----------------------------------
 * Restated from the definition, not from the kernels: a sequential scan in C order.  Voxels with
 * part[v] != 0 take part; two neighbouring voxels (6 faces, or all 26 when `fully`) that both take
 * part are connected when their values compare equal (fp32: as floats, so -0 == +0).  Each voxel
 * is joined to its already-visited neighbours, the larger root always linked under the smaller, so
 * every root is the smallest C-order index (i*J + j)*K + k of its component. */

static int values_equal(const void* p, int dtype, int64_t a, int64_t b) {
  switch (dtype) {
    case ORC_F32: return ((const float*)p)[a] == ((const float*)p)[b];
    case ORC_U8: return ((const uint8_t*)p)[a] == ((const uint8_t*)p)[b];
    case ORC_I8: return ((const int8_t*)p)[a] == ((const int8_t*)p)[b];
    case ORC_I16: return ((const int16_t*)p)[a] == ((const int16_t*)p)[b];
    case ORC_I32: return ((const int32_t*)p)[a] == ((const int32_t*)p)[b];
    default: return ((const int64_t*)p)[a] == ((const int64_t*)p)[b];
  }
}

static uint32_t cc_find(uint32_t* parent, uint32_t x) {
  uint32_t r = x;
  while (parent[r] != r) r = parent[r];
  while (parent[x] != r) { /* path compression */
    uint32_t next = parent[x];
    parent[x] = r;
    x = next;
  }
  return r;
}

/* roots[v] = the root of v's component, or 0xFFFFFFFF where part[v] == 0 */
int orc_connected_components(const void* src, int dtype, int I, int J, int K, const uint8_t* part, int fully,
                             uint32_t* roots) {
  const int64_t n = (int64_t)I * J * K;
  if (n >= ((int64_t)1 << 32)) return 1;
  for (int i = 0; i < I; ++i)
    for (int j = 0; j < J; ++j)
      for (int k = 0; k < K; ++k) {
        const uint32_t v = (uint32_t)(((int64_t)i * J + j) * K + k);
        if (!part[v]) {
          roots[v] = 0xFFFFFFFFu;
          continue;
        }
        roots[v] = v;
        for (int di = -1; di <= 0; ++di)
          for (int dj = -1; dj <= 1; ++dj)
            for (int dk = -1; dk <= 1; ++dk) {
              const int before = di < 0 || (di == 0 && (dj < 0 || (dj == 0 && dk < 0)));
              const int face = (di != 0) + (dj != 0) + (dk != 0) == 1;
              if (!before || (!fully && !face)) continue;
              const int ni = i + di, nj = j + dj, nk = k + dk;
              if (ni < 0 || nj < 0 || nj >= J || nk < 0 || nk >= K) continue;
              const uint32_t w = (uint32_t)(((int64_t)ni * J + nj) * K + nk);
              if (!part[w] || !values_equal(src, dtype, v, w)) continue;
              const uint32_t a = cc_find(roots, v), b = cc_find(roots, w);
              if (a < b) roots[b] = a;
              else if (b < a) roots[a] = b;
            }
      }
  for (int64_t v = 0; v < n; ++v)
    if (roots[v] != 0xFFFFFFFFu) roots[v] = cc_find(roots, (uint32_t)v);
  return 0;
}

typedef struct {
  double fvalue;  /* fp32 maps (+0 for -0) */
  int64_t ivalue; /* integer maps */
  uint32_t size, root;
} orc_component;

static int component_order(const void* pa, const void* pb) { /* by value, then largest, then first */
  const orc_component* a = (const orc_component*)pa;
  const orc_component* b = (const orc_component*)pb;
  if (a->fvalue != b->fvalue) return a->fvalue < b->fvalue ? -1 : 1;
  if (a->ivalue != b->ivalue) return a->ivalue < b->ivalue ? -1 : 1;
  if (a->size != b->size) return a->size > b->size ? -1 : 1;
  return a->root < b->root ? -1 : (a->root > b->root);
}

/* In place on B volumes (I, J, K): within each element and each label (a label's voxels are the
 * ones that take part and share its value), every component but the largest (equal sizes: the
 * smallest root) is overwritten with the element_size-byte `fill`.  roots: B * I*J*K. */
int orc_keep_largest(void* data, int dtype, int B, int I, int J, int K, const uint8_t* part, int fully,
                     const void* fill, uint32_t* roots) {
  const int64_t n = (int64_t)I * J * K;
  const size_t es = dtype_size(dtype);
  if (n >= ((int64_t)1 << 32)) return 1;
  uint32_t* size = (uint32_t*)calloc((size_t)(n ? n : 1), sizeof(uint32_t));
  uint8_t* keep = (uint8_t*)calloc((size_t)(n ? n : 1), 1);
  orc_component* comps = (orc_component*)malloc(sizeof(orc_component) * (size_t)(n ? n : 1));
  if (!size || !keep || !comps) return 2;
  for (int b = 0; b < B; ++b) {
    char* d = (char*)data + (size_t)b * n * es;
    uint32_t* r = roots + (size_t)b * n;
    if (orc_connected_components(d, dtype, I, J, K, part + (size_t)b * n, fully, r)) return 1;
    memset(size, 0, sizeof(uint32_t) * (size_t)n);
    memset(keep, 0, (size_t)n);
    for (int64_t v = 0; v < n; ++v)
      if (r[v] != 0xFFFFFFFFu) size[r[v]]++;
    int64_t m = 0;
    for (int64_t v = 0; v < n; ++v) {
      if (r[v] != (uint32_t)v) continue;
      orc_component c;
      c.fvalue = dtype == ORC_F32 ? (double)((const float*)d)[v] + 0.0 : 0.0;
      c.ivalue = 0;
      switch (dtype) {
        case ORC_U8: c.ivalue = ((const uint8_t*)d)[v]; break;
        case ORC_I8: c.ivalue = ((const int8_t*)d)[v]; break;
        case ORC_I16: c.ivalue = ((const int16_t*)d)[v]; break;
        case ORC_I32: c.ivalue = ((const int32_t*)d)[v]; break;
        case ORC_I64: c.ivalue = ((const int64_t*)d)[v]; break;
        default: break;
      }
      c.size = size[v];
      c.root = (uint32_t)v;
      comps[m++] = c;
    }
    qsort(comps, (size_t)m, sizeof(orc_component), component_order);
    for (int64_t c = 0; c < m; ++c) /* the first component of each value wins */
      if (c == 0 || comps[c - 1].fvalue != comps[c].fvalue || comps[c - 1].ivalue != comps[c].ivalue)
        keep[comps[c].root] = 1;
    for (int64_t v = 0; v < n; ++v)
      if (r[v] != 0xFFFFFFFFu && !keep[r[v]]) memcpy(d + v * es, fill, es);
  }
  free(size);
  free(keep);
  free(comps);
  return 0;
}

// fused_intensity.cu — K3 (separable Gaussian blur) and the fused intensity chain
//   v = src * exp(bias) -> blur_K -> blur_J -> blur_I -> + noise -> gamma
// in two HBM passes instead of the reference's ~20 (TorchIO 2.0.0a2
// transforms/intensity/{bias_field,blur,noise,gamma}.py; blur alone is
// 3 x (F.pad replicate + F.conv3d), blur.py:171-252).
//
//   pass 1  march_kernel: thread <-> (j, 4 consecutive k), marching along I
//           with a shared-memory ring of the last 2r+1 planes; bias multiply at
//           load (no halo, J/K lerp levels cached in registers), then I-conv;
//           8 B/voxel.  Without J/K blur it also applies noise and gamma and is
//           the only pass.
//   pass 2  jk_kernel:   per (b,c) plane tile (32 x 64 outputs + halo) staged in
//           shared memory; K-conv then J-conv; noise (+Rician) and gamma as the
//           store epilogue; 8 B/voxel of HBM traffic (+4 when normals are
//           supplied), halo re-reads are L2 hits.
// Replicate padding == clamped addressing, so no padded copies exist.
// Separable passes commute up to fp32 summation order (the reference runs
// I, J, K; this runs I, K, J): differences are ~1e-7 relative.
#include "common.cuh"
#include "mt19937_layout.h"
#include "mt19937_normal.cuh"
#include "tma.cuh"

namespace tio {

__device__ __forceinline__ float rician(float x, float n1, float n2) {
  float s = __fadd_rn(x, n1);
  return sqrtf(__fadd_rn(__fmul_rn(s, s), __fmul_rn(n2, n2)));
}


// Philox4x32 (Salmon et al. 2011), 7 rounds (the paper's Crush-resistant minimum;
// the name is kept for the call sites), counter = element-group index.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 7; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& n0, float& n1) {
  float u1 = ((float)(a >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
  float u2 = ((float)(b >> 8)) * (1.0f / 16777216.0f);
  float rad;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(rad) : "f"(-2.0f * __logf(u1)));
  float s, c;
  __sincosf(6.283185307179586f * u2, &s, &c);
  n0 = rad * c;
  n1 = rad * s;
}


// |x|^g = 2^(g*log2|x|) on the SFU (lg2/ex2.approx): ~3e-7 relative for the value ranges
// of normalised images, far inside the 1e-4 parity tolerance.  Neither flushes subnormals:
// (1e-40)^0.8 = 1e-32 as torch's pow gives, and a subnormal result is kept.
__device__ __forceinline__ float abs_pow(float ax, float g) {
  float l, p;
  asm("lg2.approx.f32 %0, %1;" : "=f"(l) : "f"(ax));
  asm("ex2.approx.f32 %0, %1;" : "=f"(p) : "f"(__fmul_rn(g, l)));
  return p;
}

__device__ __forceinline__ float signed_pow(float x, float gam) {
  // sign(x) * |x|^gamma (gamma.py:88-90); gamma == 1 -> x exactly (gated rows).
  // sign(+-0) = 0, so +-0 -> +0 as torch gives.
  if (gam == 1.0f) return x;
  float ax = fabsf(x);
  float p = abs_pow(ax, gam);
  p = ax == 0.0f ? 0.0f : p;
  return x < 0.0f ? -p : p;
}

constexpr int A_TJ = 32;
constexpr int A_TK = 64;
constexpr int A_PLANES = 16;  // planes per CTA (amortises table setup)

struct BiasArgs {
  const float* coarse;  // [B][C][si][sj][sk] or null
  const uint8_t* identity;
  int si, sj, sk;
  float sc_i, sc_j, sc_k;
  int divide;
};

struct BlurArgs {
  const float* taps;       // [3][B][2R+1] or null
  const int32_t* radius;   // [3][B]
  int R;
};

struct NoiseArgs {
  const float* mean;
  const float* std;
  const uint8_t* keep;
  const float* z;
  const float* z2;
  uint64_t philox_seed;
  int mode;  // 0 none, 1 supplied normals, 2 philox
  int rician;
};

// -------------------------------------------------------------------------
// pass 2
// -------------------------------------------------------------------------
template <int RMAX, bool HAS_EPI>
__global__ void __launch_bounds__(256)
jk_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int I, int J,
          int K, BlurArgs bl, NoiseArgs nz, const float* __restrict__ gamma) {
  constexpr int ROWS = A_TJ + 2 * RMAX;
  constexpr int COLS = A_TK + 2 * RMAX;
  constexpr int PITCH = (COLS + 3) / 4 * 4 + 4;  // 16-byte aligned rows
  extern __shared__ __align__(16) float smem[];
  float* A = smem;                       // [ROWS][PITCH]   input tile (+halo)
  float* Bm = A + ROWS * PITCH;          // [ROWS][A_TK]    after the K pass
  float* tapk = Bm + ROWS * A_TK;        // [2*RMAX+1]
  float* tapj = tapk + (2 * RMAX + 1);   // [2*RMAX+1]

  const int tiles_i = (I + A_PLANES - 1) / A_PLANES;
  const int bc = blockIdx.z / tiles_i;
  const int i_begin = (blockIdx.z % tiles_i) * A_PLANES;
  const int i_end = min(i_begin + A_PLANES, I);
  const int b = bc / C;
  const int j0 = blockIdx.y * A_TJ, k0 = blockIdx.x * A_TK;
  const int tid = threadIdx.x;
  const int64_t n = (int64_t)I * J * K;
  const float* x = src + (int64_t)bc * n;
  float* y = dst + (int64_t)bc * n;

  const int R = bl.taps ? bl.R : 0;
  const int rj = bl.taps ? bl.radius[1 * B + b] : 0;
  const int rk = bl.taps ? bl.radius[2 * B + b] : 0;
  const bool noise_on = HAS_EPI && nz.mode != 0 && (!nz.keep || nz.keep[b]);
  const float mu = (HAS_EPI && nz.mode) ? nz.mean[b] : 0.0f, sd = (HAS_EPI && nz.mode) ? nz.std[b] : 0.0f;
  const float gam = (HAS_EPI && gamma) ? gamma[b] : 1.0f;

  // taps shifted so that window offset s = 0..2r maps to tap (s - r); zero beyond
  if (tid < 2 * (2 * RMAX + 1)) {
    const bool is_k = tid < (2 * RMAX + 1);
    const int sft = is_k ? tid : tid - (2 * RMAX + 1);
    const int rr = is_k ? rk : rj;
    float v = 0.0f;
    if (bl.taps && rr > 0 && sft <= 2 * rr)
      v = bl.taps[((int64_t)(is_k ? 2 : 1) * B + b) * (2 * R + 1) + R - rr + sft];
    (is_k ? tapk : tapj)[sft] = v;
  }
  __syncthreads();

  float tk[2 * RMAX + 1], tj[2 * RMAX + 1];
#pragma unroll
  for (int t = 0; t < 2 * RMAX + 1; ++t) { tk[t] = tapk[t]; tj[t] = tapj[t]; }

  const int rows = A_TJ + 2 * rj, cols = A_TK + 2 * rk;
  const int lx = tid & 31, ly = tid >> 5;  // 32 x 8 loader layout

  for (int i = i_begin; i < i_end; ++i) {
    const float* xp = x + (int64_t)i * J * K;
    // ---- load (clamped = replicate padding) ----
    for (int r = ly; r < rows; r += 8) {
      const int jj = min(max(j0 - rj + r, 0), J - 1);
      const float* xr = xp + (int64_t)jj * K;
      for (int c = lx; c < cols; c += 32) {
        const int kk = min(max(k0 - rk + c, 0), K - 1);
        A[r * PITCH + c] = __ldg(xr + kk);
      }
    }
    __syncthreads();
    // ---- K pass: 16 threads x 4 outputs per row, 16 rows per sweep ----
    {
      const int k4 = (tid & 15) * 4;
      for (int r = tid >> 4; r < rows; r += 16) {
        const float* row = A + r * PITCH + k4;  // window start = output k - rk + rk
        float acc[4];
        if (rk == 0) {
#pragma unroll
          for (int o = 0; o < 4; ++o) acc[o] = row[o];
        } else {
          // window of 4 + 2*rk inputs; taps centred at index RMAX
          float win[4 + 2 * RMAX];
#pragma unroll
          for (int m = 0; m < (4 + 2 * RMAX) / 4; ++m) {
            if (4 * m < 4 + 2 * rk) {
              float4 q = *(const float4*)(row + 4 * m);
              win[4 * m] = q.x; win[4 * m + 1] = q.y; win[4 * m + 2] = q.z; win[4 * m + 3] = q.w;
            } else {
              win[4 * m] = win[4 * m + 1] = win[4 * m + 2] = win[4 * m + 3] = 0.0f;
            }
          }
#pragma unroll
          for (int o = 0; o < 4; ++o) acc[o] = 0.0f;
          // output o at window index o + rk (centre); tap t (-rk..rk) reads o + rk + t.
          // static form: iterate s = 0..2*RMAX over window offsets, tap index = s - rk + RMAX
#pragma unroll
          for (int s = 0; s < 2 * RMAX + 1; ++s) {
            if (s <= 2 * rk) {  // CTA-uniform: never touches window slots that were not loaded
#pragma unroll
              for (int o = 0; o < 4; ++o) acc[o] = __fmaf_rn(tk[s], win[o + s], acc[o]);
            }
          }
        }
        *(float4*)(Bm + r * A_TK + k4) = make_float4(acc[0], acc[1], acc[2], acc[3]);
      }
    }
    __syncthreads();
    // ---- J pass: thread = (k lane, 8 consecutive j) ----
    {
      const int kx = tid & 63, jy = (tid >> 6) * 8;
      const int k = k0 + kx;
      float acc[8];
      if (rj == 0) {
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = Bm[(jy + o) * A_TK + kx];
      } else {
        float win[8 + 2 * RMAX];
#pragma unroll
        for (int w = 0; w < 8 + 2 * RMAX; ++w)
          win[w] = (w < 8 + 2 * rj) ? Bm[(jy + w) * A_TK + kx] : 0.0f;
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = 0.0f;
#pragma unroll
        for (int s = 0; s < 2 * RMAX + 1; ++s) {
          if (s <= 2 * rj) {
#pragma unroll
            for (int o = 0; o < 8; ++o) acc[o] = __fmaf_rn(tj[s], win[o + s], acc[o]);
          }
        }
      }
      if (k < K) {
        const int64_t plane_off = (int64_t)i * J * K + k;
        if (HAS_EPI && noise_on) {
          float z1[8], z2[8];
          if (nz.mode == 1) {
#pragma unroll
            for (int o = 0; o < 8; ++o)
              if (j0 + jy + o < J) {
                const int64_t flat = (int64_t)bc * n + plane_off + (int64_t)(j0 + jy + o) * K;
                z1[o] = __ldcs(nz.z + flat);
                if (nz.rician) z2[o] = __ldcs(nz.z2 + flat);
              }
          } else {
            const uint2 key = make_uint2((uint32_t)nz.philox_seed, (uint32_t)(nz.philox_seed >> 32));
            const uint64_t gidx = (uint64_t)((int64_t)bc * n + plane_off + (int64_t)(j0 + jy) * K);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              uint4 rr = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)h, 0x6a6bu), key);
              box_muller(rr.x, rr.y, z1[4 * h], z1[4 * h + 1]);
              box_muller(rr.z, rr.w, z1[4 * h + 2], z1[4 * h + 3]);
              if (nz.rician) {
                uint4 r2 = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), (uint32_t)(2 + h), 0x6a6bu), key);
                box_muller(r2.x, r2.y, z2[4 * h], z2[4 * h + 1]);
                box_muller(r2.z, r2.w, z2[4 * h + 2], z2[4 * h + 3]);
              }
            }
          }
#pragma unroll
          for (int o = 0; o < 8; ++o) {
            const float n1 = __fadd_rn(mu, __fmul_rn(sd, z1[o]));
            if (nz.rician) acc[o] = rician(acc[o], n1, __fadd_rn(mu, __fmul_rn(sd, z2[o])));
            else acc[o] = __fadd_rn(acc[o], n1);
          }
        }
        if (HAS_EPI && gamma) {
#pragma unroll
          for (int o = 0; o < 8; ++o) acc[o] = signed_pow(acc[o], gam);
        }
        float* yp = y + plane_off;
#pragma unroll
        for (int o = 0; o < 8; ++o)
          if (j0 + jy + o < J) yp[(int64_t)(j0 + jy + o) * K] = acc[o];
      }
    }
    __syncthreads();
  }
}

// -------------------------------------------------------------------------
// pass 2, fast variant for table radius R <= 6 (sigma <= 2 voxels).
//   staging   one TMA box per plane: [j0-6, j0+38) x [k0-8, k0+72) (80 floats = 320 B
//             per row, 16-byte aligned origin), zero-filled outside the volume, two
//             buffers so plane i+1 is in flight while plane i is convolved; a single
//             thread issues it, so staging costs no issue slots.
//   padding   replicate padding is applied where the data is consumed: the K pass
//             reads the clamped source row (rows beyond the J border are the edge
//             row, and conv_K commutes with that); on K-border tiles each half-warp
//             first copies the edge column into its row's zero-filled halo.
//   K pass    (row, 4 consecutive k): five aligned LDS.128 -> 13 taps x 4 outputs.
//   J pass    (k, 8 consecutive j) from the K-pass plane (double buffered: one
//             __syncthreads per plane), normals prefetched before the FMAs,
//             noise (+Rician) and gamma at the store.
// Taps are zero-padded to 13 and held in registers; no per-tap branches.
// -------------------------------------------------------------------------
constexpr int F_R = 6;                    // taps = 13
constexpr int F_HK = 8;                   // K halo, rounded up to keep 16-byte alignment
constexpr int F_ROWS = A_TJ + 2 * F_R;    // 44
constexpr int F_COLS = A_TK + 2 * F_HK;   // 80 (dense: the TMA box pitch)
constexpr int F_ABUF = F_ROWS * F_COLS;   // floats per staged plane
constexpr int F_BBUF = F_ROWS * A_TK;     // floats per K-pass plane
constexpr size_t F_SMEM = (size_t)(2 * F_ABUF + 2 * F_BBUF + 32) * sizeof(float) + 2 * sizeof(uint64_t);

// K conv of 4 consecutive outputs (columns 8+k4 .. 8+k4+3 of a staged row), radius RK:
// aligned 16-byte loads cover columns k4+4..k4+15 (RK <= 4) or k4..k4+19.
template <int RK>
__device__ __forceinline__ float4 kconv4(const float* __restrict__ row, const int k4, const float* tk) {
  if (RK == 0) return *(const float4*)(row + F_HK + k4);
  constexpr int M0 = RK <= 4 ? 1 : 0, M1 = RK <= 4 ? 4 : 5;
  float win[20];
#pragma unroll
  for (int m = M0; m < M1; ++m) {
    const float4 q = *(const float4*)(row + k4 + 4 * m);
    win[4 * m] = q.x; win[4 * m + 1] = q.y; win[4 * m + 2] = q.z; win[4 * m + 3] = q.w;
  }
  float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
  for (int t = -RK; t <= RK; ++t)
#pragma unroll
    for (int o = 0; o < 4; ++o) acc[o] = __fmaf_rn(tk[F_R + t], win[F_HK + o + t], acc[o]);
  return make_float4(acc[0], acc[1], acc[2], acc[3]);
}

// J conv of 8 consecutive rows (F_R+jy .. F_R+jy+7 of the K-pass plane) at column kx
template <int RJ>
__device__ __forceinline__ void jconv8(const float* __restrict__ Bw, const int jy, const int kx,
                                       const float* tj, float* acc) {
  float win[8 + 2 * RJ];
#pragma unroll
  for (int w = 0; w < 8 + 2 * RJ; ++w) win[w] = Bw[(F_R - RJ + jy + w) * A_TK + kx];
  if (RJ == 0) {
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = win[o];
    return;
  }
#pragma unroll
  for (int o = 0; o < 8; ++o) acc[o] = 0.0f;
#pragma unroll
  for (int t = -RJ; t <= RJ; ++t)
#pragma unroll
    for (int o = 0; o < 8; ++o) acc[o] = __fmaf_rn(tj[F_R + t], win[o + t + RJ], acc[o]);
}

// signed_pow for g > 0, g != 1: lg2(0) = -inf -> ex2 = +0, so zero needs no select, and
// -0 -> +0 because -0 < 0 is false.  Bit-identical to signed_pow for those g.
__device__ __forceinline__ float signed_pow_pos(float x, float g) {
  const float p = abs_pow(fabsf(x), g);
  return x < 0.0f ? -p : p;
}

template <bool HAS_EPI>
__global__ void __launch_bounds__(256, 3)
jk6_kernel(const __grid_constant__ CUtensorMap tmap, float* __restrict__ dst, int B, int C, int I,
           int J, int K, BlurArgs bl, NoiseArgs nz, const float* __restrict__ gamma) {
  extern __shared__ __align__(128) float smem[];
  float* Abuf = smem;                    // [2][F_ROWS][F_COLS]  staged planes
  float* Bbuf = smem + 2 * F_ABUF;       // [2][F_ROWS][A_TK]    after the K pass
  float* taps_s = Bbuf + 2 * F_BBUF;     // [2][13] (+ padding)
  uint64_t* bars = reinterpret_cast<uint64_t*>(taps_s + 32);

  const int tiles_i = (I + A_PLANES - 1) / A_PLANES;
  const int bc = blockIdx.z / tiles_i;
  const int i_begin = (blockIdx.z % tiles_i) * A_PLANES;
  const int i_end = min(i_begin + A_PLANES, I);
  const int b = bc / C;
  const int j0 = blockIdx.y * A_TJ, k0 = blockIdx.x * A_TK;
  const int tid = threadIdx.x;
  const int64_t n = (int64_t)I * J * K;

  auto issue = [&](int i, int s) {  // one thread
    const uint32_t bar = smem_u32(bars + s);
    mbar_expect_tx(bar, (uint32_t)(F_ABUF * sizeof(float)));
    tma_load_3d(smem_u32(Abuf + s * F_ABUF), &tmap, k0 - F_HK, j0 - F_R, bc * I + i, bar);
  };
  if (tid == 0) {
    mbar_init(smem_u32(bars + 0), 1);
    mbar_init(smem_u32(bars + 1), 1);
    mbar_fence_init();
    issue(i_begin, 0);
  }

  const int R = bl.R;
  const int rj = bl.radius[1 * B + b], rk = bl.radius[2 * B + b];
  const bool noise_on = HAS_EPI && nz.mode != 0 && (!nz.keep || nz.keep[b]);
  const float mu = (HAS_EPI && nz.mode) ? nz.mean[b] : 0.0f, sd = (HAS_EPI && nz.mode) ? nz.std[b] : 0.0f;
  const float gam = (HAS_EPI && gamma) ? gamma[b] : 1.0f;
  // gamma == 1 (gated rows) passes values through exactly; gamma <= 0 or NaN never comes
  // from exp(log_gamma) but keeps the general helper
  const int gamma_mode = !(HAS_EPI && gamma) || gam == 1.0f ? 0 : (gam > 0.0f ? 1 : 2);

  if (tid < 2 * (2 * F_R + 1)) {  // 13 taps per axis, centred at index 6, zero beyond the radius
    const int axis = tid < (2 * F_R + 1) ? 2 : 1;
    const int s = tid < (2 * F_R + 1) ? tid : tid - (2 * F_R + 1);
    const int off = s - F_R, rr = axis == 2 ? rk : rj;
    float v = 0.0f;
    if (rr > 0 && off >= -rr && off <= rr) v = bl.taps[((int64_t)axis * B + b) * (2 * R + 1) + R + off];
    taps_s[(axis == 2 ? 0 : 13) + s] = v;
  }
  __syncthreads();
  float tk[2 * F_R + 1], tj[2 * F_R + 1];
#pragma unroll
  for (int t = 0; t < 2 * F_R + 1; ++t) { tk[t] = taps_s[t]; tj[t] = taps_s[13 + t]; }

  const int row_lo = F_R - rj, row_hi = F_R + A_TJ + rj;        // rows the J pass reads
  const int rsrc_lo = max(0, F_R - j0), rsrc_hi = min(F_ROWS - 1, J - 1 - j0 + F_R);  // rows inside the volume
  const int clo = max(0, F_HK - k0), chi = min(F_COLS - 1, K - 1 - k0 + F_HK);        // columns inside the volume
  const bool kfix = (clo > F_HK - rk) || (chi < F_HK + A_TK + rk - 1);                // CTA-uniform

  const int k4 = (tid & 15) * 4;
  const int kx = tid & 63, jy = (tid >> 6) * 8;
  const int k = k0 + kx;
  const int valid = (k < K) ? min(8, J - (j0 + jy)) : 0;
  const int plane_off = (j0 + jy) * K + k;  // within one plane (J*K < 2^31)

  // K pass of one staged plane -> its slot of the double-buffered K-pass plane
  auto kpass = [&](int i) {
    const int it = i - i_begin, s = it & 1;
    mbar_wait(smem_u32(bars + s), (uint32_t)((it >> 1) & 1));
    float* A = Abuf + s * F_ABUF;
    float* Bw = Bbuf + s * F_BBUF;
#pragma unroll 1
    for (int r = row_lo + (tid >> 4); r < row_hi; r += 16) {
      float* row = A + min(max(r, rsrc_lo), rsrc_hi) * F_COLS;
      if (kfix) {
        // replicate the edge column into the zero-filled halo of this half-warp's row.
        // Other warps may patch the same (clamped) row with the same values; every
        // reader has written them itself first, so any interleaving reads the same data.
        const int c_lo = (F_HK - F_R) + (tid & 15);
        if (c_lo < clo) row[c_lo] = row[clo];
#pragma unroll 1
        for (int c = chi + 1 + (tid & 15); c < F_HK + A_TK + F_R; c += 16) row[c] = row[chi];
        __syncwarp();
      }
      float4 o4;
      switch (rk) {
        case 0: o4 = kconv4<0>(row, k4, tk); break;
        case 1: o4 = kconv4<1>(row, k4, tk); break;
        case 2: o4 = kconv4<2>(row, k4, tk); break;
        case 3: o4 = kconv4<3>(row, k4, tk); break;
        case 4: o4 = kconv4<4>(row, k4, tk); break;
        case 5: o4 = kconv4<5>(row, k4, tk); break;
        default: o4 = kconv4<6>(row, k4, tk); break;
      }
      *(float4*)(Bw + r * A_TK + k4) = o4;
    }
  };

  // Software pipeline, one barrier per plane: between two barriers every thread runs the
  // K pass of plane i+1 and then the J pass + store of plane i, so the ragged K-pass rounds
  // (44 rows over 16 row slots) are amortised over a longer phase and LDS-heavy K work of
  // some warps overlaps FMA-heavy J work of others.
  if (tid == 0 && i_begin + 1 < i_end) issue(i_begin + 1, 1);
  kpass(i_begin);
  __syncthreads();
  for (int i = i_begin; i < i_end; ++i) {
    const int it = i - i_begin, s = it & 1;
    // plane i+2 replaces plane i in its staging buffer: the K pass of plane i ended before
    // the barrier that closed the previous phase
    if (tid == 0 && i + 2 < i_end) issue(i + 2, s);
    float* Bw = Bbuf + s * F_BBUF;
    // normals for this thread's 8 outputs: in flight across the K pass of the next plane
    float z1[8], z2[8];
    const int64_t flat0 = (int64_t)bc * n + (int64_t)i * J * K + plane_off;
    if (HAS_EPI && noise_on && nz.mode == 1) {
      const float* zp = nz.z + flat0;
      if (valid == 8) {
#pragma unroll
        for (int o = 0; o < 8; ++o, zp += K) z1[o] = __ldcs(zp);
      } else {
#pragma unroll
        for (int o = 0; o < 8; ++o, zp += K)
          if (o < valid) z1[o] = __ldcs(zp);
      }
      if (nz.rician) {
        const float* zq = nz.z2 + flat0;
#pragma unroll
        for (int o = 0; o < 8; ++o, zq += K)
          if (o < valid) z2[o] = __ldcs(zq);
      }
    }
    if (i + 1 < i_end) kpass(i + 1);
    // ---- J pass: thread = (k lane, 8 consecutive j), then epilogue + store ----
    float acc[8];
    switch (rj) {
      case 0: jconv8<0>(Bw, jy, kx, tj, acc); break;
      case 1: jconv8<1>(Bw, jy, kx, tj, acc); break;
      case 2: jconv8<2>(Bw, jy, kx, tj, acc); break;
      case 3: jconv8<3>(Bw, jy, kx, tj, acc); break;
      case 4: jconv8<4>(Bw, jy, kx, tj, acc); break;
      case 5: jconv8<5>(Bw, jy, kx, tj, acc); break;
      default: jconv8<6>(Bw, jy, kx, tj, acc); break;
    }
    if (valid > 0) {
      if (HAS_EPI && noise_on) {
        if (nz.mode == 2) {
          const uint2 key = make_uint2((uint32_t)nz.philox_seed, (uint32_t)(nz.philox_seed >> 32));
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint64_t gidx = (uint64_t)(flat0 + (int64_t)(4 * h) * K);
            uint4 rr = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 0u, 0x6a6bu), key);
            box_muller(rr.x, rr.y, z1[4 * h], z1[4 * h + 1]);
            box_muller(rr.z, rr.w, z1[4 * h + 2], z1[4 * h + 3]);
            if (nz.rician) {
              uint4 r2 = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 1u, 0x6a6bu), key);
              box_muller(r2.x, r2.y, z2[4 * h], z2[4 * h + 1]);
              box_muller(r2.z, r2.w, z2[4 * h + 2], z2[4 * h + 3]);
            }
          }
        }
        if (nz.rician) {
#pragma unroll
          for (int o = 0; o < 8; ++o)
            acc[o] = rician(acc[o], __fadd_rn(mu, __fmul_rn(sd, z1[o])), __fadd_rn(mu, __fmul_rn(sd, z2[o])));
        } else {
#pragma unroll
          for (int o = 0; o < 8; ++o) acc[o] = __fadd_rn(acc[o], __fadd_rn(mu, __fmul_rn(sd, z1[o])));
        }
      }
      if (gamma_mode == 1) {
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = signed_pow_pos(acc[o], gam);
      } else if (gamma_mode == 2) {
#pragma unroll
        for (int o = 0; o < 8; ++o) acc[o] = signed_pow(acc[o], gam);
      }
      float* yp = dst + flat0;
      if (valid == 8) {
#pragma unroll
        for (int o = 0; o < 8; ++o, yp += K) *yp = acc[o];
      } else {
#pragma unroll
        for (int o = 0; o < 8; ++o, yp += K)
          if (o < valid) *yp = acc[o];
      }
    }
    __syncthreads();  // K-pass plane i and staging buffer of plane i+1 are free again
  }
}

// -------------------------------------------------------------------------
// pass 1 (and the whole chain when no J/K blur is active)
// -------------------------------------------------------------------------
template <int V, bool HAS_BIAS>
__global__ void __launch_bounds__(256)
march_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int I, int J,
             int K, BlurArgs bl, BiasArgs bi, NoiseArgs nz, const float* __restrict__ gamma) {
  extern __shared__ __align__(16) float smem[];
  const int bc = blockIdx.z;
  const int b = bc / C;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  const int j = blockIdx.y * blockDim.y + threadIdx.y;
  const int64_t n = (int64_t)I * J * K;
  const float* x = src + (int64_t)bc * n;
  float* y = dst + (int64_t)bc * n;

  const int r = bl.taps ? bl.radius[0 * B + b] : 0;
  const int R = bl.taps ? bl.R : 0;
  const int W = 2 * r + 1;
  float* tapi = smem;                                   // [2R+1]
  float* g = smem + ((2 * R + 1 + 3) / 4) * 4;          // coarse bias grid
  const int ns = HAS_BIAS ? bi.si * bi.sj * bi.sk : 0;
  float* ring = g + ((ns + 3) / 4) * 4;                 // [W][256][V]
  const bool bias_on = HAS_BIAS && !(bi.identity && bi.identity[b]);
  if (r > 0)
    for (int t = tid; t < 2 * R + 1; t += 256) tapi[t] = bl.taps[((int64_t)0 * B + b) * (2 * R + 1) + t];
  if (bias_on) {
    const float* gs = bi.coarse + (int64_t)bc * ns;
    for (int t = tid; t < ns; t += 256) g[t] = gs[t];
  }
  __syncthreads();
  if (k >= K || j >= J) return;

  const bool noise_on = nz.mode != 0 && (!nz.keep || nz.keep[b]);
  const float mu = nz.mode ? nz.mean[b] : 0.0f, sd = nz.mode ? nz.std[b] : 0.0f;
  const float gam = gamma ? gamma[b] : 1.0f;

  LerpAxis lj, lk[V];
  int cur0 = -1, cur1 = -1;
  float r_lo[V], r_hi[V];
  if (bias_on) {
    lj = lerp_axis(bi.sc_j, bi.sj, j);
#pragma unroll
    for (int v = 0; v < V; ++v) lk[v] = lerp_axis(bi.sc_k, bi.sk, k + v);
  }

  auto load_plane = [&](int i, float* out) {
    const int64_t o = ((int64_t)i * J + j) * K + k;
    if (V == 4) {
      float4 t = *(const float4*)(x + o);
      out[0] = t.x; out[1] = t.y; out[2] = t.z; out[3] = t.w;
    } else {
      out[0] = x[o];
    }
    if (bias_on) {
      const LerpAxis li = lerp_axis(bi.sc_i, bi.si, i);
      if (li.i0 != cur0 || li.i1 != cur1) {
        const float* p0 = g + (li.i0 * bi.sj) * bi.sk;
        const float* p1 = g + (li.i1 * bi.sj) * bi.sk;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          float a0 = lerp2(lk[v].l0, p0[lj.i0 * bi.sk + lk[v].i0], lk[v].l1, p0[lj.i0 * bi.sk + lk[v].i1]);
          float a1 = lerp2(lk[v].l0, p0[lj.i1 * bi.sk + lk[v].i0], lk[v].l1, p0[lj.i1 * bi.sk + lk[v].i1]);
          r_lo[v] = lerp2(lj.l0, a0, lj.l1, a1);
          float b0 = lerp2(lk[v].l0, p1[lj.i0 * bi.sk + lk[v].i0], lk[v].l1, p1[lj.i0 * bi.sk + lk[v].i1]);
          float b1 = lerp2(lk[v].l0, p1[lj.i1 * bi.sk + lk[v].i0], lk[v].l1, p1[lj.i1 * bi.sk + lk[v].i1]);
          r_hi[v] = lerp2(lj.l0, b0, lj.l1, b1);
        }
        cur0 = li.i0; cur1 = li.i1;
      }
#pragma unroll
      for (int v = 0; v < V; ++v) {
        float f = expf(lerp2(li.l0, r_lo[v], li.l1, r_hi[v]));
        out[v] = bi.divide ? __fdiv_rn(out[v], f) : __fmul_rn(out[v], f);
      }
    }
  };

  auto finish = [&](int i, float* v) {
    const int64_t o = ((int64_t)i * J + j) * K + k;
    if (noise_on) {
      const int64_t flat = (int64_t)bc * n + o;
      float z1[V], z2[V];
      if (nz.mode == 1) {
        if (V == 4) {
          float4 t = __ldcs((const float4*)(nz.z + flat));
          z1[0] = t.x; z1[1] = t.y; z1[2] = t.z; z1[3] = t.w;
          if (nz.rician) {
            float4 u = __ldcs((const float4*)(nz.z2 + flat));
            z2[0] = u.x; z2[1] = u.y; z2[2] = u.z; z2[3] = u.w;
          }
        } else {
          z1[0] = nz.z[flat];
          if (nz.rician) z2[0] = nz.z2[flat];
        }
      } else {
        const uint2 key = make_uint2((uint32_t)nz.philox_seed, (uint32_t)(nz.philox_seed >> 32));
        const uint64_t gidx = (uint64_t)(flat / V);
        uint4 rr = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 0u, 0x5eedu), key);
        float nn[4];
        box_muller(rr.x, rr.y, nn[0], nn[1]);
        box_muller(rr.z, rr.w, nn[2], nn[3]);
#pragma unroll
        for (int q = 0; q < V; ++q) z1[q] = nn[q];
        if (nz.rician) {
          uint4 r2 = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 1u, 0x5eedu), key);
          box_muller(r2.x, r2.y, nn[0], nn[1]);
          box_muller(r2.z, r2.w, nn[2], nn[3]);
#pragma unroll
          for (int q = 0; q < V; ++q) z2[q] = nn[q];
        }
      }
#pragma unroll
      for (int q = 0; q < V; ++q) {
        float n1 = __fadd_rn(mu, __fmul_rn(sd, z1[q]));
        if (nz.rician) v[q] = rician(v[q], n1, __fadd_rn(mu, __fmul_rn(sd, z2[q])));
        else v[q] = __fadd_rn(v[q], n1);
      }
    }
    if (gamma) {
#pragma unroll
      for (int q = 0; q < V; ++q) v[q] = signed_pow(v[q], gam);
    }
    if (V == 4) *(float4*)(y + o) = make_float4(v[0], v[1], v[2], v[3]);
    else y[o] = v[0];
  };

  if (r == 0) {  // no I-axis blur for this element: pure streaming
    for (int i = 0; i < I; ++i) {
      float v[V];
      load_plane(i, v);
      finish(i, v);
    }
    return;
  }

  // ring[slot][tid][V]; slot = position mod W (position may be negative -> add W)
  float* mine = ring + tid * V;
  const int slot_stride = 256 * V;
  auto put = [&](int pos, const float* v) {
    int s = pos % W; if (s < 0) s += W;
    if (V == 4) *(float4*)(mine + s * slot_stride) = make_float4(v[0], v[1], v[2], v[3]);
    else mine[s * slot_stride] = v[0];
  };
  float first[V];
  load_plane(0, first);
  for (int p = -r; p <= 0; ++p) put(p, first);   // replicate padding below 0
  float last[V];
#pragma unroll
  for (int q = 0; q < V; ++q) last[q] = first[q];
  for (int p = 1; p < I + r; ++p) {
    if (p < I) load_plane(p, last);               // beyond I-1: keep the last plane
    put(p, last);
    const int o = p - r;
    if (o < 0) continue;
    float acc[V];
#pragma unroll
    for (int q = 0; q < V; ++q) acc[q] = 0.0f;
    int s = (o - r) % W; if (s < 0) s += W;
    for (int t = 0; t < W; ++t) {
      const float tp = tapi[R - r + t];
      if (V == 4) {
        float4 w4 = *(const float4*)(mine + s * slot_stride);
        acc[0] = __fmaf_rn(tp, w4.x, acc[0]); acc[1] = __fmaf_rn(tp, w4.y, acc[1]);
        acc[2] = __fmaf_rn(tp, w4.z, acc[2]); acc[3] = __fmaf_rn(tp, w4.w, acc[3]);
      } else {
        acc[0] = __fmaf_rn(tp, mine[s * slot_stride], acc[0]);
      }
      if (++s == W) s = 0;
    }
    finish(o, acc);
  }
}

// -------------------------------------------------------------------------
// pass 1, fast variant for table radius R <= 6 and 16-byte aligned rows: the ring of
// the last 13 planes lives in registers.  The plane loop is unrolled by 13 so every
// ring slot is a fixed register: no shared-memory traffic, no modular indexing.  Only the
// element's own 2r+1 taps are accumulated (a CTA-uniform predicate per tap, in the order of
// every other path): a zero tap would turn a NaN or Inf r+1..6 planes away into NaN.
//   EPI = this is the only pass (no J/K blur): noise and gamma at the store.
// -------------------------------------------------------------------------
constexpr int M6_PF = 8;  // cp.async FIFO depth of march6_kernel (power of two)

// One tile of pass 1: 256 threads, thread `tid` <-> (row j, columns k..k+3) of volume bc, all I
// planes.  BAR = 0: the 256 threads are a whole CTA (__syncthreads); BAR > 0: they are part of
// a larger CTA and meet at named barrier BAR.  `smem`: 16 floats of taps, the coarse bias grid,
// then the FIFO.
template <bool HAS_BIAS, bool EPI, int BAR>
__device__ __forceinline__ void march6_tile(float* smem, const int tid, const int k, const int j, const int bc,
                                            const float* __restrict__ src, float* __restrict__ dst, int B,
                                            int C, int I, int J, int K, const BlurArgs& bl, const BiasArgs& bi,
                                            const NoiseArgs& nz, const float* __restrict__ gamma) {
  constexpr int W = 2 * F_R + 1;
  const int b = bc / C;
  const int64_t n = (int64_t)I * J * K;
  const float* x = src + (int64_t)bc * n;
  float* y = dst + (int64_t)bc * n;

  const int r = bl.taps ? bl.radius[0 * B + b] : 0;
  float* tapi = smem;      // [13] zero-padded, centred at 6
  float* g = smem + 16;    // coarse bias grid
  const int ns = HAS_BIAS ? bi.si * bi.sj * bi.sk : 0;
  const bool bias_on = HAS_BIAS && !(bi.identity && bi.identity[b]);
  if (tid < W) {
    const int off = tid - F_R;
    tapi[tid] = (r > 0 && off >= -r && off <= r) ? bl.taps[((int64_t)0 * B + b) * (2 * bl.R + 1) + bl.R + off] : 0.0f;
  }
  if (bias_on) {
    const float* gs = bi.coarse + (int64_t)bc * ns;
    for (int t = tid; t < ns; t += 256) g[t] = gs[t];
  }
  if (BAR == 0) __syncthreads();
  else asm volatile("bar.sync %0, 256;" ::"n"(BAR) : "memory");
  if (k >= K || j >= J) return;

  const bool noise_on = EPI && nz.mode != 0 && (!nz.keep || nz.keep[b]);
  const float mu = (EPI && nz.mode) ? nz.mean[b] : 0.0f, sd = (EPI && nz.mode) ? nz.std[b] : 0.0f;
  const float gam = (EPI && gamma) ? gamma[b] : 1.0f;
  const int gamma_mode = !(EPI && gamma) || gam == 1.0f ? 0 : (gam > 0.0f ? 1 : 2);

  LerpAxis lj, lk[4];
  int o00[4], o01[4], o10[4], o11[4];
  int cur0 = -1, cur1 = -1;
  float r_lo[4], r_hi[4];
  if (bias_on) {
    lj = lerp_axis(bi.sc_j, bi.sj, j);
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      lk[v] = lerp_axis(bi.sc_k, bi.sk, k + v);
      o00[v] = lj.i0 * bi.sk + lk[v].i0; o01[v] = lj.i0 * bi.sk + lk[v].i1;
      o10[v] = lj.i1 * bi.sk + lk[v].i0; o11[v] = lj.i1 * bi.sk + lk[v].i1;
    }
  }
  const int col = j * K + k;  // within one plane
  const int plane = J * K;

  // Input planes arrive through a per-thread cp.async FIFO (M6_PF slots of 16 bytes in shared
  // memory, no registers): M6_PF-1 loads are in flight per thread while a plane is processed.
  // Without it the unrolled phases issue one dependent load at a time (8 KB in flight per SM,
  // far less than HBM bandwidth x DRAM latency needs to keep the memory system busy).  Planes are consumed strictly in
  // order; slot = plane mod M6_PF; the slot of plane i-1 is refilled while plane i is consumed.
  float4* fifo = reinterpret_cast<float4*>(g + ((ns + 3) / 4) * 4) + tid;  // [M6_PF][256]
  auto fifo_issue = [&](int pl) {
    if (pl < I) {
      const uint32_t sa = (uint32_t)__cvta_generic_to_shared(fifo + (pl & (M6_PF - 1)) * 256);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(x + (int64_t)pl * plane + col) : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
#pragma unroll
  for (int pl = 0; pl < M6_PF - 1; ++pl) fifo_issue(pl);

  auto load_plane = [&](int i, float* out) {
    fifo_issue(i + M6_PF - 1);  // into the slot of plane i-1 (consumed one call ago)
    asm volatile("cp.async.wait_group %0;" ::"n"(M6_PF - 1) : "memory");
    const float4 t = fifo[(i & (M6_PF - 1)) * 256];
    out[0] = t.x; out[1] = t.y; out[2] = t.z; out[3] = t.w;
    if (bias_on) {
      const LerpAxis li = lerp_axis(bi.sc_i, bi.si, i);
      if (li.i0 != cur0 || li.i1 != cur1) {
        const float* p0 = g + (li.i0 * bi.sj) * bi.sk;
        const float* p1 = g + (li.i1 * bi.sj) * bi.sk;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          const float a0 = lerp2(lk[v].l0, p0[o00[v]], lk[v].l1, p0[o01[v]]);
          const float a1 = lerp2(lk[v].l0, p0[o10[v]], lk[v].l1, p0[o11[v]]);
          r_lo[v] = lerp2(lj.l0, a0, lj.l1, a1);
          const float b0 = lerp2(lk[v].l0, p1[o00[v]], lk[v].l1, p1[o01[v]]);
          const float b1 = lerp2(lk[v].l0, p1[o10[v]], lk[v].l1, p1[o11[v]]);
          r_hi[v] = lerp2(lj.l0, b0, lj.l1, b1);
        }
        cur0 = li.i0; cur1 = li.i1;
      }
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const float f = expf(lerp2(li.l0, r_lo[v], li.l1, r_hi[v]));
        out[v] = bi.divide ? __fdiv_rn(out[v], f) : __fmul_rn(out[v], f);
      }
    }
  };

  auto finish = [&](int i, float* v) {
    const int64_t o = (int64_t)i * plane + col;
    if (EPI) {
      if (noise_on) {
        const int64_t flat = (int64_t)bc * n + o;
        float z1[4], z2[4];
        if (nz.mode == 1) {
          const float4 t = __ldcs((const float4*)(nz.z + flat));
          z1[0] = t.x; z1[1] = t.y; z1[2] = t.z; z1[3] = t.w;
          if (nz.rician) {
            const float4 u = __ldcs((const float4*)(nz.z2 + flat));
            z2[0] = u.x; z2[1] = u.y; z2[2] = u.z; z2[3] = u.w;
          }
        } else {
          const uint2 key = make_uint2((uint32_t)nz.philox_seed, (uint32_t)(nz.philox_seed >> 32));
          const uint64_t gidx = (uint64_t)(flat / 4);
          uint4 rr = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 0u, 0x5eedu), key);
          box_muller(rr.x, rr.y, z1[0], z1[1]);
          box_muller(rr.z, rr.w, z1[2], z1[3]);
          if (nz.rician) {
            uint4 r2 = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 1u, 0x5eedu), key);
            box_muller(r2.x, r2.y, z2[0], z2[1]);
            box_muller(r2.z, r2.w, z2[2], z2[3]);
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float n1 = __fadd_rn(mu, __fmul_rn(sd, z1[q]));
          if (nz.rician) v[q] = rician(v[q], n1, __fadd_rn(mu, __fmul_rn(sd, z2[q])));
          else v[q] = __fadd_rn(v[q], n1);
        }
      }
      if (gamma_mode == 1) {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = signed_pow_pos(v[q], gam);
      } else if (gamma_mode == 2) {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = signed_pow(v[q], gam);
      }
    }
    *(float4*)(y + o) = make_float4(v[0], v[1], v[2], v[3]);
  };

  if (r == 0) {  // no I-axis blur for this element: pure streaming
    for (int i = 0; i < I; ++i) {
      float v[4];
      load_plane(i, v);
      finish(i, v);
    }
    return;
  }

  float tp[W];
#pragma unroll
  for (int t = 0; t < W; ++t) tp[t] = tapi[t];
  float ring[W][4];
  {
    float first[4];
    load_plane(0, first);  // replicate padding below plane 0
#pragma unroll
    for (int sl = 0; sl < W; ++sl)
#pragma unroll
      for (int q = 0; q < 4; ++q) ring[sl][q] = first[q];
  }
  // position p enters slot p mod 13; output o = p - 6 reads positions p-12 .. p
  for (int base = 0; base < I + F_R; base += W) {
#pragma unroll
    for (int ph = 0; ph < W; ++ph) {
      const int p = base + ph;
      if (p >= I + F_R) break;
      if (p > 0 && p < I) load_plane(p, ring[ph]);
      else if (p >= I) {  // replicate padding above plane I-1: the previous slot holds it
#pragma unroll
        for (int q = 0; q < 4; ++q) ring[ph][q] = ring[(ph + W - 1) % W][q];
      }
      const int o = p - F_R;
      if (o >= 0) {
        float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
        for (int t = 0; t < W; ++t) {
          if (t < F_R - r || t > F_R + r) continue;  // CTA-uniform
          const int sl = (ph + 1 + t) % W;  // position p - 12 + t
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[q] = __fmaf_rn(tp[t], ring[sl][q], acc[q]);
        }
        finish(o, acc);
      }
    }
  }
}

template <bool HAS_BIAS, bool EPI>
__global__ void __launch_bounds__(256, EPI ? 1 : 2)
march6_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int I, int J,
              int K, BlurArgs bl, BiasArgs bi, NoiseArgs nz, const float* __restrict__ gamma) {
  extern __shared__ __align__(16) float smem[];
  march6_tile<HAS_BIAS, EPI, 0>(smem, threadIdx.y * blockDim.x + threadIdx.x,
                                (blockIdx.x * blockDim.x + threadIdx.x) * 4,
                                blockIdx.y * blockDim.y + threadIdx.y, blockIdx.z, src, dst, B, C, I, J, K,
                                bl, bi, nz, gamma);
}

// -------------------------------------------------------------------------
// pass 1 and the normal stage of the exact-noise replay (mt19937_normal.cuh) in one persistent
// kernel, one CTA of 7 warpgroups per SM.  Pass 1 is bound by HBM and leaves most issue slots
// empty; the normal stage is bound by issue and writes 4 B/voxel.  As two kernels they cannot
// share an SM (either one's CTAs fill the register file), so here the two roles split one CTA's
// registers with setmaxnreg: the kernel starts at 72 registers per thread (896 x 72 = 64 512),
//   warpgroups 0-1  the 256 threads of march6_kernel<HAS_BIAS, false>, raised to 152 registers
//                   (at 128 the bias variant spills):
//                   tiles (k-block, j-block, b*c) of that kernel's grid, x fastest, handed out by
//                   a global counter;
//   warpgroups 2-6  lowered to 40 registers: the first MT_THREADS threads run segment after
//                   segment of the normal stage compiled for aligned [0, n) draws
//                   (q = q_lo + blockIdx.x, + gridDim.x, ...), the other 64 leave;
// 256 x 152 + 640 x 40 = 64 512 registers after the exchange.  Both bodies are the device
// functions the stand-alone kernels run (the normal stage with the same Box-Muller arithmetic),
// so the outputs are theirs bit for bit.  Named barriers:
// 1..5 inside the normal stage, P1N_BAR_SEGMENT between its segments, P1N_BAR_MARCH for pass 1;
// barrier 0 is never used after the roles part.
// -------------------------------------------------------------------------
constexpr int P1N_MARCH_THREADS = 256;
constexpr int P1N_THREADS = P1N_MARCH_THREADS + 5 * 128;  // 896
constexpr int P1N_BAR_SEGMENT = 6, P1N_BAR_MARCH = 7;
constexpr int P1N_RING_FLOATS = MT_RING_WORDS + 4;  // the normal stage's ring, then the tile slot

template <bool HAS_BIAS>
__global__ void __launch_bounds__(P1N_THREADS, 1)
pass1_normals_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int I, int J,
                     int K, BlurArgs bl, BiasArgs bi, unsigned int* __restrict__ tile_counter,
                     const uint32_t* __restrict__ states, int q_lo, int q_hi, unsigned long long L,
                     unsigned long long offset, unsigned long long n, float* __restrict__ z) {
  extern __shared__ __align__(16) float smem[];
  if (threadIdx.x < P1N_MARCH_THREADS) {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 152;");
    const int tid = threadIdx.x;
    volatile int* next_tile = reinterpret_cast<int*>(smem + MT_RING_WORDS);
    const int kb_n = (K + 255) / 256, jb_n = (J + 3) / 4;
    const int tiles = kb_n * jb_n * B * C;
    for (;;) {
      if (tid == 0) *next_tile = (int)atomicAdd(tile_counter, 1u);
      // every thread has left the previous tile: its taps and bias grid may be replaced
      asm volatile("bar.sync %0, 256;" ::"n"(P1N_BAR_MARCH) : "memory");
      const int tile = *next_tile;  // rewritten only after the barrier inside march6_tile
      if (tile >= tiles) break;
      const int kb = tile % kb_n, jb = (tile / kb_n) % jb_n, bc = tile / (kb_n * jb_n);
      march6_tile<HAS_BIAS, false, P1N_BAR_MARCH>(smem + P1N_RING_FLOATS, tid, (kb * 64 + (tid & 63)) * 4,
                                                  jb * 4 + (tid >> 6), bc, src, dst, B, C, I, J, K, bl, bi,
                                                  NoiseArgs{}, nullptr);
    }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    const int tid = threadIdx.x - P1N_MARCH_THREADS;
    if (tid >= MT_THREADS) return;
    for (int q = q_lo + blockIdx.x; q < q_hi; q += gridDim.x) {
      mt_normal_segment<false>(reinterpret_cast<uint32_t*>(smem), tid, states, q, L, offset, n, 0, n, z);
      // the last consumers have left the ring before the next segment's start state enters it
      mt_bar_sync<P1N_BAR_SEGMENT, MT_THREADS>();
    }
  }
}

// -------------------------------------------------------------------------
// one blur axis for tables with R > 16 (sigma > 16/3 voxels), any radius: thread <-> output
// voxel, clamped (replicate) reads along the axis, the element's 2r+1 taps in shared memory,
// accumulated from offset -r to +r as every other path does.  Consecutive threads are
// consecutive k, so every tap read is coalesced; the windows of neighbours overlap in L1/L2.
//   HAS_EPI = last launch of the chain: noise and gamma at the store.
// -------------------------------------------------------------------------
constexpr int WIDE_RMAX = 6143;  // 2R+1 fp32 taps in 48 KiB of shared memory

template <bool HAS_EPI>
__global__ void __launch_bounds__(256)
axis_kernel(const float* __restrict__ src, float* __restrict__ dst, int B, int C, int I, int J,
            int K, int axis, BlurArgs bl, NoiseArgs nz, const float* __restrict__ gamma) {
  extern __shared__ float taps_s[];  // [2r+1]
  const int bc = blockIdx.y;
  const int b = bc / C;
  const int tid = threadIdx.x;
  const int64_t n = (int64_t)I * J * K;
  const int r = bl.radius[axis * B + b];
  for (int t = tid; t < 2 * r + 1; t += 256)
    taps_s[t] = bl.taps[((int64_t)axis * B + b) * (2 * bl.R + 1) + bl.R - r + t];
  __syncthreads();
  const int64_t e = (int64_t)blockIdx.x * 256 + tid;  // voxel within the (b, c) volume
  if (e >= n) return;
  const int L = axis == 0 ? I : (axis == 1 ? J : K);
  const int64_t s = axis == 0 ? (int64_t)J * K : (axis == 1 ? K : 1);
  const int pos = (int)((e / s) % L);
  const float* x = src + (int64_t)bc * n + (e - pos * s);
  float acc;
  if (r == 0) {
    acc = x[pos * s];
  } else {
    acc = 0.0f;
    for (int t = 0; t <= 2 * r; ++t) {
      const int q = min(max(pos - r + t, 0), L - 1);
      acc = __fmaf_rn(taps_s[t], __ldg(x + q * s), acc);
    }
  }
  const int64_t flat = (int64_t)bc * n + e;
  if (HAS_EPI) {
    if (nz.mode != 0 && (!nz.keep || nz.keep[b])) {
      const float mu = nz.mean[b], sd = nz.std[b];
      float z1, z2 = 0.0f;
      if (nz.mode == 1) {
        z1 = nz.z[flat];
        if (nz.rician) z2 = nz.z2[flat];
      } else {
        const uint2 key = make_uint2((uint32_t)nz.philox_seed, (uint32_t)(nz.philox_seed >> 32));
        float unused;
        uint4 rr = philox4x32_10(make_uint4((uint32_t)flat, (uint32_t)((uint64_t)flat >> 32), 0u, 0x77ffu), key);
        box_muller(rr.x, rr.y, z1, unused);
        if (nz.rician) box_muller(rr.z, rr.w, z2, unused);
      }
      const float n1 = __fadd_rn(mu, __fmul_rn(sd, z1));
      acc = nz.rician ? rician(acc, n1, __fadd_rn(mu, __fmul_rn(sd, z2))) : __fadd_rn(acc, n1);
    }
    if (gamma) acc = signed_pow(acc, gamma[b]);
  }
  dst[flat] = acc;
}

static inline bool aligned16f(const void* p) { return ((uintptr_t)p & 15) == 0; }

static float up_scale(int n_in, int n_out) {
  if (n_in == n_out) return 1.0f;
  return n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.0f;
}

template <int RMAX>
static int launch_jk(const float* src, float* dst, int B, int C, int I, int J, int K,
                     const BlurArgs& bl, const NoiseArgs& nz, const float* gamma, cudaStream_t st) {
  constexpr int ROWS = A_TJ + 2 * RMAX, COLS = A_TK + 2 * RMAX, PITCH = (COLS + 3) / 4 * 4 + 4;
  const size_t smem = (size_t)(ROWS * PITCH + ROWS * A_TK + 2 * (2 * RMAX + 1)) * sizeof(float);
  const int tiles_i = (I + A_PLANES - 1) / A_PLANES;
  dim3 grid((K + A_TK - 1) / A_TK, (J + A_TJ - 1) / A_TJ, B * C * tiles_i);
  if (nz.mode != 0 || gamma) {
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(jk_kernel<RMAX, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    jk_kernel<RMAX, true><<<grid, 256, smem, st>>>(src, dst, B, C, I, J, K, bl, nz, gamma);
  } else {
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(jk_kernel<RMAX, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    jk_kernel<RMAX, false><<<grid, 256, smem, st>>>(src, dst, B, C, I, J, K, bl, nz, gamma);
  }
  launched();
  return 0;
}

// pass 1: bias + I-conv (ib.taps == null: no I-conv) + the noise/gamma epilogue when nz1 / gamma1
// are set; march6_kernel when the table radius is <= 6 and rows are 16-byte aligned
static int launch_march(const float* cur, float* out, int B, int C, int I, int J, int K,
                        const BiasArgs& bi, const BlurArgs& ib, const NoiseArgs& nz1,
                        const float* gamma1, cudaStream_t st, const char* who) {
  {
    const bool vec = (K % 4 == 0) && aligned16f(cur) && aligned16f(out) &&
                     (nz1.mode != 1 || (aligned16f(nz1.z) && (!nz1.z2 || aligned16f(nz1.z2))));
    const int V = vec ? 4 : 1;
    dim3 block(64, 4);
    dim3 grid((K + 64 * V - 1) / (64 * V), (J + 3) / 4, B * C);
    TIO_CHECK_ARG(grid.y <= 65535, "%s: J too large", who);
    const int R = ib.taps ? ib.R : 0;
    const int ns = bi.coarse ? bi.si * bi.sj * bi.sk : 0;
    const size_t smem = ((size_t)((2 * R + 1 + 3) / 4 * 4) + (size_t)((ns + 3) / 4 * 4) +
                         (ib.taps ? (size_t)(2 * R + 1) * 256 * V : 0)) * sizeof(float);
#define TIO_LAUNCH_MARCH(VV, BB)                                                              \
  do {                                                                                        \
    if (smem > 48 * 1024)                                                                     \
      cudaFuncSetAttribute(march_kernel<VV, BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)smem);                                                        \
    march_kernel<VV, BB><<<grid, block, smem, st>>>(cur, out, B, C, I, J, K, ib, bi, nz1, gamma1); \
    launched();                                                                               \
  } while (0)
    if (vec && R <= F_R) {
      const size_t smem6 = (size_t)(16 + (ns + 3) / 4 * 4) * sizeof(float) + (size_t)M6_PF * 256 * 16;
#define TIO_LAUNCH_MARCH6(BB, EE)                                                              \
  do {                                                                                         \
    if (smem6 > 48 * 1024)                                                                     \
      cudaFuncSetAttribute(march6_kernel<BB, EE>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)smem6);                                                        \
    march6_kernel<BB, EE><<<grid, block, smem6, st>>>(cur, out, B, C, I, J, K, ib, bi, nz1, gamma1); \
    launched();                                                                                \
  } while (0)
      const bool epi = nz1.mode != 0 || gamma1 != nullptr;
      if (bi.coarse) { if (epi) TIO_LAUNCH_MARCH6(true, true); else TIO_LAUNCH_MARCH6(true, false); }
      else { if (epi) TIO_LAUNCH_MARCH6(false, true); else TIO_LAUNCH_MARCH6(false, false); }
#undef TIO_LAUNCH_MARCH6
    } else if (vec) { if (bi.coarse) TIO_LAUNCH_MARCH(4, true); else TIO_LAUNCH_MARCH(4, false); }
    else { if (bi.coarse) TIO_LAUNCH_MARCH(1, true); else TIO_LAUNCH_MARCH(1, false); }
#undef TIO_LAUNCH_MARCH
  }
  return 0;
}

// Tables with R > 16: bias (pass 1 without taps), then one axis_kernel launch per active
// axis in the order I, K, J of the other paths; the epilogue rides on the last launch.  The
// launches ping-pong between scratch and dst so that the last one writes dst.
static int wide_impl(const float* src, float* dst, float* scratch, int B, int C, int I, int J,
                     int K, const BiasArgs& bi, const BlurArgs& bl, int axes_mask,
                     const NoiseArgs& nz, const float* gamma, cudaStream_t st, const char* who) {
  TIO_CHECK_ARG(bl.R <= WIDE_RMAX, "%s: blur radius R=%d > %d unsupported", who, bl.R, WIDE_RMAX);
  int axes[3], na = 0;
  for (int a : {0, 2, 1})
    if (axes_mask & (1 << a)) axes[na++] = a;
  const int steps = na + (bi.coarse ? 1 : 0);
  TIO_CHECK_ARG(src != dst && (steps < 2 || (scratch && scratch != src && scratch != dst)),
                "%s: blur radius R=%d > 16 needs src != dst and a scratch buffer", who, bl.R);
  const int64_t n = (int64_t)I * J * K;
  TIO_CHECK_ARG((n + 255) / 256 <= 0x7fffffff, "%s: volume too large", who);
  const float* cur = src;
  int left = steps;
  auto next_out = [&]() { return (--left % 2 == 0) ? dst : scratch; };
  if (bi.coarse) {
    BlurArgs none = bl;
    none.taps = nullptr;
    float* out = next_out();
    if (launch_march(cur, out, B, C, I, J, K, bi, none, NoiseArgs{}, nullptr, st, who)) return 1;
    cur = out;
  }
  const size_t smem = (size_t)(2 * bl.R + 1) * sizeof(float);
  dim3 grid((unsigned)((n + 255) / 256), B * C);
  for (int s = 0; s < na; ++s) {
    float* out = next_out();
    if (s == na - 1 && (nz.mode != 0 || gamma))
      axis_kernel<true><<<grid, 256, smem, st>>>(cur, out, B, C, I, J, K, axes[s], bl, nz, gamma);
    else
      axis_kernel<false><<<grid, 256, smem, st>>>(cur, out, B, C, I, J, K, axes[s], bl, nz, gamma);
    launched();
    cur = out;
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

static int fused_impl(const float* src, float* dst, float* scratch, int B, int C, int I, int J,
                      int K, BiasArgs bi, BlurArgs bl, int axes_mask, NoiseArgs nz,
                      const float* gamma, cudaStream_t st, const char* who) {
  TIO_CHECK_ARG(src && dst, "%s: null src/dst", who);
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "%s: bad shape", who);
  TIO_CHECK_ARG((int64_t)B * C <= 65535, "%s: B*C must be <= 65535", who);
  if (!bl.taps) axes_mask = 0;
  TIO_CHECK_ARG(!bl.taps || (bl.radius && bl.R >= 0), "%s: blur radius table missing or R=%d < 0", who, bl.R);
  if (bi.coarse) {
    bi.sc_i = up_scale(bi.si, I); bi.sc_j = up_scale(bi.sj, J); bi.sc_k = up_scale(bi.sk, K);
    TIO_CHECK_ARG((size_t)bi.si * bi.sj * bi.sk * 4 <= 64 * 1024, "%s: coarse bias grid too large", who);
  }
  if (axes_mask != 0 && bl.R > 16)
    return wide_impl(src, dst, scratch, B, C, I, J, K, bi, bl, axes_mask, nz, gamma, st, who);
  const bool need_jk = (axes_mask & 6) != 0;
  const bool need_i = (axes_mask & 1) != 0;
  const bool need_march = !need_jk || need_i || bi.coarse != nullptr;
  TIO_CHECK_ARG(!need_jk || src != dst, "%s: blur along J/K needs src != dst", who);
  // J/K alone (the caller ran pass 1 itself: tio_intensity_pass1_with_normals) reads src directly
  TIO_CHECK_ARG(!(need_jk && need_march) || (scratch && scratch != src && scratch != dst),
                "%s: blur along J/K after bias or blur along I needs a scratch buffer", who);
  TIO_CHECK_ARG(!((axes_mask & 1) && src == dst && !need_jk), "%s: blur along I needs src != dst", who);
  const float* cur = src;
  if (need_jk) {
    // checked before any launch
    const int64_t tiles = (int64_t)B * C * ((I + A_PLANES - 1) / A_PLANES);
    TIO_CHECK_ARG(tiles <= 65535, "%s: batch too large for the blur grid", who);
  }
  if (need_march) {
    BlurArgs ib = bl;
    if (!need_i) ib.taps = nullptr;
    float* out = need_jk ? scratch : dst;
    if (launch_march(cur, out, B, C, I, J, K, bi, ib, need_jk ? NoiseArgs{} : nz,
                     need_jk ? nullptr : gamma, st, who))
      return 1;
    cur = out;
  }
  if (need_jk) {
    // pass 2: K-conv, J-conv, then noise and gamma at the store
    // TMA: 16-byte aligned base and row pitch; coordinates must fit int32
    const bool tma_ok = bl.R <= F_R && (K % 4 == 0) && aligned16f(cur) && (int64_t)B * C * I < (1ll << 31);
    EncodeTiledFn encode = tma_ok ? encode_tiled_fn() : nullptr;
    CUtensorMap tm;
    bool have_map = false;
    if (encode) {
      const cuuint64_t gdim[3] = {(cuuint64_t)K, (cuuint64_t)J, (cuuint64_t)B * C * I};
      const cuuint64_t gstride[2] = {(cuuint64_t)K * 4, (cuuint64_t)J * K * 4};
      const cuuint32_t bdim[3] = {(cuuint32_t)F_COLS, (cuuint32_t)F_ROWS, 1};
      const cuuint32_t estr[3] = {1, 1, 1};
      have_map = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(cur), gdim, gstride,
                        bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
    }
    if (have_map) {
      const int tiles_i = (I + A_PLANES - 1) / A_PLANES;
      dim3 grid((K + A_TK - 1) / A_TK, (J + A_TJ - 1) / A_TJ, B * C * tiles_i);
      if (nz.mode != 0 || gamma) {
        cudaFuncSetAttribute(jk6_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F_SMEM);
        jk6_kernel<true><<<grid, 256, F_SMEM, st>>>(tm, dst, B, C, I, J, K, bl, nz, gamma);
      } else {
        cudaFuncSetAttribute(jk6_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)F_SMEM);
        jk6_kernel<false><<<grid, 256, F_SMEM, st>>>(tm, dst, B, C, I, J, K, bl, nz, gamma);
      }
      launched();
    } else if (bl.R <= F_R) {
      launch_jk<6>(cur, dst, B, C, I, J, K, bl, nz, gamma, st);
    } else {
      launch_jk<16>(cur, dst, B, C, I, J, K, bl, nz, gamma, st);
    }
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

}  // namespace tio

using namespace tio;

extern "C" int tio_blur(const float* src, float* dst, float* scratch, int B, int C, int I, int J,
                        int K, const float* taps, const int32_t* radius, int R, int axes_mask,
                        const uint8_t* identity, void* stream) {
  (void)identity;  // rows whose radii are all 0 stream through as bit-exact copies
  TIO_CHECK_ARG(taps && radius, "tio_blur: null taps/radius");
  TIO_CHECK_ARG(src != dst, "tio_blur: src and dst must not alias");
  BiasArgs bi{};
  BlurArgs bl{taps, radius, R};
  NoiseArgs nz{};
  return fused_impl(src, dst, scratch, B, C, I, J, K, bi, bl, axes_mask & 7, nz, nullptr,
                    (cudaStream_t)stream, "tio_blur");
}

extern "C" int tio_intensity_fused(const float* src, float* dst, float* scratch, int B, int C,
                                   int I, int J, int K, const float* coarse, int si, int sj,
                                   int sk, const uint8_t* bias_identity, int bias_divide,
                                   const float* taps, const int32_t* radius, int R,
                                   int axes_mask, const float* mean, const float* std,
                                   const uint8_t* keep, const float* z, const float* z2,
                                   uint64_t philox_seed, int noise_mode, int rician_flag,
                                   const float* gamma, void* stream) {
  BiasArgs bi{};
  bi.coarse = coarse; bi.identity = bias_identity; bi.si = si; bi.sj = sj; bi.sk = sk;
  bi.divide = bias_divide;
  BlurArgs bl{taps, radius, R};
  NoiseArgs nz{};
  nz.mode = noise_mode;
  TIO_CHECK_ARG(noise_mode >= 0 && noise_mode <= 2, "tio_intensity_fused: bad noise_mode");
  if (noise_mode) {
    TIO_CHECK_ARG(mean && std, "tio_intensity_fused: noise needs mean/std");
    TIO_CHECK_ARG(noise_mode != 1 || (z && (!rician_flag || z2)), "tio_intensity_fused: normals missing");
    nz.mean = mean; nz.std = std; nz.keep = keep; nz.z = z; nz.z2 = z2;
    nz.philox_seed = philox_seed; nz.rician = rician_flag;
  }
  return fused_impl(src, dst, scratch, B, C, I, J, K, bi, bl, taps ? (axes_mask & 7) : 0, nz,
                    gamma, (cudaStream_t)stream, "tio_intensity_fused");
}

extern "C" size_t tio_intensity_pass1_with_normals_workspace_bytes(uint64_t offset, uint64_t n) {
  return tio_randn_mt19937_workspace_bytes(offset, n) + 16;  // start states, then the tile counter
}

extern "C" int tio_intensity_pass1_with_normals(const float* src, float* dst, int B, int C, int I, int J,
                                                int K, const float* coarse, int si, int sj, int sk,
                                                const uint8_t* bias_identity, int bias_divide,
                                                const float* taps, const int32_t* radius, int R,
                                                int axes_mask, uint64_t seed, uint64_t offset, uint64_t n,
                                                float* z, const void* table, void* workspace,
                                                size_t workspace_bytes, void* stream) {
  const char* who = "tio_intensity_pass1_with_normals";
  TIO_CHECK_ARG(src && dst && z, "%s: null src/dst/z", who);
  TIO_CHECK_ARG(src != dst, "%s: src and dst must not alias", who);
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "%s: bad shape", who);
  const bool need_i = taps && (axes_mask & 1);
  TIO_CHECK_ARG(!need_i || (radius && R >= 0 && R <= F_R), "%s: needs a radius table and R <= %d, got R=%d", who,
                F_R, R);
  TIO_CHECK_ARG(K % 4 == 0 && aligned16f(src) && aligned16f(dst) && aligned16f(z),
                "%s: needs K %% 4 == 0 and 16-byte aligned src, dst and z", who);
  const int64_t tiles = (int64_t)((K + 255) / 256) * ((J + 3) / 4) * B * C;
  TIO_CHECK_ARG(tiles < (1ll << 31) - (1 << 20), "%s: batch too large", who);
  BiasArgs bi{};
  bi.coarse = coarse; bi.identity = bias_identity; bi.si = si; bi.sj = sj; bi.sk = sk;
  bi.divide = bias_divide;
  if (coarse) {
    bi.sc_i = up_scale(si, I); bi.sc_j = up_scale(sj, J); bi.sc_k = up_scale(sk, K);
    TIO_CHECK_ARG(si > 0 && sj > 0 && sk > 0 && (size_t)si * sj * sk * 4 <= 64 * 1024,
                  "%s: coarse bias grid empty or too large", who);
  }
  BlurArgs bl{need_i ? taps : nullptr, radius, R};
  TIO_CHECK_ARG(n >= 16 && (n % 16) == 0 && (offset % 16) == 0, "%s: n and offset must be multiples of 16 (n >= 16)",
                who);
  TIO_CHECK_ARG(workspace_bytes >= tio_intensity_pass1_with_normals_workspace_bytes(offset, n),
                "%s: workspace too small", who);
  cudaStream_t st = (cudaStream_t)stream;
  int q_lo, q_hi;
  const size_t states_bytes = tio_randn_mt19937_workspace_bytes(offset, n);
  if (int rc = mt_start_states(seed, offset, offset + n - 16, table, workspace, states_bytes, st, who, &q_lo, &q_hi))
    return rc;
  unsigned int* tile_counter = reinterpret_cast<unsigned int*>((char*)workspace + states_bytes);
  cudaMemsetAsync(tile_counter, 0, sizeof(unsigned int), st);
  const int ns = coarse ? si * sj * sk : 0;
  const size_t smem = (size_t)(P1N_RING_FLOATS + 16 + (ns + 3) / 4 * 4) * sizeof(float) + (size_t)M6_PF * 256 * 16;
  const unsigned long long seg = 1ull << tio_mt::kLog2L;
  const int grid = num_sms();
#define TIO_LAUNCH_P1N(BB)                                                                                   \
  do {                                                                                                       \
    cudaFuncSetAttribute(pass1_normals_kernel<BB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);  \
    pass1_normals_kernel<BB><<<grid, P1N_THREADS, smem, st>>>(src, dst, B, C, I, J, K, bl, bi, tile_counter, \
                                                              (const uint32_t*)workspace, q_lo, q_hi, seg,   \
                                                              offset, n, z);                                 \
    launched();                                                                                              \
  } while (0)
  if (coarse) TIO_LAUNCH_P1N(true); else TIO_LAUNCH_P1N(false);
#undef TIO_LAUNCH_P1N
  TIO_CHECK_LAUNCH();
  return 0;
}

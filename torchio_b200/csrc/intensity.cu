// intensity.cu — K2 bias field, K3 separable blur, K4 noise, K5 gamma.
//
// Replaces the tensor math of TorchIO 2.0.0a2's
//   transforms/intensity/bias_field.py:201-255,296-341
//   transforms/intensity/blur.py:129-252
//   transforms/intensity/noise.py:98-178
//   transforms/intensity/gamma.py:80-120
// All kernels are HBM-bound elementwise / stencil passes: 128-bit accesses
// along K, grid sized to the volume, no tensor cores.
#include "common.cuh"
#include "intensity_common.cuh"

namespace tio {

// ---------------------------------------------------------------------------
// K2: dst = src * exp(trilerp(coarse))     (or / for the inverse)
// thread <-> V consecutive k of one (j) row, walking TI planes along I; the
// J/K levels of the nested lerp stay in registers across the walk.
// ---------------------------------------------------------------------------
constexpr int B_TI = 16;

template <int V>
__global__ void __launch_bounds__(256)
bias_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, int I, int J, int K,
            const float* __restrict__ coarse, int si, int sj, int sk, float sc_i, float sc_j,
            float sc_k, const uint8_t* __restrict__ identity, int divide) {
  extern __shared__ float g[];
  const int tiles_i = (I + B_TI - 1) / B_TI;
  const int bc = blockIdx.z / tiles_i;
  const int i_begin = (blockIdx.z % tiles_i) * B_TI;
  const int i_end = min(i_begin + B_TI, I);
  const int b = bc / C;
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  const int j = blockIdx.y * blockDim.y + threadIdx.y;
  const int64_t n = (int64_t)I * J * K;
  const float* x = src + (int64_t)bc * n;
  float* y = dst + (int64_t)bc * n;
  const bool ident = identity && identity[b];
  if (!ident) {
    const int ns = si * sj * sk;
    const float* gs = coarse + (int64_t)bc * ns;
    for (int t = threadIdx.y * blockDim.x + threadIdx.x; t < ns; t += blockDim.x * blockDim.y)
      g[t] = gs[t];
    __syncthreads();
  }
  if (k >= K || j >= J) return;
  if (ident) {
    if (x != y)
      for (int i = i_begin; i < i_end; ++i) {
        int64_t o = ((int64_t)i * J + j) * K + k;
        if (V == 4) *(float4*)(y + o) = *(const float4*)(x + o);
        else y[o] = x[o];
      }
    return;
  }
  const LerpAxis lj = lerp_axis(sc_j, sj, j);
  LerpAxis lk[V];
#pragma unroll
  for (int v = 0; v < V; ++v) lk[v] = lerp_axis(sc_k, sk, k + v);
  int cur0 = -1, cur1 = -1;
  float r_lo[V], r_hi[V];
  for (int i = i_begin; i < i_end; ++i) {
    const LerpAxis li = lerp_axis(sc_i, si, i);
    if (li.i0 != cur0 || li.i1 != cur1) {
      const float* p0 = g + (li.i0 * sj) * sk;
      const float* p1 = g + (li.i1 * sj) * sk;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        float a0 = lerp2(lk[v].l0, p0[lj.i0 * sk + lk[v].i0], lk[v].l1, p0[lj.i0 * sk + lk[v].i1]);
        float a1 = lerp2(lk[v].l0, p0[lj.i1 * sk + lk[v].i0], lk[v].l1, p0[lj.i1 * sk + lk[v].i1]);
        r_lo[v] = lerp2(lj.l0, a0, lj.l1, a1);
        float b0 = lerp2(lk[v].l0, p1[lj.i0 * sk + lk[v].i0], lk[v].l1, p1[lj.i0 * sk + lk[v].i1]);
        float b1 = lerp2(lk[v].l0, p1[lj.i1 * sk + lk[v].i0], lk[v].l1, p1[lj.i1 * sk + lk[v].i1]);
        r_hi[v] = lerp2(lj.l0, b0, lj.l1, b1);
      }
      cur0 = li.i0;
      cur1 = li.i1;
    }
    const int64_t o = ((int64_t)i * J + j) * K + k;
    float xv[V], yv[V];
    if (V == 4) {
      float4 t = *(const float4*)(x + o);
      xv[0] = t.x; xv[1] = t.y; xv[2] = t.z; xv[3] = t.w;
    } else {
      xv[0] = x[o];
    }
#pragma unroll
    for (int v = 0; v < V; ++v) {
      float f = expf(lerp2(li.l0, r_lo[v], li.l1, r_hi[v]));
      yv[v] = divide ? __fdiv_rn(xv[v], f) : __fmul_rn(xv[v], f);
    }
    if (V == 4) *(float4*)(y + o) = make_float4(yv[0], yv[1], yv[2], yv[3]);
    else y[o] = yv[0];
  }
}

// ---------------------------------------------------------------------------
// K4: noise (given normals) / Philox variant;  K5: gamma
// ---------------------------------------------------------------------------
template <int V, bool RICIAN>
__global__ void __launch_bounds__(256)
noise_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t per_elem,
             const float* __restrict__ mean, const float* __restrict__ std,
             const uint8_t* __restrict__ keep, const float* __restrict__ z,
             const float* __restrict__ z2) {
  const int b = blockIdx.y;
  const float mu = mean[b], sd = std[b];
  const bool kept = !keep || keep[b];
  const int64_t base = (int64_t)b * per_elem;
  const int64_t nvec = per_elem / V;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nvec;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = base + t * V;
    float xv[V], zv[V], z2v[V];
    if (V == 4) {
      float4 a = *(const float4*)(src + o);
      xv[0] = a.x; xv[1] = a.y; xv[2] = a.z; xv[3] = a.w;
      if (kept) {
        float4 c = __ldcs((const float4*)(z + o));
        zv[0] = c.x; zv[1] = c.y; zv[2] = c.z; zv[3] = c.w;
        if (RICIAN) {
          float4 e = __ldcs((const float4*)(z2 + o));
          z2v[0] = e.x; z2v[1] = e.y; z2v[2] = e.z; z2v[3] = e.w;
        }
      }
    } else {
      xv[0] = src[o];
      if (kept) { zv[0] = z[o]; if (RICIAN) z2v[0] = z2[o]; }
    }
    float yv[V];
#pragma unroll
    for (int v = 0; v < V; ++v) {
      if (!kept) { yv[v] = xv[v]; continue; }
      // reference: mean + std*base, then data + noise (noise.py:178,119)
      float n1 = __fadd_rn(mu, __fmul_rn(sd, zv[v]));
      if (RICIAN) yv[v] = rician(xv[v], n1, __fadd_rn(mu, __fmul_rn(sd, z2v[v])));
      else yv[v] = __fadd_rn(xv[v], n1);
    }
    if (V == 4) *(float4*)(dst + o) = make_float4(yv[0], yv[1], yv[2], yv[3]);
    else dst[o] = yv[0];
  }
}

template <bool RICIAN>
__global__ void __launch_bounds__(256)
noise_philox_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t per_elem,
                    const float* __restrict__ mean, const float* __restrict__ std,
                    const uint8_t* __restrict__ keep, uint64_t seed) {
  const int b = blockIdx.y;
  const float mu = mean[b], sd = std[b];
  const bool kept = !keep || keep[b];
  const int64_t base = (int64_t)b * per_elem;
  const int64_t ngrp = (per_elem + 3) / 4;
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const bool vec = ((per_elem & 3) == 0);
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < ngrp;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = base + t * 4;
    const int cnt = (int)min((int64_t)4, per_elem - t * 4);
    float xv[4] = {0.f, 0.f, 0.f, 0.f}, yv[4];
    if (vec) {
      float4 a = *(const float4*)(src + o);
      xv[0] = a.x; xv[1] = a.y; xv[2] = a.z; xv[3] = a.w;
    } else {
      for (int v = 0; v < cnt; ++v) xv[v] = src[o + v];
    }
    if (kept) {
      const uint64_t gidx = (uint64_t)t;  // group index inside element b
      uint4 r = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 0u, (uint32_t)b), key);
      float n[4];
      box_muller(r.x, r.y, n[0], n[1]);
      box_muller(r.z, r.w, n[2], n[3]);
      float m2[4];
      if (RICIAN) {
        uint4 r2 = philox4x32_10(make_uint4((uint32_t)gidx, (uint32_t)(gidx >> 32), 1u, (uint32_t)b), key);
        box_muller(r2.x, r2.y, m2[0], m2[1]);
        box_muller(r2.z, r2.w, m2[2], m2[3]);
      }
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        float n1 = __fadd_rn(mu, __fmul_rn(sd, n[v]));
        if (RICIAN) yv[v] = rician(xv[v], n1, __fadd_rn(mu, __fmul_rn(sd, m2[v])));
        else yv[v] = __fadd_rn(xv[v], n1);
      }
    } else {
#pragma unroll
      for (int v = 0; v < 4; ++v) yv[v] = xv[v];
    }
    if (vec) *(float4*)(dst + o) = make_float4(yv[0], yv[1], yv[2], yv[3]);
    else for (int v = 0; v < cnt; ++v) dst[o + v] = yv[v];
  }
}

template <int V>
__global__ void __launch_bounds__(256)
gamma_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t per_elem,
             const float* __restrict__ gamma) {
  const int b = blockIdx.y;
  const float gam = gamma[b];
  const int64_t base = (int64_t)b * per_elem;
  const int64_t nvec = per_elem / V;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nvec;
       t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = base + t * V;
    if (V == 4) {
      float4 a = *(const float4*)(src + o);
      *(float4*)(dst + o) = make_float4(signed_pow(a.x, gam), signed_pow(a.y, gam),
                                        signed_pow(a.z, gam), signed_pow(a.w, gam));
    } else {
      dst[o] = signed_pow(src[o], gam);
    }
  }
}

static inline int ew_blocks(int64_t nvec) {
  int64_t blocks = (nvec + 255) / 256;
  int64_t cap = (int64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

static inline bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

}  // namespace tio

using namespace tio;

extern "C" int tio_bias_field(const float* src, float* dst, int B, int C, int I, int J, int K,
                              const float* coarse, int si, int sj, int sk,
                              const uint8_t* identity, int divide, void* stream) {
  TIO_CHECK_ARG(src && dst && coarse, "tio_bias_field: null pointer");
  TIO_CHECK_ARG(B > 0 && C > 0 && I > 0 && J > 0 && K > 0, "tio_bias_field: bad shape");
  TIO_CHECK_ARG(si >= 1 && sj >= 1 && sk >= 1 && (size_t)si * sj * sk * 4 <= 200 * 1024,
                "tio_bias_field: coarse grid %dx%dx%d unsupported", si, sj, sk);
  auto scale = [](int n_in, int n_out) {
    if (n_in == n_out) return 1.0f;
    return n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.0f;
  };
  const int tiles_i = (I + B_TI - 1) / B_TI;
  TIO_CHECK_ARG((int64_t)B * C * tiles_i <= 65535, "tio_bias_field: batch too large");
  const size_t smem = (size_t)si * sj * sk * sizeof(float);
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (K % 4 == 0) && aligned16(src) && aligned16(dst);
  if (vec) {
    dim3 block(64, 4);
    dim3 grid((K / 4 + 63) / 64, (J + 3) / 4, B * C * tiles_i);
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(bias_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    bias_kernel<4><<<grid, block, smem, st>>>(src, dst, C, I, J, K, coarse, si, sj, sk,
                                              scale(si, I), scale(sj, J), scale(sk, K), identity,
                                              divide);
  } else {
    dim3 block(64, 4);
    dim3 grid((K + 63) / 64, (J + 3) / 4, B * C * tiles_i);
    if (smem > 48 * 1024)
      cudaFuncSetAttribute(bias_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    bias_kernel<1><<<grid, block, smem, st>>>(src, dst, C, I, J, K, coarse, si, sj, sk,
                                              scale(si, I), scale(sj, J), scale(sk, K), identity,
                                              divide);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_noise(const float* src, float* dst, int B, int64_t per_elem, const float* mean,
                         const float* std, const uint8_t* keep, const float* z, const float* z2,
                         void* stream) {
  TIO_CHECK_ARG(src && dst && mean && std && z, "tio_noise: null pointer");
  TIO_CHECK_ARG(B > 0 && B <= 65535 && per_elem > 0, "tio_noise: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (per_elem % 4 == 0) && aligned16(src) && aligned16(dst) && aligned16(z) &&
                   (!z2 || aligned16(z2));
  const int64_t nvec = vec ? per_elem / 4 : per_elem;
  dim3 grid(ew_blocks(nvec), B);
  if (vec) {
    if (z2) noise_kernel<4, true><<<grid, 256, 0, st>>>(src, dst, per_elem, mean, std, keep, z, z2);
    else noise_kernel<4, false><<<grid, 256, 0, st>>>(src, dst, per_elem, mean, std, keep, z, z2);
  } else {
    if (z2) noise_kernel<1, true><<<grid, 256, 0, st>>>(src, dst, per_elem, mean, std, keep, z, z2);
    else noise_kernel<1, false><<<grid, 256, 0, st>>>(src, dst, per_elem, mean, std, keep, z, z2);
  }
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_noise_philox(const float* src, float* dst, int B, int64_t per_elem,
                                const float* mean, const float* std, const uint8_t* keep,
                                uint64_t seed, int rician_flag, void* stream) {
  TIO_CHECK_ARG(src && dst && mean && std, "tio_noise_philox: null pointer");
  TIO_CHECK_ARG(B > 0 && B <= 65535 && per_elem > 0, "tio_noise_philox: bad shape");
  TIO_CHECK_ARG(aligned16(src) && aligned16(dst) || (per_elem & 3), "tio_noise_philox: misaligned");
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid(ew_blocks((per_elem + 3) / 4), B);
  if (rician_flag)
    noise_philox_kernel<true><<<grid, 256, 0, st>>>(src, dst, per_elem, mean, std, keep, seed);
  else
    noise_philox_kernel<false><<<grid, 256, 0, st>>>(src, dst, per_elem, mean, std, keep, seed);
  TIO_CHECK_LAUNCH();
  return 0;
}

extern "C" int tio_gamma(const float* src, float* dst, int B, int64_t per_elem, const float* gamma,
                         void* stream) {
  TIO_CHECK_ARG(src && dst && gamma, "tio_gamma: null pointer");
  TIO_CHECK_ARG(B > 0 && B <= 65535 && per_elem > 0, "tio_gamma: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = (per_elem % 4 == 0) && aligned16(src) && aligned16(dst);
  dim3 grid(ew_blocks(vec ? per_elem / 4 : per_elem), B);
  if (vec) gamma_kernel<4><<<grid, 256, 0, st>>>(src, dst, per_elem, gamma);
  else gamma_kernel<1><<<grid, 256, 0, st>>>(src, dst, per_elem, gamma);
  TIO_CHECK_LAUNCH();
  return 0;
}


// ---- tio_upload: table upload by an SM kernel (see include/tio_b200.h) ----------
namespace tio {
__global__ void upload_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, size_t bytes) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool vec = (((uintptr_t)src | (uintptr_t)dst) & 15) == 0;
  if (vec) {
    const size_t n16 = bytes >> 4;
    if (i < n16) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
    if (i == 0)
      for (size_t t = n16 << 4; t < bytes; ++t) dst[t] = src[t];
  } else {
    for (size_t t = i * 16; t < bytes && t < (i + 1) * 16; ++t) dst[t] = src[t];
  }
}
}  // namespace tio

extern "C" int tio_upload(const void* host_pinned, void* dst_device, size_t bytes, void* stream) {
  TIO_CHECK_ARG(host_pinned && dst_device, "tio_upload: null pointer");
  if (bytes == 0) return 0;
  const size_t items = (bytes + 15) / 16;
  const unsigned blocks = (unsigned)((items + 255) / 256);
  tio::upload_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((const uint8_t*)host_pinned,
                                                             (uint8_t*)dst_device, bytes);
  TIO_CHECK_LAUNCH();
  return 0;
}

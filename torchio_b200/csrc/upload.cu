// upload.cu — tio_upload: table upload by an SM kernel (see include/tio_b200.h).
#include "common.cuh"

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
  tio::launched();
  TIO_CHECK_LAUNCH();
  return 0;
}

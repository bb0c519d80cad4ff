// mt19937_layout.h — layout of the MT19937 jump-ahead table, shared by its builder
// (mt19937_jump.cpp) and the device replay (mt19937.cu).
//
// The stream is cut into segments of L = 2^kLog2L words.  The table holds the
// fine polynomials x^(r*L), r = 1 .. kS2-1, then the coarse ones x^(m*kS2*L),
// m = 1 .. kS1-1, so it reaches kS1 * kS2 * L = 2^31 stream words.  Each
// polynomial takes kStride uint16 entries (count, then set-bit positions).
#pragma once

#include <stdint.h>

namespace tio_mt {

constexpr uint32_t kMagic = 0x4d544a31u;  // "MTJ1"
constexpr int kLog2L = 21, kS2 = 16, kS1 = 64;
constexpr int kStride = 10496;  // >= 2 + max popcount observed (~10.1k), multiple of 64
constexpr int kPolys = (kS2 - 1) + (kS1 - 1);
constexpr int kHeaderBytes = 32;  // uint32 {magic, log2(L), S2, S1, n_polys, stride_u16, 0, 0}

}  // namespace tio_mt

// mt19937_jump.cpp — host side of K4a: jump-ahead tables for MT19937.
//
// The reference draws its noise with torch.randn on a CPU mt19937 generator
// (transforms/intensity/noise.py:166-178), one sequential stream per call.  To
// replay that stream on the GPU the stream is cut into segments of L = 2^21
// words (mt19937_layout.h) whose start states are obtained by jump-ahead (Haramoto, Matsumoto,
// Nishimura, Panneton, L'Ecuyer 2008): with F the one-word state transition and
// phi its characteristic polynomial, F^J = g_J(F), g_J = x^J mod phi.  This file
// computes phi (Berlekamp-Massey on 2*19937 output bits) and the polynomials
//   h_r = x^(r*L)       r = 1 .. S2-1      (fine level)
//   b_m = x^(m*L*S2)    m = 1 .. S1-1      (coarse level)
// as lists of set-bit positions.  The table depends on nothing but MT19937
// itself; the caller keeps it (the library holds no state).
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/tio_b200.h"
#include "mt19937_layout.h"

namespace {

constexpr int kDeg = 19937;
constexpr int kWords = (2 * kDeg + 63) / 64 + 1;  // room for products

struct Bits {
  std::vector<uint64_t> w;
  explicit Bits(int words = kWords) : w(words, 0) {}
  bool get(int i) const { return (w[i >> 6] >> (i & 63)) & 1u; }
  void flip(int i) { w[i >> 6] ^= (uint64_t)1 << (i & 63); }
  void set(int i) { w[i >> 6] |= (uint64_t)1 << (i & 63); }
};

// a ^= b << s   (bit shift), over `nw` words of b
static void xor_shifted(Bits& a, const Bits& b, int s, int nw) {
  const int ws = s >> 6, bs = s & 63;
  const int limit = (int)a.w.size();
  if (bs == 0) {
    for (int i = 0; i < nw && i + ws < limit; ++i) a.w[i + ws] ^= b.w[i];
  } else {
    for (int i = 0; i < nw; ++i) {
      const uint64_t v = b.w[i];
      if (!v) continue;
      if (i + ws < limit) a.w[i + ws] ^= v << bs;
      if (i + ws + 1 < limit) a.w[i + ws + 1] ^= v >> (64 - bs);
    }
  }
}

struct Mt {
  uint32_t s[624];
  int idx;
  void seed(uint32_t v) {
    s[0] = v;
    for (int j = 1; j < 624; ++j) s[j] = 1812433253u * (s[j - 1] ^ (s[j - 1] >> 30)) + (uint32_t)j;
    idx = 624;
  }
  uint32_t raw() {  // untempered next word x[624 + n]
    if (idx >= 624) {
      for (int k = 0; k < 624; ++k) {
        uint32_t y = (s[k] & 0x80000000u) | (s[(k + 1) % 624] & 0x7fffffffu);
        s[k] = s[(k + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
      }
      idx = 0;
    }
    return s[idx++];
  }
};

struct Field {
  Bits phi;  // characteristic polynomial, degree kDeg (bit kDeg set)
  std::vector<int> phi_terms;  // exponents < kDeg of the non-leading terms

  void reduce(Bits& a) const {  // a mod phi, in place; a has up to 2*kDeg bits
    for (int d = 2 * kDeg; d >= kDeg; --d) {
      if (!a.get(d)) continue;
      const int s = d - kDeg;
      a.flip(d);
      for (int e : phi_terms) a.flip(e + s);
    }
  }
  Bits mul(const Bits& a, const Bits& b) const {
    Bits r;
    const int nw = (kDeg + 63) / 64;
    for (int i = 0; i < kDeg; ++i)
      if (a.get(i)) xor_shifted(r, b, i, nw);
    reduce(r);
    return r;
  }
};

static bool build_field(Field& f) {
  // LSB of the raw word sequence: a linear functional of the state
  Mt g;
  g.seed(19650218u);
  std::vector<uint8_t> seq(2 * kDeg + 64);
  for (auto& v : seq) v = (uint8_t)(g.raw() & 1u);
  // Berlekamp-Massey over GF(2), word-packed: the discrepancy is the parity of
  // C AND (reversed sliding window of the sequence)
  const int n = (int)seq.size();
  const int W = (kDeg + 64) / 64 + 1;
  std::vector<uint64_t> c(W, 0), b(W, 0), t(W, 0), rev(W, 0);
  c[0] = 1;
  b[0] = 1;
  int L = 0, m = 1;
  for (int i = 0; i < n; ++i) {
    // rev holds s_i at bit 0, s_{i-1} at bit 1, ...
    for (int k = W - 1; k > 0; --k) rev[k] = (rev[k] << 1) | (rev[k - 1] >> 63);
    rev[0] = (rev[0] << 1) | seq[i];
    uint64_t acc = 0;
    for (int k = 0; k < W; ++k) acc ^= c[k] & rev[k];
    const int d = __builtin_popcountll(acc) & 1;
    if (d) {
      t = c;
      const int ws = m >> 6, bs = m & 63;
      for (int k = 0; k + ws < W; ++k) {
        c[k + ws] ^= b[k] << bs;
        if (bs && k + ws + 1 < W) c[k + ws + 1] ^= b[k] >> (64 - bs);
      }
      if (2 * L <= i) {
        L = i + 1 - L;
        b = t;
        m = 1;
      } else {
        ++m;
      }
    } else {
      ++m;
    }
  }
  if (L != kDeg) return false;
  // characteristic polynomial = reciprocal of the connection polynomial
  f.phi = Bits();
  f.phi_terms.clear();
  for (int j = 0; j <= kDeg; ++j)
    if ((c[j >> 6] >> (j & 63)) & 1u) {
      f.phi.set(kDeg - j);
      if (kDeg - j < kDeg) f.phi_terms.push_back(kDeg - j);
    }
  return f.phi.get(kDeg);
}

}  // namespace

// ---- table layout (mt19937_layout.h) ---------------------------------------------
//   uint32 header[8] = {magic, log2(L), S2, S1, n_polys, stride_u16, 0, 0}
//   per polynomial (n_polys = (S2-1) + (S1-1)), `stride_u16` uint16 entries:
//       [count_lo, count_hi, idx0, idx1, ...]   (set-bit positions, ascending)
//   fine polynomials h_1..h_{S2-1} first, then coarse b_1..b_{S1-1}.
using tio_mt::kLog2L;
using tio_mt::kMagic;
using tio_mt::kS1;
using tio_mt::kS2;
using tio_mt::kStride;

extern "C" size_t tio_mt19937_table_bytes(void) {
  return tio_mt::kHeaderBytes + (size_t)tio_mt::kPolys * kStride * sizeof(uint16_t);
}

extern "C" int tio_mt19937_build_table(void* blob, size_t bytes) {
  if (!blob || bytes < tio_mt19937_table_bytes()) return 1;
  Field f;
  if (!build_field(f)) return 2;
  uint32_t* header = (uint32_t*)blob;
  header[0] = kMagic; header[1] = kLog2L; header[2] = kS2; header[3] = kS1;
  header[4] = tio_mt::kPolys; header[5] = kStride; header[6] = header[7] = 0;
  uint16_t* out = (uint16_t*)((char*)blob + tio_mt::kHeaderBytes);
  auto emit = [&](const Bits& p, int slot) -> bool {
    uint16_t* dst = out + (size_t)slot * kStride;
    uint32_t count = 0;
    for (int i = 0; i < kDeg; ++i)
      if (p.get(i)) {
        if (2 + count >= (uint32_t)kStride) return false;
        dst[2 + count++] = (uint16_t)i;
      }
    dst[0] = (uint16_t)(count & 0xffffu);
    dst[1] = (uint16_t)(count >> 16);
    return true;
  };
  // x^(2^kLog2L) by repeated squaring of x
  Bits h1;
  h1.set(1);
  for (int i = 0; i < kLog2L; ++i) h1 = f.mul(h1, h1);
  Bits cur = h1;
  for (int r = 1; r < kS2; ++r) {
    if (!emit(cur, r - 1)) return 3;
    cur = f.mul(cur, h1);
  }
  const Bits b1 = cur;  // h1^S2 = x^(L*S2)
  cur = b1;
  for (int m = 1; m < kS1; ++m) {
    if (!emit(cur, (kS2 - 1) + (m - 1))) return 3;
    if (m + 1 < kS1) cur = f.mul(cur, b1);
  }
  return 0;
}

// Host application of one table polynomial to a 624-word window (test hook):
// out = g(F) * in, evaluated as XOR of shifted copies of the generated sequence.
extern "C" int tio_mt19937_apply_poly_host(const void* blob, int slot, const uint32_t* in,
                                           uint32_t* out) {
  const uint32_t* header = (const uint32_t*)blob;
  if (header[0] != kMagic || slot < 0 || slot >= (int)header[4]) return 1;
  const uint16_t* p = (const uint16_t*)((const char*)blob + tio_mt::kHeaderBytes) + (size_t)slot * header[5];
  const uint32_t count = p[0] | ((uint32_t)p[1] << 16);
  std::vector<uint32_t> seq(kDeg + 624 + 8);
  memcpy(seq.data(), in, 624 * 4);
  for (int k = 0; k + 624 < (int)seq.size(); ++k) {
    uint32_t y = (seq[k] & 0x80000000u) | (seq[k + 1] & 0x7fffffffu);
    seq[k + 624] = seq[k + 397] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
  }
  for (int j = 0; j < 624; ++j) out[j] = 0;
  for (uint32_t t = 0; t < count; ++t) {
    const uint32_t* s = seq.data() + p[2 + t];
    for (int j = 0; j < 624; ++j) out[j] ^= s[j];
  }
  return 0;
}

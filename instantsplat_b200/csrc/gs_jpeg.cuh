// Baseline JPEG arithmetic shared by the decoder kernels (gs_jpeg.cu) and the CPU suite (tests/host_jpeg.cpp, built
// by g++): the per-symbol Huffman step and its state, libjpeg-turbo's islow IDCT with its range-limit wrap, the fancy
// upsampling taps and the YCbCr->RGB fixed point.  Everything is integer arithmetic.  DESIGN.md 4.24.
#pragma once
#include <stdint.h>

#include "../../include/gsb200.h"

#if defined(__CUDACC__)
#define GSJ_HD __host__ __device__ __forceinline__
#else
#define GSJ_HD inline
#endif

namespace gsj {

// jpeg_natural_order: zigzag index -> natural (row-major) index.
#if defined(__CUDACC__)
__constant__ const uint8_t kNatural[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
    41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
    30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
#endif

GSJ_HD int natural(int k) {
#if defined(__CUDA_ARCH__)
  return kNatural[k];
#else
  static const uint8_t t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
  return t[k];
#endif
}

// Decoder state between two symbols: bit position in the interval's unstuffed bytes, block within the MCU (c) and
// zigzag index (k, 0 = the DC symbol is next).  Packed in 64 bits so that one load or store moves it whole:
// pos in bits 0..31, c in 32..39, k in 40..47, bit 63 = invalid (a decode from this start failed).
struct State {
  uint32_t pos;
  int c, k;
};
constexpr uint64_t kInvalid = 1ull << 63;
GSJ_HD uint64_t pack(State s) { return (uint64_t)s.pos | ((uint64_t)s.c << 32) | ((uint64_t)s.k << 40); }
GSJ_HD State unpack(uint64_t v) {
  State s;
  s.pos = (uint32_t)v;
  s.c = (int)((v >> 32) & 0xff);
  s.k = (int)((v >> 40) & 0xff);
  return s;
}

// Reads 32 bits starting at bit pos of the interval's bytes [0, nbytes); bytes past the end read as zero, as
// libjpeg's fill_bit_buffer zero-fills past a marker.
GSJ_HD uint32_t peek32(const uint8_t* p, uint32_t nbytes, uint32_t pos) {
  const uint32_t b = pos >> 3, sh = pos & 7;
  uint64_t v = 0;
  for (int i = 0; i < 5; ++i) v = (v << 8) | (b + i < nbytes ? p[b + i] : 0u);
  return (uint32_t)(v >> (8 - sh));
}

GSJ_HD int extend(int r, int s) { return r < (1 << (s - 1)) ? r - (1 << s) + 1 : r; }  // HUFF_EXTEND

enum StepResult { kSymbol = 0, kBlockEnd = 1, kBadCode = -1, kPastEnd = -2, kRunPast63 = -3 };

// One Huffman symbol of jdhuff.c's decode_mcu (baseline): s.k == 0 decodes the DC difference into *dc; else one AC
// run/size, writing a nonzero coefficient's natural index and value to *ci / *cv (ci = -1 when none).  Returns
// kBlockEnd when the symbol finished the block (s is then at the next block's DC), kSymbol otherwise, or an error:
// a code no table entry matches, bits needed past end_bits, or a run that takes k past 63 (libjpeg writes those to
// coefficient 63 through jpeg_natural_order's padding; such streams are handed back instead).
GSJ_HD int step(State& s, const GsbJpegHuff* dc_tbl, const GsbJpegHuff* ac_tbl, const uint8_t* p, uint32_t nbytes,
                uint32_t end_bits, int* dc, int* ci, int* cv) {
  const GsbJpegHuff* t = s.k == 0 ? dc_tbl : ac_tbl;
  const uint32_t w = peek32(p, nbytes, s.pos);
  int len, sym;
  const uint16_t look = t->look[w >> (32 - GSB_JPEG_LOOKAHEAD)];
  if (look) {
    len = look >> 8;
    sym = look & 0xff;
  } else {                                               // jpeg_huff_decode's slow path
    len = GSB_JPEG_LOOKAHEAD + 1;
    int32_t code = (int32_t)(w >> (32 - len));
    while (len <= 16 && code > t->maxcode[len]) {
      ++len;
      code = (int32_t)(w >> (32 - len));
    }
    if (len > 16) return kBadCode;
    sym = t->huffval[(code + t->valoffset[len]) & 0xff];
  }
  const int size = s.k == 0 ? sym : (sym & 15);
  const uint32_t used = (uint32_t)(len + size);
  if (s.pos + used > end_bits) return kPastEnd;
  int value = 0;
  if (size) value = extend((int)((w << len) >> (32 - size)), size);
  s.pos += used;
  *ci = -1;
  if (s.k == 0) {
    *dc = value;
    s.k = 1;
    return kSymbol;
  }
  const int run = sym >> 4;
  if (size) {
    s.k += run;
    if (s.k > 63) return kRunPast63;
    *ci = natural(s.k);
    *cv = value;
    s.k += 1;
  } else if (run == 15) {
    s.k += 16;
    if (s.k > 64) return kRunPast63;
  } else {
    s.k = 64;                                            // EOB
  }
  return s.k >= 64 ? kBlockEnd : kSymbol;
}

// The self-synchronising decode of one subsequence: from state st (packed) until the position reaches hi, in an
// interval ending at bit iend of p.  Returns the end state (kInvalid after an error) and the blocks started.
GSJ_HD uint64_t decode_span(uint64_t st, uint32_t hi, uint32_t iend, const uint8_t* p, const GsbJpegFile& F, int H,
                            int V, int32_t* count) {
  *count = 0;
  if (st & kInvalid) return st;
  State s = unpack(st);
  const int hv = H * V;
  int dc, ci, cv;
  while (s.pos < hi) {
    const int comp = s.c < hv ? 0 : s.c - hv + 1;
    if (s.k == 0) ++*count;
    const int r = step(s, &F.dc[comp], &F.ac[comp], p, iend >> 3, iend, &dc, &ci, &cv);
    if (r < 0) return kInvalid;
    if (r == kBlockEnd) {
      s.k = 0;
      s.c = s.c + 1 == hv + 2 ? 0 : s.c + 1;
    }
  }
  return pack(s);
}

// ---- jidctint.c jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2) ----
constexpr int kConstBits = 13, kPass1Bits = 2;
GSJ_HD int64_t descale(int64_t x, int n) { return (x + ((int64_t)1 << (n - 1))) >> n; }

// IDCT_range_limit(x & RANGE_MASK): the low 10 bits read as signed, plus CENTERJSAMPLE, clamped to 0..255.
GSJ_HD uint8_t range_limit_idct(int64_t x) {
  int v = (int)(x & 1023);
  v = v >= 512 ? v - 1024 : v;
  v += 128;
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// One pass of the 1-D islow transform, even part then odd part in jidctint.c's order, in 64 bits as its JLONG is
// on LP64 hosts (the odd part's sums pass 2^31 for large coefficients).  The 8 outputs before descaling go to o[].
GSJ_HD void idct_1d(int64_t i0, int64_t i1, int64_t i2, int64_t i3, int64_t i4, int64_t i5, int64_t i6, int64_t i7,
                    int64_t* o) {
  int64_t z1, z2, z3, z4, z5, tmp0, tmp1, tmp2, tmp3, tmp10, tmp11, tmp12, tmp13;
  z2 = i2;
  z3 = i6;
  z1 = (z2 + z3) * 4433;                                  // FIX_0_541196100
  tmp2 = z1 + z3 * (-15137);                              // FIX_1_847759065
  tmp3 = z1 + z2 * 6270;                                  // FIX_0_765366865
  tmp0 = (int64_t)((uint64_t)(i0 + i4) << kConstBits);
  tmp1 = (int64_t)((uint64_t)(i0 - i4) << kConstBits);
  tmp10 = tmp0 + tmp3;
  tmp13 = tmp0 - tmp3;
  tmp11 = tmp1 + tmp2;
  tmp12 = tmp1 - tmp2;
  tmp0 = i7;
  tmp1 = i5;
  tmp2 = i3;
  tmp3 = i1;
  z1 = tmp0 + tmp3;
  z2 = tmp1 + tmp2;
  z3 = tmp0 + tmp2;
  z4 = tmp1 + tmp3;
  z5 = (z3 + z4) * 9633;                                  // FIX_1_175875602
  tmp0 = tmp0 * 2446;                                     // FIX_0_298631336
  tmp1 = tmp1 * 16819;                                    // FIX_2_053119869
  tmp2 = tmp2 * 25172;                                    // FIX_3_072711026
  tmp3 = tmp3 * 12299;                                    // FIX_1_501321110
  z1 = z1 * (-7373);                                      // FIX_0_899976223
  z2 = z2 * (-20995);                                     // FIX_2_562915447
  z3 = z3 * (-16069);                                     // FIX_1_961570560
  z4 = z4 * (-3196);                                      // FIX_0_390180644
  z3 += z5;
  z4 += z5;
  tmp0 += z1 + z3;
  tmp1 += z2 + z4;
  tmp2 += z2 + z3;
  tmp3 += z1 + z4;
  o[0] = tmp10 + tmp3;
  o[7] = tmp10 - tmp3;
  o[1] = tmp11 + tmp2;
  o[6] = tmp11 - tmp2;
  o[2] = tmp12 + tmp1;
  o[5] = tmp12 - tmp1;
  o[3] = tmp13 + tmp0;
  o[4] = tmp13 - tmp0;
}

// Dequantised block (natural order, each entry already coef * quant and inside int16) -> 8x8 samples, out row r at
// out[r * stride].  The zero-AC shortcuts of jidctint.c give the same values as the full transform, so they are not
// taken.
GSJ_HD void idct_islow(const int32_t* in, uint8_t* out, int stride) {
  int32_t ws[64];
  int64_t o[8];
  for (int c = 0; c < 8; ++c) {
    idct_1d(in[c], in[8 + c], in[16 + c], in[24 + c], in[32 + c], in[40 + c], in[48 + c], in[56 + c], o);
    for (int r = 0; r < 8; ++r) ws[r * 8 + c] = (int32_t)descale(o[r], kConstBits - kPass1Bits);
  }
  for (int r = 0; r < 8; ++r) {
    const int32_t* w = ws + r * 8;
    idct_1d(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7], o);
    for (int c = 0; c < 8; ++c) out[r * stride + c] = range_limit_idct(descale(o[c], kConstBits + kPass1Bits + 3));
  }
}

// ---- jdsample.c: the chroma sample a full-resolution pixel takes ----
// Horizontal taps of h2v1_fancy_upsample / h2v2_fancy_upsample at output column x over a row of width w (> 2):
// the nearer sample i and the farther one j, with edge columns replicated.
GSJ_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// h2v1_fancy_upsample: row r of width w, output column x.
GSJ_HD uint8_t up_h2v1(const uint8_t* r, int w, int x) {
  const int i = x >> 1;
  if ((x & 1) == 0) return i == 0 ? r[0] : (uint8_t)((r[i] * 3 + r[i - 1] + 1) >> 2);
  return i == w - 1 ? r[i] : (uint8_t)((r[i] * 3 + r[i + 1] + 2) >> 2);
}

// h2v2_fancy_upsample: rows r0 (nearest) and r1 (next nearest, replicated at the plane's edges), output column x.
GSJ_HD uint8_t up_h2v2(const uint8_t* r0, const uint8_t* r1, int w, int x) {
  const int i = x >> 1;
  const int t = r0[i] * 3 + r1[i];
  if ((x & 1) == 0) {
    if (i == 0) return (uint8_t)((t * 4 + 8) >> 4);
    return (uint8_t)((t * 3 + r0[i - 1] * 3 + r1[i - 1] + 8) >> 4);
  }
  if (i == w - 1) return (uint8_t)((t * 4 + 7) >> 4);
  return (uint8_t)((t * 3 + r0[i + 1] * 3 + r1[i + 1] + 7) >> 4);
}

// h1v2_fancy_upsample: nearest and next nearest samples; odd = the lower output row of the pair.
GSJ_HD uint8_t up_h1v2(int a, int b, bool odd) { return (uint8_t)((a * 3 + b + (odd ? 2 : 1)) >> 2); }

// The chroma sample of full-resolution pixel (x, y) of a plane of w x h samples (stride ld) at luma sampling (H, V):
// jdsample.c's choice of method (fancy when the downsampled width is > 2 for 2h, box otherwise; fancy 1h2v), with
// jdmainct.c's context rows: the first row above the top, the last real row below the bottom.
GSJ_HD uint8_t chroma(const uint8_t* pl, int ld, int w, int h, int H, int V, int x, int y) {
  if (H == 1 && V == 1) return pl[y * ld + x];
  if (H == 2 && V == 1) return w > 2 ? up_h2v1(pl + y * ld, w, x) : pl[y * ld + (x >> 1)];
  const int i = y >> 1;
  const bool odd = y & 1;
  const int j = clampi(odd ? i + 1 : i - 1, 0, h - 1);
  if (H == 1) return up_h1v2(pl[i * ld + x], pl[j * ld + x], odd);
  if (w <= 2) return pl[i * ld + (x >> 1)];
  return up_h2v2(pl + i * ld, pl + j * ld, w, x);
}

// jdcolor.c ycc_rgb_convert with build_ycc_rgb_table's entries (SCALEBITS 16), then range_limit's clamp.
GSJ_HD uint8_t clamp255(int v) { return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v)); }
GSJ_HD void ycc_to_rgb(int y, int cb, int cr, uint8_t* rgb) {
  const int32_t xb = cb - 128, xr = cr - 128;
  const int32_t half = 1 << 15;
  rgb[0] = clamp255(y + ((91881 * xr + half) >> 16));
  rgb[1] = clamp255(y + ((-22554 * xb + half + -46802 * xr) >> 16));
  rgb[2] = clamp255(y + ((116130 * xb + half) >> 16));
}

}  // namespace gsj

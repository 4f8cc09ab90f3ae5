// The JPEG decoder's shared arithmetic (instantsplat_b200/csrc/gs_jpeg.cuh) built for the host by g++, for the CPU
// suite (tests/test_jpeg_cpu.py): a sequential Huffman decode, the subsequence synchronisation the kernels run,
// serially, and the per-block and per-pixel stages.  Input: one file's unstuffed entropy bytes and the first bit of
// each restart interval (ibits[0..n_int], the last entry the end), as tests/_jpeg.py splits them.
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../instantsplat_b200/csrc/gs_jpeg.cuh"

namespace {

struct Geo {
  int mcus_x, mcus_y, bpm, ri, H, V;
  int bw[3], bh[3];
  int64_t cblock[3], blocks;
};

Geo geo(const GsbJpegFile* f) {
  Geo g;
  g.H = f->h;
  g.V = f->v;
  g.mcus_x = (f->width + 8 * f->h - 1) / (8 * f->h);
  g.mcus_y = (f->height + 8 * f->v - 1) / (8 * f->v);
  g.bpm = f->h * f->v + 2;
  const int64_t mcus = (int64_t)g.mcus_x * g.mcus_y;
  g.ri = f->restart_interval > 0 ? f->restart_interval : (int)mcus;
  int64_t cb = 0;
  for (int c = 0; c < 3; ++c) {
    g.bw[c] = g.mcus_x * (c == 0 ? f->h : 1);
    g.bh[c] = g.mcus_y * (c == 0 ? f->v : 1);
    g.cblock[c] = cb;
    cb += (int64_t)g.bw[c] * g.bh[c];
  }
  g.blocks = cb;
  return g;
}

// The raster block (component-major) of block c of MCU mcu.
int64_t raster(const Geo& g, int64_t mcu, int c, int* comp) {
  const int hv = g.H * g.V;
  const int cp = c < hv ? 0 : c - hv + 1, j = cp == 0 ? c : 0, hc = cp == 0 ? g.H : 1, vc = cp == 0 ? g.V : 1;
  const int64_t mx = mcu % g.mcus_x, my = mcu / g.mcus_x;
  *comp = cp;
  return g.cblock[cp] + (my * vc + j / hc) * g.bw[cp] + mx * hc + j % hc;
}

int error_bit(int r) {
  return r == gsj::kBadCode ? GSB_JPEG_BAD_CODE : (r == gsj::kPastEnd ? GSB_JPEG_PAST_END : GSB_JPEG_RUN_PAST_63);
}

int64_t expected_blocks(const Geo& g, int i) {
  const int64_t mcus = (int64_t)g.mcus_x * g.mcus_y, mcu0 = (int64_t)i * g.ri;
  return (mcus - mcu0 < g.ri ? mcus - mcu0 : g.ri) * g.bpm;
}

}  // namespace

extern "C" {

int64_t hj_blocks(const GsbJpegFile* f) { return geo(f).blocks; }

// Sequential decode (jdhuff.c's order): coef [blocks, 64] raster blocks, natural order, DC already predicted (the
// int32 sum stored as int16).  Returns GSB_JPEG_* bits (0: decoded exactly).
int hj_decode_seq(const GsbJpegFile* f, const uint8_t* bytes, const uint32_t* ibits, int n_int, int16_t* coef) {
  const Geo g = geo(f);
  memset(coef, 0, sizeof(int16_t) * 64 * g.blocks);
  int status = 0;
  for (int i = 0; i < n_int; ++i) {
    gsj::State s{ibits[i], 0, 0};
    const uint32_t iend = ibits[i + 1];
    int64_t pred[3] = {0, 0, 0};
    const int64_t E = expected_blocks(g, i);
    for (int64_t b = 0; b < E; ++b) {
      int comp;
      const int64_t rb = raster(g, (int64_t)i * g.ri + b / g.bpm, (int)(b % g.bpm), &comp);
      int dc = 0, ci, cv, r;
      do {
        const bool was_dc = s.k == 0;
        r = gsj::step(s, &f->dc[comp], &f->ac[comp], bytes, iend >> 3, iend, &dc, &ci, &cv);
        if (r < 0) return status | error_bit(r);
        if (was_dc) {
          pred[comp] += dc;
          if (pred[comp] < INT32_MIN || pred[comp] > INT32_MAX) status |= GSB_JPEG_COEF_RANGE;
          coef[rb * 64] = (int16_t)(int32_t)pred[comp];
        } else if (ci >= 0) {
          coef[rb * 64 + ci] = (int16_t)cv;
        }
      } while (r != gsj::kBlockEnd);
      s.k = 0;
      s.c = s.c + 1 == g.bpm ? 0 : s.c + 1;
    }
    if (iend - s.pos >= 8) status |= GSB_JPEG_TRAILING;
  }
  return status;
}

// The kernels' algorithm run serially: per interval, subsequences of S bits decoded from guessed states and
// re-decoded from their predecessors' end states in rounds until none changes, the blocks each starts scanned into
// offsets, and a second pass writing from the synchronised states.  Same output as hj_decode_seq; *rounds: the
// rounds after the first that changed a state (the most over the intervals).
int hj_decode_sync(const GsbJpegFile* f, const uint8_t* bytes, const uint32_t* ibits, int n_int, int S,
                   int16_t* coef, int* rounds) {
  const Geo g = geo(f);
  memset(coef, 0, sizeof(int16_t) * 64 * g.blocks);
  int status = 0;
  *rounds = 0;
  std::vector<int64_t> dcd(g.blocks, 0);
  for (int i = 0; i < n_int; ++i) {
    const uint32_t istart = ibits[i], iend = ibits[i + 1] > istart ? ibits[i + 1] : istart;
    const int64_t nseq_l = ((int64_t)(iend - istart) + S - 1) / S;
    const int nseq = nseq_l > 0 ? (int)nseq_l : 1;
    std::vector<uint64_t> start(nseq), end(nseq);
    std::vector<int32_t> count(nseq + 1, 0);
    auto hi_of = [&](int t) {
      const uint32_t lo = istart + (uint32_t)t * S;
      return lo + (uint32_t)S < iend ? lo + (uint32_t)S : iend;
    };
    auto guess = [&](int t) { return gsj::pack(gsj::State{t == 0 ? istart : istart + (uint32_t)t * S, 0, 0}); };
    for (int t = 0; t < nseq; ++t) {
      start[t] = guess(t);
      end[t] = gsj::decode_span(start[t], hi_of(t), iend, bytes, *f, g.H, g.V, &count[t]);
    }
    for (int round = 1;; ++round) {
      bool changed = false;
      for (int t = 1; t < nseq; ++t) {
        // the predecessor's end, or this subsequence's own guess while the predecessor's decode fails
        const uint64_t want = (end[t - 1] & gsj::kInvalid) ? guess(t) : end[t - 1];
        if (want != start[t]) {
          start[t] = want;
          end[t] = gsj::decode_span(start[t], hi_of(t), iend, bytes, *f, g.H, g.V, &count[t]);
          changed = true;
        }
      }
      if (!changed) break;
      if (round > *rounds) *rounds = round;
    }
    int64_t acc = 0;
    for (int t = 0; t <= nseq; ++t) {
      const int32_t c = count[t];
      count[t] = (int32_t)acc;
      acc += c;
    }
    const int64_t E = expected_blocks(g, i);
    bool done = false;
    for (int t = 0; t < nseq; ++t) {
      if (start[t] & gsj::kInvalid) continue;
      gsj::State s = gsj::unpack(start[t]);
      int64_t blk = (int64_t)count[t] - 1;
      int dc, ci, cv;
      while (s.pos < hi_of(t)) {
        if (s.k == 0) {
          ++blk;
          if (blk >= E) break;
          if (s.c != (int)(blk % g.bpm)) { status |= GSB_JPEG_UNSYNCED; break; }
        }
        if (blk < 0) { status |= GSB_JPEG_UNSYNCED; break; }
        int comp;
        const int64_t mcu = (int64_t)i * g.ri + blk / g.bpm;
        const int64_t rb = raster(g, mcu, s.c, &comp);
        const bool was_dc = s.k == 0;
        const int r = gsj::step(s, &f->dc[comp], &f->ac[comp], bytes, iend >> 3, iend, &dc, &ci, &cv);
        if (r < 0) {
          status |= error_bit(r);
          break;
        }
        if (was_dc) dcd[rb] = dc;
        else if (ci >= 0) coef[rb * 64 + ci] = (int16_t)cv;
        if (r == gsj::kBlockEnd) {
          s.k = 0;
          s.c = s.c + 1 == g.bpm ? 0 : s.c + 1;
          if (blk == E - 1) {
            done = true;
            if (iend - s.pos >= 8) status |= GSB_JPEG_TRAILING;
            break;
          }
        }
      }
    }
    if (!done) status |= GSB_JPEG_MCUS_LEFT;
    // DC prediction, per component, in decode order
    int64_t pred[3] = {0, 0, 0};
    for (int64_t b = 0; b < E; ++b) {
      int comp;
      const int64_t rb = raster(g, (int64_t)i * g.ri + b / g.bpm, (int)(b % g.bpm), &comp);
      pred[comp] += dcd[rb];
      if (pred[comp] < INT32_MIN || pred[comp] > INT32_MAX) status |= GSB_JPEG_COEF_RANGE;
      coef[rb * 64] = (int16_t)(int32_t)pred[comp];
    }
  }
  return status;
}

// Dequantisation, the islow IDCT, upsampling and colour conversion of raster coefficient blocks into rgb [H, W, 3].
int hj_pixels(const GsbJpegFile* f, const int16_t* coef, uint8_t* rgb) {
  const Geo g = geo(f);
  int status = 0;
  std::vector<std::vector<uint8_t>> planes(3);
  for (int c = 0; c < 3; ++c) {
    const int ld = g.bw[c] * 8;
    planes[c].assign((size_t)ld * g.bh[c] * 8, 0);
    for (int by = 0; by < g.bh[c]; ++by)
      for (int bx = 0; bx < g.bw[c]; ++bx) {
        const int16_t* cb = coef + (g.cblock[c] + (int64_t)by * g.bw[c] + bx) * 64;
        int32_t in[64];
        for (int k = 0; k < 64; ++k) {
          in[k] = (int32_t)cb[k] * (int32_t)f->quant[c][k];
          if (in[k] < -32768 || in[k] > 32767) status |= GSB_JPEG_COEF_RANGE;
        }
        gsj::idct_islow(in, planes[c].data() + (size_t)by * 8 * ld + bx * 8, ld);
      }
  }
  const int ldy = g.bw[0] * 8, ldc = g.bw[1] * 8;
  const int cw = (f->width + g.H - 1) / g.H, ch = (f->height + g.V - 1) / g.V;
  for (int y = 0; y < f->height; ++y)
    for (int x = 0; x < f->width; ++x) {
      const int Y = planes[0][(size_t)y * ldy + x];
      const int cb = gsj::chroma(planes[1].data(), ldc, cw, ch, g.H, g.V, x, y);
      const int cr = gsj::chroma(planes[2].data(), ldc, cw, ch, g.H, g.V, x, y);
      gsj::ycc_to_rgb(Y, cb, cr, rgb + ((size_t)y * f->width + x) * 3);
    }
  return status;
}

}  // extern "C"

// PNG encoding of 8-bit RGB frames on the GPU (C ABI in include/gsb200.h), in its own translation unit so that the
// training, tracking and metrics kernels are compiled exactly as before.  DESIGN.md 4.19.
//
// An 8-bit RGB PNG is a zlib stream of filtered scanlines.  Three kernels build it:
//
//   k_png_filter   one CTA per (frame, row).  Pillow's ZipEncode adaptive filter: of None (0), Sub (1), Up (2) and
//                  Paeth (4) (never Average), the type whose filtered bytes have the smallest sum of |int8| wins, the
//                  first in that order on a tie; row 0 filters against a zero row, 3 bytes per pixel.  The four costs
//                  are integer sums, so the choice is exact.  Writes the frame's filtered stream, H (3W + 1) bytes.
//   k_png_deflate  one CTA per (frame, 32 KiB segment of the filtered stream).  The segment and the 32 KiB before it
//                  are staged in shared memory; LZ77 matches (3..256 bytes, distance <= 32768) are found among distance 1,
//                  distance 3 (the same channel one pixel left), the row above and up to 64 links of a 3-byte hash
//                  chain built chunk by chunk (links within a warp's 32 positions or to before the chunk) -- and
//                  parsed lazily within fixed 256-byte sub-blocks, one thread each.  One dynamic Huffman block
//                  (codes length-limited to 15 bits, 7 for the code-length code, at least two codes per alphabet so
//                  every code is complete) or a stored block, whichever is shorter, then an empty stored block (a sync
//                  flush), so the segment ends byte-aligned with BFINAL 0.  Also the segment's Adler-32 partial sums.
//   k_png_pack     one CTA per (frame, segment): the segment's offset is the sum of the sizes before it; the CTAs of
//                  the first and last segment add the zlib header, the final empty fixed-Huffman block (03 00), the
//                  big-endian Adler-32 combined from the partials, and the stream's length.
//
// Every sum is an integer sum and the only atomics are shared-memory histogram counts, maxima and bit ORs, whose
// results do not depend on their order: a frame's bytes are a function of its pixels alone, whatever the batch, the
// frame's place in it, the stream or the timing.
#include <cuda_runtime.h>
#include <stdio.h>

#include "../../include/gsb200.h"

void gsb_set_error(const char* s);
void gsb_count_launch(int n);

namespace {

constexpr int kSeg = 32768;             // filtered bytes per segment
constexpr int kHist = 32768;            // deflate's window: how far back a match may reach
constexpr int kSub = 256;               // bytes per parse sub-block (one thread); a match never crosses one
constexpr int kSubs = kSeg / kSub;      // parse threads
constexpr int kThreads = 256;
constexpr int kHashBits = 12;
constexpr int kChain = 64;          // hash-chain candidates tried per position
constexpr int kLazy = 64;           // matches at least this long are taken without looking one position ahead
constexpr int kSegSlot = kSeg + 16;     // scratch bytes per compressed segment (a stored one is n + 10)
constexpr int kFilterThreads = 128;
constexpr int kPackThreads = 256;
constexpr uint32_t kAdlerMod = 65521;
constexpr size_t kDeflateSmem = (size_t)(kHist + kSeg) + (size_t)kSeg * 4 + ((size_t)4 << kHashBits);

struct SegInfo {
  uint32_t bytes, a, b, pad;            // compressed size; Adler-32 sums of the segment from (0, 0)
};

int check(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return GSB_OK;
  char buf[256];
  snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
  gsb_set_error(buf);
  return GSB_ERR_CUDA;
}

struct Geometry {
  int64_t N;        // filtered bytes per frame
  int64_t nseg;
  size_t filt_stride, bound;
};

bool geometry(int32_t H, int32_t W, Geometry* g) {
  if (H <= 0 || W <= 0 || W > (INT32_MAX - 1) / 3) return false;
  const int64_t N = (int64_t)H * (3 * (int64_t)W + 1);
  if (N > ((int64_t)1 << 31) - 4096) return false;
  g->N = N;
  g->nseg = (N + kSeg - 1) / kSeg;
  g->filt_stride = (size_t)((N + 15) / 16 * 16);
  g->bound = (size_t)(2 + N + 10 * g->nseg + 2 + 4);
  return true;
}

// ---- filter -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t absi8(int d) {
  const uint32_t v = (uint32_t)d & 255u;
  return v < 128u ? v : 256u - v;
}

__device__ __forceinline__ int paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__global__ void __launch_bounds__(kFilterThreads) k_png_filter(int H, int W, const uint8_t* __restrict__ rgb,
                                                               uint8_t* __restrict__ filt, size_t filt_stride) {
  constexpr int kWarps = kFilterThreads / 32;
  __shared__ uint32_t part[4][kWarps];
  __shared__ int kind;
  const int y = blockIdx.x, v = blockIdx.y, RB = 3 * W;
  const uint8_t* cur = rgb + ((size_t)v * H + y) * RB;
  const uint8_t* up = y > 0 ? cur - RB : nullptr;
  uint32_t c0 = 0, c1 = 0, c2 = 0, c4 = 0;
  for (int i = threadIdx.x; i < RB; i += kFilterThreads) {
    const int x = cur[i], a = i >= 3 ? cur[i - 3] : 0, b = up ? up[i] : 0, c = (up && i >= 3) ? up[i - 3] : 0;
    c0 += absi8(x);
    c1 += absi8(x - a);
    c2 += absi8(x - b);
    c4 += absi8(x - paeth(a, b, c));
  }
  for (int o = 16; o > 0; o >>= 1) {
    c0 += __shfl_xor_sync(0xffffffffu, c0, o);
    c1 += __shfl_xor_sync(0xffffffffu, c1, o);
    c2 += __shfl_xor_sync(0xffffffffu, c2, o);
    c4 += __shfl_xor_sync(0xffffffffu, c4, o);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    part[0][warp] = c0;
    part[1][warp] = c1;
    part[2][warp] = c2;
    part[3][warp] = c4;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t s[4] = {0, 0, 0, 0};
    for (int k = 0; k < 4; ++k)
      for (int w = 0; w < kWarps; ++w) s[k] += part[k][w];
    int best = 0;
    for (int k = 1; k < 4; ++k)
      if (s[k] < s[best]) best = k;
    kind = best == 3 ? 4 : best;
  }
  __syncthreads();
  const int k = kind;
  uint8_t* out = filt + (size_t)v * filt_stride + (size_t)y * (RB + 1);
  if (threadIdx.x == 0) out[0] = (uint8_t)k;
  for (int i = threadIdx.x; i < RB; i += kFilterThreads) {
    const int x = cur[i], a = i >= 3 ? cur[i - 3] : 0, b = up ? up[i] : 0, c = (up && i >= 3) ? up[i - 3] : 0;
    const int p = k == 0 ? 0 : k == 1 ? a : k == 2 ? b : paeth(a, b, c);
    out[1 + i] = (uint8_t)(x - p);
  }
}

// ---- deflate ----------------------------------------------------------------------------------------------------
// Length 3..258 -> symbol 257..285 and its extra bits; distance 1..32768 -> symbol 0..29 and its extra bits.
__device__ __forceinline__ void len_code(int len, int* sym, int* nextra, int* extra) {
  const int l = len - 3;
  if (l < 8) { *sym = 257 + l; *nextra = 0; *extra = 0; return; }
  if (l == 255) { *sym = 285; *nextra = 0; *extra = 0; return; }
  const int e = 29 - __clz(l), m = (l >> e) & 3;
  *sym = 261 + 4 * e + m;
  *nextra = e;
  *extra = l - ((4 + m) << e);
}

__device__ __forceinline__ void dist_code(int dist, int* sym, int* nextra, int* extra) {
  const int d = dist - 1;
  if (d < 4) { *sym = d; *nextra = 0; *extra = 0; return; }
  const int e = 30 - __clz(d), m = (d >> e) & 1;
  *sym = 2 * e + 2 + m;
  *nextra = e;
  *extra = d - ((2 + m) << e);
}

__device__ __forceinline__ int lit_extra_bits(int s) { return (s < 265 || s == 285) ? 0 : (s - 261) >> 2; }
__device__ __forceinline__ int dist_extra_bits(int s) { return s < 4 ? 0 : (s - 2) >> 1; }

// LSB-first bit writer into a zeroed shared buffer of 32-bit words; the words it shares with other writers are ORed.
struct BitWriter {
  uint32_t* words;
  int w, nbits;
  uint64_t acc;
  __device__ BitWriter(uint32_t* out, uint32_t pos) : words(out), w((int)(pos >> 5)), nbits((int)(pos & 31)), acc(0) {}
  __device__ __forceinline__ void put(uint32_t val, int n) {
    acc |= (uint64_t)val << nbits;
    nbits += n;
    if (nbits >= 32) {
      atomicOr(&words[w++], (uint32_t)acc);
      acc >>= 32;
      nbits -= 32;
    }
  }
  __device__ __forceinline__ void flush() {
    if (nbits > 0) atomicOr(&words[w], (uint32_t)acc);
  }
};

// Huffman code lengths of nsym symbols, at most `limit` bits, by one warp.  Symbols with a zero count get no code;
// when fewer than two counts are non-zero the first zero-count symbols are given a count of one, as zlib does, so the
// code is complete.  Leaves are ranked by (count, symbol), merged by the two-queue method (a leaf before an internal
// node of equal weight), and lengths over the limit are folded back with the Kraft-sum correction; the lengths are
// then handed out from the most frequent symbol.  scratch: 8 * nsym + 16 words.
__device__ void huff_lengths(const uint32_t* count, int nsym, int limit, uint8_t* len, uint32_t* scratch) {
  const int lane = threadIdx.x & 31;
  uint32_t* f = scratch;                            // [nsym] counts used for the code
  uint32_t* sorted = f + nsym;                      // [nsym]
  uint32_t* wt = sorted + nsym;                     // [2 nsym] node weights
  uint32_t* par = wt + 2 * nsym;                    // [2 nsym]
  uint32_t* dep = par + 2 * nsym;                   // [2 nsym]
  uint32_t* num = dep + 2 * nsym;                   // [16]
  for (int s = lane; s < nsym; s += 32) { f[s] = count[s]; len[s] = 0; }
  __syncwarp();
  if (lane == 0) {
    int nz = 0;
    for (int s = 0; s < nsym; ++s) nz += f[s] != 0;
    for (int s = 0; s < nsym && nz < 2; ++s)
      if (f[s] == 0) { f[s] = 1; ++nz; }
  }
  __syncwarp();
  for (int s = lane; s < nsym; s += 32) {
    if (f[s] == 0) continue;
    int r = 0;
    for (int j = 0; j < nsym; ++j) r += f[j] != 0 && (f[j] < f[s] || (f[j] == f[s] && j < s));
    sorted[r] = (uint32_t)s;
  }
  __syncwarp();
  if (lane == 0) {
    int m = 0;
    for (int s = 0; s < nsym; ++s) m += f[s] != 0;
    for (int k = 0; k < m; ++k) wt[k] = f[sorted[k]];
    int li = 0, ii = m, ni = m;                     // next leaf, next internal node, next free node
    for (int k = 0; k < m - 1; ++k) {
      int pick[2];
      for (int t = 0; t < 2; ++t) {
        if (li < m && (ii >= ni || wt[li] <= wt[ii])) pick[t] = li++;
        else pick[t] = ii++;
      }
      wt[ni] = wt[pick[0]] + wt[pick[1]];
      par[pick[0]] = par[pick[1]] = (uint32_t)ni;
      ++ni;
    }
    dep[ni - 1] = 0;
    for (int x = ni - 2; x >= 0; --x) dep[x] = dep[par[x]] + 1;
    for (int i = 0; i < 16; ++i) num[i] = 0;
    for (int k = 0; k < m; ++k) num[min((int)dep[k], limit)]++;
    uint32_t total = 0;
    for (int i = 1; i <= limit; ++i) total += num[i] << (limit - i);
    while (total != (1u << limit)) {
      num[limit]--;
      for (int i = limit - 1; i > 0; --i)
        if (num[i]) { num[i]--; num[i + 1] += 2; break; }
      total--;
    }
    int k = m - 1;
    for (int i = 1; i <= limit; ++i)
      for (uint32_t j = 0; j < num[i]; ++j) len[sorted[k--]] = (uint8_t)i;
  }
  __syncwarp();
}

// Canonical codes (RFC 1951 3.2.2), bit-reversed for LSB-first output.  tmp: 32 words of shared scratch.
__device__ void huff_codes(const uint8_t* len, int nsym, uint16_t* code, uint32_t* tmp) {
  uint32_t* bl = tmp;
  uint32_t* next = tmp + 16;
  for (int b = 0; b < 16; ++b) bl[b] = 0;
  for (int s = 0; s < nsym; ++s) bl[len[s]]++;
  bl[0] = 0;
  uint32_t c = 0;
  for (int b = 1; b < 16; ++b) { c = (c + bl[b - 1]) << 1; next[b] = c; }
  for (int s = 0; s < nsym; ++s)
    if (len[s]) code[s] = (uint16_t)(__brev(next[len[s]]++) >> (32 - len[s]));
}

// The order in which the code-length code's lengths are sent (RFC 1951 3.2.7).
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ uint32_t hash3(const uint8_t* p) {
  const uint32_t x = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
  return (x * 2654435761u) >> (32 - kHashBits);
}

__device__ __forceinline__ int match_len(const uint8_t* win, int p, int r, int maxlen) {
  int l = 0;
  while (l < maxlen && win[p + l] == win[r + l]) ++l;
  return l;
}

template <typename T>
__device__ __forceinline__ T block_sum(T x, T* red) {
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  T s = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
  return s;
}

__global__ void __launch_bounds__(kThreads, 1) k_png_deflate(int64_t N, int stride, const uint8_t* __restrict__ filt,
                                                             size_t filt_stride, uint8_t* __restrict__ segs,
                                                             SegInfo* __restrict__ info, int nseg) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* win = smem;                                                     // history + segment; later the output
  uint16_t* slot = reinterpret_cast<uint16_t*>(smem + kHist + kSeg);       // per position: hash-chain link
  uint16_t* tok = slot + kSeg;                                             // each sub-block's tokens
  uint32_t* head = reinterpret_cast<uint32_t*>(tok + kSeg);                // hash heads, then Huffman scratch
  __shared__ uint32_t f_lit[288], f_dist[32], f_cl[19];
  __shared__ uint8_t l_lit[288], l_dist[32], l_cl[19];
  __shared__ uint16_t c_lit[288], c_dist[32], c_cl[19];
  __shared__ uint16_t items[320];                   // code-length code: symbol | extra << 8
  __shared__ uint32_t tok_bits[kSubs + 1];
  __shared__ uint16_t ntok[kSubs];
  __shared__ uint64_t red[kThreads / 32];
  __shared__ int n_items, hclen, hlit, hdist;
  __shared__ uint32_t hdr_bits;

  const int tid = threadIdx.x, s = blockIdx.x, v = blockIdx.y;
  const uint8_t* src = filt + (size_t)v * filt_stride;
  const int64_t seg0 = (int64_t)s * kSeg;
  const int n = (int)min((int64_t)kSeg, N - seg0);
  const int hist = s > 0 ? kHist : 0;
  const int wn = hist + n;
  const uint8_t* wsrc = src + seg0 - hist;

  // stage the window (16-byte aligned: filt_stride and seg0 - hist are multiples of 16)
  for (int i = tid; i < wn / 16; i += kThreads)
    reinterpret_cast<uint4*>(win)[i] = reinterpret_cast<const uint4*>(wsrc)[i];
  for (int i = wn / 16 * 16 + tid; i < wn; i += kThreads) win[i] = wsrc[i];
  for (int i = tid; i < (1 << kHashBits); i += kThreads) head[i] = 0;
  for (int i = tid; i < 288; i += kThreads) f_lit[i] = 0;
  if (tid < 32) f_dist[tid] = 0;
  __syncthreads();
  if (tid == 0) f_lit[256] = 1;                     // end of block

  // Adler-32 of the segment from (0, 0): a = sum b_j, b = sum (n - j) b_j = n a - sum j b_j
  uint64_t A = 0, J = 0;
  for (int j = tid; j < n; j += kThreads) {
    const uint32_t b = win[hist + j];
    A += b;
    J += (uint64_t)j * b;
  }
  A = block_sum(A, red);
  J = block_sum(J, red);
  const uint32_t adler_a = (uint32_t)(A % kAdlerMod), adler_b = (uint32_t)(((uint64_t)n * A - J) % kAdlerMod);

  // hash chains: slot[q] is the distance from segment position q back to the last earlier position with the same
  // 3-byte hash in its warp's 32 positions or, when there is none, before its 256-position chunk (0: none).  The heads
  // hold position + 1 of the last occurrence as a maximum, so the insertion order does not matter; the history's
  // positions have heads but no links.
  for (int p = tid; p < hist; p += kThreads)
    if (p + 2 < wn) atomicMax(&head[hash3(win + p)], (uint32_t)(p + 1));
  __syncthreads();
  const int lane = tid & 31;
  for (int c = 0; c < n; c += kThreads) {
    const int q = c + tid, p = hist + q;
    const bool hashed = q + 2 < n;
    const uint32_t h = hashed ? hash3(win + p) : 0u;
    const uint32_t same = __match_any_sync(0xffffffffu, hashed ? h : (1u << 16) + lane) & ((1u << lane) - 1u);
    if (q < n) {
      uint32_t d = 0;
      if (hashed && same) {
        d = (uint32_t)(lane - (31 - __clz(same)));
      } else if (hashed) {
        const uint32_t last = head[h];
        if (last != 0 && (uint32_t)p - (last - 1) <= (uint32_t)kHist) d = (uint32_t)p - (last - 1);
      }
      slot[q] = (uint16_t)(d & 0xffff);             // 32768 wraps to 0x8000; decoded below
    }
    __syncthreads();
    if (hashed) atomicMax(&head[h], (uint32_t)(p + 1));
    __syncthreads();
  }

  // parse of each sub-block with one step of lazy matching (a match shorter than kLazy is deferred when the next
  // position starts a longer one).  Candidates: distances 1, 3 and the row above, then up to kChain links of the
  // position's hash chain.  Tokens go to the sub-block's own range of tok: a literal takes one slot for the one
  // position it covers, a match two for at least three.
  if (tid < kSubs) {
    const int beg = tid * kSub, end = min(n, beg + kSub);
    auto find = [&](int q, int* bd) {
      const int p = hist + q, maxlen = min(258, end - q);
      int best = 0;
      *bd = 0;
      if (maxlen < 3) return 0;
      const int fixed[3] = {1, 3, stride};
      for (int k = 0; k < 3 && best < maxlen; ++k) {
        const int d = fixed[k];
        if (d > p || d > kHist) continue;
        const int l = match_len(win, p, p - d, maxlen);
        if (l > best) { best = l; *bd = d; }
      }
      uint32_t link = slot[q];
      for (int k = 0, r = p; k < kChain && link != 0 && best < maxlen; ++k) {
        r -= link == 0x8000u ? kHist : (int)link;
        if (p - r > kHist) break;
        if (best == 0 || win[r + best] == win[p + best]) {      // else it cannot be longer
          const int l = match_len(win, p, r, maxlen);
          if (l > best) { best = l; *bd = p - r; }
        }
        if (r < hist) break;
        link = slot[r - hist];
      }
      return best;
    };
    int w = beg, next = -1, next_d = 0;
    for (int q = beg; q < end;) {
      const int p = hist + q;
      int bd, best;
      if (next >= 0) { best = next; bd = next_d; next = -1; }
      else best = find(q, &bd);
      if (best >= 3 && best < kLazy && q + 1 < end) {
        int d2;
        const int b2 = find(q + 1, &d2);
        if (b2 > best) { next = b2; next_d = d2; best = 0; }
      }
      if (best >= 3) {
        int sym, ne, ex;
        len_code(best, &sym, &ne, &ex);
        atomicAdd(&f_lit[sym], 1u);
        dist_code(bd, &sym, &ne, &ex);
        atomicAdd(&f_dist[sym], 1u);
        tok[w] = (uint16_t)best;
        tok[w + 1] = (uint16_t)(bd - 1);
        w += 2;
        q += best;
      } else {
        atomicAdd(&f_lit[win[p]], 1u);
        tok[w++] = (uint16_t)(0x8000u | win[p]);
        ++q;
      }
    }
    ntok[tid] = (uint16_t)(w - beg);
  }
  __syncthreads();

  // code lengths: literal/length by warp 0, distance by warp 1 (scratch in the hash heads)
  const int warp = tid >> 5;
  if (warp == 0) huff_lengths(f_lit, 286, 15, l_lit, head);
  if (warp == 1) huff_lengths(f_dist, 30, 15, l_dist, head + 2304);
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      huff_codes(l_lit, 286, c_lit, head + 2560);
      huff_codes(l_dist, 30, c_dist, head + 2560);
      int hl = 286, hd = 30;
      while (hl > 257 && l_lit[hl - 1] == 0) --hl;
      while (hd > 1 && l_dist[hd - 1] == 0) --hd;
      hlit = hl;
      hdist = hd;
      // run-length code of the concatenated lengths (runs may cross from the literal to the distance lengths)
      const int total = hl + hd;
      auto L = [&](int i) { return i < hl ? (int)l_lit[i] : (int)l_dist[i - hl]; };
      int ni = 0;
      for (int i = 0; i < 19; ++i) f_cl[i] = 0;
      for (int i = 0; i < total;) {
        const int cur = L(i);
        int run = 1;
        while (i + run < total && L(i + run) == cur) ++run;
        i += run;
        if (cur == 0) {
          while (run >= 11) { const int r = min(run, 138); items[ni++] = (uint16_t)(18 | (r - 11) << 8); f_cl[18]++; run -= r; }
          if (run >= 3) { items[ni++] = (uint16_t)(17 | (run - 3) << 8); f_cl[17]++; run = 0; }
        } else {
          items[ni++] = (uint16_t)cur; f_cl[cur]++; --run;
          while (run >= 3) { const int r = min(run, 6); items[ni++] = (uint16_t)(16 | (r - 3) << 8); f_cl[16]++; run -= r; }
        }
        while (run > 0) { items[ni++] = (uint16_t)cur; f_cl[cur]++; --run; }
      }
      n_items = ni;
    }
    __syncwarp();
    huff_lengths(f_cl, 19, 7, l_cl, head);
    if (lane == 0) {
      huff_codes(l_cl, 19, c_cl, head + 2560);
      int hc = 19;
      while (hc > 4 && l_cl[kClOrder[hc - 1]] == 0) --hc;
      hclen = hc;
      uint32_t bits = 3 + 5 + 5 + 4 + 3 * hc;
      for (int i = 0; i < n_items; ++i) {
        const int sym = items[i] & 31;
        bits += l_cl[sym] + (sym == 16 ? 2 : sym == 17 ? 3 : sym == 18 ? 7 : 0);
      }
      hdr_bits = bits;
    }
  }
  __syncthreads();

  // exact size of the dynamic block; the stored alternative is n + 10 bytes
  uint64_t db = 0;
  for (int i = tid; i < 286; i += kThreads) db += (uint64_t)f_lit[i] * (l_lit[i] + lit_extra_bits(i));
  if (tid < 30) db += (uint64_t)f_dist[tid] * (l_dist[tid] + dist_extra_bits(tid));
  const uint64_t data_bits = block_sum(db, red);
  const uint64_t end_bits = hdr_bits + data_bits;   // after the end-of-block code
  const int dyn_bytes = (int)((end_bits + 3 + 7) / 8) + 4;
  uint8_t* dst = segs + ((size_t)v * nseg + s) * kSegSlot;
  int bytes;
  if (dyn_bytes < n + 10) {
    bytes = dyn_bytes;
    // bits of each sub-block's tokens, then their offsets
    if (tid < kSubs) {
      uint32_t b = 0;
      const uint16_t* t = tok + tid * kSub;
      for (int i = 0; i < ntok[tid];) {
        if (t[i] & 0x8000u) { b += l_lit[t[i] & 255]; ++i; continue; }
        int sym, ne, ex;
        len_code(t[i], &sym, &ne, &ex);
        b += l_lit[sym] + ne;
        dist_code(t[i + 1] + 1, &sym, &ne, &ex);
        b += l_dist[sym] + ne;
        i += 2;
      }
      tok_bits[tid] = b;
    }
    uint32_t* out = reinterpret_cast<uint32_t*>(win);
    for (int i = tid; i < (dyn_bytes + 3) / 4 + 1; i += kThreads) out[i] = 0;
    __syncthreads();
    if (tid == 0) {
      uint32_t acc = hdr_bits;
      for (int k = 0; k < kSubs; ++k) { const uint32_t b = tok_bits[k]; tok_bits[k] = acc; acc += b; }
      tok_bits[kSubs] = acc;
      BitWriter bw(out, 0);
      bw.put(0, 1);                                  // BFINAL 0
      bw.put(2, 2);                                  // BTYPE 10: dynamic Huffman
      bw.put(hlit - 257, 5);
      bw.put(hdist - 1, 5);
      bw.put(hclen - 4, 4);
      for (int i = 0; i < hclen; ++i) bw.put(l_cl[kClOrder[i]], 3);
      for (int i = 0; i < n_items; ++i) {
        const int sym = items[i] & 31, ex = items[i] >> 8;
        bw.put(c_cl[sym], l_cl[sym]);
        if (sym == 16) bw.put(ex, 2);
        else if (sym == 17) bw.put(ex, 3);
        else if (sym == 18) bw.put(ex, 7);
      }
      bw.flush();
    }
    __syncthreads();
    if (tid < kSubs) {
      BitWriter bw(out, tok_bits[tid]);
      const uint16_t* t = tok + tid * kSub;
      for (int i = 0; i < ntok[tid];) {
        if (t[i] & 0x8000u) { const int c = t[i] & 255; bw.put(c_lit[c], l_lit[c]); ++i; continue; }
        int sym, ne, ex;
        len_code(t[i], &sym, &ne, &ex);
        bw.put(c_lit[sym], l_lit[sym]);
        if (ne) bw.put(ex, ne);
        dist_code(t[i + 1] + 1, &sym, &ne, &ex);
        bw.put(c_dist[sym], l_dist[sym]);
        if (ne) bw.put(ex, ne);
        i += 2;
      }
      if (tid == kSubs - 1) bw.put(c_lit[256], l_lit[256]);
      bw.flush();
    }
    __syncthreads();
    // sync flush: an empty stored block (3 zero bits, the pad, LEN 0000, NLEN FFFF)
    uint8_t* ob = win;
    if (tid == 0) {
      const int at = dyn_bytes - 4;
      ob[at] = 0; ob[at + 1] = 0; ob[at + 2] = 0xff; ob[at + 3] = 0xff;
    }
    __syncthreads();
    for (int i = tid; i < bytes; i += kThreads) dst[i] = ob[i];
  } else {
    bytes = n + 10;
    if (tid == 0) {
      dst[0] = 0;                                    // BFINAL 0, BTYPE 00, pad
      dst[1] = (uint8_t)(n & 255); dst[2] = (uint8_t)(n >> 8);
      dst[3] = (uint8_t)(~n & 255); dst[4] = (uint8_t)((~n >> 8) & 255);
      dst[5 + n] = 0; dst[6 + n] = 0; dst[7 + n] = 0; dst[8 + n] = 0xff; dst[9 + n] = 0xff;
    }
    for (int i = tid; i < n; i += kThreads) dst[5 + i] = win[hist + i];
  }
  if (tid == 0) info[(size_t)v * nseg + s] = SegInfo{(uint32_t)bytes, adler_a, adler_b, 0u};
}

// ---- pack -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kPackThreads) k_png_pack(int64_t N, int nseg, const uint8_t* __restrict__ segs,
                                                           const SegInfo* __restrict__ info, uint8_t* __restrict__ out,
                                                           size_t bound, int64_t* __restrict__ sizes) {
  __shared__ uint64_t red[kPackThreads / 32];
  const int s = blockIdx.x, v = blockIdx.y, tid = threadIdx.x;
  const SegInfo* fi = info + (size_t)v * nseg;
  uint64_t off = 0;
  for (int r = tid; r < s; r += kPackThreads) off += fi[r].bytes;
  off = block_sum(off, red);
  uint8_t* o = out + (size_t)v * bound;
  const uint32_t bytes = fi[s].bytes;
  const uint8_t* src = segs + ((size_t)v * nseg + s) * kSegSlot;
  for (uint32_t i = tid; i < bytes; i += kPackThreads) o[2 + off + i] = src[i];
  if (s == 0 && tid == 0) { o[0] = 0x78; o[1] = 0x5e; }    // deflate, 32 KiB window, FCHECK
  if (s == nseg - 1) {
    // Adler-32 of the whole stream from (1, 0): byte i of N weighs N - i in s2, which is its weight inside its
    // segment plus N - (the segment's end)
    uint64_t s1 = 0, s2 = 0;
    for (int r = tid; r < nseg; r += kPackThreads) {
      const uint64_t endr = (uint64_t)min(N, (int64_t)(r + 1) * kSeg);
      s1 += fi[r].a;
      s2 += fi[r].b + ((uint64_t)N - endr) % kAdlerMod * fi[r].a % kAdlerMod;
    }
    s1 = block_sum(s1, red);
    s2 = block_sum(s2, red);
    if (tid == 0) {
      const uint32_t a = (uint32_t)((1 + s1) % kAdlerMod), b = (uint32_t)(((uint64_t)N % kAdlerMod + s2) % kAdlerMod);
      uint8_t* t = o + 2 + off + bytes;
      t[0] = 0x03; t[1] = 0x00;                      // final empty fixed-Huffman block
      t[2] = (uint8_t)(b >> 8); t[3] = (uint8_t)b; t[4] = (uint8_t)(a >> 8); t[5] = (uint8_t)a;
      sizes[v] = (int64_t)(2 + off + bytes + 6);
    }
  }
}

}  // namespace

extern "C" GSB_API size_t gsb_png_bound(int32_t H, int32_t W) {
  Geometry g;
  return geometry(H, W, &g) ? g.bound : 0;
}

extern "C" GSB_API size_t gsb_png_scratch_bytes(int32_t V, int32_t H, int32_t W) {
  Geometry g;
  if (V <= 0 || !geometry(H, W, &g)) return 0;
  return (size_t)V * (g.filt_stride + (size_t)g.nseg * (kSegSlot + sizeof(SegInfo)));
}

extern "C" GSB_API int gsb_png_encode_batch(int32_t V, int32_t H, int32_t W, const uint8_t* rgb, void* scratch,
                                            size_t scratch_bytes, uint8_t* out, int64_t* sizes, gsb_stream_t stream) {
  Geometry g;
  if (V <= 0 || V > 65535 || !geometry(H, W, &g) || !rgb || !scratch || !out || !sizes ||
      reinterpret_cast<uintptr_t>(scratch) % 16 != 0 || reinterpret_cast<uintptr_t>(sizes) % 8 != 0) {
    gsb_set_error("gsb_png_encode_batch: bad argument");
    return GSB_ERR_INVALID;
  }
  if (scratch_bytes < gsb_png_scratch_bytes(V, H, W)) {
    gsb_set_error("gsb_png_encode_batch: scratch smaller than gsb_png_scratch_bytes()");
    return GSB_ERR_INVALID;
  }
  uint8_t* filt = static_cast<uint8_t*>(scratch);
  uint8_t* segs = filt + (size_t)V * g.filt_stride;
  SegInfo* info = reinterpret_cast<SegInfo*>(segs + (size_t)V * g.nseg * kSegSlot);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = check(cudaFuncSetAttribute(k_png_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDeflateSmem),
                 "k_png_deflate shared memory");
  if (rc != GSB_OK) return rc;
  gsb_count_launch(3);
  k_png_filter<<<dim3((unsigned)H, (unsigned)V), kFilterThreads, 0, st>>>(H, W, rgb, filt, g.filt_stride);
  rc = check(cudaGetLastError(), "k_png_filter");
  if (rc != GSB_OK) return rc;
  const dim3 grid((unsigned)g.nseg, (unsigned)V);
  k_png_deflate<<<grid, kThreads, kDeflateSmem, st>>>(g.N, 3 * W + 1, filt, g.filt_stride, segs, info, (int)g.nseg);
  rc = check(cudaGetLastError(), "k_png_deflate");
  if (rc != GSB_OK) return rc;
  k_png_pack<<<grid, kPackThreads, 0, st>>>(g.N, (int)g.nseg, segs, info, out, g.bound, sizes);
  return check(cudaGetLastError(), "k_png_pack");
}

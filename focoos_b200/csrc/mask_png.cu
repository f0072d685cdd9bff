// PNG encoding of the kept segmentation masks on the device (utils/vision.py:264-293 trim_mask + binary_mask_to_base64,
// fai_mf/processor.py:275-304): every crop m[y1:min(y2,H), x1:min(x2,W)] becomes the byte stream `cv2.imencode(".png", crop * 255)`
// writes, i.e. libpng with its defaults on a single-channel 8-bit image:
//   - signature, IHDR (bit depth 8, colour type 0), IDAT chunks of 8192 zlib bytes (the last one shorter), IEND;
//   - every row filtered with SUB (filter byte 1), so on 0/255 data each filtered byte is 0, 1 or 255; a crop one pixel wide is filtered
//     with NONE (filter byte 0);
//   - zlib: CMF with the smallest window >= 256 bytes covering the h*(w+1) filtered bytes (capped at 32 KiB), FLEVEL 0; the body is
//     what zlib's deflate emits with strategy Z_RLE and memLevel 8; the stream ends with the Adler-32 of the filtered bytes.
// So the deflate body reproduces zlib's deflate_rle: the greedy parse (a match has distance 1, needs the previous byte to equal the
// next three, and is at most 258 long), a block flushed after every 16383 symbols and one last block after the final symbol (empty
// when the symbol count is a multiple of 16383), and _tr_flush_block's choice of fixed or dynamic trees, with the trees built as
// zlib builds them (heap with the depth tie-break, the bit-length overflow fix, the bit-length tree with its repeat codes).
//
// Data-parallel plan, one launch sequence for all masks of a call, nothing synchronises with the host:
//   count  (thread / row)   symbols of the row in closed form per run of equal filtered bytes; Adler-32 partial sums
//   scan   (block / mask)   first symbol of every row; symbol count -> block count; Adler-32
//   hist   (thread / row)   per-block literal/length and distance histograms
//   tree   (thread / block) Huffman trees, fixed-or-dynamic choice, the code tables and the block header as a bit string
//   bits   (thread / row)   bits of the row's symbols (plus the block headers / end-of-block codes that fall in the row)
//   scan   (block / mask)   first bit of every row; zlib and PNG lengths; exclusive scan over masks -> compact offsets
//   emit   (thread / row)   the row's bits into a zeroed per-mask zlib buffer (boundary words with atomicOr, interior words stored)
//   finish (thread / mask)  zlib header and Adler-32
//   copy   (thread / 256 B) zlib bytes into the IDAT chunks of the compact output; CRC-32 of each piece, shifted and XOR-combined
//   close  (thread / chunk) chunk lengths / types / CRCs, signature + IHDR, IEND
#include <algorithm>

#include "common.cuh"

#define FB_HD __host__ __device__ __forceinline__

namespace fb200 {
namespace png {

constexpr int kSymBuf = 16383;  // symbols per deflate block: zlib's symbol buffer (memLevel 8 -> 1 << 14 entries) holds one less
constexpr int kChunk = 8192;    // IDAT payload bytes (libpng's compression buffer)
constexpr int kPiece = 256;     // zlib bytes per thread of the copy / CRC pass
constexpr int kHead = 33;       // signature (8) + IHDR chunk (25)
constexpr int LCODES = 286, DCODES = 30, BLCODES = 19, NCODES = LCODES + DCODES, MAXBITS = 15;
constexpr int FSTRIDE = NCODES + 1;  // per-block counts: literal/length codes, distance codes, filtered bytes covered
constexpr int kHdrBytes = 320;  // dynamic block header: at most 3 + 14 + 19*3 + 316*(7+7) bits
constexpr int kAdlerMod = 65521;

struct MaskInfo {
  int h, w;               // crop size (0 rows or columns: nothing is encoded)
  int x1, y1;
  int64_t nbytes;         // filtered bytes h*(w+1)
  int nsym, nblk;
  int64_t bits;           // bits of the zlib stream before the Adler-32 (header included)
  int zlen, png_len, png_off;
  uint32_t adler;
  int err;
};

struct BlockHdr {
  int bits;               // header bits: block type, and the tree description of a dynamic block
  int stored;             // _tr_flush_block would pick a stored block (never seen on 0/255 data; reported as an error)
  uint8_t b[kHdrBytes];
};

struct Ctx {
  const uint8_t* masks;
  int n, H, W, maxblk, maxchunk;
  int64_t zstride;        // bytes of each mask's zlib scratch (multiple of 8)
  const int* bbox;
  uint8_t* out;
  int* lengths;
  MaskInfo* info;
  int* row_nsym;  int* row_sym0;
  int64_t* row_bits; int64_t* row_bit0; int64_t* row_s1; int64_t* row_s2;
  uint32_t* codes;        // [n*maxblk][NCODES]: (reversed code) | (length << 16)
  BlockHdr* hdr;          // [n*maxblk]
  int* freq;              // [n*maxblk][FSTRIDE] (zeroed)
  uint32_t* crc;          // [n*maxchunk] (zeroed)
  uint8_t* z;             // [n][zstride] (zeroed)
};

FB_HD void at_add(int* p, int v) {
#ifdef __CUDA_ARCH__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}
FB_HD void at_or(uint32_t* p, uint32_t v) {
#ifdef __CUDA_ARCH__
  atomicOr(p, v);
#else
  *p |= v;
#endif
}
FB_HD void at_xor(uint32_t* p, uint32_t v) {
#ifdef __CUDA_ARCH__
  atomicXor(p, v);
#else
  *p ^= v;
#endif
}

// ---- sizes -----------------------------------------------------------------------------------------------------------
// A block never takes more than its fixed-tree size (_tr_flush_block keeps the smaller one): at most 9 bits per filtered byte
// (a literal 255), plus 3 header and 7 end-of-block bits, rounded up to whole bytes as zlib's length estimate is.
static inline int64_t zlib_bound(int64_t N) { return 2 + (9 * N + 7) / 8 + 3 * (N / kSymBuf + 2) + 4; }
static inline int64_t png_bound(int64_t N) { const int64_t zb = zlib_bound(N); return kHead + zb + 12 * ((zb + kChunk - 1) / kChunk) + 12; }

// ---- the symbols of one run of equal filtered bytes, in closed form ----------------------------------------------------
// Group = [literal t] + E x [literal 0] + C(R), C(R) = R/258 matches of 258, then one match of R%258 if that is >= 3, else R%258
// literals 0.  A row is the group of its filter byte (t = 1) followed by one group per run of equal pixels.
struct Group { int t, E, R; };

FB_HD int group_nsym(Group g) {
  const int q = g.R / 258, r = g.R % 258;
  return 1 + g.E + q + (r >= 3 ? 1 : r);
}
// symbol k of the group: a literal byte (0..255) or 256 + match length
FB_HD int group_sym(Group g, int k) {
  if (k == 0) return g.t;
  if (k <= g.E) return 0;
  const int j = k - 1 - g.E, q = g.R / 258, r = g.R % 258;
  if (j < q) return 256 + 258;
  return r >= 3 ? 256 + r : 0;
}

// calls f(Group) for every group of the crop row in stream order
template <class F>
FB_HD void walk_row(const uint8_t* row, int w, F&& f) {
  f(Group{1, 0, 0});
  int p = 0;
  while (p < w) {
    const bool v = row[p] != 0;
    int q = p + 1;
    while (q < w && (row[q] != 0) == v) ++q;
    const int n = q - p;
    if (p == 0 && !v) f(Group{0, 0, n - 1});
    else {
      const int t = p == 0 ? 255 : (v ? 255 : 1);  // first pixel raw, else the SUB difference 255 (0 -> 255) or 1 (255 -> 0)
      if (n == 1) f(Group{t, 0, 0});
      else f(Group{t, 1, n - 2});
    }
    p = q;
  }
}

// a crop one pixel wide: libpng filters its rows with NONE (filter byte 0), so runs of 0 cross rows and the whole stream
// [0, v0, 0, v1, ...] is walked at once, by the thread of row 0
template <class F>
FB_HD void walk_column(const uint8_t* col, int64_t pitch, int h, F&& f) {
  const int64_t N = 2 * (int64_t)h;
  auto byte = [&](int64_t j) { return (j & 1) && col[(j >> 1) * pitch] ? 255 : 0; };
  for (int64_t j = 0; j < N;) {
    const int v = byte(j);
    int64_t k = j + 1;
    while (k < N && byte(k) == v) ++k;
    f(Group{v, 0, (int)(k - j - 1)});
    j = k;
  }
}

template <class F>
FB_HD void walk_crop_row(const uint8_t* row, int64_t pitch, int w, int h, int y, F&& f) {
  if (w > 1) walk_row(row, w, f);
  else if (y == 0) walk_column(row, pitch, h, f);
}

// deflate length code of a match length 3..258: symbol 257..285 and its extra bits
FB_HD void len_code(int L, int& sym, int& xbits, int& xval) {
  const int lc = L - 3;
  if (lc == 255) { sym = 285; xbits = 0; xval = 0; return; }
  if (lc < 8) { sym = 257 + lc; xbits = 0; xval = 0; return; }
  int e = 1, base = 8, c = 8;  // codes 8..27 come in fours with 1..5 extra bits
  while (lc >= base + (4 << e)) { base += 4 << e; c += 4; ++e; }
  const int k = (lc - base) >> e;
  sym = 257 + c + k;
  xbits = e;
  xval = lc - base - (k << e);
}

FB_HD bool crop_of(const Ctx& c, int i, int& h, int& w, int& x1, int& y1) {
  const int* b = c.bbox + 4 * i;
  x1 = b[0]; y1 = b[1];
  h = max(0, min(b[3], c.H) - y1);
  w = max(0, min(b[2], c.W) - x1);
  return x1 >= 0 && y1 >= 0;
}

// ---- count ------------------------------------------------------------------------------------------------------------
FB_HD void count_row(const Ctx& c, int64_t r) {
  const int i = (int)(r / c.H), y = (int)(r % c.H);
  int h, w, x1, y1;
  const bool ok = crop_of(c, i, h, w, x1, y1);
  if (!ok || y >= h || w == 0) { c.row_nsym[r] = 0; c.row_s1[r] = 0; c.row_s2[r] = 0; return; }
  const uint8_t* row = c.masks + ((int64_t)i * c.H + y1 + y) * c.W + x1;
  int ns = 0;
  walk_crop_row(row, c.W, w, h, y, [&](Group g) { ns += group_nsym(g); });
  // Adler-32 partials over this row's filtered bytes j0 .. j0+w: s1 += b, s2 += (N - j) * b   (mod 65521)
  const int64_t N = (int64_t)h * (w + 1), j0 = (int64_t)y * (w + 1);
  const int fb = w > 1 ? 1 : 0;  // the filter byte: SUB, or NONE on a one-pixel-wide crop
  uint64_t s1 = fb, s2 = ((N - j0) % kAdlerMod) * fb;
  int prev = 0;
  for (int x = 0; x < w; ++x) {
    const int v = row[x] ? 255 : 0, b = (v - prev) & 255;
    prev = v;
    s1 += b;
    s2 += (uint64_t)((N - j0 - 1 - x) % kAdlerMod) * b;
  }
  c.row_nsym[r] = ns;
  c.row_s1[r] = (int64_t)(s1 % kAdlerMod);
  c.row_s2[r] = (int64_t)(s2 % kAdlerMod);
}

// ---- histogram --------------------------------------------------------------------------------------------------------
FB_HD void hist_row(const Ctx& c, int64_t r) {
  const int i = (int)(r / c.H), y = (int)(r % c.H);
  int h, w, x1, y1;
  if (!crop_of(c, i, h, w, x1, y1) || y >= h || w == 0) return;
  const uint8_t* row = c.masks + ((int64_t)i * c.H + y1 + y) * c.W + x1;
  int* fr = c.freq + (int64_t)i * c.maxblk * FSTRIDE;
  int g0 = c.row_sym0[r];
  // literal 0 / 1 / 255, matches of 258, all matches (distance code 0) and bytes of the current block, flushed on a block change
  int cur = g0 / kSymBuf, n0 = 0, n1 = 0, n255 = 0, n258 = 0, nm = 0, nb = 0;
  auto flush = [&]() {
    int* f = fr + (int64_t)cur * FSTRIDE;
    if (n0) at_add(f + 0, n0);
    if (n1) at_add(f + 1, n1);
    if (n255) at_add(f + 255, n255);
    if (n258) at_add(f + 285, n258);
    if (nm) at_add(f + LCODES, nm);
    if (nb) at_add(f + NCODES, nb);
    n0 = n1 = n255 = n258 = nm = nb = 0;
  };
  walk_crop_row(row, c.W, w, h, y, [&](Group g) {
    const int ns = group_nsym(g);
    for (int k = 0; k < ns; ++k, ++g0) {
      const int b = g0 / kSymBuf;
      if (b != cur) { flush(); cur = b; }
      const int s = group_sym(g, k);
      if (s < 256) { if (s == 0) ++n0; else if (s == 1) ++n1; else ++n255; ++nb; continue; }
      ++nm;
      nb += s - 256;
      if (s == 256 + 258) { ++n258; continue; }
      int sym, xb, xv;
      len_code(s - 256, sym, xb, xv);
      at_add(fr + (int64_t)b * FSTRIDE + sym, 1);
    }
  });
  flush();
}

// ---- Huffman trees exactly as zlib builds them (trees.c: build_tree, gen_bitlen, gen_codes, scan_tree, send_tree) ------------
// HS >= 2 * elems + 1 nodes; zlib sorts the nodes downwards from the top of its heap array, so any HS gives the same tree.
template <int HS>
struct Tree {
  uint16_t freq[HS], dad[HS], len[HS + 1], code[HS];  // len: + the guard scan_tree writes past max_code
  uint16_t heap[HS];
  uint8_t depth[HS];
  int heap_len, heap_max;
};
struct Lens {
  int64_t opt_len, static_len;
  int bl_count[MAXBITS + 1];
};

template <int HS>
FB_HD bool smaller(const Tree<HS>& t, int n, int m) {
  return t.freq[n] < t.freq[m] || (t.freq[n] == t.freq[m] && t.depth[n] <= t.depth[m]);
}

template <int HS>
FB_HD void pqdownheap(Tree<HS>& t, int k) {
  const int v = t.heap[k];
  int j = k << 1;
  while (j <= t.heap_len) {
    if (j < t.heap_len && smaller(t, t.heap[j + 1], t.heap[j])) j++;
    if (smaller(t, v, t.heap[j])) break;
    t.heap[k] = t.heap[j];
    k = j;
    j <<= 1;
  }
  t.heap[k] = (uint16_t)v;
}

FB_HD unsigned bi_reverse(unsigned code, int len) {
  unsigned r = 0;
  do { r |= code & 1; code >>= 1; r <<= 1; } while (--len > 0);
  return r >> 1;
}

FB_HD int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }

// elems symbols; stree_len(n): static code length (has_static); extra(n - base) extra bits of symbol n >= base; returns max_code
template <int HS, class SLen, class Extra>
FB_HD int build_tree(Tree<HS>& t, Lens& s, int elems, int max_length, bool has_static, SLen stree_len, int base, Extra extra) {
  int max_code = -1;
  t.heap_len = 0;
  t.heap_max = HS;
  for (int n = 0; n < elems; n++) {
    if (t.freq[n] != 0) { t.heap[++t.heap_len] = (uint16_t)(max_code = n); t.depth[n] = 0; }
    else t.len[n] = 0;
  }
  while (t.heap_len < 2) {  // at least two codes of non-zero frequency
    const int node = max_code < 2 ? ++max_code : 0;
    t.heap[++t.heap_len] = (uint16_t)node;
    t.freq[node] = 1;
    t.depth[node] = 0;
    s.opt_len--;
    if (has_static) s.static_len -= stree_len(node);
  }
  for (int n = t.heap_len / 2; n >= 1; n--) pqdownheap(t, n);
  int node = elems;
  do {
    const int n = t.heap[1];
    t.heap[1] = t.heap[t.heap_len--];
    pqdownheap(t, 1);
    const int m = t.heap[1];
    t.heap[--t.heap_max] = (uint16_t)n;
    t.heap[--t.heap_max] = (uint16_t)m;
    t.freq[node] = (uint16_t)(t.freq[n] + t.freq[m]);
    t.depth[node] = (uint8_t)((t.depth[n] >= t.depth[m] ? t.depth[n] : t.depth[m]) + 1);
    t.dad[n] = t.dad[m] = (uint16_t)node;
    t.heap[1] = (uint16_t)node++;
    pqdownheap(t, 1);
  } while (t.heap_len >= 2);
  t.heap[--t.heap_max] = t.heap[1];

  // gen_bitlen
  for (int b = 0; b <= MAXBITS; b++) s.bl_count[b] = 0;
  t.len[t.heap[t.heap_max]] = 0;
  int overflow = 0, h;
  for (h = t.heap_max + 1; h < HS; h++) {
    const int n = t.heap[h];
    int bits = t.len[t.dad[n]] + 1;
    if (bits > max_length) bits = max_length, overflow++;
    t.len[n] = (uint16_t)bits;
    if (n > max_code) continue;
    s.bl_count[bits]++;
    const int xbits = n >= base ? extra(n - base) : 0;
    const int64_t f = t.freq[n];
    s.opt_len += f * (bits + xbits);
    if (has_static) s.static_len += f * (stree_len(n) + xbits);
  }
  if (overflow) {
    do {
      int bits = max_length - 1;
      while (s.bl_count[bits] == 0) bits--;
      s.bl_count[bits]--;
      s.bl_count[bits + 1] += 2;
      s.bl_count[max_length]--;
      overflow -= 2;
    } while (overflow > 0);
    for (int bits = max_length; bits != 0; bits--) {
      int n = s.bl_count[bits];
      while (n != 0) {
        const int m = t.heap[--h];
        if (m > max_code) continue;
        if (t.len[m] != bits) {
          s.opt_len += ((int64_t)bits - t.len[m]) * t.freq[m];
          t.len[m] = (uint16_t)bits;
        }
        n--;
      }
    }
  }
  // gen_codes
  int next_code[MAXBITS + 1];
  unsigned code = 0;
  for (int bits = 1; bits <= MAXBITS; bits++) { code = (code + s.bl_count[bits - 1]) << 1; next_code[bits] = (int)code; }
  for (int n = 0; n <= max_code; n++) {
    const int l = t.len[n];
    if (l == 0) continue;
    t.code[n] = (uint16_t)bi_reverse((unsigned)next_code[l]++, l);
  }
  return max_code;
}

FB_HD int extra_lbits(int c) { return c < 8 ? 0 : c < 28 ? (c - 4) / 4 : 0; }
FB_HD int extra_blbits(int c) { return c == 0 ? 2 : c == 1 ? 3 : 7; }

// scan_tree (emit == false: bit-length tree frequencies) / send_tree (emit == true: the codes, through put(value, bits))
template <int HS, int HB, class Put>
FB_HD void scan_send_tree(Tree<HS>& t, int max_code, Tree<HB>& bl, bool emit, Put&& put) {
  int prevlen = -1, nextlen = t.len[0], count = 0, max_count = 7, min_count = 4;
  if (nextlen == 0) max_count = 138, min_count = 3;
  t.len[max_code + 1] = 0xffff;  // guard
  auto sym = [&](int s) { if (emit) put(bl.code[s], bl.len[s]); else bl.freq[s]++; };
  for (int n = 0; n <= max_code; n++) {
    const int curlen = nextlen;
    nextlen = t.len[n + 1];
    if (++count < max_count && curlen == nextlen) continue;
    if (count < min_count) {
      if (emit) { do { sym(curlen); } while (--count != 0); }
      else bl.freq[curlen] += count;
    } else if (curlen != 0) {
      if (curlen != prevlen) { sym(curlen); count--; }
      sym(16);
      if (emit) put(count - 3, 2);
    } else if (count <= 10) {
      sym(17);
      if (emit) put(count - 3, 3);
    } else {
      sym(18);
      if (emit) put(count - 11, 7);
    }
    count = 0;
    prevlen = curlen;
    if (nextlen == 0) max_count = 138, min_count = 3;
    else if (curlen == nextlen) max_count = 6, min_count = 3;
    else max_count = 7, min_count = 4;
  }
}

constexpr int HL = 2 * LCODES + 1, HD = 2 * DCODES + 1, HB = 2 * BLCODES + 1;

__device__ __host__ inline void tree_block(const Ctx& c, int64_t bi, Tree<HL>& lt, Tree<HD>& dt, Tree<HB>& bt) {
  const int i = (int)(bi / c.maxblk), b = (int)(bi % c.maxblk);
  const MaskInfo& mi = c.info[i];
  if (mi.err || mi.h == 0 || mi.w == 0 || b >= mi.nblk) return;
  const bool last = b == mi.nblk - 1;
  const int* f = c.freq + bi * FSTRIDE;
  for (int n = 0; n < LCODES; n++) lt.freq[n] = (uint16_t)f[n];
  for (int n = 0; n < DCODES; n++) dt.freq[n] = (uint16_t)f[LCODES + n];
  for (int n = 0; n < BLCODES; n++) bt.freq[n] = 0;
  lt.freq[256] = 1;  // end of block
  Lens s;
  s.opt_len = s.static_len = 0;
  const int lmax = build_tree(lt, s, LCODES, MAXBITS, true, [](int n) { return static_llen(n); }, 257, [](int e) { return extra_lbits(e); });
  const int dmax = build_tree(dt, s, DCODES, MAXBITS, true, [](int) { return 5; }, 0, [](int) { return 0; });
  auto nop = [](int, int) {};
  scan_send_tree(lt, lmax, bt, false, nop);
  scan_send_tree(dt, dmax, bt, false, nop);
  build_tree(bt, s, BLCODES, 7, false, [](int) { return 0; }, 16, [](int e) { return extra_blbits(e); });
  const uint8_t bl_order[BLCODES] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  int max_blindex;
  for (max_blindex = BLCODES - 1; max_blindex >= 3; max_blindex--)
    if (bt.len[bl_order[max_blindex]] != 0) break;
  s.opt_len += 3 * ((int64_t)max_blindex + 1) + 5 + 5 + 4;
  int64_t opt_lenb = (s.opt_len + 3 + 7) >> 3;
  const int64_t static_lenb = (s.static_len + 3 + 7) >> 3;
  if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
  // zlib stores a block whose filtered bytes plus 4 do not exceed opt_lenb; no 0/255 mask has been seen to reach that (tests/golden/
  // png_deflate.npz records the search), so such a block is reported as an error instead of being encoded
  BlockHdr& hd = c.hdr[bi];
  hd.stored = (int64_t)f[NCODES] + 4 <= opt_lenb;
  for (int k = 0; k < kHdrBytes; k++) hd.b[k] = 0;
  int nb = 0;
  auto put = [&](int v, int bits) {
    for (int k = 0; k < bits; k++, nb++) if ((v >> k) & 1) hd.b[nb >> 3] |= (uint8_t)(1u << (nb & 7));
  };
  uint32_t* code = c.codes + bi * NCODES;
  if (static_lenb == opt_lenb) {
    put(2 + (last ? 1 : 0), 3);
    for (int n = 0; n < LCODES; n++) {
      const int l = static_llen(n);
      const int cv = n < 144 ? 0x30 + n : n < 256 ? 0x190 + (n - 144) : n < 280 ? n - 256 : 0xc0 + (n - 280);
      code[n] = bi_reverse((unsigned)cv, l) | ((uint32_t)l << 16);
    }
    for (int n = 0; n < DCODES; n++) code[LCODES + n] = bi_reverse((unsigned)n, 5) | (5u << 16);
  } else {
    put(4 + (last ? 1 : 0), 3);
    put(lmax + 1 - 257, 5);
    put(dmax + 1 - 1, 5);
    put(max_blindex + 1 - 4, 4);
    for (int rank = 0; rank <= max_blindex; rank++) put(bt.len[bl_order[rank]], 3);
    scan_send_tree(lt, lmax, bt, true, put);
    scan_send_tree(dt, dmax, bt, true, put);
    for (int n = 0; n < LCODES; n++) code[n] = n <= lmax && lt.len[n] ? (uint32_t)lt.code[n] | ((uint32_t)lt.len[n] << 16) : 0u;
    for (int n = 0; n < DCODES; n++) code[LCODES + n] = n <= dmax && dt.len[n] ? (uint32_t)dt.code[n] | ((uint32_t)dt.len[n] << 16) : 0u;
  }
  hd.bits = nb;
}

// ---- the bits of one row: symbols, and the end-of-block codes / block headers that fall between them ----------------------
template <class Put>
FB_HD void row_stream(const Ctx& c, int64_t r, Put&& put) {
  const int i = (int)(r / c.H), y = (int)(r % c.H);
  const MaskInfo& mi = c.info[i];
  if (mi.err || y >= mi.h || mi.w == 0) return;
  const uint8_t* row = c.masks + ((int64_t)i * c.H + mi.y1 + y) * c.W + mi.x1;
  const int64_t bb = (int64_t)i * c.maxblk;
  int g = c.row_sym0[r];
  auto header = [&](int b) {
    const BlockHdr& hd = c.hdr[bb + b];
    for (int k = 0; k < hd.bits; k += 8) put(hd.b[k >> 3], min(8, hd.bits - k));
  };
  auto eob = [&](int b) { const uint32_t e = c.codes[(bb + b) * NCODES + 256]; put((int)(e & 0xffff), (int)(e >> 16)); };
  walk_crop_row(row, c.W, mi.w, mi.h, y, [&](Group gr) {
    const int ns = group_nsym(gr);
    for (int k = 0; k < ns; ++k, ++g) {
      const int b = g / kSymBuf;
      if (g % kSymBuf == 0) { if (b > 0) eob(b - 1); header(b); }
      const uint32_t* cd = c.codes + (bb + b) * NCODES;
      const int s = group_sym(gr, k);
      if (s < 256) { put((int)(cd[s] & 0xffff), (int)(cd[s] >> 16)); }
      else {
        int sym, xb, xv;
        len_code(s - 256, sym, xb, xv);
        put((int)(cd[sym] & 0xffff), (int)(cd[sym] >> 16));
        if (xb) put(xv, xb);
        put((int)(cd[LCODES] & 0xffff), (int)(cd[LCODES] >> 16));  // distance 1: distance code 0, no extra bits
      }
      if (g == mi.nsym - 1) {
        eob(b);
        if (b + 1 < mi.nblk) { header(b + 1); eob(b + 1); }  // the symbol count is a multiple of 16383: an empty last block
      }
    }
  });
}

FB_HD void bits_row(const Ctx& c, int64_t r) {
  int64_t nb = 0;
  row_stream(c, r, [&](int, int bits) { nb += bits; });
  c.row_bits[r] = nb;
}

FB_HD void emit_row(const Ctx& c, int64_t r) {
  const int i = (int)(r / c.H);
  if (c.info[i].err || (int)(r % c.H) >= c.info[i].h || c.info[i].w == 0) return;
  uint32_t* zw = reinterpret_cast<uint32_t*>(c.z + (int64_t)i * c.zstride);
  const int64_t p0 = c.row_bit0[r];
  int64_t word = p0 >> 5;
  const int64_t first = word;
  uint64_t acc = 0;
  int nacc = (int)(p0 & 31);
  // words shared with the neighbouring rows (the first and the last) are OR-ed; the ones in between belong to this row alone
  row_stream(c, r, [&](int v, int bits) {
    acc |= (uint64_t)(uint32_t)v << nacc;
    nacc += bits;
    while (nacc >= 32) {
      if (word == first) at_or(zw + word, (uint32_t)acc);
      else zw[word] = (uint32_t)acc;
      ++word;
      acc >>= 32;
      nacc -= 32;
    }
  });
  if (nacc > 0) at_or(zw + word, (uint32_t)acc);
}

// ---- CRC-32 (reflected, polynomial 0xedb88320) and its combination over pieces ----------------------------------------------
FB_HD uint32_t crc_raw(uint32_t c, const uint8_t* p, int n) {
  for (int k = 0; k < n; k++) {
    c ^= p[k];
    for (int j = 0; j < 8; j++) c = (c >> 1) ^ (0xedb88320u & (0u - (c & 1u)));
  }
  return c;
}
// a * b modulo the CRC polynomial, bit 31 = x^0 (a != 0)
FB_HD uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
  }
  return p;
}
// the CRC register after n more zero bytes: c * x^(8n)
FB_HD uint32_t crc_shift(uint32_t c, int64_t n) {
  uint32_t p = 1u << 31, sq = 1u << 23;  // x^0, x^8
  for (; n; n >>= 1) {
    if (n & 1) p = multmodp(sq, p);
    sq = multmodp(sq, sq);
  }
  return c ? multmodp(p, c) : 0u;
}

FB_HD void put_be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }

// zlib byte j of mask i -> position in the PNG file
FB_HD int64_t zpos(int64_t j) { return kHead + (j / kChunk) * 12 + 8 + j; }

FB_HD void copy_piece(const Ctx& c, int i, int64_t piece) {
  const MaskInfo& mi = c.info[i];
  const int64_t j0 = piece * kPiece;
  if (mi.err || mi.png_len == 0 || j0 >= mi.zlen) return;
  const int n = (int)min((int64_t)kPiece, (int64_t)mi.zlen - j0);
  const uint8_t* src = c.z + (int64_t)i * c.zstride + j0;
  uint8_t* dst = c.out + mi.png_off + zpos(j0);
  for (int k = 0; k < n; k++) dst[k] = src[k];
  const int64_t ch = j0 / kChunk;
  uint32_t cr = 0;
  if (j0 % kChunk == 0) { const uint8_t idat[4] = {'I', 'D', 'A', 'T'}; cr = crc_raw(0, idat, 4); }
  cr = crc_raw(cr, src, n);
  const int64_t chunk_end = min((ch + 1) * kChunk, (int64_t)mi.zlen);
  at_xor(c.crc + (int64_t)i * c.maxchunk + ch, crc_shift(cr, chunk_end - j0 - n));
}

FB_HD void close_chunk(const Ctx& c, int i, int ch) {
  const MaskInfo& mi = c.info[i];
  if (mi.err || mi.png_len == 0) return;
  const int nch = (mi.zlen + kChunk - 1) / kChunk;
  if (ch >= nch) return;
  uint8_t* o = c.out + mi.png_off;
  const int len = min(kChunk, mi.zlen - ch * kChunk);
  uint8_t* hd = o + zpos((int64_t)ch * kChunk) - 8;
  put_be32(hd, (uint32_t)len);
  hd[4] = 'I'; hd[5] = 'D'; hd[6] = 'A'; hd[7] = 'T';
  const uint32_t crc = c.crc[(int64_t)i * c.maxchunk + ch] ^ crc_shift(0xffffffffu, 4 + len) ^ 0xffffffffu;
  put_be32(hd + 8 + len, crc);
  if (ch == 0) {
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    for (int k = 0; k < 8; k++) o[k] = sig[k];
    uint8_t* ih = o + 8;
    put_be32(ih, 13);
    ih[4] = 'I'; ih[5] = 'H'; ih[6] = 'D'; ih[7] = 'R';
    put_be32(ih + 8, (uint32_t)mi.w);
    put_be32(ih + 12, (uint32_t)mi.h);
    ih[16] = 8; ih[17] = 0; ih[18] = 0; ih[19] = 0; ih[20] = 0;
    put_be32(ih + 21, crc_raw(0xffffffffu, ih + 4, 17) ^ 0xffffffffu);
  }
  if (ch == nch - 1) {
    uint8_t* ie = hd + 8 + len + 4;
    const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xae, 0x42, 0x60, 0x82};
    for (int k = 0; k < 12; k++) ie[k] = iend[k];
  }
}

// ---- per-mask scans ---------------------------------------------------------------------------------------------------
// mask i, after the symbol scan: crop, block count, Adler-32, CMF
FB_HD void mask_after_syms(const Ctx& c, int i, int64_t nsym, int64_t s1, int64_t s2) {
  MaskInfo& mi = c.info[i];
  int h, w, x1, y1;
  mi.err = crop_of(c, i, h, w, x1, y1) ? 0 : 1;
  mi.h = h; mi.w = w; mi.x1 = x1; mi.y1 = y1;
  mi.nbytes = (int64_t)h * (w + 1);
  mi.nsym = (int)nsym;
  mi.nblk = (int)(nsym / kSymBuf) + 1;
  mi.adler = (uint32_t)(((s2 + mi.nbytes) % kAdlerMod) << 16 | ((s1 + 1) % kAdlerMod));
}

FB_HD void mask_after_bits(const Ctx& c, int i, int64_t bits) {
  MaskInfo& mi = c.info[i];
  mi.bits = 16 + bits;
  if (mi.err || mi.h == 0 || mi.w == 0) { mi.zlen = 0; mi.png_len = 0; return; }
  for (int b = 0; b < mi.nblk; b++)
    if (c.hdr[(int64_t)i * c.maxblk + b].stored) mi.err = 1;
  mi.zlen = (int)((mi.bits + 7) / 8 + 4);
  mi.png_len = kHead + mi.zlen + 12 * ((mi.zlen + kChunk - 1) / kChunk) + 12;
}

FB_HD void finish_mask(const Ctx& c, int i) {
  const MaskInfo& mi = c.info[i];
  c.lengths[i] = mi.err ? -1 : mi.png_len;
  if (mi.err || mi.png_len == 0) return;
  uint8_t* z = c.z + (int64_t)i * c.zstride;
  int ci = 0;
  while (ci < 7 && mi.nbytes > (256 << ci)) ci++;
  z[0] = (uint8_t)(ci << 4 | 8);
  z[1] = (uint8_t)(31 - ((z[0] << 8) % 31));
  put_be32(z + mi.zlen - 4, mi.adler);
}

#ifdef __CUDACC__
// exclusive scan of one int64 per thread over a 256-thread block; *total = block sum
__device__ int64_t block_scan(int64_t v, int64_t* total) {
  __shared__ int64_t ws[8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int64_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int64_t t = lane < 8 ? ws[lane] : 0;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) { const int64_t y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
    if (lane < 8) ws[lane] = t;
  }
  __syncthreads();
  const int64_t r = x - v + (wid ? ws[wid - 1] : 0);
  *total = ws[7];
  __syncthreads();
  return r;
}

__global__ void count_kernel(Ctx c) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < (int64_t)c.n * c.H) count_row(c, r);
}
__global__ void scan_syms_kernel(Ctx c) {
  const int i = blockIdx.x;
  int64_t carry = 0, s1 = 0, s2 = 0;
  for (int y0 = 0; y0 < c.H; y0 += 256) {
    const int y = y0 + threadIdx.x;
    const int64_t r = (int64_t)i * c.H + y;
    int64_t tot;
    const int64_t e = block_scan(y < c.H ? c.row_nsym[r] : 0, &tot);
    if (y < c.H) c.row_sym0[r] = (int)(carry + e);
    carry += tot;
    block_scan(y < c.H ? c.row_s1[r] : 0, &tot); s1 += tot;
    block_scan(y < c.H ? c.row_s2[r] : 0, &tot); s2 += tot;
  }
  if (threadIdx.x == 0) mask_after_syms(c, i, carry, s1 % kAdlerMod, s2 % kAdlerMod);
}
__global__ void hist_kernel(Ctx c) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < (int64_t)c.n * c.H) hist_row(c, r);
}
__global__ void tree_kernel(Ctx c) {  // one single-thread block per deflate block: the trees live in shared memory
  const int64_t bi = blockIdx.x;
  __shared__ Tree<HL> lt;
  __shared__ Tree<HD> dt;
  __shared__ Tree<HB> bt;
  tree_block(c, bi, lt, dt, bt);
}
__global__ void bits_kernel(Ctx c) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < (int64_t)c.n * c.H) bits_row(c, r);
}
__global__ void scan_bits_kernel(Ctx c) {
  const int i = blockIdx.x;
  int64_t carry = 0;
  for (int y0 = 0; y0 < c.H; y0 += 256) {
    const int y = y0 + threadIdx.x;
    const int64_t r = (int64_t)i * c.H + y;
    int64_t tot;
    const int64_t e = block_scan(y < c.H ? c.row_bits[r] : 0, &tot);
    if (y < c.H) c.row_bit0[r] = 16 + carry + e;
    carry += tot;
  }
  if (threadIdx.x == 0) mask_after_bits(c, i, carry);
}
__global__ void offsets_kernel(Ctx c) {  // one block: compact PNG offsets over the masks
  int64_t carry = 0;
  for (int i0 = 0; i0 < c.n; i0 += 256) {
    const int i = i0 + threadIdx.x;
    int64_t tot;
    const int64_t e = block_scan(i < c.n ? c.info[i].png_len : 0, &tot);
    if (i < c.n) c.info[i].png_off = (int)(carry + e);
    carry += tot;
  }
}
__global__ void emit_kernel(Ctx c) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < (int64_t)c.n * c.H) emit_row(c, r);
}
__global__ void finish_kernel(Ctx c) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < c.n) finish_mask(c, i);
}
__global__ void copy_kernel(Ctx c) {
  const int64_t piece = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  copy_piece(c, blockIdx.y, piece);
}
__global__ void close_kernel(Ctx c) {
  const int ch = blockIdx.x * blockDim.x + threadIdx.x;
  close_chunk(c, blockIdx.y, ch);
}
#endif

struct Layout {
  int maxblk, maxchunk;
  int64_t zstride, off_info, off_rows, off_codes, off_hdr, off_zero, off_crc, off_z, total;
};

static inline int64_t align256(int64_t v) { return (v + 255) / 256 * 256; }

static inline Layout layout(int n, int H, int W) {
  Layout L;
  const int64_t N = (int64_t)H * (W + 1);
  L.maxblk = (int)(N / kSymBuf) + 2;
  const int64_t zb = zlib_bound(N);
  L.zstride = align256(zb);
  L.maxchunk = (int)((zb + kChunk - 1) / kChunk);
  const int64_t rows = (int64_t)n * H;
  int64_t o = 0;
  L.off_info = o; o = align256(o + (int64_t)n * sizeof(MaskInfo));
  L.off_rows = o; o = align256(o + rows * (2 * sizeof(int) + 4 * sizeof(int64_t)));
  L.off_codes = o; o = align256(o + (int64_t)n * L.maxblk * NCODES * sizeof(uint32_t));
  L.off_hdr = o; o = align256(o + (int64_t)n * L.maxblk * sizeof(BlockHdr));
  L.off_zero = o; o = align256(o + (int64_t)n * L.maxblk * FSTRIDE * sizeof(int));
  L.off_crc = o; o = align256(o + (int64_t)n * L.maxchunk * sizeof(uint32_t));
  L.off_z = o; o += (int64_t)n * L.zstride;
  L.total = o;
  return L;
}

static inline Ctx make_ctx(const Layout& L, const uint8_t* masks, int n, int H, int W, const int* bbox, uint8_t* out, int* lengths, uint8_t* ws) {
  Ctx c;
  c.masks = masks; c.n = n; c.H = H; c.W = W; c.maxblk = L.maxblk; c.maxchunk = L.maxchunk; c.zstride = L.zstride;
  c.bbox = bbox; c.out = out; c.lengths = lengths;
  c.info = reinterpret_cast<MaskInfo*>(ws + L.off_info);
  const int64_t rows = (int64_t)n * H;
  int64_t* r64 = reinterpret_cast<int64_t*>(ws + L.off_rows);
  c.row_bits = r64; c.row_bit0 = r64 + rows; c.row_s1 = r64 + 2 * rows; c.row_s2 = r64 + 3 * rows;
  c.row_nsym = reinterpret_cast<int*>(r64 + 4 * rows); c.row_sym0 = c.row_nsym + rows;
  c.codes = reinterpret_cast<uint32_t*>(ws + L.off_codes);
  c.hdr = reinterpret_cast<BlockHdr*>(ws + L.off_hdr);
  c.freq = reinterpret_cast<int*>(ws + L.off_zero);
  c.crc = reinterpret_cast<uint32_t*>(ws + L.off_crc);
  c.z = ws + L.off_z;
  return c;
}

}  // namespace png
}  // namespace fb200

#ifdef __CUDACC__
using namespace fb200;

extern "C" int64_t fb200_mask_png_workspace_bytes(int n, int H, int W) {
  if (n <= 0 || H <= 0 || W <= 0) return 0;
  return png::layout(n, H, W).total;
}

extern "C" int fb200_mask_png_bound(int H, int W) {
  if (H <= 0 || W <= 0) return 0;
  const int64_t b = png::png_bound((int64_t)H * (W + 1));
  return b > INT32_MAX / 2 ? -1 : (int)b;
}

extern "C" int fb200_mask_png(const uint8_t* masks, int n, int H, int W, const int* bbox, uint8_t* out, int* lengths, void* workspace, void* stream) {
  FB_CHECK_ARG(masks && bbox && out && lengths && workspace && n > 0 && H > 0 && W > 0, "mask_png: bad arguments");
  FB_CHECK_ARG(fb200_mask_png_bound(H, W) > 0 && (int64_t)n * fb200_mask_png_bound(H, W) <= INT32_MAX, "mask_png: %d masks of %dx%d exceed 2 GiB of PNG bounds", n, H, W);
  cudaStream_t st = (cudaStream_t)stream;
  const png::Layout L = png::layout(n, H, W);
  uint8_t* ws = static_cast<uint8_t*>(workspace);
  const png::Ctx c = png::make_ctx(L, masks, n, H, W, bbox, out, lengths, ws);
  if (cudaMemsetAsync(ws + L.off_zero, 0, (size_t)(L.total - L.off_zero), st) != cudaSuccess) { set_error("mask_png: memset failed"); return FB200_ERR_CUDA; }
  const int64_t rows = (int64_t)n * H;
  const unsigned rb = (unsigned)cdiv(rows, 128);
  png::count_kernel<<<rb, 128, 0, st>>>(c);
  png::scan_syms_kernel<<<n, 256, 0, st>>>(c);
  png::hist_kernel<<<rb, 128, 0, st>>>(c);
  png::tree_kernel<<<(unsigned)(n * L.maxblk), 1, 0, st>>>(c);
  png::bits_kernel<<<rb, 128, 0, st>>>(c);
  png::scan_bits_kernel<<<n, 256, 0, st>>>(c);
  png::offsets_kernel<<<1, 256, 0, st>>>(c);
  png::emit_kernel<<<rb, 128, 0, st>>>(c);
  png::finish_kernel<<<(unsigned)cdiv(n, 128), 128, 0, st>>>(c);
  png::copy_kernel<<<dim3((unsigned)cdiv(cdiv(L.zstride, png::kPiece), 128), (unsigned)n), 128, 0, st>>>(c);
  png::close_kernel<<<dim3((unsigned)cdiv(L.maxchunk, 64), (unsigned)n), 64, 0, st>>>(c);
  FB_CHECK_LAUNCH("mask_png");
  return FB200_OK;
}
#endif

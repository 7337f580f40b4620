/*
 * pinot_oracle.c — CPU restatement (plain C) of Apache Pinot's per-segment
 * DocIdSetOperator / filter operators / ProjectionOperator / GroupByOperator /
 * AggregationOperator path, block-at-a-time like the reference.
 *
 * TEST INFRASTRUCTURE ONLY (see pinot_oracle.h).  Every function names the
 * reference file:line whose behaviour it restates.
 *   CTR  = pinot-core/src/main/java/org/apache/pinot/core
 *   SEGL = pinot-segment-local/src/main/java/org/apache/pinot/segment/local
 */
#include "pinot_oracle.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define ORC_EOF (-1)                   /* Constants.EOF */
#define MAX_DOC_PER_CALL 10000         /* CTR/plan/DocIdSetPlanNode.java:29 */
#define SCAN_BATCH 256                 /* BlockDocIdIterator.OPTIMAL_ITERATOR_BATCH_SIZE */

static __thread char g_err[512];
const char* orc_last_error(void) { return g_err; }
static void set_err(const char* m) { snprintf(g_err, sizeof g_err, "%s", m); }
void orc_free(void* p) { free(p); }

/* ------------------------------------------------------------------ */
/* big-endian primitive reads (PinotDataBuffer is BIG_ENDIAN)          */
/* ------------------------------------------------------------------ */
static inline uint32_t be32(const uint8_t* p) {
  return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | (uint32_t)p[3];
}
static inline uint64_t be64(const uint8_t* p) { return ((uint64_t)be32(p) << 32) | be32(p + 4); }
static inline float be_f32(const uint8_t* p) { uint32_t u = be32(p); float f; memcpy(&f, &u, 4); return f; }
static inline double be_f64(const uint8_t* p) { uint64_t u = be64(p); double d; memcpy(&d, &u, 8); return d; }

/* SEGL/io/util/PinotDataBitSet.java:61-72 */
int32_t orc_num_bits_per_value(int32_t max_value) {
  if (max_value <= 1) return 1;
  int32_t n = 0;
  uint32_t v = (uint32_t)max_value;
  while (v) { n++; v >>= 1; }
  return n;
}

/* SEGL/io/util/PinotDataBitSet.java:80-102 (readInt): MSB-first big-endian bitstream */
int32_t orc_read_dict_id(const uint8_t* fwd, int32_t bits, int64_t doc) {
  int64_t bit_offset = doc * (int64_t)bits;
  int64_t byte_offset = bit_offset / 8;
  int32_t in_first = (int32_t)(bit_offset % 8);
  int32_t cur = fwd[byte_offset] & (0xff >> in_first);
  int32_t left = bits - (8 - in_first);
  if (left <= 0) return cur >> -left;
  while (left > 8) {
    byte_offset++;
    cur = (cur << 8) | fwd[byte_offset];
    left -= 8;
  }
  return (int32_t)(((uint32_t)cur << left) | (uint32_t)(fwd[byte_offset + 1] >> (8 - left)));
}

/* ------------------------------------------------------------------ */
/* chunk codecs of raw forward indexes                                  */
/* ------------------------------------------------------------------ */
/* LZ4 block format, as lz4-java's safeDecompressor reads it (SEGL/io/compression/LZ4Decompressor.java:41-52; the format is
 * the public "LZ4 Block Format Description"): token = literal length : match length - 4, 15 = more length bytes follow (each
 * adds 0..255, 255 = another one), literals, 2-byte little-endian offset, match copied byte by byte (it may overlap its own
 * output).  The last sequence stops after its literals.  Returns the decoded size, -1 on a malformed stream. */
static int64_t lz4_block_decode(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_cap) {
  int64_t ip = 0, op = 0;
  while (ip < in_len) {
    uint32_t token = in[ip++];
    int64_t lit = token >> 4;
    if (lit == 15) { uint32_t b; do { if (ip >= in_len) return -1; b = in[ip++]; lit += b; } while (b == 255); }
    if (ip + lit > in_len || op + lit > out_cap) return -1;
    memcpy(out + op, in + ip, (size_t)lit); ip += lit; op += lit;
    if (ip >= in_len) break;
    if (ip + 2 > in_len) return -1;
    int64_t off = (int64_t)in[ip] | ((int64_t)in[ip + 1] << 8); ip += 2;
    int64_t ml = token & 15u;
    if (ml == 15) { uint32_t b; do { if (ip >= in_len) return -1; b = in[ip++]; ml += b; } while (b == 255); }
    ml += 4;
    if (off == 0 || off > op || op + ml > out_cap) return -1;
    for (int64_t i = 0; i < ml; i++) out[op + i] = out[op + i - off];
    op += ml;
  }
  return op;
}
/* raw Snappy block, as snappy-java's Snappy.uncompress reads it (SEGL/io/compression/SnappyDecompressor.java; public
 * "Snappy compressed format description"): varint decoded length, then elements tagged in their low two bits --
 * 00 literal (length - 1 in the upper six bits, 60..63 = that many + 1 - 60 length bytes follow), 01 copy with 11-bit offset
 * and length 4..11, 10 / 11 copy with 2- / 4-byte little-endian offset and length 1..64. */
static int64_t snappy_block_decode(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_cap) {
  int64_t ip = 0, op = 0;
  uint64_t want = 0; int sh = 0;
  for (;;) { if (ip >= in_len || sh > 28) return -1; uint32_t b = in[ip++]; want |= (uint64_t)(b & 127u) << sh; sh += 7; if (!(b & 128u)) break; }
  if ((int64_t)want > out_cap) return -1;
  while (ip < in_len) {
    uint32_t tag = in[ip++];
    int64_t len, off;
    if ((tag & 3u) == 0) {
      len = tag >> 2;
      if (len >= 60) { int nb = (int)len - 59; if (ip + nb > in_len) return -1; len = 0; for (int k = 0; k < nb; k++) len |= (int64_t)in[ip + k] << (8 * k); ip += nb; }
      len += 1;
      if (ip + len > in_len || op + len > out_cap) return -1;
      memcpy(out + op, in + ip, (size_t)len); ip += len; op += len;
      continue;
    }
    if ((tag & 3u) == 1) { if (ip + 1 > in_len) return -1; len = 4 + ((tag >> 2) & 7u); off = ((int64_t)(tag >> 5) << 8) | in[ip]; ip += 1; }
    else { int nb = (tag & 3u) == 2 ? 2 : 4; if (ip + nb > in_len) return -1; len = (tag >> 2) + 1; off = 0; for (int k = 0; k < nb; k++) off |= (int64_t)in[ip + k] << (8 * k); ip += nb; }
    if (off == 0 || off > op || op + len > out_cap) return -1;
    for (int64_t i = 0; i < len; i++) out[op + i] = out[op + i - off];
    op += len;
  }
  return op == (int64_t)want ? op : -1;
}
int64_t orc_lz4_block_decode(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_cap) { return lz4_block_decode(in, in_len, out, out_cap); }
int64_t orc_snappy_block_decode(const uint8_t* in, int64_t in_len, uint8_t* out, int64_t out_cap) { return snappy_block_decode(in, in_len, out, out_cap); }

/* BaseChunkForwardIndexReader.decompressChunk for every chunk of a fixed-width single-value raw forward index
 * (SEGL/segment/index/readers/forward/BaseChunkForwardIndexReader.java:61-160, FixedByteChunkSVForwardIndexReader.java):
 * rewrites the index as the equivalent PASS_THROUGH one (same version, same chunking) so that the readers below see
 * plain values.  out == NULL returns the size needed; -1 = malformed / unsupported codec (ZSTANDARD, GZIP). */
int64_t orc_raw_forward_decompress(const uint8_t* b, int64_t len, int32_t width, int32_t num_docs, uint8_t* out, int64_t out_cap) {
  if (len < 16) { set_err("raw forward index header"); return -1; }
  int32_t version = (int32_t)be32(b), num_chunks = (int32_t)be32(b + 4), docs_per_chunk = (int32_t)be32(b + 8);
  int32_t total_docs, codec, data_header_start;
  if (version > 1) { if (len < 28) { set_err("raw forward index header"); return -1; } total_docs = (int32_t)be32(b + 16); codec = (int32_t)be32(b + 20); data_header_start = (int32_t)be32(b + 24); }
  else if (num_docs >= 0) { total_docs = num_docs; codec = 1; data_header_start = 16; }   /* version 1: four header ints, always SNAPPY */
  else { set_err("raw forward index v1 carries no doc count"); return -1; }
  int32_t entry = version <= 2 ? 4 : 8;
  int64_t raw_start = (int64_t)data_header_start + (int64_t)num_chunks * entry;
  int64_t need = 28 + (int64_t)num_chunks * entry + (int64_t)total_docs * width;
  if (!out) return need;
  if (out_cap < need || raw_start > len) { set_err("raw forward index: buffer"); return -1; }
  memcpy(out, b, 16);
  if (version == 1) { out[0] = out[1] = out[2] = 0; out[3] = 2; }   /* the same int offsets as version 2 */
  uint8_t hdr[12] = {0};
  hdr[0] = (uint8_t)(total_docs >> 24); hdr[1] = (uint8_t)(total_docs >> 16); hdr[2] = (uint8_t)(total_docs >> 8); hdr[3] = (uint8_t)total_docs;
  hdr[11] = 28;                                   /* compression 0, dataHeaderStart 28 */
  memcpy(out + 16, hdr, 12);
  int64_t chunk_bytes = (int64_t)docs_per_chunk * width, vals0 = 28 + (int64_t)num_chunks * entry;
  for (int32_t k = 0; k < num_chunks; k++) {
    int64_t o = entry == 4 ? (int64_t)be32(b + data_header_start + 4 * (int64_t)k) : (int64_t)be64(b + data_header_start + 8 * (int64_t)k);
    int64_t e = k + 1 < num_chunks ? (entry == 4 ? (int64_t)be32(b + data_header_start + 4 * (int64_t)(k + 1)) : (int64_t)be64(b + data_header_start + 8 * (int64_t)(k + 1))) : len;
    int64_t left = (int64_t)total_docs * width - (int64_t)k * chunk_bytes;
    int64_t want = left < chunk_bytes ? left : chunk_bytes;
    uint8_t* dst = out + vals0 + (int64_t)k * chunk_bytes;
    int64_t po = vals0 + (int64_t)k * chunk_bytes;
    if (entry == 4) { uint8_t* q = out + 28 + 4 * (int64_t)k; q[0] = (uint8_t)(po >> 24); q[1] = (uint8_t)(po >> 16); q[2] = (uint8_t)(po >> 8); q[3] = (uint8_t)po; }
    else { uint8_t* q = out + 28 + 8 * (int64_t)k; for (int i = 0; i < 8; i++) q[i] = (uint8_t)((uint64_t)po >> (56 - 8 * i)); }
    if (o < raw_start || e > len || e < o) { set_err("raw forward index: chunk offsets"); return -1; }
    int64_t got;
    switch (codec) {
      case 0: if (e - o < want) { set_err("raw forward index: short chunk"); return -1; } memcpy(dst, b + o, (size_t)want); got = want; break;
      case 1: got = snappy_block_decode(b + o, e - o, dst, want); break;
      case 3: got = lz4_block_decode(b + o, e - o, dst, want); break;
      case 4:   /* lz4-java LZ4DecompressorWithLength: little-endian decoded length first */
        if (e - o < 4 || ((int64_t)b[o] | ((int64_t)b[o + 1] << 8) | ((int64_t)b[o + 2] << 16) | ((int64_t)b[o + 3] << 24)) != want) { set_err("raw forward index: LZ4 length prefix"); return -1; }
        got = lz4_block_decode(b + o + 4, e - o - 4, dst, want); break;
      default: set_err("raw forward index: codec not restated (ZSTANDARD / GZIP)"); return -1;
    }
    if (got != want) { set_err("raw forward index: chunk does not decode to its size"); return -1; }
  }
  return need;
}

/* ------------------------------------------------------------------ */
/* column readers                                                      */
/* ------------------------------------------------------------------ */
typedef struct {
  const orc_column* c;
  int32_t num_docs;
  int64_t raw_data_start;   /* raw forward index: offset of the first value */
} col_reader;

/* SEGL/segment/index/readers/forward/BaseChunkForwardIndexReader.java:61-104 */
static int col_reader_init(col_reader* r, const orc_column* c, int32_t num_docs) {
  r->c = c; r->num_docs = num_docs; r->raw_data_start = 0;
  if (!c->has_dictionary) {
    const uint8_t* b = c->forward_index;
    int32_t version = (int32_t)be32(b);
    int32_t num_chunks = (int32_t)be32(b + 4);
    int32_t off = 16;
    int32_t data_header_start = off;
    if (version > 1) {
      int32_t compression = (int32_t)be32(b + off + 4);
      if (compression != 0) { set_err("raw forward index is compressed (only PASS_THROUGH supported)"); return -1; }
      data_header_start = (int32_t)be32(b + off + 8);
    } else { set_err("raw forward index v1 (snappy) unsupported"); return -1; }
    int32_t entry = version <= 2 ? 4 : 8;
    r->raw_data_start = (int64_t)data_header_start + (int64_t)num_chunks * entry;
  }
  return 0;
}

/* SEGL/segment/index/readers/sorted/SortedIndexReaderImpl.java:37-116 */
static inline int32_t sorted_start(const orc_column* c, int32_t dict_id) { return (int32_t)be32(c->forward_index + 8 * (int64_t)dict_id); }
static inline int32_t sorted_end(const orc_column* c, int32_t dict_id) { return (int32_t)be32(c->forward_index + 8 * (int64_t)dict_id + 4); }
static int32_t sorted_dict_id_of_doc(const orc_column* c, int32_t doc) {
  int32_t lo = 0, hi = c->cardinality - 1;
  while (lo < hi) {
    int32_t mid = (lo + hi) >> 1;
    if (sorted_end(c, mid) < doc) lo = mid + 1; else hi = mid;
  }
  return lo;
}

/* dictId of a doc: FixedBitSVForwardIndexReaderV2.readDictIds
 * (SEGL/segment/index/readers/forward/FixedBitSVForwardIndexReaderV2.java:65-99) or sorted index */
static inline int32_t dict_id_of(const col_reader* r, int32_t doc) {
  const orc_column* c = r->c;
  if (c->is_sorted) return sorted_dict_id_of_doc(c, doc);
  /* fast 64-bit window; equal to orc_read_dict_id (checked in tests) */
  int64_t bit = (int64_t)doc * c->bits_per_element;
  int64_t byte = bit >> 3;
  int32_t sh = (int32_t)(bit & 7);
  uint64_t w;
  if (byte + 8 <= c->forward_index_len) w = be64(c->forward_index + byte);
  else {
    uint8_t tmp[8] = {0};
    memcpy(tmp, c->forward_index + byte, (size_t)(c->forward_index_len - byte));
    w = be64(tmp);
  }
  return (int32_t)((w << sh) >> (64 - c->bits_per_element));
}

/* dictionary value reads: SEGL/segment/index/readers/BaseImmutableDictionary.java:45-58,124-139 */
static inline int64_t dict_long(const orc_column* c, int32_t id) {
  return c->data_type == ORC_INT ? (int64_t)(int32_t)be32(c->dictionary + 4 * (int64_t)id)
                                 : (int64_t)be64(c->dictionary + 8 * (int64_t)id);
}
static inline double dict_double(const orc_column* c, int32_t id) {
  switch (c->data_type) {
    case ORC_INT: return (double)(int32_t)be32(c->dictionary + 4 * (int64_t)id);
    case ORC_LONG: return (double)(int64_t)be64(c->dictionary + 8 * (int64_t)id);
    case ORC_FLOAT: return (double)be_f32(c->dictionary + 4 * (int64_t)id);
    default: return be_f64(c->dictionary + 8 * (int64_t)id);
  }
}
static inline int64_t raw_long(const col_reader* r, int32_t doc) {
  const orc_column* c = r->c;
  return c->data_type == ORC_INT ? (int64_t)(int32_t)be32(c->forward_index + r->raw_data_start + 4 * (int64_t)doc)
                                 : (int64_t)be64(c->forward_index + r->raw_data_start + 8 * (int64_t)doc);
}
static inline double raw_double(const col_reader* r, int32_t doc) {
  const orc_column* c = r->c;
  const uint8_t* p = c->forward_index + r->raw_data_start;
  switch (c->data_type) {
    case ORC_INT: return (double)(int32_t)be32(p + 4 * (int64_t)doc);
    case ORC_LONG: return (double)(int64_t)be64(p + 8 * (int64_t)doc);
    case ORC_FLOAT: return (double)be_f32(p + 4 * (int64_t)doc);
    default: return be_f64(p + 8 * (int64_t)doc);
  }
}
/* java.lang.Math.min / max on doubles: NaN if either is NaN; -0.0 < 0.0 */
static inline double java_math_min(double a, double b) {
  if (a != a || b != b) return NAN;
  if (a == 0.0 && b == 0.0) return signbit(a) ? a : b;
  return a < b ? a : b;
}
static inline double java_math_max(double a, double b) {
  if (a != a || b != b) return NAN;
  if (a == 0.0 && b == 0.0) return signbit(a) ? b : a;
  return a > b ? a : b;
}
/* BlockValSet.getDoubleValuesSV for one doc (CTR/common/DataFetcher.java:376-386) */
static inline double value_as_double(const col_reader* r, int32_t doc) {
  return r->c->has_dictionary ? dict_double(r->c, dict_id_of(r, doc)) : raw_double(r, doc);
}

/* Dictionary.insertionIndexOf: Arrays.binarySearch convention
 * (SEGL/segment/index/readers/BaseImmutableDictionary.java:141-260) */
static int32_t dict_insertion_index_long(const orc_column* c, int64_t v) {
  int32_t lo = 0, hi = c->cardinality - 1;
  while (lo <= hi) {
    int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi) >> 1);
    int64_t m = dict_long(c, mid);
    if (m < v) lo = mid + 1; else if (m > v) hi = mid - 1; else return mid;
  }
  return -(lo + 1);
}
static int32_t dict_insertion_index_double(const orc_column* c, double v) {
  /* FloatDictionary.insertionIndexOf: binarySearch(Float.parseFloat(stringValue)) -- the literal is rounded to float first
   * (SEGL/segment/index/readers/FloatDictionary.java:43-45), so "0.1" finds the entry 0.1f */
  if (c->data_type == ORC_FLOAT) v = (double)(float)v;
  int32_t lo = 0, hi = c->cardinality - 1;
  while (lo <= hi) {
    int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi) >> 1);
    double m = c->data_type == ORC_FLOAT ? (double)be_f32(c->dictionary + 4 * (int64_t)mid)
                                         : be_f64(c->dictionary + 8 * (int64_t)mid);
    if (m < v) lo = mid + 1; else if (m > v) hi = mid - 1; else return mid;
  }
  return -(lo + 1);
}
/* STRING dictionary entry `id` as (pointer, length).  Two on-disk forms (BaseImmutableDictionary picks the ValueReader:
 * SEGL/segment/index/readers/BaseImmutableDictionary.java:45-58):
 *   fixed width  FixedByteValueReaderWriter: entries of lengthOfEachEntry bytes, padded with 0
 *   var length   VarLengthValueReader (SEGL/io/util/VarLengthValueReader.java:41-96): magic ".vl;", int version = 1,
 *                int numValues, int dataSectionStartOffset, then numValues + 1 big-endian offsets, then the bytes */
static int dict_is_var_length(const orc_column* c) {
  return c->dictionary_len >= 20 && memcmp(c->dictionary, ".vl;", 4) == 0 && be32(c->dictionary + 4) == 1;
}
static const uint8_t* str_entry(const orc_column* c, int32_t id, int32_t* len) {
  if (dict_is_var_length(c)) {
    const uint32_t data0 = be32(c->dictionary + 12);
    const uint32_t a = be32(c->dictionary + data0 + 4 * (int64_t)id), b = be32(c->dictionary + data0 + 4 * (int64_t)id + 4);
    *len = (int32_t)(b - a);
    return c->dictionary + a;
  }
  const uint8_t* e = c->dictionary + (int64_t)id * c->dict_entry_bytes;
  int32_t n = c->dict_entry_bytes, elen = 0;
  while (elen < n && e[elen] != 0) elen++;
  *len = elen;
  return e;
}
/* String compare against a dictionary entry, in the order the dictionary was sorted in: String.compareTo, i.e. by UTF-16
 * code units (ValueReaderComparisons.compareUtf8Bytes, SEGL/io/util/ValueReaderComparisons.java:68-139: find the first byte
 * that differs, step back to the start of its UTF-8 sequence, decode both sides and compare the UTF-16 units).  Byte order
 * and UTF-16 order differ only between a supplementary character (4-byte UTF-8 = a surrogate pair, 0xD800-0xDFFF) and a BMP
 * character at or above U+E000.  A shorter string that is a prefix sorts first (the padding byte 0 is the smallest unit). */
static void utf16_units_at(const uint8_t* p, int64_t avail, uint32_t* u1, uint32_t* u2) {
  *u1 = 0xfffd; *u2 = 0xfffd;
  if (avail <= 0) { *u1 = 0; return; }
  uint8_t b = p[0];
  if (b < 0x80) *u1 = b;
  else if ((b & 0xF0) < 0xE0) *u1 = ((uint32_t)(b & 0x1F) << 6) | (avail > 1 ? (p[1] & 0x3Fu) : 0);
  else if ((b & 0xF0) == 0xE0) *u1 = ((uint32_t)(b & 0x0F) << 12) | ((avail > 1 ? (p[1] & 0x3Fu) : 0) << 6) | (avail > 2 ? (p[2] & 0x3Fu) : 0);
  else {
    uint32_t cp = ((uint32_t)(b & 0x07) << 18) | ((avail > 1 ? (p[1] & 0x3Fu) : 0) << 12) | ((avail > 2 ? (p[2] & 0x3Fu) : 0) << 6) | (avail > 3 ? (p[3] & 0x3Fu) : 0);
    if (cp >= 0x10000 && cp <= 0x10FFFF) { *u1 = 0xD800 + ((cp - 0x10000) >> 10); *u2 = 0xDC00 + ((cp - 0x10000) & 0x3FF); }
  }
}
static int utf8_cmp_utf16_order(const uint8_t* a, int64_t alen, const uint8_t* b, int64_t blen) {
  int64_t m = alen < blen ? alen : blen, i = 0;
  while (i < m && a[i] == b[i]) i++;
  if (i == m) return (alen > blen) - (alen < blen);
  while (i > 0 && (b[i] & 0xC0) == 0x80) i--;            /* back to the start of the sequence (identical before the mismatch) */
  uint32_t a1, a2, b1, b2;
  utf16_units_at(a + i, alen - i, &a1, &a2);
  utf16_units_at(b + i, blen - i, &b1, &b2);
  if (a1 != b1) return a1 < b1 ? -1 : 1;
  return (a2 > b2) - (a2 < b2);
}
static int str_cmp_entry(const orc_column* c, int32_t id, const char* s) {
  int32_t elen = 0;
  const uint8_t* e = str_entry(c, id, &elen);
  return utf8_cmp_utf16_order(e, elen, (const uint8_t*)s, (int64_t)strlen(s));
}
static int32_t dict_insertion_index_string(const orc_column* c, const char* s) {
  int32_t lo = 0, hi = c->cardinality - 1;
  while (lo <= hi) {
    int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi) >> 1);
    int r = str_cmp_entry(c, mid, s);
    if (r < 0) lo = mid + 1; else if (r > 0) hi = mid - 1; else return mid;
  }
  return -(lo + 1);
}
static int32_t dict_insertion_index(const orc_column* c, const orc_predicate* p, int32_t vi) {
  switch (c->data_type) {
    case ORC_INT: case ORC_LONG: return dict_insertion_index_long(c, p->int_values[vi]);
    case ORC_FLOAT: case ORC_DOUBLE: return dict_insertion_index_double(c, p->double_values[vi]);
    default: return dict_insertion_index_string(c, p->string_values[vi]);
  }
}

/* ------------------------------------------------------------------ */
/* flat doc bitmaps (stand-in for RoaringBitmap set semantics)         */
/* ------------------------------------------------------------------ */
typedef struct { uint64_t* w; int64_t nwords; int32_t num_docs; } bitmap;
static bitmap bm_new(int32_t num_docs) {
  bitmap b; b.num_docs = num_docs; b.nwords = ((int64_t)num_docs + 63) / 64;
  b.w = (uint64_t*)calloc((size_t)(b.nwords > 0 ? b.nwords : 1), 8); return b;
}
static void bm_free(bitmap* b) { free(b->w); b->w = NULL; }
static inline void bm_set(bitmap* b, int32_t d) { b->w[d >> 6] |= 1ull << (d & 63); }
static inline int bm_get(const bitmap* b, int32_t d) { return (int)((b->w[d >> 6] >> (d & 63)) & 1); }
static void bm_set_range(bitmap* b, int32_t lo, int32_t hi_incl) { for (int32_t d = lo; d <= hi_incl; d++) bm_set(b, d); }
static void bm_flip(bitmap* b) {   /* flip(0, numDocs) */
  for (int64_t i = 0; i < b->nwords; i++) b->w[i] = ~b->w[i];
  int32_t tail = b->num_docs & 63;
  if (tail && b->nwords) b->w[b->nwords - 1] &= (1ull << tail) - 1ull;
}
static int64_t bm_card(const bitmap* b) { int64_t n = 0; for (int64_t i = 0; i < b->nwords; i++) n += __builtin_popcountll(b->w[i]); return n; }
static int32_t bm_next(const bitmap* b, int32_t from) {   /* first set bit >= from, or EOF */
  if (from >= b->num_docs) return ORC_EOF;
  int64_t wi = from >> 6;
  uint64_t cur = b->w[wi] & (~0ull << (from & 63));
  while (1) {
    if (cur) { int32_t d = (int32_t)(wi * 64 + __builtin_ctzll(cur)); return d < b->num_docs ? d : ORC_EOF; }
    if (++wi >= b->nwords) return ORC_EOF;
    cur = b->w[wi];
  }
}

/* RoaringBitmap portable format -> docIds (third-party spec, RoaringBitmap 1.3.0; reached through
 * SEGL/segment/index/readers/BitmapInvertedIndexReader.java:45-62) */
static inline uint32_t le16(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8); }
static inline uint32_t le32(const uint8_t* p) { return le16(p) | (le16(p + 2) << 16); }
typedef void (*doc_sink)(void* ctx, uint32_t doc);
static int roaring_for_each(const uint8_t* blob, int64_t len, doc_sink sink, void* ctx) {
  if (len < 4) return -1;
  uint32_t cookie = le32(blob);
  int64_t p;
  uint32_t n;
  const uint8_t* run_bitmap = NULL;
  int has_offsets;
  if ((cookie & 0xffff) == 12347u) {
    n = (cookie >> 16) + 1;
    run_bitmap = blob + 4;
    p = 4 + (n + 7) / 8;
    has_offsets = n >= 4;
  } else if (cookie == 12346u) {
    n = le32(blob + 4);
    p = 8;
    has_offsets = 1;
  } else return -1;
  const uint8_t* hdr = blob + p;
  p += 4 * (int64_t)n;
  if (has_offsets) p += 4 * (int64_t)n;
  for (uint32_t c = 0; c < n; c++) {
    uint32_t key = le16(hdr + 4 * c);
    uint32_t card = le16(hdr + 4 * c + 2) + 1;
    int is_run = run_bitmap && ((run_bitmap[c / 8] >> (c % 8)) & 1);
    uint32_t base = key << 16;
    if (is_run) {
      uint32_t nr = le16(blob + p); p += 2;
      for (uint32_t r = 0; r < nr; r++) {
        uint32_t s = le16(blob + p), l = le16(blob + p + 2); p += 4;
        for (uint32_t k = 0; k <= l; k++) sink(ctx, base | (s + k));
      }
    } else if (card <= 4096) {
      for (uint32_t k = 0; k < card; k++) { sink(ctx, base | le16(blob + p)); p += 2; }
    } else {
      for (uint32_t wv = 0; wv < 1024; wv++) {
        uint64_t word = (uint64_t)le32(blob + p) | ((uint64_t)le32(blob + p + 4) << 32); p += 8;
        while (word) { int b = __builtin_ctzll(word); sink(ctx, base | (wv * 64 + (uint32_t)b)); word &= word - 1; }
      }
    }
    if (p > len) return -1;
  }
  return 0;
}
typedef struct { uint32_t* out; int64_t n, cap; } list_ctx;
static void list_sink(void* ctx, uint32_t d) { list_ctx* l = (list_ctx*)ctx; if (l->n < l->cap) l->out[l->n] = d; l->n++; }
int64_t orc_roaring_to_doc_ids(const uint8_t* blob, int64_t len, uint32_t* out, int64_t cap) {
  list_ctx l = {out, 0, cap};
  if (roaring_for_each(blob, len, list_sink, &l) != 0) return -1;
  return l.n;
}
static void bm_sink(void* ctx, uint32_t d) { bitmap* b = (bitmap*)ctx; if ((int32_t)d < b->num_docs) bm_set(b, (int32_t)d); }
/* BitmapInvertedIndexReader.getDocIds(dictId): offsets are big-endian, relative to the first one */
static int inverted_or_into(const orc_column* c, int32_t dict_id, bitmap* b) {
  const uint8_t* inv = c->inverted_index;
  uint32_t first = be32(inv);
  uint32_t s = be32(inv + 4 * (int64_t)dict_id), e = be32(inv + 4 * (int64_t)dict_id + 4);
  int64_t base = 4 * ((int64_t)c->cardinality + 1);
  return roaring_for_each(inv + base + (s - first), (int64_t)(e - s), bm_sink, b);
}

/* ------------------------------------------------------------------ */
/* predicate evaluators                                                */
/* ------------------------------------------------------------------ */
typedef struct {
  const orc_predicate* p;
  const orc_column* c;
  col_reader reader;
  int dict_based;
  int always_true, always_false;
  int exclusive;            /* NEQ / NOT_IN */
  int is_range;
  int32_t start_dict_id, end_dict_id;   /* sorted-dictionary RANGE: [start, end) */
  int32_t* dict_ids; int32_t n_dict_ids;  /* EQ/IN: matching ids; NEQ/NOT_IN: non-matching ids (sorted) */
  uint8_t* dict_member;     /* membership over the dictionary for dict_ids */
  /* raw-value evaluators */
  int64_t ilo, ihi;         /* inclusive bounds (INT/LONG) */
  double dlo, dhi; int dlo_incl, dhi_incl;
} pred_eval;

static int cmp_i32(const void* a, const void* b) { int32_t x = *(const int32_t*)a, y = *(const int32_t*)b; return (x > y) - (x < y); }

/* CTR/operator/filter/predicate/PredicateEvaluatorProvider.java:45-95 and the per-type factories:
 * RangePredicateEvaluatorFactory.java:119-169 (sorted dictionary range), :326-400 (raw ranges, bounds
 * made inclusive :334-345); EqualsPredicateEvaluatorFactory.java:83-110; NotEqualsPredicateEvaluatorFactory.java:83-110;
 * InPredicateEvaluatorFactory.java:158-188; NotInPredicateEvaluatorFactory.java:155-172 */
static int pred_eval_init(pred_eval* e, const orc_segment* seg, const orc_predicate* p) {
  memset(e, 0, sizeof *e);
  e->p = p; e->c = &seg->columns[p->column];
  const orc_column* c = e->c;
  if (col_reader_init(&e->reader, c, seg->num_docs) != 0) return -1;
  e->dict_based = c->has_dictionary;
  e->exclusive = (p->type == ORC_NEQ || p->type == ORC_NOT_IN);
  e->is_range = (p->type == ORC_RANGE);
  if (c->has_dictionary) {
    int32_t card = c->cardinality;
    if (p->type == ORC_RANGE) {
      if (p->lower_unbounded) e->start_dict_id = 0;
      else {
        int32_t ii = dict_insertion_index(c, p, 0);
        e->start_dict_id = ii < 0 ? -(ii + 1) : (p->lower_inclusive ? ii : ii + 1);
      }
      if (p->upper_unbounded) e->end_dict_id = card;
      else {
        int32_t ii = dict_insertion_index(c, p, 1);
        e->end_dict_id = ii < 0 ? -(ii + 1) : (p->upper_inclusive ? ii + 1 : ii);
      }
      int32_t nm = e->end_dict_id - e->start_dict_id; if (nm < 0) nm = 0;
      if (nm == 0) e->always_false = 1; else if (nm == card) e->always_true = 1;
    } else {
      e->dict_ids = (int32_t*)malloc(sizeof(int32_t) * (size_t)(p->num_values > 0 ? p->num_values : 1));
      e->dict_member = (uint8_t*)calloc((size_t)card + 1, 1);
      for (int32_t i = 0; i < p->num_values; i++) {
        int32_t id = dict_insertion_index(c, p, i);     /* Dictionary.indexOf */
        if (id >= 0 && !e->dict_member[id]) { e->dict_member[id] = 1; e->dict_ids[e->n_dict_ids++] = id; }
      }
      qsort(e->dict_ids, (size_t)e->n_dict_ids, sizeof(int32_t), cmp_i32);
      if (!e->exclusive) { if (e->n_dict_ids == 0) e->always_false = 1; else if (e->n_dict_ids == card) e->always_true = 1; }
      else { if (e->n_dict_ids == 0) e->always_true = 1; else if (e->n_dict_ids == card) e->always_false = 1; }
    }
  } else {
    if (c->data_type == ORC_STRING) { set_err("raw STRING predicate unsupported"); return -1; }
    int is_int = (c->data_type == ORC_INT || c->data_type == ORC_LONG);
    if (p->type == ORC_RANGE) {
      if (is_int) {
        int64_t tmin = c->data_type == ORC_INT ? INT32_MIN : INT64_MIN;
        int64_t tmax = c->data_type == ORC_INT ? INT32_MAX : INT64_MAX;
        if (p->lower_unbounded) e->ilo = tmin;
        else { e->ilo = p->int_values[0]; if (!p->lower_inclusive) { if (e->ilo == tmax) e->always_false = 1; else e->ilo++; } }
        if (p->upper_unbounded) e->ihi = tmax;
        else { e->ihi = p->int_values[1]; if (!p->upper_inclusive) { if (e->ihi == tmin) e->always_false = 1; else e->ihi--; } }
        if (e->ilo > e->ihi) e->always_false = 1;
      } else {
        e->dlo = p->lower_unbounded ? -INFINITY : p->double_values[0];
        e->dhi = p->upper_unbounded ? INFINITY : p->double_values[1];
        /* FloatRawValueBasedRangePredicateEvaluator holds Float.parseFloat(bound) (RangePredicateEvaluatorFactory.java) */
        if (c->data_type == ORC_FLOAT) { e->dlo = (double)(float)e->dlo; e->dhi = (double)(float)e->dhi; }
        e->dlo_incl = p->lower_unbounded || p->lower_inclusive;
        e->dhi_incl = p->upper_unbounded || p->upper_inclusive;
      }
    }
  }
  return 0;
}
static void pred_eval_free(pred_eval* e) { free(e->dict_ids); free(e->dict_member); }

/* PredicateEvaluator.applySV(dictId) / applySV(value) */
static inline int pred_match_dict_id(const pred_eval* e, int32_t id) {
  if (e->is_range) return e->start_dict_id <= id && e->end_dict_id > id;
  return e->exclusive ? !e->dict_member[id] : e->dict_member[id];
}
static int pred_match_doc(const pred_eval* e, int32_t doc) {
  if (e->dict_based) return pred_match_dict_id(e, dict_id_of(&e->reader, doc));
  const orc_column* c = e->c; const orc_predicate* p = e->p;
  if (c->data_type == ORC_INT || c->data_type == ORC_LONG) {
    int64_t v = raw_long(&e->reader, doc);
    if (e->is_range) return v >= e->ilo && v <= e->ihi;
    int found = 0;
    for (int32_t i = 0; i < p->num_values; i++) if (p->int_values[i] == v) { found = 1; break; }
    return e->exclusive ? !found : found;
  } else {
    double v = raw_double(&e->reader, doc);
    if (e->is_range) {
      int lo_ok = e->dlo_incl ? v >= e->dlo : v > e->dlo;
      int hi_ok = e->dhi_incl ? v <= e->dhi : v < e->dhi;
      return lo_ok && hi_ok;
    }
    /* EQ / NOT_EQ compare with == / != (EqualsPredicateEvaluatorFactory.java:336-337, NotEqualsPredicateEvaluatorFactory.java:
     * 298-299: 0.0 equals -0.0, NaN equals nothing); IN / NOT_IN ask a fastutil DoubleSet / FloatSet, which compares
     * Double.doubleToLongBits (InPredicateEvaluatorFactory.java:341-362: -0.0 is not in {0.0}; every NaN is the canonical NaN) */
    const int by_bits = p->type == ORC_IN || p->type == ORC_NOT_IN;
    int found = 0;
    for (int32_t i = 0; i < p->num_values; i++) {
      double q = c->data_type == ORC_FLOAT ? (double)(float)p->double_values[i] : p->double_values[i];
      if (by_bits) {
        uint64_t a, b; memcpy(&a, &q, 8); memcpy(&b, &v, 8);
        if (q != q) a = 0x7ff8000000000000ull;
        if (v != v) b = 0x7ff8000000000000ull;
        if (a == b) { found = 1; break; }
      } else if (q == v) { found = 1; break; }
    }
    return e->exclusive ? !found : found;
  }
}

/* ------------------------------------------------------------------ */
/* filter operators and docId iterators                                */
/* ------------------------------------------------------------------ */
enum { OP_EMPTY, OP_MATCH_ALL, OP_SORTED, OP_BITMAP, OP_SCAN, OP_AND, OP_OR, OP_NOT };
typedef struct { int32_t lo, hi; } irange;   /* inclusive */

typedef struct fop {
  int kind;
  int32_t num_docs;
  /* OP_SORTED */ irange* ranges; int32_t n_ranges;
  /* OP_BITMAP */ bitmap bm;
  /* OP_SCAN   */ pred_eval* ev;
  /* AND/OR/NOT */ struct fop** kids; int32_t n_kids;
} fop;

static fop* fop_new(int kind, int32_t num_docs) { fop* f = (fop*)calloc(1, sizeof(fop)); f->kind = kind; f->num_docs = num_docs; return f; }
static void fop_free(fop* f) {
  if (!f) return;
  for (int32_t i = 0; i < f->n_kids; i++) fop_free(f->kids[i]);
  free(f->kids); free(f->ranges);
  if (f->kind == OP_BITMAP) bm_free(&f->bm);
  if (f->ev) { pred_eval_free(f->ev); free(f->ev); }
  free(f);
}

/* CTR/operator/filter/SortedIndexBasedFilterOperator.java:53-131 */
static fop* make_sorted_op(pred_eval* e, int32_t num_docs) {
  const orc_column* c = e->c;
  fop* f = fop_new(OP_SORTED, num_docs);
  if (e->is_range) {
    f->ranges = (irange*)malloc(sizeof(irange)); f->n_ranges = 1;
    f->ranges[0].lo = sorted_start(c, e->start_dict_id);
    f->ranges[0].hi = sorted_end(c, e->end_dict_id - 1);
    return f;
  }
  int32_t n = e->n_dict_ids;
  irange* r = (irange*)malloc(sizeof(irange) * (size_t)(n + 2));
  int32_t nr = 0;
  irange last = { sorted_start(c, e->dict_ids[0]), sorted_end(c, e->dict_ids[0]) };
  for (int32_t i = 1; i < n; i++) {
    irange cur = { sorted_start(c, e->dict_ids[i]), sorted_end(c, e->dict_ids[i]) };
    if (cur.lo == last.hi + 1) last.hi = cur.hi; else { r[nr++] = last; last = cur; }
  }
  r[nr++] = last;
  if (e->exclusive) {
    irange* inv = (irange*)malloc(sizeof(irange) * (size_t)(nr + 2));
    int32_t ni = 0;
    if (r[0].lo > 0) { inv[ni].lo = 0; inv[ni].hi = r[0].lo - 1; ni++; }
    for (int32_t i = 0; i + 1 < nr; i++) { inv[ni].lo = r[i].hi + 1; inv[ni].hi = r[i + 1].lo - 1; ni++; }
    if (r[nr - 1].hi < num_docs - 1) { inv[ni].lo = r[nr - 1].hi + 1; inv[ni].hi = num_docs - 1; ni++; }
    free(r); r = inv; nr = ni;
  }
  f->ranges = r; f->n_ranges = nr;
  return f;
}

/* CTR/operator/filter/InvertedIndexFilterOperator.java:60-96 */
static fop* make_inverted_op(pred_eval* e, int32_t num_docs) {
  if (e->n_dict_ids == 0) return fop_new(OP_EMPTY, num_docs);
  fop* f = fop_new(OP_BITMAP, num_docs);
  f->bm = bm_new(num_docs);
  for (int32_t i = 0; i < e->n_dict_ids; i++) inverted_or_into(e->c, e->dict_ids[i], &f->bm);
  if (e->exclusive) bm_flip(&f->bm);
  return f;
}

/* CTR/operator/filter/FilterOperatorUtils.java:74-133 (index selection) */
static fop* make_leaf_op(const orc_segment* seg, const orc_query* q, const orc_predicate* p) {
  /* FilterPlanNode.java:294-307: IS NULL / IS NOT NULL are a BitmapBasedFilterOperator over the column's null-value vector
   * (NullValueVectorReaderImpl: one RoaringBitmap of the null docIds; BitmapBasedFilterOperator.java:35-47 flips it over
   * [0, numDocs) when exclusive); without a vector IS NULL is empty and IS NOT NULL matches all */
  if (p->type == ORC_IS_NULL || p->type == ORC_IS_NOT_NULL) {
    const orc_column* nc = &seg->columns[p->column];
    if (!nc->null_value_vector) return fop_new(p->type == ORC_IS_NULL ? OP_EMPTY : OP_MATCH_ALL, seg->num_docs);
    fop* f = fop_new(OP_BITMAP, seg->num_docs);
    f->bm = bm_new(seg->num_docs);
    if (roaring_for_each(nc->null_value_vector, nc->null_value_vector_len, bm_sink, &f->bm) != 0) { set_err("malformed null-value vector"); fop_free(f); return NULL; }
    if (p->type == ORC_IS_NOT_NULL) bm_flip(&f->bm);
    return f;
  }
  pred_eval* e = (pred_eval*)malloc(sizeof(pred_eval));
  if (pred_eval_init(e, seg, p) != 0) { free(e); return NULL; }
  int32_t n = seg->num_docs;
  fop* f;
  if (e->always_false) f = fop_new(OP_EMPTY, n);
  else if (e->always_true) f = fop_new(OP_MATCH_ALL, n);
  else if (e->c->is_sorted && e->c->has_dictionary) f = make_sorted_op(e, n);
  else if (p->type != ORC_RANGE && e->c->inverted_index != NULL && !q->skip_inverted_index) f = make_inverted_op(e, n);
  else { f = fop_new(OP_SCAN, n); f->ev = e; return f; }
  pred_eval_free(e); free(e);
  return f;
}

static int fop_priority(const fop* f) {   /* FilterOperatorUtils.java:205-252 */
  switch (f->kind) {
    case OP_SORTED: return 0;
    case OP_BITMAP: return 100;
    case OP_AND: return 300;
    case OP_OR: return 400;
    case OP_NOT: return fop_priority(f->kids[0]);
    case OP_SCAN: return 500;
    default: return 10000;
  }
}

/* FilterOperatorUtils.java:136-195 */
static fop* make_and_op(fop** kids, int32_t n, int32_t num_docs) {
  fop** keep = (fop**)malloc(sizeof(fop*) * (size_t)(n > 0 ? n : 1));
  int32_t nk = 0;
  for (int32_t i = 0; i < n; i++) {
    if (kids[i]->kind == OP_EMPTY) {
      for (int32_t j = 0; j < n; j++) fop_free(kids[j]);
      free(keep); return fop_new(OP_EMPTY, num_docs);
    }
  }
  for (int32_t i = 0; i < n; i++) { if (kids[i]->kind == OP_MATCH_ALL) fop_free(kids[i]); else keep[nk++] = kids[i]; }
  if (nk == 0) { free(keep); return fop_new(OP_MATCH_ALL, num_docs); }
  if (nk == 1) { fop* r = keep[0]; free(keep); return r; }
  /* stable sort by priority (List.sort is a stable merge sort) */
  for (int32_t i = 1; i < nk; i++) {
    fop* x = keep[i]; int px = fop_priority(x); int32_t j = i - 1;
    while (j >= 0 && fop_priority(keep[j]) > px) { keep[j + 1] = keep[j]; j--; }
    keep[j + 1] = x;
  }
  fop* f = fop_new(OP_AND, num_docs); f->kids = keep; f->n_kids = nk; return f;
}
static fop* make_or_op(fop** kids, int32_t n, int32_t num_docs) {
  fop** keep = (fop**)malloc(sizeof(fop*) * (size_t)(n > 0 ? n : 1));
  int32_t nk = 0;
  for (int32_t i = 0; i < n; i++) {
    if (kids[i]->kind == OP_MATCH_ALL) {
      for (int32_t j = 0; j < n; j++) fop_free(kids[j]);
      free(keep); return fop_new(OP_MATCH_ALL, num_docs);
    }
  }
  for (int32_t i = 0; i < n; i++) { if (kids[i]->kind == OP_EMPTY) fop_free(kids[i]); else keep[nk++] = kids[i]; }
  if (nk == 0) { free(keep); return fop_new(OP_EMPTY, num_docs); }
  if (nk == 1) { fop* r = keep[0]; free(keep); return r; }
  fop* f = fop_new(OP_OR, num_docs); f->kids = keep; f->n_kids = nk; return f;
}
static fop* make_not_op(fop* kid, int32_t num_docs) {
  if (kid->kind == OP_MATCH_ALL) { fop_free(kid); return fop_new(OP_EMPTY, num_docs); }
  if (kid->kind == OP_EMPTY) { fop_free(kid); return fop_new(OP_MATCH_ALL, num_docs); }
  fop* f = fop_new(OP_NOT, num_docs); f->kids = (fop**)malloc(sizeof(fop*)); f->kids[0] = kid; f->n_kids = 1; return f;
}

/* CTR/plan/FilterPlanNode.java:195-320 (constructPhysicalOperator) from the postfix tree */
/* ---- enableNullHandling: three-valued filters.  The operator tree is the same; what changes is how its doc sets are
 * taken: BaseFilterOperator.getTrues() / getNulls() / getFalses() (CTR/operator/filter/BaseFilterOperator.java:88-113).
 *   column leaf (BaseColumnFilterOperator.java:46-70)  trues = matches AND NOT nulls; nulls = the null-value vector
 *   IS [NOT] NULL (BitmapBasedFilterOperator), Empty, MatchAll: no nulls; falses = NOT trues
 *   AND (AndFilterOperator.java:52-88)  trues = AND trues_i;  falses = NOT AND_i (trues_i OR nulls_i)
 *   OR  (OrFilterOperator.java:51-87)   trues = OR trues_i;   falses = NOT OR_i (trues_i OR nulls_i)
 *   NOT (NotFilterOperator.java:52-63)  trues = falses of the child; falses = its trues
 * nulls_i is taken from DIRECT column-leaf children only (And / Or / Not do not override getNulls()).  The filter of the
 * query is the trues of the root.  Built here as an ordinary two-valued operator tree over the same leaves. ---- */
typedef struct nexpr { int kind; int pred; int32_t n; struct nexpr** kids; } nexpr;
static void nexpr_free(nexpr* e) { if (!e) return; for (int32_t i = 0; i < e->n; i++) nexpr_free(e->kids[i]); free(e->kids); free(e); }
static fop* null_bitmap_op(const orc_segment* seg, int32_t column, int not_null) {
  const orc_column* nc = &seg->columns[column];
  if (!nc->null_value_vector) return NULL;
  fop* f = fop_new(OP_BITMAP, seg->num_docs);
  f->bm = bm_new(seg->num_docs);
  if (roaring_for_each(nc->null_value_vector, nc->null_value_vector_len, bm_sink, &f->bm) != 0) { set_err("malformed null-value vector"); fop_free(f); return NULL; }
  if (not_null) bm_flip(&f->bm);
  return f;
}
static fop* nh_trues(const orc_segment* seg, const orc_query* q, const nexpr* e);
/* nulls of a node: non-NULL only for a column leaf whose column has a (non-empty) null-value vector and whose own operator is
 * neither Empty nor MatchAll (those are EmptyFilterOperator / MatchAllFilterOperator, not column operators) */
static fop* nh_nulls(const orc_segment* seg, const orc_query* q, const nexpr* e) {
  if (e->kind != ORC_PRED) return NULL;
  const orc_predicate* p = &q->predicates[e->pred];
  if (p->type == ORC_IS_NULL || p->type == ORC_IS_NOT_NULL) return NULL;
  if (!seg->columns[p->column].null_value_vector) return NULL;
  fop* base = make_leaf_op(seg, q, p);
  if (!base) return NULL;
  int trivial = base->kind == OP_EMPTY || base->kind == OP_MATCH_ALL;
  fop_free(base);
  return trivial ? NULL : null_bitmap_op(seg, p->column, 0);
}
/* trues_i OR nulls_i of one child, as And / OrFilterOperator.getFalses() collect them */
static fop* nh_trues_or_nulls(const orc_segment* seg, const orc_query* q, const nexpr* e) {
  fop* t = nh_trues(seg, q, e);
  if (!t) return NULL;
  fop* nl = nh_nulls(seg, q, e);
  if (!nl) return t;
  fop* kids[2] = { t, nl };
  return make_or_op(kids, 2, seg->num_docs);
}
static fop* nh_falses(const orc_segment* seg, const orc_query* q, const nexpr* e) {
  const int32_t n = seg->num_docs;
  if (e->kind == ORC_NOT) return nh_trues(seg, q, e->kids[0]);
  if (e->kind == ORC_PRED) {   /* BaseFilterOperator.getFalses: NOT (trues OR nulls) */
    fop* x = nh_trues_or_nulls(seg, q, e);
    return x ? make_not_op(x, n) : NULL;
  }
  fop** kids = (fop**)malloc(sizeof(fop*) * (size_t)e->n);
  for (int32_t i = 0; i < e->n; i++) {
    kids[i] = nh_trues_or_nulls(seg, q, e->kids[i]);
    if (!kids[i]) { for (int32_t j = 0; j < i; j++) fop_free(kids[j]); free(kids); return NULL; }
  }
  fop* inner = e->kind == ORC_AND ? make_and_op(kids, e->n, n) : make_or_op(kids, e->n, n);
  free(kids);
  return make_not_op(inner, n);
}
static fop* nh_trues(const orc_segment* seg, const orc_query* q, const nexpr* e) {
  const int32_t n = seg->num_docs;
  if (e->kind == ORC_NOT) return nh_falses(seg, q, e->kids[0]);
  if (e->kind == ORC_PRED) {
    const orc_predicate* p = &q->predicates[e->pred];
    fop* base = make_leaf_op(seg, q, p);
    if (!base || p->type == ORC_IS_NULL || p->type == ORC_IS_NOT_NULL || base->kind == OP_EMPTY) return base;
    if (base->kind == OP_MATCH_ALL) {
      /* FilterOperatorUtils.java:78-88: an always-true predicate on a column with nulls is a BitmapBasedFilterOperator over
       * the flipped null bitmap (which, not being a column operator, reports no nulls of its own) */
      fop* nn0 = seg->columns[p->column].null_value_vector ? null_bitmap_op(seg, p->column, 1) : NULL;
      if (!nn0) return base;
      fop_free(base);
      return nn0;
    }
    fop* nn = seg->columns[p->column].null_value_vector ? null_bitmap_op(seg, p->column, 1) : NULL;
    if (!nn) return base;
    fop* kids[2] = { base, nn };                       /* excludeNulls: AND(matches, flip(nullBitmap)) */
    return make_and_op(kids, 2, n);
  }
  fop** kids = (fop**)malloc(sizeof(fop*) * (size_t)e->n);
  for (int32_t i = 0; i < e->n; i++) {
    kids[i] = nh_trues(seg, q, e->kids[i]);
    if (!kids[i]) { for (int32_t j = 0; j < i; j++) fop_free(kids[j]); free(kids); return NULL; }
  }
  fop* f = e->kind == ORC_AND ? make_and_op(kids, e->n, n) : make_or_op(kids, e->n, n);
  free(kids);
  return f;
}
static fop* build_filter_null_handling(const orc_segment* seg, const orc_query* q) {
  nexpr** stack = (nexpr**)calloc((size_t)q->num_filter_nodes, sizeof(nexpr*));
  int32_t sp = 0;
  for (int32_t i = 0; i < q->num_filter_nodes; i++) {
    const orc_filter_node* nd = &q->filter_nodes[i];
    nexpr* e = (nexpr*)calloc(1, sizeof(nexpr));
    e->kind = nd->kind; e->pred = nd->predicate;
    int32_t k = nd->kind == ORC_PRED ? 0 : nd->kind == ORC_NOT ? 1 : nd->n_children;
    e->n = k; e->kids = (nexpr**)malloc(sizeof(nexpr*) * (size_t)(k > 0 ? k : 1));
    for (int32_t j = 0; j < k; j++) e->kids[j] = stack[sp - k + j];
    sp -= k; stack[sp++] = e;
  }
  nexpr* root = stack[0];
  free(stack);
  fop* f = nh_trues(seg, q, root);
  nexpr_free(root);
  return f;
}

static fop* build_filter(const orc_segment* seg, const orc_query* q) {
  int32_t n = seg->num_docs;
  if (q->num_filter_nodes == 0) return fop_new(OP_MATCH_ALL, n);
  if (q->null_handling) return build_filter_null_handling(seg, q);
  fop** stack = (fop**)malloc(sizeof(fop*) * (size_t)q->num_filter_nodes);
  int32_t sp = 0;
  for (int32_t i = 0; i < q->num_filter_nodes; i++) {
    const orc_filter_node* nd = &q->filter_nodes[i];
    if (nd->kind == ORC_PRED) {
      fop* f = make_leaf_op(seg, q, &q->predicates[nd->predicate]);
      if (!f) { for (int32_t j = 0; j < sp; j++) fop_free(stack[j]); free(stack); return NULL; }
      stack[sp++] = f;
    } else if (nd->kind == ORC_NOT) {
      stack[sp - 1] = make_not_op(stack[sp - 1], n);
    } else {
      int32_t k = nd->n_children;
      fop* f = nd->kind == ORC_AND ? make_and_op(&stack[sp - k], k, n) : make_or_op(&stack[sp - k], k, n);
      sp -= k; stack[sp++] = f;
    }
  }
  fop* root = stack[0];
  free(stack);
  return root;
}

/* ---- iterators (CTR/operator/dociditerators) ---- */
enum { IT_EMPTY, IT_MATCH_ALL, IT_SORTED, IT_BITMAP, IT_SCAN, IT_AND, IT_OR, IT_NOT };
typedef struct dit {
  int kind;
  int32_t num_docs;
  int32_t next_doc;                       /* MATCH_ALL, SORTED, BITMAP, AND, NOT */
  const irange* ranges; int32_t n_ranges; int32_t cur_range;     /* SORTED */
  bitmap* bm; int owns_bm;                /* BITMAP */
  const pred_eval* ev;                    /* SCAN */
  int32_t batch[SCAN_BATCH]; int32_t first_mismatch, cursor; int64_t entries;   /* SCAN */
  struct dit** kids; int32_t n_kids;      /* AND / OR / NOT */
  int32_t* next_ids; int32_t n_live; int32_t prev_doc;          /* OR */
  int32_t next_non_matching;              /* NOT */
} dit;

static int32_t dit_next(dit* it);
static int32_t dit_advance(dit* it, int32_t target);

static dit* dit_new(int kind, int32_t num_docs) { dit* d = (dit*)calloc(1, sizeof(dit)); d->kind = kind; d->num_docs = num_docs; return d; }
static void dit_free(dit* d) {
  if (!d) return;
  for (int32_t i = 0; i < d->n_kids; i++) dit_free(d->kids[i]);
  free(d->kids); free(d->next_ids);
  if (d->owns_bm && d->bm) { bm_free(d->bm); free(d->bm); }
  free(d);
}
static int64_t dit_entries(const dit* d) {
  int64_t n = d->kind == IT_SCAN ? d->entries : 0;
  for (int32_t i = 0; i < d->n_kids; i++) n += dit_entries(d->kids[i]);
  return n;
}

/* SVScanDocIdIterator.java:76-98 (next), :101-113 (advance) */
static int32_t scan_next(dit* it) {
  if (it->cursor >= it->first_mismatch) {
    int32_t limit, bs = 0;
    do {
      limit = it->num_docs - it->next_doc; if (limit > SCAN_BATCH) limit = SCAN_BATCH;
      if (limit > 0) {
        bs = 0;
        for (int32_t i = 0; i < limit; i++) if (pred_match_doc(it->ev, it->next_doc + i)) it->batch[bs++] = it->next_doc + i;
        it->next_doc += limit;
        it->entries += limit;
      }
    } while (limit > 0 && bs == 0);
    it->first_mismatch = bs; it->cursor = 0;
    if (bs == 0) return ORC_EOF;
  }
  return it->batch[it->cursor++];
}
static int32_t scan_advance(dit* it, int32_t target) {
  it->next_doc = target; it->first_mismatch = 0;
  while (it->next_doc < it->num_docs) {
    int32_t d = it->next_doc++;
    it->entries++;
    if (pred_match_doc(it->ev, d)) return d;
  }
  return ORC_EOF;
}
/* SortedDocIdIterator */
static int32_t sorted_next(dit* it) {
  while (it->cur_range < it->n_ranges) {
    const irange* r = &it->ranges[it->cur_range];
    if (it->next_doc < r->lo) it->next_doc = r->lo;
    if (it->next_doc <= r->hi) return it->next_doc++;
    it->cur_range++;
  }
  return ORC_EOF;
}
/* AndDocIdIterator.java:40-68 */
static int32_t and_next(dit* it) {
  int32_t max_doc = it->next_doc, max_idx = -1, idx = 0;
  while (idx < it->n_kids) {
    if (idx == max_idx) { idx++; continue; }
    int32_t d = dit_advance(it->kids[idx], max_doc);
    if (d == ORC_EOF) return ORC_EOF;
    if (d == max_doc) idx++; else { max_doc = d; max_idx = idx; idx = 0; }
  }
  it->next_doc = max_doc;
  return it->next_doc++;
}
/* OrDocIdIterator.java:51-117 */
static void or_remove_exhausted(dit* it) {
  int32_t i = 0;
  while (i < it->n_live) {
    if (it->next_ids[i] == ORC_EOF) {
      it->n_live--;
      dit* t = it->kids[i]; it->kids[i] = it->kids[it->n_live]; it->kids[it->n_live] = t;
      it->next_ids[i] = it->next_ids[it->n_live];
    } else i++;
  }
}
static int32_t or_step(dit* it, int use_target, int32_t target) {
  int32_t best = INT32_MAX; int exhausted = 0;
  for (int32_t i = 0; i < it->n_live; i++) {
    int32_t d = it->next_ids[i];
    if (use_target ? (d < target) : (d == it->prev_doc)) {
      d = use_target ? dit_advance(it->kids[i], target) : dit_next(it->kids[i]);
      it->next_ids[i] = d;
      if (d == ORC_EOF) { exhausted = 1; continue; }
    }
    if (d < best) best = d;
  }
  if (exhausted) or_remove_exhausted(it);
  if (best != INT32_MAX) { it->prev_doc = best; return best; }
  return ORC_EOF;
}
/* NotDocIdIterator.java:30-75 */
static int32_t not_next(dit* it) {
  if (it->next_doc >= it->num_docs) return ORC_EOF;
  while (it->next_doc == it->next_non_matching) {
    it->next_doc++;
    int32_t n = dit_next(it->kids[0]);
    it->next_non_matching = n == ORC_EOF ? it->num_docs : n;
  }
  if (it->next_doc >= it->num_docs) return ORC_EOF;
  return it->next_doc++;
}

static int32_t dit_next(dit* it) {
  switch (it->kind) {
    case IT_EMPTY: return ORC_EOF;
    case IT_MATCH_ALL: return it->next_doc < it->num_docs ? it->next_doc++ : ORC_EOF;
    case IT_SORTED: return sorted_next(it);
    case IT_BITMAP: { int32_t d = bm_next(it->bm, it->next_doc); if (d == ORC_EOF) { it->next_doc = it->num_docs; return ORC_EOF; } it->next_doc = d + 1; return d; }
    case IT_SCAN: return scan_next(it);
    case IT_AND: return and_next(it);
    case IT_OR: return or_step(it, 0, 0);
    default: return not_next(it);
  }
}
static int32_t dit_advance(dit* it, int32_t target) {
  switch (it->kind) {
    case IT_EMPTY: return ORC_EOF;
    case IT_MATCH_ALL: it->next_doc = target; return dit_next(it);
    case IT_SORTED:
      /* SortedDocIdIterator.advance: move to the range containing / following target */
      while (it->cur_range < it->n_ranges && it->ranges[it->cur_range].hi < target) it->cur_range++;
      if (target > it->next_doc) it->next_doc = target;
      return sorted_next(it);
    case IT_BITMAP: it->next_doc = target; return dit_next(it);
    case IT_SCAN: return scan_advance(it, target);
    case IT_AND: it->next_doc = target; return and_next(it);
    case IT_OR: return or_step(it, 1, target);
    default:
      it->next_doc = target;
      if (target > it->next_non_matching) {
        int32_t n = dit_advance(it->kids[0], target);
        it->next_non_matching = n == ORC_EOF ? it->num_docs : n;
      }
      return not_next(it);
  }
}

static dit* make_iterator(fop* f, int64_t* extra_entries);

/* AndDocIdSet.iterator(): CTR/operator/docidsets/AndDocIdSet.java:72-186 */
static dit* make_and_iterator(fop* f, int64_t* extra_entries) {
  int32_t n = f->n_kids, num_docs = f->num_docs;
  dit** all = (dit**)malloc(sizeof(dit*) * (size_t)n);
  int32_t n_sorted = 0, n_bitmap = 0, n_scan = 0, n_rem = 0;
  for (int32_t i = 0; i < n; i++) {
    all[i] = make_iterator(f->kids[i], extra_entries);
    switch (all[i]->kind) { case IT_SORTED: n_sorted++; break; case IT_BITMAP: n_bitmap++; break; case IT_SCAN: n_scan++; break; default: n_rem++; }
  }
  int32_t n_index = n_sorted + n_bitmap;
  if ((n_index > 0 && n_scan > 0) || n_index > 1) {
    bitmap* acc = (bitmap*)malloc(sizeof(bitmap)); *acc = bm_new(num_docs);
    int first = 1;
    /* sorted ranges: intersect (SortedRangeIntersection) then -> bitmap */
    for (int32_t i = 0; i < n; i++) if (all[i]->kind == IT_SORTED) {
      bitmap t = bm_new(num_docs);
      for (int32_t r = 0; r < all[i]->n_ranges; r++) bm_set_range(&t, all[i]->ranges[r].lo, all[i]->ranges[r].hi);
      if (first) { memcpy(acc->w, t.w, (size_t)acc->nwords * 8); first = 0; }
      else for (int64_t k = 0; k < acc->nwords; k++) acc->w[k] &= t.w[k];
      bm_free(&t);
    }
    for (int32_t i = 0; i < n; i++) if (all[i]->kind == IT_BITMAP) {
      if (first) { memcpy(acc->w, all[i]->bm->w, (size_t)acc->nwords * 8); first = 0; }
      else for (int64_t k = 0; k < acc->nwords; k++) acc->w[k] &= all[i]->bm->w[k];
    }
    /* scans restricted to survivors: SVScanDocIdIterator.applyAnd (:115-142): entries += incoming docs */
    for (int32_t i = 0; i < n; i++) if (all[i]->kind == IT_SCAN) {
      int64_t incoming = bm_card(acc);
      if (incoming == 0) continue;                 /* !docIdIterator.hasNext() */
      for (int32_t d = bm_next(acc, 0); d != ORC_EOF; d = bm_next(acc, d + 1))
        if (!pred_match_doc(all[i]->ev, d)) acc->w[d >> 6] &= ~(1ull << (d & 63));
      *extra_entries += incoming;
    }
    dit* merged = dit_new(IT_BITMAP, num_docs); merged->bm = acc; merged->owns_bm = 1;
    dit* result;
    if (n_rem == 0) result = merged;
    else {
      result = dit_new(IT_AND, num_docs);
      result->kids = (dit**)malloc(sizeof(dit*) * (size_t)(n_rem + 1));
      result->kids[result->n_kids++] = merged;
      for (int32_t i = 0; i < n; i++) if (all[i]->kind != IT_SORTED && all[i]->kind != IT_BITMAP && all[i]->kind != IT_SCAN) { result->kids[result->n_kids++] = all[i]; all[i] = NULL; }
    }
    for (int32_t i = 0; i < n; i++) dit_free(all[i]);
    free(all);
    return result;
  }
  dit* result = dit_new(IT_AND, num_docs);
  result->kids = all; result->n_kids = n;
  return result;
}

/* OrDocIdSet.iterator(): CTR/operator/docidsets/OrDocIdSet.java:63-127 */
static dit* make_or_iterator(fop* f, int64_t* extra_entries) {
  int32_t n = f->n_kids, num_docs = f->num_docs;
  dit** all = (dit**)malloc(sizeof(dit*) * (size_t)n);
  int32_t n_index = 0;
  for (int32_t i = 0; i < n; i++) {
    all[i] = make_iterator(f->kids[i], extra_entries);
    if (all[i]->kind == IT_SORTED || all[i]->kind == IT_BITMAP) n_index++;
  }
  dit* result = dit_new(IT_OR, num_docs);
  if (n_index > 1) {
    bitmap* acc = (bitmap*)malloc(sizeof(bitmap)); *acc = bm_new(num_docs);
    for (int32_t i = 0; i < n; i++) {
      if (all[i]->kind == IT_SORTED) for (int32_t r = 0; r < all[i]->n_ranges; r++) bm_set_range(acc, all[i]->ranges[r].lo, all[i]->ranges[r].hi);
      else if (all[i]->kind == IT_BITMAP) for (int64_t k = 0; k < acc->nwords; k++) acc->w[k] |= all[i]->bm->w[k];
    }
    dit* merged = dit_new(IT_BITMAP, num_docs); merged->bm = acc; merged->owns_bm = 1;
    int32_t n_rem = n - n_index;
    if (n_rem == 0) { for (int32_t i = 0; i < n; i++) dit_free(all[i]); free(all); dit_free(result); return merged; }
    result->kids = (dit**)malloc(sizeof(dit*) * (size_t)(n_rem + 1));
    result->kids[result->n_kids++] = merged;
    for (int32_t i = 0; i < n; i++) {
      if (all[i]->kind == IT_SORTED || all[i]->kind == IT_BITMAP) dit_free(all[i]); else result->kids[result->n_kids++] = all[i];
    }
    free(all);
  } else { result->kids = all; result->n_kids = n; }
  result->n_live = result->n_kids;
  result->next_ids = (int32_t*)malloc(sizeof(int32_t) * (size_t)result->n_kids);
  for (int32_t i = 0; i < result->n_kids; i++) result->next_ids[i] = -1;
  result->prev_doc = -1;
  return result;
}

static dit* make_iterator(fop* f, int64_t* extra_entries) {
  switch (f->kind) {
    case OP_EMPTY: return dit_new(IT_EMPTY, f->num_docs);
    case OP_MATCH_ALL: return dit_new(IT_MATCH_ALL, f->num_docs);
    case OP_SORTED: { dit* d = dit_new(IT_SORTED, f->num_docs); d->ranges = f->ranges; d->n_ranges = f->n_ranges; return d; }
    case OP_BITMAP: { dit* d = dit_new(IT_BITMAP, f->num_docs); d->bm = &f->bm; return d; }
    case OP_SCAN: { dit* d = dit_new(IT_SCAN, f->num_docs); d->ev = f->ev; return d; }
    case OP_AND: return make_and_iterator(f, extra_entries);
    case OP_OR: return make_or_iterator(f, extra_entries);
    default: {
      dit* d = dit_new(IT_NOT, f->num_docs);
      d->kids = (dit**)malloc(sizeof(dit*)); d->kids[0] = make_iterator(f->kids[0], extra_entries); d->n_kids = 1;
      int32_t first = dit_next(d->kids[0]);
      d->next_non_matching = first == ORC_EOF ? f->num_docs : first;
      return d;
    }
  }
}

int64_t orc_filter_doc_ids(const orc_segment* seg, const orc_query* q, int32_t** out, int64_t* entries_scanned) {
  fop* root = build_filter(seg, q);
  if (!root) return -1;
  int64_t extra = 0;
  dit* it = make_iterator(root, &extra);
  int64_t cap = 1024, n = 0;
  int32_t* docs = (int32_t*)malloc(sizeof(int32_t) * (size_t)cap);
  for (int32_t d = dit_next(it); d != ORC_EOF; d = dit_next(it)) {
    if (n == cap) { cap *= 2; docs = (int32_t*)realloc(docs, sizeof(int32_t) * (size_t)cap); }
    docs[n++] = d;
  }
  if (entries_scanned) *entries_scanned = extra + dit_entries(it);
  dit_free(it); fop_free(root);
  *out = docs;
  return n;
}

/* ------------------------------------------------------------------ */
/* group-by / aggregation                                              */
/* ------------------------------------------------------------------ */
struct orc_result {
  int32_t num_groups, num_group_by, num_aggs;
  orc_stats stats;
  int64_t* group_keys;          /* [num_groups][num_group_by] */
  double** dbl;                 /* per agg */
  int64_t** lng;                /* per agg */
  int64_t** dc_offsets;         /* per agg (DISTINCTCOUNT) */
  int32_t** dc_ids;
  int64_t** dc_values;          /* DISTINCTCOUNT on a raw column: value bits, ascending per group */
};

void orc_result_free(orc_result* r) {
  if (!r) return;
  for (int32_t a = 0; a < r->num_aggs; a++) {
    if (r->dbl) free(r->dbl[a]);
    if (r->lng) free(r->lng[a]);
    if (r->dc_offsets) free(r->dc_offsets[a]);
    if (r->dc_ids) free(r->dc_ids[a]);
    if (r->dc_values) free(r->dc_values[a]);
  }
  free(r->dbl); free(r->lng); free(r->dc_offsets); free(r->dc_ids); free(r->dc_values); free(r->group_keys); free(r);
}
int32_t orc_result_num_groups(const orc_result* r) { return r->num_groups; }
const orc_stats* orc_result_stats(const orc_result* r) { return &r->stats; }
const int64_t* orc_result_group_keys(const orc_result* r) { return r->group_keys; }
const double* orc_result_double(const orc_result* r, int32_t a) { return r->dbl[a]; }
const int64_t* orc_result_long(const orc_result* r, int32_t a) { return r->lng[a]; }
const int64_t* orc_result_distinct_offsets(const orc_result* r, int32_t a) { return r->dc_offsets[a]; }
const int32_t* orc_result_distinct_dict_ids(const orc_result* r, int32_t a) { return r->dc_ids[a]; }
const int64_t* orc_result_distinct_values(const orc_result* r, int32_t a) { return r->dc_values[a]; }

/* tuple-keyed open-addressing map, ids in first-seen order — stands in for IntGroupIdMap /
 * Long2IntOpenHashMap / Object2IntOpenHashMap<IntArray> (DictionaryBasedGroupKeyGenerator.java:416-495,
 * 629-705, 809-885, 993-1138) and the NoDictionary*GroupKeyGenerator maps.  Iteration order is not
 * part of the contract (tests look groups up by key: CTEST QueriesTestUtils.java:61-83). */
typedef struct {
  int32_t arity;
  int64_t cap, size;
  int32_t* slot_id;     /* -1 empty */
  int64_t* keys;        /* [size][arity], in id order */
  int64_t keys_cap;
} gmap;
static void gmap_init(gmap* m, int32_t arity) {
  m->arity = arity; m->cap = 1024; m->size = 0;
  m->slot_id = (int32_t*)malloc(sizeof(int32_t) * (size_t)m->cap);
  memset(m->slot_id, 0xff, sizeof(int32_t) * (size_t)m->cap);
  m->keys_cap = 1024; m->keys = (int64_t*)malloc(sizeof(int64_t) * (size_t)(m->keys_cap * arity));
}
static void gmap_free(gmap* m) { free(m->slot_id); free(m->keys); }
static inline uint64_t gmap_hash(const int64_t* k, int32_t arity) {
  uint64_t h = 0x9E3779B97F4A7C15ull;
  for (int32_t i = 0; i < arity; i++) { h ^= (uint64_t)k[i]; h *= 0xff51afd7ed558ccdull; h ^= h >> 32; }
  return h;
}
static void gmap_grow(gmap* m) {
  int64_t ncap = m->cap * 2;
  int32_t* ns = (int32_t*)malloc(sizeof(int32_t) * (size_t)ncap);
  memset(ns, 0xff, sizeof(int32_t) * (size_t)ncap);
  for (int64_t id = 0; id < m->size; id++) {
    uint64_t s = gmap_hash(m->keys + id * m->arity, m->arity) & (uint64_t)(ncap - 1);
    while (ns[s] >= 0) s = (s + 1) & (uint64_t)(ncap - 1);
    ns[s] = (int32_t)id;
  }
  free(m->slot_id); m->slot_id = ns; m->cap = ncap;
}
/* returns group id, or -1 (INVALID_ID) when the key is new and the limit is reached
 * (DictionaryBasedGroupKeyGenerator.java:1033-1035, 660-668) */
static int32_t gmap_get_or_add(gmap* m, const int64_t* key, int64_t limit) {
  uint64_t s = gmap_hash(key, m->arity) & (uint64_t)(m->cap - 1);
  while (m->slot_id[s] >= 0) {
    if (memcmp(m->keys + (int64_t)m->slot_id[s] * m->arity, key, sizeof(int64_t) * (size_t)m->arity) == 0) return m->slot_id[s];
    s = (s + 1) & (uint64_t)(m->cap - 1);
  }
  if (m->size >= limit) return -1;
  if (m->size == m->keys_cap) { m->keys_cap *= 2; m->keys = (int64_t*)realloc(m->keys, sizeof(int64_t) * (size_t)(m->keys_cap * m->arity)); }
  memcpy(m->keys + m->size * m->arity, key, sizeof(int64_t) * (size_t)m->arity);
  int32_t id = (int32_t)m->size++;
  m->slot_id[s] = id;
  if (m->size * 4 > m->cap * 3) gmap_grow(m);
  return id;
}

typedef struct { double* v; int64_t cap; double dflt; } dholder;   /* DoubleGroupByResultHolder.java:42-98 */
static void dholder_ensure(dholder* h, int64_t n) {
  if (n <= h->cap) return;
  int64_t nc = h->cap ? h->cap : 16; while (nc < n) nc *= 2;
  h->v = (double*)realloc(h->v, sizeof(double) * (size_t)nc);
  for (int64_t i = h->cap; i < nc; i++) h->v[i] = h->dflt;
  h->cap = nc;
}
typedef struct { uint64_t** sets; int64_t cap; int64_t words; } bholder;   /* per-group dictId bitmaps */
static void bholder_ensure(bholder* h, int64_t n) {
  if (n <= h->cap) return;
  int64_t nc = h->cap ? h->cap : 16; while (nc < n) nc *= 2;
  h->sets = (uint64_t**)realloc(h->sets, sizeof(uint64_t*) * (size_t)nc);
  for (int64_t i = h->cap; i < nc; i++) h->sets[i] = NULL;
  h->cap = nc;
}

/* DISTINCTCOUNT on a raw (no-dictionary) column keeps per-group VALUE sets (IntOpenHashSet / LongOpenHashSet /
 * FloatOpenHashSet / DoubleOpenHashSet, BaseDistinctAggregateAggregationFunction.java:157-226).  Restated as a list of
 * (holder index, value bits) pairs, sorted and de-duplicated at the end; float values are widened to double and NaNs
 * canonicalised, which preserves the sets' notion of equality (Float.floatToIntBits / Double.doubleToLongBits). */
typedef struct { int64_t* h; int64_t* v; int64_t n, cap; } pholder;
static void pholder_add(pholder* p, int64_t h, int64_t v) {
  if (p->n == p->cap) {
    p->cap = p->cap ? p->cap * 2 : 1024;
    p->h = (int64_t*)realloc(p->h, sizeof(int64_t) * (size_t)p->cap);
    p->v = (int64_t*)realloc(p->v, sizeof(int64_t) * (size_t)p->cap);
  }
  p->h[p->n] = h; p->v[p->n] = v; p->n++;
}
static inline int64_t raw_value_bits(const col_reader* r, int32_t doc) {
  if (r->c->data_type == ORC_INT || r->c->data_type == ORC_LONG) return raw_long(r, doc);
  double d = raw_double(r, doc);
  if (d != d) return 0x7ff8000000000000LL;
  int64_t b; memcpy(&b, &d, 8); return b;
}
typedef struct { int64_t h, v; } hv_pair;
static int hv_cmp(const void* a, const void* b) {
  const hv_pair* x = (const hv_pair*)a; const hv_pair* y = (const hv_pair*)b;
  if (x->h != y->h) return x->h < y->h ? -1 : 1;
  return x->v < y->v ? -1 : (x->v > y->v ? 1 : 0);
}

orc_result* orc_execute(const orc_segment* seg, const orc_query* q) {
  g_err[0] = 0;
  const int32_t nG = q->num_group_by, nA = q->num_aggregations, num_docs = seg->num_docs;
  /* ---- swim-lanes: AggregationFunctionUtils.buildFilteredAggregationInfos
   * (CTR/query/aggregation/function/AggregationFunctionUtils.java:312-400).  A plain query is one lane. ---- */
  typedef struct { fop* root; dit* it; uint8_t* has; int64_t docs, extra; int32_t ncols; } lane_t;
  const int32_t nF = q->num_agg_filters;
  lane_t* lanes = (lane_t*)calloc((size_t)nF + 2, sizeof(lane_t));
  int32_t n_lanes = 0;
  {
    fop* main_root = build_filter(seg, q);
    if (!main_root) { free(lanes); return NULL; }
    uint8_t* in_main = (uint8_t*)calloc((size_t)(nA > 0 ? nA : 1), 1);   /* functions of the non-filtered lane */
    int any_main = 0;
    if (nF == 0 || main_root->kind == OP_EMPTY) {
      /* no FILTER clause, or ":317-326": an empty main filter needs no sub-filters: one lane, every function */
      for (int32_t a = 0; a < nA; a++) in_main[a] = 1;
      any_main = 1;
    } else {
      for (int32_t f = 0; f < nF; f++) {
        orc_query sub = *q;
        sub.num_filter_nodes = q->agg_filters[f].num_nodes; sub.filter_nodes = q->agg_filters[f].nodes; sub.predicates = q->agg_filters[f].predicates;
        fop* sub_root = build_filter(seg, &sub);
        if (!sub_root) { fop_free(main_root); free(in_main); free(lanes); return NULL; }
        fop* combined;
        if (main_root->kind == OP_MATCH_ALL || sub_root->kind == OP_EMPTY) combined = sub_root;                 /* :346-347 */
        else if (sub_root->kind == OP_MATCH_ALL) {                                                            /* :348-349, 370-372 */
          for (int32_t a = 0; a < nA; a++) if (q->agg_filter_of[a] == f) { in_main[a] = 1; any_main = 1; }
          fop_free(sub_root);
          continue;
        } else {                                                                                              /* CombinedFilterOperator: AND of the two docId sets */
          fop* kids[2]; kids[0] = build_filter(seg, q); kids[1] = sub_root;
          combined = make_and_op(kids, 2, num_docs);
        }
        lane_t* L = &lanes[n_lanes++];
        L->root = combined;
        L->has = (uint8_t*)calloc((size_t)(nA > 0 ? nA : 1), 1);
        for (int32_t a = 0; a < nA; a++) if (q->agg_filter_of[a] == f) L->has[a] = 1;
      }
      for (int32_t a = 0; a < nA; a++) if (q->agg_filter_of[a] < 0) { in_main[a] = 1; any_main = 1; }
    }
    /* :381-396: the non-filtered lane; a group-by keeps it even without functions so that every group of the main filter exists */
    if (any_main || nG > 0) {
      lane_t* L = &lanes[n_lanes++];
      L->root = main_root; L->has = in_main;
    } else { fop_free(main_root); free(in_main); }
    for (int32_t l = 0; l < n_lanes; l++) {
      lanes[l].it = make_iterator(lanes[l].root, &lanes[l].extra);
      /* ProjectPlanNode.java:69-78: distinct columns projected by the lane = group-by columns + inputs of its functions */
      int32_t cols[128]; int32_t nc = 0;
      for (int32_t j = 0; j < nG; j++) { int32_t c = q->group_by_columns[j]; int seen = 0; for (int32_t k = 0; k < nc; k++) if (cols[k] == c) seen = 1; if (!seen && nc < 128) cols[nc++] = c; }
      for (int32_t a = 0; a < nA; a++) { if (!lanes[l].has[a]) continue; int32_t c = q->aggregations[a].column; if (c < 0) continue; int seen = 0; for (int32_t k = 0; k < nc; k++) if (cols[k] == c) seen = 1; if (!seen && nc < 128) cols[nc++] = c; }
      lanes[l].ncols = nc;
    }
  }
  fop* root = NULL; dit* it = NULL;     /* (owned by the lanes) */

  col_reader* greaders = (col_reader*)calloc((size_t)(nG > 0 ? nG : 1), sizeof(col_reader));
  col_reader* areaders = (col_reader*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(col_reader));
  int all_dict = 1;
  for (int32_t j = 0; j < nG; j++) {
    if (col_reader_init(&greaders[j], &seg->columns[q->group_by_columns[j]], num_docs) != 0) goto fail;
    if (!greaders[j].c->has_dictionary) all_dict = 0;
  }
  for (int32_t a = 0; a < nA; a++) {
    if (q->aggregations[a].column >= 0) {
      if (col_reader_init(&areaders[a], &seg->columns[q->aggregations[a].column], num_docs) != 0) goto fail;
      if (q->aggregations[a].op == ORC_DISTINCTCOUNT && !areaders[a].c->has_dictionary && areaders[a].c->data_type == ORC_STRING) { set_err("DISTINCTCOUNT on raw STRING column unsupported in oracle"); goto fail; }
      if (q->aggregations[a].op != ORC_DISTINCTCOUNT && areaders[a].c->data_type == ORC_STRING) { set_err("numeric aggregation on STRING"); goto fail; }
    }
  }

  /* key-holder strategy: DictionaryBasedGroupKeyGenerator.java:120-185; DefaultGroupByExecutor.java:106-121 */
  int holder = 0; int64_t card_product = 1; int overflow = 0;
  if (nG > 0) {
    if (!all_dict) holder = 5;
    else {
      for (int32_t j = 0; j < nG; j++) {
        int64_t card = greaders[j].c->cardinality;
        if (!overflow) { if (card_product > INT64_MAX / card) overflow = 1; else card_product *= card; }
      }
      if (overflow) holder = 4;
      else if (card_product > INT32_MAX) holder = 3;
      else if (card_product > q->max_initial_result_holder_capacity || q->num_groups_limit < card_product) holder = 2;
      else holder = 1;
    }
  }
  const int64_t limit = q->num_groups_limit;

  gmap map; int have_map = 0;
  uint8_t* array_flags = NULL;       /* ArrayBasedHolder._flags */
  int64_t num_keys = 0;              /* number of groups created */
  if (holder >= 2) { gmap_init(&map, nG); have_map = 1; }
  else if (holder == 1) array_flags = (uint8_t*)calloc((size_t)card_product, 1);

  dholder* dh = (dholder*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(dholder));   /* SUM/MIN/MAX/COUNT(double)/AVG sum */
  dholder* ch = (dholder*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(dholder));   /* AVG count */
  bholder* bh = (bholder*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(bholder));
  pholder* ph = (pholder*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(pholder));   /* DISTINCTCOUNT on raw columns */
  for (int32_t a = 0; a < nA; a++) {
    int op = q->aggregations[a].op;
    dh[a].dflt = op == ORC_MIN ? INFINITY : (op == ORC_MAX ? -INFINITY : 0.0);
    ch[a].dflt = 0.0;
    if (op == ORC_DISTINCTCOUNT && areaders[a].c->has_dictionary) bh[a].words = ((int64_t)areaders[a].c->cardinality + 63) / 64;
  }
  /* enableNullHandling (NullableSingleInputAggregationFunction.java:63-134 forEachNotNull / foldNotNull): a function only
   * sees the docs of a block whose input is not null -- the null docs of its column (anull, none = w NULL) are dropped from
   * the block before the function's loop runs -- and nn counts the inputs it saw per group: 0 = the result is SQL NULL
   * (ObjectGroupByResultHolder never set, e.g. SumAggregationFunction.java:160-179, 206-220) */
  bitmap* anull = (bitmap*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(bitmap));
  dholder* nn = (dholder*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(dholder));
  int32_t* nn_docs = (int32_t*)malloc(sizeof(int32_t) * MAX_DOC_PER_CALL);
  int32_t* nn_groups = (int32_t*)malloc(sizeof(int32_t) * MAX_DOC_PER_CALL);
  uint8_t* nn_brk = (uint8_t*)malloc(MAX_DOC_PER_CALL);     /* element starts a new non-null range of the block */
  if (q->null_handling)
    for (int32_t a = 0; a < nA; a++) {
      int32_t c = q->aggregations[a].column;
      if (c < 0 || !seg->columns[c].null_value_vector) continue;
      anull[a] = bm_new(num_docs);
      roaring_for_each(seg->columns[c].null_value_vector, seg->columns[c].null_value_vector_len, bm_sink, &anull[a]);
    }
  /* keyless native-type MIN/MAX state (MinAggregationFunction.java:69-148) */
  int64_t* kl_long = (int64_t*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(int64_t));
  int* kl_long_set = (int*)calloc((size_t)(nA > 0 ? nA : 1), sizeof(int));
  int64_t kl_count = 0;

  int32_t* doc_ids = (int32_t*)malloc(sizeof(int32_t) * MAX_DOC_PER_CALL);
  int32_t* group_ids = (int32_t*)malloc(sizeof(int32_t) * MAX_DOC_PER_CALL);
  double* values = (double*)malloc(sizeof(double) * MAX_DOC_PER_CALL);
  int32_t* dict_buf = (int32_t*)malloc(sizeof(int32_t) * MAX_DOC_PER_CALL);
  int64_t key[64];
  if (nG > 64) { set_err("too many group-by columns"); goto fail2; }
  int64_t num_docs_scanned = 0;
  if (nG == 0) for (int32_t a = 0; a < nA; a++) { dholder_ensure(&dh[a], 1); dholder_ensure(&ch[a], 1); bholder_ensure(&bh[a], 1); dholder_ensure(&nn[a], 1); }

  /* GroupByOperator.getNextBlock (CTR/operator/query/GroupByOperator.java:101-140) /
   * AggregationOperator.getNextBlock (CTR/operator/query/AggregationOperator.java:64-80) */
  /* FilteredGroupByOperator.getNextBlock (CTR/operator/query/FilteredGroupByOperator.java:108-159) /
   * FilteredAggregationOperator.getNextBlock (FilteredAggregationOperator.java:68-103): lane after lane, one shared
   * group-key generator, result holders indexed by function */
  for (int32_t lane = 0; lane < n_lanes; lane++) {
  const uint8_t* lane_has = lanes[lane].has;
  it = lanes[lane].it;
  int lane_eof = 0;
  while (!lane_eof) {
    /* DocIdSetOperator.getNextBlock: CTR/operator/DocIdSetOperator.java:59-86 (":63 if (_currentDocId == Constants.EOF) return
     * null": the iterator is never asked again once it has returned EOF -- And / Not iterators are not idempotent there) */
    int32_t len = 0;
    for (; len < MAX_DOC_PER_CALL; len++) { int32_t d = dit_next(it); if (d == ORC_EOF) { lane_eof = 1; break; } doc_ids[len] = d; }
    if (len == 0) break;
    num_docs_scanned += len;
    lanes[lane].docs += len;

    if (nG > 0) {
      /* generateKeysForBlock: DictionaryBasedGroupKeyGenerator.java:210-217, 290-305, 341-347, 424-446 */
      for (int32_t i = 0; i < len; i++) {
        int32_t d = doc_ids[i];
        if (holder == 1) {
          int64_t raw = 0, mult = 1;
          for (int32_t j = 0; j < nG; j++) { raw += (int64_t)dict_id_of(&greaders[j], d) * mult; mult *= greaders[j].c->cardinality; }
          if (!array_flags[raw]) { array_flags[raw] = 1; num_keys++; }
          group_ids[i] = (int32_t)raw;
        } else {
          for (int32_t j = 0; j < nG; j++) {
            const col_reader* r = &greaders[j];
            if (r->c->has_dictionary) key[j] = dict_id_of(r, d);
            else if (r->c->data_type == ORC_INT || r->c->data_type == ORC_LONG) key[j] = raw_long(r, d);
            else { double v = raw_double(r, d); memcpy(&key[j], &v, 8); }
          }
          group_ids[i] = gmap_get_or_add(&map, key, limit);
        }
      }
      int64_t need = holder == 1 ? card_product : map.size;
      for (int32_t a = 0; a < nA; a++) {
        int op = q->aggregations[a].op;
        dholder_ensure(&dh[a], need);
        if (op == ORC_AVG) dholder_ensure(&ch[a], need);
        if (op == ORC_DISTINCTCOUNT) bholder_ensure(&bh[a], need);
        if (!lane_has[a]) continue;
        const int32_t* D = doc_ids; const int32_t* G = group_ids; int32_t L = len;
        if (anull[a].w) {   /* forEachNotNull: only the non-null docs of the block reach the function */
          L = 0;
          for (int32_t i = 0; i < len; i++) if (!bm_get(&anull[a], doc_ids[i])) { nn_docs[L] = doc_ids[i]; nn_groups[L] = group_ids[i]; L++; }
          D = nn_docs; G = nn_groups;
        }
        if (q->null_handling) { dholder_ensure(&nn[a], need); for (int32_t i = 0; i < L; i++) if (G[i] >= 0) nn[a].v[G[i]] += 1.0; }
        if (op == ORC_COUNT) {   /* CountAggregationFunction.java:178-185 */
          for (int32_t i = 0; i < L; i++) if (G[i] >= 0) dh[a].v[G[i]] += 1.0;
          continue;
        }
        if (op == ORC_DISTINCTCOUNT && !areaders[a].c->has_dictionary) {   /* BaseDistinctAggregateAggregationFunction.java:323-400 */
          for (int32_t i = 0; i < L; i++) if (G[i] >= 0) pholder_add(&ph[a], G[i], raw_value_bits(&areaders[a], D[i]));
          continue;
        }
        if (op == ORC_DISTINCTCOUNT) {  /* BaseDistinctAggregateAggregationFunction.java:306-321 */
          for (int32_t i = 0; i < L; i++) {
            int32_t g = G[i]; if (g < 0) continue;
            if (!bh[a].sets[g]) bh[a].sets[g] = (uint64_t*)calloc((size_t)bh[a].words, 8);
            int32_t id = dict_id_of(&areaders[a], D[i]);
            bh[a].sets[g][id >> 6] |= 1ull << (id & 63);
          }
          continue;
        }
        for (int32_t i = 0; i < L; i++) values[i] = value_as_double(&areaders[a], D[i]);
        double* hv = dh[a].v;
        switch (op) {
          case ORC_SUM:  /* SumAggregationFunction.java:160-179 */
            for (int32_t i = 0; i < L; i++) if (G[i] >= 0) hv[G[i]] += values[i];
            break;
          case ORC_MIN:  /* MinAggregationFunction.java:163-188: strict < in double */
            for (int32_t i = 0; i < L; i++) if (G[i] >= 0 && values[i] < hv[G[i]]) hv[G[i]] = values[i];
            break;
          case ORC_MAX:
            for (int32_t i = 0; i < L; i++) if (G[i] >= 0 && values[i] > hv[G[i]]) hv[G[i]] = values[i];
            break;
          case ORC_AVG:  /* AvgAggregationFunction.java:106-127 */
            for (int32_t i = 0; i < L; i++) if (G[i] >= 0) { hv[G[i]] += values[i]; ch[a].v[G[i]] += 1.0; }
            break;
          default: break;
        }
      }
    } else {
      kl_count += len;
      for (int32_t a = 0; a < nA; a++) {
        int op = q->aggregations[a].op;
        if (!lane_has[a]) continue;
        const int32_t* D = doc_ids; int32_t L = len;
        if (anull[a].w) {   /* foldNotNull over the non-null ranges of the block */
          L = 0;
          int prev_null = 1;
          for (int32_t i = 0; i < len; i++) {
            if (bm_get(&anull[a], doc_ids[i])) { prev_null = 1; continue; }
            nn_docs[L] = doc_ids[i]; nn_brk[L] = (uint8_t)prev_null; prev_null = 0; L++;
          }
          D = nn_docs;
        }
        if (q->null_handling) nn[a].v[0] += (double)L;
        if (L == 0 && anull[a].w) continue;          /* the entire block is null: the holder is not touched */
        if (op == ORC_COUNT) { dh[a].v[0] += (double)L; continue; }   /* CountAggregationFunction.java:110-116 */
        const col_reader* r = &areaders[a];
        if (op == ORC_DISTINCTCOUNT && !r->c->has_dictionary) {   /* BaseDistinctAggregateAggregationFunction.java:157-226 */
          for (int32_t i = 0; i < L; i++) pholder_add(&ph[a], 0, raw_value_bits(r, D[i]));
          continue;
        }
        if (op == ORC_DISTINCTCOUNT) {   /* BaseDistinctAggregateAggregationFunction.java:144-155 */
          if (!bh[a].sets[0]) bh[a].sets[0] = (uint64_t*)calloc((size_t)bh[a].words, 8);
          for (int32_t i = 0; i < L; i++) { int32_t id = dict_id_of(r, D[i]); bh[a].sets[0][id >> 6] |= 1ull << (id & 63); }
          continue;
        }
        int is_long_typed = (r->c->data_type == ORC_INT || r->c->data_type == ORC_LONG);
        if ((op == ORC_MIN || op == ORC_MAX) && is_long_typed) {
          /* keyless MIN/MAX fold in the native type, then doubleValue() */
          for (int32_t i = 0; i < L; i++) {
            int64_t v = r->c->has_dictionary ? dict_long(r->c, dict_id_of(r, D[i])) : raw_long(r, D[i]);
            if (!kl_long_set[a] || (op == ORC_MIN ? v < kl_long[a] : v > kl_long[a])) { kl_long[a] = v; kl_long_set[a] = 1; }
          }
          dh[a].v[0] = (double)kl_long[a];
          continue;
        }
        for (int32_t i = 0; i < L; i++) values[i] = value_as_double(r, D[i]);
        if (op == ORC_SUM || op == ORC_AVG) {   /* SumAggregationFunction.java:69-145: per-block innerSum */
          if (anull[a].w) {
            /* foldNotNull: one innerSum per non-null range, acum == null ? innerSum : acum + innerSum; then sum + otherSum */
            double acc = 0; int have = 0;
            for (int32_t i = 0; i < L;) {
              double inner = values[i]; int32_t k = i + 1;
              while (k < L && !nn_brk[k]) inner += values[k++];
              acc = have ? acc + inner : inner; have = 1; i = k;
            }
            dh[a].v[0] = acc + dh[a].v[0];
            if (op == ORC_AVG) ch[a].v[0] += (double)L;
            continue;
          }
          double inner = 0; for (int32_t i = 0; i < L; i++) inner += values[i];
          dh[a].v[0] += inner;
          if (op == ORC_AVG) ch[a].v[0] += (double)L;
        } else if (op == ORC_MIN || op == ORC_MAX) {
          /* keyless MIN / MAX of a FLOAT / DOUBLE column fold with Math.min / Math.max (MinAggregationFunction.java:97-124,
           * 147-157): a NaN input makes the result NaN, and -0.0 is smaller than 0.0 -- unlike the strict "<" of the
           * group-by path (:163-188), which never lets a NaN in */
          double acc = dh[a].v[0];
          for (int32_t i = 0; i < L; i++) acc = op == ORC_MIN ? java_math_min(acc, values[i]) : java_math_max(acc, values[i]);
          dh[a].v[0] = acc;
        }
        (void)dict_buf;
      }
    }
  }
  }   /* lanes */
  if (nG > 0) {   /* holders of functions whose lane saw no block still cover every group (FilteredGroupByOperator.java:161-163) */
    int64_t need = holder == 1 ? card_product : map.size;
    for (int32_t a = 0; a < nA; a++) { dholder_ensure(&dh[a], need); dholder_ensure(&ch[a], need); bholder_ensure(&bh[a], need); dholder_ensure(&nn[a], need); }
  }

  /* ---- build the result ---- */
  orc_result* res = (orc_result*)calloc(1, sizeof(orc_result));
  res->num_group_by = nG; res->num_aggs = nA;
  int64_t ng;
  int32_t* id_of_group = NULL;    /* result row -> holder index */
  if (nG == 0) ng = 1;
  else if (holder == 1) {
    ng = num_keys;
    id_of_group = (int32_t*)malloc(sizeof(int32_t) * (size_t)(ng > 0 ? ng : 1));
    int64_t k = 0;
    for (int64_t raw = 0; raw < card_product; raw++) if (array_flags[raw]) id_of_group[k++] = (int32_t)raw;
  } else ng = map.size;
  res->num_groups = (int32_t)ng;
  res->group_keys = (int64_t*)calloc((size_t)((ng > 0 ? ng : 1) * (nG > 0 ? nG : 1)), sizeof(int64_t));
  for (int64_t g = 0; g < ng && nG > 0; g++) {
    if (holder == 1) {   /* decode: DictionaryBasedGroupKeyGenerator.java:578-591 */
      int64_t raw = id_of_group[g];
      for (int32_t j = 0; j < nG; j++) { int64_t card = greaders[j].c->cardinality; res->group_keys[g * nG + j] = raw % card; raw /= card; }
    } else memcpy(res->group_keys + g * nG, map.keys + g * nG, sizeof(int64_t) * (size_t)nG);
  }
  res->dbl = (double**)calloc((size_t)(nA > 0 ? nA : 1), sizeof(double*));
  res->lng = (int64_t**)calloc((size_t)(nA > 0 ? nA : 1), sizeof(int64_t*));
  res->dc_offsets = (int64_t**)calloc((size_t)(nA > 0 ? nA : 1), sizeof(int64_t*));
  res->dc_ids = (int32_t**)calloc((size_t)(nA > 0 ? nA : 1), sizeof(int32_t*));
  res->dc_values = (int64_t**)calloc((size_t)(nA > 0 ? nA : 1), sizeof(int64_t*));
  for (int32_t a = 0; a < nA; a++) {
    int op = q->aggregations[a].op;
    res->dbl[a] = (double*)calloc((size_t)(ng > 0 ? ng : 1), sizeof(double));
    res->lng[a] = (int64_t*)calloc((size_t)(ng > 0 ? ng : 1), sizeof(int64_t));
    if (op == ORC_DISTINCTCOUNT) res->dc_offsets[a] = (int64_t*)calloc((size_t)ng + 1, sizeof(int64_t));
    if (op == ORC_DISTINCTCOUNT && !areaders[a].c->has_dictionary) {
      /* sort (holder index, value), drop duplicates, then hand the sets out in result-group order */
      hv_pair* pr = (hv_pair*)malloc(sizeof(hv_pair) * (size_t)(ph[a].n > 0 ? ph[a].n : 1));
      for (int64_t i = 0; i < ph[a].n; i++) { pr[i].h = ph[a].h[i]; pr[i].v = ph[a].v[i]; }
      qsort(pr, (size_t)ph[a].n, sizeof(hv_pair), hv_cmp);
      int64_t nu = 0;
      for (int64_t i = 0; i < ph[a].n; i++) if (i == 0 || pr[i].h != pr[i - 1].h || pr[i].v != pr[i - 1].v) pr[nu++] = pr[i];
      res->dc_values[a] = (int64_t*)malloc(sizeof(int64_t) * (size_t)(nu > 0 ? nu : 1));
      int64_t k = 0;
      for (int64_t g = 0; g < ng; g++) {
        int64_t h = (nG > 0 && holder == 1) ? id_of_group[g] : g;
        int64_t lo = 0, hi = nu;                       /* first pair with holder index >= h */
        while (lo < hi) { int64_t mid = (lo + hi) >> 1; if (pr[mid].h < h) lo = mid + 1; else hi = mid; }
        int64_t n = 0;
        for (int64_t i = lo; i < nu && pr[i].h == h; i++) { res->dc_values[a][k++] = pr[i].v; n++; }
        res->lng[a][g] = n; res->dc_offsets[a][g + 1] = k;
      }
      free(pr);
      continue;
    }
    int64_t total_ids = 0;
    for (int64_t g = 0; g < ng; g++) {
      int64_t h = (nG > 0 && holder == 1) ? id_of_group[g] : g;
      switch (op) {
        case ORC_COUNT: res->lng[a][g] = (int64_t)dh[a].v[h]; res->dbl[a][g] = dh[a].v[h]; break;
        case ORC_AVG: res->dbl[a][g] = dh[a].v[h]; res->lng[a][g] = (int64_t)ch[a].v[h]; break;
        case ORC_DISTINCTCOUNT: {
          int64_t n = 0;
          if (bh[a].sets[h]) for (int64_t w = 0; w < bh[a].words; w++) n += __builtin_popcountll(bh[a].sets[h][w]);
          res->lng[a][g] = n; total_ids += n; res->dc_offsets[a][g + 1] = total_ids;
          break;
        }
        default: res->dbl[a][g] = dh[a].v[h]; if (q->null_handling) res->lng[a][g] = (int64_t)nn[a].v[h]; break;   /* 0 inputs = SQL NULL */
      }
    }
    if (op == ORC_DISTINCTCOUNT) {
      res->dc_ids[a] = (int32_t*)malloc(sizeof(int32_t) * (size_t)(total_ids > 0 ? total_ids : 1));
      int64_t k = 0;
      for (int64_t g = 0; g < ng; g++) {
        int64_t h = (nG > 0 && holder == 1) ? id_of_group[g] : g;
        if (!bh[a].sets[h]) continue;
        for (int64_t w = 0; w < bh[a].words; w++) { uint64_t x = bh[a].sets[h][w]; while (x) { res->dc_ids[a][k++] = (int32_t)(w * 64 + __builtin_ctzll(x)); x &= x - 1; } }
      }
    }
  }
  /* ExecutionStatistics: GroupByOperator.java:148-153; ProjectPlanNode.java:69-78 (distinct projected columns) */
  {
    int32_t cols[128]; int32_t nc = 0;
    for (int32_t j = 0; j < nG; j++) { int32_t c = q->group_by_columns[j]; int seen = 0; for (int32_t k = 0; k < nc; k++) if (cols[k] == c) seen = 1; if (!seen && nc < 128) cols[nc++] = c; }
    for (int32_t a = 0; a < nA; a++) { int32_t c = q->aggregations[a].column; if (c < 0) continue; int seen = 0; for (int32_t k = 0; k < nc; k++) if (cols[k] == c) seen = 1; if (!seen && nc < 128) cols[nc++] = c; }
    (void)nc;
    int64_t in_filter = 0, post_filter = 0;
    for (int32_t l = 0; l < n_lanes; l++) { in_filter += lanes[l].extra + dit_entries(lanes[l].it); post_filter += lanes[l].docs * lanes[l].ncols; }
    res->stats.num_docs_scanned = num_docs_scanned;
    res->stats.num_entries_scanned_in_filter = in_filter;
    res->stats.num_entries_scanned_post_filter = post_filter;
    res->stats.num_total_docs = num_docs;
    res->stats.num_groups_limit_reached = (nG > 0 && ng >= limit) ? 1 : 0;   /* GroupByOperator.java:116 */
    res->stats.key_holder = holder;
  }
  free(id_of_group);
  free(doc_ids); free(group_ids); free(values); free(dict_buf);
  for (int32_t a = 0; a < nA; a++) {
    free(dh[a].v); free(ch[a].v);
    for (int64_t i = 0; i < bh[a].cap; i++) free(bh[a].sets[i]);
    free(bh[a].sets);
    free(ph[a].h); free(ph[a].v);
  }
  for (int32_t a = 0; a < nA; a++) { free(nn[a].v); if (anull[a].w) bm_free(&anull[a]); }
  free(nn); free(anull); free(nn_docs); free(nn_groups); free(nn_brk);
  free(dh); free(ch); free(bh); free(ph); free(kl_long); free(kl_long_set);
  if (have_map) gmap_free(&map);
  free(array_flags); free(greaders); free(areaders);
  for (int32_t l = 0; l < n_lanes; l++) { dit_free(lanes[l].it); fop_free(lanes[l].root); free(lanes[l].has); }
  free(lanes);
  (void)kl_count; (void)root;
  return res;

fail2:
  free(doc_ids); free(group_ids); free(values); free(dict_buf);
  for (int32_t a = 0; a < nA; a++) if (anull[a].w) bm_free(&anull[a]);
  free(nn); free(anull); free(nn_docs); free(nn_groups); free(nn_brk);
  free(dh); free(ch); free(bh); free(ph); free(kl_long); free(kl_long_set);
  if (have_map) gmap_free(&map);
  free(array_flags);
fail:
  free(greaders); free(areaders);
  for (int32_t l = 0; l < n_lanes; l++) { if (lanes[l].it) dit_free(lanes[l].it); if (lanes[l].root) fop_free(lanes[l].root); free(lanes[l].has); }
  free(lanes);
  (void)it;
  return NULL;
}


/* ---- CombineOperator-style driver: the segments of one query on `threads` worker threads (a shared work queue, as
 * BaseCombineOperator hands segments to its tasks: CTR/operator/combine/BaseCombineOperator.java:100-141).  Test / bench
 * infrastructure: lets the CPU baseline use every host core without the Python interpreter in the timed loop. ---- */
#include <pthread.h>
/* ---- the same pass WITH the cross-segment merge done natively, the way GroupByCombineOperator does it: every worker thread
 * folds the result of the segment it just executed into an IndexedTable keyed by the DECODED group key (CTR/operator/combine/
 * GroupByCombineOperator.java:132-147 -> IndexedTable.upsert, CTR/data/table/IndexedTable.java:99-125: SUM / COUNT add, MIN
 * min, MAX max, AVG (sum, count) add).  Here each worker owns a private table and the tables are merged at the end (the
 * reference's workers share one ConcurrentIndexedTable; the result is the same).  Numeric group keys and COUNT / SUM / MIN /
 * MAX / AVG only: what the CPU baseline of the benchmark needs.  Worker threads are created once and kept (a query server
 * runs a thread pool; fresh threads would pay for fresh malloc arenas on every query). ---- */
typedef struct { int64_t* keys; double* dbl; int64_t* lng; uint8_t* used; int64_t cap, size; int32_t nG, nA; } ctable;
static void ctable_init(ctable* t, int32_t nG, int32_t nA) {
  t->nG = nG; t->nA = nA; t->cap = 1024; t->size = 0;
  t->keys = (int64_t*)malloc(sizeof(int64_t) * (size_t)(t->cap * (nG > 0 ? nG : 1)));
  t->dbl = (double*)malloc(sizeof(double) * (size_t)(t->cap * nA)); t->lng = (int64_t*)malloc(sizeof(int64_t) * (size_t)(t->cap * nA));
  t->used = (uint8_t*)calloc((size_t)t->cap, 1);
}
static void ctable_free(ctable* t) { free(t->keys); free(t->dbl); free(t->lng); free(t->used); }
static int64_t ctable_slot(ctable* t, const int64_t* key) {
  uint64_t h = 1469598103934665603ull;
  for (int32_t j = 0; j < t->nG; j++) { h ^= (uint64_t)key[j]; h *= 1099511628211ull; h ^= h >> 29; }
  int64_t i = (int64_t)(h & (uint64_t)(t->cap - 1));
  while (t->used[i] && memcmp(t->keys + i * t->nG, key, sizeof(int64_t) * (size_t)t->nG) != 0) i = (i + 1) & (t->cap - 1);
  return i;
}
static void ctable_upsert(ctable* t, const int32_t* ops, const int64_t* key, const double* d, const int64_t* l);
static void ctable_grow(ctable* t, const int32_t* ops) {
  ctable o = *t;
  t->cap = o.cap * 2; t->size = 0;
  t->keys = (int64_t*)malloc(sizeof(int64_t) * (size_t)(t->cap * (t->nG > 0 ? t->nG : 1)));
  t->dbl = (double*)malloc(sizeof(double) * (size_t)(t->cap * t->nA)); t->lng = (int64_t*)malloc(sizeof(int64_t) * (size_t)(t->cap * t->nA));
  t->used = (uint8_t*)calloc((size_t)t->cap, 1);
  for (int64_t i = 0; i < o.cap; i++) if (o.used[i]) ctable_upsert(t, ops, o.keys + i * o.nG, o.dbl + i * o.nA, o.lng + i * o.nA);
  ctable_free(&o);
}
static void ctable_upsert(ctable* t, const int32_t* ops, const int64_t* key, const double* d, const int64_t* l) {
  if ((t->size + 1) * 2 > t->cap) ctable_grow(t, ops);
  int64_t i = ctable_slot(t, key);
  double* td = t->dbl + i * t->nA; int64_t* tl = t->lng + i * t->nA;
  if (!t->used[i]) {
    t->used[i] = 1; t->size++;
    memcpy(t->keys + i * t->nG, key, sizeof(int64_t) * (size_t)t->nG);
    memcpy(td, d, sizeof(double) * (size_t)t->nA); memcpy(tl, l, sizeof(int64_t) * (size_t)t->nA);
    return;
  }
  for (int32_t a = 0; a < t->nA; a++) {
    switch (ops[a]) {
      case ORC_COUNT: tl[a] += l[a]; td[a] += d[a]; break;
      case ORC_SUM: td[a] += d[a]; break;
      case ORC_MIN: if (d[a] < td[a]) td[a] = d[a]; break;
      case ORC_MAX: if (d[a] > td[a]) td[a] = d[a]; break;
      default: td[a] += d[a]; tl[a] += l[a]; break;     /* AVG */
    }
  }
}
/* fold one segment's result into a table, decoding dictIds to values (keys of FLOAT / DOUBLE columns as their bit patterns) */
static void ctable_fold(ctable* t, const orc_segment* seg, const orc_query* q, const orc_result* r, const int32_t* ops) {
  int64_t key[64]; double d[64]; int64_t l[64];
  for (int32_t g = 0; g < r->num_groups; g++) {
    for (int32_t j = 0; j < q->num_group_by; j++) {
      const orc_column* c = &seg->columns[q->group_by_columns[j]];
      int64_t k = r->group_keys[(int64_t)g * q->num_group_by + j];
      if (c->has_dictionary) {
        if (c->data_type == ORC_INT || c->data_type == ORC_LONG) k = dict_long(c, (int32_t)k);
        else { double v = dict_double(c, (int32_t)k); memcpy(&k, &v, 8); }
      }
      key[j] = k;
    }
    for (int32_t a = 0; a < q->num_aggregations; a++) { d[a] = r->dbl[a][g]; l[a] = r->lng[a][g]; }
    ctable_upsert(t, ops, key, d, l);
  }
}

typedef struct orc_pool orc_pool;
typedef struct { const orc_segment* const* segs; const orc_query* const* qs; orc_result** out; int32_t n; volatile int32_t next;
                 ctable* tables; const int32_t* ops; volatile int32_t failed; } orc_job;
struct orc_pool {
  pthread_mutex_t mu; pthread_cond_t wake, done;
  pthread_t* th; int32_t n_threads;
  orc_job* job; int64_t epoch; int32_t want, busy;      /* `want` workers take part in the current job */
};
static orc_pool g_pool = { PTHREAD_MUTEX_INITIALIZER, PTHREAD_COND_INITIALIZER, PTHREAD_COND_INITIALIZER, NULL, 0, NULL, 0, 0, 0 };
static void orc_job_run(orc_job* b, int32_t worker) {
  for (;;) {
    int32_t i = __sync_fetch_and_add(&b->next, 1);
    if (i >= b->n) break;
    orc_result* r = orc_execute(b->segs[i], b->qs[i]);
    if (!r) { __sync_fetch_and_add(&b->failed, 1); continue; }
    if (b->tables) { ctable_fold(&b->tables[worker], b->segs[i], b->qs[i], r, b->ops); orc_result_free(r); }
    else b->out[i] = r;
  }
}
static void* orc_pool_worker(void* arg) {
  const int32_t id = (int32_t)(intptr_t)arg;            /* worker 0 is the calling thread */
  int64_t seen = 0;
  pthread_mutex_lock(&g_pool.mu);
  for (;;) {
    while (g_pool.epoch == seen) pthread_cond_wait(&g_pool.wake, &g_pool.mu);
    seen = g_pool.epoch;
    orc_job* job = g_pool.job;
    if (!job || id >= g_pool.want) continue;
    pthread_mutex_unlock(&g_pool.mu);
    orc_job_run(job, id);
    pthread_mutex_lock(&g_pool.mu);
    if (--g_pool.busy == 0) pthread_cond_signal(&g_pool.done);
  }
  return NULL;
}
/* run a job on `threads` threads: the caller plus threads - 1 pooled workers */
static void orc_pool_run(orc_job* job, int32_t threads) {
  pthread_mutex_lock(&g_pool.mu);
  if (g_pool.n_threads < threads) {
    g_pool.th = (pthread_t*)realloc(g_pool.th, sizeof(pthread_t) * (size_t)threads);
    for (int32_t t = g_pool.n_threads; t < threads; t++) {
      if (t == 0) continue;
      if (pthread_create(&g_pool.th[t], NULL, orc_pool_worker, (void*)(intptr_t)t) != 0) { threads = t; break; }
    }
    if (g_pool.n_threads < threads) g_pool.n_threads = threads;
  }
  g_pool.job = job; g_pool.want = threads; g_pool.busy = threads - 1; g_pool.epoch++;
  pthread_cond_broadcast(&g_pool.wake);
  pthread_mutex_unlock(&g_pool.mu);
  orc_job_run(job, 0);
  pthread_mutex_lock(&g_pool.mu);
  while (g_pool.busy > 0) pthread_cond_wait(&g_pool.done, &g_pool.mu);
  g_pool.job = NULL;
  pthread_mutex_unlock(&g_pool.mu);
}

/* One combine pass: executes the n segments on `threads` threads and merges their results.  Returns the number of groups
 * (or -1), and hands out malloc'ed arrays: keys[num_groups][num_group_by] (decoded values), dbl / lng [num_groups][num_aggs].
 * orc_free() them. */
int64_t orc_execute_combined(const orc_segment* const* segs, const orc_query* const* qs, int32_t n, int32_t threads,
                             int64_t** keys_out, double** dbl_out, int64_t** lng_out) {
  if (n <= 0) return -1;
  const orc_query* q0 = qs[0];
  const int32_t nG = q0->num_group_by, nA = q0->num_aggregations;
  if (nG > 64 || nA > 64) { set_err("orc_execute_combined: too many columns"); return -1; }
  int32_t ops[64];
  for (int32_t a = 0; a < nA; a++) {
    ops[a] = q0->aggregations[a].op;
    if (ops[a] == ORC_DISTINCTCOUNT) { set_err("orc_execute_combined: DISTINCTCOUNT is merged by the Python combine"); return -1; }
  }
  for (int32_t i = 0; i < n; i++)
    for (int32_t j = 0; j < nG; j++) if (segs[i]->columns[qs[i]->group_by_columns[j]].data_type == ORC_STRING) { set_err("orc_execute_combined: STRING group keys are merged by the Python combine"); return -1; }
  if (threads < 1) threads = 1;
  if (threads > n) threads = n;
  ctable* tables = (ctable*)malloc(sizeof(ctable) * (size_t)threads);
  for (int32_t t = 0; t < threads; t++) ctable_init(&tables[t], nG, nA);
  orc_job job = { segs, qs, NULL, n, 0, tables, ops, 0 };
  orc_pool_run(&job, threads);
  for (int32_t t = 1; t < threads; t++) {                 /* merge the workers' tables into the first */
    for (int64_t i = 0; i < tables[t].cap; i++) if (tables[t].used[i]) ctable_upsert(&tables[0], ops, tables[t].keys + i * nG, tables[t].dbl + i * nA, tables[t].lng + i * nA);
    ctable_free(&tables[t]);
  }
  int64_t ng = job.failed ? -1 : tables[0].size;
  if (ng >= 0) {
    *keys_out = (int64_t*)malloc(sizeof(int64_t) * (size_t)((ng > 0 ? ng : 1) * (nG > 0 ? nG : 1)));
    *dbl_out = (double*)malloc(sizeof(double) * (size_t)((ng > 0 ? ng : 1) * nA)); *lng_out = (int64_t*)malloc(sizeof(int64_t) * (size_t)((ng > 0 ? ng : 1) * nA));
    int64_t k = 0;
    for (int64_t i = 0; i < tables[0].cap; i++) if (tables[0].used[i]) {
      memcpy(*keys_out + k * nG, tables[0].keys + i * nG, sizeof(int64_t) * (size_t)nG);
      memcpy(*dbl_out + k * nA, tables[0].dbl + i * nA, sizeof(double) * (size_t)nA); memcpy(*lng_out + k * nA, tables[0].lng + i * nA, sizeof(int64_t) * (size_t)nA);
      k++;
    }
  }
  ctable_free(&tables[0]); free(tables);
  return ng;
}

int32_t orc_execute_batch(const orc_segment* const* segs, const orc_query* const* qs, int32_t n, int32_t threads, orc_result** out) {
  if (n <= 0) return 0;
  if (threads < 1) threads = 1;
  if (threads > n) threads = n;
  for (int32_t i = 0; i < n; i++) out[i] = NULL;
  orc_job job = { segs, qs, out, n, 0, NULL, NULL, 0 };
  orc_pool_run(&job, threads);
  int32_t failed = 0;
  for (int32_t i = 0; i < n; i++) if (!out[i]) failed++;
  return failed;
}

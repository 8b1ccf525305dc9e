// parquet.cu — a10: Parquet -> device columns (Table.readParquet(ParquetOptions, HostMemoryBuffer)).
// Reference: MakeParquetTableProducer / ParquetTableReader (GpuParquetScan.scala:3322-3503), host
// reassembly readPartFile (:2089-2127: "PAR1" + needed column chunks + rewritten footer + len +
// "PAR1"), getParquetOptions (:2234-2244: columns selected by name, in includeColumn order),
// timestamps delivered as microseconds.  The file format is Apache Parquet (external spec).
//
// Host: parse the thrift-compact footer and walk every page header of the selected column chunks
// (headers are tiny; payloads are never touched on the CPU).  Device: (1) snappy-decompress all
// pages, one warp per page; (2) decode definition levels (RLE / bit-packed hybrid) per page;
// (3) decode values per page — PLAIN, PLAIN/RLE_DICTIONARY, FIXED_LEN_BYTE_ARRAY decimals — with
// one CTA per page: one thread parses a batch of run headers, all warps expand the runs;
// (4) strings: lengths -> scan -> chars copy; (5) only if a column really has NULLs, scatter the
// dense values to their rows.  Flat schemas (what Spark/TPC-H tables are); nested -> UNSUPPORTED.
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <chrono>
#include <thread>
#include <atomic>
#include <map>
#include "prim.cuh"

namespace b2 {

// ------------------------------------------------------------------------------------------------
// thrift compact protocol reader (host)
struct TReader {
  const uint8_t* p;
  const uint8_t* end;
  explicit TReader(const uint8_t* b, const uint8_t* e) : p(b), end(e) {}
  uint8_t byte() { if (p >= end) throw Error(B2_ERR_INVALID, "parquet: truncated thrift data"); return *p++; }
  uint64_t varint() {
    uint64_t v = 0; int shift = 0;
    while (true) { uint8_t b = byte(); v |= (uint64_t)(b & 0x7f) << shift; if (!(b & 0x80)) break; shift += 7; if (shift > 63) throw Error(B2_ERR_INVALID, "parquet: bad varint"); }
    return v;
  }
  int64_t zigzag() { uint64_t v = varint(); return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
  std::string str() { uint64_t n = varint(); if ((uint64_t)(end - p) < n) throw Error(B2_ERR_INVALID, "parquet: truncated string"); std::string s((const char*)p, n); p += n; return s; }
  // field header: returns false at STOP.  type: 1/2 bool true/false, 3 i8, 4 i16, 5 i32, 6 i64, 7 double, 8 binary, 9 list, 10 set, 11 map, 12 struct
  bool field(int& id, int& type, int& last) {
    uint8_t b = byte();
    if (b == 0) return false;
    type = b & 0x0f;
    int delta = b >> 4;
    if (delta) id = last + delta; else id = (int)zigzag();
    last = id;
    return true;
  }
  void list_header(int& n, int& etype) { uint8_t b = byte(); etype = b & 0x0f; n = b >> 4; if (n == 15) n = (int)varint(); }
  void skip(int type) {
    switch (type) {
      case 1: case 2: break;
      case 3: byte(); break;
      case 4: case 5: case 6: zigzag(); break;
      case 7: for (int i = 0; i < 8; i++) byte(); break;
      case 8: str(); break;
      case 9: case 10: { int n, et; list_header(n, et); for (int i = 0; i < n; i++) skip(et == 1 || et == 2 ? 3 : et); } break;
      case 11: { uint64_t n = varint(); if (n) { uint8_t kv = byte(); for (uint64_t i = 0; i < n; i++) { skip(kv >> 4); skip(kv & 15); } } } break;
      case 12: { int id, t, last = 0; while (field(id, t, last)) skip(t); } break;
      default: throw Error(B2_ERR_INVALID, "parquet: unknown thrift type");
    }
  }
};

enum { PT_BOOLEAN = 0, PT_INT32 = 1, PT_INT64 = 2, PT_INT96 = 3, PT_FLOAT = 4, PT_DOUBLE = 5, PT_BYTE_ARRAY = 6, PT_FLBA = 7 };
enum { ENC_PLAIN = 0, ENC_PLAIN_DICT = 2, ENC_RLE = 3, ENC_BIT_PACKED = 4, ENC_DELTA_BINARY = 5, ENC_RLE_DICT = 8 };
enum { PG_DATA = 0, PG_INDEX = 1, PG_DICT = 2, PG_DATA_V2 = 3 };
enum { CODEC_NONE = 0, CODEC_SNAPPY = 1 };

struct SchemaElem {
  int type = -1, type_length = 0, repetition = 0, num_children = 0, converted = -1, scale = 0, precision = 0;
  std::string name;
  bool lt_decimal = false, lt_date = false, lt_timestamp = false, lt_string = false;
  int lt_ts_unit = 0;  // 1 millis 2 micros 3 nanos
  int lt_int_bits = 0;
};
struct ChunkMeta {
  int type = -1, codec = 0;
  int64_t num_values = 0, total_compressed = 0, total_uncompressed = 0, data_page_offset = 0, dict_page_offset = -1;
  std::vector<std::string> path;
};
struct RowGroupMeta { int64_t num_rows = 0; std::vector<ChunkMeta> chunks; };
struct FileMeta { std::vector<SchemaElem> schema; int64_t num_rows = 0; std::vector<RowGroupMeta> row_groups; };

static void parse_logical_type(TReader& r, SchemaElem& e) {
  int id, t, last = 0;
  while (r.field(id, t, last)) {
    if (t != 12) { r.skip(t); continue; }
    int id2, t2, last2 = 0;
    switch (id) {
      case 1: e.lt_string = true; r.skip(12); break;
      case 5: e.lt_decimal = true; while (r.field(id2, t2, last2)) { if (id2 == 1) e.scale = (int)r.zigzag(); else if (id2 == 2) e.precision = (int)r.zigzag(); else r.skip(t2); } break;
      case 6: e.lt_date = true; r.skip(12); break;
      case 8:
        e.lt_timestamp = true;
        while (r.field(id2, t2, last2)) {
          if (id2 == 2 && t2 == 12) { int id3, t3, last3 = 0; while (r.field(id3, t3, last3)) { e.lt_ts_unit = id3; r.skip(t3); } }
          else r.skip(t2);
        }
        break;
      case 10: while (r.field(id2, t2, last2)) { if (id2 == 1) e.lt_int_bits = (int8_t)r.byte(); else r.skip(t2); } break;
      default: r.skip(12); break;
    }
  }
}

static FileMeta parse_footer(const uint8_t* buf, int64_t len) {
  if (len < 12 || memcmp(buf, "PAR1", 4) != 0 || memcmp(buf + len - 4, "PAR1", 4) != 0) throw Error(B2_ERR_INVALID, "parquet: missing PAR1 magic");
  uint32_t flen;
  memcpy(&flen, buf + len - 8, 4);
  if ((int64_t)flen + 12 > len) throw Error(B2_ERR_INVALID, "parquet: bad footer length");
  TReader r(buf + len - 8 - flen, buf + len - 8);
  FileMeta fm;
  int id, t, last = 0;
  while (r.field(id, t, last)) {
    if (id == 2 && t == 9) {
      int n, et; r.list_header(n, et);
      for (int i = 0; i < n; i++) {
        SchemaElem e; int id2, t2, last2 = 0;
        while (r.field(id2, t2, last2)) {
          switch (id2) {
            case 1: e.type = (int)r.zigzag(); break;
            case 2: e.type_length = (int)r.zigzag(); break;
            case 3: e.repetition = (int)r.zigzag(); break;
            case 4: e.name = r.str(); break;
            case 5: e.num_children = (int)r.zigzag(); break;
            case 6: e.converted = (int)r.zigzag(); break;
            case 7: e.scale = (int)r.zigzag(); break;
            case 8: e.precision = (int)r.zigzag(); break;
            case 10: if (t2 == 12) parse_logical_type(r, e); else r.skip(t2); break;
            default: r.skip(t2); break;
          }
        }
        fm.schema.push_back(e);
      }
    } else if (id == 3) {
      fm.num_rows = r.zigzag();
    } else if (id == 4 && t == 9) {
      int n, et; r.list_header(n, et);
      for (int i = 0; i < n; i++) {
        RowGroupMeta rg; int id2, t2, last2 = 0;
        while (r.field(id2, t2, last2)) {
          if (id2 == 1 && t2 == 9) {
            int nc, ect; r.list_header(nc, ect);
            for (int c = 0; c < nc; c++) {
              ChunkMeta cm; int id3, t3, last3 = 0;
              while (r.field(id3, t3, last3)) {
                if (id3 == 3 && t3 == 12) {
                  int id4, t4, last4 = 0;
                  while (r.field(id4, t4, last4)) {
                    switch (id4) {
                      case 1: cm.type = (int)r.zigzag(); break;
                      case 3: { int np, pt; r.list_header(np, pt); for (int k = 0; k < np; k++) cm.path.push_back(r.str()); } break;
                      case 4: cm.codec = (int)r.zigzag(); break;
                      case 5: cm.num_values = r.zigzag(); break;
                      case 6: cm.total_uncompressed = r.zigzag(); break;
                      case 7: cm.total_compressed = r.zigzag(); break;
                      case 9: cm.data_page_offset = r.zigzag(); break;
                      case 11: cm.dict_page_offset = r.zigzag(); break;
                      default: r.skip(t4); break;
                    }
                  }
                } else r.skip(t3);
              }
              rg.chunks.push_back(cm);
            }
          } else if (id2 == 3) rg.num_rows = r.zigzag();
          else r.skip(t2);
        }
        fm.row_groups.push_back(rg);
      }
    } else r.skip(t);
  }
  return fm;
}

// ------------------------------------------------------------------------------------------------
// device-side descriptors
struct PageD {
  int64_t src_off;      // payload offset in the file buffer
  int64_t dst_off;      // payload offset in the scratch buffer (-1: read in place from the file buffer)
  int32_t comp_size, uncomp_size;
  int32_t num_values;   // rows in the page (nulls included)
  int32_t encoding;
  int32_t kind;         // PG_*
  int32_t chunk;        // index into ChunkD
  int32_t lvl_bytes;    // v2: bytes of (uncompressed) rep+def levels in front of the values
  int32_t compressed;   // payload (v2: the part after the levels) is snappy compressed
  int64_t row_start;    // first row of this page inside the output column
  int64_t value_base;   // first dense value of this page inside the column
};
struct ChunkD {
  int32_t col;          // output column
  int32_t phys;         // PT_*
  int32_t type_length;
  int32_t max_def;      // 0 REQUIRED, 1 OPTIONAL
  int32_t dict_page;    // page index or -1
  int32_t dict_count;
  int64_t dict_str_off; // strings: first entry of this chunk in the dictionary offset arrays
};
struct ColD {
  int32_t out_dtype, out_width;
  int32_t phys, type_length;
  int32_t conv;         // 0 copy, 1 *1000 (millis -> micros), 2 big-endian FLBA -> integer, 3 narrow int32, 4 boolean bits, 5 string
  void* dense;          // fixed width: dense values
  int64_t* str_src;     // strings: absolute source address of each value's bytes
  int32_t* str_len;
  uint8_t* lvl;         // per-row validity bytes (max_def > 0)
};

__device__ __forceinline__ const uint8_t* page_ptr(const PageD& pg, const uint8_t* file, const uint8_t* scratch) {
  return pg.dst_off >= 0 ? scratch + pg.dst_off : file + pg.src_off;
}

// ---- snappy: one warp per page, 32 candidate element starts parsed per step ---------------------
// An LZ77 stream is sequential per page; pages are independent (tens of thousands per partition).
// Per warp the compressed input is staged through a shared-memory ring and the output through a
// second ring that serves back-references up to 2 KB and is flushed to HBM as 16-byte stores.
// Each step looks at a 32-byte window of the input: every lane decodes the element that WOULD start
// at its byte (header size, lengths, offset), the true element chain is then walked from lane 0 with
// shuffles (two elements per hop), output positions come from a warp scan, all short literals are
// copied by their own lanes at once, and only the back-references are replayed in order.
constexpr int SN_WARPS = 1;            // pages (warps) per CTA: finest scheduling grain, ~24 pages resident per SM
constexpr int SN_IN = 1024;            // input ring bytes
constexpr int SN_OUT = 8192;           // output ring bytes
constexpr int SN_HIST = 4096;          // back-reference distance served from the ring (older bytes are already in HBM)

struct SnappyWarp {
  uint8_t in[SN_IN];
  uint8_t out[SN_OUT];
};

// Input positions are counted from the 16-byte aligned address at or below the page's first byte (the caller
// starts ip at that misalignment), so a refill is one 16-byte load + one 16-byte shared store per lane.
// Reads up to 15 bytes outside [in, in + len): inside the file buffer (>= 16 bytes in front: "PAR1" + the first
// page header; >= 16 bytes of slack behind, see b2_parquet_decode_device).
__device__ __forceinline__ void sn_refill(SnappyWarp& w, const uint8_t* __restrict__ src_al, uint32_t in_len, uint32_t& loaded, uint32_t ip, int lane) {
  while (loaded < in_len && loaded <= ip + (SN_IN - 512)) {   // (ip starts at the misalignment, above loaded == 0)
    const uint32_t pos = loaded + lane * 16;
    if (pos < in_len) *reinterpret_cast<uint4*>(&w.in[pos & (SN_IN - 1)]) = *reinterpret_cast<const uint4*>(src_al + pos);
    loaded = min(loaded + 512u, in_len);
  }
  __syncwarp();
}

// byte copy between two non-overlapping ranges that do not wrap: loads of a group are issued before its stores
__device__ __forceinline__ void sn_copy(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, uint32_t len) {
  uint32_t k = 0;
  for (; k + 4 <= len; k += 4) {
    const uint8_t a = s[k], b = s[k + 1], c = s[k + 2], e = s[k + 3];
    d[k] = a; d[k + 1] = b; d[k + 2] = c; d[k + 3] = e;
  }
  for (; k < len; k++) d[k] = s[k];
}
__device__ __forceinline__ bool sn_nowrap(uint32_t p, uint32_t len, uint32_t size) { return (p & (size - 1)) + len <= size; }

// write ring bytes [flushed, target) to HBM: byte head up to 16-byte alignment, 512-byte slabs of
// 16-byte stores, and (when `all`) a byte tail
__device__ __forceinline__ void sn_flush(SnappyWarp& w, uint8_t* __restrict__ dst, uint32_t& flushed, uint32_t target, int lane, bool all) {
  if (flushed >= target) return;
  // 16-byte stores need the HBM address and the ring index aligned together
  const bool can_vec = (reinterpret_cast<uintptr_t>(dst) & 15) == 0;
  if (!can_vec) all = true;
  if (can_vec && (flushed & 15) && (all || target - flushed >= 512 + 16)) {
    const uint32_t n = min(16 - (flushed & 15), target - flushed);
    if (lane < (int)n) dst[flushed + lane] = w.out[(flushed + lane) & (SN_OUT - 1)];
    flushed += n;
  }
  if (can_vec && (flushed & 15) == 0) {
    while (target - flushed >= 512) {
      const uint4 v = *reinterpret_cast<const uint4*>(&w.out[(flushed + lane * 16) & (SN_OUT - 1)]);
      *reinterpret_cast<uint4*>(dst + flushed + lane * 16) = v;
      flushed += 512;
    }
  }
  if (all) {
    for (uint32_t k = flushed + lane; k < target; k += 32) dst[k] = w.out[k & (SN_OUT - 1)];
    flushed = target;
  }
}

__global__ void __launch_bounds__(SN_WARPS * 32) snappy_kernel(const PageD* __restrict__ pages, const int32_t* __restrict__ todo, int ntodo,
                                                               const uint8_t* __restrict__ file, uint8_t* __restrict__ scratch, int32_t* __restrict__ errors,
                                                               const int32_t* __restrict__ gate) {
  __shared__ __align__(16) SnappyWarp s_w[SN_WARPS];
  const int lane = threadIdx.x & 31;
  const int wi = threadIdx.x >> 5;
  const int wg = blockIdx.x * SN_WARPS + wi;
  if (wg >= ntodo) return;
  if (gate && gate[wg] == 0) return;  // big page already decoded by the CTA-wide kernel
  SnappyWarp& w = s_w[wi];
  const PageD pg = pages[todo[wg]];
  const uint8_t* in = file + pg.src_off;
  uint8_t* out = scratch + pg.dst_off;
  uint32_t in_len = (uint32_t)pg.comp_size, out_len = (uint32_t)pg.uncomp_size;
  if (pg.lvl_bytes) {  // v2: levels are stored uncompressed in front of the compressed values
    const uint32_t lvl = (uint32_t)pg.lvl_bytes;
    for (uint32_t k = lane; k < lvl; k += 32) out[k] = in[k];
    in += lvl; out += lvl; in_len -= lvl; out_len -= lvl;
  }
  uint8_t* dst = out;
  const uint32_t a0 = (uint32_t)(reinterpret_cast<uintptr_t>(in) & 15);
  in -= a0; in_len += a0;                 // positions are relative to the aligned address from here on
  uint32_t ip = a0, op = 0, loaded = 0, flushed = 0;
  sn_refill(w, in, in_len, loaded, ip, lane);
  uint32_t ulen = 0;
  { int shift = 0; while (ip < in_len) { const uint8_t b = w.in[ip & (SN_IN - 1)]; ip++; ulen |= (uint32_t)(b & 0x7f) << shift; if (!(b & 0x80)) break; shift += 7; } }
  bool bad = ulen != out_len;
  while (!bad && ip < in_len && op < out_len) {
    if (loaded - ip < 40 && loaded < in_len) sn_refill(w, in, in_len, loaded, ip, lane);
    // ---- 1. every lane decodes the element that would start at byte ip + lane
    const uint32_t q = ip + lane;
    const uint32_t tag = w.in[q & (SN_IN - 1)];
    const uint32_t b1 = w.in[(q + 1) & (SN_IN - 1)], b2 = w.in[(q + 2) & (SN_IN - 1)], b3 = w.in[(q + 3) & (SN_IN - 1)], b4 = w.in[(q + 4) & (SN_IN - 1)];
    const uint32_t t = tag & 3;
    uint32_t len, off = 0, hdr;
    if (t == 0) {
      len = tag >> 2;
      if (len < 60) { len += 1; hdr = 1; }
      else { const uint32_t nb = len - 59; const uint32_t v = b1 | (b2 << 8) | (b3 << 16) | (b4 << 24); len = (nb == 4 ? v : (v & ((1u << (8 * nb)) - 1))) + 1; hdr = 1 + nb; }
    } else if (t == 1) { len = 4 + ((tag >> 2) & 7); off = ((tag >> 5) << 8) | b1; hdr = 2; }
    else if (t == 2) { len = (tag >> 2) + 1; off = b1 | (b2 << 8); hdr = 3; }
    else { len = (tag >> 2) + 1; off = b1 | (b2 << 8) | (b3 << 16) | (b4 << 24); hdr = 5; }
    const bool is_lit = t == 0;
    const uint32_t esz = hdr + (is_lit ? len : 0);          // compressed bytes of this element
    const uint32_t avail = min(32u, in_len - ip);
    // a literal whose data does not end inside the window is streamed separately ("long")
    const bool is_long = is_lit && (lane + esz > 32 || len > 31);
    const uint32_t n1 = (lane >= avail) ? 64u : (is_long ? 64u : min(lane + esz, 64u));  // next start, 64 = leaves the window
    uint32_t n2 = __shfl_sync(0xffffffffu, n1, n1 & 31);
    if (n1 >= 32) n2 = 64u;
    // ---- 2. walk the true chain from lane 0, two elements per hop
    uint32_t M = 0, cur = 0;
    while (cur < 32) {
      M |= 1u << cur;
      const uint32_t a = __shfl_sync(0xffffffffu, n1, cur);
      const uint32_t c2 = __shfl_sync(0xffffffffu, n2, cur);
      if (a < 32) M |= 1u << a;
      cur = c2;
    }
    M &= (avail >= 32 ? 0xffffffffu : ((1u << avail) - 1u));
    const bool mine = (M >> lane) & 1u;
    // the last true element may be a long literal (handled after the window) — never two of them
    const uint32_t longmask = __ballot_sync(0xffffffffu, mine && is_long);
    const int long_lane = longmask ? (__ffs(longmask) - 1) : -1;
    // header bytes of a true element must be loaded; a truncated stream is an error
    const bool trunc = mine && (q + hdr > in_len || (is_lit && !is_long && q + esz > in_len));
    // ---- 3. output positions by warp scan over the true short elements
    const uint32_t myo = (mine && !is_long) ? len : 0;
    uint32_t inc = myo;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
    const uint32_t opos = op + inc - myo;
    const bool badcopy = mine && !is_lit && (off == 0 || off > opos);
    if (__any_sync(0xffffffffu, trunc || badcopy) || op + total > out_len) { bad = true; break; }
    // ---- 4a. everything that does not depend on this window's own output, all lanes at once:
    //          short literals, back-references into earlier output (ring), far back-references (HBM:
    //          anything older than SN_HIST is already flushed because < 1 KB is ever pending here)
    const bool indep = mine && !is_lit && (opos - off + len <= op);
    if (mine && is_lit && !is_long) {
      if (sn_nowrap(opos, len, SN_OUT) && sn_nowrap(q + hdr, len, SN_IN)) sn_copy(&w.out[opos & (SN_OUT - 1)], &w.in[(q + hdr) & (SN_IN - 1)], len);
      else for (uint32_t k = 0; k < len; k++) w.out[(opos + k) & (SN_OUT - 1)] = w.in[(q + hdr + k) & (SN_IN - 1)];
    } else if (indep) {
      if (off <= SN_HIST) {
        if (sn_nowrap(opos, len, SN_OUT) && sn_nowrap(opos - off, len, SN_OUT)) sn_copy(&w.out[opos & (SN_OUT - 1)], &w.out[(opos - off) & (SN_OUT - 1)], len);
        else for (uint32_t k = 0; k < len; k++) w.out[(opos + k) & (SN_OUT - 1)] = w.out[(opos - off + k) & (SN_OUT - 1)];
      } else {
        // far back-reference: the bytes are in HBM (flushed by this warp).  Two aligned 8-byte loads cover 8 source
        // bytes at any alignment: 4x fewer L1 transactions than byte loads, and both loads are in flight together.
        const uint8_t* src = dst + opos - off;
        for (uint32_t k = 0; k < len; k += 8) {
          const uintptr_t ad = reinterpret_cast<uintptr_t>(src + k);
          const uint64_t* al = reinterpret_cast<const uint64_t*>(ad & ~uintptr_t(7));
          const uint32_t sh = (uint32_t)(ad & 7) * 8;
          const uint64_t w0 = al[0], w1 = al[1];
          const uint64_t v = sh ? (w0 >> sh) | (w1 << (64 - sh)) : w0;
          const uint32_t n = min(8u, len - k);
          for (uint32_t b = 0; b < n; b++) w.out[(opos + k + b) & (SN_OUT - 1)] = (uint8_t)(v >> (8 * b));
        }
      }
    }
    __syncwarp();
    // ---- 4b. back-references into this window's output, replayed in stream order
    uint32_t cm = __ballot_sync(0xffffffffu, mine && !is_lit && !indep);
    while (cm) {
      const int l = __ffs(cm) - 1;
      cm &= cm - 1;
      const uint32_t o = __shfl_sync(0xffffffffu, opos, l), f = __shfl_sync(0xffffffffu, off, l), n = __shfl_sync(0xffffffffu, len, l);
      uint8_t v = 0, v2 = 0;  // f <= window span here, always inside the ring
      if (lane < (int)n) v = w.out[(o - f + (f >= n ? lane : lane % f)) & (SN_OUT - 1)];
      if (lane + 32 < (int)n) v2 = w.out[(o - f + (f >= n ? lane + 32 : (lane + 32) % f)) & (SN_OUT - 1)];
      __syncwarp();
      if (lane < (int)n) w.out[(o + lane) & (SN_OUT - 1)] = v;
      if (lane + 32 < (int)n) w.out[(o + lane + 32) & (SN_OUT - 1)] = v2;
      __syncwarp();
    }
    op += total;
    // end of the short elements = start of the long literal, or the next window
    const uint32_t endp = mine ? (is_long ? lane : lane + esz) : 0;
    ip += __reduce_max_sync(0xffffffffu, endp);
    // ---- 4c. a long literal streams through the rings
    if (long_lane >= 0) {
      const uint32_t llen = __shfl_sync(0xffffffffu, len, long_lane), lhdr = __shfl_sync(0xffffffffu, hdr, long_lane);
      if (ip + lhdr + llen > in_len || op + llen > out_len) { bad = true; break; }
      ip += lhdr;
      uint32_t left = llen;
      while (left) {
        const uint32_t n = min(left, 512u);
        if (loaded - ip < n) sn_refill(w, in, in_len, loaded, ip, lane);
        const uint32_t have = min(n, loaded - ip);
        if (have == 0) { bad = true; break; }
        for (uint32_t k = lane; k < have; k += 32) w.out[(op + k) & (SN_OUT - 1)] = w.in[(ip + k) & (SN_IN - 1)];
        __syncwarp();
        ip += have; op += have; left -= have;
        if (op - flushed >= 1024) { sn_flush(w, dst, flushed, op, lane, false); __syncwarp(); }
      }
    }
    if (op - flushed >= 512) { sn_flush(w, dst, flushed, op, lane, false); __syncwarp(); }
  }
  __syncwarp();
  sn_flush(w, dst, flushed, op, lane, true);
  if ((bad || op != out_len) && lane == 0) atomicExch(errors, 1);
}

// ---- snappy for LARGE pages: one CTA (32 warps) per page, fully parallel LZ77 --------------------
// A 1 MB dictionary page is ~260 k LZ77 elements; on one warp it is the critical path of the whole
// decode.  Here the compressed stream is cut into 32 chunks.  (1) Each warp finds an element boundary
// near its chunk start by self-synchronisation: 32 lanes parse forward from 32 consecutive byte offsets
// until they agree.  (2) Each warp walks its chunk from its boundary and must land EXACTLY on the next
// warp's boundary; warp 0 starts at the true stream start, so success of every check proves every
// boundary by induction (otherwise the page falls back to the one-warp kernel).  (3) Output offsets
// by prefix sum.  (4) Second walk: literal bytes go to their final place, and every output byte j gets
// a source S[j] (itself for literals, j - offset for back-references).  (5) Pointer jumping
// S[j] = S[S[j]] until every byte points at a literal byte (log2(chain depth) rounds).
// (6) out[j] = out[S[j]].
constexpr int SB_WARPS = 32;
constexpr uint32_t SB_MIN_BYTES = 192 * 1024;   // uncompressed size from which a page takes this path

struct SnE { uint32_t esz, len, off, hdr; bool lit, ok; };
__device__ __forceinline__ SnE sn_parse(const uint8_t* __restrict__ in, uint32_t q, uint32_t in_len) {
  SnE e; e.esz = 1; e.len = 0; e.off = 0; e.hdr = 1; e.lit = true; e.ok = false;
  if (q >= in_len) return e;
  const uint32_t tag = in[q];
  const uint32_t b1 = q + 1 < in_len ? in[q + 1] : 0, b2 = q + 2 < in_len ? in[q + 2] : 0, b3 = q + 3 < in_len ? in[q + 3] : 0, b4 = q + 4 < in_len ? in[q + 4] : 0;
  const uint32_t t = tag & 3;
  if (t == 0) {
    uint32_t len = tag >> 2;
    if (len < 60) { e.len = len + 1; e.hdr = 1; }
    else { const uint32_t nb = len - 59; const uint32_t v = b1 | (b2 << 8) | (b3 << 16) | (b4 << 24); e.len = (nb == 4 ? v : (v & ((1u << (8 * nb)) - 1))) + 1; e.hdr = 1 + nb; }
    e.lit = true; e.esz = e.hdr + e.len;
    e.ok = (uint64_t)q + e.esz <= in_len;
  } else {
    e.lit = false;
    if (t == 1) { e.len = 4 + ((tag >> 2) & 7); e.off = ((tag >> 5) << 8) | b1; e.hdr = 2; }
    else if (t == 2) { e.len = (tag >> 2) + 1; e.off = b1 | (b2 << 8); e.hdr = 3; }
    else { e.len = (tag >> 2) + 1; e.off = b1 | (b2 << 8) | (b3 << 16) | (b4 << 24); e.hdr = 5; }
    e.esz = e.hdr;
    e.ok = q + e.hdr <= in_len && e.off != 0;
  }
  return e;
}

// Walk elements [ip_start, ip_stop) with the 32-byte window method.  EMIT = false: only sum output
// lengths.  EMIT = true: place literals and write the source map.  Returns false on any inconsistency
// (including not landing exactly on ip_stop).
template <bool EMIT>
__device__ bool sn_walk(const uint8_t* __restrict__ in, uint32_t in_len, uint32_t ip_start, uint32_t ip_stop, uint32_t op_start, uint32_t out_len,
                        uint8_t* __restrict__ out, uint32_t* __restrict__ S, uint32_t sbase, uint32_t& out_total) {
  const int lane = threadIdx.x & 31;
  uint32_t ip = ip_start, op = op_start;
  while (ip < ip_stop) {
    const uint32_t q = ip + lane;
    const uint32_t avail = min(32u, ip_stop - ip);
    const SnE e = sn_parse(in, q, in_len);
    const bool is_long = e.lit && (lane + e.esz > 32 || e.len > 31);
    const uint32_t n1 = (lane >= avail) ? 64u : (is_long ? 64u : min(lane + e.esz, 64u));
    uint32_t n2 = __shfl_sync(0xffffffffu, n1, n1 & 31);
    if (n1 >= 32) n2 = 64u;
    uint32_t M = 0, cur = 0;
    while (cur < 32) {
      M |= 1u << cur;
      const uint32_t a = __shfl_sync(0xffffffffu, n1, cur);
      const uint32_t c2 = __shfl_sync(0xffffffffu, n2, cur);
      if (a < 32) M |= 1u << a;
      cur = c2;
    }
    M &= (avail >= 32 ? 0xffffffffu : ((1u << avail) - 1u));
    const bool mine = (M >> lane) & 1u;
    const uint32_t longmask = __ballot_sync(0xffffffffu, mine && is_long);
    const int long_lane = longmask ? (__ffs(longmask) - 1) : -1;
    const uint32_t myo = (mine && !is_long) ? e.len : 0;
    uint32_t inc = myo;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
    const uint32_t total = __shfl_sync(0xffffffffu, inc, 31);
    const uint32_t opos = op + inc - myo;
    const bool bad = mine && (!e.ok || (EMIT && !e.lit && e.off > opos));  // offsets can only be checked with absolute positions
    if (__any_sync(0xffffffffu, bad) || (uint64_t)op + total > out_len) return false;
    if (EMIT && mine && !is_long) {
      if (e.lit) { for (uint32_t k = 0; k < e.len; k++) { out[opos + k] = in[q + e.hdr + k]; S[opos + k] = sbase + opos + k; } }
      else { for (uint32_t k = 0; k < e.len; k++) S[opos + k] = sbase + opos + k - e.off; }
    }
    op += total;
    const uint32_t endp = mine ? (is_long ? lane : lane + e.esz) : 0;
    ip += __reduce_max_sync(0xffffffffu, endp);
    if (long_lane >= 0) {
      const uint32_t llen = __shfl_sync(0xffffffffu, e.len, long_lane), lhdr = __shfl_sync(0xffffffffu, e.hdr, long_lane);
      const bool lok = __shfl_sync(0xffffffffu, (uint32_t)e.ok, long_lane) != 0;
      if (!lok || (uint64_t)op + llen > out_len) return false;
      if (EMIT) for (uint32_t k = lane; k < llen; k += 32) { out[op + k] = in[ip + lhdr + k]; S[op + k] = sbase + op + k; }
      ip += lhdr + llen; op += llen;
    }
  }
  out_total = op - op_start;
  return ip == ip_stop;
}

__global__ void __launch_bounds__(SB_WARPS * 32) snappy_big_kernel(const PageD* __restrict__ pages, const int32_t* __restrict__ todo,
                                                                   const int64_t* __restrict__ s_off, const uint8_t* __restrict__ file,
                                                                   uint8_t* __restrict__ scratch, uint32_t* __restrict__ S_all, int32_t* __restrict__ fail) {
  __shared__ uint32_t s_cand[SB_WARPS + 1], s_olen[SB_WARPS], s_op[SB_WARPS + 1];
  __shared__ int s_bad;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const PageD pg = pages[todo[blockIdx.x]];
  const uint8_t* in = file + pg.src_off;
  uint8_t* out = scratch + pg.dst_off;
  uint32_t in_len = (uint32_t)pg.comp_size, out_len = (uint32_t)pg.uncomp_size;
  if (pg.lvl_bytes) {
    const uint32_t lvl = (uint32_t)pg.lvl_bytes;
    for (uint32_t k = threadIdx.x; k < lvl; k += blockDim.x) out[k] = in[k];
    in += lvl; out += lvl; in_len -= lvl; out_len -= lvl;
  }
  uint32_t* S = S_all + s_off[blockIdx.x];
  if (threadIdx.x == 0) s_bad = 0;
  // every phase below walks the compressed bytes with dependent loads: pull the whole page into L2 first
  for (uint32_t k = threadIdx.x * 128u; k < in_len; k += blockDim.x * 128u) asm volatile("prefetch.global.L2 [%0];" ::"l"(in + k));
  __syncthreads();
  // preamble
  uint32_t ip0 = 0, ulen = 0;
  { int shift = 0; while (ip0 < in_len) { const uint8_t b = in[ip0++]; ulen |= (uint32_t)(b & 0x7f) << shift; if (!(b & 0x80)) break; shift += 7; } }
  if (ulen != out_len) { if (threadIdx.x == 0) fail[blockIdx.x] = 1; return; }  // fail codes: 1 preamble, 2 boundary, 3 verify, 4 length, 5 emit
  const uint32_t C = (in_len - ip0 + SB_WARPS - 1) / SB_WARPS;
  // ---- (1) boundary near each chunk start
  {
    uint32_t cand;
    if (w == 0) cand = ip0;
    else {
      const uint32_t b = min(ip0 + (uint32_t)w * C, in_len);
      uint32_t pos = min(b + lane, in_len);
      uint32_t T = b + 256;
      bool agreed = false;
      uint32_t best = in_len;
      // chains that start inside literal bytes misparse; most re-synchronise within a few elements,
      // a few run off the end.  Take the position a majority of the 32 chains agrees on — the
      // verification walk of the previous warp proves (or refutes) it.
      for (int att = 0; att < 16 && !agreed; att++, T += 512) {
        while (pos < T && pos < in_len) { const SnE e = sn_parse(in, pos, in_len); if (!e.ok) { pos = 0xffffffffu; break; } pos += e.esz; }
        const uint32_t grp = __match_any_sync(0xffffffffu, pos);
        const bool maj = pos != 0xffffffffu && __popc(grp) >= 17;
        const uint32_t who = __ballot_sync(0xffffffffu, maj);
        if (who) { best = __shfl_sync(0xffffffffu, pos, __ffs(who) - 1); agreed = true; }
      }
      cand = min(best, in_len);
      if (!agreed && lane == 0) s_bad = 1;
    }
    if (lane == 0) s_cand[w] = cand;
    if (threadIdx.x == 0) s_cand[SB_WARPS] = in_len;
  }
  __syncthreads();
  if (s_bad) { if (threadIdx.x == 0) fail[blockIdx.x] = 2; return; }
  // boundaries must be non-decreasing (a later chunk may start inside an earlier warp's overshoot)
  // ---- (2) verification walk + output length per chunk
  {
    const uint32_t a = s_cand[w], b = s_cand[w + 1];
    uint32_t olen = 0;
    bool ok = a <= b;
    if (ok && a < b) ok = sn_walk<false>(in, in_len, a, b, 0, 0xffffffffu, nullptr, nullptr, 0, olen);
    if (lane == 0) { s_olen[w] = olen; if (!ok) s_bad = 1; }
  }
  __syncthreads();
  if (s_bad) { if (threadIdx.x == 0) fail[blockIdx.x] = 3; return; }
  // ---- (3) output offsets
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int k = 0; k < SB_WARPS; k++) { s_op[k] = run; run += s_olen[k]; }
    s_op[SB_WARPS] = run;
    if (run != out_len) s_bad = 1;
  }
  __syncthreads();
  if (s_bad) { if (threadIdx.x == 0) fail[blockIdx.x] = 4; return; }
  // ---- (4) emit literals + source map
  {
    const uint32_t a = s_cand[w], b = s_cand[w + 1];
    uint32_t olen = 0;
    bool ok = true;
    if (a < b) ok = sn_walk<true>(in, in_len, a, b, s_op[w], out_len, out, S, (uint32_t)s_off[blockIdx.x], olen);
    if (lane == 0 && !ok) s_bad = 1;
  }
  __threadfence_block();
  __syncthreads();
  if (s_bad) { if (threadIdx.x == 0) fail[blockIdx.x] = 5; return; }
}

// (5) one pointer-jumping round over the source maps of ALL large pages (values are absolute indexes
// into S): S[j] = S[S[j]].  20 rounds resolve chains of up to 2^20 back-references.
__global__ void __launch_bounds__(256) snappy_jump_kernel(uint32_t* __restrict__ S, uint32_t total) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j0 = blockIdx.x * blockDim.x + threadIdx.x; j0 < total; j0 += 4 * stride) {
    uint32_t j[4], s1[4], s2[4];
#pragma unroll
    for (int u = 0; u < 4; u++) { j[u] = j0 + u * stride; s1[u] = j[u] < total ? S[j[u]] : j[u]; }
#pragma unroll
    for (int u = 0; u < 4; u++) s2[u] = (s1[u] != j[u] && s1[u] < total) ? *reinterpret_cast<volatile uint32_t*>(&S[s1[u]]) : s1[u];
#pragma unroll
    for (int u = 0; u < 4; u++) if (s2[u] != s1[u]) S[j[u]] = s2[u];
  }
}
// (6) every non-literal byte copies the literal byte its chain ends at
__global__ void __launch_bounds__(256) snappy_resolve_kernel(const uint32_t* __restrict__ S, uint8_t* __restrict__ out, uint32_t total) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < total; j += gridDim.x * blockDim.x) {
    const uint32_t s1 = S[j];
    if (s1 != j && s1 < total) out[j] = out[s1];
  }
}

// ---- RLE / bit-packed hybrid ---------------------------------------------------------------------
struct RunD { int32_t start, count, packed; uint32_t value; const uint8_t* data; };
constexpr int PQ_NT = 256;
constexpr int PQ_RUNS = 64;

__device__ __forceinline__ uint32_t extract_bits(const uint8_t* data, uint64_t bitpos, int bw) {
  const uint8_t* a = data + (bitpos >> 3);
  const uintptr_t base = reinterpret_cast<uintptr_t>(a) & ~(uintptr_t)7;
  const uint64_t w0 = *reinterpret_cast<const uint64_t*>(base), w1 = *reinterpret_cast<const uint64_t*>(base + 8);
  const int sh = (int)((reinterpret_cast<uintptr_t>(a) & 7) * 8 + (bitpos & 7));
  uint64_t v = w0 >> sh;
  if (sh) v |= w1 << (64 - sh);
  return (uint32_t)(v & ((bw >= 32) ? 0xffffffffull : ((1ull << bw) - 1)));
}

// CTA-cooperative decode of `count` values; Sink::put(k, v) is called once per value by some thread
template <typename Sink>
__device__ void decode_hybrid(const uint8_t* p, const uint8_t* end, int bw, int count, Sink& sink) {
  __shared__ RunD s_runs[PQ_RUNS];
  __shared__ int s_nruns, s_done;
  __shared__ const uint8_t* s_pos;
  if (threadIdx.x == 0) { s_pos = p; s_done = 0; }
  __syncthreads();
  const int vbytes = (bw + 7) >> 3;
  while (true) {
    if (threadIdx.x == 0) {
      const uint8_t* q = s_pos;
      int done = s_done, n = 0;
      while (n < PQ_RUNS && done < count && q < end) {
        uint32_t h = 0; int shift = 0;
        while (q < end) { uint8_t b = *q++; h |= (uint32_t)(b & 0x7f) << shift; if (!(b & 0x80)) break; shift += 7; }
        RunD r; r.start = done;
        if (h & 1) { const int groups = (int)(h >> 1); r.packed = 1; r.count = min(groups * 8, count - done); r.data = q; r.value = 0; q += (size_t)groups * bw; }
        else { r.packed = 0; r.count = min((int)(h >> 1), count - done); uint32_t v = 0; for (int k = 0; k < vbytes && q < end; k++) v |= (uint32_t)(*q++) << (8 * k); r.value = v; r.data = nullptr; }
        if (r.count <= 0) { if (!(h & 1) && (h >> 1) == 0) { done = count; } break; }
        done += r.count;
        s_runs[n++] = r;
      }
      if (n == 0) done = count;  // malformed / exhausted stream: stop
      s_nruns = n; s_done = done; s_pos = q;
    }
    __syncthreads();
    const int n = s_nruns;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int r = warp; r < n; r += PQ_NT / 32) {
      const RunD run = s_runs[r];
      if (run.packed) {
        // four values per lane in flight: bits -> index -> dictionary entry -> store is a chain of dependent loads
        int k = lane;
        for (; k + 96 < run.count; k += 128) {
          const uint32_t v0 = extract_bits(run.data, (uint64_t)k * bw, bw), v1 = extract_bits(run.data, (uint64_t)(k + 32) * bw, bw),
                         v2 = extract_bits(run.data, (uint64_t)(k + 64) * bw, bw), v3 = extract_bits(run.data, (uint64_t)(k + 96) * bw, bw);
          sink.put4(run.start + k, v0, v1, v2, v3);
        }
        for (; k < run.count; k += 32) sink.put(run.start + k, extract_bits(run.data, (uint64_t)k * bw, bw));
      } else for (int k = lane; k < run.count; k += 32) sink.put(run.start + k, run.value);
    }
    __syncthreads();
    if (s_done >= count) break;
  }
}

// ---- pass 1: definition levels -> per-row validity bytes + per-page non-null count ---------------
struct LevelSink {
  uint8_t* lvl; int max_def; unsigned int* cnt;
  __device__ __forceinline__ void put(int k, uint32_t v) { const bool ok = (int)v == max_def; lvl[k] = ok; if (ok) atomicAdd(cnt, 1u); }
  __device__ __forceinline__ void put4(int k, uint32_t a, uint32_t b, uint32_t c, uint32_t d) { put(k, a); put(k + 32, b); put(k + 64, c); put(k + 96, d); }
};
__device__ __forceinline__ const uint8_t* levels_of(const PageD& pg, const uint8_t* d, const uint8_t*& lv_end, const uint8_t*& values) {
  if (pg.kind == PG_DATA_V2) { lv_end = d + pg.lvl_bytes; values = d + pg.lvl_bytes; return d; }
  uint32_t n; memcpy(&n, d, 4);
  lv_end = d + 4 + n; values = d + 4 + n;
  return d + 4;
}
__global__ void __launch_bounds__(PQ_NT) levels_kernel(const PageD* __restrict__ pages, const int32_t* __restrict__ todo, const ChunkD* __restrict__ chunks,
                                                       const ColD* __restrict__ cols, const uint8_t* __restrict__ file, const uint8_t* __restrict__ scratch,
                                                       int32_t* __restrict__ nonnull) {
  __shared__ unsigned int s_cnt;
  const int pi = todo[blockIdx.x];
  const PageD pg = pages[pi];
  const ChunkD ch = chunks[pg.chunk];
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const uint8_t* d = page_ptr(pg, file, scratch);
  const uint8_t *lv_end, *vals;
  const uint8_t* lv = levels_of(pg, d, lv_end, vals);
  uint8_t* out_lvl = cols[ch.col].lvl + pg.row_start;
  // the usual page of a nullable column without NULLs: one RLE run "every level = max_def" — no per-row work
  {
    const uint8_t* q = lv;
    uint32_t hdr = 0; int sh = 0;
    while (q < lv_end && sh < 35) { const uint8_t b = *q++; hdr |= (uint32_t)(b & 0x7f) << sh; if (!(b & 0x80)) break; sh += 7; }
    if (q < lv_end && (hdr & 1u) == 0 && (int)(hdr >> 1) >= pg.num_values && pg.num_values > 0) {
      // (the per-row bytes are not written here: when the column turns out to have NULLs in other pages,
      //  fill_uniform_levels_kernel writes them for the all-valid / all-NULL pages afterwards)
      const bool ok = (int)(*q & 1u) == ch.max_def;
      if (threadIdx.x == 0) nonnull[pi] = ok ? pg.num_values : 0;
      return;
    }
  }
  LevelSink sink{out_lvl, ch.max_def, &s_cnt};
  decode_hybrid(lv, lv_end, 1, pg.num_values, sink);  // flat schema: max_def == 1 -> bit width 1
  __syncthreads();
  if (threadIdx.x == 0) nonnull[pi] = (int32_t)s_cnt;
}

// per-row validity bytes of the pages levels_kernel short-cut (every row valid, or every row NULL); launched only for
// columns that do contain NULLs somewhere
__global__ void __launch_bounds__(PQ_NT) fill_uniform_levels_kernel(const PageD* __restrict__ pages, const int32_t* __restrict__ todo, const ChunkD* __restrict__ chunks,
                                                                    const ColD* __restrict__ cols, const int32_t* __restrict__ nonnull,
                                                                    const uint8_t* __restrict__ col_has_nulls) {
  const int pi = todo[blockIdx.x];
  const PageD pg = pages[pi];
  const ChunkD ch = chunks[pg.chunk];
  if (!col_has_nulls[ch.col]) return;
  const int nn = nonnull[pi];
  if (nn != 0 && nn != pg.num_values) return;   // mixed page: the level decoder wrote its bytes
  uint8_t* out_lvl = cols[ch.col].lvl + pg.row_start;
  const uint8_t v = nn != 0;
  for (int k = threadIdx.x; k < pg.num_values; k += PQ_NT) out_lvl[k] = v;
}

// ---- pass 2: values ---------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t load_le(const uint8_t* p, int nbytes) {
  uint64_t v = 0;
  if ((reinterpret_cast<uintptr_t>(p) & (nbytes - 1)) == 0) {
    if (nbytes == 8) return *reinterpret_cast<const uint64_t*>(p);
    if (nbytes == 4) return *reinterpret_cast<const uint32_t*>(p);
  }
  if (nbytes == 8 || nbytes == 4) {
    // PLAIN values start right behind the (odd-sized) level bytes, so they are rarely aligned: two aligned 8-byte
    // loads and a funnel shift instead of a byte loop (the page buffers have >= 16 bytes of slack)
    const uintptr_t ad = reinterpret_cast<uintptr_t>(p);
    const uint64_t* al = reinterpret_cast<const uint64_t*>(ad & ~uintptr_t(7));
    const int sh = (int)(ad & 7) * 8;
    const uint64_t w0 = al[0];
    uint64_t x = w0 >> sh;
    if (sh + nbytes * 8 > 64) x |= al[1] << (64 - sh);
    return nbytes == 8 ? x : (x & 0xffffffffull);
  }
  for (int k = 0; k < nbytes; k++) v |= (uint64_t)p[k] << (8 * k);
  return v;
}
// big-endian two's complement of `len` bytes -> sign-extended (lo, hi)
__device__ __forceinline__ void load_be_int(const uint8_t* p, int len, uint64_t& lo, uint64_t& hi) {
  const uint64_t sign = (p[0] & 0x80) ? ~0ull : 0ull;
  lo = sign; hi = sign;
  for (int k = 0; k < len; k++) {
    hi = (hi << 8) | (lo >> 56);
    lo = (lo << 8) | p[k];
  }
}

struct ValueWriter {
  ColD col; int64_t base;  // dense index of this page's first value
  const uint8_t* dict; int dict_count; const int64_t* dict_src; const int32_t* dict_len;
  __device__ __forceinline__ void write_fixed(int64_t k, const uint8_t* src) {
    void* out = col.dense;
    const int64_t o = base + k;
    switch (col.conv) {
      case 0:
        if (col.out_width == 4) reinterpret_cast<uint32_t*>(out)[o] = (uint32_t)load_le(src, 4);
        else reinterpret_cast<uint64_t*>(out)[o] = load_le(src, 8);
        break;
      case 1: reinterpret_cast<int64_t*>(out)[o] = (int64_t)load_le(src, 8) * 1000; break;
      case 2: {
        uint64_t lo, hi; load_be_int(src, col.type_length, lo, hi);
        if (col.out_width == 4) reinterpret_cast<uint32_t*>(out)[o] = (uint32_t)lo;
        else if (col.out_width == 8) reinterpret_cast<uint64_t*>(out)[o] = lo;
        else { reinterpret_cast<uint64_t*>(out)[2 * o] = lo; reinterpret_cast<uint64_t*>(out)[2 * o + 1] = hi; }
      } break;
      case 3:
        if (col.out_width == 1) reinterpret_cast<int8_t*>(out)[o] = (int8_t)load_le(src, 4);
        else reinterpret_cast<int16_t*>(out)[o] = (int16_t)load_le(src, 4);
        break;
      default: break;
    }
  }
};
struct DictSink {
  ValueWriter w; int src_width; int32_t* errors;
  __device__ __forceinline__ void put(int k, uint32_t idx) {
    if ((int)idx >= w.dict_count) { atomicExch(errors, 2); return; }
    if (w.col.conv == 5) { w.col.str_src[w.base + k] = w.dict_src[idx]; w.col.str_len[w.base + k] = w.dict_len[idx]; }
    else w.write_fixed(k, w.dict + (size_t)idx * src_width);
  }
  // rows k, k+32, k+64, k+96: the four dictionary entries are fetched before the first store
  __device__ __forceinline__ void put4(int k, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    if (w.col.conv == 0 && (src_width == 4 || src_width == 8) && w.col.out_width == src_width &&
        (reinterpret_cast<uintptr_t>(w.dict) & (uintptr_t)(src_width - 1)) == 0 && (int)max(max(a, b), max(c, d)) < w.dict_count) {
      if (src_width == 4) {
        const uint32_t* dp = reinterpret_cast<const uint32_t*>(w.dict);
        const uint32_t x0 = dp[a], x1 = dp[b], x2 = dp[c], x3 = dp[d];
        uint32_t* o = reinterpret_cast<uint32_t*>(w.col.dense) + w.base + k; o[0] = x0; o[32] = x1; o[64] = x2; o[96] = x3;
      } else {
        const uint64_t* dp = reinterpret_cast<const uint64_t*>(w.dict);
        const uint64_t x0 = dp[a], x1 = dp[b], x2 = dp[c], x3 = dp[d];
        uint64_t* o = reinterpret_cast<uint64_t*>(w.col.dense) + w.base + k; o[0] = x0; o[32] = x1; o[64] = x2; o[96] = x3;
      }
      return;
    }
    put(k, a); put(k + 32, b); put(k + 64, c); put(k + 96, d);
  }
};

// ---- DELTA_BINARY_PACKED (INT32 / INT64) ----------------------------------------------------------------------
// header: block size, miniblocks per block, value count, first value (zigzag); then per block: min delta (zigzag),
// one bit width per miniblock, the bit-packed miniblocks.  value[i] = value[i-1] + min_delta + delta[i], wrapping.
// Block headers are varints, so one thread walks them — PQ_NT miniblocks at a time; then every thread sums its own
// miniblock, an exclusive scan of the miniblock totals gives each thread its starting value, and the miniblocks
// are expanded in parallel.
__device__ __forceinline__ uint64_t dl_uleb(const uint8_t*& p, const uint8_t* end) {
  uint64_t v = 0; int sh = 0;
  while (p < end) { const uint8_t b = *p++; v |= (uint64_t)(b & 0x7f) << sh; if (!(b & 0x80)) break; sh += 7; if (sh > 63) break; }
  return v;
}
__device__ __forceinline__ int64_t dl_zigzag(uint64_t v) { return (int64_t)(v >> 1) ^ -(int64_t)(v & 1); }
__device__ __forceinline__ uint64_t extract_bits64(const uint8_t* data, uint64_t bitpos, int bw) {
  if (bw == 0) return 0;
  const uint8_t* a = data + (bitpos >> 3);
  const uintptr_t base = reinterpret_cast<uintptr_t>(a) & ~(uintptr_t)7;
  const uint64_t w0 = *reinterpret_cast<const uint64_t*>(base), w1 = *reinterpret_cast<const uint64_t*>(base + 8);
  const int sh = (int)((reinterpret_cast<uintptr_t>(a) & 7) * 8 + (bitpos & 7));
  uint64_t v = w0 >> sh;
  if (sh) v |= w1 << (64 - sh);
  return bw >= 64 ? v : (v & ((1ull << bw) - 1));
}

__device__ void decode_delta_binary(const uint8_t* p, const uint8_t* end, int nvals, ValueWriter w, int32_t* errors) {
  __shared__ const uint8_t* s_ptr[PQ_NT];
  __shared__ int64_t s_md[PQ_NT];
  __shared__ uint64_t s_tot[PQ_NT];
  __shared__ uint8_t s_bw[PQ_NT];
  __shared__ uint64_t s_carry;
  __shared__ const uint8_t* s_p;
  __shared__ int s_n, s_vpm, s_mpb, s_j, s_bad;
  __shared__ int64_t s_cur_md;
  __shared__ const uint8_t* s_bws;
  const int t = threadIdx.x;
  if (t == 0) {
    const uint64_t block = dl_uleb(p, end), mpb = dl_uleb(p, end), total = dl_uleb(p, end);
    const int64_t first = dl_zigzag(dl_uleb(p, end));
    s_bad = (mpb == 0 || block == 0 || block % 128 != 0 || block % mpb != 0 || (block / mpb) % 32 != 0 || (nvals > 0 && total < (uint64_t)nvals)) ? 1 : 0;
    s_vpm = s_bad ? 32 : (int)(block / mpb); s_mpb = (int)mpb; s_j = (int)mpb;   // j == mpb: a block header comes next
    s_carry = (uint64_t)first; s_p = p; s_cur_md = 0; s_bws = p;
    if (!s_bad && nvals > 0) { const uint64_t v = (uint64_t)first; w.write_fixed(0, reinterpret_cast<const uint8_t*>(&v)); }
  }
  __syncthreads();
  if (s_bad) { if (t == 0) atomicExch(errors, 5); return; }
  const int vpm = s_vpm;
  int done = 1;   // values written so far
  while (done < nvals) {
    if (t == 0) {
      const uint8_t* q = s_p;
      int m = 0, sched = done;
      while (m < PQ_NT && sched < nvals) {
        if (s_j == s_mpb) {   // block header: min delta + one bit width per miniblock
          if (q >= end) break;
          s_cur_md = dl_zigzag(dl_uleb(q, end)); s_bws = q; q += s_mpb; s_j = 0;
          if (q > end) { s_bad = 1; break; }
        }
        const int bw = s_bws[s_j];
        if (bw > 64 || q + (size_t)vpm * bw / 8 > end) { s_bad = 1; break; }   // (width-0 miniblocks occupy no bytes)
        s_ptr[m] = q; s_bw[m] = (uint8_t)bw; s_md[m] = s_cur_md;
        q += (size_t)vpm * bw / 8;
        s_j++; m++; sched += vpm;
      }
      if (m == 0) s_bad = 1;   // ran out of bytes before the announced value count
      s_n = m; s_p = q;
    }
    __syncthreads();
    if (s_bad) { if (t == 0) atomicExch(errors, 5); return; }
    const int n = s_n;
    uint64_t tot = 0;
    if (t < n) { const uint64_t md = (uint64_t)s_md[t]; const int bw = s_bw[t]; for (int i = 0; i < vpm; i++) tot += md + extract_bits64(s_ptr[t], (uint64_t)i * bw, bw); }
    s_tot[t] = t < n ? tot : 0;
    __syncthreads();
    if (t == 0) { uint64_t run = s_carry; for (int u = 0; u < n; u++) { const uint64_t x = s_tot[u]; s_tot[u] = run; run += x; } s_carry = run; }
    __syncthreads();
    if (t < n) {
      uint64_t v = s_tot[t];
      const uint64_t md = (uint64_t)s_md[t]; const int bw = s_bw[t];
      const int k0 = done + t * vpm;
      for (int i = 0; i < vpm && k0 + i < nvals; i++) {
        v += md + extract_bits64(s_ptr[t], (uint64_t)i * bw, bw);
        w.write_fixed(k0 + i, reinterpret_cast<const uint8_t*>(&v));
      }
    }
    __syncthreads();
    done += n * vpm;
  }
}

__global__ void __launch_bounds__(PQ_NT) values_kernel(const PageD* __restrict__ pages, const int32_t* __restrict__ todo, const ChunkD* __restrict__ chunks,
                                                       const ColD* __restrict__ cols, const uint8_t* __restrict__ file, const uint8_t* __restrict__ scratch,
                                                       const int32_t* __restrict__ nonnull, const int64_t* __restrict__ dict_src,
                                                       const int32_t* __restrict__ dict_len, int32_t* __restrict__ errors) {
  const int pi = todo[blockIdx.x];
  const PageD pg = pages[pi];
  const ChunkD ch = chunks[pg.chunk];
  const ColD col = cols[ch.col];
  const uint8_t* d = page_ptr(pg, file, scratch);
  const uint8_t* vals = d;
  const uint8_t* pend = d + pg.uncomp_size;
  if (ch.max_def > 0) { const uint8_t* lv_end; levels_of(pg, d, lv_end, vals); }
  else if (pg.kind == PG_DATA_V2) vals = d + pg.lvl_bytes;
  const int nvals = ch.max_def > 0 ? nonnull[pi] : pg.num_values;
  ValueWriter w; w.col = col; w.base = pg.value_base; w.dict = nullptr; w.dict_count = 0;
  w.dict_src = dict_src + ch.dict_str_off; w.dict_len = dict_len + ch.dict_str_off;
  const int src_width = ch.phys == PT_INT32 || ch.phys == PT_FLOAT ? 4 : (ch.phys == PT_FLBA ? ch.type_length : 8);
  if (pg.encoding == ENC_PLAIN_DICT || pg.encoding == ENC_RLE_DICT) {
    if (ch.dict_page < 0) { if (threadIdx.x == 0) atomicExch(errors, 3); return; }
    w.dict = page_ptr(pages[ch.dict_page], file, scratch);
    w.dict_count = ch.dict_count;
    const int bw = vals[0];
    DictSink sink{w, src_width, errors};
    if (bw == 0) { for (int k = threadIdx.x; k < nvals; k += PQ_NT) sink.put(k, 0); }
    else decode_hybrid(vals + 1, pend, bw, nvals, sink);
  } else if (pg.encoding == ENC_PLAIN) {
    if (ch.phys == PT_BOOLEAN) {
      for (int k = threadIdx.x; k < nvals; k += PQ_NT) reinterpret_cast<int8_t*>(col.dense)[w.base + k] = (vals[k >> 3] >> (k & 7)) & 1;
    } else if (ch.phys == PT_BYTE_ARRAY) {
      // length-prefixed values: a sequential walk (dictionary pages normally carry the strings)
      if (threadIdx.x == 0) {
        const uint8_t* q = vals;
        int k = 0;
        for (; k < nvals && q + 4 <= pend; k++) {
          uint32_t n; memcpy(&n, q, 4);
          if (n > (uint32_t)(pend - (q + 4))) break;   // length runs past the page
          col.str_src[w.base + k] = (int64_t)reinterpret_cast<uintptr_t>(q + 4);
          col.str_len[w.base + k] = (int32_t)n;
          q += 4 + n;
        }
        if (k < nvals) {   // truncated / corrupt page: flag it and leave the remaining rows as empty strings
          atomicExch(errors, 5);
          for (; k < nvals; k++) { col.str_src[w.base + k] = (int64_t)reinterpret_cast<uintptr_t>(vals); col.str_len[w.base + k] = 0; }
        }
      }
    } else if (vals > pend || (size_t)nvals * (size_t)src_width > (size_t)(pend - vals)) {
      if (threadIdx.x == 0) atomicExch(errors, 5);   // fewer value bytes than the header promises
    } else {
      for (int k = threadIdx.x; k < nvals; k += PQ_NT) w.write_fixed(k, vals + (size_t)k * src_width);
    }
  } else if (pg.encoding == ENC_DELTA_BINARY && (ch.phys == PT_INT32 || ch.phys == PT_INT64)) {
    decode_delta_binary(vals, pend, nvals, w, errors);
  } else if (pg.encoding == ENC_RLE && ch.phys == PT_BOOLEAN) {
    // RLE booleans (data page v2 writers): 4-byte length, then the hybrid stream at bit width 1
    struct BoolSink {
      int8_t* out;
      __device__ __forceinline__ void put(int k, uint32_t v) { out[k] = (int8_t)(v & 1); }
      __device__ __forceinline__ void put4(int k, uint32_t a, uint32_t b, uint32_t c, uint32_t d) { put(k, a); put(k + 32, b); put(k + 64, c); put(k + 96, d); }
    };
    BoolSink sink{reinterpret_cast<int8_t*>(col.dense) + w.base};
    decode_hybrid(vals + 4, pend, 1, nvals, sink);
  } else {
    if (threadIdx.x == 0) atomicExch(errors, 4);
  }
}

// string dictionaries: walk the length-prefixed entries of each dictionary page once
__global__ void dict_strings_kernel(const PageD* __restrict__ pages, const ChunkD* __restrict__ chunks, int nchunks, const uint8_t* __restrict__ file,
                                    const uint8_t* __restrict__ scratch, int64_t* __restrict__ dict_src, int32_t* __restrict__ dict_len,
                                    int32_t* __restrict__ errors) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= nchunks) return;
  const ChunkD ch = chunks[c];
  if (ch.phys != PT_BYTE_ARRAY || ch.dict_page < 0) return;
  const PageD pg = pages[ch.dict_page];
  const uint8_t* q = page_ptr(pg, file, scratch);
  const uint8_t* end = q + pg.uncomp_size;
  int k = 0;
  for (; k < ch.dict_count && q + 4 <= end; k++) {
    uint32_t n; memcpy(&n, q, 4);
    if (n > (uint32_t)(end - (q + 4))) break;   // entry runs past the dictionary page
    dict_src[ch.dict_str_off + k] = (int64_t)reinterpret_cast<uintptr_t>(q + 4);
    dict_len[ch.dict_str_off + k] = (int32_t)n;
    q += 4 + n;
  }
  if (k < ch.dict_count) {   // corrupt dictionary: the missing entries become empty strings, the decode reports an error
    atomicExch(errors, 5);
    for (; k < ch.dict_count; k++) { dict_src[ch.dict_str_off + k] = (int64_t)reinterpret_cast<uintptr_t>(end); dict_len[ch.dict_str_off + k] = 0; }
  }
}

__global__ void string_chars_kernel(const int64_t* __restrict__ src, const int32_t* __restrict__ offsets, int64_t n, uint8_t* __restrict__ chars) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < n; i += nwarps) {
    const int32_t o = offsets[i], len = offsets[i + 1] - o;
    const uint8_t* s = reinterpret_cast<const uint8_t*>((uintptr_t)src[i]);
    for (int k = lane; k < len; k += 32) chars[o + k] = s[k];
  }
}

// NULL expansion: out[row] = lvl[row] ? dense[idx[row]] : 0, validity bits by ballot
__global__ void expand_nulls_kernel(const uint8_t* __restrict__ lvl, const int64_t* __restrict__ idx, int64_t n, int width,
                                    const uint8_t* __restrict__ dense, uint8_t* __restrict__ out, uint32_t* __restrict__ valid) {
  const int64_t nround = (n + 31) & ~(int64_t)31;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
    const bool v = i < n && lvl[i] != 0;
    if (i < n) {
      const int64_t s = idx[i];
      for (int b = 0; b < width; b++) out[i * width + b] = v ? dense[s * width + b] : 0;
    }
    const uint32_t bits = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && i < n) valid[i >> 5] = bits;
  }
}
__global__ void expand_null_lengths_kernel(const uint8_t* __restrict__ lvl, const int64_t* __restrict__ idx, int64_t n, const int32_t* __restrict__ dense_len,
                                           const int64_t* __restrict__ dense_src, int32_t* __restrict__ out_len, int64_t* __restrict__ out_src,
                                           uint32_t* __restrict__ valid) {
  const int64_t nround = (n + 31) & ~(int64_t)31;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nround; i += (int64_t)gridDim.x * blockDim.x) {
    const bool v = i < n && lvl[i] != 0;
    if (i < n) { out_len[i] = v ? dense_len[idx[i]] : 0; out_src[i] = v ? dense_src[idx[i]] : 0; }
    const uint32_t bits = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && i < n) valid[i >> 5] = bits;
  }
}

// ------------------------------------------------------------------------------------------------
struct OutColPlan {
  int schema_idx;
  int out_dtype, out_scale, out_width, conv;
  int phys, type_length, max_def;
};

static OutColPlan plan_column(const SchemaElem& e, int schema_idx) {
  OutColPlan p; memset(&p, 0, sizeof(p));
  p.schema_idx = schema_idx; p.phys = e.type; p.type_length = e.type_length;
  if (e.repetition == 2) throw Error(B2_ERR_UNSUPPORTED, "parquet: repeated (nested) column '" + e.name + "'");
  p.max_def = e.repetition == 1 ? 1 : 0;
  const bool dec = e.converted == 5 || e.lt_decimal;
  switch (e.type) {
    case PT_BOOLEAN: p.out_dtype = B2_BOOL8; p.out_width = 1; p.conv = 4; break;
    case PT_INT32:
      p.out_width = 4; p.conv = 0;
      if (dec) { p.out_dtype = B2_DECIMAL32; p.out_scale = e.scale; }
      else if (e.converted == 6 || e.lt_date) p.out_dtype = B2_DATE32;
      else if (e.converted == 15 || e.lt_int_bits == 8) { p.out_dtype = B2_INT8; p.out_width = 1; p.conv = 3; }
      else if (e.converted == 16 || e.lt_int_bits == 16) { p.out_dtype = B2_INT16; p.out_width = 2; p.conv = 3; }
      else p.out_dtype = B2_INT32;
      break;
    case PT_INT64:
      p.out_width = 8; p.conv = 0;
      if (dec) { p.out_dtype = B2_DECIMAL64; p.out_scale = e.scale; }
      else if (e.converted == 10 || (e.lt_timestamp && e.lt_ts_unit == 2)) p.out_dtype = B2_TIMESTAMP_US;
      else if (e.converted == 9 || (e.lt_timestamp && e.lt_ts_unit == 1)) { p.out_dtype = B2_TIMESTAMP_US; p.conv = 1; }
      else if (e.lt_timestamp) throw Error(B2_ERR_UNSUPPORTED, "parquet: nanosecond timestamps");
      else p.out_dtype = B2_INT64;
      break;
    case PT_FLOAT: p.out_dtype = B2_FLOAT32; p.out_width = 4; break;
    case PT_DOUBLE: p.out_dtype = B2_FLOAT64; p.out_width = 8; break;
    case PT_BYTE_ARRAY: p.out_dtype = B2_STRING; p.out_width = 0; p.conv = 5; break;
    case PT_FLBA:
      if (!dec) throw Error(B2_ERR_UNSUPPORTED, "parquet: FIXED_LEN_BYTE_ARRAY that is not a decimal");
      if (e.type_length > 16) throw Error(B2_ERR_UNSUPPORTED, "parquet: decimal wider than 16 bytes");
      p.conv = 2; p.out_scale = e.scale;
      if (e.precision <= 9) { p.out_dtype = B2_DECIMAL32; p.out_width = 4; }
      else if (e.precision <= 18) { p.out_dtype = B2_DECIMAL64; p.out_width = 8; }
      else { p.out_dtype = B2_DECIMAL128; p.out_width = 16; }
      break;
    default: throw Error(B2_ERR_UNSUPPORTED, "parquet: physical type " + std::to_string(e.type) + " (INT96?) is not supported");
  }
  return p;
}

static std::string lower(std::string s) { for (auto& c : s) c = (char)tolower(c); return s; }

static thread_local int64_t t_pq_stats[5];

Table* parquet_decode(const uint8_t* host, const uint8_t* dev_in, int64_t len, const char* const* names, int ncols, int rg_begin = 0, int rg_end = 0x7fffffff) {
  const auto t_host0 = std::chrono::steady_clock::now();
  FileMeta fm = parse_footer(host, len);
  if (fm.schema.empty()) throw Error(B2_ERR_INVALID, "parquet: empty schema");
  // leaves in depth-first order = column-chunk order; only top-level (flat) leaves can be selected
  std::vector<int> leaf_schema;     // schema index of every leaf
  std::vector<bool> leaf_flat;
  {
    std::vector<int> remaining;     // children still to visit at each depth
    remaining.push_back(fm.schema[0].num_children);
    for (size_t i = 1; i < fm.schema.size(); i++) {
      while (!remaining.empty() && remaining.back() == 0) remaining.pop_back();
      if (remaining.empty()) break;
      remaining.back()--;
      const int depth = (int)remaining.size();
      if (fm.schema[i].num_children > 0) remaining.push_back(fm.schema[i].num_children);
      else { leaf_schema.push_back((int)i); leaf_flat.push_back(depth == 1); }
    }
  }
  std::vector<OutColPlan> plans;
  std::vector<int> leaf_of_col;
  for (int c = 0; c < ncols; c++) {
    int found = -1;
    for (size_t l = 0; l < leaf_schema.size(); l++)
      if (leaf_flat[l] && fm.schema[leaf_schema[l]].name == names[c]) found = (int)l;
    if (found < 0)  // case-insensitive fallback (GpuParquetScan.scala:965-1070 isCaseSensitive=false)
      for (size_t l = 0; l < leaf_schema.size(); l++)
        if (lower(fm.schema[leaf_schema[l]].name) == lower(names[c])) found = (int)l;
    if (found < 0) throw Error(B2_ERR_INVALID, std::string("parquet: column '") + names[c] + "' not in file");
    if (!leaf_flat[found]) throw Error(B2_ERR_UNSUPPORTED, std::string("parquet: column '") + names[c] + "' is nested");
    plans.push_back(plan_column(fm.schema[leaf_schema[found]], leaf_schema[found]));
    leaf_of_col.push_back(found);
  }
  // split clipping (GpuParquetScan.scala filterBlocks: a task reads the row groups whose midpoint falls in its split)
  rg_begin = std::max(0, rg_begin); rg_end = std::min<int>(rg_end, (int)fm.row_groups.size());
  if (rg_begin > 0 || rg_end < (int)fm.row_groups.size()) {
    std::vector<RowGroupMeta> sel;
    for (int g = rg_begin; g < rg_end; g++) sel.push_back(fm.row_groups[g]);
    fm.row_groups.swap(sel);
  }
  int64_t total_rows = 0;
  for (auto& rg : fm.row_groups) total_rows += rg.num_rows;
  if (total_rows > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "parquet: more than 2^31-1 rows in one read; use chunked reads");

  // walk page headers.  Column chunks are independent page chains, so they are walked by a few host threads;
  // offsets that depend on the chunks in front (scratch position, first row, dictionary-string base) are local
  // to the chunk here and rebased in file order below.
  struct ChunkWalk {
    ChunkD cd; std::vector<PageD> pages; int64_t rows = 0, scratch = 0, dict_strs = 0;
    int err = 0; std::string msg;
  };
  struct ChunkRef { const ChunkMeta* cm; int c; };
  std::vector<ChunkRef> refs;
  for (auto& rg : fm.row_groups)
    for (int c = 0; c < ncols; c++) {
      if (leaf_of_col[c] >= (int)rg.chunks.size()) throw Error(B2_ERR_INVALID, "parquet: row group lacks a column chunk");
      refs.push_back({&rg.chunks[leaf_of_col[c]], c});
    }
  std::vector<ChunkWalk> walks(refs.size());
  auto walk_chunk = [&](const ChunkRef& ref, ChunkWalk& w) {
    const ChunkMeta& cm = *ref.cm;
    const int c = ref.c;
    if (cm.codec != CODEC_NONE && cm.codec != CODEC_SNAPPY) throw Error(B2_ERR_UNSUPPORTED, "parquet: codec " + std::to_string(cm.codec) + " (only UNCOMPRESSED / SNAPPY)");
    ChunkD& cd = w.cd; memset(&cd, 0, sizeof(cd));
    cd.col = c; cd.phys = cm.type; cd.type_length = plans[c].type_length; cd.max_def = plans[c].max_def; cd.dict_page = -1;
    int64_t pos = cm.data_page_offset;
    if (cm.dict_page_offset > 0 && cm.dict_page_offset < pos) pos = cm.dict_page_offset;
    const int64_t chunk_end = pos + cm.total_compressed;
    if (cm.num_values == 0) return;  // empty row group
    if (pos < 4 || chunk_end > len - 8) throw Error(B2_ERR_INVALID, "parquet: column chunk outside the buffer");
    int64_t values_seen = 0;
    while (pos < chunk_end && values_seen < cm.num_values) {
      TReader r(host + pos, host + chunk_end);
      int id, t, last = 0;
      int ptype = -1, usize = 0, csize = 0, nvals = 0, enc = 0, v2_def_len = 0, v2_rep_len = 0, v2_compressed = 1;
      while (r.field(id, t, last)) {
        if (id == 1) ptype = (int)r.zigzag();
        else if (id == 2) usize = (int)r.zigzag();
        else if (id == 3) csize = (int)r.zigzag();
        else if ((id == 5 || id == 7 || id == 8) && t == 12) {
          int id2, t2, last2 = 0;
          while (r.field(id2, t2, last2)) {
            if (id2 == 1) nvals = (int)r.zigzag();
            else if (id == 5 && id2 == 2) enc = (int)r.zigzag();
            else if (id == 7 && id2 == 2) enc = (int)r.zigzag();
            else if (id == 8 && id2 == 4) enc = (int)r.zigzag();
            else if (id == 8 && id2 == 5) v2_def_len = (int)r.zigzag();
            else if (id == 8 && id2 == 6) v2_rep_len = (int)r.zigzag();
            else if (id == 8 && id2 == 7) v2_compressed = (t2 == 1);
            else r.skip(t2);
          }
        } else r.skip(t);
      }
      const int64_t payload = r.p - host;
      // untrusted input: sizes and counts are zigzag varints and may decode negative (a negative csize would move
      // `pos` backwards: endless loop / reads before the chunk)
      if (csize < 0 || usize < 0 || nvals < 0 || v2_def_len < 0 || v2_rep_len < 0) throw Error(B2_ERR_INVALID, "parquet: negative size in a page header");
      if ((int64_t)v2_def_len + v2_rep_len > usize) throw Error(B2_ERR_INVALID, "parquet: level bytes exceed the page");
      if (payload + csize > chunk_end) throw Error(B2_ERR_INVALID, "parquet: page runs past its chunk");
      if (csize == 0 && (ptype == PG_DATA || ptype == PG_DATA_V2) && nvals > 0 && usize > 0) throw Error(B2_ERR_INVALID, "parquet: empty data page with values");
      if (ptype == PG_INDEX) { pos = payload + csize; continue; }
      PageD pg; memset(&pg, 0, sizeof(pg));
      pg.src_off = payload; pg.comp_size = csize; pg.uncomp_size = usize; pg.num_values = nvals; pg.encoding = enc; pg.kind = ptype;
      pg.lvl_bytes = ptype == PG_DATA_V2 ? v2_def_len + v2_rep_len : 0;
      pg.compressed = cm.codec == CODEC_SNAPPY && (ptype != PG_DATA_V2 || v2_compressed);
      if (ptype == PG_DATA_V2 && v2_rep_len) throw Error(B2_ERR_UNSUPPORTED, "parquet: repetition levels");
      if (pg.compressed && pg.lvl_bytes == 0 && csize > usize && usize > 0) {
        // Incompressible pages (bit-packed dictionary indexes, mostly) are stored by snappy as ONE literal: the
        // page bytes sit verbatim in the file behind the length preamble and the literal header.  Read them in
        // place instead of copying them through the decompressor.
        const uint8_t* p = host + payload;
        const uint8_t* pend = p + csize;
        uint64_t ulen = 0; int shift = 0;
        while (p < pend && shift < 35) { const uint8_t b = *p++; ulen |= (uint64_t)(b & 0x7f) << shift; if (!(b & 0x80)) break; shift += 7; }
        if (ulen == (uint64_t)usize && p < pend && (*p & 3) == 0) {
          uint64_t len = *p >> 2; int nb = 0;
          if (len >= 60) { nb = (int)len - 59; len = 0; for (int k = 0; k < nb && p + 1 + k < pend; k++) len |= (uint64_t)p[1 + k] << (8 * k); }
          len += 1;
          const uint8_t* data = p + 1 + nb;
          if (len == (uint64_t)usize && data + len == pend) { pg.compressed = 0; pg.src_off = data - host; pg.comp_size = usize; }
        }
      }
      if (pg.compressed) { pg.dst_off = w.scratch; w.scratch += ((int64_t)usize + 15) & ~15LL; }
      else pg.dst_off = -1;
      if (ptype == PG_DICT) {
        if (enc != ENC_PLAIN && enc != ENC_PLAIN_DICT) throw Error(B2_ERR_UNSUPPORTED, "parquet: dictionary page encoding " + std::to_string(enc));
        cd.dict_page = (int)w.pages.size(); cd.dict_count = nvals;
        if (cm.type == PT_BYTE_ARRAY) w.dict_strs += nvals;
      } else if (ptype == PG_DATA || ptype == PG_DATA_V2) {
        if (enc != ENC_PLAIN && enc != ENC_PLAIN_DICT && enc != ENC_RLE_DICT && !(enc == ENC_RLE && cm.type == PT_BOOLEAN) &&
            !(enc == ENC_DELTA_BINARY && (cm.type == PT_INT32 || cm.type == PT_INT64)))
          throw Error(B2_ERR_UNSUPPORTED, "parquet: value encoding " + std::to_string(enc) + " (DELTA_BYTE_ARRAY / DELTA_LENGTH_BYTE_ARRAY / BYTE_STREAM_SPLIT are not supported)");
        pg.row_start = w.rows;
        w.rows += nvals; values_seen += nvals;
      } else throw Error(B2_ERR_INVALID, "parquet: unknown page type");
      w.pages.push_back(pg);
      pos = payload + csize;
    }
  };
  {
    int64_t walk_bytes = 0;
    for (auto& ref : refs) walk_bytes += ref.cm->total_compressed;
    const int nthreads = (refs.size() >= 4 && walk_bytes >= (8 << 20)) ? (int)std::min<size_t>({(size_t)(getenv("B2_PQ_WALK_THREADS") ? atoi(getenv("B2_PQ_WALK_THREADS")) : 8), refs.size(), std::max(1u, std::thread::hardware_concurrency())}) : 1;
    std::atomic<size_t> next{0};
    auto worker = [&]() {
      for (size_t i = next.fetch_add(1); i < refs.size(); i = next.fetch_add(1)) {
        try { walk_chunk(refs[i], walks[i]); }
        catch (const Error& e) { walks[i].err = e.code; walks[i].msg = e.what(); }
        catch (const std::exception& e) { walks[i].err = B2_ERR_INVALID; walks[i].msg = e.what(); }
      }
    };
    std::vector<std::thread> pool;
    for (int t = 1; t < nthreads; t++) pool.emplace_back(worker);
    worker();
    for (auto& th : pool) th.join();
  }
  std::vector<PageD> pages;
  std::vector<ChunkD> chunks;
  std::vector<int64_t> col_rows(ncols, 0);
  int64_t scratch_bytes = 0, dict_str_total = 0;
  for (size_t i = 0; i < walks.size(); i++) {
    ChunkWalk& w = walks[i];
    if (w.err) throw Error(w.err, w.msg);   // first failing chunk in file order, as a serial walk would report
    const int c = refs[i].c;
    const int chunk_idx = (int)chunks.size();
    w.cd.dict_str_off = dict_str_total;
    if (w.cd.dict_page >= 0) w.cd.dict_page += (int)pages.size();
    for (PageD& pg : w.pages) {
      pg.chunk = chunk_idx;
      if (pg.compressed) pg.dst_off += scratch_bytes;
      if (pg.kind == PG_DATA || pg.kind == PG_DATA_V2) pg.row_start += col_rows[c];
      pages.push_back(pg);
    }
    scratch_bytes += w.scratch; dict_str_total += w.dict_strs; col_rows[c] += w.rows;
    chunks.push_back(w.cd);
  }
  for (int c = 0; c < ncols; c++)
    if (col_rows[c] != total_rows) throw Error(B2_ERR_INVALID, "parquet: page row counts disagree with the footer");
  if (getenv("B2_PQ_DEBUG"))
    fprintf(stderr, "[b2 parquet] footer + page-header walk: %.3f ms for %zu pages\n",
            std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_host0).count(), pages.size());

  {
    int64_t comp = 0, prod = 0, unc = 0;
    for (auto& pg : pages) {
      unc += pg.uncomp_size;
      if (pg.compressed) { comp += pg.comp_size - pg.lvl_bytes; prod += pg.uncomp_size - pg.lvl_bytes; }
    }
    t_pq_stats[0] = comp; t_pq_stats[1] = prod; t_pq_stats[2] = unc; t_pq_stats[3] = 0; t_pq_stats[4] = (int64_t)pages.size();
  }
  std::vector<int32_t> todo_snappy, todo_big, todo_levels, todo_values;
  std::vector<int64_t> big_soff;
  int64_t big_S = 0;
  for (size_t i = 0; i < pages.size(); i++) {
    if (pages[i].compressed) {
      if ((uint32_t)pages[i].uncomp_size >= SB_MIN_BYTES && pages[i].lvl_bytes == 0) {
        // large pages decode into one contiguous region at the end of the scratch buffer so that the
        // source map and the output share one index space
        todo_big.push_back((int32_t)i); big_soff.push_back(big_S);
        pages[i].dst_off = scratch_bytes + big_S;   // scratch_bytes = start of the large-page region
        big_S += ((int64_t)pages[i].uncomp_size + 15) & ~15LL;
      } else todo_snappy.push_back((int32_t)i);
    }
    if (pages[i].kind != PG_DICT) { todo_values.push_back((int32_t)i); if (chunks[pages[i].chunk].max_def > 0) todo_levels.push_back((int32_t)i); }
  }
  const int64_t big_region = scratch_bytes;
  scratch_bytes += big_S;
  cudaStream_t s = stream();
  // device copy of the file bytes (H2D inside the call unless the caller already has them resident)
  DevBuf file_buf;
  const uint8_t* d_file = dev_in;
  if (!d_file) {
    file_buf = DevBuf((size_t)len + 64);
    CUDA_CHECK(cudaMemcpyAsync(file_buf.p, host, (size_t)len, cudaMemcpyHostToDevice, s));
    d_file = file_buf.as<uint8_t>();
  }
  DevBuf scratch((size_t)scratch_bytes + 64);
  DevBuf d_pages(std::max<size_t>(1, pages.size()) * sizeof(PageD)), d_chunks(std::max<size_t>(1, chunks.size()) * sizeof(ChunkD));
  DevBuf d_err(4), d_nonnull(std::max<size_t>(1, pages.size()) * 4);
  CUDA_CHECK(cudaMemsetAsync(d_err.p, 0, 4, s));
  CUDA_CHECK(cudaMemsetAsync(d_nonnull.p, 0, d_nonnull.bytes, s));
  if (!chunks.empty()) h2d(d_chunks.p, chunks.data(), chunks.size());

  // outputs
  std::vector<ColD> cold(ncols);
  std::vector<DevBuf> dense(ncols), str_src(ncols), str_len(ncols), lvl(ncols);
  for (int c = 0; c < ncols; c++) {
    ColD& cd = cold[c]; memset(&cd, 0, sizeof(cd));
    cd.out_dtype = plans[c].out_dtype; cd.out_width = plans[c].out_width; cd.phys = plans[c].phys; cd.type_length = plans[c].type_length; cd.conv = plans[c].conv;
    if (cd.conv == 5) {
      str_src[c] = DevBuf((size_t)std::max<int64_t>(total_rows, 1) * 8); str_len[c] = DevBuf((size_t)(total_rows + 1) * 4);
      cd.str_src = str_src[c].as<int64_t>(); cd.str_len = str_len[c].as<int32_t>();
    } else {
      dense[c] = DevBuf((size_t)std::max<int64_t>(total_rows, 1) * cd.out_width);
      cd.dense = dense[c].p;
    }
    if (plans[c].max_def > 0) { lvl[c] = DevBuf((size_t)std::max<int64_t>(total_rows, 1)); cd.lvl = lvl[c].as<uint8_t>(); }
  }
  DevBuf d_cols((size_t)ncols * sizeof(ColD));
  h2d(d_cols.p, cold.data(), cold.size());

  // value_base is only known after the level pass when a column has NULLs; start with rows
  for (auto& pg : pages) pg.value_base = pg.row_start;
  if (!pages.empty()) h2d(d_pages.p, pages.data(), pages.size());
  auto upload = [&](const std::vector<int32_t>& v, DevBuf& b) { b = DevBuf(std::max<size_t>(1, v.size()) * 4); if (!v.empty()) h2d(b.p, v.data(), v.size()); };
  DevBuf d_todo_s, d_todo_l, d_todo_v;
  // longest pages first: a page is one serial LZ77 chain, so the kernel ends when the slowest page does
  std::stable_sort(todo_snappy.begin(), todo_snappy.end(), [&](int32_t a, int32_t b) { return pages[a].uncomp_size > pages[b].uncomp_size; });
  upload(todo_snappy, d_todo_s); upload(todo_levels, d_todo_l); upload(todo_values, d_todo_v);
  DevBuf d_todo_b, d_big_soff, d_big_S, d_big_fail;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaStream_t ws = s;   // stream of the small-page kernel
  if (!todo_big.empty()) {
    // Large pages: CTA-wide parallel decode; pages it declines are redone by the one-warp kernel.  Its 1024-thread
    // CTAs need an SM to themselves, so they must be dispatched BEFORE the thousands of one-warp CTAs of the
    // small-page kernel: the wide kernel goes first on the main stream and the small-page kernel runs on the aux
    // stream, released by an event recorded just in front of the wide kernel, so the two paths overlap.  (With the
    // wide kernel on the aux stream the order flipped whenever the main stream had been blocked on an upload event
    // and the two paths ran back to back on the host-buffer path.)
    upload(todo_big, d_todo_b);
    d_big_soff = DevBuf(big_soff.size() * 8);
    h2d(d_big_soff.p, big_soff.data(), big_soff.size());
    d_big_S = DevBuf((size_t)big_S * 4);
    d_big_fail = DevBuf(todo_big.size() * 4);
    CUDA_CHECK(cudaMemsetAsync(d_big_fail.p, 0, d_big_fail.bytes, s));
    if (!todo_snappy.empty()) {
      ws = aux_stream();
      CUDA_CHECK(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
      CUDA_CHECK(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
      CUDA_CHECK(cudaEventRecord(ev_fork, s));
      CUDA_CHECK(cudaStreamWaitEvent(ws, ev_fork, 0));
    }
    launch("snappy_big_kernel", snappy_big_kernel, (int)todo_big.size(), SB_WARPS * 32, 0, s, d_pages.as<PageD>(), d_todo_b.as<int32_t>(),
           d_big_soff.as<int64_t>(), d_file, scratch.as<uint8_t>(), d_big_S.as<uint32_t>(), d_big_fail.as<int32_t>());
  }
  if (!todo_snappy.empty()) {
    launch("snappy_kernel", snappy_kernel, ((int)todo_snappy.size() + SN_WARPS - 1) / SN_WARPS, SN_WARPS * 32, 0, ws, d_pages.as<PageD>(),
           d_todo_s.as<int32_t>(), (int)todo_snappy.size(), d_file, scratch.as<uint8_t>(), d_err.as<int32_t>(), nullptr);
    if (ev_join) CUDA_CHECK(cudaEventRecord(ev_join, ws));
  }
  if (!todo_big.empty()) {
    {
      KernelTimer kt("snappy_jump_resolve_kernels");
      const uint32_t total = (uint32_t)big_S;
      const int grid = grid_for((int64_t)total, 256 * 4, 8);
      for (int round = 0; round < 20; round++) launch(snappy_jump_kernel, grid, 256, 0, s, d_big_S.as<uint32_t>(), total);
      launch(snappy_resolve_kernel, grid_for((int64_t)total, 256, 8), 256, 0, s, d_big_S.as<uint32_t>(), scratch.as<uint8_t>() + big_region, total);
    }
    launch("snappy_fallback_kernel", snappy_kernel, ((int)todo_big.size() + SN_WARPS - 1) / SN_WARPS, SN_WARPS * 32, 0, s, d_pages.as<PageD>(),
           d_todo_b.as<int32_t>(), (int)todo_big.size(), d_file, scratch.as<uint8_t>(), d_err.as<int32_t>(), d_big_fail.as<int32_t>());
  }
  if (ev_join) {
    CUDA_CHECK(cudaStreamWaitEvent(s, ev_join, 0));
    cudaEventDestroy(ev_fork); cudaEventDestroy(ev_join);
  }
  std::vector<int64_t> col_nonnull(ncols, 0);
  std::vector<bool> has_nulls(ncols, false);
  if (!todo_levels.empty()) {
    launch("levels_kernel", levels_kernel, (int)todo_levels.size(), PQ_NT, 0, s, d_pages.as<PageD>(), d_todo_l.as<int32_t>(), d_chunks.as<ChunkD>(),
           d_cols.as<ColD>(), d_file, scratch.as<uint8_t>(), d_nonnull.as<int32_t>());
    std::vector<int32_t> nn(pages.size());
    d2h(nn.data(), d_nonnull.p, nn.size());
    sync();
    std::vector<int64_t> run(ncols, 0);
    for (size_t i = 0; i < pages.size(); i++) {
      PageD& pg = pages[i];
      if (pg.kind == PG_DICT) continue;
      const int c = chunks[pg.chunk].col;
      if (chunks[pg.chunk].max_def > 0) { pg.value_base = run[c]; run[c] += nn[i]; }
    }
    bool any_nulls = false;
    for (int c = 0; c < ncols; c++) if (plans[c].max_def > 0) { col_nonnull[c] = run[c]; has_nulls[c] = run[c] != total_rows; any_nulls = any_nulls || has_nulls[c]; }
    h2d(d_pages.p, pages.data(), pages.size());
    if (any_nulls) {
      std::vector<uint8_t> hn(ncols, 0);
      for (int c = 0; c < ncols; c++) hn[c] = has_nulls[c] ? 1 : 0;
      DevBuf d_hn((size_t)ncols);
      h2d(d_hn.p, hn.data(), hn.size());
      launch(fill_uniform_levels_kernel, (int)todo_levels.size(), PQ_NT, 0, s, d_pages.as<PageD>(), d_todo_l.as<int32_t>(), d_chunks.as<ChunkD>(),
             d_cols.as<ColD>(), d_nonnull.as<int32_t>(), d_hn.as<uint8_t>());
    }
  }
  DevBuf d_dict_src((size_t)std::max<int64_t>(dict_str_total, 1) * 8), d_dict_len((size_t)std::max<int64_t>(dict_str_total, 1) * 4);
  if (dict_str_total)
    launch(dict_strings_kernel, ((int)chunks.size() + 63) / 64, 64, 0, s, d_pages.as<PageD>(), d_chunks.as<ChunkD>(), (int)chunks.size(), d_file,
           scratch.as<uint8_t>(), d_dict_src.as<int64_t>(), d_dict_len.as<int32_t>(), d_err.as<int32_t>());
  if (!todo_values.empty())
    launch("values_kernel", values_kernel, (int)todo_values.size(), PQ_NT, 0, s, d_pages.as<PageD>(), d_todo_v.as<int32_t>(), d_chunks.as<ChunkD>(),
           d_cols.as<ColD>(), d_file, scratch.as<uint8_t>(), d_nonnull.as<int32_t>(), d_dict_src.as<int64_t>(), d_dict_len.as<int32_t>(),
           d_err.as<int32_t>());
  // assemble output columns
  ColsGuard outs;
  for (int c = 0; c < ncols; c++) {
    std::unique_ptr<Column> oc(new Column());
    oc->dtype = plans[c].out_dtype; oc->scale = plans[c].out_scale; oc->size = total_rows;
    DevBuf idx;
    if (has_nulls[c]) {
      idx = DevBuf((size_t)(total_rows + 1) * 8);
      exclusive_scan<uint8_t, int64_t>(lvl[c].as<uint8_t>(), idx.as<int64_t>(), total_rows, false);
      oc->valid = DevBuf(validity_bytes(total_rows)); oc->null_count = total_rows - col_nonnull[c];
    }
    if (plans[c].conv == 5) {
      int32_t* lens = str_len[c].as<int32_t>();
      int64_t* srcs = str_src[c].as<int64_t>();
      DevBuf xl, xs;
      if (has_nulls[c]) {
        xl = DevBuf((size_t)(total_rows + 1) * 4); xs = DevBuf((size_t)std::max<int64_t>(total_rows, 1) * 8);
        if (total_rows)
          launch(expand_null_lengths_kernel, grid_for(total_rows, 256), 256, 0, s, lvl[c].as<uint8_t>(), idx.as<int64_t>(), total_rows, lens, srcs,
                 xl.as<int32_t>(), xs.as<int64_t>(), oc->valid.as<uint32_t>());
        lens = xl.as<int32_t>(); srcs = xs.as<int64_t>();
      }
      oc->offsets = DevBuf((size_t)(total_rows + 1) * 4);
      DevBuf sums = exclusive_scan<int32_t, int32_t>(lens, oc->offsets.as<int32_t>(), total_rows, true);
      int64_t chars = 0;
      d2h(&chars, sums.as<int64_t>() + std::max<int64_t>(1, (total_rows + SCAN_TILE - 1) / SCAN_TILE), 1);
      sync();
      if (chars > 0x7fffffffLL) throw Error(B2_ERR_SIZE_OVERFLOW, "parquet: string column exceeds 2^31-1 chars");
      oc->chars_bytes = chars;
      oc->data = DevBuf((size_t)chars);
      if (chars) {
        launch(string_chars_kernel, grid_for(total_rows * 32, 256), 256, 0, s, srcs, oc->offsets.as<int32_t>(), total_rows, oc->data.as<uint8_t>());
        sync();  // srcs / scratch are read by the kernel; keep them alive
      }
    } else if (has_nulls[c]) {
      oc->data = DevBuf((size_t)total_rows * plans[c].out_width);
      launch(expand_nulls_kernel, grid_for(total_rows, 256), 256, 0, s, lvl[c].as<uint8_t>(), idx.as<int64_t>(), total_rows, plans[c].out_width,
             dense[c].as<uint8_t>(), oc->data.as<uint8_t>(), oc->valid.as<uint32_t>());
    } else {
      oc->data = std::move(dense[c]);  // no NULLs: the dense decode IS the column
    }
    t_pq_stats[3] += (int64_t)oc->data.bytes + (int64_t)oc->offsets.bytes + (int64_t)oc->valid.bytes;
    outs.v.push_back(oc.release());
  }
  int32_t err = 0;
  d2h(&err, d_err.p, 1);
  sync();
  if (err == 1) throw Error(B2_ERR_INVALID, "parquet: corrupt snappy stream");
  if (err) throw Error(B2_ERR_INVALID, "parquet: corrupt page data (code " + std::to_string(err) + ")");
  return new_table(outs.release());
}

}  // namespace b2

using namespace b2;
extern "C" {

int b2_parquet_last_stats(int64_t* out5) {
  for (int i = 0; i < 5; i++) out5[i] = t_pq_stats[i];
  return B2_OK;
}

int b2_parquet_decode(const uint8_t* host_buf, int64_t len, const char* const* column_names, int32_t ncols, b2_handle* out_table) {
  B2_TRY
  B2_CHECK(host_buf && len > 0 && ncols >= 1, "bad arguments");
  *out_table = to_handle(parquet_decode(host_buf, nullptr, len, column_names, ncols));
  B2_CATCH
}

int b2_parquet_decode_device(const uint8_t* host_buf, const uint8_t* dev_buf, int64_t len, const char* const* column_names, int32_t ncols,
                             b2_handle* out_table) {
  B2_TRY
  B2_CHECK(host_buf && dev_buf && len > 0 && ncols >= 1, "bad arguments");
  *out_table = to_handle(parquet_decode(host_buf, dev_buf, len, column_names, ncols));
  B2_CATCH
}

int b2_parquet_decode_row_groups(const uint8_t* host_buf, const uint8_t* dev_buf, int64_t len, const char* const* column_names, int32_t ncols,
                                 int32_t rg_begin, int32_t rg_end, b2_handle* out_table) {
  B2_TRY
  B2_CHECK(host_buf && len > 0 && ncols >= 1 && rg_begin >= 0 && rg_end >= rg_begin, "bad arguments");
  *out_table = to_handle(parquet_decode(host_buf, dev_buf, len, column_names, ncols, rg_begin, rg_end));
  B2_CATCH
}

// ParquetChunkedReader (GpuParquetScan.scala:3403-3407, 3497-3498: `new ParquetChunkedReader(chunkSizeByteLimit, ...)`, then
// hasNext / readChunk): the buffer is decoded in pieces whose decoded size stays under the limit (spark.rapids.sql.reader.
// chunked + batchSizeBytes, RapidsConf.scala:660-668) and under the 2^31-1 row / char limits of a column.  The unit here is
// the row group: a chunk is a run of consecutive row groups whose selected columns decode to <= limit bytes (always at
// least one row group; a single row group larger than the limit is decoded whole).
struct ParquetChunked {
  const uint8_t* host; int64_t len;
  std::vector<std::string> names;
  std::vector<int64_t> rg_rows, rg_bytes;
  int next_rg = 0;
  int64_t limit = 0;
};
int b2_parquet_chunked_open(const uint8_t* host_buf, int64_t len, const char* const* column_names, int32_t ncols, int64_t chunk_byte_limit,
                            b2_handle* out_reader) {
  B2_TRY
  B2_CHECK(host_buf && len > 0 && ncols >= 1, "bad arguments");
  std::unique_ptr<ParquetChunked> r(new ParquetChunked());
  r->host = host_buf; r->len = len; r->limit = chunk_byte_limit;
  for (int i = 0; i < ncols; i++) r->names.push_back(column_names[i]);
  FileMeta fm = parse_footer(host_buf, len);
  for (auto& rg : fm.row_groups) {
    int64_t bytes = 0;
    for (auto& cm : rg.chunks)
      for (auto& nm : r->names) if (!cm.path.empty() && cm.path[0] == nm) bytes += cm.total_uncompressed > 0 ? cm.total_uncompressed : cm.total_compressed;
    r->rg_rows.push_back(rg.num_rows); r->rg_bytes.push_back(bytes);
  }
  *out_reader = to_handle(r.release());
  B2_CATCH
}
int b2_parquet_chunked_has_next(b2_handle reader, int32_t* out) {
  B2_TRY
  B2_CHECK(reader, "null reader");
  auto* r = reinterpret_cast<ParquetChunked*>((intptr_t)reader);
  *out = r->next_rg < (int)r->rg_rows.size() ? 1 : 0;
  B2_CATCH
}
int b2_parquet_chunked_next(b2_handle reader, b2_handle* out_table) {
  B2_TRY
  B2_CHECK(reader, "null reader");
  auto* r = reinterpret_cast<ParquetChunked*>((intptr_t)reader);
  B2_CHECK(r->next_rg < (int)r->rg_rows.size(), "chunked reader is exhausted");
  int end = r->next_rg;
  int64_t bytes = 0, rows = 0;
  while (end < (int)r->rg_rows.size()) {
    const bool first = end == r->next_rg;
    if (!first && ((r->limit > 0 && bytes + r->rg_bytes[end] > r->limit) || rows + r->rg_rows[end] > 0x7fffffffLL)) break;
    bytes += r->rg_bytes[end]; rows += r->rg_rows[end]; end++;
  }
  std::vector<const char*> cn;
  for (auto& s : r->names) cn.push_back(s.c_str());
  *out_table = to_handle(parquet_decode(r->host, nullptr, r->len, cn.data(), (int)cn.size(), r->next_rg, end));
  r->next_rg = end;
  B2_CATCH
}
int b2_parquet_chunked_close(b2_handle reader) {
  B2_TRY
  delete reinterpret_cast<ParquetChunked*>((intptr_t)reader);
  B2_CATCH
}

int b2_parquet_num_row_groups(const uint8_t* host_buf, int64_t len, int32_t* out_count) {
  B2_TRY
  B2_CHECK(host_buf && len >= 12 && out_count, "bad arguments");
  *out_count = (int32_t)parse_footer(host_buf, len).row_groups.size();
  B2_CATCH
}

}  // extern "C"

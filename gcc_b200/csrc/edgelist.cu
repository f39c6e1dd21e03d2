// edgelist.cu -- corpus builder: ASCII edge lists parsed into the directed 64-bit keys s*n + d.
//
// Replaces (reference file:line):
//   the per-line loop of yuxiao_kdd17_graph_to_dgl   gcc/utils/x2dgl.py:28-47
//     (header n, n skipped vertex lines, header m, m lines "u v w"; self loops dropped, both orientations kept)
//
// The host streams the file in chunks that hold whole lines (each staging chunk is cut at its last '\n' and the
// tail goes to the front of the next one).  Per chunk, in stream order:
//   1. line index: a ballot/popc count of '\n' per 4 KiB tile, an exclusive scan of the tile counts, and a second
//      ballot pass that writes every newline's offset at its rank (64-bit offsets throughout);
//   2. .lscc only: one thread reads the header lines (n, m) that fall into the chunk;
//   3. parse: one thread per line, 256 lines per tile.  A count pass (validation, errors, kept lines per tile),
//      an exclusive scan of the tile counts, and a write pass that parses again and stores each kept line's two
//      keys at its rank.  The key order is the file's line order and no atomics decide a key's slot, so the
//      output is bit-reproducible;
//   4. one thread advances the running state (lines and keys so far).
// Errors never fault: the kind and the line of the first offending line go to the state's first_error word
// (atomicMin on (line << 4) | kind), which the host reads after the last chunk.
#include "common.cuh"

namespace gccb {

constexpr int kNlTile = 4096;       // bytes per block of the newline passes (8 warps x 16 x 32 bytes)
constexpr int kLineTile = 256;      // lines per tile of the parse passes (one thread per line)
constexpr int kMaxParseBlocks = GCCB_NUM_SMS * 8;
constexpr long long kPlainMult = 1LL << 31;   // key multiplier of a plain edge list until n is known

// scratch words of the workspace after the state: [0] newlines of the chunk, [1] lines of the chunk,
// [2] kept lines of the chunk
constexpr int kScratchWords = 4;

__host__ __device__ inline size_t el_align(size_t b) { return (b + 255) & ~(size_t)255; }
struct ElLayout {
  size_t scratch, tile_cnt, line_end, keep_cnt, total;
};
__host__ __device__ inline ElLayout el_layout(int64_t nbytes) {
  ElLayout L;
  const int64_t tiles = (nbytes + kNlTile - 1) / kNlTile;
  const int64_t max_lines = nbytes + 1;
  const int64_t line_tiles = (max_lines + kLineTile - 1) / kLineTile;
  L.scratch = el_align(sizeof(gccb_edgelist_state_t));
  L.tile_cnt = L.scratch + el_align(kScratchWords * sizeof(int64_t));
  L.line_end = L.tile_cnt + el_align((size_t)tiles * sizeof(int64_t));
  L.keep_cnt = L.line_end + el_align((size_t)max_lines * sizeof(int64_t));
  L.total = L.keep_cnt + el_align((size_t)line_tiles * sizeof(int64_t));
  return L;
}

__device__ __forceinline__ void el_error(gccb_edgelist_state_t* st, long long line, int kind) {
  atomicMin((unsigned long long*)&st->first_error, ((unsigned long long)line << 4) | (unsigned)kind);
  atomicOr((int*)&st->error_flags, 1 << kind);
}

__device__ __forceinline__ bool el_sep(uint8_t c) { return c == ' ' || c == '\t' || c == '\r'; }

// Token [a, b) as -?[0-9]+ into *v.  Returns 0, GCCB_EL_ERR_CHAR or GCCB_EL_ERR_OVERFLOW (outside int64).
__device__ __forceinline__ int el_int(const uint8_t* t, int64_t a, int64_t b, long long* v) {
  const bool neg = t[a] == '-';
  if (neg) ++a;
  if (a == b) return GCCB_EL_ERR_CHAR;
  const unsigned long long lim = neg ? (1ULL << 63) : (1ULL << 63) - 1;
  unsigned long long mag = 0;
  int err = 0;
  for (int64_t i = a; i < b; ++i) {
    const unsigned d = (unsigned)t[i] - '0';
    if (d > 9) return GCCB_EL_ERR_CHAR;
    if (mag > (lim - d) / 10) err = GCCB_EL_ERR_OVERFLOW;    // keep scanning: a bad character wins
    else mag = mag * 10 + d;
  }
  if (err) return err;
  *v = neg ? (long long)(0ULL - mag) : (long long)mag;
  return 0;
}

// Splits the line [a, b) into tokens separated by runs of ' ', '\t', '\r'.  Tokens lo .. lo+nv-1 (nv <= 3) are
// read as integers into v0, v1, v2; an overflow of token lo+k is ignored when bit k of ovf_ok is set.  Returns the
// token count; err = the first error of the tokens read, first = the first non-separator character (0 if none).
__device__ __forceinline__ int el_tokens(const uint8_t* t, int64_t a, int64_t b, int lo, int nv, unsigned ovf_ok,
                                         long long& v0, long long& v1, long long& v2, int& err, uint8_t& first) {
  int ntok = 0;
  err = 0;
  int64_t i = a;
  while (i < b && el_sep(t[i])) ++i;
  first = i < b ? t[i] : 0;
  while (i < b) {
    const int64_t s = i;
    while (i < b && !el_sep(t[i])) ++i;
    const int k = ntok - lo;
    if (k >= 0 && k < nv) {
      long long x = 0;
      int e = el_int(t, s, i, &x);
      if (e == GCCB_EL_ERR_OVERFLOW && (ovf_ok >> k & 1)) e = 0;
      if (e && !err) err = e;
      if (k == 0) v0 = x;
      else if (k == 1) v1 = x;
      else v2 = x;
    }
    ++ntok;
    while (i < b && el_sep(t[i])) ++i;
  }
  return ntok;
}

__device__ __forceinline__ void el_line_span(const int64_t* line_end, int64_t i, int64_t* a, int64_t* b) {
  *a = i == 0 ? 0 : line_end[i - 1] + 1;
  *b = line_end[i];
}

// One line of the chunk: 1 when it is an edge line that yields keys (*s, *d), with *edge = 1 for every edge
// line (kept or a self loop).  *err: the error kind of the line (0 = none).
__device__ int el_parse_line(const uint8_t* t, const int64_t* line_end, int64_t i, long long g, int format,
                             long long n, long long m, long long* s, long long* d, int* edge, int* err) {
  *edge = 0;
  *err = 0;
  const bool lscc = format == GCCB_EL_LSCC;
  if (lscc && (n < 0 || m < 0 || g < n + 2 || g >= n + 2 + m)) return 0;    // header, vertex or trailing line
  int64_t a, b;
  el_line_span(line_end, i, &a, &b);
  long long u = 0, w = 0, unused = 0;
  uint8_t first;
  int e;
  const int ntok = el_tokens(t, a, b, 0, lscc ? 3 : 2, lscc ? 4u : 0u, u, w, unused, e, first);
  if (!lscc && (ntok == 0 || first == '#' || first == '%')) return 0;       // blank or comment line
  *edge = 1;
  if (e) { *err = e; return 0; }
  if (lscc ? ntok != 3 : ntok < 2) { *err = GCCB_EL_ERR_TOKENS; return 0; }
  if (u == w) return 0;                                                     // self loop (x2dgl.py:41-42)
  const long long hi = lscc ? n : kPlainMult;
  if (u < 0 || u >= hi || w < 0 || w >= hi) { *err = GCCB_EL_ERR_RANGE; return 0; }
  *s = u < w ? u : w;
  *d = u < w ? w : u;
  return 1;
}

// ---- line index --------------------------------------------------------------------------------------------
// grid = tiles, block = 256: newlines per 4 KiB tile.
__global__ void __launch_bounds__(256)
el_nl_count_kernel(const uint8_t* __restrict__ text, int64_t nbytes, int64_t* __restrict__ tile_cnt) {
  __shared__ int warp_cnt[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * kNlTile + w * (kNlTile / 8);
  int cnt = 0;
  for (int it = 0; it < kNlTile / 8 / 32; ++it) {
    const int64_t p = base + it * 32 + lane;
    cnt += __popc(__ballot_sync(0xffffffffu, p < nbytes && text[p] == '\n'));
  }
  if (lane == 0) warp_cnt[w] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long s = 0;
    for (int k = 0; k < 8; ++k) s += warp_cnt[k];
    tile_cnt[blockIdx.x] = s;
  }
}

__device__ __forceinline__ long long el_warp_scan_incl(long long v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  return v;
}

// Exclusive scan of a[0 .. len) in place; *total = the sum.  len = the host's value, or, when lines is set,
// the line tiles of *lines.  One block of 1024 threads.
__global__ void __launch_bounds__(1024)
el_scan_kernel(int64_t* __restrict__ a, int64_t len, const int64_t* __restrict__ lines, int64_t* __restrict__ total) {
  __shared__ long long wsum[32];
  __shared__ long long carry;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (lines) len = (*lines + kLineTile - 1) / kLineTile;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int64_t b0 = 0; b0 < len; b0 += 1024) {
    const int64_t i = b0 + tid;
    const long long v = i < len ? (long long)a[i] : 0;
    const long long incl = el_warp_scan_incl(v, lane);
    if (lane == 31) wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
      const long long s = wsum[lane];
      wsum[lane] = el_warp_scan_incl(s, lane) - s;
    }
    __syncthreads();
    const long long c = carry;
    if (i < len) a[i] = c + wsum[w] + incl - v;
    __syncthreads();
    if (tid == 1023) carry = c + wsum[31] + incl;
    __syncthreads();
  }
  if (tid == 0) *total = carry;
}

// grid = tiles, block = 256: line_end[rank] = offset of every newline; the last block also closes a final line
// without a newline (line_end = nbytes) and stores the chunk's line count in scratch[1].
__global__ void __launch_bounds__(256)
el_nl_write_kernel(const uint8_t* __restrict__ text, int64_t nbytes, const int64_t* __restrict__ tile_off,
                   int64_t* __restrict__ line_end, int64_t* __restrict__ scratch) {
  __shared__ int warp_cnt[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * kNlTile + w * (kNlTile / 8);
  const unsigned below = (1u << lane) - 1u;
  int cnt = 0;
  for (int it = 0; it < kNlTile / 8 / 32; ++it) {
    const int64_t p = base + it * 32 + lane;
    cnt += __popc(__ballot_sync(0xffffffffu, p < nbytes && text[p] == '\n'));
  }
  if (lane == 0) warp_cnt[w] = cnt;
  __syncthreads();
  long long rank = tile_off[blockIdx.x];
  for (int k = 0; k < w; ++k) rank += warp_cnt[k];
  for (int it = 0; it < kNlTile / 8 / 32; ++it) {
    const int64_t p = base + it * 32 + lane;
    const bool nl = p < nbytes && text[p] == '\n';
    const unsigned mask = __ballot_sync(0xffffffffu, nl);
    if (nl) line_end[rank + __popc(mask & below)] = p;
    rank += __popc(mask);
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    const long long nl = scratch[0];
    const bool tail = text[nbytes - 1] != '\n';
    if (tail) line_end[nl] = nbytes;
    scratch[1] = nl + (tail ? 1 : 0);
  }
}

// ---- .lscc header ------------------------------------------------------------------------------------------
// One thread: the second token of line 0 is n, the second token of line n + 1 is m (x2dgl.py:30-36).
__device__ long long el_header_value(const uint8_t* t, const int64_t* line_end, int64_t i, long long g,
                                     gccb_edgelist_state_t* st) {
  int64_t a, b;
  el_line_span(line_end, i, &a, &b);
  long long v = 0, unused1 = 0, unused2 = 0;
  uint8_t first;
  int e;
  const int ntok = el_tokens(t, a, b, 1, 1, 0u, v, unused1, unused2, e, first);
  if (ntok < 2) e = GCCB_EL_ERR_TOKENS;
  else if (!e && (v < 0 || v >= kPlainMult)) e = GCCB_EL_ERR_RANGE;   // the CSR holds int32 vertex ids
  if (e) {
    el_error(st, g, e);
    return -2;
  }
  return v;
}

__global__ void el_header_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ line_end,
                                 const int64_t* __restrict__ scratch, gccb_edgelist_state_t* st) {
  const long long lines = scratch[1], g0 = st->lines;
  if (g0 == 0 && lines > 0) st->n = el_header_value(text, line_end, 0, 0, st);
  const long long n = st->n;
  if (n >= 0 && st->m == -1 && n + 1 >= g0 && n + 1 < g0 + lines)
    st->m = el_header_value(text, line_end, n + 1 - g0, n + 1, st);
}

// ---- parse -------------------------------------------------------------------------------------------------
// Count pass: errors, edge lines, max id (plain), kept lines per line tile.  Grid-stride over line tiles.
__global__ void __launch_bounds__(256)
el_parse_count_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ line_end,
                      const int64_t* __restrict__ scratch, int format, gccb_edgelist_state_t* st,
                      int64_t* __restrict__ keep_cnt) {
  __shared__ int red_keep[8], red_edge[8];
  __shared__ long long red_max[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long lines = scratch[1], g0 = st->lines, n = st->n, m = st->m;
  const long long tiles = (lines + kLineTile - 1) / kLineTile;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long i = tile * kLineTile + threadIdx.x;
    long long s = 0, d = 0;
    int keep = 0, edge = 0, err = 0;
    if (i < lines) {
      keep = el_parse_line(text, line_end, i, g0 + i, format, n, m, &s, &d, &edge, &err);
      if (err) el_error(st, g0 + i, err);
    }
    int k = warp_sum_i(keep), e = warp_sum_i(edge);
    long long mx = keep ? d + 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const long long t = __shfl_xor_sync(0xffffffffu, mx, o);
      mx = t > mx ? t : mx;
    }
    if (lane == 0) { red_keep[w] = k; red_edge[w] = e; red_max[w] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
      long long kk = 0, ee = 0, mm = 0;
      for (int q = 0; q < 8; ++q) {
        kk += red_keep[q];
        ee += red_edge[q];
        mm = red_max[q] > mm ? red_max[q] : mm;
      }
      keep_cnt[tile] = kk;
      if (ee) atomicAdd((unsigned long long*)&st->edge_lines, (unsigned long long)ee);
      if (format == GCCB_EL_PLAIN && mm) atomicMax((long long*)&st->n, mm);
    }
    __syncthreads();
  }
}

// Write pass: the kept lines' keys min*mult + max, max*mult + min at 2 * (their rank among kept lines).
__global__ void __launch_bounds__(256)
el_parse_write_kernel(const uint8_t* __restrict__ text, const int64_t* __restrict__ line_end,
                      const int64_t* __restrict__ scratch, int format, const int64_t* __restrict__ keep_off,
                      const gccb_edgelist_state_t* st_c, gccb_edgelist_state_t* st, int64_t* __restrict__ keys,
                      int64_t keys_cap) {
  __shared__ int scan_scratch[33];
  const long long lines = scratch[1], g0 = st_c->lines, key0 = st_c->keys;
  const long long n = format == GCCB_EL_LSCC ? st_c->n : 0, m = st_c->m;
  const long long mult = format == GCCB_EL_LSCC ? n : kPlainMult;
  const long long tiles = (lines + kLineTile - 1) / kLineTile;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long i = tile * kLineTile + threadIdx.x;
    long long s = 0, d = 0;
    int keep = 0, edge, err;
    if (i < lines) keep = el_parse_line(text, line_end, i, g0 + i, format, n, m, &s, &d, &edge, &err);
    int tot;
    const int r = block_scan_excl(keep, scan_scratch, &tot);
    if (keep) {
      const long long slot = key0 + 2 * (keep_off[tile] + r);
      if (slot + 2 > keys_cap) {
        el_error(st, g0 + i, GCCB_EL_ERR_CAPACITY);
      } else {
        keys[slot] = s * mult + d;
        keys[slot + 1] = d * mult + s;
      }
    }
  }
}

__global__ void el_advance_kernel(const int64_t* __restrict__ scratch, gccb_edgelist_state_t* st) {
  st->lines += scratch[1];
  st->keys += 2 * scratch[2];
}

// ---- end of file ---------------------------------------------------------------------------------------------
// .lscc: a header line or edge lines missing (the reference's readline returns "" there and the unpack raises).
__global__ void el_finish_lscc_kernel(gccb_edgelist_state_t* st) {
  const long long n = st->n, m = st->m;
  if (n == -1) el_error(st, 0, GCCB_EL_ERR_SHORT);
  else if (n >= 0 && m == -1) el_error(st, n + 1, GCCB_EL_ERR_SHORT);
  else if (n >= 0 && m >= 0 && st->edge_lines < m) el_error(st, n + 2 + st->edge_lines, GCCB_EL_ERR_SHORT);
}

// plain: n is known now; keys s * 2^31 + d become s * n + d (same order).
__global__ void __launch_bounds__(256)
el_rekey_kernel(const gccb_edgelist_state_t* st, int64_t* __restrict__ keys) {
  const long long count = st->keys, n = st->n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x) {
    const long long k = keys[i];
    keys[i] = (k >> 31) * n + (k & (kPlainMult - 1));
  }
}

__global__ void el_begin_kernel(gccb_edgelist_state_t* st, int format) {
  st->lines = 0;
  st->n = format == GCCB_EL_LSCC ? -1 : 0;
  st->m = -1;
  st->edge_lines = 0;
  st->keys = 0;
  st->first_error = ~0ULL;
  st->error_flags = 0;
  st->_pad = 0;
}

}  // namespace gccb

using namespace gccb;

extern "C" size_t gccb_edgelist_workspace(int64_t chunk_bytes) {
  return chunk_bytes <= 0 ? 0 : el_layout(chunk_bytes).total;
}

extern "C" int gccb_edgelist_begin(int32_t format, void* workspace, size_t workspace_bytes, gccb_stream_t stream) {
  if ((format != GCCB_EL_LSCC && format != GCCB_EL_PLAIN) || !workspace ||
      workspace_bytes < sizeof(gccb_edgelist_state_t)) {
    set_last_error("gccb_edgelist_begin: bad argument");
    return GCCB_ERR_BADARG;
  }
  GCCB_LAUNCH(el_begin_kernel, 1, 1, 0, stream, (gccb_edgelist_state_t*)workspace, (int)format);
  return check_launch("gccb_edgelist_begin");
}

extern "C" int gccb_edgelist_parse(const char* text, int64_t nbytes, int32_t format, int64_t* keys, int64_t keys_cap,
                                   void* workspace, size_t workspace_bytes, gccb_stream_t stream) {
  if ((format != GCCB_EL_LSCC && format != GCCB_EL_PLAIN) || !workspace || nbytes < 0 || (nbytes > 0 && !text) ||
      (keys_cap > 0 && !keys) || keys_cap < 0 || workspace_bytes < gccb_edgelist_workspace(nbytes)) {
    set_last_error("gccb_edgelist_parse: bad argument (nbytes %lld, workspace %zu bytes, %zu needed)",
                   (long long)nbytes, workspace_bytes, (size_t)gccb_edgelist_workspace(nbytes));
    return GCCB_ERR_BADARG;
  }
  if (nbytes == 0) return GCCB_OK;
  const ElLayout L = el_layout(nbytes);
  char* ws = (char*)workspace;
  gccb_edgelist_state_t* st = (gccb_edgelist_state_t*)ws;
  int64_t* scratch = (int64_t*)(ws + L.scratch);
  int64_t* tile_cnt = (int64_t*)(ws + L.tile_cnt);
  int64_t* line_end = (int64_t*)(ws + L.line_end);
  int64_t* keep_cnt = (int64_t*)(ws + L.keep_cnt);
  const uint8_t* t = (const uint8_t*)text;
  const int64_t tiles = (nbytes + kNlTile - 1) / kNlTile;
  const int64_t line_tiles = (nbytes + 1 + kLineTile - 1) / kLineTile;
  const int parse_grid = (int)(line_tiles < kMaxParseBlocks ? line_tiles : kMaxParseBlocks);
  GCCB_LAUNCH(el_nl_count_kernel, (unsigned)tiles, 256, 0, stream, t, nbytes, tile_cnt);
  GCCB_LAUNCH(el_scan_kernel, 1, 1024, 0, stream, tile_cnt, tiles, (const int64_t*)nullptr, scratch);
  GCCB_LAUNCH(el_nl_write_kernel, (unsigned)tiles, 256, 0, stream, t, nbytes, (const int64_t*)tile_cnt, line_end,
              scratch);
  if (format == GCCB_EL_LSCC)
    GCCB_LAUNCH(el_header_kernel, 1, 1, 0, stream, t, (const int64_t*)line_end, (const int64_t*)scratch, st);
  GCCB_LAUNCH(el_parse_count_kernel, parse_grid, 256, 0, stream, t, (const int64_t*)line_end,
              (const int64_t*)scratch, (int)format, st, keep_cnt);
  GCCB_LAUNCH(el_scan_kernel, 1, 1024, 0, stream, keep_cnt, (int64_t)0, (const int64_t*)(scratch + 1), scratch + 2);
  GCCB_LAUNCH(el_parse_write_kernel, parse_grid, 256, 0, stream, t, (const int64_t*)line_end,
              (const int64_t*)scratch, (int)format, (const int64_t*)keep_cnt, (const gccb_edgelist_state_t*)st, st,
              keys, keys_cap);
  GCCB_LAUNCH(el_advance_kernel, 1, 1, 0, stream, (const int64_t*)scratch, st);
  return check_launch("gccb_edgelist_parse");
}

extern "C" int gccb_edgelist_finish(int32_t format, int64_t* keys, void* workspace, size_t workspace_bytes,
                                    gccb_stream_t stream) {
  if ((format != GCCB_EL_LSCC && format != GCCB_EL_PLAIN) || !workspace ||
      workspace_bytes < sizeof(gccb_edgelist_state_t) || (format == GCCB_EL_PLAIN && !keys)) {
    set_last_error("gccb_edgelist_finish: bad argument");
    return GCCB_ERR_BADARG;
  }
  gccb_edgelist_state_t* st = (gccb_edgelist_state_t*)workspace;
  if (format == GCCB_EL_LSCC) GCCB_LAUNCH(el_finish_lscc_kernel, 1, 1, 0, stream, st);
  else GCCB_LAUNCH(el_rekey_kernel, kMaxParseBlocks, 256, 0, stream, (const gccb_edgelist_state_t*)st, keys);
  return check_launch("gccb_edgelist_finish");
}

// sampler.cu -- seed draw, random walk with restart, ego-net induction, batching.
//
// Replaces (reference file:line):
//   LoadBalanceGraphDataset.__iter__ seed draw            gcc/datasets/graph_dataset.py:85-92
//   budget + dgl...random_walk_with_restart([s, s])        gcc/datasets/graph_dataset.py:113-130
//   _rwr_trace_to_dgl_graph (unique, sort, seed first,
//     g.subgraph, seed one-hot)                            gcc/datasets/data_util.py:218-239
//   batcher() / dgl.batch                                  gcc/datasets/data_util.py:26-32
//
// Design (H100): one CTA per (sample, view).  Trace lengths depend only on the
// counter-based RNG, so the stopping trace T* is found without touching memory;
// then all traces are walked in parallel (dependent-load depth = longest single
// trace, not the whole budget).  The visited list is bitonic-sorted / uniqued in
// shared memory; induction streams each visited vertex's neighbour list with
// coalesced warp loads and binary-searches the shared-memory frontier.  Every neighbour
// list is read ONCE: the local ids of the hits are parked in a scratch pool while the induced
// degrees are counted, the per-view scan fixes the (deterministic) output layout, and the fill
// kernel only copies pool -> batched CSR.  Hits wait in a per-warp shared-memory stage until their row's
// count is known (rows with more than 128 induced neighbours are the exception: counted first, recorded on a
// second look).  A one-hash membership filter of the frontier rejects most scanned neighbours with one shared-
// memory load.  Hub rows (degree > 16 n) are not streamed: the ego-net's vertices are looked up in the hub's
// sorted list, by the whole CTA at once.
#include "common.cuh"

namespace gccb {

__global__ void draw_seeds_kernel(const double* __restrict__ cdf, int64_t n, uint64_t key,
                                  int64_t first, int count, int64_t* __restrict__ seeds,
                                  int64_t* __restrict__ sample_ids) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  uint64_t sample = (uint64_t)(first + i);
  u32x4 w = philox_at(key, sample, 0, 0, 0, GCCB_TAG_SEED);
  uint64_t u53 = ((uint64_t)w.x << 21) | (uint64_t)(w.y >> 11);
  double u = (double)u53 * (1.0 / 9007199254740992.0);
  int64_t lo = 0, hi = n;                  // first index with cdf[i] > u
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  seeds[i] = lo < n ? lo : n - 1;
  if (sample_ids) sample_ids[i] = first + i;
}

// membership of u in the ego-net: local id or -1.  keys[0] = seed, keys[1..n) ascending.
__device__ __forceinline__ int local_id(const int* keys, int n, int seed, int u) {
  if (u == seed) return 0;
  int lo = 1, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (keys[mid] < u) lo = mid + 1; else hi = mid;
  }
  return (lo < n && keys[lo] == u) ? lo : -1;
}

// bit of the membership filter for parent id u (Knuth's multiplicative hash, top 16 bits)
__device__ __forceinline__ unsigned bloom_bit(int u) { return ((unsigned)u * 2654435761u) >> 16; }

// neighbour lists are ascending (gccb_graph_t contract): membership of u in adj(v) by bisection
__device__ __forceinline__ bool adj_find(const int32_t* __restrict__ indices, int64_t beg, int64_t end, int u) {
  const int64_t stop = end;
  while (beg < end) {
    int64_t mid = (beg + end) >> 1;
    if (indices[mid] < u) beg = mid + 1; else end = mid;
  }
  return beg < stop && indices[beg] == u;
}
// A hub row (parent degree >> ego-net size) is not streamed: each ego-net vertex is looked up in the
// hub's sorted neighbour list instead (n log deg probes instead of deg reads).
#define GCCB_REVERSE_FACTOR 16
#ifndef GCCB_ST
#define GCCB_ST 1024           // threads per CTA of the walk / fill kernels: hub ego-nets (thousands of
                               // vertices, ~1e5..1e6 neighbour probes) are the tail of these kernels
#endif
#define GCCB_SW (GCCB_ST / 32)
#ifndef GCCB_SCAN_UNROLL
#define GCCB_SCAN_UNROLL 4     // 32-element chunks of a neighbour list loaded before the first is searched
#endif
#ifndef GCCB_BLOOM
#define GCCB_BLOOM 1           // A/B switches (profiles/build_variant.py)
#endif
#define GCCB_BLOOM_WORDS 2048   // 65,536 bits: 0.6 % false positives at n = 400, 7 % at n = 5,000
#define GCCB_HUB_LIST 1024     // hub rows per ego-net handled CTA-wide (further ones fall back to one warp each)
#define GCCB_HIT_STAGE 128     // hits of one row parked in shared memory before their pool slot is known

// Pass 1: walk + sort/unique + induced-degree count.  grid = 2B, block = GCCB_ST.
// dyn smem: keys[P] ints, P = pow2 >= max_budget + HOPCAP.
__global__ void __launch_bounds__(GCCB_ST)
rwr_walk_unique_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int64_t n_nodes,
                       const int32_t* __restrict__ budget_table, int budget_table_len,
                       uint32_t restart_thresh, uint64_t key, const int64_t* __restrict__ seeds,
                       const int64_t* __restrict__ sample_ids, int B, int cap_n,
                       int32_t* __restrict__ subv_scratch, int32_t* __restrict__ subdeg_scratch,
                       int32_t* __restrict__ rowstart_scratch, int32_t* __restrict__ pool, int pool_cap,
                       unsigned long long* __restrict__ pool_counter,
                       int64_t* __restrict__ counters, int32_t* __restrict__ flags) {
  GCCB_DYN_SMEM(int, keys);
  __shared__ int scan_scratch[33];
  __shared__ int stage[GCCB_SW][GCCB_HIT_STAGE];      // per-warp parking of one row's hits
  __shared__ int s_tstar, s_m;
  __shared__ unsigned long long s_sumdeg;
  __shared__ int s_nhub, s_pos;
  __shared__ unsigned bloom[GCCB_BLOOM_WORDS];        // one-hash membership filter of the frontier (8 KB)
  __shared__ int hub_rows[GCCB_HUB_LIST];             // hub rows of this ego-net: probed by the whole CTA
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int slot = blockIdx.x;            // view-major: slot = view * B + g
  const int view = slot / B, g = slot - view * B;
  int64_t seed64 = seeds[g];
  seed64 = seed64 < 0 ? 0 : (seed64 >= n_nodes ? n_nodes - 1 : seed64);   // caller-supplied seeds: never read out of bounds
  const int seed = (int)seed64;
  const uint64_t sample = (uint64_t)sample_ids[g];
  int64_t sdeg = indptr[seed64 + 1] - indptr[seed64];
  const int budget = budget_table[sdeg < budget_table_len ? (int)sdeg : budget_table_len - 1];

  if (tid == 0) { s_tstar = 0x7fffffff; s_m = 0; s_sumdeg = 0ull; }
  __syncthreads();

  // ---- phase A+B: trace lengths (RNG only), stopping trace, parallel walk ------------
  int base = 0;          // recorded nodes before this chunk
  int total = 0;
  for (int chunk = 0;; ++chunk) {
    const uint32_t t = (uint32_t)(chunk * GCCB_ST + tid);
    int len = 1;         // hop 0 is always taken
    for (uint32_t hop = 1; hop < GCCB_HOPCAP; ++hop) {
      u32x4 w = philox_at(key, sample, t, hop, (uint32_t)view, GCCB_TAG_WALK);
      if (w.x < restart_thresh) break;
      ++len;
    }
    int chunk_total;
    int excl = block_scan_excl(len, scan_scratch, &chunk_total);
    int cum = base + excl + len;           // inclusive cumulative count after trace t
    if (cum >= budget && cum - len < budget) s_tstar = (int)t;   // exactly one thread
    __syncthreads();
    const int tstar = s_tstar;
    if ((int)t <= tstar) {
      // walk this trace; its nodes land at keys[base+excl .. +len)
      int64_t cur = seed64;
      int pos = base + excl;
      for (uint32_t hop = 0; hop < (uint32_t)len; ++hop) {
        u32x4 w = philox_at(key, sample, t, hop, (uint32_t)view, GCCB_TAG_WALK);
        int64_t beg = indptr[cur];
        uint32_t deg = (uint32_t)(indptr[cur + 1] - beg);
        if (deg == 0u) { atomicOr(flags, (int)GCCB_FLAG_ZERO_DEGREE); keys[pos++] = (int)cur; continue; }
        cur = indices[beg + __umulhi(w.y, deg)];
        keys[pos++] = (int)cur;
      }
    }
    if (tstar != 0x7fffffff) {
      // total = cumulative count after trace tstar (held by the thread that owns it)
      if ((int)t == tstar) s_m = cum;
      __syncthreads();
      total = s_m;
      break;
    }
    base += chunk_total;
    __syncthreads();
  }
  __syncthreads();
  if (tid == 0) s_m = 0;

  // ---- phase C: bitonic sort of keys[0..total), padded to a power of two --------------
  int P = 1;
  while (P < total) P <<= 1;
  for (int i = total + tid; i < P; i += GCCB_ST) keys[i] = 0x7fffffff;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += GCCB_ST) {
        int ixj = i ^ j;
        if (ixj > i) {
          int a = keys[i], b = keys[ixj];
          bool asc = (i & k) == 0;
          if ((a > b) == asc) { keys[i] = b; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  // ---- unique, drop the seed; subv = [seed] + sorted rest (data_util.py:221-226) -------
  int32_t* subv = subv_scratch + (size_t)slot * cap_n;
  int n_rest = 0;
  for (int b0 = 0; b0 < total; b0 += GCCB_ST) {
    int i = b0 + tid;
    int head = 0, v = 0;
    if (i < total) {
      v = keys[i];
      head = (v != seed) && (i == 0 || keys[i - 1] != v);
    }
    int cnt;
    int ex = block_scan_excl(head, scan_scratch, &cnt);
    if (head) subv[1 + n_rest + ex] = v;
    n_rest += cnt;
  }
  const int n = n_rest + 1;
  if (tid == 0) subv[0] = seed;
  __syncthreads();                       // global writes of this block visible to the block
  for (int i = tid; i < n; i += GCCB_ST) keys[i] = subv[i];
  for (int i = tid; i < GCCB_BLOOM_WORDS; i += GCCB_ST) bloom[i] = 0u;
  __syncthreads();
  // 99 % of the scanned neighbours are not in the ego-net: one shared-memory load rejects them, only the
  // filter's candidates pay for the binary search of the frontier
  for (int i = tid; i < n; i += GCCB_ST) {
    const unsigned b = bloom_bit(keys[i]);
    atomicOr(&bloom[b >> 5], 1u << (b & 31u));
  }
  __syncthreads();

  // ---- phase D: induced neighbours of every ego-net vertex (warp per vertex), ONE look at each list ------
  // Hits (local ids, in the order a scan of adj(v) meets them) are parked per warp, then moved to a slot of
  // the scratch pool claimed with one atomic per row; the fill kernel copies pool -> batched CSR.
  int32_t* subdeg = subdeg_scratch + (size_t)slot * cap_n;
  int32_t* rowstart = rowstart_scratch + (size_t)slot * cap_n;
  int* wstage = stage[warp];
  const unsigned lt_mask = (1u << lane) - 1u;
  int m_local = 0;
  unsigned long long sumdeg_local = 0ull;
  int sr = 0;                                            // rank of the seed among the sorted non-seed keys
  {
    int lo = 1, hi = n;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (keys[mid] < seed) lo = mid + 1; else hi = mid; }
    sr = lo - 1;
  }
  // Hub rows first, with the whole CTA: a reverse probe is a chain of ~log2(deg) dependent global loads per key, so
  // one warp needs n/32 such chains back to back for ONE row (a 326k-neighbour RMAT hub in a 400-vertex ego-net:
  // ~120 us, and hub-rich ego-nets hold dozens of them); 1024 threads probe all keys of the row at once.
  if (tid == 0) s_nhub = 0;
  __syncthreads();
  for (int i = tid; i < n; i += GCCB_ST) {
    const int64_t v = keys[i];
    int mark = -3;
    if (indptr[v + 1] - indptr[v] > (int64_t)GCCB_REVERSE_FACTOR * n) {
      const int idx = atomicAdd(&s_nhub, 1);
      if (idx < GCCB_HUB_LIST) { hub_rows[idx] = i; mark = -2; }
    }
    rowstart[i] = mark;                                  // -2: handled below, not by the warp loop
  }
  __syncthreads();
  const int n_hub = min(s_nhub, GCCB_HUB_LIST);
  for (int h = 0; h < n_hub; ++h) {
    const int i = hub_rows[h];
    const int64_t v = keys[i];
    const int64_t beg = indptr[v], end = indptr[v + 1];
    int cnt = 0, my_j = -1, my_ex = 0;
    for (int t0 = 0; t0 < n; t0 += GCCB_ST) {            // count (ascending parent id, the seed spliced in at rank sr)
      const int t = t0 + tid;
      int j = -1;
      if (t < n) {
        const int loc = t < sr ? t + 1 : (t == sr ? 0 : t);
        if (adj_find(indices, beg, end, keys[loc])) j = loc;
      }
      int tot;
      const int ex = block_scan_excl(j >= 0 ? 1 : 0, scan_scratch, &tot);
      if (t0 == 0) { my_j = j; my_ex = ex; }
      cnt += tot;
    }
    if (tid == 0) {
      const unsigned long long p64 = cnt > 0 ? atomicAdd(pool_counter, (unsigned long long)cnt) : 0ull;
      s_pos = p64 + (unsigned long long)cnt > (unsigned long long)pool_cap ? -1 : (int)p64;   // exhausted: the fill kernel looks again itself
    }
    __syncthreads();
    const int pos = s_pos;
    if (pos >= 0) {
      if (n <= GCCB_ST) {
        if (my_j >= 0) pool[pos + my_ex] = my_j;
      } else {
        int w = 0;
        for (int t0 = 0; t0 < n; t0 += GCCB_ST) {
          const int t = t0 + tid;
          int j = -1;
          if (t < n) {
            const int loc = t < sr ? t + 1 : (t == sr ? 0 : t);
            if (adj_find(indices, beg, end, keys[loc])) j = loc;
          }
          int tot;
          const int ex = block_scan_excl(j >= 0 ? 1 : 0, scan_scratch, &tot);
          if (j >= 0) pool[pos + w + ex] = j;
          w += tot;
        }
      }
    }
    if (tid == 0) {
      subdeg[i] = cnt;
      rowstart[i] = pos;
      m_local += cnt;
      sumdeg_local += (unsigned long long)(end - beg);
    }
    __syncthreads();                                     // s_pos / scan_scratch are reused by the next hub row
  }
  for (int i = warp; i < n; i += GCCB_SW) {
    if (rowstart[i] != -3) continue;                     // a hub row: done above
    const int64_t v = keys[i];
    const int64_t beg = indptr[v], end = indptr[v + 1];
    const bool reverse = end - beg > (int64_t)GCCB_REVERSE_FACTOR * n;
    // Hits are parked in the warp's shared-memory stage until the row's count is known, then moved to a pool
    // slot claimed with one atomic.  A row with more hits than the stage holds (> 128 induced neighbours) is
    // counted first and recorded on a second look.  (Claiming an upper bound min(deg, n) on the spot instead --
    // one look -- was measured on the RMAT sweep: the slack exhausts the pool and costs more than the re-scan.)
    int pos = 0, w = 0, round = 0;
    auto emit = [&](int j) {                             // called by all lanes; j < 0: no hit on this lane
      const unsigned hit = __ballot_sync(0xffffffffu, j >= 0);
      if (j >= 0) {
        const int q = w + __popc(hit & lt_mask);
        if (round == 1) pool[pos + q] = j;
        else if (q < GCCB_HIT_STAGE) wstage[q] = j;
      }
      w += __popc(hit);
    };
    auto scan_row = [&]() {
      w = 0;
      if (reverse) {
        // hub row (beyond the CTA-wide list): probe adj(v) for every ego-net vertex in ascending parent id (= the
        // order a scan of adj(v) would meet them): keys[1..n) is ascending, the seed (local id 0) is spliced in at rank sr
        for (int t0 = 0; t0 < n; t0 += 32) {
          const int t = t0 + lane;
          int j = -1;
          if (t < n) {
            const int loc = t < sr ? t + 1 : (t == sr ? 0 : t);
            if (adj_find(indices, beg, end, keys[loc])) j = loc;
          }
          emit(j);
        }
      } else {
        // four independent 128-byte loads in flight per warp before the first search: the scan of a cold
        // neighbour list is bound by memory-level parallelism, not by the searches (-18 % on the RMAT sweep)
        for (int64_t e0 = beg; e0 < end; e0 += 32 * GCCB_SCAN_UNROLL) {
          int u[GCCB_SCAN_UNROLL];
#pragma unroll
          for (int k = 0; k < GCCB_SCAN_UNROLL; ++k) {
            const int64_t e = e0 + 32 * k + lane;
            u[k] = e < end ? indices[e] : -1;
          }
#pragma unroll
          for (int k = 0; k < GCCB_SCAN_UNROLL; ++k) {
            if (e0 + 32 * k >= end) break;                  // warp-uniform
            int j = -1;
            if (u[k] >= 0) {
#if GCCB_BLOOM
              const unsigned b = bloom_bit(u[k]);
              if ((bloom[b >> 5] >> (b & 31u)) & 1u)
#endif
                j = local_id(keys, n, seed, u[k]);
            }
            emit(j);
          }
        }
      }
    };
    scan_row();
    const int cnt = w;
    if (lane == 0) {
      const unsigned long long p64 = cnt > 0 ? atomicAdd(pool_counter, (unsigned long long)cnt) : 0ull;
      pos = p64 + (unsigned long long)cnt > (unsigned long long)pool_cap ? -1 : (int)p64;   // exhausted: the fill kernel looks again itself
    }
    pos = __shfl_sync(0xffffffffu, pos, 0);
    if (pos >= 0) {
      if (cnt <= GCCB_HIT_STAGE) {
        __syncwarp();
        for (int q = lane; q < cnt; q += 32) pool[pos + q] = wstage[q];
      } else {
        round = 1;
        scan_row();
      }
    }
    __syncwarp();                                          // wstage is reused by the next row
    if (lane == 0) {
      subdeg[i] = cnt;
      rowstart[i] = pos;
      m_local += cnt;
      sumdeg_local += (unsigned long long)(end - beg);
    }
  }
  if (lane == 0) {
    atomicAdd(&s_m, m_local);
    atomicAdd(&s_sumdeg, sumdeg_local);
  }
  __syncthreads();
  if (tid == 0) {
    counters[(size_t)slot * 4 + 0] = n;
    counters[(size_t)slot * 4 + 1] = s_m;
    counters[(size_t)slot * 4 + 2] = total;
    counters[(size_t)slot * 4 + 3] = (int64_t)s_sumdeg;
  }
}

// Pass 2: per-view exclusive scans of n and m -> node_off / edge_off.  grid = 2, block = 256.
__global__ void __launch_bounds__(256)
batch_offsets_kernel(const int64_t* __restrict__ counters, int B, int node_cap, int edge_cap,
                     int32_t* __restrict__ node_off, int32_t* __restrict__ edge_off,
                     int32_t* __restrict__ flags) {
  __shared__ int scan_scratch[33];
  const int view = blockIdx.x, tid = threadIdx.x;
  long long nbase = 0, ebase = 0;
  for (int b0 = 0; b0 < B; b0 += 256) {
    int g = b0 + tid;
    int n = 0, m = 0;
    if (g < B) {
      n = (int)counters[(size_t)(view * B + g) * 4 + 0];
      m = (int)counters[(size_t)(view * B + g) * 4 + 1];
    }
    int tn, tm;
    int en = block_scan_excl(n, scan_scratch, &tn);
    int em = block_scan_excl(m, scan_scratch, &tm);
    if (g < B) {
      long long no = nbase + en, eo = ebase + em;
      node_off[view * (B + 1) + g] = (int)(no > 0x7fffffffLL ? 0x7fffffffLL : no);
      edge_off[view * (B + 1) + g] = (int)(eo > 0x7fffffffLL ? 0x7fffffffLL : eo);
    }
    nbase += tn;
    ebase += tm;
  }
  if (tid == 0) {
    int f = 0;
    if (nbase > node_cap) { f |= GCCB_FLAG_NODE_OVERFLOW; }
    if (ebase > edge_cap) { f |= GCCB_FLAG_EDGE_OVERFLOW; }
    // on overflow publish an EMPTY view so that no consumer runs out of bounds
    node_off[view * (B + 1) + B] = f ? -1 : (int)nbase;
    edge_off[view * (B + 1) + B] = f ? -1 : (int)ebase;
    if (f) atomicOr(flags, f);
  }
}

// Pass 3: fill the batched CSR.  grid = 2B, block = GCCB_ST, dyn smem keys[P].
__global__ void __launch_bounds__(GCCB_ST)
induce_fill_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                   const int64_t* __restrict__ counters, int B, int cap_n, int node_cap,
                   int edge_cap, const int32_t* __restrict__ subv_scratch,
                   const int32_t* __restrict__ subdeg_scratch, const int32_t* __restrict__ rowstart_scratch,
                   const int32_t* __restrict__ pool,
                   int32_t* __restrict__ node_off, const int32_t* __restrict__ edge_off,
                   int32_t* __restrict__ out_indptr, int32_t* __restrict__ out_indices,
                   int32_t* __restrict__ out_subdeg, int32_t* __restrict__ out_graph_id,
                   int32_t* __restrict__ out_orig_id) {
  GCCB_DYN_SMEM(int, keys);
  __shared__ int scan_scratch[33];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int slot = blockIdx.x;
  const int view = slot / B, g = slot - view * B;
  const int Nv = node_off[view * (B + 1) + B];
  if (Nv < 0) return;                                   // view overflowed: published empty
  const int n = (int)counters[(size_t)slot * 4 + 0];
  const int noff = node_off[view * (B + 1) + g];
  const int eoff = edge_off[view * (B + 1) + g];
  const int32_t* subv = subv_scratch + (size_t)slot * cap_n;
  const int32_t* subdeg = subdeg_scratch + (size_t)slot * cap_n;
  const int32_t* rowstart = rowstart_scratch + (size_t)slot * cap_n;
  int32_t* v_indptr = out_indptr + (size_t)view * (node_cap + 1);
  int32_t* v_indices = out_indices + (size_t)view * edge_cap;
  const size_t nb = (size_t)view * node_cap;
  for (int i = tid; i < n; i += GCCB_ST) keys[i] = subv[i];
  const int seed = subv[0];
  // row starts (view-local edge positions) = eoff + exclusive scan of induced degrees
  int run = 0;
  for (int b0 = 0; b0 < n; b0 += GCCB_ST) {
    int i = b0 + tid;
    int d = i < n ? subdeg[i] : 0;
    int tot;
    int ex = block_scan_excl(d, scan_scratch, &tot);
    if (i < n) {
      v_indptr[noff + i] = eoff + run + ex;
      out_subdeg[nb + noff + i] = d;
      out_graph_id[nb + noff + i] = g;
      out_orig_id[nb + noff + i] = subv[i];
    }
    run += tot;
  }
  if (g == B - 1 && tid == 0) v_indptr[noff + n] = eoff + run;   // closing entry = E_v
  __syncthreads();                                               // keys[] + v_indptr visible
  for (int i = warp; i < n; i += GCCB_SW) {
    int wpos = v_indptr[noff + i];
    const int rs = rowstart[i];
    if (rs >= 0) {                                       // the walk kernel parked this row's hits: copy
      const int d = subdeg[i];
      for (int q = lane; q < d; q += 32) v_indices[wpos + q] = noff + pool[rs + q];
      continue;
    }
    // (pool exhausted while this row was counted: look at its neighbour list again)
    const int64_t v = keys[i];
    const int64_t beg = indptr[v], end = indptr[v + 1];
    if (end - beg > (int64_t)GCCB_REVERSE_FACTOR * n) {
      // candidates in ascending parent id = the order a scan of adj(v) would meet them:
      // keys[1..n) is ascending, the seed (local id 0) is spliced in at its rank sr
      int lo = 1, hi = n;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (keys[mid] < seed) lo = mid + 1; else hi = mid; }
      const int sr = lo - 1;                             // number of non-seed keys below the seed
      for (int t0 = 0; t0 < n; t0 += 32) {
        const int t = t0 + lane;
        int j = -1;
        if (t < n) {
          const int loc = t < sr ? t + 1 : (t == sr ? 0 : t);
          if (adj_find(indices, beg, end, keys[loc])) j = loc;
        }
        unsigned hit = __ballot_sync(0xffffffffu, j >= 0);
        if (j >= 0) v_indices[wpos + __popc(hit & ((1u << lane) - 1u))] = noff + j;
        wpos += __popc(hit);
      }
      continue;
    }
    for (int64_t e0 = beg; e0 < end; e0 += 32) {
      int64_t e = e0 + lane;
      int j = -1;
      if (e < end) j = local_id(keys, n, seed, indices[e]);
      unsigned hit = __ballot_sync(0xffffffffu, j >= 0);
      if (j >= 0) v_indices[wpos + __popc(hit & ((1u << lane) - 1u))] = noff + j;
      wpos += __popc(hit);
    }
  }
}

}  // namespace gccb

using namespace gccb;

static int pow2_ge(int x) { int p = 1; while (p < x) p <<= 1; return p; }

extern "C" int gccb_draw_seeds(const double* cdf, int64_t n_nodes, uint64_t key,
                               int64_t first_sample, int32_t count, int64_t* seeds_out,
                               int64_t* sample_ids_out, gccb_stream_t stream) {
  if (!cdf || !seeds_out || n_nodes <= 0 || count < 0) {
    set_last_error("gccb_draw_seeds: bad argument");
    return GCCB_ERR_BADARG;
  }
  if (count == 0) return GCCB_OK;
  GCCB_LAUNCH(draw_seeds_kernel, (count + 127) / 128, 128, 0, stream, cdf, n_nodes, key,
              first_sample, count, seeds_out, sample_ids_out);
  return check_launch("draw_seeds_kernel");
}

// workspace layout: subv[2B][cap_n] | subdeg[2B][cap_n] | rowstart[2B][cap_n] | pool counter (16 ints) | pool[2*edge_cap]
static int sampler_cap_n(int max_budget) { return (max_budget + (int)GCCB_HOPCAP + 1 + 3) & ~3; }

extern "C" size_t gccb_sample_batch_workspace(int32_t batch, int32_t max_budget, int32_t edge_cap) {
  return ((size_t)3 * (size_t)(2 * batch) * (size_t)sampler_cap_n(max_budget) + 16 + (size_t)2 * (size_t)edge_cap) *
         sizeof(int32_t);
}

extern "C" int gccb_sample_batch(const gccb_graph_t* graph, const int64_t* seeds,
                                 const int64_t* sample_ids, const gccb_batch_t* batch,
                                 void* workspace, size_t workspace_bytes, gccb_stream_t stream) {
  if (!graph || !batch || !seeds || !sample_ids || !workspace || batch->batch <= 0 ||
      graph->max_budget <= 0 || !graph->indptr || !graph->indices || !graph->budget_table) {
    set_last_error("gccb_sample_batch: bad argument");
    return GCCB_ERR_BADARG;
  }
  const int B = batch->batch;
  const int cap_n = sampler_cap_n(graph->max_budget);
  if (workspace_bytes < gccb_sample_batch_workspace(B, graph->max_budget, batch->edge_cap)) {
    set_last_error("gccb_sample_batch: workspace too small");
    return GCCB_ERR_CAPACITY;
  }
  const int P = pow2_ge(graph->max_budget + (int)GCCB_HOPCAP);
  const size_t smem = (size_t)P * sizeof(int);
  if (smem > 200 * 1024) {
    set_last_error("gccb_sample_batch: walk budget %d needs %zu B of shared memory (> 200 KiB)",
                   graph->max_budget, smem);
    return GCCB_ERR_CAPACITY;
  }
  int32_t* subv = (int32_t*)workspace;
  int32_t* subdeg = subv + (size_t)2 * B * cap_n;
  int32_t* rowstart = subdeg + (size_t)2 * B * cap_n;
  unsigned long long* pool_counter = (unsigned long long*)(rowstart + (size_t)2 * B * cap_n);   // 16 ints reserved, 8-byte aligned
  int32_t* pool = (int32_t*)pool_counter + 16;
  // pool positions are stored per row as int32: the pool is capped below 2^31 entries (2 * edge_cap overflows
  // an int for edge_cap > 2^30 -- the 65,536-ego-net sweep of config 5)
  const long long want_cap = 2ll * (long long)batch->edge_cap;
  const int pool_cap = (int)(want_cap < 0x7fff0000ll ? want_cap : 0x7fff0000ll);
  cudaMemsetAsync(pool_counter, 0, sizeof(unsigned long long), (cudaStream_t)stream);
  auto k1 = rwr_walk_unique_kernel;
  auto k3 = induce_fill_kernel;
  if (smem > 48 * 1024) {
    gccb::ensure_dyn_smem(k1, smem);
    gccb::ensure_dyn_smem(k3, smem);
  }
  GCCB_LAUNCH(k1, 2 * B, GCCB_ST, smem, stream, graph->indptr, graph->indices, graph->n_nodes, graph->budget_table,
              graph->budget_table_len, graph->restart_thresh, graph->key, seeds, sample_ids, B,
              cap_n, subv, subdeg, rowstart, pool, pool_cap, pool_counter, batch->counters, batch->flags);
  GCCB_LAUNCH(batch_offsets_kernel, 2, 256, 0, stream, batch->counters, B, batch->node_cap,
              batch->edge_cap, batch->node_off, batch->edge_off, batch->flags);
  GCCB_LAUNCH(k3, 2 * B, GCCB_ST, smem, stream, graph->indptr, graph->indices, batch->counters, B,
              cap_n, batch->node_cap, batch->edge_cap, subv, subdeg, rowstart, pool, batch->node_off,
              batch->edge_off, batch->indptr, batch->indices, batch->sub_deg, batch->graph_id,
              batch->orig_id);
  return check_launch("gccb_sample_batch");
}

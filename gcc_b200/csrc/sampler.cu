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
// sorted list, by the whole CTA at once; a vertex listed c times (parallel edges) is emitted c times.
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

// neighbour lists are non-decreasing (gccb_graph_t contract), a value repeated c times being c parallel edges:
// multiplicity of u in adj(v) by a lower bound, then, on a hit only, an upper bound.  A simple graph's hit costs
// one more load, of the entry next to it.
__device__ __forceinline__ int adj_count(const int32_t* __restrict__ indices, int64_t beg, int64_t end, int u) {
  const int64_t stop = end;
  while (beg < end) {
    int64_t mid = (beg + end) >> 1;
    if (indices[mid] < u) beg = mid + 1; else end = mid;
  }
  if (beg >= stop || indices[beg] != u) return 0;
  // first entry > u, as a 32-bit offset from the first == u (64-bit bounds cost the fill kernel 8 registers)
  const int32_t* run = indices + beg;
  int lo = 1, hi = (int)min(stop - beg, (int64_t)0x7fffffff);
  if (lo == hi || run[lo] != u) return 1;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (run[mid] <= u) lo = mid + 1; else hi = mid;
  }
  return lo;
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
#ifndef GCCB_HUB_LIST
#define GCCB_HUB_LIST 1024     // hub rows per ego-net handled CTA-wide (further ones fall back to one warp each)
#endif
#define GCCB_HIT_STAGE 128     // hits of one row parked in shared memory before their pool slot is known
// Walk CTAs keep the trace in GCCB_WALK_KEYS ints of dynamic shared memory (128 KiB): a sample whose walk budget
// + HOPCAP exceeds it is walked and induced by the wide kernels below, from a key array in global memory.
// (The emulator build lowers it, so that the kernel-logic tests reach the wide path on small graphs.)
#ifndef GCCB_WALK_KEYS
#define GCCB_WALK_KEYS 32768
#endif
#define GCCB_WALK_BUDGET_MAX (GCCB_WALK_KEYS - (int)GCCB_HOPCAP)
#define GCCB_WIDE_CTAS 32      // wide walk CTAs in flight, each with its own key array; they claim slots in turn
#define GCCB_WIDE_KEYS_MAX (1 << 30)   // a wide trace's int32 positions: pow2 >= budget + HOPCAP up to 2^30

// Block-wide ascending bitonic sort of a[0..cnt), padded with INT_MAX to a power of two (the buffer must hold it).
__device__ void block_sort_pad(int* a, int cnt) {
  const int tid = threadIdx.x;
  int P = 1;
  while (P < cnt) P <<= 1;
  for (int i = cnt + tid; i < P; i += GCCB_ST) a[i] = 0x7fffffff;
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < P; i += GCCB_ST) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const int x = a[i], y = a[ixj];
          if ((x > y) == ((i & k) == 0)) { a[i] = y; a[ixj] = x; }
        }
      }
      __syncthreads();
    }
  }
}

__device__ __forceinline__ bool in_sorted(const int* a, int n, int u) {
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (a[mid] < u) lo = mid + 1; else hi = mid; }
  return lo < n && a[lo] == u;
}

// Neighbour-sampled ego-net of `seed` (aug="ns", reference graph_dataset.py:131-162), built in shared memory:
//   V[cap]  the union of all layers so far, ascending (the seed included);
//   F[cap]  the current layer, ascending (a vertex's position in it keys its draws);
//   S[Ps]   candidates of the next layer, then the merge buffer (Ps = pow2 >= max(k, 2) * cap >= k |F|, 2 cap).
// Layer h = the de-duplicated union over u of layer h-1 of all neighbour entries of u if deg(u) <= k, else k distinct
// entries drawn without replacement (Floyd's algorithm: draw t of u uses Philox (sample, position of u | t << 16,
// hop, view, GCCB_TAG_NS)).  A layer is not reduced by the earlier ones: only the final union is.  The loop stops
// early when a layer is empty or when V is closed under neighbourhood (every later layer then lies inside V); a
// layer that merely adds nothing new does not stop it, because the next one draws afresh.
// Writes subv = [seed, V \ {seed} ascending] and returns |V|, or -1 when |V| would exceed cap.  *layers = layers
// expanded.  Every return value is uniform over the block.
__device__ int ns_expand(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, uint64_t key,
                         uint64_t sample, uint32_t view, int seed, int hops, int k, int cap, int* V, int* F, int* S,
                         int* scan_scratch, int32_t* __restrict__ subv, int* layers) {
  __shared__ int s_miss;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int nV = 1, nF = 1, checked = 0, hop = 1;
  if (tid == 0) { V[0] = seed; F[0] = seed; }
  __syncthreads();
  for (; hop <= hops; ++hop) {
    const uint32_t c3hop = (uint32_t)hop & 0xffu, c3tag = GCCB_TAG_NS | (((uint32_t)hop >> 8) << 8);
    // candidates: min(deg, k) entries per vertex of the layer, at the vertex's offset in S
    int nc = 0;
    for (int b0 = 0; b0 < nF; b0 += GCCB_ST) {
      const int i = b0 + tid;
      int64_t beg = 0, d = 0;
      if (i < nF) { beg = indptr[F[i]]; d = indptr[F[i] + 1] - beg; }
      int tot;
      const int ex = block_scan_excl(d <= k ? (int)d : k, scan_scratch, &tot);
      if (i < nF) {
        int* out = S + nc + ex;
        if (d <= k) {
          for (int e = 0; e < (int)d; ++e) out[e] = indices[beg + e];
        } else {
          for (int t = 0; t < k; ++t) {                   // entry positions: k distinct of [0, d)
            const uint32_t j = (uint32_t)(d - k + t);
            const u32x4 w = philox_at(key, sample, (uint32_t)i | ((uint32_t)t << 16), c3hop, view, c3tag);
            const int r = (int)__umulhi(w.x, j + 1u);
            bool dup = false;
            for (int q = 0; q < t; ++q) dup |= out[q] == r;
            out[t] = dup ? (int)j : r;
          }
          for (int t = 0; t < k; ++t) out[t] = indices[beg + out[t]];
        }
      }
      nc += tot;
    }
    __syncthreads();
    block_sort_pad(S, nc);
    // the layer: unique candidates
    int nF2 = 0;
    for (int b0 = 0; b0 < nc; b0 += GCCB_ST) {
      const int i = b0 + tid;
      const int head = i < nc && (i == 0 || S[i - 1] != S[i]);
      int tot;
      const int ex = block_scan_excl(head, scan_scratch, &tot);
      if (head && nF2 + ex < cap) F[nF2 + ex] = S[i];
      nF2 += tot;
    }
    if (nF2 > cap) return -1;                             // the layer alone: so would be the union
    nF = nF2;
    __syncthreads();
    if (nF == 0) break;
    // new vertices of the union, appended to a copy of V and merged by a sort
    int nNew = 0;
    for (int b0 = 0; b0 < nF; b0 += GCCB_ST) {
      const int i = b0 + tid;
      const int fresh = i < nF && !in_sorted(V, nV, F[i]);
      int tot;
      const int ex = block_scan_excl(fresh, scan_scratch, &tot);
      if (fresh) S[nV + nNew + ex] = F[i];
      nNew += tot;
    }
    if (nV + nNew > cap) return -1;
    if (nNew > 0) {
      for (int i = tid; i < nV; i += GCCB_ST) S[i] = V[i];
      block_sort_pad(S, nV + nNew);                       // (syncs before it reads)
      nV += nNew;
      for (int i = tid; i < nV; i += GCCB_ST) V[i] = S[i];
      __syncthreads();
    } else if (nV != checked) {
      // nothing new: stop if no neighbour entry of V lies outside V (one look per size of V)
      if (tid == 0) s_miss = 0;
      __syncthreads();
      int miss = 0;
      for (int i = warp; i < nV; i += GCCB_SW) {
        const int64_t end = indptr[V[i] + 1];
        for (int64_t e = indptr[V[i]] + lane; e < end && !miss; e += 32) miss = !in_sorted(V, nV, indices[e]);
      }
      if (miss) s_miss = 1;
      __syncthreads();
      const bool closed = s_miss == 0;
      __syncthreads();
      if (closed) break;
      checked = nV;
    }
  }
  *layers = hop > hops ? hops : hop;
  for (int i = tid; i < nV; i += GCCB_ST) {
    const int v = V[i];
    subv[v < seed ? i + 1 : (v == seed ? 0 : i)] = v;
  }
  return nV;
}

// RWR node set of one (sample, view) (reference graph_dataset.py:113-130, data_util.py:221-226): the traces from
// seed64 until `budget` vertices are recorded, sorted and uniqued in keys[]; writes rest[0..n-1) = the visited
// vertices but the seed, ascending, and returns n (the caller puts the seed in front).  rest may be keys itself:
// the unique pass writes each vertex at or below the position it reads it from.  *steps = recorded vertices.
// s_tstar and s_m are the kernel's shared words (s_m is left 0).
__device__ __forceinline__ int rwr_node_set(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                            int budget, uint32_t restart_thresh, uint64_t key, uint64_t sample,
                                            int view, int64_t seed64, int seed, int* keys, int* scan_scratch,
                                            int* s_tstar, int* s_m, int32_t* __restrict__ flags,
                                            int32_t* rest, int* steps) {
  const int tid = threadIdx.x;
  if (tid == 0) *s_tstar = 0x7fffffff;
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
    if (cum >= budget && cum - len < budget) *s_tstar = (int)t;   // exactly one thread
    __syncthreads();
    const int tstar = *s_tstar;
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
      if ((int)t == tstar) *s_m = cum;
      __syncthreads();
      total = *s_m;
      break;
    }
    base += chunk_total;
    __syncthreads();
  }
  __syncthreads();
  if (tid == 0) *s_m = 0;

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
    if (head) rest[n_rest + ex] = v;
    n_rest += cnt;
  }
  *steps = total;
  return n_rest + 1;
}

enum { kModeRwr = 0, kModePairs = 1, kModeNs = 2 };

// Pass 1: walk + sort/unique + induced-degree count.  grid = 2B, block = GCCB_ST.
// dyn smem: keys[P] ints, P = pow2 >= max_budget + HOPCAP.
// kMode = kModeRwr: both views walk from seeds[g] (gccb_sample_batch).  kModePairs: view 1 walks from and induces
// around seeds_k[g]; both budgets come from seeds[g]'s degree.  kModeNs: the node set is ns_expand's from seeds[g] /
// seeds_k[g] (dyn smem: its V, F and S, ns_cap = cap_n); a view over cap_n vertices is counted node_cap + 1 vertices,
// no edges, so that batch_offsets_kernel publishes the view empty.  The arguments after `flags` are unused by kModeRwr.
//
// Wide ego-nets (walk budget > GCCB_WALK_BUDGET_MAX: their trace does not fit the CTA's keys[]).  The walk CTA of such
// a slot only writes subv[0] = -1 and leaves it to rwr_walk_wide_kernel, whose GCCB_WIDE_CTAS CTAs claim the slots in
// turn and run the same walk, sort and unique on a key array of their own in global memory.  The node set then moves to
// a region of its view (WideWs), where induction reads it in place of the shared-memory copy; its offset there is
// parked in the slot's subv[1] for induce_fill_wide_kernel.
struct WideWs {
  int32_t* subv;                  // [2][region]: node sets of the view's wide ego-nets, back to back
  int32_t* subdeg;                // [2][region]
  int32_t* rowstart;              // [2][region]
  unsigned long long* used;       // [2] entries of each view's region claimed so far
  unsigned* next;                 // next slot for a wide walk CTA to claim
  int region;
};

template <int kMode, bool kWide>
__device__ __forceinline__ void
walk_slot(const int slot, int* keys, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
          int64_t n_nodes, const int32_t* __restrict__ budget_table, int budget_table_len, uint32_t restart_thresh,
          uint64_t key, const int64_t* __restrict__ seeds, const int64_t* __restrict__ sample_ids, int B, int cap_n,
          int32_t* __restrict__ subv_scratch, int32_t* __restrict__ subdeg_scratch,
          int32_t* __restrict__ rowstart_scratch, int32_t* __restrict__ pool, int pool_cap,
          unsigned long long* __restrict__ pool_counter, int64_t* __restrict__ counters,
          int32_t* __restrict__ flags, const int64_t* __restrict__ seeds_k, int ns_hops, int ns_k, int node_cap,
          const WideWs& wide) {
  __shared__ int scan_scratch[33];
  __shared__ int stage[GCCB_SW][GCCB_HIT_STAGE];      // per-warp parking of one row's hits
  __shared__ int s_tstar, s_m;
  __shared__ unsigned long long s_sumdeg;
  __shared__ int s_nhub, s_pos;
  __shared__ unsigned bloom[GCCB_BLOOM_WORDS];        // one-hash membership filter of the frontier (8 KB)
  __shared__ int hub_rows[GCCB_HUB_LIST];             // hub rows of this ego-net: probed by the whole CTA
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = slot / B, g = slot - view * B;    // view-major: slot = view * B + g
  int64_t seed64 = seeds[g];
  seed64 = seed64 < 0 ? 0 : (seed64 >= n_nodes ? n_nodes - 1 : seed64);   // caller-supplied seeds: never read out of bounds
  const int64_t q64 = seed64;
  if constexpr (kMode != kModeRwr) {
    if (view == 1) {
      seed64 = seeds_k[g];
      seed64 = seed64 < 0 ? 0 : (seed64 >= n_nodes ? n_nodes - 1 : seed64);
    }
  }
  const int seed = (int)seed64;
  const uint64_t sample = (uint64_t)sample_ids[g];
  int32_t* subv = subv_scratch + (size_t)slot * cap_n;
  int32_t* subdeg = subdeg_scratch + (size_t)slot * cap_n;
  int32_t* rowstart = rowstart_scratch + (size_t)slot * cap_n;
  if (tid == 0) { s_m = 0; s_sumdeg = 0ull; }
  int n, total = 0;                                       // total: counters[2] (walk steps / ns layers expanded)
  if constexpr (kMode == kModeNs) {
    n = ns_expand(indptr, indices, key, sample, (uint32_t)view, seed, ns_hops, ns_k, cap_n, keys, keys + cap_n,
                  keys + 2 * cap_n, scan_scratch, subv, &total);
    if (n < 0) {                                          // too large: the whole view is published empty
      if (tid == 0) {
        counters[(size_t)slot * 4 + 0] = (int64_t)node_cap + 1;
        counters[(size_t)slot * 4 + 1] = 0;
        counters[(size_t)slot * 4 + 2] = total;
        counters[(size_t)slot * 4 + 3] = 0;
        atomicOr(flags, (int)GCCB_FLAG_NODE_OVERFLOW);
      }
      return;
    }
    __syncthreads();                                      // subv complete before it is copied to keys
  } else {
    const int64_t sdeg = indptr[q64 + 1] - indptr[q64];   // the budget's seed: the q view's
    const int budget = budget_table[sdeg < budget_table_len ? (int)sdeg : budget_table_len - 1];
    if constexpr (!kWide) {
      if (budget > GCCB_WALK_BUDGET_MAX) {               // rwr_walk_wide_kernel's
        if (tid == 0) subv[0] = -1;
        return;
      }
    }
    n = rwr_node_set(indptr, indices, budget, restart_thresh, key, sample, view, seed64, seed, keys, scan_scratch,
                     &s_tstar, &s_m, flags, kWide ? keys : subv + 1, &total);
  }
  if constexpr (kWide) {
    // room for the node set in the view's region.  None left: the view overflows (gccb_sample_batch_workspace), so
    // the ego-net is only counted, its m as n - 1, a lower bound (every vertex but the seed was entered through an
    // edge inside the ego-net), which keeps the view's edge total above what the region's size allows.
    if (tid == 0) {
      const unsigned long long off = atomicAdd(wide.used + view, (unsigned long long)n);
      s_pos = off + (unsigned long long)n <= (unsigned long long)wide.region ? (int)off : -1;
      subv[1] = s_pos;
    }
    __syncthreads();                                     // also: the node set in keys[] visible to the block
    const int off = s_pos;
    if (off < 0) {
      if (tid == 0) {
        counters[(size_t)slot * 4 + 0] = n;
        counters[(size_t)slot * 4 + 1] = n - 1;
        counters[(size_t)slot * 4 + 2] = total;
        counters[(size_t)slot * 4 + 3] = 0;
      }
      return;
    }
    const size_t at = (size_t)view * wide.region + off;
    subv = wide.subv + at;
    subdeg = wide.subdeg + at;
    rowstart = wide.rowstart + at;
    for (int i = tid; i < n - 1; i += GCCB_ST) subv[1 + i] = keys[i];
    if (tid == 0) subv[0] = seed;
    keys = subv;                                         // induction reads the node set where it is
  } else {
    if (tid == 0) subv[0] = seed;
    __syncthreads();                     // global writes of this block visible to the block
    for (int i = tid; i < n; i += GCCB_ST) keys[i] = subv[i];
  }
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
    // count (ascending parent id, the seed spliced in at rank sr); a key met c times takes c consecutive slots
    int cnt = 0, my_j = 0, my_c = 0, my_ex = 0;
    for (int t0 = 0; t0 < n; t0 += GCCB_ST) {
      const int t = t0 + tid;
      int j = 0, c = 0;
      if (t < n) {
        j = t < sr ? t + 1 : (t == sr ? 0 : t);
        c = adj_count(indices, beg, end, keys[j]);
      }
      int tot;
      const int ex = block_scan_excl(c, scan_scratch, &tot);
      if (t0 == 0) { my_j = j; my_c = c; my_ex = ex; }
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
        for (int k = 0; k < my_c; ++k) pool[pos + my_ex + k] = my_j;
      } else {
        int w = 0;
        for (int t0 = 0; t0 < n; t0 += GCCB_ST) {
          const int t = t0 + tid;
          int j = 0, c = 0;
          if (t < n) {
            j = t < sr ? t + 1 : (t == sr ? 0 : t);
            c = adj_count(indices, beg, end, keys[j]);
          }
          int tot;
          const int ex = block_scan_excl(c, scan_scratch, &tot);
          for (int k = 0; k < c; ++k) pool[pos + w + ex + k] = j;
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
        // order a scan of adj(v) would meet them): keys[1..n) is ascending, the seed (local id 0) is spliced in at rank sr.
        // A key met c times (parallel edges) takes c consecutive slots: a warp prefix sum of the counts.
        for (int t0 = 0; t0 < n; t0 += 32) {
          const int t = t0 + lane;
          int j = 0, c = 0;
          if (t < n) {
            j = t < sr ? t + 1 : (t == sr ? 0 : t);
            c = adj_count(indices, beg, end, keys[j]);
          }
          const int incl = warp_scan_incl(c, lane);
          for (int q = w + incl - c; q < w + incl; ++q) {
            if (round == 1) pool[pos + q] = j;
            else if (q < GCCB_HIT_STAGE) wstage[q] = j;
          }
          w += __shfl_sync(0xffffffffu, incl, 31);
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

template <int kMode>
__global__ void __launch_bounds__(GCCB_ST)
rwr_walk_unique_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int64_t n_nodes,
                       const int32_t* __restrict__ budget_table, int budget_table_len,
                       uint32_t restart_thresh, uint64_t key, const int64_t* __restrict__ seeds,
                       const int64_t* __restrict__ sample_ids, int B, int cap_n,
                       int32_t* __restrict__ subv_scratch, int32_t* __restrict__ subdeg_scratch,
                       int32_t* __restrict__ rowstart_scratch, int32_t* __restrict__ pool, int pool_cap,
                       unsigned long long* __restrict__ pool_counter,
                       int64_t* __restrict__ counters, int32_t* __restrict__ flags,
                       const int64_t* __restrict__ seeds_k, int ns_hops, int ns_k, int node_cap) {
  GCCB_DYN_SMEM(int, keys);
  walk_slot<kMode, false>(blockIdx.x, keys, indptr, indices, n_nodes, budget_table, budget_table_len, restart_thresh,
                          key, seeds, sample_ids, B, cap_n, subv_scratch, subdeg_scratch, rowstart_scratch, pool,
                          pool_cap, pool_counter, counters, flags, seeds_k, ns_hops, ns_k, node_cap, WideWs{});
}

// Pass 1 of the wide ego-nets (kModeRwr / kModePairs), after rwr_walk_unique_kernel.  grid = min(2B, GCCB_WIDE_CTAS),
// block = GCCB_ST, no dynamic shared memory: CTA c walks in wide_keys[c][keys_len] (keys_len = pow2 >= max_budget +
// HOPCAP) and claims slots one by one, taking those whose walk CTA left them (subv[0] = -1).
template <int kMode>
__global__ void __launch_bounds__(GCCB_ST)
rwr_walk_wide_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int64_t n_nodes,
                     const int32_t* __restrict__ budget_table, int budget_table_len,
                     uint32_t restart_thresh, uint64_t key, const int64_t* __restrict__ seeds,
                     const int64_t* __restrict__ sample_ids, int B, int cap_n,
                     int32_t* __restrict__ subv_scratch, int32_t* __restrict__ pool, int pool_cap,
                     unsigned long long* __restrict__ pool_counter,
                     int64_t* __restrict__ counters, int32_t* __restrict__ flags,
                     const int64_t* __restrict__ seeds_k, WideWs wide, int32_t* __restrict__ wide_keys,
                     size_t keys_len) {
  __shared__ int s_slot;
  int* keys = wide_keys + (size_t)blockIdx.x * keys_len;
  for (;;) {
    if (threadIdx.x == 0) s_slot = (int)atomicAdd(wide.next, 1u);
    __syncthreads();
    const int slot = s_slot;
    if (slot >= 2 * B) return;
    if (subv_scratch[(size_t)slot * cap_n] < 0)
      walk_slot<kMode, true>(slot, keys, indptr, indices, n_nodes, budget_table, budget_table_len, restart_thresh,
                             key, seeds, sample_ids, B, cap_n, subv_scratch, nullptr, nullptr, pool, pool_cap,
                             pool_counter, counters, flags, seeds_k, 0, 0, 0, wide);
    __syncthreads();                                     // s_slot and walk_slot's shared words: next slot's
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

// Pass 3: fill the batched CSR of one ego-net.  keys: its node set, a shared-memory copy of subv made here, or (kWide)
// subv itself.
template <bool kWide>
__device__ __forceinline__ void
fill_slot(const int slot, int* keys, const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
          const int64_t* __restrict__ counters, int B, int node_cap, int edge_cap, const int32_t* __restrict__ subv,
          const int32_t* __restrict__ subdeg, const int32_t* __restrict__ rowstart, const int32_t* __restrict__ pool,
          int32_t* __restrict__ node_off, const int32_t* __restrict__ edge_off, int32_t* __restrict__ out_indptr,
          int32_t* __restrict__ out_indices, int32_t* __restrict__ out_subdeg, int32_t* __restrict__ out_graph_id,
          int32_t* __restrict__ out_orig_id) {
  __shared__ int scan_scratch[33];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int view = slot / B, g = slot - view * B;
  const int Nv = node_off[view * (B + 1) + B];
  if (Nv < 0) return;                                   // view overflowed: published empty
  const int n = (int)counters[(size_t)slot * 4 + 0];
  const int noff = node_off[view * (B + 1) + g];
  const int eoff = edge_off[view * (B + 1) + g];
  int32_t* v_indptr = out_indptr + (size_t)view * (node_cap + 1);
  int32_t* v_indices = out_indices + (size_t)view * edge_cap;
  const size_t nb = (size_t)view * node_cap;
  if constexpr (!kWide)
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
        int j = 0, c = 0;
        if (t < n) {
          j = t < sr ? t + 1 : (t == sr ? 0 : t);
          c = adj_count(indices, beg, end, keys[j]);
        }
        const int incl = warp_scan_incl(c, lane);      // parallel edges: c consecutive slots
        for (int q = wpos + incl - c; q < wpos + incl; ++q) v_indices[q] = noff + j;
        wpos += __shfl_sync(0xffffffffu, incl, 31);
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

// grid = 2B, block = GCCB_ST, dyn smem keys[P]
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
  const int slot = blockIdx.x;
  const size_t at = (size_t)slot * cap_n;
  if (subv_scratch[at] < 0) return;                     // a wide ego-net: induce_fill_wide_kernel's
  fill_slot<false>(slot, keys, indptr, indices, counters, B, node_cap, edge_cap, subv_scratch + at,
                   subdeg_scratch + at, rowstart_scratch + at, pool, node_off, edge_off, out_indptr, out_indices,
                   out_subdeg, out_graph_id, out_orig_id);
}

// Pass 3 of the wide ego-nets, after induce_fill_kernel.  grid = 2B, block = GCCB_ST, no dynamic shared memory: the
// CTA of a slot that rwr_walk_wide_kernel induced fills it from the view's region.
__global__ void __launch_bounds__(GCCB_ST)
induce_fill_wide_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                        const int64_t* __restrict__ counters, int B, int cap_n, int node_cap, int edge_cap,
                        const int32_t* __restrict__ subv_scratch, WideWs wide, const int32_t* __restrict__ pool,
                        int32_t* __restrict__ node_off, const int32_t* __restrict__ edge_off,
                        int32_t* __restrict__ out_indptr, int32_t* __restrict__ out_indices,
                        int32_t* __restrict__ out_subdeg, int32_t* __restrict__ out_graph_id,
                        int32_t* __restrict__ out_orig_id) {
  const int slot = blockIdx.x;
  const int32_t* mark = subv_scratch + (size_t)slot * cap_n;
  if (mark[0] >= 0 || mark[1] < 0) return;             // an ordinary slot, or one without room (its view overflowed)
  const size_t at = (size_t)(slot / B) * wide.region + mark[1];
  fill_slot<true>(slot, wide.subv + at, indptr, indices, counters, B, node_cap, edge_cap, wide.subv + at,
                  wide.subdeg + at, wide.rowstart + at, pool, node_off, edge_off, out_indptr, out_indices,
                  out_subdeg, out_graph_id, out_orig_id);
}

// One thread per sample: step ~ step_dist (first index with cdf > u, 53 Philox bits, GCCB_TAG_STEP), then `step`
// uniform hops of a plain walk from seeds_q[i] (hop h: GCCB_TAG_KHOP, hop field h).  A vertex without neighbours ends
// the walk where it is.
__global__ void pair_seeds_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                  int64_t n_nodes, uint64_t key, double cdf0, double cdf1, int n_steps,
                                  const int64_t* __restrict__ seeds_q, const int64_t* __restrict__ sample_ids,
                                  int count, int64_t* __restrict__ seeds_k) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const uint64_t sample = (uint64_t)sample_ids[i];
  const u32x4 w = philox_at(key, sample, 0, 0, 0, GCCB_TAG_STEP);
  const double u = (double)(((uint64_t)w.x << 21) | (uint64_t)(w.y >> 11)) * (1.0 / 9007199254740992.0);
  int step = 0;
  if (step < n_steps - 1 && !(cdf0 > u)) ++step;
  if (step == 1 && step < n_steps - 1 && !(cdf1 > u)) ++step;
  int64_t cur = seeds_q[i];
  cur = cur < 0 ? 0 : (cur >= n_nodes ? n_nodes - 1 : cur);
  for (int h = 1; h <= step; ++h) {
    const int64_t beg = indptr[cur];
    const uint32_t deg = (uint32_t)(indptr[cur + 1] - beg);
    if (deg == 0u) break;
    const u32x4 r = philox_at(key, sample, 0, (uint32_t)h, 0, GCCB_TAG_KHOP);
    cur = indices[beg + __umulhi(r.y, deg)];
  }
  seeds_k[i] = cur;
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
// and, when max_budget > GCCB_WALK_BUDGET_MAX (cap_n then that of GCCB_WALK_BUDGET_MAX):
//   | wide subv[2][R] | wide subdeg[2][R] | wide rowstart[2][R] | wide keys[min(2B, GCCB_WIDE_CTAS)][pow2 >= max_budget + HOPCAP]
// with R = min(edge_cap + B, 2^31 - 1).  The 16 ints hold the pool counter, the next wide slot and each view's R used.
static int sampler_cap_n(int max_budget) { return (max_budget + (int)GCCB_HOPCAP + 1 + 3) & ~3; }
static bool sampler_wide(int max_budget) { return max_budget > GCCB_WALK_BUDGET_MAX; }
static int wide_region(int batch, int edge_cap) {
  const long long r = (long long)edge_cap + batch;
  return (int)(r < 0x7fffffffll ? r : 0x7fffffffll);
}
static int wide_ctas(int batch) { return 2 * batch < GCCB_WIDE_CTAS ? 2 * batch : GCCB_WIDE_CTAS; }
static size_t wide_keys_len(int max_budget) {
  size_t p = 1;
  while (p < (size_t)max_budget + GCCB_HOPCAP) p <<= 1;
  return p;
}

extern "C" size_t gccb_sample_batch_workspace(int32_t batch, int32_t max_budget, int32_t edge_cap) {
  const bool wide = sampler_wide(max_budget);
  const int cap_n = sampler_cap_n(wide ? GCCB_WALK_BUDGET_MAX : max_budget);
  size_t ints = (size_t)3 * (size_t)(2 * batch) * (size_t)cap_n + 16 + (size_t)2 * (size_t)edge_cap;
  if (wide)
    ints += (size_t)6 * (size_t)wide_region(batch, edge_cap) + (size_t)wide_ctas(batch) * wide_keys_len(max_budget);
  return ints * sizeof(int32_t);
}

// gccb_sample_batch (kModeRwr: seeds_k unused) and gccb_sample_batch_pairs (kModePairs)
template <int kMode>
static int sample_batch_rwr(const char* what, const gccb_graph_t* graph, const int64_t* seeds, const int64_t* seeds_k,
                            const int64_t* sample_ids, const gccb_batch_t* batch, void* workspace,
                            size_t workspace_bytes, gccb_stream_t stream) {
  const int B = batch->batch;
  const bool wide = sampler_wide(graph->max_budget);
  if (wide && wide_keys_len(graph->max_budget) > (size_t)GCCB_WIDE_KEYS_MAX) {
    set_last_error("%s: walk budget %d: a trace of up to %d vertices does not fit int32 positions", what,
                   graph->max_budget, graph->max_budget + (int)GCCB_HOPCAP - 1);
    return GCCB_ERR_CAPACITY;
  }
  const int cap_n = sampler_cap_n(wide ? GCCB_WALK_BUDGET_MAX : graph->max_budget);
  if (workspace_bytes < gccb_sample_batch_workspace(B, graph->max_budget, batch->edge_cap)) {
    set_last_error("%s: workspace too small", what);
    return GCCB_ERR_CAPACITY;
  }
  const int P = wide ? GCCB_WALK_KEYS : pow2_ge(graph->max_budget + (int)GCCB_HOPCAP);
  const size_t smem = (size_t)P * sizeof(int);
  int32_t* subv = (int32_t*)workspace;
  int32_t* subdeg = subv + (size_t)2 * B * cap_n;
  int32_t* rowstart = subdeg + (size_t)2 * B * cap_n;
  unsigned long long* pool_counter = (unsigned long long*)(rowstart + (size_t)2 * B * cap_n);   // 16 ints reserved, 8-byte aligned
  int32_t* pool = (int32_t*)pool_counter + 16;
  // pool positions are stored per row as int32: the pool is capped below 2^31 entries (2 * edge_cap overflows
  // an int for edge_cap > 2^30 -- the 65,536-ego-net sweep of config 5)
  const long long want_cap = 2ll * (long long)batch->edge_cap;
  const int pool_cap = (int)(want_cap < 0x7fff0000ll ? want_cap : 0x7fff0000ll);
  cudaMemsetAsync(pool_counter, 0, wide ? 16 * sizeof(int32_t) : sizeof(unsigned long long), (cudaStream_t)stream);
  auto k1 = rwr_walk_unique_kernel<kMode>;
  auto k3 = induce_fill_kernel;
  if (smem > 48 * 1024) {
    gccb::ensure_dyn_smem(k1, smem);
    gccb::ensure_dyn_smem(k3, smem);
  }
  GCCB_LAUNCH(k1, 2 * B, GCCB_ST, smem, stream, graph->indptr, graph->indices, graph->n_nodes, graph->budget_table,
              graph->budget_table_len, graph->restart_thresh, graph->key, seeds, sample_ids, B,
              cap_n, subv, subdeg, rowstart, pool, pool_cap, pool_counter, batch->counters, batch->flags,
              seeds_k, 0, 0, 0);
  WideWs ww = {};
  if (wide) {
    ww.region = wide_region(B, batch->edge_cap);
    ww.subv = pool + (size_t)2 * batch->edge_cap;
    ww.subdeg = ww.subv + (size_t)2 * ww.region;
    ww.rowstart = ww.subdeg + (size_t)2 * ww.region;
    ww.used = pool_counter + 2;
    ww.next = (unsigned*)(pool_counter + 1);
    int32_t* wide_keys = ww.rowstart + (size_t)2 * ww.region;
    GCCB_LAUNCH(rwr_walk_wide_kernel<kMode>, wide_ctas(B), GCCB_ST, 0, stream, graph->indptr, graph->indices,
                graph->n_nodes, graph->budget_table, graph->budget_table_len, graph->restart_thresh, graph->key,
                seeds, sample_ids, B, cap_n, subv, pool, pool_cap, pool_counter, batch->counters, batch->flags,
                seeds_k, ww, wide_keys, wide_keys_len(graph->max_budget));
  }
  GCCB_LAUNCH(batch_offsets_kernel, 2, 256, 0, stream, batch->counters, B, batch->node_cap,
              batch->edge_cap, batch->node_off, batch->edge_off, batch->flags);
  GCCB_LAUNCH(k3, 2 * B, GCCB_ST, smem, stream, graph->indptr, graph->indices, batch->counters, B,
              cap_n, batch->node_cap, batch->edge_cap, subv, subdeg, rowstart, pool, batch->node_off,
              batch->edge_off, batch->indptr, batch->indices, batch->sub_deg, batch->graph_id,
              batch->orig_id);
  if (wide)
    GCCB_LAUNCH(induce_fill_wide_kernel, 2 * B, GCCB_ST, 0, stream, graph->indptr, graph->indices, batch->counters,
                B, cap_n, batch->node_cap, batch->edge_cap, subv, ww, pool, batch->node_off, batch->edge_off,
                batch->indptr, batch->indices, batch->sub_deg, batch->graph_id, batch->orig_id);
  return check_launch(what);
}

extern "C" int gccb_sample_batch(const gccb_graph_t* graph, const int64_t* seeds,
                                 const int64_t* sample_ids, const gccb_batch_t* batch,
                                 void* workspace, size_t workspace_bytes, gccb_stream_t stream) {
  if (!graph || !batch || !seeds || !sample_ids || !workspace || batch->batch <= 0 ||
      graph->max_budget <= 0 || !graph->indptr || !graph->indices || !graph->budget_table) {
    set_last_error("gccb_sample_batch: bad argument");
    return GCCB_ERR_BADARG;
  }
  return sample_batch_rwr<kModeRwr>("gccb_sample_batch", graph, seeds, (const int64_t*)nullptr, sample_ids, batch,
                                    workspace, workspace_bytes, stream);
}

// ---- the reference's other views: k-hop key seeds (step_dist) and neighbour sampling (aug="ns") ----------------

extern "C" int gccb_pair_seeds(const gccb_graph_t* graph, const double* step_cdf, int32_t n_steps,
                               const int64_t* seeds_q, const int64_t* sample_ids, int32_t count, int64_t* seeds_k,
                               gccb_stream_t stream) {
  if (!graph || !graph->indptr || !graph->indices || graph->n_nodes <= 0 || !step_cdf || n_steps < 1 ||
      n_steps > 3 || !seeds_q || !sample_ids || !seeds_k || count < 0) {
    set_last_error("gccb_pair_seeds: bad argument");
    return GCCB_ERR_BADARG;
  }
  if (count == 0) return GCCB_OK;
  GCCB_LAUNCH(pair_seeds_kernel, (count + 127) / 128, 128, 0, stream, graph->indptr, graph->indices, graph->n_nodes,
              graph->key, step_cdf[0], n_steps > 1 ? step_cdf[1] : 1.0, (int)n_steps, seeds_q, sample_ids, (int)count,
              seeds_k);
  return check_launch("pair_seeds_kernel");
}

extern "C" int gccb_sample_batch_pairs(const gccb_graph_t* graph, const int64_t* seeds_q, const int64_t* seeds_k,
                                       const int64_t* sample_ids, const gccb_batch_t* batch, void* workspace,
                                       size_t workspace_bytes, gccb_stream_t stream) {
  if (!graph || !batch || !seeds_q || !seeds_k || !sample_ids || !workspace || batch->batch <= 0 ||
      graph->max_budget <= 0 || !graph->indptr || !graph->indices || !graph->budget_table) {
    set_last_error("gccb_sample_batch_pairs: bad argument");
    return GCCB_ERR_BADARG;
  }
  return sample_batch_rwr<kModePairs>("gccb_sample_batch_pairs", graph, seeds_q, seeds_k, sample_ids, batch,
                                      workspace, workspace_bytes, stream);
}

// shared memory of an ns ego-net of cap vertices: V[cap] | F[cap] | S[pow2 >= max(k, 2) * cap]
static size_t ns_smem(int cap, int k) { return (size_t)4 * (2 * (size_t)cap + (size_t)pow2_ge((k < 2 ? 2 : k) * cap)); }
#define GCCB_NS_SMEM (192 * 1024)
// An ego-net over its cap is counted node_cap + 1 vertices, so that batch_offsets_kernel publishes its view empty.
// That kernel sums the counts of 256 samples in an int block scan: 256 * (node_cap + 1) must stay below 2^31.
#define GCCB_NS_NODE_CAP_MAX (0x7fffffff / 256 - 1)

extern "C" int32_t gccb_ns_ego_cap(int32_t num_neighbors) {
  if (num_neighbors < 1 || num_neighbors > 0xffff) return 0;
  for (int cap = 65536; cap >= 64; cap >>= 1)
    if ((long long)num_neighbors * cap <= (1 << 24) && ns_smem(cap, num_neighbors) <= GCCB_NS_SMEM) return cap;
  return 0;
}

extern "C" size_t gccb_ns_batch_workspace(int32_t batch, int32_t num_neighbors, int32_t edge_cap) {
  const int cap = gccb_ns_ego_cap(num_neighbors);
  return ((size_t)3 * (size_t)(2 * batch) * (size_t)cap + 16 + (size_t)2 * (size_t)edge_cap) * sizeof(int32_t);
}

extern "C" int gccb_ns_batch(const gccb_graph_t* graph, const int64_t* seeds_q, const int64_t* seeds_k,
                             const int64_t* sample_ids, int32_t num_hops, int32_t num_neighbors,
                             const gccb_batch_t* batch, void* workspace, size_t workspace_bytes,
                             gccb_stream_t stream) {
  const int cap = gccb_ns_ego_cap(num_neighbors);
  if (!graph || !batch || !seeds_q || !seeds_k || !sample_ids || !workspace || batch->batch <= 0 ||
      !graph->indptr || !graph->indices || graph->n_nodes <= 0 || num_hops < 0 || num_hops > 0xffff || cap == 0) {
    set_last_error("gccb_ns_batch: bad argument (num_hops 0..65535, num_neighbors 1..%d)", 0xffff);
    return GCCB_ERR_BADARG;
  }
  if (batch->node_cap > GCCB_NS_NODE_CAP_MAX) {
    set_last_error("gccb_ns_batch: node_cap %d above %d", batch->node_cap, GCCB_NS_NODE_CAP_MAX);
    return GCCB_ERR_CAPACITY;
  }
  const int B = batch->batch;
  if (workspace_bytes < gccb_ns_batch_workspace(B, num_neighbors, batch->edge_cap)) {
    set_last_error("gccb_ns_batch: workspace too small");
    return GCCB_ERR_CAPACITY;
  }
  const size_t smem1 = ns_smem(cap, num_neighbors), smem3 = (size_t)cap * sizeof(int);
  int32_t* subv = (int32_t*)workspace;
  int32_t* subdeg = subv + (size_t)2 * B * cap;
  int32_t* rowstart = subdeg + (size_t)2 * B * cap;
  unsigned long long* pool_counter = (unsigned long long*)(rowstart + (size_t)2 * B * cap);
  int32_t* pool = (int32_t*)pool_counter + 16;
  const long long want_cap = 2ll * (long long)batch->edge_cap;
  const int pool_cap = (int)(want_cap < 0x7fff0000ll ? want_cap : 0x7fff0000ll);
  cudaMemsetAsync(pool_counter, 0, sizeof(unsigned long long), (cudaStream_t)stream);
  auto k1 = rwr_walk_unique_kernel<kModeNs>;
  auto k3 = induce_fill_kernel;
  if (smem1 > 48 * 1024) gccb::ensure_dyn_smem(k1, smem1);
  if (smem3 > 48 * 1024) gccb::ensure_dyn_smem(k3, smem3);
  GCCB_LAUNCH(k1, 2 * B, GCCB_ST, smem1, stream, graph->indptr, graph->indices, graph->n_nodes,
              (const int32_t*)nullptr, 0, 0u, graph->key, seeds_q, sample_ids, B, cap, subv, subdeg, rowstart, pool,
              pool_cap, pool_counter, batch->counters, batch->flags, seeds_k, (int)num_hops, (int)num_neighbors,
              batch->node_cap);
  GCCB_LAUNCH(batch_offsets_kernel, 2, 256, 0, stream, batch->counters, B, batch->node_cap,
              batch->edge_cap, batch->node_off, batch->edge_off, batch->flags);
  GCCB_LAUNCH(k3, 2 * B, GCCB_ST, smem3, stream, graph->indptr, graph->indices, batch->counters, B,
              cap, batch->node_cap, batch->edge_cap, subv, subdeg, rowstart, pool, batch->node_off,
              batch->edge_off, batch->indptr, batch->indices, batch->sub_deg, batch->graph_id,
              batch->orig_id);
  return check_launch("gccb_ns_batch");
}

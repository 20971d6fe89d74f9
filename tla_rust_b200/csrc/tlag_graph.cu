// tlag_graph.cu -- liveness building blocks on sm_90a (H100): SCC decomposition of a masked state graph and the
// Emerson-Lei fair-cycle search over it (include/tlag.h: tlag_scc, tlag_fair_cycles).
//
// The graph is uploaded once as an edge list; edges outside the masks and self-loops are compacted away, and a
// forward and a reverse CSR are built with CUB radix sorts.  A vertex's component id lives in scc[v]: kActive while
// unassigned, kOut when outside the (current) mask, else the index of one state of its SCC.  The decomposition is
// the usual GPU recipe (trim / forward-backward / colouring, Hong et al. SC'13, Slota et al. IPDPS'14):
//   1. trim: a vertex with no active in- or out-neighbour is an SCC of its own;
//   2. forward-backward from the vertex of largest degree product takes the giant component in one piece;
//   3. colouring, round by round: the largest hashed priority is pushed along forward edges, each vertex whose own
//      priority survived is a root, and the vertices of the root's colour it reaches backwards are its SCC.
// Every reachability step is the same "push a larger value to the neighbours whose group matches" kernel, run to a
// fixpoint with changed-vertex flags so a pass only touches the vertices whose value moved in the pass before.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <string>
#include <utility>
#include <vector>
#include <cub/device/device_radix_sort.cuh>

#include "../../include/tlag.h"

namespace {

constexpr uint32_t kActive = 0xFFFFFFFEu;   // in the graph, no component yet
constexpr uint32_t kOut = 0xFFFFFFFFu;      // outside the (current) state mask
constexpr int kBlock = 256;
constexpr int kTrimPasses = 16;             // trim passes per round before the (always correct) colouring takes over

thread_local std::string g_err;

#define GK(call)                                                                         \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess) {                                                             \
      g_err = std::string(#call) + ": " + cudaGetErrorString(_e);                        \
      if (_e != cudaErrorMemoryAllocation) return TLAG_ECUDA;                            \
      cudaGetLastError();                                                                \
      g_err += " (the graph does not fit in device memory)";                             \
      return TLAG_ENOMEM;                                                                \
    }                                                                                    \
  } while (0)
#define GR(call)                                                                         \
  do {                                                                                   \
    int _r = (call);                                                                     \
    if (_r != TLAG_OK) return _r;                                                        \
  } while (0)

typedef unsigned long long u64;

// colour of a vertex: a hashed priority above its index, so that colours are distinct and roots are not all at one
// end of a numbered chain
__device__ __forceinline__ u64 prio(uint32_t v) {
  uint32_t h = v * 0x9E3779B1u;
  h ^= h >> 15; h *= 0x85EBCA77u; h ^= h >> 13;
  return (u64)h << 32 | v;
}

#define GRID_STRIDE(i, n) for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < (n); \
                               i += (uint64_t)gridDim.x * blockDim.x)

// keep edge i iff it is in both masks and not a self-loop; warp-aggregated append into count[0].  An endpoint >= n
// is never kept and sets count[1]: the call fails with TLAG_EINVAL.
__global__ void k_keep_edges(uint32_t n, uint64_t m, const uint32_t* src, const uint32_t* dst, const uint32_t* lab,
                             const uint8_t* emask, const uint8_t* vmask, uint32_t* osrc, uint32_t* odst,
                             uint32_t* olab, unsigned int* count) {
  GRID_STRIDE(i, m) {
    uint32_t s = src[i], d = dst[i];
    bool in_range = s < n && d < n;
    if (!in_range) atomicOr(&count[1], 1u);
    bool keep = in_range && s != d && (!emask || emask[i]) && vmask[s] && vmask[d];
    unsigned act = __activemask();
    unsigned bal = __ballot_sync(act, keep);
    int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
    unsigned base = 0;
    if (lane == leader && bal) base = atomicAdd(count, (unsigned)__popc(bal));
    base = __shfl_sync(act, base, leader);
    if (keep) {
      unsigned at = base + __popc(bal & ((1u << lane) - 1));
      osrc[at] = s; odst[at] = d; olab[at] = lab ? lab[i] : 0u;
    }
  }
}

// off[v] = first position of key v in the sorted key array (off[n] = m)
__global__ void k_offsets(uint32_t n, uint32_t m, const uint32_t* keys, uint32_t* off) {
  GRID_STRIDE(v, (uint64_t)n + 1) {
    uint32_t lo = 0, hi = m;
    while (lo < hi) {
      uint32_t mid = (lo + hi) >> 1;
      if (keys[mid] < (uint32_t)v) lo = mid + 1; else hi = mid;
    }
    off[v] = lo;
  }
}

__global__ void k_init_scc(uint32_t n, const uint8_t* alive, uint32_t* scc) {
  GRID_STRIDE(v, n) scc[v] = alive[v] ? kActive : kOut;
}

__device__ __forceinline__ bool has_active(const uint32_t* off, const uint32_t* adj, const uint32_t* scc, uint32_t v) {
  for (uint32_t j = off[v], e = off[v + 1]; j < e; ++j)
    if (scc[adj[j]] == kActive) return true;
  return false;
}

// Trim v, which has no active neighbour along (off, adj), then keep walking: the first neighbour along the other
// direction (woff, wadj) that is left without an active neighbour along (off, adj) is trimmed next.  One thread so
// takes a whole chain in one pass instead of one vertex per pass.  Claims are CASes, so two walks never trim one
// vertex twice; stale reads only end a walk early, they never trim a vertex that still has an active neighbour.
__device__ void trim_walk(uint32_t v, const uint32_t* off, const uint32_t* adj, const uint32_t* woff, const uint32_t* wadj,
                          uint32_t* scc, unsigned int* changed) {
  for (;;) {
    if (atomicCAS(&scc[v], kActive, v) != kActive) return;
    *changed = 1;
    uint32_t next = kOut;
    for (uint32_t j = woff[v], e = woff[v + 1]; j < e && next == kOut; ++j) {
      uint32_t w = wadj[j];
      if (scc[w] == kActive && !has_active(off, adj, scc, w)) next = w;
    }
    if (next == kOut) return;
    v = next;
  }
}

// a vertex without an active in- or out-neighbour is its own SCC
__global__ void k_trim(uint32_t n, const uint32_t* foff, const uint32_t* fadj, const uint32_t* roff, const uint32_t* radj,
                       uint32_t* scc, unsigned int* changed) {
  GRID_STRIDE(v, n) {
    if (scc[v] != kActive) continue;
    if (!has_active(roff, radj, scc, (uint32_t)v)) trim_walk((uint32_t)v, roff, radj, foff, fadj, scc, changed);
    else if (!has_active(foff, fadj, scc, (uint32_t)v)) trim_walk((uint32_t)v, foff, fadj, roff, radj, scc, changed);
  }
}

// pivot of forward-backward: the active vertex of largest (out-degree x in-degree), ties to the larger index; the
// packed key is 1 + product above the index, so *best stays 0 only when no vertex is active
__global__ void k_pivot(uint32_t n, const uint32_t* foff, const uint32_t* roff, const uint32_t* scc, u64* best) {
  GRID_STRIDE(v, n) {
    if (scc[v] != kActive) continue;
    u64 d = (u64)(foff[v + 1] - foff[v]) * (roff[v + 1] - roff[v]);
    atomicMax(best, ((d < 0x7FFFFFFFull ? d : 0x7FFFFFFFull) + 1) << 32 | v);
  }
}

// val[v] = seed ? 1 : 0 (or the colour prio(v) when colour != 0) for active vertices; cur[v] = the vertex pushes first
__global__ void k_seed(uint32_t n, const uint32_t* scc, u64* val, uint8_t* cur, uint32_t pivot, int colour) {
  GRID_STRIDE(v, n) {
    bool a = scc[v] == kActive;
    u64 x = !a ? 0 : (colour ? prio((uint32_t)v) : (u64)((uint32_t)v == pivot));
    val[v] = x;
    cur[v] = a && x != 0;
  }
}

// roots of a colouring round: active vertices whose own colour survived; they seed the backward search
__global__ void k_roots(uint32_t n, const uint32_t* scc, const u64* colour, u64* bw, uint8_t* cur) {
  GRID_STRIDE(v, n) {
    bool r = scc[v] == kActive && colour[v] == prio((uint32_t)v);
    bw[v] = r;
    cur[v] = r;
  }
}

// one pass of max-propagation: every flagged vertex offers its value to the neighbours that are eligible (active when
// scc is given, same group value when grp is given) and flags those it raised
__global__ void k_push(uint32_t n, const uint32_t* off, const uint32_t* adj, u64* val, const uint32_t* scc,
                       const u64* grp, const uint8_t* cur, uint8_t* nxt, unsigned int* changed) {
  GRID_STRIDE(v, n) {
    if (!cur[v]) continue;
    u64 x = val[v];
    u64 g = grp ? grp[v] : 0;
    for (uint32_t j = off[v], e = off[v + 1]; j < e; ++j) {
      uint32_t w = adj[j];
      if (scc && scc[w] != kActive) continue;
      if (grp && grp[w] != g) continue;
      if (val[w] >= x) continue;
      if (atomicMax(&val[w], x) < x) {
        nxt[w] = 1;
        *changed = 1;
      }
    }
  }
}

// component assignment: forward-backward (both searches reached v) or colouring (v reached backwards from its root)
__global__ void k_assign(uint32_t n, uint32_t* scc, const u64* a, const u64* b, uint32_t pivot, int colour,
                         unsigned int* left) {
  GRID_STRIDE(v, n) {
    if (scc[v] != kActive) continue;
    if (colour ? b[v] != 0 : (a[v] != 0 && b[v] != 0)) scc[v] = colour ? (uint32_t)a[v] : pivot;
    else atomicAdd(left, 1u);
  }
}

// ---- fair-cycle search: per-SCC aggregates indexed by the SCC id
__global__ void k_state_agg(uint32_t n, const uint32_t* scc, const uint32_t* lab, uint32_t* s_or, uint32_t* s_and) {
  GRID_STRIDE(v, n) {
    uint32_t c = scc[v];
    if (c >= kActive) continue;
    uint32_t x = lab ? lab[v] : 0u;
    if (x) atomicOr(&s_or[c], x);
    if (~x) atomicAnd(&s_and[c], x);
  }
}

__global__ void k_edge_agg(uint32_t m, const uint32_t* src, const uint32_t* dst, const uint32_t* lab, const uint32_t* scc,
                           uint32_t* e_or) {
  GRID_STRIDE(i, m) {
    uint32_t x = lab[i];
    if (!x) continue;
    uint32_t c = scc[src[i]];
    if (c < kActive && c == scc[dst[i]]) atomicOr(&e_or[c], x);
  }
}

struct FairSet {
  uint32_t n_wf, n_sf;
  uint32_t en[64], act[64];      // per condition: enabled bit mask, action bit mask; WF first, then SF
  uint32_t need_clear;
};

// judge v's SCC: v leaves the graph when the SCC fails a WF or need_clear test, or when it is an EN state of a
// failed SF condition (then the SCC must be decomposed again: *resplit)
__global__ void k_judge(uint32_t n, const uint32_t* scc, const uint32_t* lab, const uint32_t* s_or, const uint32_t* s_and,
                        const uint32_t* e_or, FairSet fs, uint8_t* alive, unsigned int* resplit) {
  GRID_STRIDE(v, n) {
    uint32_t c = scc[v];
    if (c >= kActive) continue;
    uint32_t so = s_or[c], sa = s_and[c], eo = e_or[c], x = lab ? lab[v] : 0u;
    bool drop = (sa & fs.need_clear) != 0, sf_drop = false;
    for (uint32_t k = 0; k < fs.n_wf && !drop; ++k)
      drop = (sa & fs.en[k]) && !(eo & fs.act[k]);
    for (uint32_t k = fs.n_wf; k < fs.n_wf + fs.n_sf && !drop; ++k)
      if ((so & fs.en[k]) && !(eo & fs.act[k]) && (x & fs.en[k])) sf_drop = true;
    if (drop || sf_drop) alive[v] = 0;
    if (!drop && sf_drop) *resplit = 1;
  }
}

__global__ void k_result(uint32_t n, const uint32_t* scc, const uint8_t* alive, const u64* reach, uint32_t* out,
                         unsigned int* witness, unsigned int* n_fair) {
  GRID_STRIDE(v, n) {
    uint32_t c = alive[v] ? scc[v] : kOut;
    out[v] = c;
    if (c == kOut) continue;
    if (c == (uint32_t)v) atomicAdd(n_fair, 1u);
    if (!reach || reach[v]) atomicMin(witness, (unsigned)v);
  }
}

// reach[v] = v is a seed inside the state mask; it pushes first
__global__ void k_reach_seed(uint32_t n, const uint8_t* seeds, const uint8_t* vmask, u64* reach, uint8_t* cur) {
  GRID_STRIDE(v, n) {
    bool r = seeds[v] && vmask[v];
    reach[v] = r;
    cur[v] = r;
  }
}

__global__ void k_count_roots(uint32_t n, const uint32_t* scc, unsigned int* cnt) {
  GRID_STRIDE(v, n) if (scc[v] == (uint32_t)v) atomicAdd(cnt, 1u);
}

// ---- the engine's labelled graph (tlag_live_check)
// the source row of every CSR edge
__global__ void k_csr_src(uint32_t n, const u64* off, uint32_t* src) {
  GRID_STRIDE(v, n) for (u64 j = off[v], e = off[v + 1]; j < e; ++j) src[j] = (uint32_t)v;
}

// the restriction and the seeds from the label words
__global__ void k_live_masks(uint32_t n, const uint32_t* slab, uint32_t keep_set, uint32_t keep_clear, uint32_t seed_set,
                             uint32_t seed_clear, uint64_t seed_rows, uint8_t* vmask, uint8_t* seeds) {
  GRID_STRIDE(v, n) {
    const uint32_t x = slab[v];
    vmask[v] = (x & keep_set) == keep_set && !(x & keep_clear);
    seeds[v] = v < seed_rows && (x & seed_set) == seed_set && !(x & seed_clear);
  }
}

__global__ void k_edge_drop(uint64_t m, const uint32_t* elab, uint32_t drop, uint8_t* em) {
  GRID_STRIDE(i, m) em[i] = !(elab[i] & drop);
}

__global__ void k_first_seed(uint32_t n, const uint8_t* seeds, unsigned int* first) {
  GRID_STRIDE(v, n) if (seeds[v]) atomicMin(first, (unsigned)v);
}

// ---- lasso: breadth-first search with parent pointers inside `allowed`, from the vertices with par[v] == v
__global__ void k_bfs_init(uint32_t n, const uint8_t* src, uint32_t one, uint32_t* par, uint8_t* cur) {
  GRID_STRIDE(v, n) {
    const bool s = src ? src[v] != 0 : (uint32_t)v == one;
    par[v] = s ? (uint32_t)v : kOut;
    cur[v] = s;
  }
}

__global__ void k_bfs_step(uint32_t n, const uint32_t* off, const uint32_t* adj, const uint8_t* allowed, uint32_t* par,
                           const uint8_t* cur, uint8_t* nxt, const uint8_t* target, unsigned int* flag) {
  GRID_STRIDE(v, n) {
    if (!cur[v]) continue;
    for (uint32_t j = off[v], e = off[v + 1]; j < e; ++j) {
      const uint32_t w = adj[j];
      if (!allowed[w] || par[w] != kOut) continue;
      if (atomicCAS(&par[w], kOut, (uint32_t)v) == kOut) {
        nxt[w] = 1;
        flag[0] = 1;
        if (target[w]) atomicMin(&flag[1], w);
      }
    }
  }
}

__global__ void k_bfs_hit(uint32_t n, const uint8_t* cur, const uint8_t* target, unsigned int* flag) {
  GRID_STRIDE(v, n) if (cur[v] && target[v]) atomicMin(&flag[1], (unsigned)v);
}

// targets inside SCC c: the states with a `clear` bit clear (clear != 0), or the sources of the SCC's edges with an
// `act` bit, next[source] = the edge's destination
__global__ void k_scc_targets(uint32_t n, uint32_t m, const uint32_t* res, uint32_t c, const uint32_t* word, uint32_t clear,
                              const uint32_t* src, const uint32_t* dst, const uint32_t* lab, uint32_t act, uint8_t* target,
                              uint32_t* next) {
  GRID_STRIDE(i, (uint64_t)n > m ? n : m) {
    if (clear && i < n) target[i] = res[i] == c && (~word[i] & clear) != 0;
    if (act && i < m && res[src[i]] == c && res[dst[i]] == c && (lab[i] & act)) {
      target[src[i]] = 1;
      next[src[i]] = dst[i];
    }
  }
}

// the path from v back along par[] to its root (par[root] == root), v first: out[0, min(len, cap)), *len
__global__ void k_walk_parents(const uint32_t* par, uint32_t v, uint32_t cap, uint32_t* out, unsigned int* len) {
  uint32_t k = 0;
  for (;;) {
    if (k < cap) out[k] = v;
    ++k;
    const uint32_t p = par[v];
    if (p == v || k > cap) break;
    v = p;
  }
  *len = k;
}

__global__ void k_in_scc(uint32_t n, const uint32_t* res, uint32_t c, uint8_t* in) {
  GRID_STRIDE(v, n) in[v] = res[v] == c;
}

template <class T>
struct DevBuf {
  T* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(uint64_t n) { return cudaMalloc((void**)&p, (n ? n : 1) * sizeof(T)); }
};

// the calling thread's current device, restored when the call returns (declared before the Graph, so the Graph's
// buffers are freed on the graph's device first)
struct DeviceGuard {
  int prev = -1;
  DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// the uploaded, compacted graph with both CSRs and the decomposition's scratch
struct Graph {
  uint32_t n = 0, m = 0;
  cudaStream_t st = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int grid = 0;
  DevBuf<uint32_t> src, dst, lab, foff, fadj, roff, radj, scc, word;
  DevBuf<uint8_t> vmask, alive, cur, nxt;   // vmask: the caller's state mask; alive: what the fair-cycle search keeps
  DevBuf<u64> a, b;
  DevBuf<unsigned int> flag;
  DevBuf<unsigned char> tmp;
  unsigned int* h_flag = nullptr;
  ~Graph() {
    if (h_flag) cudaFreeHost(h_flag);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (st) cudaStreamDestroy(st);
  }

  int grid_for(uint64_t k) const {
    uint64_t b = (k + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > (uint64_t)grid ? grid : b));
  }

  int read_flag(unsigned int* out) {
    GK(cudaMemcpyAsync(h_flag, flag.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    GK(cudaStreamSynchronize(st));
    *out = *h_flag;
    return TLAG_OK;
  }
  int clear_flag() {
    GK(cudaMemsetAsync(flag.p, 0, sizeof(unsigned int), st));
    return TLAG_OK;
  }

  // the stream, events and flags on the graph's device, for n_states states and n_edges edges
  int init(uint64_t n_states, uint64_t n_edges, int device, const char* what) {
    if (n_states >= kActive || n_edges >= 0xFFFFFFFFull) {
      g_err = std::string(what) + ": n_states >= 2^32 - 2 or n_edges >= 2^32 - 1";
      return TLAG_EINVAL;
    }
    n = (uint32_t)n_states;
    GK(cudaSetDevice(device));
    int sms = 0;
    GK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    grid = sms * 8;
    GK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    GK(cudaEventCreate(&ev0));
    GK(cudaEventCreate(&ev1));
    GK(cudaMallocHost((void**)&h_flag, 2 * sizeof(unsigned int)));
    GK(flag.alloc(2));
    GK(vmask.alloc(n)); GK(alive.alloc(n)); GK(word.alloc(n));
    return TLAG_OK;
  }

  // a host edge list: copied to the device, then build()
  int upload(const tlag_graph* g) {
    if (!g || !g->src || !g->dst) {
      g_err = "tlag_graph: missing edge arrays";
      return TLAG_EINVAL;
    }
    GR(init(g->n_states, g->n_edges, g->device, "tlag_graph"));
    uint64_t m0 = g->n_edges;
    DevBuf<uint32_t> rs, rd, rl;
    DevBuf<uint8_t> em;
    GK(rs.alloc(m0)); GK(rd.alloc(m0));
    GK(cudaMemcpyAsync(rs.p, g->src, m0 * 4, cudaMemcpyHostToDevice, st));
    GK(cudaMemcpyAsync(rd.p, g->dst, m0 * 4, cudaMemcpyHostToDevice, st));
    if (g->edge_label) {
      GK(rl.alloc(m0));
      GK(cudaMemcpyAsync(rl.p, g->edge_label, m0 * 4, cudaMemcpyHostToDevice, st));
    }
    if (g->edge_mask) {
      GK(em.alloc(m0));
      GK(cudaMemcpyAsync(em.p, g->edge_mask, m0, cudaMemcpyHostToDevice, st));
    }
    if (g->state_mask) GK(cudaMemcpyAsync(vmask.p, g->state_mask, n, cudaMemcpyHostToDevice, st));
    else GK(cudaMemsetAsync(vmask.p, 1, n, st));
    if (g->state_label) GK(cudaMemcpyAsync(word.p, g->state_label, (uint64_t)n * 4, cudaMemcpyHostToDevice, st));
    else GK(cudaMemsetAsync(word.p, 0, (uint64_t)n * 4, st));
    GK(cudaEventRecord(ev0, st));
    return build(rs, rd, rl.p, em.p, m0);
  }

  // device compaction and both CSRs: the edges (rs, rd; labels rl, mask em may be null) of m0 edges, vmask and word set;
  // rs and rd are the sorts' scratch afterwards
  int build(DevBuf<uint32_t>& rs, DevBuf<uint32_t>& rd, const uint32_t* rl, const uint8_t* em, uint64_t m0) {
    GK(cudaMemcpyAsync(alive.p, vmask.p, n, cudaMemcpyDeviceToDevice, st));
    GK(src.alloc(m0)); GK(dst.alloc(m0)); GK(lab.alloc(m0));
    GK(cudaMemsetAsync(flag.p, 0, 2 * sizeof(unsigned int), st));
    if (m0)
      k_keep_edges<<<grid_for(m0), kBlock, 0, st>>>(n, m0, rs.p, rd.p, rl, em, vmask.p, src.p, dst.p, lab.p, flag.p);
    GK(cudaGetLastError());
    GK(cudaMemcpyAsync(h_flag, flag.p, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    GK(cudaStreamSynchronize(st));
    if (h_flag[1]) {
      g_err = "tlag_graph: an edge endpoint is >= n_states";
      return TLAG_EINVAL;
    }
    m = h_flag[0];
    // forward CSR: sort (src, dst) by src; reverse CSR: sort (dst, src) by dst
    GK(foff.alloc((uint64_t)n + 1)); GK(fadj.alloc(m)); GK(roff.alloc((uint64_t)n + 1)); GK(radj.alloc(m));
    GK(scc.alloc(n)); GK(cur.alloc(n)); GK(nxt.alloc(n)); GK(a.alloc(n)); GK(b.alloc(n));
    int end_bit = 1;
    while (end_bit < 32 && (1ull << end_bit) < (uint64_t)n) ++end_bit;
    DevBuf<uint32_t> k2, v2;
    GK(k2.alloc(m)); GK(v2.alloc(m));
    size_t tb = 0;
    {
      cub::DoubleBuffer<uint32_t> kk(rs.p, k2.p), vv(rd.p, v2.p);
      GK(cub::DeviceRadixSort::SortPairs(nullptr, tb, kk, vv, m, 0, end_bit, st));
    }
    GK(tmp.alloc(tb));
    for (int dir = 0; dir < 2; ++dir) {
      GK(cudaMemcpyAsync(rs.p, dir ? dst.p : src.p, (uint64_t)m * 4, cudaMemcpyDeviceToDevice, st));
      GK(cudaMemcpyAsync(rd.p, dir ? src.p : dst.p, (uint64_t)m * 4, cudaMemcpyDeviceToDevice, st));
      cub::DoubleBuffer<uint32_t> kk(rs.p, k2.p), vv(rd.p, v2.p);
      size_t t = tb;
      if (m) GK(cub::DeviceRadixSort::SortPairs(tmp.p, t, kk, vv, m, 0, end_bit, st));
      uint32_t* off = dir ? roff.p : foff.p;
      GK(cudaMemcpyAsync(dir ? radj.p : fadj.p, vv.Current(), (uint64_t)m * 4, cudaMemcpyDeviceToDevice, st));
      k_offsets<<<grid_for((uint64_t)n + 1), kBlock, 0, st>>>(n, m, kk.Current(), off);
      GK(cudaGetLastError());
    }
    return TLAG_OK;
  }

  // push values to a fixpoint along one CSR (cur holds the first pass's flags)
  int propagate(const uint32_t* off, const uint32_t* adj, u64* val, const uint32_t* gate, const u64* grp) {
    uint8_t *c = cur.p, *x = nxt.p;
    for (;;) {
      GK(cudaMemsetAsync(x, 0, n, st));
      GR(clear_flag());
      k_push<<<grid_for(n), kBlock, 0, st>>>(n, off, adj, val, gate, grp, c, x, flag.p);
      GK(cudaGetLastError());
      unsigned int ch = 0;
      GR(read_flag(&ch));
      std::swap(c, x);
      if (!ch) break;
    }
    return TLAG_OK;
  }

  int trim() {
    for (int pass = 0; pass < kTrimPasses; ++pass) {
      GR(clear_flag());
      k_trim<<<grid_for(n), kBlock, 0, st>>>(n, foff.p, fadj.p, roff.p, radj.p, scc.p, flag.p);
      GK(cudaGetLastError());
      unsigned int ch = 0;
      GR(read_flag(&ch));
      if (!ch) break;
    }
    return TLAG_OK;
  }

  // SCCs of the vertices with alive[v] != 0, into scc[]
  int decompose() {
    if (!n) return TLAG_OK;
    k_init_scc<<<grid_for(n), kBlock, 0, st>>>(n, alive.p, scc.p);
    GK(cudaGetLastError());
    GR(trim());
    // forward-backward from the pivot
    GK(cudaMemsetAsync(a.p, 0, 8, st));
    k_pivot<<<grid_for(n), kBlock, 0, st>>>(n, foff.p, roff.p, scc.p, a.p);
    GK(cudaGetLastError());
    u64 best = 0;
    GK(cudaMemcpyAsync(&best, a.p, 8, cudaMemcpyDeviceToHost, st));
    GK(cudaStreamSynchronize(st));
    unsigned int left = 0;
    if (best) {   // an active vertex with an active in- and out-neighbour exists
      uint32_t pivot = (uint32_t)best;
      k_seed<<<grid_for(n), kBlock, 0, st>>>(n, scc.p, a.p, cur.p, pivot, 0);
      GR(propagate(foff.p, fadj.p, a.p, scc.p, nullptr));
      k_seed<<<grid_for(n), kBlock, 0, st>>>(n, scc.p, b.p, cur.p, pivot, 0);
      GR(propagate(roff.p, radj.p, b.p, scc.p, a.p));   // backwards, within the forward set (a == 1)
      GR(clear_flag());
      k_assign<<<grid_for(n), kBlock, 0, st>>>(n, scc.p, a.p, b.p, pivot, 0, flag.p);
      GK(cudaGetLastError());
      GR(read_flag(&left));
    }
    // colouring rounds over what is left
    while (left) {
      GR(trim());
      k_seed<<<grid_for(n), kBlock, 0, st>>>(n, scc.p, a.p, cur.p, 0, 1);
      GR(propagate(foff.p, fadj.p, a.p, scc.p, nullptr));
      k_roots<<<grid_for(n), kBlock, 0, st>>>(n, scc.p, a.p, b.p, cur.p);
      GR(propagate(roff.p, radj.p, b.p, scc.p, a.p));   // backwards, within the root's colour
      GR(clear_flag());
      k_assign<<<grid_for(n), kBlock, 0, st>>>(n, scc.p, a.p, b.p, 0, 1, flag.p);
      GK(cudaGetLastError());
      GR(read_flag(&left));
    }
    return TLAG_OK;
  }

  int elapsed(float* ms) {
    GK(cudaEventRecord(ev1, st));
    GK(cudaEventSynchronize(ev1));
    GK(cudaEventElapsedTime(ms, ev0, ev1));
    return TLAG_OK;
  }
};


// The Emerson-Lei search of tlag_fair_cycles and tlag_live_check on a built Graph: decompose, drop what fails, decompose
// again while an SF test split an SCC; then the accepted SCCs reachable from the seeds (device flags, or all).
// res[v] = accepted SCC id of v or kOut; s_or / s_and / e_or: the last decomposition's aggregates, exact for accepted SCCs.
struct FairSearch {
  DevBuf<uint32_t> s_or, s_and, e_or, res;
  DevBuf<unsigned int> cnt;     // {witness, accepted SCCs}
  unsigned int h_cnt[2] = {kOut, 0};
  uint32_t rounds = 0;
  const u64* reach = nullptr;   // G.b: reachable from the seeds (null: no seeds)

  int run(Graph& G, const FairSet& fs, const uint8_t* seeds) {
    const uint32_t n = G.n;
    GK(s_or.alloc(n)); GK(s_and.alloc(n)); GK(e_or.alloc(n)); GK(res.alloc(n));
    for (;;) {
      ++rounds;
      GR(G.decompose());
      if (!n) break;
      GK(cudaMemsetAsync(s_or.p, 0, (uint64_t)n * 4, G.st));
      GK(cudaMemsetAsync(s_and.p, 0xFF, (uint64_t)n * 4, G.st));
      GK(cudaMemsetAsync(e_or.p, 0, (uint64_t)n * 4, G.st));
      k_state_agg<<<G.grid_for(n), kBlock, 0, G.st>>>(n, G.scc.p, G.word.p, s_or.p, s_and.p);
      if (G.m) k_edge_agg<<<G.grid_for(G.m), kBlock, 0, G.st>>>(G.m, G.src.p, G.dst.p, G.lab.p, G.scc.p, e_or.p);
      GR(G.clear_flag());
      k_judge<<<G.grid_for(n), kBlock, 0, G.st>>>(n, G.scc.p, G.word.p, s_or.p, s_and.p, e_or.p, fs, G.alive.p, G.flag.p);
      GK(cudaGetLastError());
      unsigned int resplit = 0;
      GR(G.read_flag(&resplit));
      if (!resplit) break;
    }
    // reachability from the seeds over the whole restricted graph (every compacted edge), into b[]
    GK(cnt.alloc(2));
    GK(cudaMemcpyAsync(cnt.p, h_cnt, sizeof h_cnt, cudaMemcpyHostToDevice, G.st));
    if (seeds && n) {
      k_reach_seed<<<G.grid_for(n), kBlock, 0, G.st>>>(n, seeds, G.vmask.p, G.b.p, G.cur.p);
      GK(cudaGetLastError());
      GR(G.propagate(G.foff.p, G.fadj.p, G.b.p, nullptr, nullptr));
      reach = G.b.p;
    }
    if (n) k_result<<<G.grid_for(n), kBlock, 0, G.st>>>(n, G.scc.p, G.alive.p, reach, res.p, cnt.p, cnt.p + 1);
    GK(cudaGetLastError());
    GK(cudaMemcpyAsync(h_cnt, cnt.p, sizeof h_cnt, cudaMemcpyDeviceToHost, G.st));
    GK(cudaStreamSynchronize(G.st));
    return TLAG_OK;
  }
};

}  // namespace

extern "C" const char* tlag_graph_last_error(void) { return g_err.c_str(); }

extern "C" int tlag_scc(const tlag_graph* g, uint32_t* scc_out, uint64_t* n_scc_out, float* device_ms) {
  g_err.clear();
  DeviceGuard dg;
  Graph G;
  GR(G.upload(g));
  GR(G.decompose());
  GR(G.clear_flag());
  if (G.n) k_count_roots<<<G.grid_for(G.n), kBlock, 0, G.st>>>(G.n, G.scc.p, G.flag.p);
  GK(cudaGetLastError());
  float ms = 0;
  GR(G.elapsed(&ms));
  unsigned int roots = 0;
  GR(G.read_flag(&roots));
  if (scc_out && G.n) GK(cudaMemcpy(scc_out, G.scc.p, (uint64_t)G.n * 4, cudaMemcpyDeviceToHost));
  if (n_scc_out) *n_scc_out = roots;
  if (device_ms) *device_ms = ms;
  return TLAG_OK;
}

// the conditions of a query, WF first, then SF
static int fair_set(const tlag_fairness* fair, uint32_t n_fair, uint32_t need_clear, FairSet* fs, const char* what) {
  if ((n_fair && !fair) || n_fair > 64) {
    g_err = std::string(what) + ": missing fairness conditions, or more than 64";
    return TLAG_EINVAL;
  }
  memset(fs, 0, sizeof *fs);
  fs->need_clear = need_clear;
  for (int kind = TLAG_FAIR_WF; kind <= TLAG_FAIR_SF; ++kind)
    for (uint32_t k = 0; k < n_fair; ++k) {
      const tlag_fairness& f = fair[k];
      if (f.kind > TLAG_FAIR_SF || f.enabled_bit > 31 || f.action_bit > 31) {
        g_err = std::string(what) + ": fairness condition " + std::to_string(k) + " has a bad kind or bit";
        return TLAG_EINVAL;
      }
      if ((int)f.kind != kind) continue;
      uint32_t at = fs->n_wf + fs->n_sf;
      fs->en[at] = 1u << f.enabled_bit;
      fs->act[at] = 1u << f.action_bit;
      if (kind == TLAG_FAIR_WF) ++fs->n_wf; else ++fs->n_sf;
    }
  return TLAG_OK;
}

extern "C" int tlag_fair_cycles(const tlag_graph* g, const tlag_fair_query* q, uint32_t* scc_out, tlag_fair_result* out) {
  g_err.clear();
  if (!q || !out) {
    g_err = "tlag_fair_cycles: missing query or result";
    return TLAG_EINVAL;
  }
  FairSet fs;
  GR(fair_set(q->fair, q->n_fair, q->need_clear, &fs, "tlag_fair_cycles"));
  DeviceGuard dg;
  Graph G;
  GR(G.upload(g));
  const uint32_t n = G.n;
  FairSearch F;
  DevBuf<uint8_t> sd;
  if (q->seeds && n) {
    GK(sd.alloc(n));
    GK(cudaMemcpyAsync(sd.p, q->seeds, n, cudaMemcpyHostToDevice, G.st));
  }
  GR(F.run(G, fs, q->seeds ? sd.p : nullptr));
  float ms = 0;
  GR(G.elapsed(&ms));
  if (scc_out && n) GK(cudaMemcpy(scc_out, F.res.p, (uint64_t)n * 4, cudaMemcpyDeviceToHost));
  out->violated = F.h_cnt[0] != kOut;
  out->witness = F.h_cnt[0];
  out->fair_sccs = F.h_cnt[1];
  out->rounds = F.rounds;
  out->device_ms = ms;
  return TLAG_OK;
}

namespace {

// A shortest path inside `allowed` from the sources (flags src, or the vertex one) to a vertex with target[v] != 0, the
// source first and the target last, appended to path; the search and the path are the graph's forward CSR.
int bfs_path(Graph& G, const uint8_t* src, uint32_t one, const uint8_t* allowed, const uint8_t* target, uint32_t* par,
             uint32_t* walk, std::vector<uint32_t>& path) {
  const uint32_t n = G.n;
  k_bfs_init<<<G.grid_for(n), kBlock, 0, G.st>>>(n, src, one, par, G.cur.p);
  const unsigned int init[2] = {0, kOut};
  GK(cudaMemcpyAsync(G.flag.p, init, sizeof init, cudaMemcpyHostToDevice, G.st));
  k_bfs_hit<<<G.grid_for(n), kBlock, 0, G.st>>>(n, G.cur.p, target, G.flag.p);
  GK(cudaGetLastError());
  uint8_t *c = G.cur.p, *x = G.nxt.p;
  for (bool first = true;; first = false) {
    GK(cudaMemcpyAsync(G.h_flag, G.flag.p, 2 * sizeof(unsigned int), cudaMemcpyDeviceToHost, G.st));
    GK(cudaStreamSynchronize(G.st));
    if (G.h_flag[1] != kOut) break;
    if (!first && !G.h_flag[0]) {      // the last step reached no new vertex
      g_err = "tlag_live_check: the lasso search found no path to its target (internal error)";
      return TLAG_EINVAL;
    }
    GK(cudaMemsetAsync(x, 0, n, G.st));
    GK(cudaMemsetAsync(G.flag.p, 0, sizeof(unsigned int), G.st));
    k_bfs_step<<<G.grid_for(n), kBlock, 0, G.st>>>(n, G.foff.p, G.fadj.p, allowed, par, c, x, target, G.flag.p);
    GK(cudaGetLastError());
    std::swap(c, x);
  }
  // the parent chain from the target, walked on the device and read back in one copy
  k_walk_parents<<<1, 1, 0, G.st>>>(par, G.h_flag[1], n, walk, G.flag.p);
  GK(cudaGetLastError());
  GK(cudaMemcpyAsync(G.h_flag, G.flag.p, sizeof(unsigned int), cudaMemcpyDeviceToHost, G.st));
  GK(cudaStreamSynchronize(G.st));
  std::vector<uint32_t> back(G.h_flag[0]);
  GK(cudaMemcpyAsync(back.data(), walk, back.size() * 4, cudaMemcpyDeviceToHost, G.st));
  GK(cudaStreamSynchronize(G.st));
  path.insert(path.end(), back.rbegin(), back.rend());
  return TLAG_OK;
}

}  // namespace

extern "C" int tlag_live_check(const tlag_graph_dev* g, const tlag_live_query* q, uint32_t* lasso_out, uint32_t lasso_cap,
                               tlag_live_result* out) {
  g_err.clear();
  if (!g || !q || !out || !g->off || !g->dst || !g->state_label || !g->edge_label) {
    g_err = "tlag_live_check: missing graph, labels, query or result";
    return TLAG_EINVAL;
  }
  if (g->n_edges >= 0xFFFFFFFFull) {
    g_err = "tlag_live_check: the graph has 2^32 - 1 edges or more (the SCC core indexes edges with 32 bits)";
    return TLAG_EINVAL;
  }
  memset(out, 0, sizeof *out);
  FairSet fs;
  GR(fair_set(q->fair, q->n_fair, q->need_clear, &fs, "tlag_live_check"));
  const u64* off = (const u64*)(uintptr_t)g->off;
  const uint32_t* slab = (const uint32_t*)(uintptr_t)g->state_label;
  const uint32_t* elab = (const uint32_t*)(uintptr_t)g->edge_label;
  DeviceGuard dg;
  Graph G;
  GR(G.init(g->n_states, g->n_edges, g->device, "tlag_live_check"));
  const uint32_t n = G.n;
  const uint64_t m0 = g->n_edges;
  GK(cudaEventRecord(G.ev0, G.st));
  DevBuf<uint32_t> rs, rd;
  DevBuf<uint8_t> em, seeds;
  GK(rs.alloc(m0)); GK(rd.alloc(m0)); GK(em.alloc(m0)); GK(seeds.alloc(n));
  if (n) {
    k_csr_src<<<G.grid_for(n), kBlock, 0, G.st>>>(n, off, rs.p);
    k_live_masks<<<G.grid_for(n), kBlock, 0, G.st>>>(n, slab, q->keep_set, q->keep_clear, q->seed_set, q->seed_clear,
                                                     q->seed_rows ? q->seed_rows : n, G.vmask.p, seeds.p);
    GK(cudaMemcpyAsync(G.word.p, slab, (uint64_t)n * 4, cudaMemcpyDeviceToDevice, G.st));
  }
  if (m0) {
    GK(cudaMemcpyAsync(rd.p, (const uint32_t*)(uintptr_t)g->dst, m0 * 4, cudaMemcpyDeviceToDevice, G.st));
    k_edge_drop<<<G.grid_for(m0), kBlock, 0, G.st>>>(m0, elab, q->edge_drop, em.p);
  }
  GK(cudaGetLastError());
  uint32_t witness = kOut;
  FairSearch F;
  if (q->flags & TLAG_LIVE_ANY_SEED) {
    GK(F.cnt.alloc(2));
    GK(cudaMemcpyAsync(F.cnt.p, F.h_cnt, sizeof F.h_cnt, cudaMemcpyHostToDevice, G.st));
    if (n) k_first_seed<<<G.grid_for(n), kBlock, 0, G.st>>>(n, seeds.p, F.cnt.p);
    GK(cudaGetLastError());
    GK(cudaMemcpyAsync(F.h_cnt, F.cnt.p, sizeof F.h_cnt, cudaMemcpyDeviceToHost, G.st));
    GK(cudaStreamSynchronize(G.st));
    witness = F.h_cnt[0];
  } else {
    GR(G.build(rs, rd, elab, em.p, m0));
    GR(F.run(G, fs, (q->flags & TLAG_LIVE_SEEDS) ? seeds.p : nullptr));
    witness = F.h_cnt[0];
    out->fair_sccs = F.h_cnt[1];
    out->rounds = F.rounds;
  }
  GR(G.elapsed(&out->check_ms));
  out->violated = witness != kOut;
  out->witness = witness;
  if (!out->violated || (q->flags & TLAG_LIVE_ANY_SEED)) {
    if (out->violated) {
      out->prefix_len = 1;
      if (lasso_cap < 1) return TLAG_EOVERFLOW;
      if (lasso_out) lasso_out[0] = witness;
    }
    return TLAG_OK;
  }
  // the lasso
  GK(cudaEventRecord(G.ev0, G.st));
  std::vector<uint32_t> prefix, cycle;
  DevBuf<uint32_t> par, next, walk;
  DevBuf<uint8_t> target, inscc;
  GK(par.alloc(n)); GK(next.alloc(n)); GK(walk.alloc(n)); GK(target.alloc(n)); GK(inscc.alloc(n));
  if (q->flags & TLAG_LIVE_SEEDS) {   // seed -> witness inside the restriction
    GK(cudaMemsetAsync(target.p, 0, n, G.st));
    GK(cudaMemsetAsync(target.p + witness, 1, 1, G.st));
    GR(bfs_path(G, seeds.p, 0, G.vmask.p, target.p, par.p, walk.p, prefix));
  } else {
    prefix.push_back(witness);
  }
  uint32_t c = 0, s_and = 0, e_or = 0;
  GK(cudaMemcpy(&c, F.res.p + witness, 4, cudaMemcpyDeviceToHost));
  GK(cudaMemcpy(&s_and, F.s_and.p + c, 4, cudaMemcpyDeviceToHost));
  GK(cudaMemcpy(&e_or, F.e_or.p + c, 4, cudaMemcpyDeviceToHost));
  k_in_scc<<<G.grid_for(n), kBlock, 0, G.st>>>(n, F.res.p, c, inscc.p);
  GK(cudaGetLastError());
  // the cycle's stops: an A-edge of every condition whose action occurs in the SCC, else (WF) a ~EN state; a state with
  // each need_clear bit clear
  std::vector<std::pair<uint32_t, uint32_t>> stops;   // (state bits to find clear, edge bits to take)
  for (uint32_t k = 0; k < fs.n_wf + fs.n_sf; ++k) {
    if (e_or & fs.act[k]) stops.push_back({0u, fs.act[k]});
    else if (k < fs.n_wf && (s_and & fs.en[k])) {
      g_err = "tlag_live_check: an accepted SCC fails a WF condition (internal error)";
      return TLAG_EINVAL;
    } else if (k < fs.n_wf) stops.push_back({fs.en[k], 0u});
  }
  for (uint32_t b = 0; b < 32; ++b)
    if (fs.need_clear & (1u << b)) stops.push_back({1u << b, 0u});
  cycle.push_back(witness);
  uint32_t at = witness;
  for (const auto& st : stops) {
    GK(cudaMemsetAsync(target.p, 0, n, G.st));
    const uint32_t grid_n = n > G.m ? n : G.m;
    k_scc_targets<<<G.grid_for(grid_n ? grid_n : 1), kBlock, 0, G.st>>>(n, G.m, F.res.p, c, G.word.p, st.first, G.src.p,
                                                                        G.dst.p, G.lab.p, st.second, target.p, next.p);
    GK(cudaGetLastError());
    std::vector<uint32_t> leg;
    GR(bfs_path(G, nullptr, at, inscc.p, target.p, par.p, walk.p, leg));
    cycle.insert(cycle.end(), leg.begin() + 1, leg.end());
    at = leg.back();
    if (st.second) {
      GK(cudaMemcpy(&at, next.p + at, 4, cudaMemcpyDeviceToHost));
      cycle.push_back(at);
    }
  }
  if (at != witness) {
    GK(cudaMemsetAsync(target.p, 0, n, G.st));
    GK(cudaMemsetAsync(target.p + witness, 1, 1, G.st));
    std::vector<uint32_t> leg;
    GR(bfs_path(G, nullptr, at, inscc.p, target.p, par.p, walk.p, leg));
    cycle.insert(cycle.end(), leg.begin() + 1, leg.end() - 1);
  } else if (cycle.size() > 1) {
    cycle.pop_back();
  }
  GR(G.elapsed(&out->lasso_ms));
  out->prefix_len = (uint32_t)prefix.size();
  out->cycle_len = (uint32_t)cycle.size();
  if ((uint64_t)prefix.size() + cycle.size() > lasso_cap) return TLAG_EOVERFLOW;
  if (lasso_out) {
    memcpy(lasso_out, prefix.data(), prefix.size() * 4);
    memcpy(lasso_out + prefix.size(), cycle.data(), cycle.size() * 4);
  }
  return TLAG_OK;
}

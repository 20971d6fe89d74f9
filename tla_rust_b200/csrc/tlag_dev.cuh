// tlag_dev.cuh -- device-side definitions shared by the engine (tlag_engine.cu) and by the translation units of a
// sliced native build (tla_rust_b200/compile/sliced.py writes one .cu per group of slices; they are compiled in
// parallel and linked into one library): counters, kernel parameters, the seen-set probe, the appends to the store and
// to the send regions, and the slice runtime.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/tlag.h"
#include "tlag_vm.h"

struct Counters {
  unsigned long long n_states;      // tail of the state store
  unsigned long long generated;
  unsigned long long work;          // chunk dispenser
  unsigned long long viol_inv;      // min key: idx<<20 | detail
  unsigned long long viol_assert;
  unsigned long long viol_trap;     // idx<<20 | code<<16 | line
  unsigned long long viol_deadlock;
  unsigned long long store_overflow;
  unsigned long long table_full;
  unsigned long long route_overflow;
  unsigned long long send_count[16];
  unsigned long long stop;          // TLAG_F_EXACT: an error was found, no further state is dequeued
};

struct DevParams {
  const uint64_t* code; uint32_t code_len; int code_in_smem;
  const int32_t* cpool;
  const tlag_slot* layout; int n_slots;
  uint32_t entry_inv, entry_next;
  uint32_t n_off, p_off;
  int W;
  uint32_t* states; uint32_t* parent; uint32_t* meta;
  unsigned long long cap_states;    // append limit: a row at or past it is counted in n_states, not written
  // Where appended rows go: row pos's W words at app + pos * app_stride, its parent and meta words at app_parent and
  // app_meta + pos * pm_stride.  That is the store (strides W and 1), or while a level is discovered its discovery
  // buffer of records [W words, parent, meta] (both strides W + 2), which the host clusters into the store when the level
  // ends.  For the buffer the host offsets the pointers by the level's first row, so that appends take no branch.
  uint32_t* app; uint32_t* app_parent; uint32_t* app_meta;
  unsigned app_stride, pm_stride;
  unsigned long long* table; unsigned long long mask;
  Counters* ctr;
  uint32_t flags;
  int n_inv;
  uint8_t* succ_flag;               // sliced build: one byte per frontier state, set when a slice produced a successor
  // route mode
  int route;                        // sliced build: successors go to the send regions instead of the local seen-set
  int owner_words;                  // trailing packed words the ownership hash covers (tlag_owner_k; 2 = clustering key)
  uint32_t* send; unsigned long long region_cap; int n_ranks; int rank;
  unsigned long long* sent_cache; unsigned long long sent_mask;   // direct-mapped filter of fingerprints already routed
  int skip_self;                    // sliced build: a successor equal to its parent is counted, never fingerprinted or probed
  int stage;                        // sliced build, scalar form: cap on the per-warp staging slots used (0: none, all direct)
};

// ---- random simulation (tlag_simulate) ----
// A walk's status between the kernels of a step
enum { SIM_RUN = 0, SIM_ENDED = 1, SIM_FAILED = 2 /* this step: no successor is enumerated */,
       SIM_FAILED_NEXT = 3 /* this step, while its successors were enumerated: the enumeration goes on */ };

struct SimCtl {
  unsigned long long stopped;       // 1 + the first step of the batch that held an error (0: none): later steps are no-ops
  unsigned long long checked;       // states whose invariants were evaluated
};

// One step t of a batch.  The history is `depth` rows of B walks x W words; the step reads row t (DevParams::states,
// walks [0, n)) and writes each walk's pick into row t + 1.
struct SimParams {
  unsigned long long seed, first;   // seed of the run, global id of the batch's walk 0
  uint32_t t, depth, B, flags;      // step, behaviour length bound, walks per row, TLAG_F_DEADLOCK_CHECK
  uint32_t* hist; int16_t* act;     // history rows; action id of each row's state (-1: initial)
  uint8_t* status; uint32_t* cnt;   // per walk: SIM_*, candidates seen this step
  uint32_t* len;                    // per walk: states checked
  SimCtl* ctl;
};

__device__ __forceinline__ bool sim_stopped(const SimParams& s) {
  return *(volatile const unsigned long long*)&s.ctl->stopped != 0;
}

// the pick so far of walk idx at step s.t: its successor goes to row t + 1
__device__ __forceinline__ void sim_pick(const SimParams& s, unsigned long long idx, uint32_t j, int aid, const uint32_t* w,
                                         int W) {
  if (!tlag_sim_take(s.seed, s.first + idx, s.t, j)) return;
  uint32_t* dst = s.hist + ((unsigned long long)(s.t + 1) * s.B + idx) * (unsigned long long)W;
  for (int i = 0; i < W; ++i) dst[i] = w[i];
  s.act[(unsigned long long)(s.t + 1) * s.B + idx] = (int16_t)aid;
}

// ---- peer-memory exchange (tlag_engine.cu: k_push / k_insert_inbox) ----
struct P2PMeta {                       // lives in the OWNER's memory, one per source rank
  unsigned long long count[2];         // records the source pushed into buffer (seq & 1)            [written by the source]
  unsigned long long seq[2];           // chunk number whose records are complete in that buffer      [written by the source]
  unsigned long long ack;              // as a source: last chunk of MINE that this peer has consumed [written by the peer]
  unsigned long long pad[3];
};

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

struct P2PParams {
  int n_ranks, rank, rec_words;
  unsigned long long inbox_cap;        // records per (owner, source, buffer) region
  unsigned long long region_cap;       // records per destination in the local send buffer
  const uint32_t* send;                // local send regions [n_ranks][region_cap][rec_words]
  uint32_t* peer_inbox[16];            // rank r's inbox base as mapped in this process
  P2PMeta* peer_meta[16];              // rank r's meta array as mapped in this process
  uint32_t* inbox; P2PMeta* meta;      // this rank's own
  unsigned int* tickets;               // [0..16): k_push "last block per destination", [16]: k_insert_inbox
};


// ------------------------------------------------------------------ seen-set
// returns 1 if fp was inserted by this call, 0 if already present, -1 if the table is full
__device__ __forceinline__ int seen_insert(unsigned long long* table, unsigned long long mask,
                                           unsigned long long fp) {
  // read first, CAS only on an empty slot: atomics are throughput-limited at L2, and duplicates need no atomic at all
  unsigned long long i = fp & mask;
  for (unsigned long long probes = 0; probes <= mask; ++probes) {
    const unsigned long long cur = __ldcv(&table[i]);
    if (cur == fp) return 0;
    if (cur == 0ULL) {
      const unsigned long long old = atomicCAS(&table[i], 0ULL, fp);
      if (old == 0ULL) return 1;
      if (old == fp) return 0;
    }
    i = (i + 1) & mask;
  }
  return -1;
}

// seen_insert for a caller that has already loaded the home slot (table[fp & mask]) as cur, so that it can keep several
// such loads in flight: an empty slot is claimed with a CAS, one that holds another state runs the whole probe
__device__ __forceinline__ int seen_insert_at(unsigned long long* table, unsigned long long mask, unsigned long long fp,
                                              unsigned long long cur) {
  if (cur == fp) return 0;
  if (cur == 0ULL) {
    const unsigned long long old = atomicCAS(&table[fp & mask], 0ULL, fp);
    if (old == 0ULL) return 1;
    if (old == fp) return 0;
  }
  return seen_insert(table, mask, fp);
}

// the result of a probe, with a full table (-1) reported in table_full: 1 if the state is new, else 0
__device__ __forceinline__ int seen_report(Counters* ctr, int ins) {
  if (ins < 0) { atomicExch(&ctr->table_full, 1ULL); return 0; }
  return ins;
}

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// meta word of a stored state: the action that produced it, and the rank that expanded its parent (whose store the
// parent index points into)
__device__ __forceinline__ uint32_t tlag_meta(int aid, int rank) { return ((uint32_t)aid << 8) | (uint32_t)(rank & 0xFF); }

// Where new row pos (< cap_states) is written: its W words, its parent and its meta word (DevParams::app)
struct RowDst { uint32_t* w; uint32_t* parent; uint32_t* meta; };
__device__ __forceinline__ RowDst row_dst(const DevParams& p, unsigned long long pos) {
  return {p.app + pos * p.app_stride, p.app_parent + pos * p.pm_stride, p.app_meta + pos * p.pm_stride};
}

// Appends a new state to the tail of the store.  Only the lanes of `group` call it, each with a new state: one tail
// atomic for the group, rows in lane order.  A row past cap_states is still counted in n_states (the host sizes the
// rerun of the level from it) and is reported in store_overflow.
__device__ __forceinline__ void store_append(const DevParams& p, unsigned group, const uint32_t* w, int W, uint32_t parent,
                                             uint32_t meta) {
  const int leader = __ffs((int)group) - 1;
  unsigned long long base = 0;
  if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(&p.ctr->n_states, (unsigned long long)__popc(group));
  base = __shfl_sync(group, base, leader);
  const unsigned long long pos = base + (unsigned long long)__popc(group & lanemask_lt());
  if (pos < p.cap_states) {
    const RowDst d = row_dst(p, pos);
    for (int i = 0; i < W; ++i) d.w[i] = w[i];
    *d.parent = parent;
    *d.meta = meta;
  } else {
    atomicExch(&p.ctr->store_overflow, 1ULL);
  }
}

// Route mode: appends a successor that `owner` holds to that rank's send region (W words, parent, meta), with one
// atomic per group of lanes present that route to the same owner.  A successor whose fingerprint this rank has already
// routed is known to its owner and is dropped (direct-mapped exact-compare cache: a miss only costs a redundant record).
// The cache slot is written only once the record is in the send region, so a chunk that is re-run after a region
// overflow finds none of its dropped records there.
__device__ __forceinline__ void route_append(const DevParams& p, const uint32_t* w, int W, unsigned long long fp, int owner,
                                             uint32_t parent, uint32_t meta) {
  unsigned long long* cslot = p.sent_cache ? p.sent_cache + (fp & p.sent_mask) : nullptr;
  if (cslot && __ldcv(cslot) == fp) return;
  const unsigned peers = __match_any_sync(__activemask(), owner);
  const int leader = __ffs((int)peers) - 1;
  unsigned long long base = 0;
  if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(&p.ctr->send_count[owner], (unsigned long long)__popc(peers));
  base = __shfl_sync(peers, base, leader);
  const unsigned long long pos = base + (unsigned long long)__popc(peers & lanemask_lt());
  if (pos < p.region_cap) {
    uint32_t* dst = p.send + ((unsigned long long)owner * p.region_cap + pos) * (unsigned long long)(W + 2);
    for (int i = 0; i < W; ++i) dst[i] = w[i];
    dst[W] = parent;
    dst[W + 1] = meta;
    if (cslot) *cslot = fp;
  } else {
    atomicExch(&p.ctr->route_overflow, 1ULL);
  }
}

__device__ __forceinline__ void report_min(unsigned long long* slot, unsigned long long key) {
  atomicMin(slot, key);
}

// ------------------------------------------------------------------ sliced native build
// (tla_rust_b200/compile/sliced.py)  One kernel per slice of the model's program: k_sl_inv_<i> evaluates invariant i,
// k_sl_next_<j> one disjunct of Next, each over the whole frontier, one thread per state.  All warps of a launch run
// the same few KB of straight-line code (the whole-program compiled form of round 1 lost to the interpreter on
// instruction-cache misses: 354 KB of code, every warp somewhere else); divergence inside a slice is the hardware's
// (compiler-placed reconvergence) instead of a min-pc election per block; a successor is packed where it is produced,
// then staged for a probe by the whole warp (scalar form) or fingerprinted and inserted there (array form).
// A translation unit that holds slices defines TLAG_SLICED_DEFS (the generated header with the model's constants) before
// including this file, then the slice functions, then TLAG_SL_KERNEL_INV(j) / TLAG_SL_KERNEL_NEXT(j) for its slices.
#ifdef TLAG_SLICED_DEFS
// the scalar form's emit sites test this before they hand a successor equal to its parent to TLAG_SL_EMITW
// (TLAG_SL_SIM, a simulation library: a self-loop is a candidate like any other successor)
#ifdef TLAG_SL_SIM
#define TLAG_SL_SKIPSELF 0
#else
#define TLAG_SL_SKIPSELF (cx->p->skip_self)
#endif
#include TLAG_SLICED_DEFS
struct tlag_sl_cx {
  const DevParams* p;
  unsigned long long idx;
  const uint32_t* src;              // packed words of the state being expanded (EMITD re-packs over a copy)
  unsigned long long gen;
  unsigned nsucc;
  int phase;                        // 0 = invariant slice, 1 = slice of Next
#if TLAG_SL_SCALAR                  // (only the scalar form stages: the array form's kernels are left as they were)
  unsigned stage_cap;               // staging slots this launch may use per warp (0: every successor goes direct)
#endif
#ifdef TLAG_SL_SIM
  const SimParams* sim;
  unsigned cnt;                     // candidates of this step so far
  int stat;                         // the walk's SIM_* status
#endif
};

#ifndef TLAG_SL_BLOCK
#define TLAG_SL_BLOCK 256
#endif
#ifndef TLAG_SL_OCC
#define TLAG_SL_OCC 4               /* resident CTAs per SM the slice kernels are compiled for (register cap) */
#endif

static __device__ __noinline__ void sl_emit_words(tlag_sl_cx* cx, int aid, const uint32_t* o);
static __device__ __noinline__ void sl_emit_frame(tlag_sl_cx* cx, const int32_t* f, int aid, int dirty);
#define TLAG_SL_EMIT(aid, dirty) sl_emit_frame(cx, f, (aid), (dirty))

// Per-warp staging (scalar form, Next kernels, not in route mode).  An emit site puts its successor into a slot of its
// warp's buffer; the whole warp later fingerprints and probes the staged successors together (sl_flush, tlag_dev2.cuh),
// instead of every group of lanes that reaches a site waiting on its own seen-set round trip inside divergent code.
// Budget: 3.5 KB a warp, 28 KB a 256-thread CTA, so that 4 CTAs per SM take 112 KB of the 228 KB of shared memory.
// A slot holds the W packed words, the parent index and the meta word; at fewer than 32 slots (W > 26) nothing is staged.
#define TLAG_SL_STAGE_BYTES 3584
#define TLAG_SL_STAGE_SLOTS ((TLAG_SL_STAGE_BYTES / (4 * (TLAG_SL_W + 2)) / 32) * 32)
#if TLAG_SL_SCALAR && TLAG_SL_STAGE_SLOTS >= 32 && !defined(TLAG_SL_SIM)
#define TLAG_SL_STAGED 1
// word-major: word k of slot s of warp v at [v][k][s], so that the lanes of an emit site (consecutive slots) and of a
// flush (slots lane, lane + 32, ...) hit distinct banks; the row is one word longer than the slots so that the flush's
// copy into the store (consecutive words of one slot on consecutive lanes) does too.  Words W, W + 1: parent, meta.
static __shared__ uint32_t tlag_sl_stage[TLAG_SL_BLOCK / 32][TLAG_SL_W + 2][TLAG_SL_STAGE_SLOTS + 1];
static __shared__ unsigned tlag_sl_fill[TLAG_SL_BLOCK / 32];     // slots taken; may run past the cap (those went direct)
static __shared__ unsigned short tlag_sl_row[TLAG_SL_BLOCK / 32][TLAG_SL_STAGE_SLOTS];   // flush: new row -> slot

static __device__ __forceinline__ void sl_stage_words(tlag_sl_cx* cx, int aid, const uint32_t* o) {
  constexpr int W = TLAG_SL_W;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // divergent groups of one warp can interleave here: slots are taken with one shared atomic per arriving group
  const unsigned am = __activemask();
  const int leader = __ffs((int)am) - 1;
  unsigned base = 0;
  if ((int)lane == leader) base = atomicAdd(&tlag_sl_fill[warp], (unsigned)__popc(am));
  base = __shfl_sync(am, base, leader);
  const unsigned s = base + (unsigned)__popc(am & lanemask_lt());
  if (s < cx->stage_cap) {
    cx->nsucc++; cx->gen++;
#pragma unroll
    for (int k = 0; k < W; ++k) tlag_sl_stage[warp][k][s] = o[k];
    tlag_sl_stage[warp][W][s] = (uint32_t)cx->idx;
    tlag_sl_stage[warp][W + 1][s] = tlag_meta(aid, cx->p->rank);
  } else {
    // buffer full: probe here, as without staging (a copy, so that the site's words can stay in registers)
    uint32_t w[W];
#pragma unroll
    for (int k = 0; k < W; ++k) w[k] = o[k];
    sl_emit_words(cx, aid, w);
  }
}
#define TLAG_SL_EMITW(aid, o) sl_stage_words(cx, (aid), (o))
#else
#define TLAG_SL_EMITW(aid, o) sl_emit_words(cx, (aid), (o))
#endif
#define TLAG_SL_GEN() do { cx->nsucc++; cx->gen++; } while (0)
#ifdef TLAG_SL_SIM
// as below, and the walk fails at this step (an Assert while Next is enumerated lets the enumeration go on, as the
// interpreter does)
#define TLAG_SL_SIM_FAIL() (cx->stat = cx->phase == 0 ? SIM_FAILED : (cx->stat == SIM_RUN ? SIM_FAILED_NEXT : cx->stat))
#define TLAG_SL_ASSERT(id) do { report_min(&cx->p->ctr->viol_assert, (cx->idx << 20) | (unsigned)((id) & 0xFFFFF)); TLAG_SL_SIM_FAIL(); } while (0)
#define TLAG_SL_INVF(i) do { if (cx->phase == 0) { report_min(&cx->p->ctr->viol_inv, (cx->idx << 20) | (unsigned)((i) & 0xFFFFF)); cx->stat = SIM_FAILED; } } while (0)
#define TLAG_SL_TRAP(code, line) do { report_min(&cx->p->ctr->viol_trap, (cx->idx << 20) | ((unsigned long long)((code) & 15) << 16) | (unsigned)((line) & 0xFFFF)); cx->nsucc++; cx->stat = SIM_FAILED; } while (0)
#else
#define TLAG_SL_ASSERT(id) report_min(&cx->p->ctr->viol_assert, (cx->idx << 20) | (unsigned)((id) & 0xFFFFF))
#define TLAG_SL_INVF(i) do { if (cx->phase == 0) report_min(&cx->p->ctr->viol_inv, (cx->idx << 20) | (unsigned)((i) & 0xFFFFF)); } while (0)
#define TLAG_SL_TRAP(code, line) do { report_min(&cx->p->ctr->viol_trap, (cx->idx << 20) | ((unsigned long long)((code) & 15) << 16) | (unsigned)((line) & 0xFFFF)); cx->nsucc++; } while (0)
#endif
#define TLAG_SL_SUBQ static __device__ __noinline__
// Array form with a big frame (container models): the slice is a function of its own that receives the frame as a
// pointer -- inlined, cicc tries scalar replacement of a 2 K-word array over a goto graph and takes many minutes (raft).
#if defined(TLAG_SL_SEG_NOINLINE)
#define TLAG_SL_SEGQ static __device__ __noinline__
#else
#define TLAG_SL_SEGQ static __device__ __forceinline__
#endif
// (the slice functions of this translation unit follow the #include of this header)
#define TLAG_SL_RUNTIME_PART2 1
#endif  // TLAG_SLICED_DEFS

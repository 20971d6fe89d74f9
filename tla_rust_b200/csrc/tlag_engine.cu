// tlag_engine.cu -- sm_90a (H100) BFS engine behind include/tlag.h.
//
// One wave (BFS level) = one launch of k_wave: a persistent grid pulls 32-state chunks of
// the frontier; each thread unpacks its state, runs the invariant program, then the
// next-state program.  Every EMIT event is handled warp-synchronously: pack -> 64-bit
// fingerprint -> open-addressed seen-set probe/insert (atomicCAS on 8-byte slots in HBM)
// -> __ballot_sync compaction of the newly discovered states into the tail of the state
// store (which doubles as the BFS queue: the next frontier is the slice appended by this
// wave).  Successor states never round-trip through HBM before the probe (SURVEY.md §8d:
// the fused form of K2->K1->K3->K4).  No tensor cores: integer / hash work only.
//
// Replaces TLC's Worker loop + StateQueue, action evaluator, FPSet and invariant checker
// (SURVEY.md §2b; all external to /root/reference, which only fixes the CLI contract
// Makefile:6-7 and the output format README.md:267-321).
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <string>
#include <type_traits>
#include <unordered_set>
#include <vector>
#include <cub/device/device_radix_sort.cuh>   // CUDA-toolkit header library; used only to reorder a level (not on the hot path)
#include <cub/device/device_select.cuh>       // (and by the state graph pass: duplicate edges of a chunk)

#include "tlag_dev.cuh"
// second copy of the instruction executor without the extension ops (see tlag_vm_exec.inc)
#define TLAG_VM_EXEC_FN tlag_vm_exec_lean
#define TLAG_VM_EXT 0
#include "tlag_vm_exec.inc"
#undef TLAG_VM_EXEC_FN
#undef TLAG_VM_EXT

// Resident CTAs per SM the interpreter wave kernel is compiled for (register cap = 65536 / (512 x this)).  Big frames
// (> 512 words) with the image in global memory get 4: they are latency-bound on local memory.
#define TLAG_WAVE_OCC(FRAME, SMEM) ((FRAME) <= 256 ? 4 : ((FRAME) <= 512 ? 2 : ((SMEM) ? 1 : 4)))

#define TLAG_MAXW 128
#define TLAG_BLOCK 512
#define TLAG_MAX_STEPS (1u << 26)

// The policy that picks an interpreter kernel's variant (vm_variant; a sliced library's k_graph at compile time).  The
// frame is a per-thread array of the frame class: the frame rounded up to a power of two, 64 to 8192 words.
constexpr int vm_frame_class(uint32_t words) {
  int c = 64;
  while (c < 8192 && (uint32_t)c < words) c *= 2;
  return c;
}
// The program runs from shared memory when it fits.  Big frames (container models such as raft) are bound by local-memory
// latency (ncu: long-scoreboard 37 per issue, 16 warps/SM): they run with the program in global memory (read through L1)
// so that two CTAs fit per SM.
constexpr bool vm_code_in_smem(uint32_t words, uint32_t code_len) {
  return (uint64_t)code_len * 8 <= (words > 512 ? 0 : 200 * 1024);
}

#define CK(call)                                                                         \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess) {                                                             \
      e->err = std::string(#call) + ": " + cudaGetErrorString(_e);                       \
      return TLAG_ECUDA;                                                                 \
    }                                                                                    \
  } while (0)

struct tlag_engine {
  tlag_model m;
  std::vector<uint64_t> h_code;
  std::vector<uint32_t> h_init;     // retained initial states (for tlag_restart)
  DevParams p;
  uint64_t* d_code = nullptr; int32_t* d_cpool = nullptr; tlag_slot* d_layout = nullptr;
  uint32_t* d_states = nullptr; uint32_t* d_parent = nullptr; uint32_t* d_meta = nullptr;
  unsigned long long* d_table = nullptr; unsigned table_log2 = 0;
  Counters* d_ctr = nullptr;
  uint64_t cap_states = 0;
  uint64_t lo = 0, hi = 0;          // current frontier [lo,hi)
  uint64_t level = 0;               // level of the frontier (1 = initial states)
  uint64_t init_states = 0;
  uint64_t generated = 0;
  uint64_t depth = 0;
  int verdict = TLAG_V_RUNNING; int detail = 0, detail2 = 0; uint64_t viol_idx = 0;
  double dev_seconds = 0;
  uint64_t launches = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  int sm_count = 132;
  int frame_class = 64;              // the interpreter's frame class, in words (vm_frame_class)
  bool uses_ext = false;            // the image contains LEXLT / SFIND / SINS / EMITD (full interpreter needed)
  bool restarting = false;
  bool tight = false;               // TLAG_TIGHT_HEADROOM (test hook): store and table sized for no growth, see read_env_hooks
  bool no_sort = false;             // TLAG_NO_SORT (test hook): levels go to the store in discovery order, see cluster_slice
  double growth_hint = 4.0;
  double disc_hint = 4.0;           // discovery buffer rows per state expanded, for the next level (note_growth)
  // discovery buffer: the open level's new rows (DevParams::disc), put into the store by close_level
  void* d_disc = nullptr; uint64_t disc_bytes = 0; bool disc_open = false;
  void* d_sort = nullptr; uint64_t sort_bytes = 0;    // clustering pass: (rank, index) pairs, double-buffered, CUB temp
  // clustering pass: the rank set ([RankSetCtl | keys | ranks | key lists], cluster_slice), its size carried from level to
  // level
  void* d_rset = nullptr; uint64_t rset_bytes = 0; unsigned rset_log2 = 16; bool rset_fixed = false;
  unsigned long long* d_sent = nullptr;
  uint8_t* d_succ = nullptr; uint64_t succ_cap = 0;   // sliced build: per-frontier-state "has a successor" flags
  unsigned long long* d_dig = nullptr;                // tlag_digest accumulators (XOR, SUM)
  // peer-memory exchange (tlag_p2p_*): one cudaMalloc'ed block [meta | inbox x 2 buffers], exported through CUDA IPC
  P2PParams q;
  void* d_p2p = nullptr; uint64_t p2p_bytes = 0;
  uint32_t* d_send_own = nullptr;
  unsigned int* d_tickets = nullptr;
  void* peer_base[16] = {nullptr};
  unsigned long long p2p_seq = 0;
  int p2p_slot = -1;                                   // entry of g_p2p_parked this engine's exchange buffers belong to
  bool p2p_ready = false;
  uint64_t p2p_level_start = 0, p2p_level_generated = 0;   // for tlag_p2p_rollback: store tail before the level, what it added
  // TLAG_F_KEEP_GOING: the first violation is remembered, the search goes on to the fixpoint
  int kg_verdict = 0, kg_detail = 0, kg_detail2 = 0; uint64_t kg_idx = 0;
  std::string err;
  uint32_t* d_scratch = nullptr; uint64_t scratch_words = 0; uint8_t* d_flags = nullptr; uint64_t flags_cap = 0;
  // random simulation (tlag_simulate): one batch's history and per-walk state, sized for sim_B walks x sim_D rows; the
  // last batch run stays readable (tlag_sim_trace, tlag_sim_read) until the next call
  uint32_t* d_hist = nullptr; int16_t* d_act = nullptr; uint8_t* d_sstat = nullptr; uint8_t* d_ssucc = nullptr;
  uint32_t* d_scnt = nullptr; uint32_t* d_slen = nullptr; SimCtl* d_sctl = nullptr; uint32_t* d_sinit = nullptr;
  uint64_t sim_B = 0, sim_D = 0, sim_n = 0, sim_first = 0, sim_n_init = 0;
  // state graph (tlag_build_graph): CSR over the store's rows, offsets g_states + 1, released when the search moves on
  unsigned long long* d_goff = nullptr; uint32_t* d_gdst = nullptr; uint32_t* d_gact = nullptr;
  uint64_t g_cap = 0, g_edges = 0, g_states = 0, g_expanded = 0; bool g_ready = false;
  uint64_t graph_edges = 1ULL << 24;  // edges the chunk buffer of the edge pass starts with (TLAG_GRAPH_EDGES: test hook)
  // the graph's liveness labels (tlag_label_graph): one word per row and one per edge, released with the graph
  uint32_t* d_slab = nullptr; uint32_t* d_elab = nullptr;
};

// ------------------------------------------------------------------ sliced native build
// The slice kernels live in translation units of their own (csrc/native/<tag>_part<k>.cu, generated and compiled in
// parallel: tla_rust_b200/engine.py build_sliced_library); this unit only knows their launchers.
#ifdef TLAG_SLICED_INC
#include TLAG_SLICED_INC     /* the generated constants: TLAG_SL_W, TLAG_SL_*_LIST, program length + FNV */
#ifndef TLAG_SL_BLOCK
#define TLAG_SL_BLOCK 256
#endif
// CTAs of a slice kernel over n rows: one thread per row, at most 64 CTAs per SM
static unsigned sl_blocks(const tlag_engine* e, uint64_t n) {
  const uint64_t blocks = (n + TLAG_SL_BLOCK - 1) / TLAG_SL_BLOCK, maxb = (uint64_t)e->sm_count * 64;
  return (unsigned)(blocks < maxb ? blocks : maxb);
}
typedef void (*sl_launch_t)(const DevParams*, unsigned long long, unsigned long long, unsigned, cudaStream_t);
#ifdef TLAG_SL_SIM
// a simulation library (build_sliced_library(cm, simulate=True)): its slice kernels are the simulation kernels only
typedef void (*sl_sim_launch_t)(const DevParams*, const SimParams*, unsigned long long, unsigned, cudaStream_t);
#define TLAG_SL_DECL_INV(j) extern "C" void tlag_sl_sim_launch_inv_##j(const DevParams*, const SimParams*, unsigned long long, unsigned, cudaStream_t);
#define TLAG_SL_DECL_NEXT(j) extern "C" void tlag_sl_sim_launch_next_##j(const DevParams*, const SimParams*, unsigned long long, unsigned, cudaStream_t);
TLAG_SL_INV_LIST(TLAG_SL_DECL_INV)
TLAG_SL_NEXT_LIST(TLAG_SL_DECL_NEXT)
#define TLAG_SL_ADDR_INV(j) tlag_sl_sim_launch_inv_##j,
#define TLAG_SL_ADDR_NEXT(j) tlag_sl_sim_launch_next_##j,
static const sl_sim_launch_t kSlSimInv[] = { TLAG_SL_INV_LIST(TLAG_SL_ADDR_INV) nullptr };
static const sl_sim_launch_t kSlSimNext[] = { TLAG_SL_NEXT_LIST(TLAG_SL_ADDR_NEXT) nullptr };
static const sl_launch_t kSlInv[] = { nullptr };
static const sl_launch_t kSlNext[] = { nullptr };
#define TLAG_NO_BFS(e) do { (e)->err = "this library holds the model's simulation kernels only: a search needs its BFS library"; return TLAG_EINVAL; } while (0)
#else
#define TLAG_SL_DECL_INV(j) extern "C" void tlag_sl_launch_inv_##j(const DevParams*, unsigned long long, unsigned long long, unsigned, cudaStream_t);
#define TLAG_SL_DECL_NEXT(j) extern "C" void tlag_sl_launch_next_##j(const DevParams*, unsigned long long, unsigned long long, unsigned, cudaStream_t);
TLAG_SL_INV_LIST(TLAG_SL_DECL_INV)
TLAG_SL_NEXT_LIST(TLAG_SL_DECL_NEXT)
#define TLAG_SL_ADDR_INV(j) tlag_sl_launch_inv_##j,
#define TLAG_SL_ADDR_NEXT(j) tlag_sl_launch_next_##j,
static const sl_launch_t kSlInv[] = { TLAG_SL_INV_LIST(TLAG_SL_ADDR_INV) nullptr };
static const sl_launch_t kSlNext[] = { TLAG_SL_NEXT_LIST(TLAG_SL_ADDR_NEXT) nullptr };
#endif

// deadlock = a frontier state for which no slice of Next produced a successor
__global__ void k_sl_deadlock(DevParams p, unsigned long long lo, unsigned long long hi) {
  const unsigned long long i = lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < hi && !p.succ_flag[i - lo]) report_min(&p.ctr->viol_deadlock, i << 20);
}
#endif  // TLAG_SLICED_INC

// ------------------------------------------------------------------ wave kernel
// Warp-scheduled interpreter.  A SIMT interpreter that lets every lane follow its own pc pays a
// divergent fetch/decode/dispatch per distinct opcode per step.  Here the warp executes, at every
// step, the ONE instruction at the minimum pc among its running lanes (REDUX min), for exactly the
// lanes that are at that pc: fetch (shared-memory broadcast), decode and dispatch are warp-uniform,
// frame accesses use the same word index in every lane (coalesced local memory), and lanes that
// took different branches re-join as soon as the laggards catch up (forward progress is by
// construction: the lowest pc always advances).
enum { L_RUN = 0, L_EMIT = 1, L_DONE = 2, L_STOP = 3 };
#define TLAG_PC_PARKED 0xFFFFFFFFu

// A lane that is not running parks its pc at TLAG_PC_PARKED (so it never wins the min) and keeps the
// pc to resume from in `rpc`.  Per step: one REDUX min, one shared-memory broadcast fetch, uniform
// decode/dispatch; only lanes whose pc equals the minimum execute.
template <bool SMEM, bool LEAN>
__device__ __forceinline__ void warp_vm(const uint64_t* __restrict__ gcode, const uint64_t* scode,
                                        const int32_t* __restrict__ cpool, int32_t* frame, uint32_t& pc,
                                        uint32_t& rpc, int& ev_out, int32_t& info, int32_t& info2) {
  for (;;) {
    const uint32_t pcm = __reduce_min_sync(0xffffffffu, pc);
    if (pcm == TLAG_PC_PARKED) break;
    const uint64_t w = SMEM ? scode[pcm] : __ldg(gcode + pcm);
    if (pc == pcm) {
      const int ev = LEAN ? tlag_vm_exec_lean(w, cpool, frame, &pc, &info, &info2)
                          : tlag_vm_exec(w, cpool, frame, &pc, &info, &info2);
      if (ev >= 0) { ev_out = ev; rpc = pc; pc = TLAG_PC_PARKED; }
    }
  }
}

// The program warp_vm fetches from shared memory: with SMEM the CTA copies it there first
template <bool SMEM>
__device__ __forceinline__ const uint64_t* vm_stage_code(const DevParams& p) {
  extern __shared__ uint64_t s_code[];
  if (SMEM) {
    for (uint32_t i = threadIdx.x; i < p.code_len; i += blockDim.x) s_code[i] = p.code[i];
    __syncthreads();
  }
  return s_code;
}

// Row idx of p.states (W = p.W words): its packed words into succ[], unpacked into the frame
__device__ __forceinline__ void vm_load_row(const DevParams& p, int W, unsigned long long idx, uint32_t* succ,
                                            int32_t* frame) {
  const uint32_t* src = p.states + idx * (unsigned long long)W;
  for (int i = 0; i < W; ++i) succ[i] = src[i];
  tlag_unpack(p.layout, p.n_slots, succ, frame + p.n_off);
}

// The successor at the lane's EMIT into succ[]: EMITD (info2 > 0) re-packs its dirty slot ranges into a copy of row idx,
// EMIT packs the whole frame.  Returns 0, or 1 + the slot whose value does not fit (tlag_pack).
template <bool LEAN>
__device__ __forceinline__ int vm_pack_emit(const DevParams& p, int W, unsigned long long idx, int32_t info2,
                                            const int32_t* frame, uint32_t* succ) {
  if (!LEAN && info2 > 0) {
    const uint32_t* src = p.states + idx * (unsigned long long)W;
    for (int i = 0; i < W; ++i) succ[i] = src[i];
    return tlag_pack_ranges(p.layout, p.cpool, info2, frame + p.p_off, succ);
  }
  return tlag_pack(p.layout, p.n_slots, frame + p.p_off, succ, W);
}

// v summed over the warp and added to *total, one atomic per warp
__device__ __forceinline__ void warp_add(unsigned long long* total, unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(total, v);
}

// A digest kernel's last step: the XOR and the SUM of its terms over the warp, into out2[0] and out2[1]
__device__ __forceinline__ void warp_digest(unsigned long long* out2, unsigned long long x, unsigned long long sm) {
  for (int o = 16; o > 0; o >>= 1) { x ^= __shfl_down_sync(0xffffffffu, x, o); sm += __shfl_down_sync(0xffffffffu, sm, o); }
  if ((threadIdx.x & 31) == 0) { atomicXor(&out2[0], x); atomicAdd(&out2[1], sm); }
}

#ifndef TLAG_SLICED_INC   // (a sliced library runs the interpreter only in the state graph's edge pass, k_graph)

// MODE 0: fused insert (single GPU).  MODE 1: route successors to per-owner send regions.
// LEAN: interpreter without the extension ops, for models that do not use them (small frames only).
template <int FRAME, int MODE, bool SMEM, bool LEAN = false>
__global__ void __launch_bounds__(TLAG_BLOCK, TLAG_WAVE_OCC(FRAME, SMEM))
k_wave(DevParams p, unsigned long long lo, unsigned long long hi) {
  const uint64_t* s_code = vm_stage_code<SMEM>(p);
  const uint64_t* code = p.code;
  int32_t frame[FRAME];
  uint32_t succ[TLAG_MAXW];
  const unsigned lane = threadIdx.x & 31;
  const int W = p.W;
  unsigned long long gen_local = 0;
  // TLAG_F_EXACT (launched as ONE warp): lane 0 dequeues one state at a time, in index = FIFO order, and the search
  // stops at the first Assert failure / deadlock -- TLC's single worker, on the device
  const bool exact = MODE == 0 && (p.flags & TLAG_F_EXACT) != 0;

  for (;;) {
    if (exact && *(volatile unsigned long long*)&p.ctr->stop) break;
    unsigned long long chunk = 0;
    if (lane == 0) chunk = atomicAdd(&p.ctr->work, 1ULL);
    chunk = __shfl_sync(0xffffffffu, chunk, 0);
    const unsigned long long first = lo + chunk * (exact ? 1ULL : 32ULL);
    if (first >= hi) break;
    const unsigned long long idx = first + lane;
    const bool active = idx < hi && (!exact || lane == 0);
    if (active) vm_load_row(p, W, idx, succ, frame);
    bool trapped = false;
    int st, ev = 0;
    int32_t info = 0, info2 = 0;
    uint32_t pc, rpc = 0;
    // One interpreter loop for both programs (a single copy of the dispatch switch: the first version
    // inlined it twice and stalled on instruction fetch -- ncu stall_no_instruction 14 per issue).
    // Each lane first runs the invariant program on the state it expands; at its HALT it continues
    // with the next-state program (the invariant code sits at lower pcs, so those lanes go first).
    int phase = p.n_inv > 0 ? 0 : 1;
    st = active ? L_RUN : L_DONE;
    pc = active ? (phase == 0 ? p.entry_inv : p.entry_next) : TLAG_PC_PARKED;
    unsigned nsucc = 0;
    for (;;) {
      warp_vm<SMEM, LEAN>(code, s_code, p.cpool, frame, pc, rpc, ev, info, info2);
      int32_t act = 0;
      if (st == L_RUN) {        // this lane stopped on an event
        if (ev == TLAG_EV_EMIT) { st = L_EMIT; ++nsucc; ++gen_local; }
        else if (ev == TLAG_EV_HALT) {
          if (phase == 0) { phase = 1; pc = p.entry_next; } else st = L_DONE;
        }
        else if (ev == TLAG_EV_GEN) { ++nsucc; ++gen_local; pc = rpc; }
        else if (ev == TLAG_EV_INVF) {
          if (phase == 0) report_min(&p.ctr->viol_inv, (idx << 20) | (unsigned)(info & 0xFFFFF));
          pc = rpc;
        }
        else if (ev == TLAG_EV_ASSERT) {
          report_min(&p.ctr->viol_assert, (idx << 20) | (unsigned)(info & 0xFFFFF));
          if (exact) { atomicExch(&p.ctr->stop, 1ULL); st = L_DONE; trapped = true; }   // stop here: nothing after it is generated
          else pc = rpc;
        }
        else {
          report_min(&p.ctr->viol_trap, (idx << 20) | ((unsigned long long)(info & 15) << 16) | (unsigned)(info2 & 0xFFFF));
          st = L_DONE; trapped = true;
        }
      }
      if (__any_sync(0xffffffffu, pc != TLAG_PC_PARKED)) continue;   // resume the lanes that only reported
      bool has = (st == L_EMIT);
      if (!__any_sync(0xffffffffu, has)) break;                 // every lane is done
      act = info;
      unsigned long long fp = 0;
      if (has) {
        const int ov = vm_pack_emit<LEAN>(p, W, idx, info2, frame, succ);
        if (ov) {
          report_min(&p.ctr->viol_trap, (idx << 20) | (2ULL << 16) | (unsigned)((ov - 1) & 0xFFFF));
          has = false;
        } else {
          fp = tlag_fingerprint(succ, W);
        }
      }
      if (MODE == 0) {
        const bool isnew = has && seen_report(p.ctr, seen_insert(p.table, p.mask, fp));
        const unsigned m = __ballot_sync(0xffffffffu, isnew);
        if (isnew) store_append(p, m, succ, W, (uint32_t)idx, tlag_meta(act, p.rank));
      } else if (has) {
        // route: every successor goes to the send region of its owner (tlag_owner_k: hash of its last packed words)
        route_append(p, succ, W, fp, (int)tlag_owner_k(succ, W, (uint32_t)p.n_ranks, p.owner_words), (uint32_t)idx,
                     tlag_meta(act, p.rank));
      }
      if (st == L_EMIT) { st = L_RUN; pc = rpc; }
    }
    if (active && nsucc == 0 && !trapped && (p.flags & TLAG_F_DEADLOCK_CHECK)) {
      report_min(&p.ctr->viol_deadlock, idx << 20);
      if (exact) atomicExch(&p.ctr->stop, 1ULL);
    }
  }
  warp_add(&p.ctr->generated, gen_local);
}

// ------------------------------------------------------------------ random simulation, interpreter
// Step s.t of a batch: one lane per walk of row t (p.states, walks [0, hi)), the warp-scheduled interpreter of k_wave.
// The invariant program runs first; at its HALT a walk that has not failed and is not at its last state runs Next, in
// which every EMIT is packed and offered to the walk's reservoir pick (no fingerprint, no probe, no append).
template <int FRAME, bool SMEM, bool LEAN>
__global__ void __launch_bounds__(TLAG_BLOCK, TLAG_WAVE_OCC(FRAME, SMEM))
k_sim(DevParams p, SimParams s, unsigned long long hi) {
  if (sim_stopped(s)) return;
  const uint64_t* s_code = vm_stage_code<SMEM>(p);
  const uint64_t* code = p.code;
  int32_t frame[FRAME];
  uint32_t succ[TLAG_MAXW];
  const unsigned lane = threadIdx.x & 31;
  const int W = p.W;
  const bool last = s.t + 1 >= s.depth;
  unsigned long long gen_local = 0;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < hi; base += stride) {
    const unsigned long long idx = base + lane;
    int stat = idx < hi ? s.status[idx] : SIM_ENDED;
    const bool active = stat != SIM_ENDED;
    if (active) vm_load_row(p, W, idx, succ, frame);
    int st, ev = 0;
    int32_t info = 0, info2 = 0;
    uint32_t pc, rpc = 0;
    int phase = p.n_inv > 0 ? 0 : 1;
    st = active && (phase == 0 || !last) ? L_RUN : L_DONE;
    pc = st == L_RUN ? (phase == 0 ? p.entry_inv : p.entry_next) : TLAG_PC_PARKED;
    unsigned nsucc = 0, cnt = 0;
    for (;;) {
      warp_vm<SMEM, LEAN>(code, s_code, p.cpool, frame, pc, rpc, ev, info, info2);
      if (st == L_RUN) {
        if (ev == TLAG_EV_EMIT) { st = L_EMIT; ++nsucc; ++gen_local; }
        else if (ev == TLAG_EV_HALT) {
          if (phase == 0 && !last && stat != SIM_FAILED) { phase = 1; pc = p.entry_next; } else st = L_DONE;
        }
        else if (ev == TLAG_EV_GEN) { ++nsucc; ++gen_local; pc = rpc; }
        else if (ev == TLAG_EV_INVF) {
          if (phase == 0) { report_min(&p.ctr->viol_inv, (idx << 20) | (unsigned)(info & 0xFFFFF)); stat = SIM_FAILED; }
          pc = rpc;
        }
        else if (ev == TLAG_EV_ASSERT) {
          report_min(&p.ctr->viol_assert, (idx << 20) | (unsigned)(info & 0xFFFFF));
          stat = phase == 0 ? SIM_FAILED : (stat == SIM_RUN ? SIM_FAILED_NEXT : stat);
          pc = rpc;
        }
        else {
          report_min(&p.ctr->viol_trap, (idx << 20) | ((unsigned long long)(info & 15) << 16) | (unsigned)(info2 & 0xFFFF));
          st = L_DONE; stat = SIM_FAILED;
        }
      }
      if (__any_sync(0xffffffffu, pc != TLAG_PC_PARKED)) continue;
      if (!__any_sync(0xffffffffu, st == L_EMIT)) break;
      if (st == L_EMIT) {
        const int ov = vm_pack_emit<LEAN>(p, W, idx, info2, frame, succ);
        if (ov) {
          report_min(&p.ctr->viol_trap, (idx << 20) | (2ULL << 16) | (unsigned)((ov - 1) & 0xFFFF));
          stat = SIM_FAILED;
        } else {
          sim_pick(s, idx, cnt++, info, succ, W);
        }
        st = L_RUN; pc = rpc;
      }
    }
    if (active) {
      if (stat != s.status[idx]) s.status[idx] = (uint8_t)stat;
      s.cnt[idx] = cnt;
      if (nsucc) p.succ_flag[idx] = 1;
    }
  }
  warp_add(&p.ctr->generated, gen_local);
}
#endif  // !TLAG_SLICED_INC

// ------------------------------------------------------------------ random simulation, both engines
// Each walk of the batch picks its initial state: the draw for "candidate" 0xFFFFFFFF of step 0, over the distinct
// initial states in the order the caller seeded them.
__global__ void k_sim_init(SimParams s, const uint32_t* __restrict__ init, unsigned long long n_init, int W,
                           unsigned long long n) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = tlag_sim_draw(s.seed, s.first + i, 0, 0xFFFFFFFFu) % n_init;
  for (int c = 0; c < W; ++c) s.hist[i * W + c] = init[k * W + c];
  s.act[i] = -1;
  s.status[i] = SIM_RUN; s.cnt[i] = 0; s.len[i] = 0;
}

// End of step s.t: every walk that ran it has checked one more state.  A walk that failed ends, and so does one at its
// last state, one without successors (a deadlock when that is checked) and one whose successors were none of them
// candidates.  Any error makes this the batch's last step (SimCtl::stopped); the others keep their pick in row t + 1.
__global__ void k_sim_end(DevParams p, SimParams s, unsigned long long n) {
  const unsigned long long stopped = *(volatile unsigned long long*)&s.ctl->stopped;
  if (stopped && stopped != s.t + 1ULL) return;
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long ran = 0;
  if (i < n && s.status[i] != SIM_ENDED) {
    ran = 1;
    s.len[i] = s.t + 1;
    bool err = s.status[i] != SIM_RUN, more = false;
    if (!err && s.t + 1 < s.depth) {
      if (!p.succ_flag[i]) {
        if (s.flags & TLAG_F_DEADLOCK_CHECK) { report_min(&p.ctr->viol_deadlock, i << 20); err = true; }
      } else {
        more = s.cnt[i] != 0;
      }
    }
    if (err) atomicExch(&s.ctl->stopped, s.t + 1ULL);
    s.status[i] = more ? SIM_RUN : SIM_ENDED;
    s.cnt[i] = 0; p.succ_flag[i] = 0;
  }
  warp_add(&s.ctl->checked, ran);
}

// XOR and SUM over the batch's behaviours: one term per state checked, from its fingerprint, walk, step and action
__global__ void k_sim_digest(SimParams s, int W, unsigned long long n, unsigned long long* out2) {
  unsigned long long x = 0, sm = 0;
  const unsigned long long total = n * s.depth;
  for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < total;
       k += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long i = k % n, t = k / n;
    if (t >= s.len[i]) continue;
    const unsigned long long v = tlag_sim_term(tlag_fingerprint(s.hist + (t * s.B + i) * W, W), s.first + i, (uint32_t)t,
                                               s.act[t * s.B + i]);
    x ^= v; sm += v;
  }
  warp_digest(out2, x, sm);
}

#if !defined(TLAG_SL_SIM)
// ------------------------------------------------------------------ state graph (tlag_build_graph), both engines
// The index pass maps each seen-set slot to the store row whose fingerprint it holds; the edge pass runs Next on a chunk
// of expanded rows with the interpreter and finds each successor's row by a read-only probe of the same seen-set.
struct GraphCtl {
  unsigned long long n;             // edges the chunk produced (counted past the buffer's capacity)
  unsigned long long missing;       // a fingerprint without a slot, or a successor that is not stored
  unsigned long long bad;           // the edge pass met an evaluation trap, a pack overflow or an action id out of range
};

struct GraphParams {
  const uint32_t* row_of_slot;      // seen-set slot -> store row
  unsigned long long first;         // first row of the chunk
  unsigned long long* keys;         // the chunk's edges: (s - first) << (32 + abits) | t << abits | a
  unsigned long long cap;
  unsigned abits;
  GraphCtl* ctl;
};

// the slot of fp in the seen-set, or -1 when it is not there (read-only: the probe sequence of seen_insert)
__device__ __forceinline__ long long seen_find(const unsigned long long* __restrict__ table, unsigned long long mask,
                                               unsigned long long fp) {
  unsigned long long i = fp & mask;
  for (unsigned long long probes = 0; probes <= mask; ++probes, i = (i + 1) & mask) {
    const unsigned long long v = table[i];
    if (v == fp) return (long long)i;
    if (v == 0ULL) return -1;
  }
  return -1;
}

__global__ void k_graph_index(DevParams p, unsigned long long n, uint32_t* __restrict__ row_of_slot, GraphCtl* ctl) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t w[TLAG_MAXW];
  for (int k = 0; k < p.W; ++k) w[k] = p.states[i * (unsigned long long)p.W + k];
  const long long slot = seen_find(p.table, p.mask, tlag_fingerprint(w, p.W));
  if (slot < 0) atomicExch(&ctl->missing, 1ULL);
  else row_of_slot[slot] = (uint32_t)i;
}

// Edges out of rows [g.first, hi): one lane per row, the warp-scheduled interpreter of k_wave on Next only (no invariant,
// nothing reported to the search's counters).  Each EMIT is packed, fingerprinted and looked up; a successor other than
// the row itself is appended to the chunk's buffer, one atomic per warp.
template <int FRAME, bool SMEM, bool LEAN>
__global__ void __launch_bounds__(TLAG_BLOCK, TLAG_WAVE_OCC(FRAME, SMEM))
k_graph(DevParams p, GraphParams g, unsigned long long hi) {
  const uint64_t* s_code = vm_stage_code<SMEM>(p);
  const uint64_t* code = p.code;
  int32_t frame[FRAME];
  uint32_t succ[TLAG_MAXW];
  const unsigned lane = threadIdx.x & 31;
  const int W = p.W;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long base = g.first + (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < hi;
       base += stride) {
    const unsigned long long idx = base + lane;
    const bool active = idx < hi;
    if (active) vm_load_row(p, W, idx, succ, frame);
    int st = active ? L_RUN : L_DONE, ev = 0;
    int32_t info = 0, info2 = 0;
    uint32_t pc = active ? p.entry_next : TLAG_PC_PARKED, rpc = 0;
    for (;;) {
      warp_vm<SMEM, LEAN>(code, s_code, p.cpool, frame, pc, rpc, ev, info, info2);
      if (st == L_RUN) {
        if (ev == TLAG_EV_EMIT) st = L_EMIT;
        else if (ev == TLAG_EV_HALT) st = L_DONE;
        else if (ev == TLAG_EV_GEN || ev == TLAG_EV_INVF || ev == TLAG_EV_ASSERT) pc = rpc;
        else { atomicExch(&g.ctl->bad, 1ULL); st = L_DONE; }
      }
      if (__any_sync(0xffffffffu, pc != TLAG_PC_PARKED)) continue;
      if (!__any_sync(0xffffffffu, st == L_EMIT)) break;
      bool keep = false;
      unsigned long long key = 0;
      if (st == L_EMIT) {
        const int ov = vm_pack_emit<LEAN>(p, W, idx, info2, frame, succ);
        if (ov || info < 0 || ((unsigned long long)info >> g.abits) != 0) {
          atomicExch(&g.ctl->bad, 1ULL);
        } else {
          const long long slot = seen_find(p.table, p.mask, tlag_fingerprint(succ, W));
          if (slot < 0) {
            atomicExch(&g.ctl->missing, 1ULL);
          } else {
            const unsigned long long t = g.row_of_slot[slot];
            keep = t != idx;
            key = ((idx - g.first) << (32 + g.abits)) | (t << g.abits) | (unsigned long long)info;
          }
        }
        st = L_RUN; pc = rpc;
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int leader = __ffs((int)m) - 1;
        unsigned long long pos = 0;
        if ((int)lane == leader) pos = atomicAdd(&g.ctl->n, (unsigned long long)__popc(m));
        pos = __shfl_sync(m, pos, leader) + (unsigned long long)__popc(m & lanemask_lt());
        if (pos < g.cap) g.keys[pos] = key;
      }
    }
  }
}

// Rows [0, rows] of a chunk whose sorted distinct edges are keys[0, n): off[r] = base + the first edge of row r
__global__ void k_graph_rows(const unsigned long long* __restrict__ keys, unsigned long long n, unsigned long long rows,
                             unsigned shift, unsigned long long base, unsigned long long* __restrict__ off) {
  const unsigned long long r = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > rows) return;
  unsigned long long lo = 0, hi = n;
  while (lo < hi) {
    const unsigned long long mid = (lo + hi) >> 1;
    if ((keys[mid] >> shift) < r) lo = mid + 1; else hi = mid;
  }
  off[r] = base + lo;
}

// edge i of the chunk -> its destination row and action id in the resident CSR
__global__ void k_graph_split(const unsigned long long* __restrict__ keys, unsigned long long n, unsigned abits,
                              uint32_t* __restrict__ dst, uint32_t* __restrict__ act) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  dst[i] = (uint32_t)(k >> abits);
  act[i] = (uint32_t)(k & ((1ULL << abits) - 1));
}

__global__ void k_fill_u64(unsigned long long* __restrict__ a, unsigned long long n, unsigned long long v) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// ---- liveness labels (include/tlag.h: tlag_label_graph)
struct LabelParams {
  const uint64_t* code; const int32_t* cpool;   // the label image
  uint32_t entry;                                // its state or edge program
  uint32_t all;                                  // the program's bits
  const unsigned long long* off; const uint32_t* dst;   // the resident CSR (edge labels)
  unsigned long long n;                          // lanes: rows (state labels) or edges
  unsigned long long rows;                       // rows of the CSR
  uint32_t* out;                                 // one word per lane: bit j = predicate j holds
  unsigned long long* bad;                       // a predicate trapped
};

// One lane per stored row (EDGES false) or per edge of the resident CSR (EDGES true: its source row unpacked to the current
// frame, its destination to the primed one), on the warp-scheduled interpreter of k_wave.  The program raises INVF j for
// each predicate j that is false; the lane's word gets the others.
template <int FRAME, bool EDGES>
__global__ void __launch_bounds__(TLAG_BLOCK, TLAG_WAVE_OCC(FRAME, false))
k_label(DevParams p, LabelParams l) {
  int32_t frame[FRAME];
  uint32_t w[TLAG_MAXW];
  const unsigned lane = threadIdx.x & 31;
  const int W = p.W;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < l.n;
       base += stride) {
    const unsigned long long i = base + lane;
    const bool active = i < l.n;
    if (active) {
      unsigned long long s = i;
      if (EDGES) {                       // the row whose edges hold edge i: the last s with off[s] <= i
        unsigned long long lo = 0, hi = l.rows - 1;
        while (lo < hi) {
          const unsigned long long mid = (lo + hi + 1) >> 1;
          if (l.off[mid] <= i) lo = mid; else hi = mid - 1;
        }
        s = lo;
      }
      vm_load_row(p, W, s, w, frame);
      if (EDGES) {
        const uint32_t* t = p.states + (unsigned long long)l.dst[i] * W;
        for (int k = 0; k < W; ++k) w[k] = t[k];
        tlag_unpack(p.layout, p.n_slots, w, frame + p.p_off);
      }
    }
    uint32_t fails = 0;
    int ev = 0;
    int32_t info = 0, info2 = 0;
    bool run = active;
    uint32_t pc = active ? l.entry : TLAG_PC_PARKED, rpc = 0;
    for (;;) {
      warp_vm<false, false>(l.code, nullptr, l.cpool, frame, pc, rpc, ev, info, info2);
      if (run) {
        if (ev == TLAG_EV_INVF) {
          fails |= 1u << (info & 31);
          pc = rpc;
        } else {
          if (ev != TLAG_EV_HALT) atomicExch(l.bad, 1ULL);
          run = false;
        }
      }
      if (!__any_sync(0xffffffffu, pc != TLAG_PC_PARKED)) break;
    }
    if (active) l.out[i] = ~fails & l.all;
  }
}

// state bits derived from each row's out-edges: en[b] (< 32) is set when some edge has edge bit b (ENABLED <<A_b>>_v),
// nen[b] when none has
struct EnabledMap { uint8_t en[32], nen[32]; };

__global__ void k_label_enabled(const unsigned long long* __restrict__ off, const uint32_t* __restrict__ elab,
                                unsigned long long n, EnabledMap m, uint32_t* __restrict__ slab) {
  for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < n;
       s += (unsigned long long)gridDim.x * blockDim.x) {
    uint32_t x = 0;
    for (unsigned long long j = off[s], e = off[s + 1]; j < e; ++j) x |= elab[j];
    uint32_t word = slab[s];
    for (int b = 0; b < 32; ++b) {
      if (m.en[b] < 32 && ((x >> b) & 1u)) word |= 1u << m.en[b];
      if (m.nen[b] < 32 && !((x >> b) & 1u)) word |= 1u << m.nen[b];
    }
    slab[s] = word;
  }
}

// XOR and SUM of tlag_edge_term over the edges out of rows [0, n)
__global__ void k_graph_digest(DevParams p, const unsigned long long* __restrict__ off, const uint32_t* __restrict__ dst,
                               const uint32_t* __restrict__ act, unsigned long long n, unsigned long long* out2) {
  unsigned long long x = 0, sm = 0;
  uint32_t w[TLAG_MAXW];
  for (unsigned long long s = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; s < n;
       s += (unsigned long long)gridDim.x * blockDim.x) {
    if (off[s] == off[s + 1]) continue;
    for (int k = 0; k < p.W; ++k) w[k] = p.states[s * (unsigned long long)p.W + k];
    const unsigned long long fs = tlag_fingerprint(w, p.W);
    for (unsigned long long j = off[s]; j < off[s + 1]; ++j) {
      const unsigned long long t = dst[j];
      for (int k = 0; k < p.W; ++k) w[k] = p.states[t * (unsigned long long)p.W + k];
      const unsigned long long v = tlag_edge_term(fs, tlag_fingerprint(w, p.W), (int32_t)act[j]);
      x ^= v; sm += v;
    }
  }
  warp_digest(out2, x, sm);
}
#endif  // !TLAG_SL_SIM

// ------------------------------------------------------------------ K1 alone: fingerprint + probe/insert
// One thread per candidate state, word by word: the inputs the staged form does not take (W = 1, or a batch that is not
// 16-byte aligned).
__global__ void __launch_bounds__(256) k_probe(const uint32_t* __restrict__ states, unsigned long long n, int W,
                                               unsigned long long* table, unsigned long long mask,
                                               uint8_t* __restrict__ is_new, Counters* ctr) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* src = states + i * (unsigned long long)W;
  uint64_t h = tlag_fp_init(W);
  int k = 0;
  for (; k + 1 < W; k += 2) h = tlag_fp_pair(h, __ldg(src + k), __ldg(src + k + 1));
  if (k < W) h = tlag_fp_tail(h, __ldg(src + k));
  is_new[i] = (uint8_t)seen_report(ctr, seen_insert(table, mask, tlag_fp_final(h, W)));
}

// K1, coalesced form: a CTA of 256 threads owns 256 consecutive candidates = one contiguous span of
// 256*W words.  The span is fetched with fully coalesced 128-bit loads (every 32-byte sector is read
// exactly once; ncu on the strided v0 showed 2.4x DRAM read amplification from L1 thrash), staged in
// shared memory with an odd row stride (W|1 words -> conflict-free), then each thread fingerprints its
// own row and probes the table.
__global__ void __launch_bounds__(256) k_probe_staged(const uint32_t* __restrict__ states, unsigned long long n, int W,
                                                      unsigned long long* table, unsigned long long mask,
                                                      uint8_t* __restrict__ is_new, Counters* ctr) {
  extern __shared__ uint32_t s_rows[];
  const int stride = W | 1;
  const unsigned ROWS = 256;
  const unsigned long long base = (unsigned long long)blockIdx.x * ROWS;
  const unsigned nst = (unsigned)((n - base) < (unsigned long long)ROWS ? (n - base) : (unsigned long long)ROWS);
  const uint32_t* g = states + base * (unsigned long long)W;
  const unsigned total = nst * (unsigned)W;          // words in this CTA's span
  const unsigned total4 = total >> 2;
  const uint4* g4 = reinterpret_cast<const uint4*>(g);
  for (unsigned i = threadIdx.x; i < total4; i += 256) {
    const uint4 v = __ldcs(g4 + i);                  // streaming: each word is used once
    unsigned wi = i << 2;
    unsigned row = wi / (unsigned)W, col = wi - row * (unsigned)W;
    s_rows[row * stride + col] = v.x; if (++col == (unsigned)W) { col = 0; ++row; }
    s_rows[row * stride + col] = v.y; if (++col == (unsigned)W) { col = 0; ++row; }
    s_rows[row * stride + col] = v.z; if (++col == (unsigned)W) { col = 0; ++row; }
    s_rows[row * stride + col] = v.w;
  }
  for (unsigned wi = (total4 << 2) + threadIdx.x; wi < total; wi += 256) {   // ragged tail (< 4 words)
    const unsigned row = wi / (unsigned)W, col = wi - row * (unsigned)W;
    s_rows[row * stride + col] = g[wi];
  }
  __syncthreads();
  if (threadIdx.x >= nst) return;
  const uint32_t* r = s_rows + threadIdx.x * stride;
  uint64_t h = tlag_fp_init(W);
  int k = 0;
  for (; k + 1 < W; k += 2) h = tlag_fp_pair(h, r[k], r[k + 1]);
  if (k < W) h = tlag_fp_tail(h, r[k]);
  const unsigned long long fp = tlag_fp_final(h, W);
  is_new[base + threadIdx.x] = (uint8_t)seen_report(ctr, seen_insert_at(table, mask, fp, __ldcv(&table[fp & mask])));
}

// One routed record (W state words, parent, meta) into this rank's shard: fingerprint, probe, append.  Every lane of the
// warp calls it; `has` says whether the lane holds a record.  Read through L2: the inbox of k_insert_inbox is written by
// peers over NVLink.
__device__ __forceinline__ void insert_record(const DevParams& p, const uint32_t* rec, bool has) {
  const int W = p.W;
  uint32_t w[TLAG_MAXW];
  unsigned long long fp = 0;
  if (has) {
    for (int k = 0; k < W; ++k) w[k] = __ldcg(rec + k);
    fp = tlag_fingerprint(w, W);
  }
  const bool isnew = has && seen_report(p.ctr, seen_insert(p.table, p.mask, fp));
  const unsigned m = __ballot_sync(0xffffffffu, isnew);
  if (isnew) store_append(p, m, w, W, __ldcg(rec + W), __ldcg(rec + W + 1));
}

// insert routed records into this rank's shard
__global__ void __launch_bounds__(256) k_insert_records(DevParams p, const uint32_t* __restrict__ rec,
                                                        unsigned long long n) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  insert_record(p, rec + i * (unsigned long long)(p.W + 2), i < n);
}

// ------------------------------------------------------------------ peer-memory exchange (multi-GPU)
// One process per GPU; the state space is partitioned by tlag_owner().  Instead of handing the per-owner send regions to
// NCCL (two all_to_alls and three host round trips per chunk in round 1), every rank maps every other rank's INBOX with
// CUDA IPC and the exchange is device code over NVLink / NVSwitch:
//   k_push          copies this rank's send region for owner d into d's inbox (16-byte stores over NVLink), then
//                   publishes {count, seq} in d's memory with a system-scope release;
//   k_insert_inbox  waits (acquire) until every source has published chunk `seq`, inserts the records into this
//                   rank's seen-set shard / state store (the next frontier), then acknowledges the chunk in the
//                   sources' memory so that they may reuse the buffer.
// Inboxes are double-buffered by chunk parity; a whole BFS level is enqueued on the engine's stream (expand kernels,
// push, insert per chunk) and the host synchronises once per level for the termination all-reduce.
// grid: (blocks_per_dst, n_ranks).  Copies min(send_count[dst], region_cap) records to dst's inbox.
__global__ void __launch_bounds__(256) k_push(P2PParams q, const Counters* ctr, unsigned long long seq) {
  const int dst = blockIdx.y;
  __shared__ int s_last;
  P2PMeta* mine_at_dst = q.peer_meta[dst] + q.rank;
  if (threadIdx.x == 0 && seq > 2) {
    // the buffer (seq & 1) at dst was last used for my chunk seq - 2: wait until dst has consumed it
    const unsigned long long* ack = &q.meta[dst].ack;
    while (ld_acquire_sys(ack) + 2 < seq) __nanosleep(200);
  }
  __syncthreads();
  unsigned long long n = ctr->send_count[dst];
  if (n > q.region_cap) n = q.region_cap;
  const unsigned long long words = n * (unsigned long long)q.rec_words;
  const uint32_t* src = q.send + (unsigned long long)dst * q.region_cap * q.rec_words;
  uint32_t* out = q.peer_inbox[dst] + (((seq & 1ULL) * q.n_ranks + q.rank) * q.inbox_cap) * q.rec_words;
  const unsigned long long w4 = words >> 2;
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* o4 = reinterpret_cast<uint4*>(out);
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < w4;
       i += (unsigned long long)gridDim.x * blockDim.x)
    o4[i] = s4[i];
  if (blockIdx.x == 0)
    for (unsigned long long i = (w4 << 2) + threadIdx.x; i < words; i += blockDim.x) out[i] = src[i];
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) s_last = (atomicAdd(&q.tickets[dst], 1u) == gridDim.x - 1);
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    q.tickets[dst] = 0;
    __threadfence_system();
    *(volatile unsigned long long*)&mine_at_dst->count[seq & 1ULL] = n;
    __threadfence_system();
    st_release_sys(&mine_at_dst->seq[seq & 1ULL], seq);
  }
}

// Inserts every source's records of chunk `seq` (grid-stride over sources and records, whole warps).
__global__ void __launch_bounds__(256) k_insert_inbox(DevParams p, P2PParams q, unsigned long long seq) {
  __shared__ unsigned long long s_n;
  __shared__ int s_last;
  for (int src = 0; src < q.n_ranks; ++src) {
    if (threadIdx.x == 0) {
      const P2PMeta* m = &q.meta[src];
      while (ld_acquire_sys(&m->seq[seq & 1ULL]) != seq) __nanosleep(200);
      s_n = *(volatile const unsigned long long*)&m->count[seq & 1ULL];
    }
    __syncthreads();
    const unsigned long long n = s_n;
    const uint32_t* rec = q.inbox + (((seq & 1ULL) * q.n_ranks + src) * q.inbox_cap) * q.rec_words;
    const unsigned long long n32 = (n + 31ULL) & ~31ULL;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n32;
         i += (unsigned long long)gridDim.x * blockDim.x)
      insert_record(p, rec + i * (unsigned long long)(p.W + 2), i < n);
    __syncthreads();
  }
  // every block is done with every source: the last one acknowledges the chunk to all sources
  __threadfence();
  if (threadIdx.x == 0) s_last = (atomicAdd(&q.tickets[16], 1u) == gridDim.x - 1);
  __syncthreads();
  if (s_last && threadIdx.x < (unsigned)q.n_ranks) {
    if (threadIdx.x == 0) q.tickets[16] = 0;
    __threadfence_system();
    st_release_sys(&(q.peer_meta[threadIdx.x] + q.rank)->ack, seq);
  }
}

// checksum of checksums over the state store: XOR and SUM (mod 2^64) of all fingerprints
__global__ void k_digest(DevParams p, unsigned long long n, unsigned long long* out2) {
  unsigned long long x = 0, sm = 0;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    uint32_t w[TLAG_MAXW];
    for (int k = 0; k < p.W; ++k) w[k] = p.states[i * (unsigned long long)p.W + k];
    const unsigned long long fp = tlag_fingerprint(w, p.W);
    x ^= fp; sm += fp;
  }
  warp_digest(out2, x, sm);
}

// ---- frontier clustering -----------------------------------------------------------------------
// The warp-scheduled interpreter executes the union of its 32 lanes' paths, so its efficiency is
// (mean path length) / (union length).  States that agree on the tail of the packed vector (the last
// variables, for the Paxos models the high bits of the msgs bitset) follow similar paths: measured on
// a 4096-state window of MCPaxos3_b3 level 14, lane utilisation is 0.35 in discovery order, 0.31 in random
// order and 0.54 when sorted by the last packed word.  Each newly discovered level is therefore reordered by a
// 64-bit key of its last two words, key = w[W-1] << 32 | w[W-2], stably, so equal keys keep their discovery order
// (an unstable order within a key costs the next wave time: 8 - 10 % on MCssi_4x3, 1 % on MCPaxos3_b4).
//
// A level's new rows are appended to a discovery buffer of records [W words, parent, meta] (DevParams::app), and the
// pass moves each record once, straight to its final row in the store.  A level holds few distinct keys (MCPaxos3_b4:
// 1 K - 100 K in levels of up to millions of states; Raft and SSI a few hundred), so the level is sorted on the key's
// dense rank among the level's distinct keys, not on the key itself: the same permutation, on 32-bit keys of
// ceil(log2(distinct)) bits -- 2 or 3 radix passes instead of 8 passes over 64-bit keys.  The pass:
//   k_rset_insert     puts each record's key into a small open-addressed set (the rank set, L2-resident at these sizes)
//                     and writes the key's slot;
//   k_rset_list, a sort of the distinct keys, k_rset_rank   give every slot its key's rank;
//   k_rank_states     turns each record's slot into its rank and writes its index, then a stable radix sort of
//                     (rank, index) over the rank's bits;
//   k_cluster_gather  writes record idx[i] to store row first + i, a warp per 32 rows, stores coalesced.
#define TLAG_RSET_EMPTY 0xFFFFFFFFFFFFFFFFull   /* empty slot; a key equal to it is counted aside (it is the largest) */
struct RankSetCtl { unsigned n, full, has_max, n_list; };
#define TLAG_CLUSTER_ILP 4   /* words each lane loads before it stores them (gather): latency-bound otherwise */

__device__ __forceinline__ unsigned long long rset_hash(unsigned long long k) {   // splitmix64 finaliser
  k ^= k >> 30; k *= 0xbf58476d1ce4e5b9ull; k ^= k >> 27; k *= 0x94d049bb133111ebull; return k ^ (k >> 31);
}

// The slot of `key` in the rank set (mask + 1 slots; slot mask + 1 for the TLAG_RSET_EMPTY key), inserted if absent; a
// set past half full (or full) is flagged for the host to grow and refill.
__device__ __forceinline__ unsigned long long rset_slot(unsigned long long* table, unsigned long long mask, RankSetCtl* ctl,
                                                        unsigned long long key) {
  if (key == TLAG_RSET_EMPTY) { if (!*(volatile unsigned*)&ctl->has_max) ctl->has_max = 1; return mask + 1; }
  unsigned long long h = rset_hash(key) & mask;
  for (unsigned long long probes = 0; probes <= mask; ++probes, h = (h + 1) & mask) {
    unsigned long long v = __ldcg(table + h);
    if (v == key) return h;
    if (v == TLAG_RSET_EMPTY) {
      if (*(volatile unsigned*)&ctl->full) return 0;
      v = atomicCAS(table + h, TLAG_RSET_EMPTY, key);
      if (v == TLAG_RSET_EMPTY) {                 // new distinct key
        if ((unsigned long long)atomicAdd(&ctl->n, 1u) + 1 > (mask + 1) / 2) ctl->full = 1;
        return h;
      }
      if (v == key) return h;
    }
  }
  ctl->full = 1;
  return 0;
}

// record i of the discovery buffer -> its key's slot; the key is the record's words W-1, W-2 (next to parent and meta)
__global__ void k_rset_insert(const uint32_t* __restrict__ rec, unsigned long long n, int W, unsigned long long* table,
                              unsigned long long mask, RankSetCtl* ctl, uint32_t* __restrict__ slot_of) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* r = rec + i * (unsigned long long)(W + 2);
  const unsigned long long key = ((unsigned long long)r[W - 1] << 32) | (W >= 2 ? r[W - 2] : 0u);
  // lanes of a warp often share a key (successors of like states): one lane per distinct key probes the set
  const unsigned peers = __match_any_sync(__activemask(), key);
  const int leader = __ffs(peers) - 1;
  unsigned long long h = 0;
  if ((int)(threadIdx.x & 31) == leader) h = rset_slot(table, mask, ctl, key);
  slot_of[i] = (uint32_t)__shfl_sync(peers, h, leader);
}

__global__ void k_rset_list(const unsigned long long* __restrict__ table, unsigned long long slots,
                            unsigned long long* __restrict__ list, RankSetCtl* ctl) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= slots) return;
  const unsigned long long v = table[i];
  if (v != TLAG_RSET_EMPTY) list[atomicAdd(&ctl->n_list, 1u)] = v;
}

__device__ __forceinline__ unsigned long long rset_find(const unsigned long long* __restrict__ table,
                                                        unsigned long long mask, unsigned long long key) {
  unsigned long long h = rset_hash(key) & mask;
  while (table[h] != key) h = (h + 1) & mask;     // every key looked up was inserted
  return h;
}

// sorted[r] = the distinct key of rank r (r < n); the TLAG_RSET_EMPTY key, the largest, has rank n (slot mask + 1)
__global__ void k_rset_rank(const unsigned long long* __restrict__ sorted, unsigned n,
                            const unsigned long long* __restrict__ table, unsigned long long mask, uint32_t* __restrict__ rank) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rank[rset_find(table, mask, sorted[i])] = i;
  else if (i == n) rank[mask + 1] = n;
}

// Entry i of the sort: the rank of record i and i itself (rank_out may be `slot`: each thread reads its own entry
// before it writes it).
__global__ void k_rank_states(const uint32_t* slot, unsigned long long n, const uint32_t* __restrict__ rank,
                              uint32_t* rank_out, uint32_t* __restrict__ idx) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t r = __ldg(rank + slot[i]);
  rank_out[i] = r;
  idx[i] = (uint32_t)i;
}

// Store row first + i <- record idx[i] of the discovery buffer (st, parent and meta point at row first; without idx,
// record i: discovery order).  A warp writes 32 consecutive rows: coalesced stores.
__global__ void k_cluster_gather(const uint32_t* __restrict__ rec, const uint32_t* __restrict__ idx,
                                 unsigned long long n, int W, uint32_t* __restrict__ st,
                                 uint32_t* __restrict__ parent, uint32_t* __restrict__ meta) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long r0 = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull;
  if (r0 >= n) return;
  const unsigned rows = n - r0 < 32 ? (unsigned)(n - r0) : 32u;
  const unsigned long long j = lane < rows ? (idx ? (unsigned long long)__ldcs(idx + r0 + lane) : r0 + lane) : 0;
  const uint32_t* mine = rec + j * (unsigned long long)(W + 2);
  const uint32_t par = lane < rows ? mine[W] : 0, met = lane < rows ? mine[W + 1] : 0;
  uint32_t* dst = st + r0 * (unsigned long long)W;
  const unsigned words = rows * (unsigned)W;
  for (unsigned base = 0; base < words; base += 32 * TLAG_CLUSTER_ILP) {   // warp-uniform trip count: the shuffle has every lane
    uint32_t v[TLAG_CLUSTER_ILP];
#pragma unroll
    for (int u = 0; u < TLAG_CLUSTER_ILP; ++u) {
      const unsigned k = base + u * 32 + lane, r = k / (unsigned)W, c = k - r * (unsigned)W;
      const unsigned long long jr = __shfl_sync(0xffffffffu, j, r & 31);
      v[u] = k < words ? rec[jr * (unsigned long long)(W + 2) + c] : 0;
    }
#pragma unroll
    for (int u = 0; u < TLAG_CLUSTER_ILP; ++u) {
      const unsigned k = base + u * 32 + lane;
      if (k < words) dst[k] = v[u];
    }
  }
  if (lane < rows) {
    parent[r0 + lane] = par;
    meta[r0 + lane] = met;
  }
}

// rebuild the table from the state store after growing it
__global__ void k_rehash(DevParams p, unsigned long long n) {
  const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t w[TLAG_MAXW];
  for (int k = 0; k < p.W; ++k) w[k] = p.states[i * (unsigned long long)p.W + k];
  seen_insert(p.table, p.mask, tlag_fingerprint(w, p.W));
}

// Exchange buffers outlive the engine that created them: allocating an 8 GB inbox, exporting it and mapping seven peers'
// inboxes costs seconds, and a host process that checks one model after another (bench.py's end-to-end leg does) would
// pay it per job.  tlag_destroy parks the buffers of a p2p engine here; the next engine of the same shape (device, ranks,
// record size, capacity) adopts them -- same IPC handle, peers' mappings still valid, chunk numbering continued (every
// rank has run the same number of chunks, so the inbox protocol needs no reset).
struct P2PParked {
  int device, n_ranks, rank, rec_words; uint64_t cap;
  void* d_p2p; uint64_t bytes; uint32_t* d_send; unsigned int* d_tickets;
  void* peer_base[16]; uint8_t peer_handle[16][64]; bool peer_ok[16];
  unsigned long long seq; bool in_use;
};
static std::vector<P2PParked> g_p2p_parked;

// ------------------------------------------------------------------ host side
// Big device buffers (state store, parent / meta, seen-set, sort scratch, routed-fingerprint cache, send regions) come
// from the device's stream-ordered memory pool with its release threshold lifted: a buffer freed by a growth step or by
// tlag_destroy stays in the pool, and the next allocation of that size -- the next growth step, the next engine of a
// long-lived host process -- is served without going back to the driver.  cudaMalloc / cudaFree of multi-GB buffers
// cost tens of milliseconds each, and a fresh engine performs a dozen of them while its store and table grow (the
// end-to-end leg of bench.py creates and destroys an engine per job).  The peer-memory inbox stays on cudaMalloc: CUDA
// IPC cannot export pool memory.
// On an 80 GB H100 the buffers a growing job has outgrown (the previous store and seen-set generations) can hold a third
// of the device: when free memory runs short they are handed back to the driver before the next allocation.  This runs
// only when an allocation fails or a store growth step finds too little free memory, and it empties the device's
// default pool for every engine of the process on that device (their buffers in use stay; only freed ones go).
static void trim_pool(tlag_engine* e) {
  cudaMemPool_t pool;
  cudaStreamSynchronize(e->stream);
  if (cudaDeviceGetDefaultMemPool(&pool, e->m.device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  cudaGetLastError();
}
static cudaError_t dmalloc(tlag_engine* e, void* pp, size_t bytes, bool trim = true) {
  cudaError_t r = cudaMallocAsync((void**)pp, bytes, e->stream);
  if (r == cudaErrorMemoryAllocation && trim) {
    cudaGetLastError();
    trim_pool(e);
    r = cudaMallocAsync((void**)pp, bytes, e->stream);
  }
  return r;
}
static void dfree(tlag_engine* e, void* p) {
  if (p) cudaFreeAsync(p, e->stream);
}

// DevParams::app at the store, or with the level open at its discovery buffer (row hi = record 0).  The store's append
// limit is its capacity; an open level's is set by open_level.
static void point_appends(tlag_engine* e) {
  DevParams& p = e->p;
  const unsigned W = (unsigned)e->m.words_per_state;
  if (e->disc_open) {
    const uintptr_t row0 = (uintptr_t)e->d_disc - (uintptr_t)(e->hi * (W + 2) * 4);   // never dereferenced below row hi
    p.app = (uint32_t*)row0; p.app_parent = (uint32_t*)(row0 + W * 4); p.app_meta = (uint32_t*)(row0 + (W + 1) * 4);
    p.app_stride = p.pm_stride = W + 2;
  } else {
    p.app = p.states; p.app_parent = p.parent; p.app_meta = p.meta;
    p.app_stride = W; p.pm_stride = 1;
    p.cap_states = e->cap_states;
  }
}

// Lets kernel fn take `bytes` of dynamic shared memory (past the default 48 KB it has to opt in)
template <class K>
static cudaError_t allow_smem(K fn, size_t bytes) {
  return bytes > 48 * 1024 ? cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) : cudaSuccess;
}

// The dynamic shared memory of an interpreter kernel: the program, when the engine's variant runs it from there
static inline size_t vm_smem(const tlag_engine* e) { return e->p.code_in_smem ? (size_t)e->p.code_len * 8 : 0; }

// Interpreter kernel fn over `rows` rows, one lane per row (k_wave: a warp per 32-row chunk, the same count), on a
// persistent grid: at most one resident wave of CTAs, at least one CTA.  launch_vm gives it the engine's program in
// shared memory when the engine's variant runs it from there; launch_vm_smem takes the size
template <class... P, class... A>
static cudaError_t launch_vm_smem(tlag_engine* e, size_t smem, void (*fn)(P...), uint64_t rows, const A&... args) {
  const cudaError_t r = allow_smem(fn, smem);
  if (r != cudaSuccess) return r;
  int occ = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, TLAG_BLOCK, smem) != cudaSuccess || occ < 1) occ = 1;
  uint64_t blocks = (rows + TLAG_BLOCK - 1) / TLAG_BLOCK;
  if (blocks > (uint64_t)e->sm_count * (uint64_t)occ) blocks = (uint64_t)e->sm_count * (uint64_t)occ;
  if (blocks == 0) blocks = 1;
  fn<<<(unsigned)blocks, TLAG_BLOCK, smem, e->stream>>>(args...);
  e->launches++;
  return cudaGetLastError();
}
template <class... P, class... A>
static cudaError_t launch_vm(tlag_engine* e, void (*fn)(P...), uint64_t rows, const A&... args) {
  return launch_vm_smem(e, vm_smem(e), fn, rows, args...);
}

// The engine's variant of an interpreter kernel template: its frame class, the program in shared memory or not, and up to
// 512 words the lean interpreter for a program without the extension ops.  kernel(frame, smem, lean) names the template's
// instantiation for one variant (each argument a std::integral_constant), so each template gets the 24 variants.
template <int FRAME, class K>
static auto vm_variant_of(const tlag_engine* e, K kernel) {
  using F = std::integral_constant<int, FRAME>;
  using Y = std::true_type;
  using N = std::false_type;
  const bool sm = e->p.code_in_smem != 0;
  if constexpr (FRAME <= 512)
    if (!e->uses_ext) return sm ? kernel(F{}, Y{}, Y{}) : kernel(F{}, N{}, Y{});
  return sm ? kernel(F{}, Y{}, N{}) : kernel(F{}, N{}, N{});
}

template <class K>
static auto vm_variant(const tlag_engine* e, K kernel) {
  switch (e->frame_class) {
    case 64: return vm_variant_of<64>(e, kernel);
    case 128: return vm_variant_of<128>(e, kernel);
    case 256: return vm_variant_of<256>(e, kernel);
    case 512: return vm_variant_of<512>(e, kernel);
    case 1024: return vm_variant_of<1024>(e, kernel);
    case 2048: return vm_variant_of<2048>(e, kernel);
    case 4096: return vm_variant_of<4096>(e, kernel);
    // 8192 words = 32 KB of local memory per thread (SSI at 4 transactions x 3 keys needs 6.9 K words)
    default: return vm_variant_of<8192>(e, kernel);
  }
}

#ifdef TLAG_SLICED_INC
// One BFS level (or one chunk of it, route mode) = the invariant kernels, the kernels of the slices of Next, and the
// deadlock scan, back to back on the engine's stream.
template <int MODE>
static cudaError_t launch_wave(tlag_engine* e, uint64_t lo, uint64_t hi) {
  const uint64_t n = hi - lo;
  if (n == 0) return cudaSuccess;
  const bool dl = (e->p.flags & TLAG_F_DEADLOCK_CHECK) != 0;
  if (dl) {
    if (n > e->succ_cap) {
      dfree(e, e->d_succ); e->d_succ = nullptr; e->succ_cap = 0;
      uint64_t cap = n + n / 2 + 4096;
      cudaError_t r = dmalloc(e, &e->d_succ, cap);
      if (r != cudaSuccess) return r;
      e->succ_cap = cap;
    }
    cudaError_t r = cudaMemsetAsync(e->d_succ, 0, n, e->stream);
    if (r != cudaSuccess) return r;
  }
  e->p.succ_flag = dl ? e->d_succ : nullptr;
  e->p.route = MODE;
  const unsigned blocks = sl_blocks(e, n);
  if (e->p.n_inv > 0)
    for (int j = 0; kSlInv[j]; ++j) { kSlInv[j](&e->p, lo, hi, blocks, e->stream); e->launches++; }
  for (int j = 0; kSlNext[j]; ++j) { kSlNext[j](&e->p, lo, hi, blocks, e->stream); e->launches++; }
  if (dl) { k_sl_deadlock<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(e->p, lo, hi); e->launches++; }
  return cudaGetLastError();
}
#else
template <int MODE>
static cudaError_t launch_wave(tlag_engine* e, uint64_t lo, uint64_t hi) {
  const auto fn = vm_variant(e, [](auto f, auto s, auto l) { return k_wave<f, MODE, s, l>; });
  if (MODE == 0 && (e->p.flags & TLAG_F_EXACT)) {                 // sequential replay: one warp, one state at a time
    const size_t smem = vm_smem(e);
    const cudaError_t r = allow_smem(fn, smem);
    if (r != cudaSuccess) return r;
    fn<<<1, 32, smem, e->stream>>>(e->p, lo, hi);
    e->launches++;
    return cudaGetLastError();
  }
  return launch_vm(e, fn, hi - lo, e->p, lo, hi);
}
#endif

// The counter block after everything queued on the engine's stream so far.  The stream is non-blocking, so a copy on
// the legacy stream would not wait for that work: this is the only copy of d_ctr to the host.
static cudaError_t read_counters(tlag_engine* e, Counters* hc) {
  cudaError_t r = cudaMemcpyAsync(hc, e->d_ctr, sizeof(*hc), cudaMemcpyDeviceToHost, e->stream);
  return r != cudaSuccess ? r : cudaStreamSynchronize(e->stream);
}

// The counters of a store of n_states states that has discovered nothing since: zero, and the violation slots (minimum
// keys) at "none"
static cudaError_t reset_counters(tlag_engine* e, uint64_t n_states) {
  Counters hc;
  memset(&hc, 0, sizeof(hc));
  hc.n_states = n_states;
  hc.viol_inv = hc.viol_assert = hc.viol_trap = hc.viol_deadlock = ~0ULL;
  return cudaMemcpyAsync(e->d_ctr, &hc, sizeof(hc), cudaMemcpyHostToDevice, e->stream);   // pageable: staged before return
}

// enqueue() between two events on the engine's stream; waits for it and returns its device time in *ms.  With hc the
// counters are read in the same synchronisation.
template <class F>
static int timed(tlag_engine* e, float* ms, Counters* hc, F&& enqueue) {
  CK(cudaEventRecord(e->ev0, e->stream));
  int r = enqueue();
  if (r) return r;
  CK(cudaEventRecord(e->ev1, e->stream));
  if (hc) CK(read_counters(e, hc));
  else CK(cudaEventSynchronize(e->ev1));
  CK(cudaEventElapsedTime(ms, e->ev0, e->ev1));
  return TLAG_OK;
}

// The XOR and the SUM a digest kernel accumulates: launch() enqueues it on the engine's stream, into e->d_dig zeroed first
template <class F>
static int read_digest(tlag_engine* e, uint64_t* xor_out, uint64_t* sum_out, F&& launch) {
  if (!e->d_dig) CK(cudaMalloc(&e->d_dig, 16));
  CK(cudaMemsetAsync(e->d_dig, 0, 16, e->stream));
  const int r = launch();
  if (r) return r;
  unsigned long long h2[2];
  CK(cudaMemcpyAsync(h2, e->d_dig, 16, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  *xor_out = h2[0]; *sum_out = h2[1];
  return TLAG_OK;
}

// A snapshot's store overflow or full seen-set as TLAG_ENOMEM with its message in e->err (store_msg null: the store is
// not checked)
static int overflow_error(tlag_engine* e, const Counters& hc, const char* store_msg, const char* table_msg) {
  if (store_msg && hc.store_overflow) { e->err = store_msg; return TLAG_ENOMEM; }
  if (hc.table_full) { e->err = table_msg; return TLAG_ENOMEM; }
  return TLAG_OK;
}

static int alloc_table(tlag_engine* e, unsigned log2) {
  if (e->d_table) dfree(e, e->d_table);
  e->d_table = nullptr;
  const uint64_t slots = 1ULL << log2;
  CK(dmalloc(e, &e->d_table, slots * 8));
  CK(cudaMemsetAsync(e->d_table, 0, slots * 8, e->stream));
  e->table_log2 = log2;
  e->p.table = e->d_table;
  e->p.mask = slots - 1;
  return TLAG_OK;
}

static int sync_store(tlag_engine* e, uint64_t n_states);

static int grow_table_if_needed(tlag_engine* e, uint64_t expected_states) {
  const uint64_t slots = 1ULL << e->table_log2;
  if (expected_states * (e->tight ? 1 : 2) <= slots) return TLAG_OK;
  unsigned log2 = e->table_log2;
  while ((1ULL << log2) < expected_states * (e->tight ? 1 : 4)) ++log2;
  Counters hc;
  CK(read_counters(e, &hc));
  int r = alloc_table(e, log2);
  if (r) return r;
  const uint64_t n = hc.n_states;
  r = sync_store(e, n);            // the rehash reads every row from the store
  if (r) return r;
  if (n) {
    k_rehash<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(e->p, n);
    e->launches++;
    CK(cudaGetLastError());
  }
  return TLAG_OK;
}

static int grow_store_if_needed(tlag_engine* e, uint64_t need) {
  if (need <= e->cap_states) return TLAG_OK;
  uint64_t ncap = e->cap_states;
  if (e->tight) ncap = need;
  while (ncap < need) ncap *= (ncap < (1ULL << 25) ? 4 : 2);   // few re-allocations while the store is small
  if (e->m.max_states && ncap > e->m.max_states) ncap = e->m.max_states;
  // parent links are 32-bit indices into this rank's store and 0xFFFFFFFF marks an initial state: a store never holds
  // more than 2^32 - 2 states per GPU (beyond that the wave reports a store overflow instead of wrapping a link)
  if (ncap > 0xFFFFFFFEull) ncap = 0xFFFFFFFEull;
  if (ncap <= e->cap_states) return TLAG_OK;   // at the configured limit; overflow is detected by the kernel
  size_t freeb = 0, totalb = 0;
  cudaMemGetInfo(&freeb, &totalb);
  const uint64_t per = (uint64_t)e->m.words_per_state * 4 + 8;
  if (ncap * per > freeb * 9 / 10) {
    // the clustering buffers are re-allocated by the next level that needs them: the store comes first (an open level
    // keeps its discovery buffer, which holds its rows)
    if (!e->disc_open) { dfree(e, e->d_disc); e->d_disc = nullptr; e->disc_bytes = 0; }
    dfree(e, e->d_sort); e->d_sort = nullptr; e->sort_bytes = 0;
    dfree(e, e->d_rset); e->d_rset = nullptr; e->rset_bytes = 0;
    trim_pool(e);
    cudaMemGetInfo(&freeb, &totalb);
  }
  if (ncap * per > freeb * 9 / 10) {
    ncap = e->cap_states + (freeb * 8 / 10) / per;
    if (ncap <= e->cap_states) return TLAG_OK;
  }
  uint32_t *ns = nullptr, *np = nullptr, *nm = nullptr;
  CK(dmalloc(e, &ns, ncap * (uint64_t)e->m.words_per_state * 4));
  CK(dmalloc(e, &np, ncap * 4));
  CK(dmalloc(e, &nm, ncap * 4));
  Counters hc;
  CK(read_counters(e, &hc));
  const uint64_t n = e->disc_open ? e->hi : hc.n_states;   // an open level's rows are in its discovery buffer
  CK(cudaMemcpyAsync(ns, e->d_states, n * (uint64_t)e->m.words_per_state * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(np, e->d_parent, n * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(nm, e->d_meta, n * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  dfree(e, e->d_states); dfree(e, e->d_parent); dfree(e, e->d_meta);
  e->d_states = ns; e->d_parent = np; e->d_meta = nm;
  e->cap_states = ncap;
  e->p.states = ns; e->p.parent = np; e->p.meta = nm;
  if (!e->disc_open) point_appends(e);                   // an open level keeps appending to its buffer (open_level)
  return TLAG_OK;
}

// room for a level before it runs: the store for store_need states, the seen-set for table_need
static int reserve_level(tlag_engine* e, uint64_t store_need, uint64_t table_need) {
  int r = grow_store_if_needed(e, store_need);
  return r ? r : grow_table_if_needed(e, table_need);
}

// Grows a clustering buffer to at least `bytes` (geometrically when `slack`: levels grow, a re-allocation per level is
// slow).  false: no device memory for it -- the level is then left in discovery order (the order is an optimisation).
static bool ensure_cluster_buf(tlag_engine* e, void** buf, uint64_t* cap, uint64_t bytes, bool slack) {
  if (bytes <= *cap) return true;
  dfree(e, *buf); *buf = nullptr; *cap = 0;
  uint64_t want = slack ? bytes * 2 : bytes;
  if (dmalloc(e, buf, want) != cudaSuccess) {
    cudaGetLastError();
    want = bytes;
    if (dmalloc(e, buf, want) != cudaSuccess) { cudaGetLastError(); return false; }
  }
  *cap = want;
  return true;
}

// Records [first, first + count) of the open level's discovery buffer into store rows [first, first + count): row
// first + i gets record idx[i], or without idx record i (discovery order).
static int gather_rows(tlag_engine* e, uint64_t first, uint64_t count, const uint32_t* idx) {
  if (count == 0) return TLAG_OK;
  const uint64_t W = e->m.words_per_state;
  const uint32_t* rec = (const uint32_t*)e->d_disc + (first - e->hi) * (W + 2);
  k_cluster_gather<<<(unsigned)((count + 255) / 256), 256, 0, e->stream>>>(rec, idx, count, (int)W, e->d_states + first * W,
                                                                           e->d_parent + first, e->d_meta + first);
  e->launches++;
  CK(cudaGetLastError());
  return TLAG_OK;
}

// Puts the open level's `count` discovered records into store rows [first, first + count): stably sorted by key, or in
// discovery order when the level is not clustered (under 8192 states, TLAG_NO_SORT, a single key, or no device memory
// for the pass: the order is an optimisation).
static int cluster_slice(tlag_engine* e, uint64_t first, uint64_t count) {
  if (e->no_sort || count < 8192 || count > 0xFFFFFFFFull) return gather_rows(e, first, count, nullptr);
  const uint64_t W = e->m.words_per_state;
  const uint32_t* rec = (const uint32_t*)e->d_disc + (first - e->hi) * (W + 2);
  const uint64_t cpad = (count + 63) & ~63ull;
  size_t sort_tmp = 0, list_tmp = 0;
  {
    cub::DoubleBuffer<uint32_t> k32(nullptr, nullptr), v32(nullptr, nullptr);
    cub::DoubleBuffer<unsigned long long> k64(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, k32, v32, (unsigned long long)count);
    cub::DeviceRadixSort::SortKeys(nullptr, list_tmp, k64, (unsigned long long)count);   // the distinct keys: <= count
  }
  const size_t cub_bytes = sort_tmp > list_tmp ? sort_tmp : list_tmp;
  // one scratch allocation: A = (slot, then rank | idx) | B = (rank | idx) | cub temp
  if (!ensure_cluster_buf(e, &e->d_sort, &e->sort_bytes, cpad * 8 * 2 + cub_bytes, true)) return gather_rows(e, first, count, nullptr);
  uint8_t* b = (uint8_t*)e->d_sort;
  uint32_t* rank_a = (uint32_t*)b; uint32_t* idx_a = rank_a + cpad;
  uint32_t* rank_b = idx_a + cpad; uint32_t* idx_b = rank_b + cpad;
  void* cub_tmp = b + cpad * 16;
  const unsigned blocks = (unsigned)((count + 255) / 256);

  // the level's distinct keys and each record's slot; a set past half full is grown 4x and filled again
  unsigned log2 = e->rset_log2;
  RankSetCtl hc;
  for (;;) {
    const uint64_t slots = 1ull << log2;
    // [RankSetCtl | slots keys | slots + 2 ranks | two lists of slots / 2 keys]: a set that is not full holds <= slots / 2
    if (!ensure_cluster_buf(e, &e->d_rset, &e->rset_bytes, 256 + slots * 8 + (slots + 2) * 4 + slots * 8, false))
      return gather_rows(e, first, count, nullptr);
    RankSetCtl* ctl = (RankSetCtl*)e->d_rset;
    unsigned long long* table = (unsigned long long*)((uint8_t*)e->d_rset + 256);
    CK(cudaMemsetAsync(ctl, 0, sizeof(RankSetCtl), e->stream));
    CK(cudaMemsetAsync(table, 0xFF, slots * 8, e->stream));
    k_rset_insert<<<blocks, 256, 0, e->stream>>>(rec, count, (int)W, table, slots - 1, ctl, rank_a);
    CK(cudaGetLastError());
    e->launches++;
    CK(cudaMemcpyAsync(&hc, ctl, sizeof(hc), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (!hc.full) break;
    log2 += 2;
  }
  if (!e->rset_fixed) e->rset_log2 = log2;
  const uint64_t distinct = (uint64_t)hc.n + hc.has_max;
  if (distinct <= 1) return gather_rows(e, first, count, nullptr);   // one key: the stable order is discovery order
  const uint64_t slots = 1ull << log2;
  RankSetCtl* ctl = (RankSetCtl*)e->d_rset;
  unsigned long long* table = (unsigned long long*)((uint8_t*)e->d_rset + 256);
  uint32_t* rank = (uint32_t*)(table + slots);        // per slot, and one for the TLAG_RSET_EMPTY key

  // rank of each distinct key = its position in sorted order (a key equal to the empty marker is the largest: rank n)
  unsigned long long* list_a = (unsigned long long*)(rank + slots + 2);
  unsigned long long* list_b = list_a + slots / 2;
  k_rset_list<<<(unsigned)((slots + 255) / 256), 256, 0, e->stream>>>(table, slots, list_a, ctl);
  CK(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> dk(list_a, list_b);
  size_t tb = cub_bytes;
  if (cub::DeviceRadixSort::SortKeys(cub_tmp, tb, dk, (unsigned long long)hc.n, 0, 64, e->stream) != cudaSuccess) {
    e->err = "cub sort failed"; return TLAG_ECUDA;
  }
  k_rset_rank<<<(hc.n + 1 + 255) / 256, 256, 0, e->stream>>>(dk.Current(), hc.n, table, slots - 1, rank);
  CK(cudaGetLastError());

  // stable sort of (rank, discovery index) over the rank's bits, then one gather from the buffer into the store
  // (in place over the slots)
  k_rank_states<<<blocks, 256, 0, e->stream>>>(rank_a, count, rank, rank_a, idx_a);
  CK(cudaGetLastError());
  const int end_bit = 32 - __builtin_clz((unsigned)(distinct - 1));
  cub::DoubleBuffer<uint32_t> rk(rank_a, rank_b), ix(idx_a, idx_b);
  tb = cub_bytes;
  if (cub::DeviceRadixSort::SortPairs(cub_tmp, tb, rk, ix, (unsigned long long)count, 0, end_bit, e->stream) != cudaSuccess) {
    e->err = "cub sort failed"; return TLAG_ECUDA;
  }
  e->launches += 4;
  return gather_rows(e, first, count, ix.Current());
}

// Rows the open level has discovered so far, copied into the store in discovery order, for a call that reads the store
// in the middle of a level.  The buffer keeps them: the level is still clustered when it ends.
static int sync_store(tlag_engine* e, uint64_t n_states) {
  if (!e->disc_open) return TLAG_OK;
  const uint64_t end = n_states < e->p.cap_states ? n_states : e->p.cap_states;
  if (end <= e->hi) return TLAG_OK;
  int r = gather_rows(e, e->hi, end - e->hi, nullptr);
  if (r) return r;
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
}

// The level appends to the store itself again: its discovery buffer's rows are in the store, or discarded.
static void end_appends(tlag_engine* e) {
  e->disc_open = false;
  point_appends(e);
}

// Opens the level being discovered for appends to the discovery buffer: rows [hi, hi + rows) of it, at most up to the
// store's capacity.  A row past that is counted in n_states, not written, and reported as a store overflow.  A level that
// is already open keeps the rows it has put there, and its room never shrinks.  Without device memory for the buffer the
// level appends to the store itself and is not clustered.  TLAG_F_EXACT always does: its single worker dequeues the rows
// it appends, in the same launch.
static int open_level(tlag_engine* e, uint64_t rows) {
  if (e->m.flags & TLAG_F_EXACT) return TLAG_OK;
  const uint64_t room = e->cap_states - e->hi;
  if (rows > room) rows = room;
  if (e->disc_open && e->p.cap_states >= e->hi + rows) return TLAG_OK;
  const uint64_t rb = (e->m.words_per_state + 2) * 4;
  if (rows * rb > e->disc_bytes) {
    uint64_t used = 0;
    if (e->disc_open) {
      Counters hc;
      CK(read_counters(e, &hc));
      used = (hc.n_states < e->p.cap_states ? hc.n_states : e->p.cap_states) - e->hi;
    }
    // levels grow: twice the rows asked for while the store has room for them, so that the next levels fit too (only
    // from memory that is free: the pool is not trimmed for it)
    uint64_t want = (rows * 2 < room ? rows * 2 : room) * rb;
    void* nb = nullptr;
    if (want > rows * rb && dmalloc(e, &nb, want, false) != cudaSuccess) { cudaGetLastError(); nb = nullptr; }
    if (!nb) {
      want = rows * rb;
      if (dmalloc(e, &nb, want) != cudaSuccess) {
        cudaGetLastError();
        int r = used ? gather_rows(e, e->hi, used, nullptr) : TLAG_OK;
        if (r) return r;
        dfree(e, e->d_disc); e->d_disc = nullptr; e->disc_bytes = 0;
        end_appends(e);
        return TLAG_OK;
      }
    }
    if (used) CK(cudaMemcpyAsync(nb, e->d_disc, used * rb, cudaMemcpyDeviceToDevice, e->stream));
    dfree(e, e->d_disc);
    e->d_disc = nb; e->disc_bytes = want;
  }
  e->disc_open = true;
  point_appends(e);
  e->p.cap_states = e->hi + rows;
  return TLAG_OK;
}

// Route mode with several ranks: the direct-mapped cache of the fingerprints this rank has routed (2^26 x 8 B = 512 MB).
// It is only a filter: without memory for it every successor is routed.
static int ensure_sent_cache(tlag_engine* e) {
  if (e->d_sent || e->p.n_ranks < 2) return TLAG_OK;
  const unsigned long long slots = 1ULL << 26;
  if (dmalloc(e, &e->d_sent, slots * 8) != cudaSuccess) { cudaGetLastError(); e->d_sent = nullptr; return TLAG_OK; }
  CK(cudaMemsetAsync(e->d_sent, 0, slots * 8, e->stream));
  e->p.sent_cache = e->d_sent; e->p.sent_mask = slots - 1;
  return TLAG_OK;
}

#if defined(TLAG_SLICED_INC)
extern "C" const char* tlag_version(void) { return "tlag 0.2 (sm_90a) native sliced"; }
#else
extern "C" const char* tlag_version(void) { return "tlag 0.1 (sm_90a)"; }
#endif

extern "C" const char* tlag_last_error(const tlag_engine* e) { return e ? e->err.c_str() : "null engine"; }

extern "C" uint64_t tlag_kernel_launches(const tlag_engine* e) { return e ? e->launches : 0; }

// The engine's test hooks (DESIGN.md section 4d), read once per engine: each forces a path that a test must reach and
// that the engine's own sizing would rarely or never take.  None is a tuning knob.  Called with e->p zeroed.
static void read_env_hooks(tlag_engine* e) {
  // 1: the store starts at 1024 rows, and the store and the seen-set are sized before each level for as many new states
  // as the level expands, with no slack, and a rerun for exactly what the failed attempt counted: every level that grows
  // overflows the store (or, with a small table_slots_log2, fills the table) and is rolled back and redone (rollback_wave)
  const char* s_ = getenv("TLAG_TIGHT_HEADROOM");
  e->tight = s_ && *s_ && atoi(s_) != 0;
  // set (any value): no level is clustered, each goes to the store in discovery order (cluster_slice)
  e->no_sort = getenv("TLAG_NO_SORT") != nullptr;
  // sliced build: 0 probes self-loop successors like any other successor instead of dropping them at the emit site
  s_ = getenv("TLAG_SL_SKIPSELF");
  e->p.skip_self = (s_ && *s_) ? (atoi(s_) != 0) : 1;
  // sliced build, scalar form: n caps the per-warp staging slots below the compiled number, so that the buffer fills up
  // and the direct path runs (0: every successor is probed where it is produced; tlag_dev.cuh, TLAG_SL_STAGED)
  s_ = getenv("TLAG_SL_STAGE");
  e->p.stage = (s_ && *s_) ? (atoi(s_) > 0 ? atoi(s_) : 0) : INT_MAX;
  // n starts the clustering pass's rank set at n slots (rounded up to a power of two) on every level, so that it fills
  // up and grows
  s_ = getenv("TLAG_RSET_SLOTS");
  if (s_ && *s_) {
    const long n = atol(s_);
    e->rset_log2 = 1;
    while (e->rset_log2 < 40 && (1L << e->rset_log2) < n) ++e->rset_log2;
    e->rset_fixed = true;
  }
  // n starts the state graph's edge buffer at n edges (tlag_build_graph), so that chunks overflow it and are run again
  // with fewer rows
  s_ = getenv("TLAG_GRAPH_EDGES");
  if (s_ && *s_ && atoll(s_) > 0) e->graph_edges = (uint64_t)atoll(s_);
}

// The state graph is a picture of the store after a search call: any call that changes the store drops it.
static void release_graph(tlag_engine* e) {
  dfree(e, e->d_goff); dfree(e, e->d_gdst); dfree(e, e->d_gact); dfree(e, e->d_slab); dfree(e, e->d_elab);
  e->d_goff = nullptr; e->d_gdst = e->d_gact = nullptr; e->d_slab = e->d_elab = nullptr;
  e->g_cap = e->g_edges = e->g_states = e->g_expanded = 0;
  e->g_ready = false;
}

extern "C" int tlag_create(const tlag_model* m, tlag_engine** out) {
  if (!m || !out) return TLAG_EINVAL;
  *out = nullptr;
  tlag_engine* e = new tlag_engine();
  *out = e;   // returned even on failure so that tlag_last_error works; caller destroys it
  e->m = *m;
  if (m->words_per_state == 0 || m->words_per_state > TLAG_MAXW) { e->err = "words_per_state out of range (1..128)"; return TLAG_EINVAL; }
  if (m->frame_words > 8192) { e->err = "frame_words > 8192 not supported"; return TLAG_EINVAL; }
#if defined(TLAG_SLICED_INC)
  if (m->flags & TLAG_F_EXACT) { e->err = "TLAG_F_EXACT (sequential replay) runs on the interpreter kernel: use libtlag.so"; return TLAG_EINVAL; }
  {  // this library holds ONE model's program as kernels (constant pool folded in): refuse anything else
    uint64_t h = 0xcbf29ce484222325ULL, hc = 0xcbf29ce484222325ULL;
    for (uint32_t i = 0; i < m->code_len; ++i) h = (h ^ m->code[i]) * 0x100000001b3ULL;
    for (uint32_t i = 0; i < m->cpool_len; ++i) hc = (hc ^ (uint64_t)(uint32_t)m->cpool[i]) * 0x100000001b3ULL;
    if (m->code_len != TLAG_NATIVE_CODE_LEN || h != TLAG_NATIVE_CODE_FNV || hc != TLAG_NATIVE_CPOOL_FNV ||
        m->frame_words > TLAG_SL_FRAME || m->words_per_state != TLAG_SL_W) {
      e->err = "this library was compiled for another model's program (native build)";
      return TLAG_EINVAL;
    }
  }
#endif
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { e->err = "no CUDA device available"; return TLAG_ECUDA; }
  CK(cudaSetDevice(m->device));
  // Seen-set probes are random 8-byte accesses: ncu showed every probe pulling a full 128-byte line
  // from DRAM (4 sectors) with the default L2 fetch granularity; 32 B makes a probe cost one sector.
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, m->device));
  e->sm_count = prop.multiProcessorCount;
  CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, m->device) == cudaSuccess) {
      uint64_t thr = ~0ULL;                       // keep freed buffers mapped (see dmalloc)
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    } else cudaGetLastError();
  }
  CK(cudaEventCreate(&e->ev0));
  CK(cudaEventCreate(&e->ev1));
#if defined(TLAG_SLICED_INC)
  const uint32_t vm_frame = TLAG_SL_FRAME;   // the frame the library's one interpreter kernel is compiled for (launch_graph)
#else
  const uint32_t vm_frame = m->frame_words;
#endif
  e->frame_class = vm_frame_class(vm_frame);
  for (uint32_t i = 0; i < m->code_len && !e->uses_ext; ++i) {
    const uint32_t op = (uint32_t)(m->code[i] & 0xFF);
    if (op == OP_LEXLT || op == OP_SFIND || op == OP_SINS || op == OP_EMITD || op == OP_CALL || op == OP_RET) e->uses_ext = true;
  }
  // program image
  CK(cudaMalloc(&e->d_code, (size_t)(m->code_len ? m->code_len : 1) * 8));
  CK(cudaMemcpy(e->d_code, m->code, (size_t)m->code_len * 8, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&e->d_cpool, (size_t)(m->cpool_len ? m->cpool_len : 1) * 4));
  CK(cudaMemcpy(e->d_cpool, m->cpool, (size_t)m->cpool_len * 4, cudaMemcpyHostToDevice));
  CK(cudaMalloc(&e->d_layout, (size_t)(m->n_slots ? m->n_slots : 1) * sizeof(tlag_slot)));
  CK(cudaMemcpy(e->d_layout, m->layout, (size_t)m->n_slots * sizeof(tlag_slot), cudaMemcpyHostToDevice));
  CK(cudaMalloc(&e->d_ctr, sizeof(Counters)));
  CK(reset_counters(e, 0));
  memset(&e->p, 0, sizeof(e->p));
  read_env_hooks(e);
  // state store
  uint64_t cap = m->max_states ? m->max_states : (1ULL << 20);
  if (cap < 1024) cap = 1024;
  if (!m->max_states) cap = 1ULL << 20;
  else if (cap > (1ULL << 22)) cap = 1ULL << 22;   // start modest, grow on demand up to max_states
  if (e->tight) cap = 1024;
  e->cap_states = cap;
  CK(dmalloc(e, &e->d_states, cap * (uint64_t)m->words_per_state * 4));
  CK(dmalloc(e, &e->d_parent, cap * 4));
  CK(dmalloc(e, &e->d_meta, cap * 4));
  e->p.code = e->d_code; e->p.code_len = m->code_len;
  e->p.code_in_smem = vm_code_in_smem(vm_frame, m->code_len) ? 1 : 0;
  e->p.cpool = e->d_cpool; e->p.layout = e->d_layout; e->p.n_slots = (int)m->n_slots;
  e->p.entry_inv = m->entry_inv; e->p.entry_next = m->entry_next;
  e->p.n_off = 0; e->p.p_off = m->unpacked_words; e->p.W = (int)m->words_per_state;
  e->p.states = e->d_states; e->p.parent = e->d_parent; e->p.meta = e->d_meta; e->p.cap_states = cap;
  point_appends(e);
  e->p.ctr = e->d_ctr; e->p.flags = m->flags; e->p.n_inv = (int)m->n_invariants;
  e->p.n_ranks = 1; e->p.rank = 0; e->p.owner_words = 2;
  unsigned log2 = m->table_slots_log2 ? m->table_slots_log2 : 22;
  int r = alloc_table(e, log2);
  if (r) return r;
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
}

extern "C" void tlag_destroy(tlag_engine* e) {
  if (!e) return;
  cudaFree(e->d_code); cudaFree(e->d_cpool); cudaFree(e->d_layout); cudaFree(e->d_ctr); cudaFree(e->d_dig); cudaFree(e->d_sctl);
  if (e->stream) {
    dfree(e, e->d_states); dfree(e, e->d_parent); dfree(e, e->d_meta); dfree(e, e->d_table);
    dfree(e, e->d_scratch); dfree(e, e->d_flags); dfree(e, e->d_disc); dfree(e, e->d_sort); dfree(e, e->d_rset); dfree(e, e->d_sent); dfree(e, e->d_succ);
    dfree(e, e->d_hist); dfree(e, e->d_act); dfree(e, e->d_sstat); dfree(e, e->d_ssucc); dfree(e, e->d_scnt); dfree(e, e->d_slen);
    dfree(e, e->d_sinit);
    release_graph(e);
    cudaStreamSynchronize(e->stream);
  }
  if (e->p2p_slot >= 0) {                              // exchange buffers and peer mappings are parked, not released
    if (e->stream) cudaStreamSynchronize(e->stream);
    g_p2p_parked[e->p2p_slot].seq = e->p2p_seq;
    g_p2p_parked[e->p2p_slot].in_use = false;
  }
  if (e->ev0) cudaEventDestroy(e->ev0);
  if (e->ev1) cudaEventDestroy(e->ev1);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

static int ensure_scratch(tlag_engine* e, uint64_t words, uint64_t flags) {
  if (words > e->scratch_words) {
    dfree(e, e->d_scratch); e->d_scratch = nullptr; e->scratch_words = 0;
    CK(dmalloc(e, &e->d_scratch, words * 4));
    e->scratch_words = words;
  }
  if (flags > e->flags_cap) {
    dfree(e, e->d_flags); e->d_flags = nullptr; e->flags_cap = 0;
    CK(dmalloc(e, &e->d_flags, flags));
    e->flags_cap = flags;
  }
  return TLAG_OK;
}

static int launch_probe(tlag_engine* e, const uint32_t* d_states, uint64_t n, uint8_t* d_is_new) {
  const int W = (int)e->m.words_per_state;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (n == 0) return TLAG_OK;
  if (((uintptr_t)d_states % 16) == 0 && W >= 2) {
    const size_t smem = (size_t)256 * (size_t)(W | 1) * 4;
    CK(allow_smem(k_probe_staged, smem));
    k_probe_staged<<<blocks, 256, smem, e->stream>>>(d_states, n, W, e->d_table, e->p.mask, d_is_new, e->d_ctr);
  } else {
    k_probe<<<blocks, 256, 0, e->stream>>>(d_states, n, W, e->d_table, e->p.mask, d_is_new, e->d_ctr);
  }
  e->launches++;
  CK(cudaGetLastError());
  return TLAG_OK;
}

extern "C" int tlag_probe_batch_device(tlag_engine* e, uint64_t d_states, uint64_t n, uint64_t d_is_new, float* kernel_ms) {
  if (!e) return TLAG_EINVAL;
  Counters hc;
  float ms = 0;
  int r = timed(e, &ms, &hc, [&] { return launch_probe(e, (const uint32_t*)(uintptr_t)d_states, n, (uint8_t*)(uintptr_t)d_is_new); });
  if (r) return r;
  if (kernel_ms) *kernel_ms = ms;
  return overflow_error(e, hc, nullptr, "seen-set table is full");
}

extern "C" int tlag_probe_batch(tlag_engine* e, const uint32_t* states, uint64_t n, uint8_t* is_new) {
  if (!e || (!states && n) || (!is_new && n)) return TLAG_EINVAL;
  if (n == 0) return TLAG_OK;
  const uint64_t W = e->m.words_per_state;
  int r = ensure_scratch(e, n * W, n);
  if (r) return r;
  CK(cudaMemcpyAsync(e->d_scratch, states, n * W * 4, cudaMemcpyHostToDevice, e->stream));
  r = launch_probe(e, e->d_scratch, n, e->d_flags);
  if (r) return r;
  CK(cudaMemcpyAsync(is_new, e->d_flags, n, cudaMemcpyDeviceToHost, e->stream));
  Counters hc;
  CK(read_counters(e, &hc));
  return overflow_error(e, hc, nullptr, "seen-set table is full");
}

extern "C" int tlag_reset_table(tlag_engine* e) {
  if (!e) return TLAG_EINVAL;
  CK(cudaMemsetAsync(e->d_table, 0, (1ULL << e->table_log2) * 8, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
}

extern "C" int tlag_seed(tlag_engine* e, const uint32_t* states, uint64_t n) {
  if (!e || (!states && n)) return TLAG_EINVAL;
  if (e->level != 0) { e->err = "tlag_seed after the search started"; return TLAG_ESTATE; }
  release_graph(e);
  const uint64_t W = e->m.words_per_state;
  int r = reserve_level(e, e->hi + n + 1024, e->hi + n);
  if (r) return r;
  if (n) {
    // records: W words + parent(-1) + meta(action -1)
    std::vector<uint32_t> rec(n * (W + 2));
    for (uint64_t i = 0; i < n; ++i) {
      memcpy(&rec[i * (W + 2)], states + i * W, W * 4);
      rec[i * (W + 2) + W] = 0xFFFFFFFFu;
      rec[i * (W + 2) + W + 1] = 0xFFFFFF00u;
    }
    r = ensure_scratch(e, n * (W + 2), 0);
    if (r) return r;
    CK(cudaMemcpyAsync(e->d_scratch, rec.data(), rec.size() * 4, cudaMemcpyHostToDevice, e->stream));
    if (e->m.flags & TLAG_F_EXACT) {
      // store order = the caller's order (TLC enumerates the initial states in a fixed order): one warp at a time
      for (uint64_t o = 0; o < n; o += 32) {
        const uint64_t c = n - o < 32 ? n - o : 32;
        k_insert_records<<<1, 32, 0, e->stream>>>(e->p, e->d_scratch + o * (W + 2), c);
      }
    } else {
      k_insert_records<<<(unsigned)((n + 255) / 256), 256, 0, e->stream>>>(e->p, e->d_scratch, n);
    }
    e->launches++;
    CK(cudaGetLastError());
  }
  Counters hc;
  CK(read_counters(e, &hc));
  e->generated += n;
  e->hi = hc.n_states;
  e->init_states = hc.n_states;
  if (n && !e->restarting) e->h_init.insert(e->h_init.end(), states, states + n * W);
  return TLAG_OK;
}

// Forget everything discovered and start again from the retained initial states (bench loops).
extern "C" int tlag_restart(tlag_engine* e) {
  if (!e) return TLAG_EINVAL;
  release_graph(e);
  end_appends(e);
  CK(reset_counters(e, 0));
  CK(cudaMemsetAsync(e->d_table, 0, (1ULL << e->table_log2) * 8, e->stream));
  if (e->d_sent) CK(cudaMemsetAsync(e->d_sent, 0, (e->p.sent_mask + 1) * 8, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  e->lo = e->hi = 0; e->level = 0; e->init_states = 0; e->generated = 0; e->depth = 0;
  e->verdict = TLAG_V_RUNNING; e->detail = e->detail2 = 0; e->viol_idx = 0; e->dev_seconds = 0;
  e->kg_verdict = 0;
  e->restarting = true;
  const uint64_t W = e->m.words_per_state;
  int r = tlag_seed(e, e->h_init.data(), e->h_init.size() / W);
  e->restarting = false;
  return r;
}

static void fill_result(tlag_engine* e, tlag_result* out, uint64_t n_states) {
  memset(out, 0, sizeof(*out));
  out->verdict = e->verdict;
  out->detail = e->detail;
  out->detail2 = e->detail2;
  out->state_idx = e->viol_idx;
  out->generated = e->generated;
  out->distinct = n_states;
  out->queue_left = (e->verdict == TLAG_V_OK) ? 0 : (n_states - e->hi) + 0;
  if ((e->m.flags & TLAG_F_EXACT) && (e->verdict == TLAG_V_ASSERT || e->verdict == TLAG_V_DEADLOCK) && n_states > e->viol_idx)
    out->queue_left = n_states - e->viol_idx - 1;      // discovered, not yet dequeued when the worker stopped
  out->depth = e->depth;
  out->init_states = e->init_states;
  const double n = (double)n_states, g = (double)e->generated;
  out->fp_collision_estimate = n * (g > n ? g - n : 0.0) / 18446744073709551616.0;
  out->device_seconds = e->dev_seconds;
}

// decode violation counters after a wave; sets e->verdict if something was found
static void collect_violations(tlag_engine* e, const Counters& hc) {
  unsigned long long best = ~0ULL; int kind = 0;
  if (hc.viol_trap != ~0ULL && (hc.viol_trap >> 20) < best) { best = hc.viol_trap >> 20; kind = TLAG_V_EVAL_ERROR; }
  if (hc.viol_assert != ~0ULL && (hc.viol_assert >> 20) < best) { best = hc.viol_assert >> 20; kind = TLAG_V_ASSERT; }
  if (hc.viol_inv != ~0ULL && (hc.viol_inv >> 20) < best) { best = hc.viol_inv >> 20; kind = TLAG_V_INVARIANT; }
  if (hc.viol_deadlock != ~0ULL && (hc.viol_deadlock >> 20) < best) { best = hc.viol_deadlock >> 20; kind = TLAG_V_DEADLOCK; }
  if (!kind) return;
  e->verdict = kind;
  e->viol_idx = best;
  if (kind == TLAG_V_EVAL_ERROR) { e->detail = (int)((hc.viol_trap >> 16) & 15); e->detail2 = (int)(hc.viol_trap & 0xFFFF); }
  else if (kind == TLAG_V_ASSERT) e->detail = (int)(hc.viol_assert & 0xFFFFF);
  else if (kind == TLAG_V_INVARIANT) e->detail = (int)(hc.viol_inv & 0xFFFFF);
}

// the first level call of a search: the frontier is the seeded initial states
static void start_search(tlag_engine* e) {
  if (e->level == 0) { e->level = 1; e->lo = 0; e->depth = e->hi > 0 ? 1 : 0; }
}

// the search reached its fixpoint: OK, or under TLAG_F_KEEP_GOING the first violation it went past
static void settle_verdict(tlag_engine* e) {
  e->verdict = e->kg_verdict ? e->kg_verdict : TLAG_V_OK;
  if (e->kg_verdict) { e->detail = e->kg_detail; e->detail2 = e->kg_detail2; e->viol_idx = e->kg_idx; }
}

// End of a wave, from the counters read after it: its `generated` moves to the host total (and is cleared on the
// device), a violation becomes the verdict, and out gets the wave's numbers.  keep_going: the first violation is
// remembered, the device slots are cleared and the search goes on.
static int account_wave(tlag_engine* e, const Counters& hc, bool keep_going, uint64_t expanded, float ms,
                        tlag_wave_stats* out) {
  e->generated += hc.generated;
  CK(cudaMemsetAsync(&e->d_ctr->generated, 0, 8, e->stream));
  collect_violations(e, hc);
  if (keep_going && e->verdict != TLAG_V_RUNNING) {
    if (!e->kg_verdict) { e->kg_verdict = e->verdict; e->kg_detail = e->detail; e->kg_detail2 = e->detail2; e->kg_idx = e->viol_idx; }
    e->verdict = TLAG_V_RUNNING;
    const unsigned long long ones[4] = {~0ULL, ~0ULL, ~0ULL, ~0ULL};
    CK(cudaMemcpyAsync(&e->d_ctr->viol_inv, ones, sizeof(ones), cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  if (out) {
    out->level = e->level; out->expanded = expanded; out->generated = hc.generated;
    out->distinct_total = hc.n_states; out->generated_total = e->generated; out->kernel_ms = ms;
    out->verdict = e->verdict;
  }
  return TLAG_OK;
}

// head-room for the next level: in the store twice the observed discovered/expanded ratio, at least 4x; in the discovery
// buffer the ratio plus a quarter (a level that outgrows it is rolled back and redone, tlag_step)
static void note_growth(tlag_engine* e, uint64_t expanded, uint64_t discovered) {
  const double ratio = (double)discovered / (double)(expanded ? expanded : 1);
  e->growth_hint = ratio * 2.0 > 4.0 ? ratio * 2.0 : 4.0;
  e->disc_hint = ratio * 1.25;
}

// End of a level whose store now holds n_states states: the slice it appended (if any) sets the depth and goes from the
// discovery buffer into the store, with cluster in clustering order, else in discovery order (device time in
// out->cluster_ms); then it becomes the frontier.
static int close_level(tlag_engine* e, uint64_t n_states, bool cluster, tlag_wave_stats* out) {
  if (out) {
    out->level = e->level; out->discovered = n_states - e->hi; out->distinct_total = n_states;
    out->generated_total = e->generated; out->verdict = e->verdict;
  }
  if (n_states > e->hi) {
    e->depth = e->level + 1;
    if (e->disc_open) {
      const uint64_t n = (n_states < e->p.cap_states ? n_states : e->p.cap_states) - e->hi;
      float ms = 0;
      int r = timed(e, &ms, nullptr, [&] {
        return cluster ? cluster_slice(e, e->hi, n) : gather_rows(e, e->hi, n, nullptr);
      });
      if (r) return r;
      if (out) out->cluster_ms = ms;
    }
  }
  end_appends(e);
  e->lo = e->hi; e->hi = n_states; e->level += 1;
  return TLAG_OK;
}

// Undo a wave that ran out of store or table space: the states it appended are dropped (n_states back to `hi`), the
// seen-set is rebuilt from the store (it holds fingerprints of the dropped states) and every other counter is reset --
// the level is then expanded again from scratch with more room.
static int rollback_wave(tlag_engine* e, uint64_t hi, uint64_t want_states) {
  end_appends(e);                  // the discovery buffer's rows are dropped with them
  CK(reset_counters(e, hi));
  int r = grow_store_if_needed(e, e->tight ? want_states : want_states + 4096);
  if (r) return r;
  unsigned log2 = e->table_log2;
  while ((1ULL << log2) < want_states * 2 && log2 < 40) ++log2;
  r = alloc_table(e, log2);
  if (r) return r;
  if (hi) {
    k_rehash<<<(unsigned)((hi + 255) / 256), 256, 0, e->stream>>>(e->p, hi);
    e->launches++;
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
}

extern "C" int tlag_step(tlag_engine* e, tlag_wave_stats* out) {
  if (!e) return TLAG_EINVAL;
#ifdef TLAG_NO_BFS
  TLAG_NO_BFS(e);
#endif
  if (out) memset(out, 0, sizeof(*out));
  release_graph(e);
  start_search(e);
  if (e->verdict != TLAG_V_RUNNING) { if (out) out->verdict = e->verdict; return TLAG_OK; }
  const uint64_t lo = e->lo, hi = e->hi;
  if (lo >= hi) {
    settle_verdict(e);
    if (out) out->verdict = e->verdict;
    return TLAG_OK;
  }
  int r = reserve_level(e, e->tight ? hi + (hi - lo) : hi + (uint64_t)((double)(hi - lo) * e->growth_hint) + 4096,
                        e->tight ? hi + (hi - lo)
                                 : hi + (uint64_t)((double)(hi - lo) * (e->growth_hint > 4.0 ? e->growth_hint * 0.5 : 2.0)));
  if (r) return r;
  // the level's new rows go to the discovery buffer, sized from the previous level's growth (a rerun: from its count);
  // TLAG_TIGHT_HEADROOM sizes the store alone, and the buffer takes all of its room
  uint64_t rows = e->tight ? e->cap_states - hi : (uint64_t)((double)(hi - lo) * e->disc_hint) + 4096;
  Counters hc;
  float ms = 0;
  int attempt = 0;
  for (;; ++attempt) {
    r = open_level(e, rows);
    if (r) return r;
    CK(cudaMemsetAsync(&e->d_ctr->work, 0, 8, e->stream));
    float ms1 = 0;
    r = timed(e, &ms1, &hc, [&] { CK(launch_wave<0>(e, lo, hi)); return TLAG_OK; });
    if (r) return r;
    ms += ms1;
    if (!hc.store_overflow && !hc.table_full) break;
    // The head-room heuristics were too tight for this level (its discovered / expanded ratio jumped): n_states kept
    // counting past the capacity, so it says how much room the level needs.  Redo the level with that much, twice over.
    const uint64_t need = hc.n_states > hi ? hc.n_states : hi;
    const uint64_t want = e->tight ? need : hi + (need - hi) * 2 + 4096;
    if (attempt >= 3 || (e->m.max_states && need > e->m.max_states) || need > 0xFFFFFFFEull)
      return overflow_error(e, hc, "state store overflow: raise max_states (or the model needs more than 2^32 - 2 states per GPU)",
                            "seen-set table full");
    r = rollback_wave(e, hi, want);
    if (r) return r;
    if (e->cap_states < need + (e->tight ? 0 : 1024)) { e->err = "state store overflow: not enough device memory for this level"; return TLAG_ENOMEM; }
    rows = e->tight ? e->cap_states - hi : want - hi;
  }
  e->dev_seconds += ms * 1e-3;
  r = account_wave(e, hc, (e->m.flags & TLAG_F_KEEP_GOING) != 0, hi - lo, ms, out);
  if (r) return r;
  if (out) out->retries = (uint32_t)attempt;
  r = close_level(e, hc.n_states, e->verdict == TLAG_V_RUNNING, out);
  if (r) return r;
  note_growth(e, hi - lo, e->hi - hi);
  if (e->verdict == TLAG_V_RUNNING && e->lo >= e->hi) settle_verdict(e);
  if (out) out->verdict = e->verdict;
  return TLAG_OK;
}

extern "C" int tlag_result_now(tlag_engine* e, tlag_result* out) {
  if (!e || !out) return TLAG_EINVAL;
  Counters hc;
  CK(read_counters(e, &hc));
  fill_result(e, out, hc.n_states);
  return TLAG_OK;
}

extern "C" int tlag_run(tlag_engine* e, tlag_result* out) {
  if (!e || !out) return TLAG_EINVAL;
  tlag_wave_stats ws;
  for (;;) {
    int r = tlag_step(e, &ws);
    if (r) return r;
    if (ws.verdict != TLAG_V_RUNNING) break;
  }
  return tlag_result_now(e, out);
}

extern "C" int tlag_read_states(tlag_engine* e, uint64_t first, uint64_t n, uint32_t* states_out) {
  if (!e || (!states_out && n)) return TLAG_EINVAL;
  Counters hc;
  CK(read_counters(e, &hc));
  if (first + n > hc.n_states) { e->err = "tlag_read_states: range beyond the state store"; return TLAG_EINVAL; }
  int r = sync_store(e, hc.n_states);
  if (r) return r;
  const uint64_t W = e->m.words_per_state;
  CK(cudaMemcpy(states_out, e->d_states + first * W, n * W * 4, cudaMemcpyDeviceToHost));
  return TLAG_OK;
}

extern "C" int tlag_digest(tlag_engine* e, uint64_t* xor_out, uint64_t* sum_out) {
  if (!e || !xor_out || !sum_out) return TLAG_EINVAL;
  Counters hc;
  CK(read_counters(e, &hc));
  int r = sync_store(e, hc.n_states);
  if (r) return r;
  return read_digest(e, xor_out, sum_out, [&] {
    if (hc.n_states) {
      k_digest<<<e->sm_count * 8, 256, 0, e->stream>>>(e->p, hc.n_states, e->d_dig);
      e->launches++;
      CK(cudaGetLastError());
    }
    return TLAG_OK;
  });
}

// One hop of a counterexample chain: the state at idx (when state_out) with its parent index and meta word (action id
// << 8 | rank that expanded the parent).  With several ranks the parent lives in THAT rank's store: the host follows the
// chain across ranks (tla_rust_b200/dist.py: counterexample).
static int read_link(tlag_engine* e, uint64_t idx, uint32_t* state_out, uint32_t* parent_out, uint32_t* meta_out) {
  const uint64_t W = e->m.words_per_state;
  if (state_out) CK(cudaMemcpyAsync(state_out, e->d_states + idx * W, W * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(parent_out, e->d_parent + idx, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemcpyAsync(meta_out, e->d_meta + idx, 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
}

extern "C" int tlag_trace(tlag_engine* e, uint64_t state_idx, uint32_t* states_out, int32_t* actions_out, uint32_t* len_inout) {
  if (!e || !len_inout) return TLAG_EINVAL;
  Counters hc;
  CK(read_counters(e, &hc));
  if (state_idx >= hc.n_states) { e->err = "tlag_trace: no such state"; return TLAG_EINVAL; }
  int r0 = sync_store(e, hc.n_states);
  if (r0) return r0;
  const uint64_t W = e->m.words_per_state;
  std::vector<uint32_t> words;   // the chain's states from state_idx back, while they fit the caller's buffer
  std::vector<int32_t> acts;
  uint64_t cur = state_idx;
  for (;;) {
    uint32_t par = 0, meta = 0;
    const bool keep = states_out && acts.size() < *len_inout;
    if (keep) words.resize(words.size() + W);
    int r = read_link(e, cur, keep ? words.data() + words.size() - W : nullptr, &par, &meta);
    if (r) return r;
    acts.push_back(par == 0xFFFFFFFFu ? -1 : (int32_t)(meta >> 8));
    if (par == 0xFFFFFFFFu) break;
    cur = par;
    if (acts.size() > (1u << 24)) { e->err = "tlag_trace: parent chain too long"; return TLAG_ESTATE; }
  }
  const uint32_t len = (uint32_t)acts.size();
  if (len > *len_inout) { *len_inout = len; e->err = "tlag_trace: buffer too small"; return TLAG_EINVAL; }
  for (uint32_t i = 0; i < len; ++i) {
    if (states_out) memcpy(states_out + (uint64_t)i * W, words.data() + (uint64_t)(len - 1 - i) * W, W * 4);
    if (actions_out) actions_out[i] = acts[len - 1 - i];
  }
  *len_inout = len;
  return TLAG_OK;
}

extern "C" int tlag_read_link(tlag_engine* e, uint64_t idx, uint32_t* state_out, uint32_t* parent_out, uint32_t* meta_out) {
  if (!e || !parent_out || !meta_out) return TLAG_EINVAL;
  Counters hc;
  CK(read_counters(e, &hc));
  if (idx >= hc.n_states) { e->err = "tlag_read_link: no such state"; return TLAG_EINVAL; }
  int r = sync_store(e, hc.n_states);
  return r ? r : read_link(e, idx, state_out, parent_out, meta_out);
}

// ---- multi-GPU building blocks -----------------------------------------------------
extern "C" int tlag_frontier(tlag_engine* e, uint64_t* first_idx, uint64_t* count) {
  if (!e) return TLAG_EINVAL;
  start_search(e);
  if (first_idx) *first_idx = e->lo;
  if (count) *count = e->hi - e->lo;
  return TLAG_OK;
}

// Which shard of the partitioned state space this engine holds (host-driven exchange: tlag_expand_route /
// tlag_insert_records; tlag_p2p_init sets it for the peer-memory path).  The rank goes into the meta word of every
// state this engine expands a parent of, and successors the rank owns itself are inserted in place.
// How many trailing packed words the ownership hash covers (every rank must use the same value; before any state is
// routed).  2 keeps whole clusters of like states on one rank; W balances models whose tail words carry no entropy.
extern "C" int tlag_set_owner_words(tlag_engine* e, uint32_t k) {
  if (!e || k < 2) return TLAG_EINVAL;
  e->p.owner_words = (int)(k > e->m.words_per_state ? e->m.words_per_state : k);
  return TLAG_OK;
}

extern "C" int tlag_set_rank(tlag_engine* e, uint32_t n_ranks, uint32_t rank) {
  if (!e || n_ranks == 0 || n_ranks > 16 || rank >= n_ranks) return TLAG_EINVAL;
  e->p.n_ranks = (int)n_ranks; e->p.rank = (int)rank;
  return TLAG_OK;
}

extern "C" int tlag_expand_route(tlag_engine* e, uint32_t n_ranks, uint64_t first, uint64_t count, uint64_t d_send,
                                 uint64_t cap_records, uint64_t* counts, tlag_wave_stats* out) {
  if (!e || !counts || n_ranks == 0 || n_ranks > 16) return TLAG_EINVAL;
#ifdef TLAG_NO_BFS
  TLAG_NO_BFS(e);
#endif
  if (out) memset(out, 0, sizeof(*out));
  start_search(e);
  uint64_t lo = e->lo + first, hi = lo + count;
  if (lo > e->hi) lo = e->hi;
  if (hi > e->hi) hi = e->hi;
  if ((uint32_t)e->p.n_ranks != n_ranks) {
    if (n_ranks > 1) { e->err = "tlag_expand_route: call tlag_set_rank(n_ranks, rank) first"; return TLAG_ESTATE; }
    e->p.n_ranks = 1; e->p.rank = 0;
  }
  int r = ensure_sent_cache(e);
  if (r) return r;
  // successors this rank owns itself are appended here (sliced build), room for them as tlag_p2p_level reserves it;
  // an overflow is reported by tlag_insert_records
  r = open_level(e, (uint64_t)((double)(e->hi - e->lo) * e->growth_hint) + 4096);
  if (r) return r;
  e->p.send = (uint32_t*)(uintptr_t)d_send;
  e->p.region_cap = cap_records / n_ranks;
  CK(cudaMemsetAsync(&e->d_ctr->work, 0, 8, e->stream));
  CK(cudaMemsetAsync(e->d_ctr->send_count, 0, sizeof(unsigned long long) * 16, e->stream));
  CK(cudaMemsetAsync(&e->d_ctr->route_overflow, 0, 8, e->stream));   // a failed attempt may be retried with
  CK(cudaMemsetAsync(&e->d_ctr->generated, 0, 8, e->stream));        // larger regions: start from clean counters
  Counters hc;
  float ms = 0;
  r = timed(e, &ms, &hc, [&] { if (hi > lo) CK(launch_wave<1>(e, lo, hi)); return TLAG_OK; });
  if (r) return r;
  e->dev_seconds += ms * 1e-3;
  if (hc.route_overflow) {
    // The caller re-runs this chunk with larger regions and throws this attempt's buffer away -- including the records
    // that did fit, whose fingerprints are now in the routed-fingerprint cache.  Forget them all (the cache is only a
    // filter: an empty one costs redundant records, a stale one loses states).
    if (e->d_sent) CK(cudaMemsetAsync(e->d_sent, 0, (e->p.sent_mask + 1) * 8, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    e->err = "send buffer overflow in tlag_expand_route";
    return TLAG_EOVERFLOW;
  }
  for (uint32_t k = 0; k < n_ranks; ++k) counts[k] = hc.send_count[k];
  return account_wave(e, hc, false, hi - lo, ms, out);
}

extern "C" int tlag_insert_records(tlag_engine* e, uint64_t d_recv, uint64_t n_records, uint32_t, uint64_t* n_new) {
  if (!e) return TLAG_EINVAL;
  Counters hc;
  CK(read_counters(e, &hc));
  const uint64_t before = hc.n_states;
  int r = reserve_level(e, before + n_records + 1024, before + n_records);
  if (r) return r;
  r = open_level(e, before + n_records + 1024 - e->hi);   // the reservation: a store overflow fails this call
  if (r) return r;
  if (n_records) {
    float ms = 0;
    r = timed(e, &ms, &hc, [&] {
      k_insert_records<<<(unsigned)((n_records + 255) / 256), 256, 0, e->stream>>>(e->p, (const uint32_t*)(uintptr_t)d_recv, n_records);
      e->launches++;
      CK(cudaGetLastError());
      return TLAG_OK;
    });
    if (r) return r;
    e->dev_seconds += ms * 1e-3;
  }
  r = overflow_error(e, hc, "state store overflow: raise max_states", "seen-set table full");
  if (r) return r;
  if (n_new) *n_new = hc.n_states - before;
  return TLAG_OK;
}


// ---- peer-memory exchange: set-up and one-call-per-level driver ------------------------------------------------------
static size_t p2p_meta_bytes() { return 16 * sizeof(P2PMeta); }

extern "C" int tlag_p2p_init(tlag_engine* e, uint32_t n_ranks, uint32_t rank, uint64_t cap_records, uint8_t* handle_out64) {
  if (!e || !handle_out64 || n_ranks == 0 || n_ranks > 16 || rank >= n_ranks || cap_records == 0) return TLAG_EINVAL;
  if (e->d_p2p) { e->err = "tlag_p2p_init called twice"; return TLAG_ESTATE; }
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  const uint64_t rw = e->m.words_per_state + 2;
  cap_records = (cap_records + 3) & ~3ULL;                       // regions stay 16-byte aligned
  for (size_t i = 0; i < g_p2p_parked.size() && e->p2p_slot < 0; ++i) {
    P2PParked& c = g_p2p_parked[i];
    if (c.in_use || c.device != e->m.device || c.n_ranks != (int)n_ranks || c.rank != (int)rank || c.rec_words != (int)rw ||
        c.cap != cap_records) continue;
    c.in_use = true;
    e->p2p_slot = (int)i;
    e->d_p2p = c.d_p2p; e->p2p_bytes = c.bytes; e->d_send_own = c.d_send; e->d_tickets = c.d_tickets; e->p2p_seq = c.seq;
  }
  if (e->p2p_slot < 0) {
    const uint64_t inbox_bytes = 2ULL * n_ranks * cap_records * rw * 4;
    e->p2p_bytes = p2p_meta_bytes() + inbox_bytes;
    CK(cudaMalloc(&e->d_p2p, e->p2p_bytes));
    CK(cudaMemset(e->d_p2p, 0, p2p_meta_bytes()));
    CK(cudaMalloc(&e->d_send_own, (uint64_t)n_ranks * cap_records * rw * 4));
    CK(cudaMalloc(&e->d_tickets, 32 * sizeof(unsigned int)));
    CK(cudaMemset(e->d_tickets, 0, 32 * sizeof(unsigned int)));
    P2PParked c;
    memset(&c, 0, sizeof(c));
    c.device = e->m.device; c.n_ranks = (int)n_ranks; c.rank = (int)rank; c.rec_words = (int)rw; c.cap = cap_records;
    c.d_p2p = e->d_p2p; c.bytes = e->p2p_bytes; c.d_send = e->d_send_own; c.d_tickets = e->d_tickets; c.in_use = true;
    g_p2p_parked.push_back(c);
    e->p2p_slot = (int)g_p2p_parked.size() - 1;
  }
  memset(&e->q, 0, sizeof(e->q));
  e->q.n_ranks = (int)n_ranks; e->q.rank = (int)rank; e->q.rec_words = (int)rw;
  e->q.inbox_cap = cap_records; e->q.region_cap = cap_records;
  e->q.send = e->d_send_own;
  e->q.meta = (P2PMeta*)e->d_p2p;
  e->q.inbox = (uint32_t*)((uint8_t*)e->d_p2p + p2p_meta_bytes());
  e->q.tickets = e->d_tickets;
  e->peer_base[rank] = e->d_p2p;
  e->q.peer_meta[rank] = e->q.meta; e->q.peer_inbox[rank] = e->q.inbox;
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, e->d_p2p));
  memcpy(handle_out64, &h, 64);
  e->p.n_ranks = (int)n_ranks; e->p.rank = (int)rank;
  return TLAG_OK;
}

extern "C" int tlag_p2p_attach(tlag_engine* e, uint32_t peer, const uint8_t* handle64) {
  if (!e || !handle64 || !e->d_p2p || peer >= (uint32_t)e->q.n_ranks) return TLAG_EINVAL;
  if ((int)peer == e->q.rank) return TLAG_OK;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  void* base = nullptr;
  P2PParked* c = e->p2p_slot >= 0 ? &g_p2p_parked[e->p2p_slot] : nullptr;
  if (c && c->peer_ok[peer] && memcmp(c->peer_handle[peer], handle64, 64) == 0) {
    base = c->peer_base[peer];                                  // the peer parked and re-adopted the same inbox
  } else {
    if (c && c->peer_ok[peer]) { cudaIpcCloseMemHandle(c->peer_base[peer]); c->peer_ok[peer] = false; }
    CK(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
    if (c) { c->peer_base[peer] = base; memcpy(c->peer_handle[peer], handle64, 64); c->peer_ok[peer] = true; }
  }
  e->peer_base[peer] = base;
  e->q.peer_meta[peer] = (P2PMeta*)base;
  e->q.peer_inbox[peer] = (uint32_t*)((uint8_t*)base + p2p_meta_bytes());
  int ready = 1;
  for (int r = 0; r < e->q.n_ranks; ++r) if (!e->peer_base[r]) ready = 0;
  e->p2p_ready = ready != 0;
  return TLAG_OK;
}

// One BFS level on this rank: the frontier shard in n_chunks chunks of chunk_states states; per chunk the expand
// kernels (successors bucketed by owner), k_push (NVLink stores into the owners' inboxes) and k_insert_inbox (this
// rank's share of the next frontier).  Every rank must call it with the same n_chunks (ranks with a shorter frontier
// run empty chunks: the inbox protocol counts chunks).  One host synchronisation, at the end.
extern "C" int tlag_p2p_level(tlag_engine* e, uint64_t n_chunks, uint64_t chunk_states, uint64_t expect_inbound,
                              tlag_wave_stats* out) {
  if (!e || chunk_states == 0) return TLAG_EINVAL;
#ifdef TLAG_NO_BFS
  TLAG_NO_BFS(e);
#endif
  if (!e->p2p_ready && e->q.n_ranks > 1) { e->err = "tlag_p2p_level before every peer was attached"; return TLAG_ESTATE; }
  if (out) memset(out, 0, sizeof(*out));
  start_search(e);
  const uint32_t n_ranks = (uint32_t)e->q.n_ranks;
  // room for what may arrive this level (the caller passes the all-reduced estimate; at least the heuristic)
  uint64_t expect = (uint64_t)((double)(e->hi - e->lo) * e->growth_hint) + 4096;
  if (expect_inbound > expect) expect = expect_inbound;
  Counters hc;
  CK(read_counters(e, &hc));
  const uint64_t before = hc.n_states;
  e->p2p_level_start = before; e->p2p_level_generated = 0;
  int r = reserve_level(e, before + expect, before + expect);
  if (r) return r;
  r = open_level(e, before + expect - e->hi);    // the level's reservation: a store overflow fails the level
  if (r) return r;
  e->p.n_ranks = (int)n_ranks; e->p.rank = e->q.rank;
  r = ensure_sent_cache(e);
  if (r) return r;
  e->p.send = e->d_send_own;
  e->p.region_cap = e->q.region_cap;
  CK(cudaMemsetAsync(&e->d_ctr->route_overflow, 0, 8, e->stream));
  CK(cudaMemsetAsync(&e->d_ctr->generated, 0, 8, e->stream));
  const unsigned push_blocks = 64, ins_blocks = (unsigned)e->sm_count * 4;
  float ms = 0;
  r = timed(e, &ms, &hc, [&] {
    for (uint64_t c = 0; c < n_chunks; ++c) {
      const unsigned long long seq = ++e->p2p_seq;
      uint64_t lo = e->lo + c * chunk_states, hi = lo + chunk_states;
      if (lo > e->hi) lo = e->hi;
      if (hi > e->hi) hi = e->hi;
      CK(cudaMemsetAsync(&e->d_ctr->work, 0, 8, e->stream));
      CK(cudaMemsetAsync(e->d_ctr->send_count, 0, sizeof(unsigned long long) * 16, e->stream));
      if (hi > lo) CK(launch_wave<1>(e, lo, hi));
      k_push<<<dim3(push_blocks, n_ranks), 256, 0, e->stream>>>(e->q, e->d_ctr, seq);
      k_insert_inbox<<<ins_blocks, 256, 0, e->stream>>>(e->p, e->q, seq);
      e->launches += 2;
      CK(cudaGetLastError());
    }
    return TLAG_OK;
  });
  if (r) return r;
  e->dev_seconds += ms * 1e-3;
  if (hc.route_overflow) { e->err = "send region overflow in tlag_p2p_level: use smaller chunks or larger regions"; return TLAG_EOVERFLOW; }
  r = overflow_error(e, hc, "state store overflow in tlag_p2p_level", "seen-set table full in tlag_p2p_level");
  if (r) return r;
  e->p2p_level_generated = hc.generated;
  r = account_wave(e, hc, false, e->hi - e->lo, ms, out);
  if (r) return r;
  if (out) out->discovered = hc.n_states - before;
  note_growth(e, e->hi - e->lo, hc.n_states - before);
  return TLAG_OK;
}

// Undo the level tlag_p2p_level just ran on this rank (some rank's send regions overflowed: every rank rolls back and
// the host re-runs the level with smaller chunks).  The states the level appended are dropped, the seen-set is rebuilt
// from the store, the routed-fingerprint cache is emptied; the inbox chunk numbering simply continues.
extern "C" int tlag_p2p_rollback(tlag_engine* e) {
  if (!e || !e->d_p2p) return TLAG_EINVAL;
  int r = rollback_wave(e, e->p2p_level_start, e->p2p_level_start + 4096);
  if (r) return r;
  if (e->d_sent) CK(cudaMemsetAsync(e->d_sent, 0, (e->p.sent_mask + 1) * 8, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  e->generated -= e->p2p_level_generated;
  e->p2p_level_generated = 0;
  e->verdict = TLAG_V_RUNNING; e->detail = e->detail2 = 0; e->viol_idx = 0;
  return TLAG_OK;
}

extern "C" int tlag_advance_level(tlag_engine* e, tlag_wave_stats* out) {
  if (!e) return TLAG_EINVAL;
  if (out) memset(out, 0, sizeof(*out));
  Counters hc;
  CK(read_counters(e, &hc));
  return close_level(e, hc.n_states, true, out);
}

// ---- random simulation (include/tlag.h: tlag_simulate) ------------------------------------------------------------
#if defined(TLAG_SLICED_INC)
#if defined(TLAG_SL_SIM)
static cudaError_t launch_sim_step(tlag_engine* e, const DevParams& p, const SimParams& s, uint64_t n) {
  const unsigned blocks = sl_blocks(e, n);
  if (p.n_inv > 0)
    for (int j = 0; kSlSimInv[j]; ++j) { kSlSimInv[j](&p, &s, n, blocks, e->stream); e->launches++; }
  for (int j = 0; kSlSimNext[j]; ++j) { kSlSimNext[j](&p, &s, n, blocks, e->stream); e->launches++; }
  return cudaGetLastError();
}
#endif
#else
static cudaError_t launch_sim_step(tlag_engine* e, const DevParams& p, const SimParams& s, uint64_t n) {
  return launch_vm(e, vm_variant(e, [](auto f, auto sm, auto l) { return k_sim<f, sm, l>; }), n, p, s, n);
}
#endif

#if !defined(TLAG_SLICED_INC) || defined(TLAG_SL_SIM)
// The batch's buffers: sim_B walks x sim_D rows of history, the per-walk state, and the distinct initial states in the
// order the caller seeded them (first occurrence)
static int sim_buffers(tlag_engine* e, uint64_t B, uint64_t D) {
  const uint64_t W = e->m.words_per_state;
  if (B * D > e->sim_B * e->sim_D || B > e->sim_B) {
    dfree(e, e->d_hist); dfree(e, e->d_act); dfree(e, e->d_sstat); dfree(e, e->d_ssucc); dfree(e, e->d_scnt); dfree(e, e->d_slen);
    e->d_hist = nullptr; e->d_act = nullptr; e->d_sstat = e->d_ssucc = nullptr; e->d_scnt = e->d_slen = nullptr;
    e->sim_B = e->sim_D = 0;
    CK(dmalloc(e, &e->d_hist, B * D * W * 4));
    CK(dmalloc(e, &e->d_act, B * D * 2));
    CK(dmalloc(e, &e->d_sstat, B));
    CK(dmalloc(e, &e->d_ssucc, B));
    CK(dmalloc(e, &e->d_scnt, B * 4));
    CK(dmalloc(e, &e->d_slen, B * 4));
  }
  e->sim_B = B; e->sim_D = D;
  if (!e->d_sctl) CK(cudaMalloc(&e->d_sctl, sizeof(SimCtl)));
  if (!e->d_sinit) {
    std::vector<uint32_t> distinct;
    std::unordered_set<std::string> seen;
    const uint64_t n = e->h_init.size() / W;
    for (uint64_t i = 0; i < n; ++i)
      if (seen.insert(std::string((const char*)(e->h_init.data() + i * W), W * 4)).second)
        distinct.insert(distinct.end(), e->h_init.begin() + i * W, e->h_init.begin() + (i + 1) * W);
    e->sim_n_init = distinct.size() / W;
    if (!e->sim_n_init) { e->err = "tlag_simulate: no initial state was seeded"; return TLAG_ESTATE; }
    CK(dmalloc(e, &e->d_sinit, distinct.size() * 4));
    CK(cudaMemcpyAsync(e->d_sinit, distinct.data(), distinct.size() * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  return TLAG_OK;
}

static SimParams sim_params(tlag_engine* e, const tlag_sim_params* sp, uint64_t first) {
  SimParams s;
  memset(&s, 0, sizeof(s));
  s.seed = sp->seed; s.first = first; s.depth = sp->depth; s.B = (uint32_t)e->sim_B; s.flags = sp->flags;
  s.hist = e->d_hist; s.act = e->d_act; s.status = e->d_sstat; s.cnt = e->d_scnt; s.len = e->d_slen; s.ctl = e->d_sctl;
  return s;
}
#endif

extern "C" int tlag_simulate(tlag_engine* e, const tlag_sim_params* sp, tlag_sim_result* out) {
  if (!e || !sp || !out) return TLAG_EINVAL;
  memset(out, 0, sizeof(*out));
#if defined(TLAG_SLICED_INC) && !defined(TLAG_SL_SIM)
  e->err = "this library has no simulation kernels: build the model's simulation library (build_sliced_library(cm, simulate=True))";
  return TLAG_EINVAL;
#else
  if (sp->depth < 1 || sp->depth > 1000000 || sp->num_walks == 0) { e->err = "tlag_simulate: depth must be 1..10^6 and num_walks > 0"; return TLAG_EINVAL; }
  if (e->m.n_actions > 32767) { e->err = "tlag_simulate: more than 32767 actions"; return TLAG_EINVAL; }
  if (sp->first_walk + sp->num_walks < sp->first_walk) { e->err = "tlag_simulate: walk ids past 2^64"; return TLAG_EINVAL; }
  const uint64_t W = e->m.words_per_state, D = sp->depth;
  const uint64_t B = tlag_sim_batch((uint32_t)W, sp->depth, sp->num_walks);
  int r = sim_buffers(e, B, D);
  if (r) return r;
  out->verdict = TLAG_V_OK;
  out->batch_walks = B;
  float total_ms = 0;
  for (uint64_t done = 0; done < sp->num_walks; done += B) {
    const uint64_t n = sp->num_walks - done < B ? sp->num_walks - done : B, first = sp->first_walk + done;
    e->sim_n = n; e->sim_first = first;
    CK(reset_counters(e, 0));
    CK(cudaMemsetAsync(e->d_sctl, 0, sizeof(SimCtl), e->stream));
    CK(cudaMemsetAsync(e->d_ssucc, 0, n, e->stream));
    SimParams s = sim_params(e, sp, first);
    DevParams p = e->p;
    p.succ_flag = e->d_ssucc;
    Counters hc;
    float ms = 0;
    r = timed(e, &ms, &hc, [&] {
      const unsigned blocks = (unsigned)((n + 255) / 256);
      k_sim_init<<<blocks, 256, 0, e->stream>>>(s, e->d_sinit, e->sim_n_init, (int)W, n);
      e->launches++;
      CK(cudaGetLastError());
      for (uint32_t t = 0; t < sp->depth; ++t) {
        s.t = t;
        p.states = e->d_hist + (uint64_t)t * B * W;
        CK(launch_sim_step(e, p, s, n));
        k_sim_end<<<blocks, 256, 0, e->stream>>>(p, s, n);
        e->launches++;
        CK(cudaGetLastError());
      }
      return TLAG_OK;
    });
    if (r) return r;
    total_ms += ms;
    SimCtl hs;
    CK(cudaMemcpy(&hs, e->d_sctl, sizeof(hs), cudaMemcpyDeviceToHost));
    out->generated += hc.generated;
    out->checked += hs.checked;
    out->behaviours += n;
    if (hs.stopped) {
      const int saved = e->verdict;
      collect_violations(e, hc);
      out->verdict = e->verdict; out->detail = e->detail; out->detail2 = e->detail2;
      out->walk = first + e->viol_idx; out->step = hs.stopped - 1;
      e->verdict = saved;
      break;
    }
  }
  out->device_ms = total_ms;
  return TLAG_OK;
#endif
}

#if !defined(TLAG_SLICED_INC) || defined(TLAG_SL_SIM)
// walk (a global id) -> its column in the last batch
static int sim_column(tlag_engine* e, uint64_t walk, uint64_t n, uint64_t* col) {
  if (!e->sim_n || walk < e->sim_first || walk + n > e->sim_first + e->sim_n || walk + n < walk) {
    e->err = "no such walk in the last batch of tlag_simulate";
    return TLAG_EINVAL;
  }
  *col = walk - e->sim_first;
  return TLAG_OK;
}
#endif

extern "C" int tlag_sim_read(tlag_engine* e, uint64_t walk, uint64_t n, uint32_t* states_out, int16_t* actions_out,
                             uint32_t* len_out) {
  if (!e) return TLAG_EINVAL;
#if defined(TLAG_SLICED_INC) && !defined(TLAG_SL_SIM)
  e->err = "this library has no simulation kernels";
  return TLAG_EINVAL;
#else
  uint64_t c = 0;
  int r = sim_column(e, walk, n, &c);
  if (r) return r;
  const uint64_t W = e->m.words_per_state, B = e->sim_B, D = e->sim_D;
  if (states_out)
    CK(cudaMemcpy2DAsync(states_out, n * W * 4, e->d_hist + c * W, B * W * 4, n * W * 4, D, cudaMemcpyDeviceToHost, e->stream));
  if (actions_out)
    CK(cudaMemcpy2DAsync(actions_out, n * 2, e->d_act + c, B * 2, n * 2, D, cudaMemcpyDeviceToHost, e->stream));
  if (len_out) CK(cudaMemcpyAsync(len_out, e->d_slen + c, n * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
#endif
}

extern "C" int tlag_sim_trace(tlag_engine* e, uint64_t walk, uint32_t* states_out, int32_t* actions_out, uint32_t* len_inout) {
  if (!e || !len_inout) return TLAG_EINVAL;
#if defined(TLAG_SLICED_INC) && !defined(TLAG_SL_SIM)
  e->err = "this library has no simulation kernels";
  return TLAG_EINVAL;
#else
  uint64_t c = 0;
  int r = sim_column(e, walk, 1, &c);
  if (r) return r;
  const uint64_t W = e->m.words_per_state, B = e->sim_B;
  uint32_t len = 0;
  CK(cudaMemcpy(&len, e->d_slen + c, 4, cudaMemcpyDeviceToHost));
  if (len > *len_inout) { *len_inout = len; e->err = "tlag_sim_trace: buffer too small"; return TLAG_EINVAL; }
  std::vector<int16_t> a(len);
  if (len && states_out)
    CK(cudaMemcpy2DAsync(states_out, W * 4, e->d_hist + c * W, B * W * 4, W * 4, len, cudaMemcpyDeviceToHost, e->stream));
  if (len) CK(cudaMemcpy2DAsync(a.data(), 2, e->d_act + c, B * 2, 2, len, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (actions_out) for (uint32_t i = 0; i < len; ++i) actions_out[i] = a[i];
  *len_inout = len;
  return TLAG_OK;
#endif
}

extern "C" int tlag_sim_digest(tlag_engine* e, uint64_t* xor_out, uint64_t* sum_out) {
  if (!e || !xor_out || !sum_out) return TLAG_EINVAL;
#if defined(TLAG_SLICED_INC) && !defined(TLAG_SL_SIM)
  e->err = "this library has no simulation kernels";
  return TLAG_EINVAL;
#else
  if (!e->sim_n) { e->err = "tlag_sim_digest before tlag_simulate"; return TLAG_ESTATE; }
  tlag_sim_params sp;
  memset(&sp, 0, sizeof(sp));
  sp.depth = (uint32_t)e->sim_D;
  const SimParams s = sim_params(e, &sp, e->sim_first);
  return read_digest(e, xor_out, sum_out, [&] {
    k_sim_digest<<<e->sm_count * 8, 256, 0, e->stream>>>(s, (int)e->m.words_per_state, e->sim_n, e->d_dig);
    e->launches++;
    CK(cudaGetLastError());
    return TLAG_OK;
  });
#endif
}

// ---- state graph (include/tlag.h: tlag_build_graph) -------------------------------------------------------------------
#if !defined(TLAG_SL_SIM)
static cudaError_t launch_graph(tlag_engine* e, const GraphParams& g, uint64_t hi) {
#if defined(TLAG_SLICED_INC)   // the one variant of the edge pass the policy picks for the library's model
  const auto fn = k_graph<vm_frame_class(TLAG_SL_FRAME), vm_code_in_smem(TLAG_SL_FRAME, TLAG_NATIVE_CODE_LEN), false>;
#else
  const auto fn = vm_variant(e, [](auto f, auto s, auto l) { return k_graph<f, s, l>; });
#endif
  return launch_vm(e, fn, hi - g.first, e->p, g, hi);
}

static unsigned bits_for(uint64_t n) {   // bits of n - 1, at least 1
  unsigned b = 1;
  while (b < 64 && (1ULL << b) < n) ++b;
  return b;
}

// The resident CSR holds at least `need` edges (geometric growth up to `bound`, contents kept)
static int graph_reserve(tlag_engine* e, uint64_t need, uint64_t bound) {
  if (need <= e->g_cap) return TLAG_OK;
  uint64_t cap = e->g_cap * 2 > need ? e->g_cap * 2 : need;
  if (cap > bound && bound >= need) cap = bound;
  uint32_t *nd = nullptr, *na = nullptr;
  if (dmalloc(e, &nd, cap * 4) != cudaSuccess || dmalloc(e, &na, cap * 4) != cudaSuccess) {
    cudaGetLastError();
    dfree(e, nd); dfree(e, na);
    e->err = "tlag_build_graph: not enough device memory for the state graph";
    return TLAG_ENOMEM;
  }
  if (e->g_edges) {
    CK(cudaMemcpyAsync(nd, e->d_gdst, e->g_edges * 4, cudaMemcpyDeviceToDevice, e->stream));
    CK(cudaMemcpyAsync(na, e->d_gact, e->g_edges * 4, cudaMemcpyDeviceToDevice, e->stream));
  }
  dfree(e, e->d_gdst); dfree(e, e->d_gact);
  e->d_gdst = nd; e->d_gact = na; e->g_cap = cap;
  return TLAG_OK;
}

// The passes of tlag_build_graph over n_states stored rows, n_exp of them expanded; scratch buffers freed by the caller
struct GraphScratch { uint32_t* row_of_slot = nullptr; unsigned long long* keys = nullptr; void* tmp = nullptr; GraphCtl* ctl = nullptr; };

static int graph_passes(tlag_engine* e, GraphScratch& sc, uint64_t n_states, uint64_t n_exp) {
  const uint64_t slots = e->p.mask + 1;
  const unsigned abits = bits_for(e->m.n_actions ? e->m.n_actions : 1);
  if (abits > 24) { e->err = "tlag_build_graph: more than 2^24 actions"; return TLAG_EINVAL; }
  const uint64_t max_rows = 1ULL << (32 - abits);         // (s - first) | t | a fit one 64-bit key
  uint64_t cap = e->graph_edges;
  size_t sort_tmp = 0, uniq_tmp = 0;
  {
    cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
    cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, k, (unsigned long long)cap);
    cub::DeviceSelect::Unique(nullptr, uniq_tmp, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                              (unsigned long long*)nullptr, (unsigned long long)cap);
  }
  size_t tmp_bytes = ((sort_tmp > uniq_tmp ? sort_tmp : uniq_tmp) + 255) & ~(size_t)255;   // then the count of Unique
  if (dmalloc(e, &sc.row_of_slot, slots * 4) != cudaSuccess || dmalloc(e, &sc.keys, cap * 16) != cudaSuccess ||
      dmalloc(e, &sc.tmp, tmp_bytes + 256) != cudaSuccess || dmalloc(e, &sc.ctl, sizeof(GraphCtl)) != cudaSuccess) {
    cudaGetLastError();
    e->err = "tlag_build_graph: not enough device memory for the index and edge buffers";
    return TLAG_ENOMEM;
  }
  if (dmalloc(e, &e->d_goff, (n_states + 1) * 8) != cudaSuccess) {
    cudaGetLastError();
    e->err = "tlag_build_graph: not enough device memory for the state graph";
    return TLAG_ENOMEM;
  }
  e->g_states = n_states; e->g_expanded = n_exp;
  // every edge was an EMIT the search counted in `generated`: reserve that many at once (no copy of a multi-GB CSR
  // while it grows), and grow from 2^20 edges when it does not fit
  const uint64_t init_gen = e->h_init.size() / e->m.words_per_state;
  const uint64_t bound = e->generated > init_gen ? e->generated - init_gen : 0;
  int r = graph_reserve(e, bound ? bound : 1, bound);
  if (r == TLAG_ENOMEM) r = graph_reserve(e, (1ULL << 20) < bound ? (1ULL << 20) : (bound ? bound : 1), bound);
  if (r) return r;

  // index pass: row_of_slot[slot of row i's fingerprint] = i
  CK(cudaMemsetAsync(sc.ctl, 0, sizeof(GraphCtl), e->stream));
  if (n_states) {
    k_graph_index<<<(unsigned)((n_states + 255) / 256), 256, 0, e->stream>>>(e->p, n_states, sc.row_of_slot, sc.ctl);
    e->launches++;
    CK(cudaGetLastError());
  }
  // chunks of expanded rows, sized from the search's successors per expanded state; a chunk whose edges overflow the
  // buffer is run again with half the rows (a single row: with a buffer as big as its count)
  const double ratio = n_exp ? (double)bound / (double)n_exp : 1.0;
  uint64_t rows = (uint64_t)((double)cap / (ratio + 1.0));
  GraphCtl hc;
  for (uint64_t first = 0; first < n_exp;) {
    if (rows < 1) rows = 1;
    if (rows > max_rows) rows = max_rows;
    const uint64_t n = n_exp - first < rows ? n_exp - first : rows;
    GraphParams g;
    g.row_of_slot = sc.row_of_slot; g.first = first; g.keys = sc.keys; g.cap = cap; g.abits = abits; g.ctl = sc.ctl;
    CK(cudaMemsetAsync(&sc.ctl->n, 0, 8, e->stream));
    CK(launch_graph(e, g, first + n));
    CK(cudaMemcpyAsync(&hc, sc.ctl, sizeof(hc), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    if (hc.missing) {
      e->err = "tlag_build_graph: a stored state or a successor of an expanded state is not in the seen-set (store and "
               "seen-set disagree)";
      return TLAG_ESTATE;
    }
    if (hc.bad) { e->err = "tlag_build_graph: Next trapped while its successors were enumerated again"; return TLAG_ESTATE; }
    if (hc.n > cap) {
      if (n > 1) { rows = n / 2; continue; }
      dfree(e, sc.keys); dfree(e, sc.tmp); sc.keys = nullptr; sc.tmp = nullptr;
      cap = hc.n;
      cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
      cub::DeviceRadixSort::SortKeys(nullptr, sort_tmp, k, (unsigned long long)cap);
      cub::DeviceSelect::Unique(nullptr, uniq_tmp, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                (unsigned long long*)nullptr, (unsigned long long)cap);
      tmp_bytes = ((sort_tmp > uniq_tmp ? sort_tmp : uniq_tmp) + 255) & ~(size_t)255;
      if (dmalloc(e, &sc.keys, cap * 16) != cudaSuccess || dmalloc(e, &sc.tmp, tmp_bytes + 256) != cudaSuccess) {
        cudaGetLastError();
        e->err = "tlag_build_graph: not enough device memory for the edges of one state";
        return TLAG_ENOMEM;
      }
      continue;
    }
    // sort by (s, t, a), drop duplicates, append to the CSR
    const uint64_t m = hc.n;
    unsigned long long* ka = sc.keys; unsigned long long* kb = sc.keys + cap;
    unsigned long long* d_nsel = (unsigned long long*)((uint8_t*)sc.tmp + tmp_bytes);
    uint64_t nu = 0;
    if (m) {
      cub::DoubleBuffer<unsigned long long> k(ka, kb);
      size_t tb = tmp_bytes;
      if (cub::DeviceRadixSort::SortKeys(sc.tmp, tb, k, (unsigned long long)m, 0, (int)(32 + abits + bits_for(n)),
                                         e->stream) != cudaSuccess) { e->err = "cub sort failed"; return TLAG_ECUDA; }
      unsigned long long* sorted = k.Current();
      unsigned long long* uniq = sorted == ka ? kb : ka;
      tb = tmp_bytes;
      if (cub::DeviceSelect::Unique(sc.tmp, tb, sorted, uniq, d_nsel, (unsigned long long)m, e->stream) != cudaSuccess) {
        e->err = "cub unique failed"; return TLAG_ECUDA;
      }
      e->launches += 2;
      CK(cudaMemcpyAsync(&nu, d_nsel, 8, cudaMemcpyDeviceToHost, e->stream));
      CK(cudaStreamSynchronize(e->stream));
      r = graph_reserve(e, e->g_edges + nu, bound);
      if (r) return r;
      k_graph_split<<<(unsigned)((nu + 255) / 256), 256, 0, e->stream>>>(
          uniq, nu, abits, e->d_gdst + e->g_edges, e->d_gact + e->g_edges);
      k_graph_rows<<<(unsigned)((n + 1 + 255) / 256), 256, 0, e->stream>>>(uniq, nu, n, 32 + abits, e->g_edges,
                                                                          e->d_goff + first);
      e->launches += 2;
    } else {
      k_fill_u64<<<(unsigned)((n + 1 + 255) / 256), 256, 0, e->stream>>>(e->d_goff + first, n + 1, e->g_edges);
      e->launches++;
    }
    CK(cudaGetLastError());
    e->g_edges += nu;
    first += n;
  }
  // rows past the expanded ones have no edges
  k_fill_u64<<<(unsigned)((n_states - n_exp + 1 + 255) / 256), 256, 0, e->stream>>>(e->d_goff + n_exp, n_states - n_exp + 1,
                                                                                     e->g_edges);
  e->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(&hc, sc.ctl, sizeof(hc), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (hc.missing) { e->err = "tlag_build_graph: a stored state is not in the seen-set"; return TLAG_ESTATE; }
  return TLAG_OK;
}
// The CSR keeps the edges it holds, not the bound it was reserved for (kept as it is without memory for the copy)
static int graph_shrink(tlag_engine* e) {
  if (e->g_cap <= e->g_edges + e->g_edges / 8 + (1ULL << 20)) return TLAG_OK;
  const uint64_t cap = e->g_edges ? e->g_edges : 1;
  uint32_t *nd = nullptr, *na = nullptr;
  if (dmalloc(e, &nd, cap * 4) != cudaSuccess || dmalloc(e, &na, cap * 4) != cudaSuccess) {
    cudaGetLastError();
    dfree(e, nd); dfree(e, na);
    return TLAG_OK;
  }
  CK(cudaMemcpyAsync(nd, e->d_gdst, e->g_edges * 4, cudaMemcpyDeviceToDevice, e->stream));
  CK(cudaMemcpyAsync(na, e->d_gact, e->g_edges * 4, cudaMemcpyDeviceToDevice, e->stream));
  dfree(e, e->d_gdst); dfree(e, e->d_gact);
  e->d_gdst = nd; e->d_gact = na; e->g_cap = cap;
  return TLAG_OK;
}
#endif

extern "C" int tlag_build_graph(tlag_engine* e, tlag_graph_info* out) {
  if (!e || !out) return TLAG_EINVAL;
  memset(out, 0, sizeof(*out));
#if defined(TLAG_SL_SIM)
  e->err = "this library holds the model's simulation kernels only: the state graph needs its BFS library";
  return TLAG_EINVAL;
#else
  if (e->m.flags & TLAG_F_EXACT) { e->err = "tlag_build_graph: not on a TLAG_F_EXACT (sequential replay) engine"; return TLAG_EINVAL; }
  if (e->p.n_ranks > 1 || e->q.n_ranks > 1 || e->p2p_slot >= 0) {
    e->err = "tlag_build_graph: the engine holds one shard of a multi-GPU search";
    return TLAG_EINVAL;
  }
  if (e->h_init.empty()) { e->err = "tlag_build_graph before tlag_seed"; return TLAG_ESTATE; }
  if (e->verdict == TLAG_V_EVAL_ERROR || e->kg_verdict == TLAG_V_EVAL_ERROR) {
    e->err = "tlag_build_graph: the search stopped at an evaluation trap, its successor sets are incomplete";
    return TLAG_ESTATE;
  }
  release_graph(e);
  Counters hc;
  CK(read_counters(e, &hc));
  int r = sync_store(e, hc.n_states);
  if (r) return r;
  const uint64_t n_states = hc.n_states, n_exp = e->lo;
  // the graph comes first: the clustering and discovery buffers are allocated again by the next level that needs them,
  // and the routed-fingerprint cache is only a filter
  if (!e->disc_open) { dfree(e, e->d_disc); e->d_disc = nullptr; e->disc_bytes = 0; }
  dfree(e, e->d_sort); e->d_sort = nullptr; e->sort_bytes = 0;
  dfree(e, e->d_rset); e->d_rset = nullptr; e->rset_bytes = 0;
  dfree(e, e->d_sent); e->d_sent = nullptr; e->p.sent_cache = nullptr;
  GraphScratch sc;
  float ms = 0;
  r = timed(e, &ms, nullptr, [&] { return graph_passes(e, sc, n_states, n_exp); });
  dfree(e, sc.row_of_slot); dfree(e, sc.keys); dfree(e, sc.tmp); dfree(e, sc.ctl);
  if (!r) r = graph_shrink(e);
  if (r) { cudaStreamSynchronize(e->stream); release_graph(e); return r; }
  CK(cudaStreamSynchronize(e->stream));
  e->g_ready = true;
  out->n_states = n_states; out->n_expanded = n_exp; out->n_edges = e->g_edges; out->device_ms = ms;
  return TLAG_OK;
#endif
}

extern "C" int tlag_read_graph(tlag_engine* e, uint64_t first, uint64_t n, uint64_t* off_out, uint32_t* dst_out,
                               int32_t* act_out) {
  if (!e || !off_out) return TLAG_EINVAL;
  if (!e->g_ready) { e->err = "no state graph: tlag_build_graph first (tlag_seed, tlag_step, tlag_run and tlag_restart release it)"; return TLAG_ESTATE; }
  if (first > e->g_states || n > e->g_states - first) { e->err = "tlag_read_graph: rows beyond the state graph"; return TLAG_EINVAL; }
  CK(cudaMemcpyAsync(off_out, e->d_goff + first, (n + 1) * 8, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  const uint64_t o0 = off_out[0], m = off_out[n] - o0;
  for (uint64_t i = 0; i <= n; ++i) off_out[i] -= o0;
  if (dst_out && m) CK(cudaMemcpyAsync(dst_out, e->d_gdst + o0, m * 4, cudaMemcpyDeviceToHost, e->stream));
  if (act_out && m) CK(cudaMemcpyAsync(act_out, e->d_gact + o0, m * 4, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return TLAG_OK;
}

extern "C" int tlag_graph_digest(tlag_engine* e, uint64_t* xor_out, uint64_t* sum_out) {
  if (!e || !xor_out || !sum_out) return TLAG_EINVAL;
#if defined(TLAG_SL_SIM)
  e->err = "this library holds the model's simulation kernels only";
  return TLAG_EINVAL;
#else
  if (!e->g_ready) { e->err = "no state graph: tlag_build_graph first"; return TLAG_ESTATE; }
  return read_digest(e, xor_out, sum_out, [&] {
    if (e->g_expanded) {
      k_graph_digest<<<e->sm_count * 8, 256, 0, e->stream>>>(e->p, e->d_goff, e->d_gdst, e->d_gact, e->g_expanded, e->d_dig);
      e->launches++;
      CK(cudaGetLastError());
    }
    return TLAG_OK;
  });
#endif
}

// ---- liveness labels (include/tlag.h: tlag_label_graph, tlag_graph_view) -------------------------------------------------
#if !defined(TLAG_SL_SIM)
template <bool EDGES>
static cudaError_t launch_label(tlag_engine* e, const LabelParams& l) {
#if defined(TLAG_SLICED_INC)   // the one frame class of the library's model, as its k_graph
  const auto fn = k_label<vm_frame_class(TLAG_SL_FRAME), EDGES>;
#else
  const auto fn = vm_variant(e, [](auto f, auto, auto) { return k_label<f, EDGES>; });
#endif
  return launch_vm_smem(e, 0, fn, l.n, e->p, l);
}
#endif

extern "C" int tlag_label_graph(tlag_engine* e, const tlag_label_program* lp, float* device_ms) {
  if (!e || !lp) return TLAG_EINVAL;
#if defined(TLAG_SL_SIM)
  e->err = "this library holds the model's simulation kernels only";
  return TLAG_EINVAL;
#else
  if (!e->g_ready) { e->err = "no state graph: tlag_build_graph first"; return TLAG_ESTATE; }
  if (!lp->code || !lp->code_len || lp->entry_states >= lp->code_len || lp->entry_edges >= lp->code_len ||
      lp->n_state_preds > 32 || lp->n_edge_preds > 32 || (lp->cpool_len && !lp->cpool)) {
    e->err = "tlag_label_graph: missing program, an entry outside it, or more than 32 state or edge predicates";
    return TLAG_EINVAL;
  }
  EnabledMap em;
  for (int b = 0; b < 32; ++b) {
    em.en[b] = lp->en_bit[b]; em.nen[b] = lp->nen_bit[b];
    if ((em.en[b] < 32 || em.nen[b] < 32) && (uint32_t)b >= lp->n_edge_preds) {
      e->err = "tlag_label_graph: an ENABLED bit of an edge predicate the program does not have";
      return TLAG_EINVAL;
    }
    if ((em.en[b] != 0xFF && em.en[b] >= 32) || (em.nen[b] != 0xFF && em.nen[b] >= 32)) {
      e->err = "tlag_label_graph: an ENABLED bit past bit 31";
      return TLAG_EINVAL;
    }
  }
  dfree(e, e->d_slab); dfree(e, e->d_elab);
  e->d_slab = e->d_elab = nullptr;
  uint64_t* code = nullptr; int32_t* cpool = nullptr; unsigned long long* bad = nullptr;
  if (dmalloc(e, &e->d_slab, (e->g_states ? e->g_states : 1) * 4) != cudaSuccess ||
      dmalloc(e, &e->d_elab, (e->g_edges ? e->g_edges : 1) * 4) != cudaSuccess ||
      dmalloc(e, &code, (uint64_t)lp->code_len * 8) != cudaSuccess ||
      dmalloc(e, &cpool, (uint64_t)(lp->cpool_len ? lp->cpool_len : 1) * 4) != cudaSuccess ||
      dmalloc(e, &bad, 8) != cudaSuccess) {
    cudaGetLastError();
    dfree(e, code); dfree(e, cpool); dfree(e, bad);
    dfree(e, e->d_slab); dfree(e, e->d_elab);
    e->d_slab = e->d_elab = nullptr;
    e->err = "tlag_label_graph: not enough device memory for the labels";
    return TLAG_ENOMEM;
  }
  float ms = 0;
  unsigned long long hbad = 0;
  int r = timed(e, &ms, nullptr, [&] {
    CK(cudaMemcpyAsync(code, lp->code, (uint64_t)lp->code_len * 8, cudaMemcpyHostToDevice, e->stream));
    if (lp->cpool_len) CK(cudaMemcpyAsync(cpool, lp->cpool, (uint64_t)lp->cpool_len * 4, cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemsetAsync(bad, 0, 8, e->stream));
    LabelParams l;
    l.code = code; l.cpool = cpool; l.off = e->d_goff; l.dst = e->d_gdst; l.rows = e->g_states; l.bad = bad;
    l.entry = lp->entry_states; l.all = lp->n_state_preds == 32 ? 0xFFFFFFFFu : (1u << lp->n_state_preds) - 1;
    l.n = e->g_states; l.out = e->d_slab;
    if (l.n) CK(launch_label<false>(e, l));
    l.entry = lp->entry_edges; l.all = lp->n_edge_preds == 32 ? 0xFFFFFFFFu : (1u << lp->n_edge_preds) - 1;
    l.n = e->g_edges; l.out = e->d_elab;
    if (l.n) CK(launch_label<true>(e, l));
    if (e->g_states) {
      k_label_enabled<<<e->sm_count * 8, 256, 0, e->stream>>>(e->d_goff, e->d_elab, e->g_states, em, e->d_slab);
      e->launches++;
      CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(&hbad, bad, 8, cudaMemcpyDeviceToHost, e->stream));
    return TLAG_OK;
  });
  dfree(e, code); dfree(e, cpool); dfree(e, bad);
  if (!r) CK(cudaStreamSynchronize(e->stream));
  if (!r && hbad) { e->err = "tlag_label_graph: a label predicate trapped (it cannot be evaluated on some state or edge)"; r = TLAG_EEVAL; }
  if (r) { dfree(e, e->d_slab); dfree(e, e->d_elab); e->d_slab = e->d_elab = nullptr; return r; }
  if (device_ms) *device_ms = ms;
  return TLAG_OK;
#endif
}

extern "C" int tlag_graph_view(tlag_engine* e, tlag_graph_dev* out) {
  if (!e || !out) return TLAG_EINVAL;
  memset(out, 0, sizeof(*out));
  if (!e->g_ready) { e->err = "no state graph: tlag_build_graph first"; return TLAG_ESTATE; }
  CK(cudaStreamSynchronize(e->stream));
  out->n_states = e->g_states; out->n_edges = e->g_edges; out->n_init = e->init_states;
  out->off = (uint64_t)(uintptr_t)e->d_goff; out->dst = (uint64_t)(uintptr_t)e->d_gdst;
  out->state_label = (uint64_t)(uintptr_t)e->d_slab; out->edge_label = (uint64_t)(uintptr_t)e->d_elab;
  out->device = e->m.device;
  return TLAG_OK;
}

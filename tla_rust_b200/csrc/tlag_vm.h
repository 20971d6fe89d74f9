// tlag_vm.h -- bytecode VM core, state pack/unpack and the 64-bit fingerprint.
//
// One definition of the ISA semantics, compiled by nvcc into the CUDA engine
// (tlag_engine.cu) and by gcc into the CPU bytecode oracle (oracle/tlag_cpu.c, test
// infrastructure).  The opcode order MUST match tla_rust_b200/compile/bytecode.py:OPS.
//
// Replaces (SURVEY.md §2b, all [ext] TLC components, none present under /root/reference):
//   next-state action evaluator  -> tlag_vm_run over the Next program
//   invariant checker            -> tlag_vm_run over the invariant program
//   64-bit state fingerprint     -> tlag_fingerprint (own hash; TLC's FP64 polynomial is
//                                   not observable through any reference artefact)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define TLAG_HD __host__ __device__ __forceinline__
#define TLAG_NOUNROLL   /* (tried _Pragma("unroll 1") to shrink the kernel: 34 KB instead of 58 KB of SASS but 5% slower) */
#else
#define TLAG_HD static inline
#define TLAG_NOUNROLL
#endif

enum {
  OP_HALT = 0, OP_ADD, OP_SUB, OP_MUL, OP_LT, OP_LE, OP_EQ, OP_NE,
  OP_AND, OP_OR, OP_ADDI, OP_MULI, OP_EQI, OP_NEI, OP_LTI, OP_LEI,
  OP_GTI, OP_GEI, OP_SHRI, OP_ANDI, OP_JEQ, OP_JNE, OP_JLT, OP_JGE,
  OP_JEQI, OP_JNEI, OP_JLTI, OP_JGEI, OP_JZ, OP_JNZ, OP_JNEG, OP_JGEZ,
  OP_JBT, OP_JBF, OP_JBTI, OP_JBFI, OP_JMP, OP_LI, OP_LIW, OP_MOV,
  OP_MOVN, OP_ZERO, OP_LDC, OP_DIV, OP_MOD, OP_NEG, OP_EQN, OP_NOT,
  OP_LDX, OP_STX, OP_TBL, OP_TBLT, OP_BSET, OP_BCLR, OP_BTEST, OP_BOR,
  OP_BAND, OP_BANDN, OP_BISZ, OP_BSUB, OP_BCNT, OP_BNEXT, OP_BFILL, OP_BSETI,
  OP_BTESTI, OP_UCLAMP, OP_TRAP, OP_EMIT, OP_GEN, OP_ASSERTF, OP_INVF,
  OP_MADI, OP_BANDC, OP_LEXLT, OP_SFIND, OP_SINS, OP_EMITD, OP_CALL, OP_RET,
  OP__COUNT
};

// events returned by tlag_vm_run
#define TLAG_EV_HALT 0
#define TLAG_EV_EMIT 1
#define TLAG_EV_GEN 2
#define TLAG_EV_TRAP 3
#define TLAG_EV_ASSERT 4
#define TLAG_EV_INVF 5
#define TLAG_EV_STEPS 6   /* instruction budget exhausted (runaway program) */

typedef struct { int32_t off, width, bias; } tlag_slot;

TLAG_HD int32_t tlag_imm28(uint32_t v) { return (int32_t)(v << 4) >> 4; }

TLAG_HD int32_t tlag_cp(const int32_t* cpool, int32_t i) {
#if defined(__CUDA_ARCH__)
  return __ldg(cpool + i);
#else
  return cpool[i];
#endif
}

TLAG_HD int tlag_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}

TLAG_HD int tlag_ffs(uint32_t x) {  /* 1-based index of lowest set bit, 0 if none */
#if defined(__CUDA_ARCH__)
  return __ffs((int)x);
#else
  return __builtin_ffs((int)x);
#endif
}

// Executes ONE instruction word `w` (fetched from code[*pc_io]) for the calling thread: updates the
// frame and *pc_io; returns -1 to continue or a TLAG_EV_* event.  info receives the event payload
// (action id / trap code / assert id / invariant index), info2 the secondary payload (source line).
// The scalar interpreter (tlag_vm_run) and the warp-scheduled interpreter of the CUDA engine both
// call this, so the ISA semantics have a single definition.
#define TLAG_VM_EXEC_FN tlag_vm_exec
#define TLAG_VM_EXT 1
#include "tlag_vm_exec.inc"
#undef TLAG_VM_EXEC_FN
#undef TLAG_VM_EXT

// Runs from *pc until the next event.  `code` may live in shared memory on the device.
TLAG_HD int tlag_vm_run(const uint64_t* code, const int32_t* cpool, int32_t* f, uint32_t* pc_io,
                        int32_t* info, int32_t* info2, uint64_t max_steps) {
  TLAG_NOUNROLL for (uint64_t steps = 0; steps < max_steps; ++steps) {
    const int ev = tlag_vm_exec(code[*pc_io], cpool, f, pc_io, info, info2);
    if (ev >= 0) return ev;
  }
  return TLAG_EV_STEPS;
}

// ---- packed state <-> frame ----------------------------------------------------
// Slots are laid out LSB-first in a little-endian bit stream of W 32-bit words.
// Returns 0, or 1+slot index when a value does not fit its slot (overflow trap).
TLAG_HD int tlag_pack(const tlag_slot* lay, int nslots, const int32_t* st, uint32_t* out, int W) {
  TLAG_NOUNROLL for (int i = 0; i < W; ++i) out[i] = 0;
  uint32_t bitpos = 0;
  TLAG_NOUNROLL for (int s = 0; s < nslots; ++s) {
    const int32_t width = lay[s].width;
    uint32_t v = (uint32_t)(st[lay[s].off] - lay[s].bias);
    if (width < 32 && (v >> width) != 0) return 1 + s;
    const uint32_t wi = bitpos >> 5, sh = bitpos & 31;
    out[wi] |= v << sh;
    if (sh + (uint32_t)width > 32) out[wi + 1] |= v >> (32 - sh);
    bitpos += (uint32_t)width;
  }
  return 0;
}

// Re-pack the slot ranges listed at cpool[tbl]: [n, (first_slot, n_slots, bit position of first_slot) x n] into `out`,
// which holds the packed words of the state being expanded.  Same overflow convention as tlag_pack.
TLAG_HD int tlag_pack_ranges(const tlag_slot* lay, const int32_t* cpool, int32_t tbl, const int32_t* st, uint32_t* out) {
  const int32_t n = tlag_cp(cpool, tbl);
  for (int32_t r = 0; r < n; ++r) {
    const int32_t first = tlag_cp(cpool, tbl + 1 + 3 * r), cnt = tlag_cp(cpool, tbl + 2 + 3 * r);
    uint32_t bitpos = (uint32_t)tlag_cp(cpool, tbl + 3 + 3 * r);
    for (int32_t s = first; s < first + cnt; ++s) {
      const int32_t width = lay[s].width;
      const uint32_t v = (uint32_t)(st[lay[s].off] - lay[s].bias);
      if (width < 32 && (v >> width) != 0) return 1 + s;
      const uint32_t mask = width < 32 ? ((1u << width) - 1u) : 0xFFFFFFFFu;
      const uint32_t wi = bitpos >> 5, sh = bitpos & 31;
      out[wi] = (out[wi] & ~(mask << sh)) | (v << sh);
      if (sh + (uint32_t)width > 32) out[wi + 1] = (out[wi + 1] & ~(mask >> (32 - sh))) | (v >> (32 - sh));
      bitpos += (uint32_t)width;
    }
  }
  return 0;
}

TLAG_HD void tlag_unpack(const tlag_slot* lay, int nslots, const uint32_t* in, int32_t* st) {
  uint32_t bitpos = 0;
  TLAG_NOUNROLL for (int s = 0; s < nslots; ++s) {
    const int32_t width = lay[s].width;
    const uint32_t wi = bitpos >> 5, sh = bitpos & 31;
    uint32_t v = in[wi] >> sh;
    if (sh + (uint32_t)width > 32) v |= in[wi + 1] << (32 - sh);
    if (width < 32) v &= (1u << width) - 1u;
    st[lay[s].off] = (int32_t)v + lay[s].bias;
    bitpos += (uint32_t)width;
  }
}

// ---- 64-bit fingerprint of a packed state --------------------------------------
TLAG_HD uint64_t tlag_rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

TLAG_HD uint64_t tlag_fmix64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdULL; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ULL; k ^= k >> 33;
  return k;
}

// incremental form (lets the probe kernel hash straight out of its vector loads)
TLAG_HD uint64_t tlag_fp_init(int W) { return 0x9E3779B97F4A7C15ULL ^ ((uint64_t)W * 0xD6E8FEB86659FD93ULL); }

TLAG_HD uint64_t tlag_fp_pair(uint64_t h, uint32_t lo, uint32_t hi) {
  uint64_t k = (uint64_t)lo | ((uint64_t)hi << 32);
  k *= 0x87c37b91114253d5ULL; k = tlag_rotl64(k, 31); k *= 0x4cf5ad432745937fULL;
  h ^= k;
  return tlag_rotl64(h, 27) * 5 + 0x52dce729ULL;
}

TLAG_HD uint64_t tlag_fp_tail(uint64_t h, uint32_t w) {
  uint64_t k = (uint64_t)w;
  k *= 0x87c37b91114253d5ULL; k = tlag_rotl64(k, 31); k *= 0x4cf5ad432745937fULL;
  return h ^ k;
}

TLAG_HD uint64_t tlag_fp_final(uint64_t h, int W) {
  h = tlag_fmix64(h ^ (uint64_t)W);
  return h ? h : 1ULL;   // 0 is the empty-slot marker of the seen-set
}

TLAG_HD uint64_t tlag_fingerprint(const uint32_t* w, int W) {
  uint64_t h = tlag_fp_init(W);
  int i = 0;
  TLAG_NOUNROLL for (; i + 1 < W; i += 2) h = tlag_fp_pair(h, w[i], w[i + 1]);
  if (i < W) h = tlag_fp_tail(h, w[i]);
  return tlag_fp_final(h, W);
}

// ---- random simulation ---------------------------------------------------------------
// The draw of walk w (global id) of a run with seed S at step t for candidate j (j = 0xFFFFFFFF: the initial state).
// A walk is a pure function of (S, w): the device engines and the CPU walker of the tests make the same choices.
TLAG_HD uint64_t tlag_mix64(uint64_t z) {   // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ULL; z = (z ^ (z >> 27)) * 0x94d049bb133111ebULL; return z ^ (z >> 31);
}

TLAG_HD uint64_t tlag_sim_draw(uint64_t seed, uint64_t w, uint32_t t, uint32_t j) {
  return tlag_mix64(tlag_mix64(tlag_mix64(seed + 0x9E3779B97F4A7C15ULL) ^ w) ^ (((uint64_t)t << 32) | (uint64_t)j));
}

// Reservoir sampling over a step's candidates: candidate j (0-based, in emission order) replaces the pick iff this holds,
// so that each of k candidates is picked with probability 1/k.
TLAG_HD int tlag_sim_take(uint64_t seed, uint64_t w, uint32_t t, uint32_t j) {
  return tlag_sim_draw(seed, w, t, j) % ((uint64_t)j + 1ULL) == 0ULL;
}

// One state of a behaviour in the history digest (tlag_sim_digest): its fingerprint, walk, step and action id
TLAG_HD uint64_t tlag_sim_term(uint64_t fp, uint64_t w, uint32_t t, int32_t act) {
  return tlag_mix64(fp ^ tlag_mix64(w * 0x9E3779B97F4A7C15ULL + ((uint64_t)t << 16) + (uint64_t)(uint16_t)act));
}

// ---- state graph ---------------------------------------------------------------------
// One edge s -> t with action id a in the graph digest (tlag_graph_digest), from the fingerprints of its two states: the
// XOR and the SUM of it over all edges do not depend on the order of the store.
TLAG_HD uint64_t tlag_edge_term(uint64_t fp_s, uint64_t fp_t, int32_t a) {
  return tlag_mix64(tlag_mix64(fp_s ^ 0x9E3779B97F4A7C15ULL) ^ tlag_mix64(fp_t + (uint64_t)(uint32_t)a));
}

// Walks of one batch: min(num, 2^20, what a 4 GiB history holds at depth D), rounded down to a multiple of 32 (at least
// 32).  It depends on W, D and num only, so a run's batches, and with them its first error, are the same on any GPU.
#define TLAG_SIM_BUDGET (4ULL << 30)
TLAG_HD uint64_t tlag_sim_batch(uint32_t W, uint32_t D, uint64_t num) {
  uint64_t b = TLAG_SIM_BUDGET / ((uint64_t)D * (4ULL * W + 2ULL));
  if (b > (1ULL << 20)) b = 1ULL << 20;
  if (b > num) b = num;
  b &= ~31ULL;
  return b < 32 ? 32 : b;
}

// ---- multi-GPU ownership ---------------------------------------------------------
// Owner rank of a state = hash of its LAST TWO packed words (the clustering key of the frontier sort)
// scaled to n_ranks.  All states of one cluster therefore live on, and are expanded by, the same rank, so a
// rank's level slices are as dense in like states as on a single GPU (hashing the whole state spread every
// cluster over all ranks and cost ~25 % of the per-rank interpreter efficiency at N = 2).
// k = number of trailing packed words the hash covers: 2 = the clustering key (default); up to W = the whole state, for
// models whose last two words carry too little entropy to balance the ranks (SSI: the zero tail of a half-empty
// history sequence -- 278 distinct keys in 2.4 M states, one of 8 ranks would own 70 % of them).
TLAG_HD uint32_t tlag_owner_k(const uint32_t* w, int W, uint32_t n_ranks, int k) {
  const uint64_t key = ((uint64_t)w[W - 1] << 32) | (uint64_t)(W >= 2 ? w[W - 2] : 0u);
  uint64_t h = tlag_fmix64(key * 0x9E3779B97F4A7C15ULL + 0x7F4A7C15ULL);
  for (int i = W - 3, n = 2; i >= 0 && n < k; --i, ++n)
    h = tlag_fmix64(h ^ ((uint64_t)w[i] * 0x9E3779B97F4A7C15ULL + (uint64_t)n));
  return (uint32_t)(((h >> 32) * (uint64_t)n_ranks) >> 32);
}

TLAG_HD uint32_t tlag_owner(const uint32_t* w, int W, uint32_t n_ranks) { return tlag_owner_k(w, W, n_ranks, 2); }


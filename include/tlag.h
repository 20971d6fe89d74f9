/* tlag.h -- C ABI of the H100 explicit-state BFS engine (boundary B1 of SURVEY.md §8b).
 *
 * The reference (spacejam/tla-rust) contains no FFI, plugin or operator API at all: its
 * only integration point is the process boundary `tlc FILE.tla...` (Makefile:6-7,
 * README.md:260-263), behind which the external TLC does parse -> BFS -> report.  This
 * header is the thin C-ABI the north star asks for between a host front end (which
 * parses .tla/.cfg and lowers Next / invariants to fixed-width bytecode) and the
 * sm_90a kernels that replace TLC's Worker BFS loop + StateQueue, next-state
 * evaluator, FPSet and invariant checker (SURVEY.md §2b).  A Rust host binds it with a
 * plain `extern "C"` block (see INTEGRATION.md); nothing here mentions torch or C++.
 *
 * Ownership: the caller owns every buffer it passes in or receives results in; the
 * engine copies inputs during the call.  The engine owns all device memory.  No
 * pointer returned by the engine outlives tlag_destroy (tlag_last_error is valid until
 * the next call on that engine).  Calls on one engine are not re-entrant.
 * Errors: negative return codes + tlag_last_error.  A model-checking verdict
 * (invariant violated, Assert failed, deadlock, evaluation trap) is NOT an error: it is
 * reported in tlag_result.verdict with return code 0.
 */
#ifndef TLAG_H
#define TLAG_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct tlag_engine tlag_engine;

enum { TLAG_OK = 0, TLAG_EINVAL = -1, TLAG_ENOMEM = -2, TLAG_ECUDA = -3, TLAG_ENCCL = -4,
       TLAG_EOVERFLOW = -5, TLAG_EEVAL = -6, TLAG_ESTATE = -7 };

/* verdicts (what `tlc` prints: README.md:267-321) */
enum { TLAG_V_OK = 0, TLAG_V_INVARIANT = 1, TLAG_V_ASSERT = 2, TLAG_V_DEADLOCK = 3,
       TLAG_V_EVAL_ERROR = 4, TLAG_V_RUNNING = 5 };

enum { TLAG_F_DEADLOCK_CHECK = 1u,   /* report states without successors            */
       TLAG_F_KEEP_GOING     = 2u,   /* do not stop a run at the first violation    */
       TLAG_F_EXACT          = 4u }; /* TLC-exact replay: the search runs as ONE sequential worker on the device (states
                                      * dequeued in FIFO order, successors in program order) and stops AT the first
                                      * Assert failure / deadlock, so the counts at that moment, the state reported and
                                      * its parent chain are the ones TLC's single worker prints (README.md:267-321).
                                      * Interpreter kernel only; meant for re-running a small model after an error. */

typedef struct {
  uint32_t words_per_state;      /* W: packed state vector width in u32 words (1..128)        */
  const uint64_t *code;          /* bytecode image (compile/bytecode.py), host-owned, copied   */
  uint32_t code_len;             /* in 64-bit instructions                                     */
  uint32_t entry_inv;            /* pc of the invariant program (runs on each expanded state)  */
  uint32_t entry_next;           /* pc of the next-state program (EMITs successors)            */
  const int32_t *cpool;          /* constant pool (tables), copied                             */
  uint32_t cpool_len;
  const int32_t *layout;         /* n_slots x {frame_off, width_bits, bias}: packed layout     */
  uint32_t n_slots;
  uint32_t frame_words;          /* per-thread VM frame size in words (<= 8192)                */
  uint32_t unpacked_words;       /* words of one unpacked state (primed copy follows it)       */
  uint32_t n_invariants;
  uint32_t n_actions;
  uint32_t table_slots_log2;     /* seen-set capacity (8-byte slots); grows by rehash if 0<load*/
  uint64_t max_states;           /* capacity of the state store (0 = size from free memory)    */
  uint32_t flags;                /* TLAG_F_*                                                   */
  int32_t  device;               /* CUDA device ordinal                                        */
} tlag_model;

typedef struct {
  uint64_t level;                /* BFS level just expanded (initial states are level 1)       */
  uint64_t expanded;             /* states expanded in this wave                               */
  uint64_t generated;            /* successors generated in this wave (incl. duplicates)       */
  uint64_t discovered;           /* new distinct states found in this wave                     */
  uint64_t distinct_total;
  uint64_t generated_total;
  float    kernel_ms;            /* device time of the wave kernel (CUDA events)               */
  int32_t  verdict;              /* TLAG_V_RUNNING while the search continues                  */
  float    cluster_ms;           /* device time of the level's frontier clustering pass (events) */
  uint32_t retries;              /* times the level was rolled back and run again (store or seen-set out of room) */
} tlag_wave_stats;

typedef struct {
  int32_t  verdict;              /* TLAG_V_*                                                   */
  int32_t  detail;               /* invariant index / assert id / trap code                    */
  int32_t  detail2;              /* trap source line                                           */
  int32_t  reserved;
  uint64_t state_idx;            /* index (discovery order) of the offending state             */
  uint64_t generated, distinct, queue_left, depth, init_states;
  double   fp_collision_estimate;/* n*(g-n)/2^64, as TLC's "calculated (optimistic)"           */
  double   device_seconds;       /* sum of wave-kernel times                                   */
} tlag_result;

int  tlag_create(const tlag_model *m, tlag_engine **out);
/* n initial states, W words each (host memory).  Duplicates are dropped; every one counts
 * as "generated" like TLC's "Finished computing initial states" line (testout2:3). */
int  tlag_seed(tlag_engine *e, const uint32_t *states, uint64_t n);
int  tlag_step(tlag_engine *e, tlag_wave_stats *out);          /* one BFS level; blocks       */
int  tlag_run(tlag_engine *e, tlag_result *out);               /* to fixpoint / violation     */
int  tlag_result_now(tlag_engine *e, tlag_result *out);        /* counters so far             */
/* Counterexample reconstruction: walks parent links from state_idx back to an initial
 * state.  states_out receives len*W words (initial state first), actions_out len action
 * ids (entry 0 is -1).  *len_inout: capacity in, length out. */
int  tlag_trace(tlag_engine *e, uint64_t state_idx, uint32_t *states_out, int32_t *actions_out,
                uint32_t *len_inout);
int  tlag_read_states(tlag_engine *e, uint64_t first, uint64_t n, uint32_t *states_out);
/* One hop of a parent chain: state idx (W words), its parent's index and the meta word = action id << 8 | rank whose
 * store holds the parent (multi-GPU: the host follows the chain from rank to rank).  parent 0xFFFFFFFF = initial state. */
int  tlag_read_link(tlag_engine *e, uint64_t idx, uint32_t *state_out, uint32_t *parent_out, uint32_t *meta_out);
/* Checksum of checksums over every stored state: XOR and SUM (mod 2^64) of the 64-bit fingerprints
 * (size-independent parity property for state spaces too large to read back). */
int  tlag_digest(tlag_engine *e, uint64_t *xor_out, uint64_t *sum_out);
/* K1 alone (fingerprint + seen-set probe/insert) on caller-provided HOST states: unit tests
 * and the e2e leg of the roofline bench.  is_new[i] = 1 iff state i was not in the set. */
int  tlag_probe_batch(tlag_engine *e, const uint32_t *states, uint64_t n, uint8_t *is_new);
/* Same on DEVICE-resident buffers (d_states: n*W u32, d_is_new: n bytes); returns the kernel
 * time measured with CUDA events on the engine's stream. */
int  tlag_probe_batch_device(tlag_engine *e, uint64_t d_states, uint64_t n, uint64_t d_is_new,
                             float *kernel_ms);
int  tlag_reset_table(tlag_engine *e);                         /* empty the seen-set           */
int  tlag_restart(tlag_engine *e);     /* forget all discovered states; re-seed the retained initial states */
uint64_t tlag_kernel_launches(const tlag_engine *e);           /* kernels launched so far      */
void tlag_destroy(tlag_engine *e);
const char *tlag_last_error(const tlag_engine *e);
const char *tlag_version(void);

/* ---- random simulation (tlc -simulate) ------------------------------------------------------------------------------
 * Walk w (a global id) of a run with seed S starts at the distinct initial state R(S, w, 0, 0xFFFFFFFF) mod n_init
 * (distinct seeded states, first occurrence order).  At step t it checks every invariant on its state s_t, enumerates
 * the successors of s_t in program order, and picks one of the candidates (the successors the search would store) by
 * reservoir sampling: candidate j replaces the pick iff R(S, w, t, j) mod (j + 1) == 0.  R is tlag_sim_draw
 * (csrc/tlag_vm.h).  A behaviour has at most `depth` states; its last state's invariants are checked, its successors
 * are not enumerated.  A walk ends at an error, at a state without successors (a deadlock when flags has
 * TLAG_F_DEADLOCK_CHECK), at a state whose successors are none of them candidates, or at its last state.
 * Walks run in batches of batch_walks ids, a function of W, depth and num_walks only (tlag_sim_batch in
 * csrc/tlag_vm.h); the run stops after the first batch
 * that holds an error, and the error reported is the one at the smallest step, then the smallest walk id, so the
 * result depends on (seed, first_walk, num_walks, depth) only.  The interpreter library and a model's simulation
 * library (sliced build with simulation kernels) run it; any other library returns TLAG_EINVAL. */
typedef struct {
  uint64_t seed;
  uint64_t first_walk;           /* global id of the first walk                                 */
  uint64_t num_walks;
  uint32_t depth;                /* states per behaviour at most (1..10^6)                      */
  uint32_t flags;                /* TLAG_F_DEADLOCK_CHECK                                       */
} tlag_sim_params;

typedef struct {
  int32_t  verdict;              /* TLAG_V_OK or the first error's TLAG_V_*                     */
  int32_t  detail, detail2;      /* as in tlag_result                                           */
  int32_t  reserved;
  uint64_t walk, step;           /* the first error: walk id and step (0 = the initial state)   */
  uint64_t checked;              /* states whose invariants were evaluated                      */
  uint64_t generated;            /* successors enumerated, duplicates and non-candidates included */
  uint64_t behaviours;           /* walks run (all of the batch that held the error)            */
  uint64_t batch_walks;          /* walks per batch                                             */
  double   device_ms;            /* device time of the batches (CUDA events)                    */
} tlag_sim_result;

int  tlag_simulate(tlag_engine *e, const tlag_sim_params *params, tlag_sim_result *out);
/* The behaviour of `walk` (in the last batch run): len states (W words each, initial state first) and the action id
 * of each (entry 0 is -1).  *len_inout: capacity in, length out (the states whose invariants were checked). */
int  tlag_sim_trace(tlag_engine *e, uint64_t walk, uint32_t *states_out, int32_t *actions_out, uint32_t *len_inout);
/* The history of walks [walk, walk + n) of the last batch: states_out depth x n x W words (row t = step t), actions_out
 * depth x n ids, len_out n lengths.  Rows at or past a walk's length hold no state of its behaviour.  Any output may be
 * NULL. */
int  tlag_sim_read(tlag_engine *e, uint64_t walk, uint64_t n, uint32_t *states_out, int16_t *actions_out,
                   uint32_t *len_out);
/* XOR and SUM over the last batch of one term per state checked, from its fingerprint, walk, step and action
 * (tlag_sim_term in csrc/tlag_vm.h). */
int  tlag_sim_digest(tlag_engine *e, uint64_t *xor_out, uint64_t *sum_out);

/* ---- state graph (tlc -dump dot; the input of the liveness checks) ---------------------------------------------------
 * After a search call, the state graph covers every state of the store.  Rows [0, n_expanded) are the states the search
 * expanded; the store is level-contiguous, so n_expanded is the first row of the current frontier: n_states at the
 * fixpoint, the first row of the first unexpanded level after a violation (the level that found it is finished), the
 * first row of level L after a depth-bounded stop.  There is one edge (s, t, a) per distinct triple where s is an
 * expanded row, Next enumerated from s reaches an EMIT (a successor the search would store, not a GEN) with action id a
 * (as tlag_trace reports it), the packed successor (under SYMMETRY the representative EMIT produces) is stored row t, and
 * t != s: self-loops are not edges (as for tlag_scc).  The same t reached by two actions makes two edges.  Edges are CSR
 * by source row, and within a row ordered by (t, a).  The set of (fingerprint(s), fingerprint(t), a) does not depend on
 * the store's order: both device engines and any run give the same set.
 * tlag_build_graph builds it in device memory: an index pass maps every seen-set slot to its row (4 bytes per slot), then
 * Next runs over chunks of expanded rows on the interpreter (the sliced libraries included) and each chunk's edges are
 * sorted, made distinct and appended.  The clustering and discovery buffers and the routed-fingerprint cache are freed
 * first; a graph that does not fit is TLAG_ENOMEM.  Refused: a simulation library and a TLAG_F_EXACT engine
 * (TLAG_EINVAL), an engine that holds one shard of a multi-GPU search (tlag_set_rank with n > 1, tlag_p2p_init;
 * TLAG_EINVAL), an engine not seeded (TLAG_ESTATE) and a search that stopped at an evaluation trap, whose successor sets
 * are incomplete (TLAG_ESTATE).  tlag_seed, tlag_step, tlag_run, tlag_restart and tlag_destroy release the graph; reading
 * a released graph is TLAG_ESTATE.  device_ms: from the index pass to the last append (CUDA events). */
typedef struct {
  uint64_t n_states, n_expanded, n_edges;
  float    device_ms;
} tlag_graph_info;

int  tlag_build_graph(tlag_engine *e, tlag_graph_info *out);
/* The edges of rows [first, first + n): off_out n + 1 offsets relative to row `first` (off_out[0] = 0), dst_out and
 * act_out off_out[n] destination rows and action ids.  dst_out / act_out may be NULL (sizing). */
int  tlag_read_graph(tlag_engine *e, uint64_t first, uint64_t n, uint64_t *off_out, uint32_t *dst_out, int32_t *act_out);
/* XOR and SUM (mod 2^64) over all edges (s, t, a) of the edge term of csrc/tlag_vm.h (tlag_edge_term) on the
 * fingerprints of s and t and on a: does not depend on the store's order. */
int  tlag_graph_digest(tlag_engine *e, uint64_t *xor_out, uint64_t *sum_out);

/* ---- liveness labels of the state graph (DESIGN.md §7h) ---------------------------------------------------------------
 * tlag_label_graph runs a label image (compile/lower.py compile_labels: its own bytecode and constant pool over the model's
 * layout and frame) on the graph tlag_build_graph left: the state program on every stored row (state word bit j = state
 * predicate j holds), the edge program on every edge (s, t) with s in the current frame and t in the primed one (edge word
 * bit j = <<A_j>>_v holds), each predicate that is false raising INVF j.  Then, for every edge bit b, en_bit[b] (< 32) is
 * set in the state word of each row with an out-edge that has bit b (ENABLED <<A_b>>_v over the stored successors: see
 * DESIGN.md §7h), nen_bit[b] (< 32) in the state word of each row without one; 0xFF = not derived.  A program that traps
 * on a row or an edge is TLAG_EEVAL.  The labels belong to the graph and are released with it; labelling again replaces
 * them.  device_ms: the two label passes and the ENABLED pass (CUDA events). */
typedef struct {
  const uint64_t *code;          /* the label image, copied                                     */
  uint32_t code_len;
  uint32_t entry_states;         /* pc of the state program                                     */
  uint32_t entry_edges;          /* pc of the edge program                                      */
  uint32_t n_state_preds;        /* state bits [0, n) the state program writes (<= 32)           */
  uint32_t n_edge_preds;         /* edge bits [0, n) the edge program writes (<= 32)             */
  const int32_t *cpool;          /* the image's constant pool, copied                           */
  uint32_t cpool_len;
  uint8_t  en_bit[32], nen_bit[32];
} tlag_label_program;

int  tlag_label_graph(tlag_engine *e, const tlag_label_program *prog, float *device_ms);

/* The engine's graph as device pointers (as tlag_expand_route takes them), valid until the graph is released: the CSR
 * (off: n_states + 1 uint64, dst: n_edges uint32), the labels (state_label: n_states uint32, edge_label: n_edges uint32,
 * 0 when not labelled), the device, and n_init: rows [0, n_init) are the initial states. */
typedef struct {
  uint64_t n_states, n_edges;
  uint64_t off, dst, state_label, edge_label;
  uint64_t n_init;
  int32_t  device;
} tlag_graph_dev;

int  tlag_graph_view(tlag_engine *e, tlag_graph_dev *out);

/* ---- multi-GPU building blocks (one engine per rank; the host exchanges the buffers,
 *      e.g. torch.distributed all_to_all_single over NCCL/NVLink; SURVEY.md §8e) ---------- */
/* Expand the current frontier WITHOUT inserting: successor records (W state words + parent
 * index + action id, record = W+2 u32) are bucketed by owner rank = fingerprint >> (64-log2 R)
 * ... into d_send (device, capacity cap_records), counts[r] records per rank (host out). */
int  tlag_frontier(tlag_engine *e, uint64_t *first_idx, uint64_t *count);   /* current frontier slice */
/* Which shard this engine holds (before the first tlag_expand_route of a multi-rank run): successors the rank owns
 * itself are inserted in place, and the rank is recorded in the meta word of the states whose parent it expands. */
int  tlag_set_rank(tlag_engine *e, uint32_t n_ranks, uint32_t rank);
/* Trailing packed words the ownership hash covers (same on every rank, before anything is routed): 2 (default) keeps
 * clusters of like states on one rank, words_per_state spreads models whose tail words carry little entropy. */
int  tlag_set_owner_words(tlag_engine *e, uint32_t k);
/* `first`/`count` select a sub-range of the frontier (chunked exchange with bounded buffers). */
int  tlag_expand_route(tlag_engine *e, uint32_t n_ranks, uint64_t first, uint64_t count, uint64_t d_send,
                       uint64_t cap_records, uint64_t *counts, tlag_wave_stats *out);
/* Insert received records (device buffer) into this rank's seen-set shard / state store. */
int  tlag_insert_records(tlag_engine *e, uint64_t d_recv, uint64_t n_records, uint32_t src_rank_unused,
                         uint64_t *n_new);
int  tlag_advance_level(tlag_engine *e, tlag_wave_stats *out);  /* frontier <- newly inserted  */

/* ---- peer-memory exchange (NVLink / NVSwitch; no NCCL on the data path) ---------------------------------------
 * tlag_p2p_init allocates this rank's inbox (2 buffers x n_ranks regions of cap_records records) and send regions
 * and returns a 64-byte CUDA IPC handle of the inbox; the host all-gathers the handles (any transport) and calls
 * tlag_p2p_attach for every peer.  tlag_p2p_level then runs one whole BFS level on this rank: per chunk of
 * chunk_states frontier states the expand kernels bucket successors by owner, k_push stores the buckets into the
 * owners' inboxes and publishes {count, chunk number} with a system-scope release, k_insert_inbox waits for every
 * source's chunk, inserts the records (this rank's share of the next frontier) and acknowledges.  All ranks must
 * pass the same n_chunks.  expect_inbound: upper estimate of the records this rank may receive (store head-room).
 * Follow with tlag_advance_level; termination is the host's all-reduce of `discovered`. */
int  tlag_p2p_init(tlag_engine *e, uint32_t n_ranks, uint32_t rank, uint64_t cap_records, uint8_t *handle_out64);
int  tlag_p2p_attach(tlag_engine *e, uint32_t peer, const uint8_t *handle64);
int  tlag_p2p_level(tlag_engine *e, uint64_t n_chunks, uint64_t chunk_states, uint64_t expect_inbound,
                    tlag_wave_stats *out);
/* TLAG_EOVERFLOW from tlag_p2p_level on ANY rank (a send region was too small for a chunk): every rank calls
 * tlag_p2p_rollback -- the level's appended states are dropped, the seen-set rebuilt -- and the level is run again
 * with smaller chunks. */
int  tlag_p2p_rollback(tlag_engine *e);

/* ---- liveness building blocks: strongly connected components and fair cycles of a state graph ---------------------
 * Standalone calls (no engine): the caller passes the graph as a host edge list over states 0..n_states-1; each call
 * copies it to the device, works there and returns.  Self-loops are ignored (a self-loop cannot satisfy <<A>>_v; the
 * implicit stuttering step of every state stands for it), so every SCC, a single state included, carries a cycle.
 * An edge endpoint >= n_states is TLAG_EINVAL.  The calling thread's current CUDA device is the same on return.
 * Errors: negative return codes + tlag_graph_last_error (per host thread). */
typedef struct {
  uint64_t n_states;             /* < 2^32 - 1                                                  */
  uint64_t n_edges;              /* < 2^32                                                      */
  const uint32_t *src, *dst;     /* n_edges state indices each                                  */
  const uint32_t *edge_label;    /* n_edges words: bit b = the edge satisfies <<A_b>>_v (NULL = all 0) */
  const uint32_t *state_label;   /* n_states words: state predicates, ENABLED bits (NULL = all 0) */
  const uint8_t  *state_mask;    /* nonzero = the state is in the restricted graph (NULL = all) */
  const uint8_t  *edge_mask;     /* nonzero = the edge is in the restricted graph (NULL = all)  */
  int32_t device;                /* CUDA device ordinal                                         */
} tlag_graph;

/* SCC decomposition of the restricted graph: scc_out[v] = id of v's component (the index of one of its states), or
 * 0xFFFFFFFF for a state outside the mask.  Trim, then forward-backward from the state of largest degree product,
 * then colour propagation for the rest.  device_ms: device time of the edge compaction, the CSR build and the
 * decomposition (CUDA events; the host<->device copies are not counted). */
int  tlag_scc(const tlag_graph *g, uint32_t *scc_out, uint64_t *n_scc_out, float *device_ms);

enum { TLAG_FAIR_WF = 0, TLAG_FAIR_SF = 1 };
typedef struct {
  uint32_t kind;                 /* TLAG_FAIR_WF / TLAG_FAIR_SF                                 */
  uint32_t enabled_bit;          /* state-label bit of ENABLED <<A>>_v                          */
  uint32_t action_bit;           /* edge-label bit of <<A>>_v                                   */
  uint32_t reserved;
} tlag_fairness;

typedef struct {
  const tlag_fairness *fair;     /* fairness conditions every accepted cycle must satisfy       */
  uint32_t n_fair;
  uint32_t need_clear;           /* state-label bits: an accepted SCC holds, for each bit, a state where it is clear
                                  * (the ~Y state of every <>[]Y disjunct of the obligation)    */
  const uint8_t *seeds;          /* NULL: every accepted SCC counts; else only those reachable in the restricted
                                  * graph from a state with seeds[v] != 0 (P ~> Q: P /\ ~Q states; <>P: initial ~P) */
} tlag_fair_query;

typedef struct {
  int32_t  violated;             /* 1 = a (reachable) accepted SCC exists: the obligation fails */
  uint32_t witness;              /* smallest state of such an SCC (0xFFFFFFFF if none)          */
  uint64_t fair_sccs;            /* accepted SCCs, reachable or not                             */
  uint32_t rounds;               /* SCC decompositions run (Emerson-Lei refinements + 1)        */
  float    device_ms;            /* device time from the edge compaction on (CUDA events, copies excluded) */
} tlag_fair_result;

/* Fair-cycle search (Emerson-Lei) on the restricted graph.  An SCC C is accepted when, for every condition,
 *   WF: some state of C has ~EN, or some edge inside C has the action bit;
 *   SF: no state of C has EN, or some edge inside C has the action bit;
 * and C holds a state with each need_clear bit clear.  C failing a WF or need_clear test is dropped; C failing only
 * SF tests loses its EN states and the rest is decomposed again, to a fixpoint.  scc_out[v] = accepted SCC id of v,
 * else 0xFFFFFFFF (NULL: not returned).  The cycle through every state and edge of an accepted SCC is fair and
 * violates the obligation the masks and need_clear encode.  It uploads the graph and builds both CSRs on every call;
 * tlag_live_check runs the same search on a graph the engine built in device memory. */
int  tlag_fair_cycles(const tlag_graph *g, const tlag_fair_query *q, uint32_t *scc_out, tlag_fair_result *out);

/* Obligation check on an engine's labelled graph (DESIGN.md §7h), with the decomposition and the Emerson-Lei loop of
 * tlag_fair_cycles.  The restricted graph keeps the rows whose state word has every keep_set bit and no keep_clear bit,
 * and the edges between them whose edge word has no edge_drop bit.  Seeds are the rows below seed_rows (0: all rows)
 * whose state word has every seed_set bit and no seed_clear bit.  With TLAG_LIVE_SEEDS only accepted SCCs reachable from a
 * seed in the restricted graph count; with TLAG_LIVE_ANY_SEED no SCC is searched and the obligation fails iff a seed
 * exists ([]P: the rows with ~P), the witness being the smallest.  fair: enabled_bit / action_bit are state / edge bits.
 * A graph of 2^32 edges or more is TLAG_EINVAL.
 * For a violation lasso_out receives prefix_len + cycle_len rows: the prefix, a path of the restricted graph from a seed
 * (without seeds: the witness alone) to the witness, then the cycle, from the witness through an edge with each
 * condition's action bit (or a ~EN state of a WF condition) and a state with each need_clear bit clear, inside the
 * accepted SCC, back to (not including) the witness.  cycle_len 1: the SCC is the witness alone, the behaviour stutters
 * there.  With TLAG_LIVE_ANY_SEED the cycle is empty.  lasso_cap too small: TLAG_EOVERFLOW, lengths set. */
enum { TLAG_LIVE_SEEDS = 1u, TLAG_LIVE_ANY_SEED = 2u };
typedef struct {
  const tlag_fairness *fair;
  uint32_t n_fair;
  uint32_t flags;                /* TLAG_LIVE_*                                                 */
  uint32_t keep_set, keep_clear, edge_drop, need_clear;
  uint32_t seed_set, seed_clear;
  uint64_t seed_rows;
} tlag_live_query;

typedef struct {
  int32_t  violated;
  uint32_t witness;              /* smallest row of a (reachable) accepted SCC, or the smallest seed (0xFFFFFFFF: none) */
  uint64_t fair_sccs;            /* accepted SCCs, reachable or not                             */
  uint32_t rounds;
  uint32_t prefix_len, cycle_len;
  uint32_t reserved;
  float    check_ms, lasso_ms;   /* device time of the check (from the restriction on) and of the lasso (CUDA events) */
} tlag_live_result;

int  tlag_live_check(const tlag_graph_dev *g, const tlag_live_query *q, uint32_t *lasso_out, uint32_t lasso_cap,
                     tlag_live_result *out);
const char *tlag_graph_last_error(void);

#ifdef __cplusplus
}
#endif
#endif

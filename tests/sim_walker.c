/* CPU walker of the random simulation (test infrastructure, tests/test_simulate.py): tlag_simulate's semantics
 * (include/tlag.h) on the host, one walk after another within each step, so that every device result can be checked
 * word for word.  The draws, the batch size and pack / unpack come from tla_rust_b200/csrc/tlag_vm.h, which the
 * engine includes too; the walk itself is written out again here.
 *
 * Two builds: the bytecode interpreter (default), and with -DTLAG_SLICED_INC="<file>" the sliced code of one model
 * (tla_rust_b200/compile/sliced.py), which runs every invariant slice and then every slice of Next in program order, as
 * the simulation kernels of a sliced library do.  The model struct is oracle/cpu_engine.py's CpuModel. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../tla_rust_b200/csrc/tlag_vm.h"

#define MAXW 128
#define MAX_STEPS (1ull << 38)

typedef struct {
  uint32_t W;
  const uint64_t *code; uint32_t code_len;
  uint32_t entry_inv, entry_next;
  const int32_t *cpool; uint32_t cpool_len;
  const tlag_slot *layout; uint32_t n_slots;
  uint32_t frame_words, unpacked_words, n_invariants;
  uint32_t flags;           /* 1 = deadlock check */
  uint32_t table_log2;
  uint64_t max_states;
} cpu_model;

typedef struct {
  int32_t verdict, detail, detail2, pad;
  uint64_t walk, step, checked, generated, behaviours, batch_walks;
} sim_result;

enum { RUN = 0, ENDED = 1, FAILED = 2, FAILED_NEXT = 3 };

/* one batch in progress */
typedef struct {
  const cpu_model *m;
  uint64_t seed, first, B;
  uint32_t t, depth;
  uint32_t *hist; int16_t *act;               /* depth rows of B walks */
  uint64_t viol_inv, viol_assert, viol_trap, viol_deadlock;
  uint64_t generated;
} batch;

static void vmin(uint64_t *p, uint64_t v) { if (v < *p) *p = v; }

/* the walk's pick so far: row t + 1 */
static void pick(batch *b, uint64_t i, uint32_t j, int aid, const uint32_t *w) {
  if (!tlag_sim_take(b->seed, b->first + i, b->t, j)) return;
  const int W = (int)b->m->W;
  memcpy(b->hist + ((uint64_t)(b->t + 1) * b->B + i) * W, w, (size_t)W * 4);
  b->act[(uint64_t)(b->t + 1) * b->B + i] = (int16_t)aid;
}

#ifdef TLAG_SLICED_INC
typedef struct {
  batch *b; uint64_t idx; const uint32_t *src;
  uint64_t gen; unsigned nsucc; int phase; unsigned cnt; int stat;
} tlag_sl_cx;

static void sl_emit_words(tlag_sl_cx *cx, int aid, const uint32_t *succ) {
  cx->nsucc++; cx->gen++;
  pick(cx->b, cx->idx, cx->cnt++, aid, succ);
}

static void sl_emit_frame(tlag_sl_cx *cx, const int32_t *f, int aid, int dirty) {
  const cpu_model *m = cx->b->m;
  const int W = (int)m->W;
  uint32_t succ[MAXW];
  int ov;
  if (dirty > 0) {
    memcpy(succ, cx->src, (size_t)W * 4);
    ov = tlag_pack_ranges(m->layout, m->cpool, dirty, f + m->unpacked_words, succ);
  } else ov = tlag_pack(m->layout, (int)m->n_slots, f + m->unpacked_words, succ, W);
  if (ov) {
    cx->nsucc++; cx->gen++;
    vmin(&cx->b->viol_trap, (cx->idx << 20) | (2ULL << 16) | (uint32_t)((ov - 1) & 0xFFFF));
    cx->stat = FAILED;
    return;
  }
  sl_emit_words(cx, aid, succ);
}

#define TLAG_SL_SKIPSELF 0
#define TLAG_SL_EMIT(aid, dirty) sl_emit_frame(cx, f, (aid), (dirty))
#define TLAG_SL_EMITW(aid, o) sl_emit_words(cx, (aid), (o))
#define TLAG_SL_GEN() do { cx->nsucc++; cx->gen++; } while (0)
#define TLAG_SL_ASSERT(id) do { vmin(&cx->b->viol_assert, (cx->idx << 20) | (uint32_t)((id) & 0xFFFFF)); \
    cx->stat = cx->phase == 0 ? FAILED : (cx->stat == RUN ? FAILED_NEXT : cx->stat); } while (0)
#define TLAG_SL_INVF(i) do { if (cx->phase == 0) { vmin(&cx->b->viol_inv, (cx->idx << 20) | (uint32_t)((i) & 0xFFFFF)); cx->stat = FAILED; } } while (0)
#define TLAG_SL_TRAP(code, line) do { vmin(&cx->b->viol_trap, (cx->idx << 20) | ((uint64_t)((code) & 15) << 16) | (uint32_t)((line) & 0xFFFF)); cx->nsucc++; cx->stat = FAILED; } while (0)
#define TLAG_SL_SUBQ static __attribute__((noinline))
#define TLAG_SL_SEGQ static __attribute__((noinline))
#define TLAG_SL_POISON 1
#include TLAG_SLICED_INC
typedef void (*sl_fn)(const int32_t *, const uint32_t *, tlag_sl_cx *);
#define SL_ADDR_INV(j) tlag_sl_inv_##j,
#define SL_ADDR_NEXT(j) tlag_sl_next_##j,
static const sl_fn sl_inv_fns[] = { TLAG_SL_INV_LIST(SL_ADDR_INV) NULL };
static const sl_fn sl_next_fns[] = { TLAG_SL_NEXT_LIST(SL_ADDR_NEXT) NULL };

/* step b->t of walk i: -> its status; *cnt candidates, *nsucc successors */
static int step_walk(batch *b, uint64_t i, int32_t *frame, unsigned *cnt, unsigned *nsucc) {
  (void)frame;
  const cpu_model *m = b->m;
  tlag_sl_cx cx;
  memset(&cx, 0, sizeof(cx));
  cx.b = b; cx.idx = i; cx.src = b->hist + ((uint64_t)b->t * b->B + i) * m->W; cx.stat = RUN;
  if (m->n_invariants) {
    cx.phase = 0;
    for (int j = 0; sl_inv_fns[j]; ++j) sl_inv_fns[j](m->cpool, cx.src, &cx);
  }
  if (b->t + 1 < b->depth && cx.stat != FAILED) {
    cx.phase = 1;
    for (int j = 0; sl_next_fns[j] && cx.stat != FAILED; ++j) sl_next_fns[j](m->cpool, cx.src, &cx);
  }
  b->generated += cx.gen;
  *cnt = cx.cnt; *nsucc = cx.nsucc;
  return cx.stat;
}
#else
static int step_walk(batch *b, uint64_t i, int32_t *frame, unsigned *cnt, unsigned *nsucc) {
  const cpu_model *m = b->m;
  const int W = (int)m->W;
  const uint32_t *src = b->hist + ((uint64_t)b->t * b->B + i) * W;
  uint32_t succ[MAXW];
  int stat = RUN;
  *cnt = 0; *nsucc = 0;
  tlag_unpack(m->layout, (int)m->n_slots, src, frame);
  if (m->n_invariants) {
    uint32_t pc = m->entry_inv;
    for (;;) {
      int32_t info = 0, info2 = 0;
      int ev = tlag_vm_run(m->code, m->cpool, frame, &pc, &info, &info2, MAX_STEPS);
      if (ev == TLAG_EV_HALT) break;
      if (ev == TLAG_EV_INVF) { vmin(&b->viol_inv, (i << 20) | (uint32_t)(info & 0xFFFFF)); stat = FAILED; continue; }
      if (ev == TLAG_EV_ASSERT) { vmin(&b->viol_assert, (i << 20) | (uint32_t)(info & 0xFFFFF)); stat = FAILED; continue; }
      if (ev == TLAG_EV_GEN) { ++*nsucc; ++b->generated; continue; }
      if (ev == TLAG_EV_EMIT) { ++*nsucc; ++b->generated; continue; }
      vmin(&b->viol_trap, (i << 20) | ((uint64_t)(ev == TLAG_EV_STEPS ? 15 : (info & 15)) << 16) | (uint32_t)(info2 & 0xFFFF));
      return FAILED;
    }
  }
  if (b->t + 1 >= b->depth || stat == FAILED) return stat;
  uint32_t pc = m->entry_next;
  for (;;) {
    int32_t info = 0, info2 = 0;
    int ev = tlag_vm_run(m->code, m->cpool, frame, &pc, &info, &info2, MAX_STEPS);
    if (ev == TLAG_EV_HALT) break;
    if (ev == TLAG_EV_GEN) { ++*nsucc; ++b->generated; continue; }
    if (ev == TLAG_EV_INVF) continue;
    if (ev == TLAG_EV_ASSERT) {
      vmin(&b->viol_assert, (i << 20) | (uint32_t)(info & 0xFFFFF));
      if (stat == RUN) stat = FAILED_NEXT;
      continue;
    }
    if (ev == TLAG_EV_EMIT) {
      ++*nsucc; ++b->generated;
      int ov;
      if (info2 > 0) {
        memcpy(succ, src, (size_t)W * 4);
        ov = tlag_pack_ranges(m->layout, m->cpool, info2, frame + m->unpacked_words, succ);
      } else ov = tlag_pack(m->layout, (int)m->n_slots, frame + m->unpacked_words, succ, W);
      if (ov) { vmin(&b->viol_trap, (i << 20) | (2ULL << 16) | (uint32_t)((ov - 1) & 0xFFFF)); stat = FAILED; continue; }
      pick(b, i, (*cnt)++, info, succ);
      continue;
    }
    vmin(&b->viol_trap, (i << 20) | ((uint64_t)(ev == TLAG_EV_STEPS ? 15 : (info & 15)) << 16) | (uint32_t)(info2 & 0xFFFF));
    return FAILED;
  }
  return stat;
}
#endif

/* tlag_simulate on the host.  hist_out (depth x n x W), act_out (depth x n) and len_out (n) receive the last batch's
 * history, n = its walks (at most batch_walks = tlag_sim_batch(W, depth, num)).  Returns 0, or -1 (bad arguments) /
 * -2 (memory). */
int tlagcpu_simulate(const cpu_model *m, const uint32_t *init, uint64_t n_init, uint64_t seed, uint64_t first, uint64_t num,
                     uint32_t depth, sim_result *out, uint32_t *hist_out, int16_t *act_out, uint32_t *len_out) {
  memset(out, 0, sizeof(*out));
  if (depth < 1 || num == 0 || n_init == 0) return -1;
  const int W = (int)m->W;
  /* the distinct initial states, first occurrence first */
  uint32_t *dist = (uint32_t *)malloc(n_init * (size_t)W * 4);
  uint64_t nd = 0;
  for (uint64_t k = 0; k < n_init; ++k) {
    uint64_t o = 0;
    while (o < nd && memcmp(dist + o * W, init + k * W, (size_t)W * 4)) ++o;
    if (o == nd) memcpy(dist + nd++ * W, init + k * W, (size_t)W * 4);
  }
  const uint64_t B = tlag_sim_batch((uint32_t)W, depth, num);
  batch b;
  memset(&b, 0, sizeof(b));
  b.m = m; b.seed = seed; b.B = B; b.depth = depth;
  b.hist = (uint32_t *)calloc(B * depth * (size_t)W, 4);
  b.act = (int16_t *)calloc(B * depth, 2);
  uint8_t *status = (uint8_t *)malloc(B);
  uint32_t *len = (uint32_t *)malloc(B * 4);
  int32_t *frame = (int32_t *)calloc(m->frame_words + 8, 4);
  if (!dist || !b.hist || !b.act || !status || !len || !frame) {
    free(dist); free(b.hist); free(b.act); free(status); free(len); free(frame);
    return -2;
  }
  out->batch_walks = B;
  uint64_t n = 0;
  for (uint64_t done = 0; done < num; done += B) {
    n = num - done < B ? num - done : B;
    b.first = first + done;
    b.viol_inv = b.viol_assert = b.viol_trap = b.viol_deadlock = ~0ULL;
    b.generated = 0;
    for (uint64_t i = 0; i < n; ++i) {
      const uint64_t k = tlag_sim_draw(seed, b.first + i, 0, 0xFFFFFFFFu) % nd;
      memcpy(b.hist + i * W, dist + k * W, (size_t)W * 4);
      b.act[i] = -1; status[i] = RUN; len[i] = 0;
    }
    uint64_t stopped = 0;
    for (uint32_t t = 0; t < depth && !stopped; ++t) {
      b.t = t;
      for (uint64_t i = 0; i < n; ++i) {
        if (status[i] == ENDED) continue;
        unsigned cnt = 0, nsucc = 0;
        const int st = step_walk(&b, i, frame, &cnt, &nsucc);
        out->checked++;
        len[i] = t + 1;
        int err = st != RUN, more = 0;
        if (!err && t + 1 < depth) {
          if (!nsucc) {
            if (m->flags & 1) { vmin(&b.viol_deadlock, i << 20); err = 1; }
          } else more = cnt != 0;
        }
        if (err) stopped = t + 1;
        status[i] = more ? RUN : ENDED;
      }
    }
    out->generated += b.generated;
    out->behaviours += n;
    if (stopped) {
      uint64_t best = ~0ULL; int kind = 0;
      if (b.viol_trap != ~0ULL && (b.viol_trap >> 20) < best) { best = b.viol_trap >> 20; kind = 4; }
      if (b.viol_assert != ~0ULL && (b.viol_assert >> 20) < best) { best = b.viol_assert >> 20; kind = 2; }
      if (b.viol_inv != ~0ULL && (b.viol_inv >> 20) < best) { best = b.viol_inv >> 20; kind = 1; }
      if (b.viol_deadlock != ~0ULL && (b.viol_deadlock >> 20) < best) { best = b.viol_deadlock >> 20; kind = 3; }
      out->verdict = kind; out->walk = b.first + best; out->step = stopped - 1;
      if (kind == 4) { out->detail = (int)((b.viol_trap >> 16) & 15); out->detail2 = (int)(b.viol_trap & 0xFFFF); }
      else if (kind == 2) out->detail = (int)(b.viol_assert & 0xFFFFF);
      else if (kind == 1) out->detail = (int)(b.viol_inv & 0xFFFFF);
      break;
    }
  }
  for (uint32_t t = 0; t < depth; ++t) {
    if (hist_out) memcpy(hist_out + (uint64_t)t * n * W, b.hist + (uint64_t)t * B * W, n * (size_t)W * 4);
    if (act_out) memcpy(act_out + (uint64_t)t * n, b.act + (uint64_t)t * B, n * 2);
  }
  if (len_out) memcpy(len_out, len, n * 4);
  free(dist); free(b.hist); free(b.act); free(status); free(len); free(frame);
  return 0;
}

uint64_t tlagcpu_sim_draw(uint64_t seed, uint64_t w, uint32_t t, uint32_t j) { return tlag_sim_draw(seed, w, t, j); }
uint64_t tlagcpu_sim_batch(uint32_t W, uint32_t D, uint64_t num) { return tlag_sim_batch(W, D, num); }
uint64_t tlagcpu_sim_term(uint64_t fp, uint64_t w, uint32_t t, int32_t act) { return tlag_sim_term(fp, w, t, act); }
uint64_t tlagcpu_fingerprint(const uint32_t *w, int W) { return tlag_fingerprint(w, W); }

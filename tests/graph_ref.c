/* CPU reference of the state graph (test infrastructure, tests/test_state_graph.py): tlag_build_graph's semantics
 * (include/tlag.h) on the host, over a caller's list of stored states.  Next runs on the bytecode interpreter, and pack,
 * unpack, the fingerprint and the edge term come from tla_rust_b200/csrc/tlag_vm.h, which the engine includes too; the
 * enumeration and the lookup are written out again here.  The model struct is oracle/cpu_engine.py's CpuModel. */
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
  uint32_t flags;
  uint32_t table_log2;
  uint64_t max_states;
} cpu_model;

typedef struct { uint64_t s, t; int64_t a; } edge;

static int edge_cmp(const void *x, const void *y) {
  const edge *a = (const edge *)x, *b = (const edge *)y;
  if (a->s != b->s) return a->s < b->s ? -1 : 1;
  if (a->t != b->t) return a->t < b->t ? -1 : 1;
  return a->a < b->a ? -1 : (a->a > b->a);
}

/* The edges out of rows [0, n_expanded) of `states` (n_states rows of W words), sorted by (s, t, a) and distinct.  The
 * first min(total, cap) go to src / dst / act.  Returns the total, or -1 (bad arguments or memory), -2 (a successor is
 * not in `states`), -3 (Next trapped or a successor does not pack). */
int64_t tlagcpu_graph(const cpu_model *m, const uint32_t *states, uint64_t n_states, uint64_t n_expanded, uint32_t *src,
                      uint32_t *dst, int32_t *act, uint64_t cap) {
  const int W = (int)m->W;
  if (n_expanded > n_states || W < 1 || W > MAXW) return -1;
  /* fingerprint -> row: open addressing over twice the rows */
  uint64_t slots = 2;
  while (slots < 2 * n_states) slots <<= 1;
  uint64_t *fps = (uint64_t *)calloc(slots, 8);
  uint64_t *rows = (uint64_t *)malloc(slots * 8);
  int32_t *frame = (int32_t *)calloc(m->frame_words + 8, 4);
  uint64_t n_e = 0, cap_e = 1024;
  edge *es = (edge *)malloc(cap_e * sizeof(edge));
  int64_t rc = 0;
  if (!fps || !rows || !frame || !es) { rc = -1; goto done; }
  for (uint64_t i = 0; i < n_states; ++i) {
    const uint64_t fp = tlag_fingerprint(states + i * W, W);
    uint64_t h = fp & (slots - 1);
    while (fps[h] && fps[h] != fp) h = (h + 1) & (slots - 1);
    fps[h] = fp; rows[h] = i;
  }
  for (uint64_t s = 0; s < n_expanded; ++s) {
    const uint32_t *in = states + s * W;
    uint32_t succ[MAXW];
    tlag_unpack(m->layout, (int)m->n_slots, in, frame);
    uint32_t pc = m->entry_next;
    for (;;) {
      int32_t info = 0, info2 = 0;
      const int ev = tlag_vm_run(m->code, m->cpool, frame, &pc, &info, &info2, MAX_STEPS);
      if (ev == TLAG_EV_HALT) break;
      if (ev == TLAG_EV_GEN || ev == TLAG_EV_INVF || ev == TLAG_EV_ASSERT) continue;
      if (ev != TLAG_EV_EMIT) { rc = -3; goto done; }
      int ov;
      if (info2 > 0) {
        memcpy(succ, in, (size_t)W * 4);
        ov = tlag_pack_ranges(m->layout, m->cpool, info2, frame + m->unpacked_words, succ);
      } else ov = tlag_pack(m->layout, (int)m->n_slots, frame + m->unpacked_words, succ, W);
      if (ov) { rc = -3; goto done; }
      const uint64_t fp = tlag_fingerprint(succ, W);
      uint64_t h = fp & (slots - 1);
      while (fps[h] && fps[h] != fp) h = (h + 1) & (slots - 1);
      if (!fps[h]) { rc = -2; goto done; }
      if (rows[h] == s) continue;
      if (n_e == cap_e) {
        cap_e *= 2;
        edge *ne = (edge *)realloc(es, cap_e * sizeof(edge));
        if (!ne) { rc = -1; goto done; }
        es = ne;
      }
      es[n_e].s = s; es[n_e].t = rows[h]; es[n_e].a = info;
      ++n_e;
    }
  }
  qsort(es, n_e, sizeof(edge), edge_cmp);
  for (uint64_t i = 0; i < n_e; ++i) {
    if (i && !edge_cmp(&es[i], &es[i - 1])) continue;
    if ((uint64_t)rc < cap) { src[rc] = (uint32_t)es[i].s; dst[rc] = (uint32_t)es[i].t; act[rc] = (int32_t)es[i].a; }
    ++rc;
  }
done:
  free(fps); free(rows); free(frame); free(es);
  return rc;
}

uint64_t tlagcpu_edge_term(uint64_t fp_s, uint64_t fp_t, int32_t a) { return tlag_edge_term(fp_s, fp_t, a); }
uint64_t tlagcpu_fingerprint(const uint32_t *w, int W) { return tlag_fingerprint(w, W); }

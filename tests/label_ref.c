/* CPU reference of the label pass (test infrastructure, tests/test_liveness.py): tlag_label_graph's state and edge
 * programs (include/tlag.h) run on the bytecode interpreter of tla_rust_b200/csrc/tlag_vm.h, which the engine includes
 * too, over caller-given packed states.  t == NULL: the state program on s[i]; else the edge program on (s[i], t[i]). */
#include <stdint.h>
#include <stdlib.h>

#include "../tla_rust_b200/csrc/tlag_vm.h"

/* out[i] = the predicates of [0, n_preds) that hold.  Returns 0, or -1 (bad arguments or memory), -2 (a trap) */
int tlagcpu_labels(const uint64_t *code, const int32_t *cpool, uint32_t entry, const tlag_slot *layout, int n_slots,
                   uint32_t frame_words, uint32_t unpacked_words, int W, const uint32_t *s, const uint32_t *t, uint64_t n,
                   uint32_t n_preds, uint32_t *out) {
  if (n_preds > 32 || W < 1) return -1;
  int32_t *frame = (int32_t *)calloc(frame_words + 8, 4);
  if (!frame) return -1;
  const uint32_t all = n_preds == 32 ? 0xFFFFFFFFu : (1u << n_preds) - 1;
  int rc = 0;
  for (uint64_t i = 0; i < n && !rc; ++i) {
    tlag_unpack(layout, n_slots, s + i * W, frame);
    if (t) tlag_unpack(layout, n_slots, t + i * W, frame + unpacked_words);
    uint32_t pc = entry, fails = 0;
    for (;;) {
      int32_t info = 0, info2 = 0;
      const int ev = tlag_vm_run(code, cpool, frame, &pc, &info, &info2, 1ull << 38);
      if (ev == TLAG_EV_HALT) break;
      if (ev != TLAG_EV_INVF) { rc = -2; break; }
      fails |= 1u << (info & 31);
    }
    out[i] = ~fails & all;
  }
  free(frame);
  return rc;
}

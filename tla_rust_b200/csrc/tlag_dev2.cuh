// tlag_dev2.cuh -- second half of the slice runtime: needs the generated constants (TLAG_SL_W ...), so it is included
// by a slice translation unit AFTER tlag_dev.cuh; defines the successor handling and the per-slice kernel macros.
#pragma once

#ifdef TLAG_SL_SIM
// simulation: the successor is the step's next candidate of the walk's reservoir pick
static __device__ __noinline__ void sl_emit_words(tlag_sl_cx* cx, int aid, const uint32_t* o) {
  cx->nsucc++; cx->gen++;
  sim_pick(*cx->sim, cx->idx, cx->cnt++, aid, o, TLAG_SL_W);
}
#else
// successor already packed: fingerprint -> seen-set (or owner's send region) -> store
static __device__ __noinline__ void sl_emit_words(tlag_sl_cx* cx, int aid, const uint32_t* o) {
  const DevParams& p = *cx->p;
  constexpr int W = TLAG_SL_W;
  cx->nsucc++; cx->gen++;
  uint32_t w[W];
#pragma unroll
  for (int i = 0; i < W; ++i) w[i] = o[i];
  const unsigned long long fp = tlag_fingerprint(w, W);
  // route mode: a successor this rank owns itself never leaves the GPU (1/N of the records)
  const int owner = p.route ? (int)tlag_owner_k(w, W, (uint32_t)p.n_ranks, p.owner_words) : p.rank;
  if (!p.route || owner == p.rank) {
    // the tail allocation is aggregated over whichever lanes arrived here together
    if (seen_report(p.ctr, seen_insert(p.table, p.mask, fp)))
      store_append(p, __activemask(), w, W, (uint32_t)cx->idx, tlag_meta(aid, p.rank));
  } else {
    route_append(p, w, W, fp, owner, (uint32_t)cx->idx, tlag_meta(aid, p.rank));
  }
}
#endif

// array form: pack the primed frame (all slots, or the dirty ranges over a copy of the parent) first
static __device__ __noinline__ void sl_emit_frame(tlag_sl_cx* cx, const int32_t* f, int aid, int dirty) {
  const DevParams& p = *cx->p;
  constexpr int W = TLAG_SL_W;
  uint32_t succ[W];
  int ov;
  if (dirty > 0) {
#pragma unroll
    for (int i = 0; i < W; ++i) succ[i] = cx->src[i];
    ov = tlag_pack_ranges(p.layout, p.cpool, dirty, f + TLAG_SL_USZ, succ);
  } else {
    ov = tlag_pack(p.layout, p.n_slots, f + TLAG_SL_USZ, succ, W);
  }
  if (ov) {
    cx->nsucc++; cx->gen++;
    report_min(&p.ctr->viol_trap, (cx->idx << 20) | (2ULL << 16) | (unsigned)((ov - 1) & 0xFFFF));
#ifdef TLAG_SL_SIM
    cx->stat = SIM_FAILED;
#endif
    return;
  }
  // (no self-loop test here: comparing every word with the parent's row in memory cost raft 1 % of its wave time and
  // saved SSI none; the scalar form tests its registers, compile/sliced.py: emit_stmt)
  sl_emit_words(cx, aid, succ);
}


#ifdef TLAG_SL_STAGED
// The whole warp: fingerprint the staged successors and probe the seen-set for them, then append the new ones to the
// store (its discovery buffer while the level has one) as one contiguous run (one tail atomic, coalesced stores).  Semantics as sl_emit_words: a row past the store's
// capacity is counted in n_states and reported as an overflow, a full table as table_full.
static __device__ __forceinline__ void sl_flush(const DevParams& p, unsigned cap) {
  constexpr int W = TLAG_SL_W, R = TLAG_SL_STAGE_SLOTS / 32;
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncwarp();
  const unsigned n = min(tlag_sl_fill[warp], cap);
  unsigned long long fp[R], cur[R];
  // every table load of this lane is issued before any is examined: R probes in flight per lane
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const unsigned s = r * 32 + lane;
    fp[r] = 0; cur[r] = 0;
    if (s < n) {
      uint32_t w[W];
#pragma unroll
      for (int k = 0; k < W; ++k) w[k] = tlag_sl_stage[warp][k][s];
      fp[r] = tlag_fingerprint(w, W);
      cur[r] = __ldcv(&p.table[fp[r] & p.mask]);
    }
  }
  unsigned total = 0;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int ins = r * 32 + lane < n ? seen_report(p.ctr, seen_insert_at(p.table, p.mask, fp[r], cur[r])) : 0;
    const unsigned m = __ballot_sync(0xffffffffu, ins > 0);
    if (ins > 0) tlag_sl_row[warp][total + __popc(m & lanemask_lt())] = (unsigned short)(r * 32 + lane);
    total += __popc(m);
  }
  if (total) {
    unsigned long long base = 0;
    if (lane == 0) base = atomicAdd(&p.ctr->n_states, (unsigned long long)total);
    base = __shfl_sync(0xffffffffu, base, 0);
    __syncwarp();
    for (unsigned t = lane; t < total * W; t += 32) {
      const unsigned row = t / W, k = t - row * W;
      const unsigned long long pos = base + row;
      if (pos < p.cap_states) row_dst(p, pos).w[k] = tlag_sl_stage[warp][k][tlag_sl_row[warp][row]];
    }
    for (unsigned row = lane; row < total; row += 32) {
      const unsigned long long pos = base + row;
      const unsigned s = tlag_sl_row[warp][row];
      if (pos < p.cap_states) {
        const RowDst d = row_dst(p, pos);
        *d.parent = tlag_sl_stage[warp][W][s];
        *d.meta = tlag_sl_stage[warp][W + 1][s];
      } else {
        atomicExch(&p.ctr->store_overflow, 1ULL);
      }
    }
  }
  __syncwarp();
  if (lane == 0) tlag_sl_fill[warp] = 0;
  __syncwarp();
}
#endif

// One thread per frontier state (grid-stride).  A staged Next kernel strides over whole warps, so that a warp is
// converged at the bottom of every iteration and can flush its staged successors together; the other kernels keep one
// lane per state.  FN: the slice function of this kernel.
template <int PHASE, typename FN>
__device__ __forceinline__ void sl_run(const DevParams& p, unsigned long long lo, unsigned long long hi, FN fn) {
  constexpr int W = TLAG_SL_W;
#ifdef TLAG_SL_STAGED
  constexpr bool staged = PHASE == 1;
#else
  constexpr bool staged = false;
#endif
  tlag_sl_cx cxs;
  tlag_sl_cx* cx = &cxs;
  cx->p = &p; cx->gen = 0; cx->phase = PHASE;
  const unsigned lane = threadIdx.x & 31;
#ifdef TLAG_SL_STAGED
  cx->stage_cap = 0;
  if (staged) {
    // route mode keeps the direct path: its send regions and sent-cache have their own ordering
    cx->stage_cap = p.route ? 0u : min((unsigned)p.stage, (unsigned)TLAG_SL_STAGE_SLOTS);
    if (lane == 0) tlag_sl_fill[threadIdx.x >> 5] = 0;
    __syncwarp();
  }
#endif
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long i0 = lo + (unsigned long long)blockIdx.x * blockDim.x + (staged ? threadIdx.x & ~31u : threadIdx.x);
       i0 < hi; i0 += stride) {
    const unsigned long long idx = staged ? i0 + lane : i0;
    if (!staged || idx < hi) {
      const uint32_t* src = p.states + idx * (unsigned long long)W;
      cx->idx = idx; cx->nsucc = 0;
      // the slice unpacks the slots it reads (liveness, compile/sliced.py) straight out of these registers
      uint32_t in_[W];
#pragma unroll
      for (int i = 0; i < W; ++i) in_[i] = src[i];
      cx->src = src;                 // (the global row: taking the address of in_ would force it out of registers)
      fn(p.cpool, in_, cx);
      if (PHASE == 1 && cx->nsucc && p.succ_flag) p.succ_flag[idx - lo] = 1;
    }
#ifdef TLAG_SL_STAGED
    // flush at half full: the next iteration's successors then usually fit
    if (staged) {
      __syncwarp();
      if (tlag_sl_fill[threadIdx.x >> 5] >= cx->stage_cap / 2) sl_flush(p, cx->stage_cap);
    }
#endif
  }
#ifdef TLAG_SL_STAGED
  if (staged) sl_flush(p, cx->stage_cap);
#endif
  // generated counter: warp reduce, one atomic per warp
  unsigned long long g = cx->gen;
  if (PHASE == 1) {
    for (int o = 16; o > 0; o >>= 1) g += __shfl_down_sync(0xffffffffu, g, o);
    if ((threadIdx.x & 31) == 0 && g) atomicAdd(&p.ctr->generated, g);
  }
}

#ifdef TLAG_SL_SIM
// Simulation: step s.t of a batch, one thread per walk of row t (p.states).  Ended walks are skipped, and so are walks
// that failed this step's invariants when Next runs; the reservoir count goes from one slice kernel to the next in
// s.cnt.  The slices run in program order, so the candidates come in the interpreter's order.
template <int PHASE, typename FN>
__device__ __forceinline__ void sl_sim_run(const DevParams& p, const SimParams& s, unsigned long long hi, FN fn) {
  constexpr int W = TLAG_SL_W;
  if (sim_stopped(s) || (PHASE == 1 && s.t + 1 >= s.depth)) return;
  tlag_sl_cx cxs;
  tlag_sl_cx* cx = &cxs;
  cx->p = &p; cx->sim = &s; cx->gen = 0; cx->phase = PHASE;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; idx < hi; idx += stride) {
    const int st = s.status[idx];
    if (st == SIM_ENDED || (PHASE == 1 && st == SIM_FAILED)) continue;
    const uint32_t* src = p.states + idx * (unsigned long long)W;
    cx->idx = idx; cx->nsucc = 0; cx->stat = st; cx->cnt = PHASE == 1 ? s.cnt[idx] : 0u;
    uint32_t in_[W];
#pragma unroll
    for (int i = 0; i < W; ++i) in_[i] = src[i];
    cx->src = src;
    fn(p.cpool, in_, cx);
    if (cx->stat != st) s.status[idx] = (uint8_t)cx->stat;
    if (PHASE == 1) {
      s.cnt[idx] = cx->cnt;
      if (cx->nsucc) p.succ_flag[idx] = 1;
    }
  }
  unsigned long long g = cx->gen;
  if (PHASE == 1) {
    for (int o = 16; o > 0; o >>= 1) g += __shfl_down_sync(0xffffffffu, g, o);
    if ((threadIdx.x & 31) == 0 && g) atomicAdd(&p.ctr->generated, g);
  }
}

#define TLAG_SL_KERNEL_INV(j)                                                                                      \
  __global__ void __launch_bounds__(TLAG_SL_BLOCK, TLAG_SL_OCC) k_sl_sim_inv_##j(                                  \
      const __grid_constant__ DevParams p, const __grid_constant__ SimParams s, unsigned long long hi) {            \
    sl_sim_run<0>(p, s, hi, [](const int32_t* cp, const uint32_t* f, tlag_sl_cx* cx) { tlag_sl_inv_##j(cp, f, cx); }); \
  }
#define TLAG_SL_KERNEL_NEXT(j)                                                                                     \
  __global__ void __launch_bounds__(TLAG_SL_BLOCK, TLAG_SL_OCC) k_sl_sim_next_##j(                                 \
      const __grid_constant__ DevParams p, const __grid_constant__ SimParams s, unsigned long long hi) {            \
    sl_sim_run<1>(p, s, hi, [](const int32_t* cp, const uint32_t* f, tlag_sl_cx* cx) { tlag_sl_next_##j(cp, f, cx); }); \
  }
#define TLAG_SL_LAUNCH_INV(j)                                                                                      \
  extern "C" void tlag_sl_sim_launch_inv_##j(const DevParams* p, const SimParams* s, unsigned long long hi,         \
                                             unsigned blocks, cudaStream_t st) {                                   \
    k_sl_sim_inv_##j<<<blocks, TLAG_SL_BLOCK, 0, st>>>(*p, *s, hi);                                                \
  }
#define TLAG_SL_LAUNCH_NEXT(j)                                                                                     \
  extern "C" void tlag_sl_sim_launch_next_##j(const DevParams* p, const SimParams* s, unsigned long long hi,        \
                                              unsigned blocks, cudaStream_t st) {                                  \
    k_sl_sim_next_##j<<<blocks, TLAG_SL_BLOCK, 0, st>>>(*p, *s, hi);                                               \
  }
#else
#define TLAG_SL_FARG const uint32_t*
#define TLAG_SL_KERNEL_INV(j)                                                                                     \
  __global__ void __launch_bounds__(TLAG_SL_BLOCK, TLAG_SL_OCC) k_sl_inv_##j(const __grid_constant__ DevParams p, \
                                                                            unsigned long long lo, unsigned long long hi) { \
    sl_run<0>(p, lo, hi, [](const int32_t* cp, TLAG_SL_FARG f, tlag_sl_cx* cx) { tlag_sl_inv_##j(cp, f, cx); });  \
  }
#define TLAG_SL_KERNEL_NEXT(j)                                                                                     \
  __global__ void __launch_bounds__(TLAG_SL_BLOCK, TLAG_SL_OCC) k_sl_next_##j(const __grid_constant__ DevParams p, \
                                                                             unsigned long long lo, unsigned long long hi) { \
    sl_run<1>(p, lo, hi, [](const int32_t* cp, TLAG_SL_FARG f, tlag_sl_cx* cx) { tlag_sl_next_##j(cp, f, cx); });  \
  }

// launcher the engine's translation unit calls (kernels live in the slice units)
#define TLAG_SL_LAUNCH_INV(j)                                                                                      \
  extern "C" void tlag_sl_launch_inv_##j(const DevParams* p, unsigned long long lo, unsigned long long hi, unsigned blocks, \
                                         cudaStream_t st) { k_sl_inv_##j<<<blocks, TLAG_SL_BLOCK, 0, st>>>(*p, lo, hi); }
#define TLAG_SL_LAUNCH_NEXT(j)                                                                                     \
  extern "C" void tlag_sl_launch_next_##j(const DevParams* p, unsigned long long lo, unsigned long long hi, unsigned blocks, \
                                          cudaStream_t st) { k_sl_next_##j<<<blocks, TLAG_SL_BLOCK, 0, st>>>(*p, lo, hi); }
#endif  // TLAG_SL_SIM

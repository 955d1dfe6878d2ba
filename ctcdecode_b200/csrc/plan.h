// Everything derived from (config, B, T): pruning mode, row padding, shared-memory layout, block size
// and the workspace carve-up.  Shared by the CUDA library and the CPU logic-test emulation.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>

#include "../../include/ctcdecode_b200.h"
#include "beam_core.cuh"

namespace ctc {

struct Plan {
  bool sorted;    // the reference sorts (and possibly cuts) the vocabulary every frame
  int cp_active;  // log(cutoff_prob) < 0
  int n_max;      // most characters a frame can keep
  int NP;         // row length of the pruned log-prob rows (multiple of 8, >= n_max + kRowTrailer)
  int P;          // next power of two >= V
  int F;          // frames per staged tile
  int NT;         // threads per CTA of the beam kernel
  int budget_kb;  // shared-memory budget per CTA the layout was made for (make_layout)
  SmemLayout L;
  size_t off_lp, off_idx, off_arena, off_state, total;
  long long arena_stride, state_stride;
};

static inline size_t al256(size_t x) { return (x + 255) / 256 * 256; }

// streaming multiprocessors of the H100 SXM the launch shapes are sized for (one wave = kNumSMs x CTAs per SM)
constexpr int kNumSMs = 132;
// dynamic shared memory one CTA can opt into on the H100 (cudaDevAttrMaxSharedMemoryPerBlockOptin)
constexpr int kMaxSmemPerCTA = 227 * 1024;

// Launch shape of the prune kernel (prune_program.cuh): a 2 KB head, then per warp the sort keys of the vocabulary
// (sorted mode, P u64) and, for logits, a staging row of the log-softmax; as many warps per CTA (up to 8) as ~200 KB
// hold.  The plan refuses a vocabulary whose sort keys alone exceed that (make_plan_core).
struct PruneShape {
  int wpc;      // warps per CTA, one frame per warp
  size_t smem;  // dynamic shared memory per CTA, bytes
};
static inline PruneShape prune_shape(const Plan &pl, int V, bool logits) {
  const size_t row_bytes = logits ? (size_t)((V + 3) / 4 * 4) * 4 : 0;
  const size_t per_warp = (pl.sorted ? (size_t)pl.P * 8 : 0) + row_bytes;
  int wpc = 8;
  if (per_warp > 0) wpc = (int)std::max<size_t>(1, std::min<size_t>(8, (200 * 1024 - 2048) / per_warp));
  return PruneShape{wpc, 2048 + (size_t)wpc * per_warp};
}

// Workspace carve-up: the pruned rows of `rows` input utterances, then the node arenas and state blocks of `ctas` beam
// CTAs (the same number except in a sweep of the LM weights, where P pairs decode each input row).
static inline void plan_regions(Plan *pl, int rows, int ctas, int T) {
  size_t o = 0;
  pl->off_lp = o;     o = al256(o + (size_t)rows * T * pl->NP * 4);
  pl->off_idx = o;    o = al256(o + (pl->sorted ? (size_t)rows * T * pl->NP * 2 : 0));
  pl->off_arena = o;  o = al256(o + (size_t)ctas * pl->arena_stride * sizeof(Node));
  pl->off_state = o;  o = al256(o + (size_t)ctas * pl->state_stride * 4);
  pl->total = o;
}

// b_sched: the number of utterances that will be in flight on the device together (>= B when the caller runs
// several groups of B concurrently); decides between the latency and the throughput shape of the beam kernel.
// lm: a scorer is attached.  Its beam kernel carries the [KP][WC] dictionary masks as well (make_layout(..., lm =
// true)), and pl->L is that layout.  It keeps the two-CTAs-per-SM budget at every batch size: a scorer decode spends
// its frames in the per-frame host handshake, so three CTAs per SM would not make it faster.
static inline int make_plan_core(const ctcdec_config *cfg, int B, int T, Plan *pl, char *msg, size_t msglen,
                                 int nt_override = 0, int b_sched = 0, bool lm = false) {
#define PLAN_FAIL(code, ...) do { snprintf(msg, msglen, __VA_ARGS__); return code; } while (0)
  if (!cfg) PLAN_FAIL(CTCDEC_E_INVALID, "cfg is NULL");
  const int V = cfg->vocab_size, K = cfg->beam_size;
  if (B < 0 || T < 0) PLAN_FAIL(CTCDEC_E_INVALID, "negative batch (%d) or time (%d)", B, T);
  if (V < 1 || V > 65534) PLAN_FAIL(CTCDEC_E_UNSUPPORTED, "vocab_size %d outside [1, 65534]", V);
  if (K < 1 || K > 4096) PLAN_FAIL(CTCDEC_E_UNSUPPORTED, "beam_size %d outside [1, 4096]", K);
  if (cfg->cutoff_top_n < 0) PLAN_FAIL(CTCDEC_E_INVALID, "cutoff_top_n %d < 0", cfg->cutoff_top_n);
  if (cfg->blank_id < 0) PLAN_FAIL(CTCDEC_E_INVALID, "blank_id %d < 0", cfg->blank_id);
  if ((long long)K * (long long)(T > 0 ? T : 1) + 1 > 0x7fffffffll / 2)
    PLAN_FAIL(CTCDEC_E_UNSUPPORTED, "beam_size * T too large for the node arena");
  // reference decoder_utils.cpp:15,21: sort (and possibly cut) iff log(cutoff_prob) < 0 or top_n < V
  const double log_cp = std::log(cfg->cutoff_prob);
  pl->cp_active = (log_cp < 0.0) ? 1 : 0;
  pl->sorted = pl->cp_active || cfg->cutoff_top_n < V;
  if (!pl->sorted) pl->n_max = V;
  else if (pl->cp_active) pl->n_max = std::min(V, std::max(1, cfg->cutoff_top_n));
  else pl->n_max = std::min(V, cfg->cutoff_top_n);
  pl->NP = align_up(pl->n_max + kRowTrailer, 8);
  int P = 64;  // (at least 64 sort words per warp: the partial top-n selection sorts up to 64 survivors)
  while (P < V) P <<= 1;
  pl->P = P;
  pl->F = std::max(1, std::min(32, 4096 / (pl->NP * 4)));
  const long long grid = (long long)K * pl->n_max;
  // 8 warps with 128 registers per utterance for a batch that fits the GPU in one go (an utterance is T serial
  // frames: latency counts).  A batch of several waves is a throughput problem instead: 4 warps per utterance and
  // as many CTAs per SM as shared memory allows (228 KB per SM: two CTAs of 111 KB or three of 74 KB).
  pl->NT = grid <= 512 ? 128 : 256;
  int budget_kb = 111;
  if (std::max(B, b_sched) > 2 * kNumSMs && nt_override == 0) {
    // three CTAs per SM
    pl->NT = 128;
    const SmemLayout t = make_layout(K, V, pl->NP, pl->F, pl->sorted, 128, false, 74);
    if (!lm && t.total <= 74 * 1024 && t.seg * 8 * 4 >= 8 * 1024) budget_kb = 74;
  }
  if (nt_override == 128 || nt_override == 160 || nt_override == 192 || nt_override == 256 || nt_override == 512 || nt_override == 1024) pl->NT = nt_override;
  pl->budget_kb = budget_kb;
  pl->L = make_layout(K, V, pl->NP, pl->F, pl->sorted, pl->NT, lm, budget_kb);
  if (pl->L.total > kMaxSmemPerCTA)
    PLAN_FAIL(CTCDEC_E_UNSUPPORTED,
              "beam_size %d x pruned vocab %d needs %d bytes of shared memory%s (> %d, the 227 KB a CTA can have)", K,
              pl->n_max, pl->L.total, lm ? " with a scorer" : "", kMaxSmemPerCTA);
  if (pl->sorted && 2048 + (size_t)P * 8 > 200 * 1024)
    PLAN_FAIL(CTCDEC_E_UNSUPPORTED, "vocab_size %d too large for the in-shared-memory vocabulary sort (at most 16384)", V);
  pl->arena_stride = 1 + (long long)K * T;
  pl->state_stride = (state_ints(K) + 63) / 64 * 64;
  plan_regions(pl, B, B, T);
  msg[0] = 0;
  return CTCDEC_OK;
#undef PLAN_FAIL
}

}  // namespace ctc

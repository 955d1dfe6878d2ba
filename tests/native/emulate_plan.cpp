// TEST INFRASTRUCTURE ONLY -- the launch plan (ctcdecode_b200/csrc/plan.h) of a configuration, as the library makes
// it, for tests/test_plan_envelope.py.  The product never builds or loads this file.
#define CTC_EMULATE 1
#include <cstring>

#include "../../ctcdecode_b200/csrc/beam_program.cuh"
#include "../../ctcdecode_b200/csrc/plan.h"

using namespace ctc;

extern "C" {

// The whole plan for a configuration (lm: a scorer is attached): out[0..7] = NT, KP, budget_kb, seg, smem total, F,
// NP, sorted; out[8..17] = the layout's tail offsets evcnt, mask, mask2, rmask, dmask, rank, tile_lp, tile_idx, clk,
// cli; out[18..21] = W, WC, NW, P; out[22..23] = finalize / committed kernel shared memory; out[24..27] = prune kernel
// warps per CTA and shared memory for probabilities, then for logits; out[28] = n_max.  On refusal returns the
// CTCDEC_E_* code and the plan's message in msg.
int emu_plan_full(int B, int T, int V, int K, double cutoff_prob, int cutoff_top_n, int lm, int *out, char *msg,
                  int msglen) {
  ctcdec_config cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.vocab_size = V; cfg.beam_size = K; cfg.cutoff_top_n = cutoff_top_n; cfg.cutoff_prob = cutoff_prob;
  Plan pl;
  const int rc = make_plan_core(&cfg, B, T, &pl, msg, (size_t)msglen, 0, 0, lm != 0);
  if (rc) return rc;
  const SmemLayout &L = pl.L;
  const PruneShape probs = prune_shape(pl, V, false), logits = prune_shape(pl, V, true);
  const int v[] = {pl.NT, L.KP, pl.budget_kb, L.seg, L.total, pl.F, pl.NP, pl.sorted ? 1 : 0,
                   L.evcnt, L.mask, L.mask2, L.rmask, L.dmask, L.rank, L.tile_lp, L.tile_idx, L.clk, L.cli,
                   L.W, L.WC, L.NW, pl.P, (int)finalize_smem_bytes(K), (int)committed_smem_bytes(K),
                   probs.wpc, (int)probs.smem, logits.wpc, (int)logits.smem, pl.n_max};
  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) out[i] = v[i];
  return 0;
}

}  // extern "C"

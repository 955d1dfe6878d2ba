// TEST INFRASTRUCTURE ONLY -- the offline decode of an uncut vocabulary as the device entry point runs it: one beam
// launch whose CTAs run the backtrace (finalize_cta_run) in their epilogue (BeamParams::backtrace), in the shared
// memory behind the layout's head.  Builds on emulate_cta.cpp (its host mirror of the prune scan and its beam
// launcher); tests/test_backtrace_emulation.py compiles this file into tests/native/_build/.  The product never builds
// or loads it.
#include "emulate_cta.cpp"

extern "C" {

// emu_decode_batch in one go (no chunks), with the backtrace in the beam program's epilogue and no separate finalize.
// Returns CTCDEC_E_UNSUPPORTED when the plan does not take that path (a cut vocabulary).
int emu_decode_batch_backtrace(const float *probs, const int *seq_lens, int B, int T, int V, int K, double cutoff_prob,
                               int cutoff_top_n, int blank, int log_input, int NT, int *tokens, int *timesteps,
                               float *scores, int *lens, int *n_results, int *flags) {
  ctcdec_config cfg;
  cfg.vocab_size = V; cfg.beam_size = K; cfg.blank_id = blank; cfg.log_input = log_input;
  cfg.cutoff_top_n = cutoff_top_n; cfg.cutoff_prob = cutoff_prob;
  Plan pl;
  char msg[256];
  int rc = make_plan_core(&cfg, B, T, &pl, msg, sizeof(msg));
  if (rc) { fprintf(stderr, "emu: %s\n", msg); return rc; }
  if (NT <= 0) NT = pl.NT;
  pl.NT = NT;
  pl.L = make_layout(K, V, pl.NP, pl.F, pl.sorted, NT);
  if (!cta_backtrace(pl.sorted, K, pl.L)) return CTCDEC_E_UNSUPPORTED;
  std::vector<float> lp((size_t)B * T * pl.NP + 8, 0.f);
  std::vector<Node> arena((size_t)B * pl.arena_stride);
  std::vector<int> state((size_t)B * pl.state_stride, 0);
  // exactly the layout's size: the epilogue's backtrace must fit behind the head
  std::vector<unsigned char> smem(pl.L.total);
  for (int b = 0; b < B; ++b) flags[b] = 0;
  prune_rows(cfg, pl, probs, seq_lens, B, T, lp.data(), nullptr, flags);

  BeamParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.V = V; bp.NP = pl.NP; bp.K = K; bp.blank = blank; bp.tile_frames = pl.F; bp.L = pl.L;
  bp.arena = arena.data(); bp.arena_stride = pl.arena_stride; bp.state = state.data();
  bp.state_stride = pl.state_stride; bp.arena_cap = (int)pl.arena_stride;
  bp.out_tokens = tokens; bp.out_timesteps = timesteps; bp.out_scores = scores; bp.out_lens = lens;
  bp.n_results = n_results; bp.out_T = T; bp.flags = flags;
  bp.no_fast = getenv("CTC_EMU_NO_FAST") ? atoi(getenv("CTC_EMU_NO_FAST")) : 0;
  g_emu_order = getenv("CTC_EMU_ORDER") ? atoi(getenv("CTC_EMU_ORDER")) : 0;  // test knob: order of the emulated threads
  bp.lp = lp.data(); bp.T = T; bp.seq_lens = seq_lens; bp.fresh = 1;
  bp.backtrace = 1;
  switch (NT) {
    case 128: run_beam<128>(bp, false, B, smem.data()); break;
    case 160: run_beam<160>(bp, false, B, smem.data()); break;
    case 192: run_beam<192>(bp, false, B, smem.data()); break;
    case 256: run_beam<256>(bp, false, B, smem.data()); break;
    case 1024: run_beam<1024>(bp, false, B, smem.data()); break;
    default: run_beam<512>(bp, false, B, smem.data()); break;
  }
  return 0;
}

}  // extern "C"

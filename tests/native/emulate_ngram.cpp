// TEST INFRASTRUCTURE ONLY -- the scorer path with the library's own ARPA scorer (BeamParams::lm_dev: the CTA computes
// the LM terms itself) in the single-threaded CPU emulation of the CTA program.  Builds on emulate_cta.cpp (its host
// mirror of the prune scan and its beam launcher); tests/test_ngram_emulation.py compiles this file into
// tests/native/_build/.  The product never builds or loads it.
#include "emulate_cta.cpp"

extern "C" {

// Offline decode with the ARPA model at `path` (loaded and checked as ctcdec_scorer_create_arpa does).  chunk > 0 feeds
// the frames in launches of that many frames over the saved state (the streaming shape); the read-out rescores through
// the scorer's own host hooks, as the library does.  Returns 0 or a CTCDEC_E_* code.
int emu_decode_batch_ngram(const float *probs, const int *seq_lens, int B, int T, int V, int K, double cutoff_prob,
                           int cutoff_top_n, int blank, int log_input, int NT, int chunk, const char *path,
                           double alpha, double beta, const char *const *labels, int *tokens, int *timesteps,
                           float *scores, int *lens, int *n_results, int *flags) {
  ctcdec_config cfg;
  cfg.vocab_size = V; cfg.beam_size = K; cfg.blank_id = blank; cfg.log_input = log_input;
  cfg.cutoff_top_n = cutoff_top_n; cfg.cutoff_prob = cutoff_prob;
  Plan pl;
  char msg[256];
  int rc = make_plan_core(&cfg, B, T, &pl, msg, sizeof(msg), true);
  if (rc) { fprintf(stderr, "emu: %s\n", msg); return rc; }
  if (NT <= 0) NT = pl.NT;
  pl.NT = NT;
  pl.L = make_layout(K, V, pl.NP, pl.F, pl.sorted, NT, true);

  std::shared_ptr<NgramModel> m = std::make_shared<NgramModel>();
  for (int i = 0; i < V; ++i) {
    m->labels.emplace_back(labels[i]);
    if (m->labels.back() == " ") m->space_id = i;
  }
  const std::string why = load_arpa(path, *m);
  if (!why.empty()) { fprintf(stderr, "emu: %s\n", why.c_str()); return CTCDEC_E_UNSUPPORTED; }
  HostScorer sc;
  sc.hooks.ctx = m.get(); sc.hooks.cond_log_prob = ngram_hook_cond; sc.hooks.sent_log_prob = ngram_hook_sent;
  sc.alpha = alpha; sc.beta = beta; sc.max_order = m->order; sc.is_character_based = m->is_character_based;
  sc.space_id = -2;
  for (int i = 0; i < V; ++i) { sc.labels.emplace_back(labels[i]); if (sc.labels.back() == " ") sc.space_id = i; }
  if (sc.space_id < 0 && !sc.is_character_based) return CTCDEC_E_UNSUPPORTED;
  sc.ngram = m;
  if (sc.is_character_based) {
    sc.dict = accept_all_dictionary(V);
  } else {
    sc.dict = build_dictionary(sc.labels, sc.space_id, m->vocabulary);
    pack_dictionary(sc.dict, sc.space_id);
  }
  lm_dev_word_ids(sc);

  std::vector<float> lp((size_t)B * T * pl.NP + 8, 0.f);
  std::vector<uint16_t> idx(pl.sorted ? (size_t)B * T * pl.NP + 8 : 8, 0);
  std::vector<Node> arena((size_t)B * pl.arena_stride);
  std::vector<float> lm_arena((size_t)B * pl.arena_stride, 0.f);
  std::vector<int> dstate_arena((size_t)B * pl.arena_stride, 0);
  std::vector<int> hist((size_t)B * pl.arena_stride * (sc.max_order - 1), -1);
  std::vector<int> state((size_t)B * pl.state_stride, 0);
  std::vector<float> lm_row(sc.is_character_based ? (size_t)B * pl.arena_stride * V : 1, 0.f);
  std::vector<unsigned char> smem(pl.L.total + 64);
  for (int b = 0; b < B; ++b) flags[b] = 0;
  prune_rows(cfg, pl, probs, seq_lens, B, T, lp.data(), idx.data(), flags);

  BeamParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.lp = lp.data(); bp.idx = pl.sorted ? idx.data() : nullptr; bp.seq_lens = seq_lens; bp.T = T;
  bp.V = V; bp.NP = pl.NP; bp.K = K; bp.blank = blank; bp.tile_frames = pl.F; bp.L = pl.L;
  bp.arena = arena.data(); bp.arena_stride = pl.arena_stride; bp.state = state.data();
  bp.state_stride = pl.state_stride; bp.arena_cap = (int)pl.arena_stride;
  bp.out_tokens = tokens; bp.out_timesteps = timesteps; bp.out_scores = scores; bp.out_lens = lens;
  bp.n_results = n_results; bp.out_T = T; bp.flags = flags;
  g_emu_order = getenv("CTC_EMU_ORDER") ? atoi(getenv("CTC_EMU_ORDER")) : 0;  // test knob: order of the emulated threads
  bp.dict_next = sc.dict.packed.data(); bp.dict_mask = sc.dict.mask.data(); bp.dict_wc = sc.dict.wc;
  bp.dict_start = sc.dict.start;
  bp.space_id = sc.space_id; bp.beta = beta; bp.lm_arena = lm_arena.data(); bp.dstate_arena = dstate_arena.data();
  bp.lm_char = sc.is_character_based; bp.lm_row = sc.is_character_based ? lm_row.data() : nullptr;
  bp.lm_dev = 1; bp.lm_alpha = alpha; bp.ngram = m->view();
  bp.word_of_state = sc.word_of_state.data(); bp.label_word = sc.label_word.data();
  bp.lm_hist_n = sc.max_order - 1; bp.lm_hist = hist.data();

  int tm = 0;
  for (int b = 0; b < B; ++b) tm = std::max(tm, std::min(seq_lens ? seq_lens[b] : T, T));
  for (int t0 = 0; t0 < std::max(tm, 1); t0 += (chunk > 0 ? chunk : std::max(tm, 1))) {
    bp.t0 = t0; bp.nframes = chunk > 0 ? chunk : 0; bp.fresh = t0 == 0 ? 1 : 0;
    switch (NT) {
      case 32: run_beam<32>(bp, pl.sorted, B, smem.data()); break;
      case 64: run_beam<64>(bp, pl.sorted, B, smem.data()); break;
      case 128: run_beam<128>(bp, pl.sorted, B, smem.data()); break;
      case 512: run_beam<512>(bp, pl.sorted, B, smem.data()); break;
      default: run_beam<256>(bp, pl.sorted, B, smem.data()); break;
    }
  }
  std::vector<unsigned char> fsmem(finalize_smem_bytes(K) + 64);
  for (int b = 0; b < B; ++b) finalize_cta_run<256>(bp, b, fsmem.data());
  lm_rescore_batch(sc, B, K, T, n_results, tokens, lens, scores);
  return 0;
}

}  // extern "C"

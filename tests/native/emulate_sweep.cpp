// TEST INFRASTRUCTURE ONLY -- a sweep of the LM weights (ctcdec_decode_batch_lm_sweep_async) in the single-threaded CPU
// emulation of the CTA program: P x B beam CTAs over one vocabulary scan of B utterances, CTA g decoding input row
// g % B with the pair g / B (BeamParams::sweep_B / lm_ab), then the read-out row by row with each row's pair
// (ngram_readout_row, the read-out kernel's function).  Builds on emulate_cta.cpp; tests/test_lm_sweep_emulation.py
// compiles this file into tests/native/_build/.  The product never builds or loads it.
#include "emulate_cta.cpp"
#include "../../ctcdecode_b200/csrc/ngram_kenlm.h"

extern "C" {

// alphas / betas [P] (each rounded through float32, as the library does); outputs [P, B, ...] like the library's.
// NT <= 0: the block size of a B-utterance decode.  Returns 0 or a CTCDEC_E_* code.
int emu_decode_sweep_ngram(const float *probs, const int *seq_lens, int B, int T, int V, int K, double cutoff_prob,
                           int cutoff_top_n, int blank, int log_input, int NT, const char *path, const double *alphas,
                           const double *betas, int P, const char *const *labels, int *tokens, int *timesteps,
                           float *scores, int *lens, int *n_results, int *flags) {
  ctcdec_config cfg;
  cfg.vocab_size = V; cfg.beam_size = K; cfg.blank_id = blank; cfg.log_input = log_input;
  cfg.cutoff_top_n = cutoff_top_n; cfg.cutoff_prob = cutoff_prob;
  const int G = P * B;
  Plan pl;
  char msg[256];
  int rc = make_plan_core(&cfg, B, T, &pl, msg, sizeof(msg), 0, 0, true);  // (the library's block size: a B-utterance decode's)
  if (rc) { fprintf(stderr, "emu: %s\n", msg); return rc; }
  if (NT <= 0) NT = pl.NT;
  pl.NT = NT;
  pl.L = make_layout(K, V, pl.NP, pl.F, pl.sorted, NT, true);

  std::shared_ptr<NgramModel> m = std::make_shared<NgramModel>();
  for (int i = 0; i < V; ++i) {
    m->labels.emplace_back(labels[i]);
    if (m->labels.back() == " ") m->space_id = i;
  }
  const std::string why = load_ngram_file(path, *m);
  if (!why.empty()) { fprintf(stderr, "emu: %s\n", why.c_str()); return CTCDEC_E_UNSUPPORTED; }
  HostScorer sc;
  sc.max_order = m->order; sc.is_character_based = m->is_character_based;
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
  std::vector<double> ab((size_t)2 * P);
  for (int p = 0; p < P; ++p) { ab[2 * p] = (double)(float)alphas[p]; ab[2 * p + 1] = (double)(float)betas[p]; }

  // the scan: B input rows, once; its flags go to slice 0 and are copied to the other slices
  std::vector<float> lp((size_t)B * T * pl.NP + 8, 0.f);
  std::vector<uint16_t> idx(pl.sorted ? (size_t)B * T * pl.NP + 8 : 8, 0);
  for (int g = 0; g < G; ++g) flags[g] = 0;
  prune_rows(cfg, pl, probs, seq_lens, B, T, lp.data(), idx.data(), flags);
  for (int g = B; g < G; ++g) flags[g] = flags[g % B];
  // everything else: per CTA
  std::vector<Node> arena((size_t)G * pl.arena_stride);
  std::vector<float> lm_arena((size_t)G * pl.arena_stride, 0.f);
  std::vector<int> dstate_arena((size_t)G * pl.arena_stride, 0);
  std::vector<int> hist((size_t)G * pl.arena_stride * (sc.max_order - 1), -1);
  std::vector<int> state((size_t)G * pl.state_stride, 0);
  std::vector<float> lm_row(sc.is_character_based ? (size_t)G * pl.arena_stride * V : 1, 0.f);
  std::vector<unsigned char> smem(pl.L.total + 64);

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
  bp.space_id = sc.space_id; bp.lm_arena = lm_arena.data(); bp.dstate_arena = dstate_arena.data();
  bp.lm_char = sc.is_character_based; bp.lm_row = sc.is_character_based ? lm_row.data() : nullptr;
  bp.lm_dev = 1; bp.ngram = m->view();
  bp.word_of_state = sc.word_of_state.data(); bp.label_word = sc.label_word.data();
  bp.lm_hist_n = sc.max_order - 1; bp.lm_hist = hist.data();
  // (lm_alpha / beta stay 0: a CTA that read them instead of its pair would show in the results)
  bp.sweep_B = B; bp.lm_ab = ab.data();
  bp.t0 = 0; bp.nframes = 0; bp.fresh = 1;
  switch (NT) {
    case 128: run_beam<128>(bp, pl.sorted, G, smem.data()); break;
    case 256: run_beam<256>(bp, pl.sorted, G, smem.data()); break;
    default: fprintf(stderr, "emu: NT %d\n", NT); return CTCDEC_E_INVALID;
  }
  std::vector<unsigned char> fsmem(finalize_smem_bytes(K) + 64);
  for (int g = 0; g < G; ++g) finalize_cta_run<256>(bp, g, fsmem.data());
  const NgramView v = m->view();
  const NgramFront f = m->front();
  for (int g = 0; g < G; ++g)
    for (int q = 0; q < n_results[g] && q < K; ++q) {
      const size_t r = (size_t)g * K + q;
      const int p = g / B;
      scores[r] = ngram_readout_row(v, f, tokens + r * T, lens[r], scores[r], ab[2 * p], ab[2 * p + 1]);
    }
  return 0;
}

}  // extern "C"

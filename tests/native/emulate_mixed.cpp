// TEST INFRASTRUCTURE ONLY -- a decode over several language models (ctcdec_decode_batch_lm_mixed_async) in the
// single-threaded CPU emulation of the CTA program: B beam CTAs, CTA b decoding with the LM slot lm_index[b] (its own
// model, dictionary, order and weights; BeamParams::lm_slots / lm_slot_of), then the read-out row by row with each
// row's slot (ngram_readout_row, the read-out kernel's function).  Builds on emulate_cta.cpp;
// tests/test_lm_mixed_emulation.py compiles this file into tests/native/_build/.  The product never builds or loads it.
#include <memory>

#include "emulate_cta.cpp"
#include "../../ctcdecode_b200/csrc/ngram_kenlm.h"

extern "C" {

// paths / alphas / betas [S]: the models and their weights (used as given, as a scorer created with them uses them);
// lm_index [B]; outputs [B, ...] like the library's.  NT <= 0: the block size of a B-utterance decode.  Returns 0 or a
// CTCDEC_E_* code.
int emu_decode_mixed_ngram(const float *probs, const int *seq_lens, int B, int T, int V, int K, double cutoff_prob,
                           int cutoff_top_n, int blank, int log_input, int NT, const char *const *paths,
                           const double *alphas, const double *betas, int S, const int *lm_index,
                           const char *const *labels, int *tokens, int *timesteps, float *scores, int *lens,
                           int *n_results, int *flags) {
  ctcdec_config cfg;
  cfg.vocab_size = V; cfg.beam_size = K; cfg.blank_id = blank; cfg.log_input = log_input;
  cfg.cutoff_top_n = cutoff_top_n; cfg.cutoff_prob = cutoff_prob;
  Plan pl;
  char msg[256];
  int rc = make_plan_core(&cfg, B, T, &pl, msg, sizeof(msg), 0, 0, true);
  if (rc) { fprintf(stderr, "emu: %s\n", msg); return rc; }
  if (NT <= 0) NT = pl.NT;
  pl.NT = NT;
  pl.L = make_layout(K, V, pl.NP, pl.F, pl.sorted, NT, true);

  std::vector<std::unique_ptr<HostScorer>> scorers;
  std::vector<LmSlot> slots((size_t)S);
  int hist_stride = 0;
  for (int s = 0; s < S; ++s) {
    std::shared_ptr<NgramModel> m = std::make_shared<NgramModel>();
    for (int i = 0; i < V; ++i) {
      m->labels.emplace_back(labels[i]);
      if (m->labels.back() == " ") m->space_id = i;
    }
    const std::string why = load_ngram_file(paths[s], *m);
    if (!why.empty()) { fprintf(stderr, "emu: %s\n", why.c_str()); return CTCDEC_E_UNSUPPORTED; }
    scorers.emplace_back(new HostScorer());
    HostScorer &sc = *scorers.back();
    sc.max_order = m->order; sc.is_character_based = m->is_character_based;
    sc.space_id = -2;
    for (int i = 0; i < V; ++i) { sc.labels.emplace_back(labels[i]); if (sc.labels.back() == " ") sc.space_id = i; }
    if (sc.space_id < 0 && !sc.is_character_based) return CTCDEC_E_UNSUPPORTED;
    if (sc.is_character_based != scorers[0]->is_character_based) return CTCDEC_E_UNSUPPORTED;
    sc.ngram = m;
    if (sc.is_character_based) {
      sc.dict = accept_all_dictionary(V);
    } else {
      sc.dict = build_dictionary(sc.labels, sc.space_id, m->vocabulary);
      pack_dictionary(sc.dict, sc.space_id);
    }
    lm_dev_word_ids(sc);
    LmSlot &sl = slots[s];
    sl.dict_next = sc.dict.packed.data(); sl.dict_mask = sc.dict.mask.data(); sl.dict_start = sc.dict.start;
    sl.lm_alpha = alphas[s]; sl.beta = betas[s];
    sl.ngram = m->view(); sl.front = m->front();
    sl.word_of_state = sc.word_of_state.data(); sl.label_word = sc.label_word.data(); sl.lm_hist_n = sc.max_order - 1;
    if (sl.lm_hist_n > hist_stride) hist_stride = sl.lm_hist_n;
  }
  std::vector<unsigned char> slot_of((size_t)B + 1);
  for (int b = 0; b < B; ++b) {
    if (lm_index[b] < 0 || lm_index[b] >= S) return CTCDEC_E_INVALID;
    slot_of[b] = (unsigned char)lm_index[b];
  }
  const HostScorer &s0 = *scorers[0];

  std::vector<float> lp((size_t)B * T * pl.NP + 8, 0.f);
  std::vector<uint16_t> idx(pl.sorted ? (size_t)B * T * pl.NP + 8 : 8, 0);
  for (int b = 0; b < B; ++b) flags[b] = 0;
  prune_rows(cfg, pl, probs, seq_lens, B, T, lp.data(), idx.data(), flags);
  std::vector<Node> arena((size_t)B * pl.arena_stride);
  std::vector<float> lm_arena((size_t)B * pl.arena_stride, 0.f);
  std::vector<int> dstate_arena((size_t)B * pl.arena_stride, 0);
  std::vector<int> hist((size_t)B * pl.arena_stride * hist_stride + 1, -1);
  std::vector<int> state((size_t)B * pl.state_stride, 0);
  std::vector<float> lm_row(s0.is_character_based ? (size_t)B * pl.arena_stride * V : 1, 0.f);
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
  // call-wide: the labels' space and the kind of model.  Of the call's own model fields only dict_next is set (a
  // dictionary selects the scorer kernel); the others stay 0, so a CTA that read them instead of its slot would show.
  bp.dict_next = s0.dict.packed.data();
  bp.dict_wc = s0.dict.wc; bp.space_id = s0.space_id; bp.lm_char = s0.is_character_based;
  bp.lm_arena = lm_arena.data(); bp.dstate_arena = dstate_arena.data();
  bp.lm_row = s0.is_character_based ? lm_row.data() : nullptr;
  bp.lm_dev = 1; bp.lm_hist = hist.data();
  bp.lm_slots = slots.data(); bp.lm_slot_of = slot_of.data(); bp.lm_hist_stride = hist_stride;
  bp.t0 = 0; bp.nframes = 0; bp.fresh = 1;
  switch (NT) {
    case 128: run_beam<128>(bp, pl.sorted, B, smem.data()); break;
    case 256: run_beam<256>(bp, pl.sorted, B, smem.data()); break;
    default: fprintf(stderr, "emu: NT %d\n", NT); return CTCDEC_E_INVALID;
  }
  std::vector<unsigned char> fsmem(finalize_smem_bytes(K) + 64);
  for (int b = 0; b < B; ++b) finalize_cta_run<256>(bp, b, fsmem.data());
  for (int b = 0; b < B; ++b)
    for (int q = 0; q < n_results[b] && q < K; ++q) {
      const size_t r = (size_t)b * K + q;
      const LmSlot &sl = slots[slot_of[b]];
      scores[r] = ngram_readout_row(sl.ngram, sl.front, tokens + r * T, lens[r], scores[r], sl.lm_alpha, sl.beta);
    }
  return 0;
}

}  // extern "C"

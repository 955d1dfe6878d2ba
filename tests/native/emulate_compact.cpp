// TEST INFRASTRUCTURE ONLY -- streaming decodes in the single-threaded CPU emulation of the CTA programs with the arena
// compaction (compact_program.cuh) run between chunks.  Each stream owns its arrays as a streaming state does
// (ctc_api.cu StreamState: arena, LM terms with the histories behind them, dictionary states, rows of a
// character-based model; capacity grown as grow_arenas grows it), so the beam program reads them through the
// per-stream pointer tables.  Builds on emulate_cta.cpp; tests/test_stream_compact_emulation.py compiles this file into
// tests/native/_build/.  The product never builds or loads it.
#include "emulate_cta.cpp"
#include "../../ctcdecode_b200/csrc/compact_program.cuh"

namespace {

struct EmuStream {
  std::vector<Node> arena;
  std::vector<float> lm, row;
  std::vector<int> dst, state;
  long long cap = 0, base = 1, since = 0;  // node accounting: base + K x (frames since the last compaction)
};

// new arrays of capacity `cap` holding the first `used` nodes of the old ones
void resize_stream(EmuStream &s, long long cap, long long used, int H, int V, bool lm, bool chr) {
  EmuStream n;
  n.arena.assign((size_t)cap, Node{});
  std::copy(s.arena.begin(), s.arena.begin() + used, n.arena.begin());
  if (lm) {
    n.lm.assign((size_t)cap * (1 + H), 0.f);
    n.dst.assign((size_t)cap, 0);
    std::copy(s.lm.begin(), s.lm.begin() + used, n.lm.begin());
    std::copy(s.lm.begin() + s.cap, s.lm.begin() + s.cap + used * H, n.lm.begin() + cap);
    std::copy(s.dst.begin(), s.dst.begin() + used, n.dst.begin());
    if (chr) {
      n.row.assign((size_t)cap * V, 0.f);
      std::copy(s.row.begin(), s.row.begin() + used * V, n.row.begin());
    }
  }
  s.arena.swap(n.arena); s.lm.swap(n.lm); s.dst.swap(n.dst); s.row.swap(n.row);
  s.cap = cap;
}

}  // namespace

extern "C" {

// chunks[0 .. n_chunks): frames of each chunk (every stream gets min(its remaining frames, chunk)); the frames beyond
// their sum are not decoded.  compact_every > 0: compaction after every compact_every-th chunk (also after the last,
// before the read-out), 0: never.  slack: frames of room the capacity rule leaves (ctc_api.cu uses 256).
// lm_path: an ARPA model for the device n-gram scorer, or NULL.  After every chunk the committed prefix of each stream
// goes to committed[ci][b] and com_tok / com_ts[ci][b][0 .. T).
// dump (dump_cap ints): per compaction and stream, [ci, b, n, M, A, kept] then the old arena's parents [n] and chars
// [n], the members' nodes [M], the occupied dead anchors' nodes [A], the new arena's parents, chars and jumps [kept]
// each; a final -1.  Returns 0, a CTCDEC_E_* code, or -2 when the dump overflows.
int emu_decode_stream_compact(const float *probs, const int *seq_lens, int B, int T, int V, int K, double cutoff_prob,
                              int cutoff_top_n, int blank, int log_input, int NT, const int *chunks, int n_chunks,
                              int compact_every, int slack, const char *lm_path, double alpha, double beta,
                              const char *const *labels, int *tokens, int *timesteps, float *scores, int *lens,
                              int *n_results, int *flags, int *committed, int *com_tok, int *com_ts, int *dump,
                              long long dump_cap) {
  ctcdec_config cfg;
  cfg.vocab_size = V; cfg.beam_size = K; cfg.blank_id = blank; cfg.log_input = log_input;
  cfg.cutoff_top_n = cutoff_top_n; cfg.cutoff_prob = cutoff_prob;
  const bool lm = lm_path != nullptr;
  Plan pl;
  char msg[256];
  int rc = make_plan_core(&cfg, B, T, &pl, msg, sizeof(msg), lm);
  if (rc) { fprintf(stderr, "emu: %s\n", msg); return rc; }
  if (NT <= 0) NT = pl.NT;
  pl.NT = NT;
  pl.L = make_layout(K, V, pl.NP, pl.F, pl.sorted, NT, lm);
  std::vector<float> lp((size_t)B * T * pl.NP + 8, 0.f);
  std::vector<uint16_t> idx(pl.sorted ? (size_t)B * T * pl.NP + 8 : 8, 0);
  std::vector<unsigned char> smem(pl.L.total + 64), csmem(compact_smem_bytes(K, 256) + 64);
  for (int b = 0; b < B; ++b) flags[b] = 0;
  prune_rows(cfg, pl, probs, seq_lens, B, T, lp.data(), idx.data(), flags);

  BeamParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.V = V; bp.NP = pl.NP; bp.K = K; bp.blank = blank; bp.tile_frames = pl.F; bp.L = pl.L;
  bp.out_tokens = tokens; bp.out_timesteps = timesteps; bp.out_scores = scores; bp.out_lens = lens;
  bp.n_results = n_results; bp.out_T = T; bp.flags = flags;
  g_emu_order = getenv("CTC_EMU_ORDER") ? atoi(getenv("CTC_EMU_ORDER")) : 0;  // test knob: order of the emulated threads

  std::shared_ptr<NgramModel> m;
  HostScorer sc;
  int H = 0;
  if (lm) {
    m = std::make_shared<NgramModel>();
    for (int i = 0; i < V; ++i) {
      m->labels.emplace_back(labels[i]);
      if (m->labels.back() == " ") m->space_id = i;
    }
    const std::string why = load_arpa(lm_path, *m);
    if (!why.empty()) { fprintf(stderr, "emu: %s\n", why.c_str()); return CTCDEC_E_UNSUPPORTED; }
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
    H = sc.max_order - 1;
    bp.dict_next = sc.dict.packed.data(); bp.dict_mask = sc.dict.mask.data(); bp.dict_wc = sc.dict.wc;
    bp.dict_start = sc.dict.start;
    bp.space_id = sc.space_id; bp.beta = beta;
    bp.lm_char = sc.is_character_based;
    bp.lm_dev = 1; bp.lm_alpha = alpha; bp.ngram = m->view();
    bp.word_of_state = sc.word_of_state.data(); bp.label_word = sc.label_word.data();
    bp.lm_hist_n = H;
  }
  const bool chr = lm && sc.is_character_based;

  std::vector<EmuStream> S(B);
  std::vector<Node *> arena_ptrs(B);
  std::vector<int *> state_ptrs(B), dst_ptrs(B);
  std::vector<float *> lm_ptrs(B), row_ptrs(B);
  std::vector<int> caps(B);
  for (int b = 0; b < B; ++b) {
    S[b].state.assign((size_t)state_ints(K), 0);
    resize_stream(S[b], 1 + (long long)K * slack, 0, H, V, lm, chr);
  }
  bp.arena_ptrs = arena_ptrs.data(); bp.state_ptrs = state_ptrs.data(); bp.arena_caps = caps.data();
  if (lm) { bp.lm_arena_ptrs = lm_ptrs.data(); bp.dstate_ptrs = dst_ptrs.data(); bp.lm_row_ptrs = row_ptrs.data(); }
  auto tables = [&]() {
    for (int b = 0; b < B; ++b) {
      arena_ptrs[b] = S[b].arena.data(); state_ptrs[b] = S[b].state.data(); caps[b] = (int)S[b].cap;
      lm_ptrs[b] = lm ? S[b].lm.data() : nullptr; dst_ptrs[b] = lm ? S[b].dst.data() : nullptr;
      row_ptrs[b] = chr ? S[b].row.data() : nullptr;
    }
  };

  long long dpos = 0;
  auto put = [&](int v) { if (dpos < dump_cap) dump[dpos] = v; ++dpos; };
  std::vector<int> map;
  auto compact = [&](int ci) {
    for (int b = 0; b < B; ++b) {
      EmuStream &s = S[b];
      const int *st = s.state.data();
      const int n = st[1], M = st[0], KP2 = 2 * kp_of(K);
      const int *an = st + kStateHeader + kSlotArrays * K;
      std::vector<int> anch, mem(st + kStateHeader, st + kStateHeader + M);
      for (int a = 0; a < KP2; ++a) if (an[2 * KP2 + a] >= 0) anch.push_back(an[a]);
      map.assign((size_t)n, 7);
      int kept = -1;
      compact_mark_cta_run<256>(s.arena.data(), st, K, (int)s.cap, map.data(), &kept, csmem.data());
      EmuStream t;
      const long long cap_new = std::max<long long>(1 + (long long)K * slack, kept + (long long)K * slack);
      resize_stream(t, cap_new, 0, H, V, lm, chr);
      CompactJob j;
      j.arena = s.arena.data(); j.arena_new = t.arena.data(); j.state = s.state.data(); j.map = map.data();
      j.lm = lm ? s.lm.data() : nullptr; j.lm_new = lm ? t.lm.data() : nullptr;
      j.dst = lm ? s.dst.data() : nullptr; j.dst_new = lm ? t.dst.data() : nullptr;
      j.row = chr ? s.row.data() : nullptr; j.row_new = chr ? t.row.data() : nullptr;
      j.K = K; j.cap = (int)s.cap; j.cap_new = (int)cap_new; j.H = H; j.V = V; j.kept = kept;
      compact_gather_cta_run<256>(j);
      put(ci); put(b); put(n); put(M); put((int)anch.size()); put(s.state[1]);
      for (int i = 0; i < n; ++i) put(s.arena[i].parent);
      for (int i = 0; i < n; ++i) put(s.arena[i].chr);
      for (int v : mem) put(v);
      for (int a : anch) put(a);
      for (int i = 0; i < kept; ++i) put(t.arena[i].parent);
      for (int i = 0; i < kept; ++i) put(t.arena[i].chr);
      for (int i = 0; i < kept; ++i) put(t.arena[i].jump);
      s.arena.swap(t.arena); s.lm.swap(t.lm); s.dst.swap(t.dst); s.row.swap(t.row);
      s.cap = cap_new; s.base = kept; s.since = 0;
    }
  };

  std::vector<int> chunk_lens(B);
  int t0 = 0;
  const int TT = std::max(T, 1);
  for (int ci = 0; ci < n_chunks; ++ci) {
    const int tc = std::max(0, std::min(chunks[ci], T - t0));
    bp.lp = lp.data() + (size_t)t0 * pl.NP;
    bp.idx = pl.sorted ? idx.data() + (size_t)t0 * pl.NP : nullptr;
    bp.T = T;
    for (int b = 0; b < B; ++b) {
      int len = seq_lens ? seq_lens[b] : T;
      len = std::max(0, std::min(len, T));
      chunk_lens[b] = std::max(0, std::min(len - t0, tc));
      EmuStream &s = S[b];
      // grow_arenas: room for base + K x (frames since the last compaction, this chunk included)
      const long long need = s.base + (long long)K * (s.since + chunk_lens[b]);
      if (need > s.cap) resize_stream(s, std::max(need, 2 * s.cap), std::min(s.cap, s.base + (long long)K * s.since), H, V,
                                      lm, chr);
    }
    tables();
    bp.seq_lens = chunk_lens.data();
    bp.fresh = ci == 0 ? 1 : 0;
    switch (NT) {
      case 128: run_beam<128>(bp, pl.sorted, B, smem.data()); break;
      case 256: run_beam<256>(bp, pl.sorted, B, smem.data()); break;
      case 512: run_beam<512>(bp, pl.sorted, B, smem.data()); break;
      default: return CTCDEC_E_UNSUPPORTED;
    }
    for (int b = 0; b < B; ++b) S[b].since += chunk_lens[b];
    t0 += tc;
    if (compact_every > 0 && (ci + 1) % compact_every == 0) {
      compact(ci);
      tables();
    }
    for (int b = 0; b < B; ++b) {
      const size_t row = ((size_t)ci * B + b) * TT;
      committed_cta_run<128>(S[b].arena.data(), S[b].state.data(), K, 0, &committed[(size_t)ci * B + b], com_tok + row,
                             com_ts + row, T, csmem.data());
    }
  }
  put(-1);
  if (dpos > dump_cap) return -2;
  std::vector<unsigned char> fsmem(finalize_smem_bytes(K) + 64);
  for (int b = 0; b < B; ++b) finalize_cta_run<256>(bp, b, fsmem.data());
  if (lm) lm_rescore_batch(sc, B, K, T, n_results, tokens, lens, scores);
  return 0;
}

}  // extern "C"

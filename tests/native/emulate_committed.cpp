// TEST INFRASTRUCTURE ONLY -- the committed-prefix program (committed_cta_run, beam_program.cuh) in the single-threaded
// CPU emulation of the CTA programs, run after every chunk of a streaming decode.  Builds on emulate_cta.cpp (its host
// mirror of the prune scan and its beam launcher); tests/test_committed_emulation.py compiles this file into
// tests/native/_build/.  The product never builds or loads it.
#include "emulate_cta.cpp"

extern "C" {

// The streaming decode of emu_decode_batch (chunk > 0, the same chunk loop) with committed_cta_run run after every
// chunk, three times per stream:
//   committed [n_chunks][B]              the LCA depth (-1000000 if the three calls below disagree on it);
//   full_tok / full_ts [n_chunks][B][T]  the whole committed prefix (since = 0);
//   acc_tok / acc_ts [n_chunks][B][T]    the deltas of calls with since = the previous call's depth, appended;
//   bad_tok / bad_ts [n_chunks][B][T]    a call with since = frames consumed + 1 (never a valid depth: read from 0).
// Unwritten entries stay as the caller filled them.  tokens ... flags: the final read-out, as emu_decode_batch.
int emu_decode_stream_committed(const float *probs, const int *seq_lens, int B, int T, int V, int K, double cutoff_prob,
                                int cutoff_top_n, int blank, int log_input, int NT, int chunk, int *tokens,
                                int *timesteps, float *scores, int *lens, int *n_results, int *flags, int *committed,
                                int *full_tok, int *full_ts, int *acc_tok, int *acc_ts, int *bad_tok, int *bad_ts) {
  if (chunk <= 0) return CTCDEC_E_INVALID;
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
  std::vector<float> lp((size_t)B * T * pl.NP + 8, 0.f);
  std::vector<uint16_t> idx(pl.sorted ? (size_t)B * T * pl.NP + 8 : 8, 0);
  std::vector<Node> arena((size_t)B * pl.arena_stride);
  std::vector<int> state((size_t)B * pl.state_stride, 0);
  std::vector<unsigned char> smem(pl.L.total + 64), csmem(committed_smem_bytes(K) + 64);
  for (int b = 0; b < B; ++b) flags[b] = 0;
  prune_rows(cfg, pl, probs, seq_lens, B, T, lp.data(), idx.data(), flags);

  BeamParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.V = V; bp.NP = pl.NP; bp.K = K; bp.blank = blank; bp.tile_frames = pl.F; bp.L = pl.L;
  bp.arena = arena.data(); bp.arena_stride = pl.arena_stride; bp.state = state.data();
  bp.state_stride = pl.state_stride; bp.arena_cap = (int)pl.arena_stride;
  bp.out_tokens = tokens; bp.out_timesteps = timesteps; bp.out_scores = scores; bp.out_lens = lens;
  bp.n_results = n_results; bp.out_T = T; bp.flags = flags;
  g_emu_order = getenv("CTC_EMU_ORDER") ? atoi(getenv("CTC_EMU_ORDER")) : 0;  // test knob: order of the emulated threads

  const int TT = std::max(T, 1);
  std::vector<int> chunk_lens(B), prev(B, 0), d_tok(TT), d_ts(TT);
  bool first = true;
  for (int t0 = 0, ci = 0; t0 < T || first; t0 += chunk, ++ci) {
    const int tc = std::min(chunk, T - t0);
    bp.lp = lp.data() + (size_t)t0 * pl.NP;
    bp.idx = pl.sorted ? idx.data() + (size_t)t0 * pl.NP : nullptr;
    bp.T = T;
    for (int b = 0; b < B; ++b) {
      int len = seq_lens ? seq_lens[b] : T;
      len = std::max(0, std::min(len, T));
      chunk_lens[b] = std::max(0, std::min(len - t0, tc));
    }
    bp.seq_lens = chunk_lens.data();
    bp.fresh = first ? 1 : 0;
    switch (NT) {
      case 128: run_beam<128>(bp, pl.sorted, B, smem.data()); break;
      case 256: run_beam<256>(bp, pl.sorted, B, smem.data()); break;
      default: return CTCDEC_E_UNSUPPORTED;
    }
    first = false;
    for (int b = 0; b < B; ++b) {
      const Node *nodes = bp.arena + (long long)b * bp.arena_stride;
      const int *st = bp.state + (long long)b * bp.state_stride;
      const size_t row = ((size_t)ci * B + b) * TT;
      int D = 0, D2 = 0, D3 = 0;
      committed_cta_run<128>(nodes, st, K, 0, &D, full_tok + row, full_ts + row, T, csmem.data());
      // deltas: since = the previous depth, written to scratch and appended behind the previous accumulated prefix
      committed_cta_run<128>(nodes, st, K, prev[b], &D2, d_tok.data(), d_ts.data(), T, csmem.data());
      if (ci > 0) {
        memcpy(acc_tok + row, acc_tok + row - (size_t)B * TT, (size_t)TT * 4);
        memcpy(acc_ts + row, acc_ts + row - (size_t)B * TT, (size_t)TT * 4);
      }
      const int s0 = prev[b] <= D2 ? prev[b] : 0;
      for (int i = 0; i < D2 - s0; ++i) { acc_tok[row + s0 + i] = d_tok[i]; acc_ts[row + s0 + i] = d_ts[i]; }
      int len = seq_lens ? seq_lens[b] : T;
      len = std::max(0, std::min(len, T));
      const int consumed = std::min(len, t0 + tc);
      committed_cta_run<128>(nodes, st, K, consumed + 1, &D3, bad_tok + row, bad_ts + row, T, csmem.data());
      committed[(size_t)ci * B + b] = (D == D2 && D == D3) ? D : -1000000;
      prev[b] = D2;
    }
    if (T == 0) break;
  }
  std::vector<unsigned char> fsmem(finalize_smem_bytes(K) + 64);
  for (int b = 0; b < B; ++b) finalize_cta_run<256>(bp, b, fsmem.data());
  return 0;
}

}  // extern "C"

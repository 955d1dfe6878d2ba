// TEST INFRASTRUCTURE ONLY -- the per-row read-out rescoring of the ARPA scorer (ngram_readout_row in ngram_lm.h, the
// function the library's read-out kernel runs) compiled for the CPU, over a model loaded as ctcdec_scorer_create_arpa
// loads it.  tests/test_lm_readout.py compiles this file into tests/native/_build/.  The product never builds or loads it.
#include <memory>
#include <string>

#include "../../ctcdecode_b200/csrc/ngram_arpa.h"

extern "C" {

// Rescores rows p < min(n_results[b], K) of scores [B, K] in place from tokens [B, K, row_stride] / lens [B, K].
// Returns 0, or -2 when the model is refused (the reason on stderr).
int emu_readout_rows(const char *path, const char *const *labels, int V, double alpha, double beta, const int *tokens,
                     const int *lens, const int *n_results, float *scores, int B, int K, int row_stride) {
  ctc::NgramModel m;
  for (int i = 0; i < V; ++i) {
    m.labels.emplace_back(labels[i]);
    if (m.labels.back() == " ") m.space_id = i;
  }
  const std::string why = ctc::load_arpa(path, m);
  if (!why.empty()) { fprintf(stderr, "emu: %s\n", why.c_str()); return -2; }
  const ctc::NgramView v = m.view();
  const ctc::NgramFront f = m.front();
  for (int b = 0; b < B; ++b)
    for (int p = 0; p < n_results[b] && p < K; ++p) {
      const size_t r = (size_t)b * K + p;
      scores[r] = ctc::ngram_readout_row(v, f, tokens + r * row_stride, lens[r], scores[r], alpha, beta);
    }
  return 0;
}

}  // extern "C"

// N-gram language model read from an ARPA text file: the tables, and the one lookup that reproduces the reference's
// Scorer::get_log_cond_prob (scorer.cpp:74-93) over KenLM's probing model bit for bit.  The tables and the lookup
// compile for the host and for the device (ngram_cond_ids takes plain pointers: a view of host vectors or of their
// HBM copies); the ARPA loader and the label-to-word front end are host code.
//
// What is reproduced, from KenLM's query path (lm/model.cc FullScore / ResumeScore, lm/read_arpa.cc):
//   * word ids: 0 is <unk> (also "<UNK>"), then the unigrams in file order; an unknown string is 0;
//   * every stored log10 probability has its sign bit set (KenLM's Prob() does so; 0 becomes -0.0);
//   * a backoff of 0 (or none) is stored as -0.0, "no n-gram extends this one", and turned into +0.0 when the n-gram is
//     the context of a longer one: the sign decides how long the state's history is, as in KenLM;
//   * a word is scored in the state left by the previous one: the longest matching n-gram's probability, then the
//     state's context backoffs from the matched length up, added in float in that order.
// The tables hold the file's n-grams plus the suffix entries KenLM fills in on load (ngram_arpa.h), so "not found"
// means the same thing here as in KenLM.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define CTC_NG_HD __host__ __device__ __forceinline__
#else
#define CTC_NG_HD static inline
#endif

namespace ctc {

constexpr int kNgramMaxOrder = 6;            // KENLM_MAX_ORDER of the reference build
constexpr double kNgramOovScore = -1000.0;   // reference scorer.h OOV_SCORE
constexpr float kNgramFltLogE = 0.4342944819f;  // reference decoder_utils.h NUM_FLT_LOGE (a float constant)

// One n-gram of order >= 2 in an open-addressing table; w[0] < 0 marks an empty slot.
struct NgramEntry {
  int32_t w[kNgramMaxOrder];  // word ids in text order, unused tail -1
  float prob, backoff;
};

// Read-only view of the tables: host vectors or their device copies.
struct NgramView {
  int order = 0;
  int vocab = 0;
  int bos = 0;                         // the id of "<s>"
  const float *uni_prob = nullptr;     // [vocab]
  const float *uni_backoff = nullptr;  // [vocab]
  const NgramEntry *table[kNgramMaxOrder] = {};  // [n - 1]: order n >= 2, capacity mask[n - 1] + 1 (a power of two)
  uint32_t mask[kNgramMaxOrder] = {};
};

struct NgramState {
  int len;
  int32_t words[kNgramMaxOrder - 1];  // most recent first
  float backoff[kNgramMaxOrder - 1];  // backoff[i]: of the n-gram words[i] .. words[0]
};

CTC_NG_HD uint32_t ngram_hash(const int32_t *w, int n) {
  uint64_t h = 0x9e3779b97f4a7c15ull * (uint64_t)(n + 1);
  for (int i = 0; i < n; ++i) {
    h ^= (uint64_t)(uint32_t)w[i] + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
    h *= 0xff51afd7ed558ccdull;
  }
  return (uint32_t)(h ^ (h >> 29));
}

// The entry of the n-gram w[0..n) (text order), or null.  The full key is compared.
CTC_NG_HD const NgramEntry *ngram_find(const NgramView &m, const int32_t *w, int n) {
  const NgramEntry *t = m.table[n - 1];
  const uint32_t mask = m.mask[n - 1];
  for (uint32_t s = ngram_hash(w, n) & mask;; s = (s + 1) & mask) {
    const NgramEntry &e = t[s];
    if (e.w[0] < 0) return nullptr;
    bool eq = true;
    for (int i = 0; i < n; ++i) eq = eq && e.w[i] == w[i];
    if (eq) return &e;
  }
}

CTC_NG_HD bool ngram_has_extension(float backoff) {
  uint32_t u;
  memcpy(&u, &backoff, 4);
  return u != 0x80000000u;  // anything but -0.0
}

// KenLM GenericModel::FullScore(in, w, out).prob: log10 p(w | in's history).
CTC_NG_HD float ngram_score(const NgramView &m, const NgramState &in, int32_t w, NgramState &out) {
  float prob = m.uni_prob[w];
  out.backoff[0] = m.uni_backoff[w];
  out.len = ngram_has_extension(out.backoff[0]) ? 1 : 0;
  out.words[0] = w;
  int matched = 1;
  int32_t key[kNgramMaxOrder];
  for (int j = 0; j < in.len; ++j) {  // the n-gram of the last j + 1 history words and w
    const int n = j + 2;
    for (int i = 0; i <= j; ++i) key[i] = in.words[j - i];
    key[j + 1] = w;
    const NgramEntry *e = ngram_find(m, key, n);
    if (!e) break;
    prob = e->prob;
    matched = n;
    if (n < m.order) {
      out.backoff[j + 1] = e->backoff;
      if (ngram_has_extension(e->backoff)) out.len = n;
    }
  }
  for (int i = 1; i < out.len; ++i) out.words[i] = in.words[i - 1];
  for (int i = matched - 1; i < in.len; ++i) prob += in.backoff[i];
  return prob;
}

// Scorer::get_log_cond_prob over word ids: every word scored from KenLM's null context on (the "<s>" padding words are
// scored as words); any id 0 gives OOV_SCORE.  The natural-log result of the last word.
CTC_NG_HD double ngram_cond_ids(const NgramView &m, const int32_t *ids, int n) {
  NgramState a, b;
  a.len = 0;
  float p = 0.0f;
  for (int i = 0; i < n; ++i) {
    if (ids[i] == 0) return kNgramOovScore;
    NgramState &in = (i & 1) ? b : a;
    NgramState &out = (i & 1) ? a : b;
    p = ngram_score(m, in, ids[i], out);
  }
  return (double)p / (double)kNgramFltLogE;
}

}  // namespace ctc

#undef CTC_NG_HD

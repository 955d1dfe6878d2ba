// Host side of the n-gram scorer: the model's tables (NgramModel), the ARPA text loader that fills them, and the two
// scorer hooks (ctcdec_scorer_hooks) computed from them exactly as the reference's Scorer computes them over KenLM.
// KenLM binary files are read by ngram_kenlm.h, whose load_ngram_file takes either form.
//
// The ARPA loader accepts only what it can reproduce exactly; everything else is refused with the reason:
//   * a KenLM binary file (load_ngram_file sends those to ngram_kenlm.h), or anything that is not ARPA text ("\data\",
//     counts, "\N-grams:" sections, "\end\");
//   * order 1 (KenLM needs at least bigrams) or above kNgramMaxOrder;
//   * counts that disagree with the sections, a malformed line, a duplicate n-gram or unigram;
//   * an n-gram word that is not a unigram, a missing <s> or </s> (KenLM refuses all of these too);
//   * an n-gram whose context (all words but the last) is not in the model;
//   * a positive log-prob, a NaN or +inf log-prob, a non-finite backoff, a non-zero backoff on a highest-order n-gram.
// A log-prob of -inf is read as it is, as KenLM does.  An n-gram whose suffix n-gram (all words but the first) is missing,
// as in models pruned by SRILM, gets the entries KenLM fills in on load, computed the same way (link_lower below).
#pragma once
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <unordered_map>
#include <vector>

#include "ngram_lm.h"

namespace ctc {

struct NgramModel {
  int order = 0;
  std::vector<std::string> vocabulary;  // by word id, as KenLM's EnumerateVocab reports it: "<unk>" first
  std::unordered_map<std::string, int32_t> word_id;
  std::vector<float> uni_prob, uni_backoff;
  std::vector<NgramEntry> tables[kNgramMaxOrder];
  // a KenLM probing file (layout kNgramKenlmProbing): its tables of orders 2..N byte for byte, instead of `tables`
  int layout = kNgramTables;
  std::vector<uint64_t> probing[kNgramMaxOrder];
  uint32_t buckets[kNgramMaxOrder] = {};
  // a KenLM trie file (layout kNgramKenlmTrie): its search region byte for byte, zero-padded, and where each order is
  std::vector<uint64_t> trie_bits;
  std::vector<NgramTrieOrder> trie_orders;
  // the decoder's labels, for the label-id hooks (reference Scorer::set_char_map, scorer.cpp:148-161)
  std::vector<std::string> labels;
  int space_id = -1;  // the " " label, -1 if none (reference SPACE_ID_)
  int is_character_based = 1;
  // the label-to-word front end's tables (ngram_build_front; NgramFront)
  std::vector<unsigned char> label_bytes, word_bytes;
  std::vector<int32_t> label_off;
  std::vector<NgramWordSlot> words;
  int32_t bos_id = 0, eos_id = 0;

  NgramView view() const {
    NgramView v;
    v.order = order;
    v.vocab = (int)uni_prob.size();
    v.bos = id_of("<s>");
    v.uni_prob = uni_prob.data();
    v.uni_backoff = uni_backoff.data();
    v.layout = layout;
    if (layout == kNgramKenlmTrie) {
      v.trie.bits = trie_bits.data();
      v.trie.orders = trie_orders.data();
      return v;
    }
    for (int n = 2; n <= order; ++n) {
      if (layout == kNgramKenlmProbing) {
        v.probe[n - 1] = reinterpret_cast<const uint32_t *>(probing[n - 1].data());
        v.buckets[n - 1] = buckets[n - 1];
      } else {
        v.table[n - 1] = tables[n - 1].data();
        v.mask[n - 1] = (uint32_t)tables[n - 1].size() - 1;
      }
    }
    return v;
  }
  NgramFront front() const {
    NgramFront f;
    f.space_id = space_id;
    f.is_character_based = is_character_based;
    f.bos = bos_id;
    f.eos = eos_id;
    f.label_bytes = label_bytes.data();
    f.label_off = label_off.data();
    f.word_bytes = word_bytes.data();
    f.words = words.data();
    f.word_mask = (uint32_t)words.size() - 1;
    return f;
  }
  int32_t id_of(const std::string &w) const {
    auto it = word_id.find(w);
    return it == word_id.end() ? 0 : it->second;
  }
  // The bytes of n-gram data a device holds: the unigrams and the data of orders >= 2 (the trie's order descriptors,
  // a few hundred bytes, aside).
  size_t table_bytes() const {
    size_t bytes = (uni_prob.size() + uni_backoff.size()) * 4 + trie_bits.size() * 8;
    for (int n = 2; n <= order; ++n) bytes += tables[n - 1].size() * sizeof(NgramEntry) + probing[n - 1].size() * 8;
    return bytes;
  }
};

// The front end's tables of a loaded model with its labels set: the labels' bytes, and every unigram but <unk> (id 0,
// which is also what a word missing from the table gets) in an open-addressing table keyed by its spelling.
static inline void ngram_build_front(NgramModel &m) {
  m.bos_id = m.id_of("<s>");
  m.eos_id = m.id_of("</s>");
  m.label_bytes.clear();
  m.label_off.assign(1, 0);
  for (const std::string &l : m.labels) {
    m.label_bytes.insert(m.label_bytes.end(), l.begin(), l.end());
    m.label_off.push_back((int32_t)m.label_bytes.size());
  }
  size_t cap = 2;
  while (cap < 2 * m.vocabulary.size()) cap <<= 1;
  NgramWordSlot empty;
  empty.hash = empty.off = 0;
  empty.len = -1;
  empty.id = 0;
  m.words.assign(cap, empty);
  m.word_bytes.clear();
  const uint32_t mask = (uint32_t)cap - 1;
  for (size_t id = 1; id < m.vocabulary.size(); ++id) {
    const std::string &w = m.vocabulary[id];
    NgramWordSlot e;
    e.hash = kNgramFnvBasis;
    for (char c : w) e.hash = ngram_fnv(e.hash, (unsigned char)c);
    e.off = (uint32_t)m.word_bytes.size();
    e.len = (int32_t)w.size();
    e.id = (int32_t)id;
    m.word_bytes.insert(m.word_bytes.end(), w.begin(), w.end());
    uint32_t s = e.hash & mask;
    while (m.words[s].len >= 0) s = (s + 1) & mask;
    m.words[s] = e;
  }
}

// reference Scorer::load_lm (scorer.cpp:61-71): word-based as soon as one word other than <unk> / <s> / </s> is longer
// than one UTF-8 character
static inline int ngram_character_based(const std::vector<std::string> &vocabulary) {
  for (const std::string &w : vocabulary) {
    if (w == "<unk>" || w == "<s>" || w == "</s>") continue;
    int chars = 0;
    for (char c : w) chars += ((c & 0xc0) != 0x80);
    if (chars > 1) return 0;
  }
  return 1;
}

namespace arpa_detail {

static inline bool blank_line(const std::string &s) {
  for (char c : s)
    if (!isspace((unsigned char)c)) return false;
  return true;
}

// fields separated by ' ' / '\t' (KenLM's kARPASpaces, with '\n' already cut)
static inline void split_fields(const std::string &s, std::vector<std::string> &out) {
  out.clear();
  size_t i = 0;
  while (i < s.size()) {
    while (i < s.size() && (s[i] == ' ' || s[i] == '\t')) ++i;
    size_t j = i;
    while (j < s.size() && s[j] != ' ' && s[j] != '\t') ++j;
    if (j > i) out.emplace_back(s, i, j - i);
    i = j;
  }
}

static inline bool parse_float(const std::string &s, float *v) {
  char *end = nullptr;
  *v = strtof(s.c_str(), &end);
  return end != s.c_str() && *end == 0;
}

static inline void set_sign(float &f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  u |= 0x80000000u;
  memcpy(&f, &u, 4);
}

}  // namespace arpa_detail

// Fills the open-addressing table of order n from its entries (capacity: a power of two >= 2 x count).
static inline void ngram_build_table(const std::vector<NgramEntry> &entries, int n, std::vector<NgramEntry> &table) {
  size_t cap = 2;
  while (cap < 2 * entries.size()) cap <<= 1;
  NgramEntry empty;
  for (int i = 0; i < kNgramMaxOrder; ++i) empty.w[i] = -1;
  empty.prob = empty.backoff = 0.0f;
  table.assign(cap, empty);
  const uint32_t mask = (uint32_t)cap - 1;
  for (const NgramEntry &e : entries) {
    uint32_t s = ngram_hash(e.w, n) & mask;
    while (table[s].w[0] >= 0) s = (s + 1) & mask;
    table[s] = e;
  }
}

// Returns "" on success, else the reason the file is refused.
static inline std::string load_arpa(const char *path, NgramModel &m) {
  using namespace arpa_detail;
  FILE *f = fopen(path, "rb");
  if (!f) return std::string("cannot open the file");
  std::string line;
  bool eof = false;
  auto next_line = [&]() -> bool {
    line.clear();
    int c;
    while ((c = fgetc(f)) != EOF && c != '\n') line.push_back((char)c);
    if (c == EOF && line.empty()) { eof = true; return false; }
    return true;
  };
  struct Closer { FILE *f; ~Closer() { fclose(f); } } closer{f};

  static const char kBinaryMagic[] = "mmap lm http://kheafield.com/code";
  {
    char head[sizeof(kBinaryMagic)] = {0};
    const size_t got = fread(head, 1, sizeof(kBinaryMagic) - 1, f);
    if (got == sizeof(kBinaryMagic) - 1 && memcmp(head, kBinaryMagic, got) == 0)
      return "a KenLM binary file: only ARPA text is supported";
    rewind(f);
  }
  do {
    if (!next_line()) return "not an ARPA text file: no \\data\\ line";
  } while (blank_line(line) || line[0] == '#');
  if (line != "\\data\\") return "not an ARPA text file: the first line is not \\data\\";

  std::vector<long long> counts;
  while (next_line() && !blank_line(line)) {
    int n = 0;
    long long c = -1;
    char tail = 0;
    if (sscanf(line.c_str(), "ngram %d=%lld%c", &n, &c, &tail) != 2 || c < 0)
      return "bad count line \"" + line + "\"";
    if (n != (int)counts.size() + 1) return "count lines are not consecutive from 1: \"" + line + "\"";
    counts.push_back(c);
  }
  const int order = (int)counts.size();
  if (order < 2) return "order " + std::to_string(order) + ": at least a bigram model is needed";
  if (order > kNgramMaxOrder)
    return "order " + std::to_string(order) + " is above " + std::to_string(kNgramMaxOrder);
  m.order = order;

  std::vector<std::string> fld;
  std::vector<NgramEntry> entries[kNgramMaxOrder];
  // per order: key -> index into entries (text-order ids as bytes)
  std::unordered_map<std::string, size_t> index[kNgramMaxOrder];
  auto key_of = [](const int32_t *w, int n) { return std::string(reinterpret_cast<const char *>(w), (size_t)n * 4); };
  bool saw_unk = false;
  m.vocabulary.assign(1, "<unk>");
  m.uni_prob.assign(1, -100.0f);  // KenLM's stand-in for a missing <unk> (never scored: id 0 is OOV)
  m.uni_backoff.assign(1, 0.0f);

  // What KenLM's hashed search does as it reads each n-gram w[0..n) of order n >= 2, in file order
  // (lm/search_hashed.cc FindLower / AdjustLower / ActivateLowerMiddle):
  //   * a missing suffix n-gram w[n-L..n) (L = n-1 down to the first one present) is filled in with the probability a
  //     query would give it: the longest present suffix's, plus the backoffs of the contexts in between, in float;
  //   * every context used on the way, and the n-gram's own context w[0..n-1), is marked extended (-0.0 -> +0.0);
  //     a missing own context is an error in KenLM (and here).
  auto find = [&](const int32_t *w, int len) -> NgramEntry * {
    auto it = index[len - 1].find(key_of(w, len));
    return it == index[len - 1].end() ? nullptr : &entries[len - 1][it->second];
  };
  auto mark_extended = [](float &backoff) { if (!ngram_has_extension(backoff)) backoff = 0.0f; };
  auto link_lower = [&](const int32_t *w, int n) -> bool {
    std::vector<int> blanks;  // lengths of the suffixes filled in, longest first
    int basis = 1;
    for (int len = n - 1; len >= 2; --len) {
      if (find(w + n - len, len)) { basis = len; break; }
      NgramEntry b;
      for (int k = 0; k < kNgramMaxOrder; ++k) b.w[k] = k < len ? w[n - len + k] : -1;
      b.prob = 0.0f;
      b.backoff = -0.0f;
      index[len - 1].emplace(key_of(b.w, len), entries[len - 1].size());
      entries[len - 1].push_back(b);
      blanks.push_back(len);
    }
    if (!blanks.empty()) {
      float prob = basis == 1 ? m.uni_prob[w[n - 1]] : find(w + n - basis, basis)->prob;
      set_sign(prob);
      for (int len = basis + 1; len <= n - 1; ++len) {  // the suffix of length len: context w[n-len .. n-1)
        float *bo = len == 2 ? &m.uni_backoff[w[n - 2]] : nullptr;
        if (len > 2)
          if (NgramEntry *c = find(w + n - len, len - 1)) bo = &c->backoff;
        if (bo) { mark_extended(*bo); prob += *bo; }
        float stored = prob;
        set_sign(stored);  // (KenLM's Prob() sets the sign bit on every read)
        find(w + n - len, len)->prob = stored;
      }
    }
    if (n == 2) {
      mark_extended(m.uni_backoff[w[0]]);
      return true;
    }
    NgramEntry *ctx = find(w, n - 1);
    if (!ctx) return false;
    mark_extended(ctx->backoff);
    return true;
  };

  for (int n = 1; n <= order; ++n) {
    while (next_line() && blank_line(line)) {}
    const std::string header = "\\" + std::to_string(n) + "-grams:";
    if (eof || line != header) return "expected " + header + " but found \"" + line + "\"";
    entries[n - 1].reserve((size_t)counts[n - 1]);
    for (long long i = 0; i < counts[n - 1]; ++i) {
      if (!next_line() || blank_line(line) || line[0] == '\\')
        return "the counts disagree with the sections: " + std::to_string(n) + "-grams has " + std::to_string(i) +
               " entries, \\data\\ says " + std::to_string(counts[n - 1]);
      split_fields(line, fld);
      if ((int)fld.size() != n + 1 && (int)fld.size() != n + 2) return "malformed " + std::to_string(n) + "-gram \"" + line + "\"";
      float prob, backoff = -0.0f;
      if (!parse_float(fld[0], &prob)) return "bad log-prob in \"" + line + "\"";
      if (std::isnan(prob) || prob == INFINITY) return "non-finite log-prob in \"" + line + "\"";
      if (prob > 0.0f) return "positive log-prob in \"" + line + "\"";
      if ((int)fld.size() == n + 2) {
        if (!parse_float(fld[n + 1], &backoff)) return "bad backoff in \"" + line + "\"";
        if (!std::isfinite(backoff)) return "non-finite backoff in \"" + line + "\"";
        if (n == order && backoff != 0.0f) return "non-zero backoff on a highest-order n-gram \"" + line + "\"";
        if (backoff == 0.0f) backoff = -0.0f;
      }
      set_sign(prob);  // KenLM's Prob() sets the sign bit
      if (n == 1) {
        const std::string &w = fld[1];
        if (w == "<unk>" || w == "<UNK>") {
          if (saw_unk) return "duplicate unigram \"" + w + "\"";
          saw_unk = true;
          m.uni_prob[0] = prob;
          m.uni_backoff[0] = backoff;
          continue;
        }
        if (m.word_id.count(w)) return "duplicate unigram \"" + w + "\"";
        m.word_id.emplace(w, (int32_t)m.vocabulary.size());
        m.vocabulary.push_back(w);
        m.uni_prob.push_back(prob);
        m.uni_backoff.push_back(backoff);
        continue;
      }
      NgramEntry e;
      for (int k = 0; k < kNgramMaxOrder; ++k) e.w[k] = -1;
      for (int k = 0; k < n; ++k) {
        const std::string &w = fld[1 + k];
        const bool unk = w == "<unk>" || w == "<UNK>";
        const int32_t id = unk ? 0 : m.id_of(w);
        if (id == 0 && !unk) return "word \"" + w + "\" of \"" + line + "\" is not a unigram";
        e.w[k] = id;
      }
      e.prob = prob;
      e.backoff = backoff;
      if (!index[n - 1].emplace(key_of(e.w, n), entries[n - 1].size()).second) return "duplicate n-gram \"" + line + "\"";
      entries[n - 1].push_back(e);
      if (!link_lower(e.w, n)) return "the context of \"" + line + "\" is not in the model";
    }
  }
  while (next_line() && blank_line(line)) {}
  if (eof) return "no \\end\\ line";
  if (line != "\\end\\") {
    if (line[0] == '\\') return "expected \\end\\ but found \"" + line + "\"";
    return "the counts disagree with the sections: more " + std::to_string(order) + "-grams than \\data\\ says";
  }
  while (next_line())
    if (!blank_line(line)) return "text after \\end\\";
  if (!m.word_id.count("<s>")) return "no <s> unigram";
  if (!m.word_id.count("</s>")) return "no </s> unigram";

  for (int n = 2; n <= order; ++n) ngram_build_table(entries[n - 1], n, m.tables[n - 1]);

  m.is_character_based = ngram_character_based(m.vocabulary);
  ngram_build_front(m);
  return "";
}

// ---- the two hooks: the front end of ngram_lm.h over the host tables ----

static inline double ngram_hook_cond(void *ctx, const int32_t *labels, int n) {
  const NgramModel &m = *static_cast<const NgramModel *>(ctx);
  return ngram_prefix_cond(m.view(), m.front(), labels, n);
}

static inline double ngram_hook_sent(void *ctx, const int32_t *labels, int n) {
  const NgramModel &m = *static_cast<const NgramModel *>(ctx);
  return ngram_sentence(m.view(), m.front(), labels, n);
}

}  // namespace ctc

// Host side of the scorer path (word-based language model + dictionary), shared by the CUDA library and the CPU
// logic-test emulation.
//
// The reference keeps KenLM behind its `Scorer` class and calls it from inside the time loop
// (ctc_beam_search_decoder.cpp:120-137) and once more when results are read out (:173-208).  The language
// model stays on the host here too, behind a HOOK the integrator supplies (include/ctcdecode_b200.h,
// ctcdec_scorer_hooks: the reference side wraps its own Scorer / KenLM, see INTEGRATION.md) -- this library has
// no KenLM of its own.  What moves to the GPU is everything the hook does not do:
//   * the dictionary (reference scorer.cpp:196-230, decoder_utils.cpp:147-193, path_trie.cpp:59-96) becomes a
//     dense [state][label] table the beam kernel consults when a candidate would create a node;
//   * the per-frame cutoff (:74-82, :93-95) and the application of the LM term (:134-136) run in the kernel;
//   * the LM term of a prefix depends only on the prefix (the words before the space being appended), so the host
//     asks the hook ONCE per trie node that can be followed by a space, when the node is created, and the kernel
//     reads it from a per-node array afterwards.  The host keeps a (parent, char) mirror of the trie for that.
// The frame loop is therefore: frame -> list of created nodes to the host -> hook calls -> LM terms back -> next
// frame; by default inside ONE persistent launch (per-frame handshake through device-mapped pinned memory, see
// ctc_api.cu), optionally as one launch per frame.
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/ctcdecode_b200.h"
#include "ngram_kenlm.h"

namespace ctc {

// Deterministic dictionary automaton over label ids: words spelled with `labels`, each followed by the space
// label (reference Scorer::fill_dictionary(true) -> add_word_to_dictionary -> add_word_to_fst, then
// RmEpsilon / Determinize / Minimize: language-equivalent to this prefix trie).
struct Dictionary {
  int V = 0;
  int start = 0;
  int n_words = 0;                  // reference Scorer::dict_size_
  std::vector<int> next;            // [states][V], -1 = no arc
  std::vector<unsigned char> fin;   // [states]
  // what the kernel reads (pack_dictionary): arcs with the flags of beam_core.cuh (kDictFinal, kDictSpace) and one
  // bit per (state, character) "has an arc"
  std::vector<int> packed;          // [states][V]
  std::vector<uint32_t> mask;       // [states][wc]
  int wc = 0;

  int add_state() {
    next.insert(next.end(), V, -1);
    fin.push_back(0);
    return (int)fin.size() - 1;
  }
  int states() const { return (int)fin.size(); }
};

// split into UTF-8 characters like the reference's split_utf8_str (decoder_utils.cpp:83-99)
static inline std::vector<std::string> utf8_chars(const std::string &s) {
  std::vector<std::string> out;
  std::string cur;
  for (char ch : s) {
    if ((ch & 0xc0) != 0x80 && !cur.empty()) { out.push_back(cur); cur.clear(); }
    cur.push_back(ch);
  }
  out.push_back(cur);
  return out;
}

static inline Dictionary build_dictionary(const std::vector<std::string> &labels, int space_id,
                                          const std::vector<std::string> &words) {
  Dictionary d;
  d.V = (int)labels.size();
  d.start = d.add_state();
  std::unordered_map<std::string, int> char_map;
  for (int i = 0; i < d.V; ++i) char_map[labels[i]] = i;
  for (const std::string &w : words) {
    std::vector<int> ids;
    bool ok = true;
    for (const std::string &ch : utf8_chars(w)) {
      if (ch == " ") { ids.push_back(space_id); continue; }
      auto it = char_map.find(ch);
      if (it == char_map.end()) { ok = false; break; }  // not spellable: skipped (decoder_utils.cpp:178-183)
      ids.push_back(it->second);
    }
    if (!ok) continue;
    ids.push_back(space_id);
    int s = d.start;
    for (int id : ids) {
      int &nx = d.next[(size_t)s * d.V + id];
      if (nx < 0) { const int ns = d.add_state(); d.next[(size_t)s * d.V + id] = ns; s = ns; }
      else s = nx;
    }
    d.fin[s] = 1;
    d.n_words += 1;
  }
  return d;
}

// reference path_trie.cpp:83-92: a child whose arc ends in a final state restarts at the start state; the kernel
// also wants to know, when it creates the child, whether a space can follow it (= the host must score it)
static inline void pack_dictionary(Dictionary &d, int space_id) {
  const int S = d.states(), V = d.V;
  d.wc = (V + 31) / 32;
  d.packed.assign((size_t)S * V, -1);
  d.mask.assign((size_t)S * d.wc, 0u);
  for (int s = 0; s < S; ++s)
    for (int c = 0; c < V; ++c) {
      const int nx = d.next[(size_t)s * V + c];
      if (nx < 0) continue;
      const int dst = d.fin[nx] ? d.start : nx;
      int e = nx;
      if (d.fin[nx]) e |= 1 << 30;
      if (space_id >= 0 && d.next[(size_t)dst * V + space_id] >= 0) e |= 1 << 29;
      d.packed[(size_t)s * V + c] = e;
      d.mask[(size_t)s * d.wc + (c >> 5)] |= 1u << (c & 31);
    }
}

// A character-based model has no dictionary (reference scorer.cpp:50-53, ctc_beam_search_decoder.cpp:46): the kernel
// gets the automaton that accepts everything -- one state, every character loops back to it -- with the "tell the host
// about this node" flag on every arc.
static inline Dictionary accept_all_dictionary(int V) {
  Dictionary d;
  d.V = V;
  d.start = d.add_state();
  d.wc = (V + 31) / 32;
  d.packed.assign((size_t)V, 0 | (1 << 29));
  d.mask.assign((size_t)d.wc, 0xffffffffu);
  for (int c = 0; c < V; ++c) d.next[c] = 0;
  return d;
}

struct HostScorer {
  // cond_log_prob depends only on the last max_order words of the prefix, and beams share word histories: cache it
  // keyed by that tail of the label sequence (the hook is pure, so the values are the hook's own)
  // (one cache per host worker thread: each utterance is served by one worker, so no locking)
  typedef std::unordered_map<std::string, double> CondCache;
  std::vector<CondCache> cond_caches = std::vector<CondCache>(1);
  ctcdec_scorer_hooks hooks;
  double alpha, beta;
  int max_order, is_character_based, space_id;
  std::vector<std::string> labels;
  Dictionary dict;
  // the model behind the hooks of a scorer built from an ARPA file (ctcdec_scorer_create_arpa; hooks.ctx points to
  // it), null for a scorer whose hooks the caller supplies
  std::shared_ptr<const NgramModel> ngram;
  // what the beam kernel needs besides the tables to compute an ARPA scorer's terms itself (BeamParams::lm_dev):
  // word-based, the word id each dictionary state completes with a space (0 if none); character-based, each label's
  std::vector<int> word_of_state, label_word;
  // device copies of the tables and of those two arrays (one allocation, ensure_ngram_on_device)
  void *d_ngram = nullptr;
  int ngram_device = -1;
  NgramView d_view;
  NgramFront d_front;  // the label-to-word front end's tables on the device (the read-out kernel)
  int *d_word_of_state = nullptr, *d_label_word = nullptr;
  // device copies of the dictionary (CUDA library only)
  int *d_next = nullptr;
  uint32_t *d_mask = nullptr;
  int device = -1;
};

// An ARPA scorer's word ids for the beam kernel (BeamParams::lm_dev): word-based, the word each dictionary state completes
// with a space (the dictionary is a trie from its start state: spell every state); character-based, each label's.
static inline void lm_dev_word_ids(HostScorer &sc) {
  const NgramModel &m = *sc.ngram;
  const Dictionary &d = sc.dict;
  if (sc.is_character_based) {
    sc.label_word.clear();
    for (const std::string &l : sc.labels) sc.label_word.push_back(m.id_of(l));
    return;
  }
  sc.word_of_state.assign(d.states(), 0);
  std::vector<std::string> spelled(d.states());
  std::vector<int> todo(1, d.start);
  while (!todo.empty()) {
    const int st = todo.back();
    todo.pop_back();
    for (int c = 0; c < d.V; ++c) {
      const int nx = d.next[(size_t)st * d.V + c];
      if (nx < 0) continue;
      if (c == sc.space_id) {
        if (d.fin[nx]) sc.word_of_state[st] = m.id_of(spelled[st]);
        continue;
      }
      spelled[nx] = spelled[st] + sc.labels[c];
      todo.push_back(nx);
    }
  }
}

// Per-utterance host mirror of the trie: enough to spell the prefix of any node.
struct TrieMirror {
  // Capacity for the arena is reserved up front (address space only: a frame's worth of an utterance's nodes is a few
  // hundred bytes, while filling 1 + beam x frames entries per utterance ahead of time cost config 5 fifty megabytes of
  // page faults per call); node ids arrive in increasing order, so growing the used part is amortised pushes.
  std::vector<int> parent, chr;
  void reserve(size_t nodes) {
    parent.clear(); chr.clear();
    parent.reserve(nodes > 0 ? nodes : 1); chr.reserve(nodes > 0 ? nodes : 1);
    parent.push_back(-1); chr.push_back(-1);  // node 0, the root
  }
  void add(int nid, int par, int ch) {
    if ((size_t)nid >= parent.size()) { parent.resize((size_t)nid + 1, -1); chr.resize((size_t)nid + 1, -1); }
    parent[nid] = par;
    chr[nid] = ch;
  }
  // The labels of node nid's prefix from just after the max_words-th space from the end (walking up, every space
  // ends a word): exactly the part Scorer::make_ngram looks at (scorer.cpp:163-194); the whole prefix if it has
  // fewer words.
  void tail_labels_of(int nid, int space_id, int max_words, std::vector<int> &out) const {
    out.clear();
    int words = 0;
    for (int q = nid; q > 0; q = parent[q]) {
      if (chr[q] == space_id && ++words == max_words) break;
      out.push_back(chr[q]);
    }
    for (size_t a = 0, b = out.size(); a + 1 < b; ++a, --b) std::swap(out[a], out[b - 1]);
  }
  // the last n labels of node nid's prefix (all of them if it is shorter)
  void last_labels_of(int nid, int n, std::vector<int> &out) const {
    out.clear();
    for (int q = nid; q > 0 && (int)out.size() < n; q = parent[q]) out.push_back(chr[q]);
    for (size_t a = 0, b = out.size(); a + 1 < b; ++a, --b) std::swap(out[a], out[b - 1]);
  }
};

// the same tail of a label array
static inline int tail_start(const int *labels, int n, int space_id, int max_words) {
  int words = 0;
  for (int i = n - 1; i >= 0; --i)
    if (labels[i] == space_id && ++words == max_words) return i + 1;
  return 0;
}

static inline double cached_cond(const HostScorer &sc, HostScorer::CondCache &cache, const int *labels, int n) {
  std::string key(reinterpret_cast<const char *>(labels), (size_t)n * sizeof(int));
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  const double v = sc.hooks.cond_log_prob(sc.hooks.ctx, labels, n);
  if (cache.size() > (1u << 20)) cache.clear();
  cache.emplace(std::move(key), v);
  return v;
}

// The two per-utterance exchange blocks (beam_core.cuh BeamParams::newlist / lm_upd): strides in ints, each a
// multiple of 128 bytes so that no two utterances (host workers, CTAs) share a line.  row_len: 0 for a word-based
// model ((node, term) pairs), the vocabulary size for a character-based one ((node, V terms) entries).
static inline void exchange_strides(int K, int row_len, int *nl_stride, int *up_stride) {
  *nl_stride = (4 + 4 * K + 31) / 32 * 32;
  *up_stride = (2 + (row_len > 0 ? 1 + row_len : 2) * K + 31) / 32 * 32;
}
static inline int exchange_row_len(const struct HostScorer &sc) { return sc.is_character_based ? (int)sc.labels.size() : 0; }

// Character-based model: the V terms float(cond_log_prob(prefix + c) * alpha) of one node (reference :125-133 with
// prefix_to_score = prefix_new; Scorer::make_ngram looks at the last max_order characters only, scorer.cpp:172-174).
// labels: the node's last min(depth, max_order - 1) labels; scratch has room for one more.
static inline void lm_char_row(const HostScorer &sc, HostScorer::CondCache &cache, std::vector<int> &labels, int *out) {
  const int V = (int)sc.labels.size();
  labels.push_back(0);
  for (int c = 0; c < V; ++c) {
    labels.back() = c;
    const float val = (float)(cached_cond(sc, cache, labels.data(), (int)labels.size()) * sc.alpha);
    memcpy(&out[c], &val, 4);
  }
  labels.pop_back();
}

// Before the first frame of an utterance with a character-based model: the root's row, as the block's only entry.
static inline void lm_char_root_entry(const HostScorer &sc, HostScorer::CondCache &cache, int *upd, std::vector<int> &scratch) {
  scratch.clear();
  upd[1] = 1;
  upd[2] = 0;
  lm_char_row(sc, cache, scratch, upd + 3);
}

// After a frame: register the created nodes and compute the LM term of those a space can follow.
// newlist: one utterance's block ([0] = count, from [4]: 16-byte entries node / parent / chr / needs_lm); writes
// the answer into the utterance's lm_upd block: [1] = number of pairs, from [2]: (node, float bits) pairs.  The
// caller publishes it ([0], the go flag) afterwards.  Returns the number of pairs.
static inline int lm_after_frame(const HostScorer &sc, HostScorer::CondCache &cache, TrieMirror &mirror,
                                 const int *newlist, int *upd, std::vector<int> &scratch) {
  const int cnt = newlist[0];
  int nu = 0;
  for (int q = 0; q < cnt; ++q) {
    const int *e = newlist + 4 + 4 * q;
    if (e[0] < 0) continue;  // a revived node: already known
    mirror.add(e[0], e[1], e[2]);
    if (sc.is_character_based) {
      const int V = (int)sc.labels.size();
      mirror.last_labels_of(e[0], sc.max_order - 1, scratch);
      upd[2 + (1 + V) * nu] = e[0];
      lm_char_row(sc, cache, scratch, upd + 2 + (1 + V) * nu + 1);
      ++nu;
    } else if (e[3]) {
      mirror.tail_labels_of(e[0], sc.space_id, sc.max_order, scratch);
      const double cond = cached_cond(sc, cache, scratch.data(), (int)scratch.size());
      const float val = (float)(cond * sc.alpha);  // reference :133 `score = get_log_cond_prob(ngram) * alpha` (float)
      upd[2 + 2 * nu] = e[0];
      memcpy(&upd[3 + 2 * nu], &val, 4);
      ++nu;
    }
  }
  upd[1] = nu;
  return nu;
}

// DecoderState::decode with a scorer (reference ctc_beam_search_decoder.cpp:164-211): the order of the
// results is by the raw prefix score (decoder_utils.cpp:59), the reported score is the LM-corrected approx_ctc.
// tokens / lens / scores are one utterance's rows as written by the finalize kernel (scores = -raw score).
// cond_rows[p] must hold cond_log_prob of row p's prefix when the row does not end in a space (computed by the
// caller through the cache, single-threaded); the sentence hook is called here, so this function may run on
// several threads over disjoint utterances.
static inline void lm_rescore(const HostScorer &sc, int n_results, int row_stride, const int *tokens, const int *lens,
                              const double *cond_rows, float *scores) {
  for (int p = 0; p < n_results; ++p) {
    const int len = lens[p];
    const int *tok = tokens + (size_t)p * row_stride;
    const bool last_word = !sc.is_character_based && len > 0 && tok[len - 1] != sc.space_id;  // :173-185
    scores[p] = lm_readout_score(scores[p], len, last_word, cond_rows[p], sc.hooks.sent_log_prob(sc.hooks.ctx, tok, len),
                                 sc.alpha, sc.beta);
  }
}

}  // namespace ctc

namespace ctc {

// Result read-out for a whole batch: last-word terms through the cache, sentence terms on a few host threads.
static inline void lm_rescore_batch(HostScorer &sc, int B, int K, int T, const int *n_results, const int *tokens,
                                    const int *lens, float *scores) {
  std::vector<double> cond((size_t)B * K, 0.0);
  for (int b = 0; b < B; ++b)
    for (int p = 0; p < n_results[b] && p < K; ++p) {
      const int len = lens[(size_t)b * K + p];
      const int *tok = tokens + ((size_t)b * K + p) * T;
      if (!sc.is_character_based && len > 0 && tok[len - 1] != sc.space_id) {
        const int st = tail_start(tok, len, sc.space_id, sc.max_order);
        cond[(size_t)b * K + p] = cached_cond(sc, sc.cond_caches[0], tok + st, len - st);
      }
    }
  unsigned nt = std::thread::hardware_concurrency();
  nt = nt == 0 ? 1 : (nt > 32 ? 32 : nt);  // (the sentence hook of a result row costs ~15 us; config 5 has 6400 rows)
  if ((unsigned)B < nt) nt = (unsigned)B;
  std::vector<std::thread> pool;
  for (unsigned w = 0; w < nt; ++w)
    pool.emplace_back([&, w]() {
      for (int b = (int)w; b < B; b += (int)nt)
        lm_rescore(sc, n_results[b] < K ? n_results[b] : K, T, tokens + (size_t)b * K * T, lens + (size_t)b * K,
                   cond.data() + (size_t)b * K, scores + (size_t)b * K);
    });
  for (auto &th : pool) th.join();
}

}  // namespace ctc

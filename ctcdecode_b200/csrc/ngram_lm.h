// N-gram language model read from an ARPA text file or a KenLM binary file: the tables, the one lookup that reproduces
// the reference's Scorer::get_log_cond_prob (scorer.cpp:74-93) over KenLM bit for bit, the reference's label-to-word
// front end (make_ngram, split_labels, get_sent_log_prob) and the read-out rescoring of a result row.  All of it
// compiles for the host and for the device (plain pointers: views of host vectors or of their HBM copies); the loaders
// and the building of the tables are host code (ngram_arpa.h, ngram_kenlm.h).
//
// What is reproduced, from KenLM's query path (lm/model.cc FullScore / ResumeScore, lm/read_arpa.cc):
//   * word ids: 0 is <unk> (also "<UNK>"), then the unigrams in file order (a binary file's own id order); an unknown
//     string is 0;
//   * log10 probabilities are read as KenLM returns them: from ARPA text and probing files with the sign bit set (its
//     Prob() does so; 0 becomes -0.0), from a trie file as stored;
//   * a backoff of 0 (or none) is stored as -0.0, "no n-gram extends this one", and turned into +0.0 when the n-gram is
//     the context of a longer one: the sign decides how long the state's history is, as in KenLM;
//   * a word is scored in the state left by the previous one: the longest matching n-gram's probability, then the
//     state's context backoffs from the matched length up, added in float in that order.
// The tables hold the file's n-grams plus the suffix entries KenLM fills in on load (ngram_arpa.h), or what a KenLM
// binary file holds (ngram_kenlm.h), so "not found" means the same thing here as in KenLM.
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

// How the tables of orders >= 2 are laid out.
enum NgramLayout {
  kNgramTables = 0,        // NgramEntry tables with the full key (ARPA text)
  kNgramKenlmProbing = 1,  // a KenLM probing file's own tables, searched by their 64-bit keys (ngram_probe)
  kNgramKenlmTrie = 2,     // a KenLM trie file's search data, walked as it is (ngram_trie_*)
};

// Where one order's data lies in a KenLM trie file's search region (NgramTrie::bits); all positions are in bits from
// the region's start.  Order n >= 2 (index n - 1): entry i has its word id at bit + i * total_bits, then quant_bits of
// value (unquantized: a 31-bit probability without its sign, then a 32-bit backoff below the highest order; quantized:
// the backoff code, then the probability code), then, below the highest order, the low inline_bits of its next
// pointer.  Index 0 describes the unigram array of {float prob, float backoff, uint64 next} records.
struct NgramTrieOrder {
  uint64_t bit = 0;          // entry 0 (n >= 2), or the unigram array (index 0)
  uint64_t entries = 0;      // entries of the order (the array has one more, the last pointer's end)
  uint64_t offsets = 0;      // array tries, n < order: the offset array of n_offsets uint64 values (lm/bhiksha.cc);
  uint64_t n_offsets = 0;    // a next pointer's high bits are the last index whose value is <= the entry's index
  uint64_t prob_bins = 0, backoff_bins = 0;  // quantized: this order's bins, 2^prob_bits / 2^backoff_bits floats
  uint8_t word_bits = 0, quant_bits = 0, inline_bits = 0, total_bits = 0;
  uint8_t prob_bits = 0, backoff_bits = 0;   // 0: unquantized
};

// A trie file's search region (8-byte aligned, zero-padded by at least 8 bytes) and its order descriptors [order].
struct NgramTrie {
  const uint64_t *bits;
  const NgramTrieOrder *orders;
};

// Read-only view of the tables: host vectors or their device copies.  It is a kernel parameter of the beam and read-out
// kernels, and its size is kept: the layouts share the per-order fields.
struct NgramView {
  int order = 0;
  int vocab = 0;
  int bos = 0;                         // the id of "<s>"
  int layout = kNgramTables;
  const float *uni_prob = nullptr;     // [vocab]; a probing file's raw values, the sign bit its independent-left flag
  const float *uni_backoff = nullptr;  // [vocab]
  // [n - 1]: order n >= 2.  kNgramTables: capacity mask[n - 1] + 1 (a power of two).  kNgramKenlmProbing: the table's
  // bytes, buckets[n - 1] entries of 16 bytes (key, prob, backoff) below the highest order and of 12 bytes (key, prob)
  // at it, both packed to 4 bytes (so a key is read as two 32-bit words).  kNgramKenlmTrie: `trie`, for all orders.
  union {
    const NgramEntry *table[kNgramMaxOrder] = {};
    const uint32_t *probe[kNgramMaxOrder];
    NgramTrie trie;
  };
  union {
    uint32_t mask[kNgramMaxOrder] = {};
    uint32_t buckets[kNgramMaxOrder];
  };
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

CTC_NG_HD uint32_t ngram_bits(float f) {
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
}
CTC_NG_HD float ngram_float(uint32_t u) {
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// KenLM's key of an n-gram in a probing file (lm/search_hashed.hh CombineWordHash): it starts as the newest word's id,
// and each older word is folded in.
CTC_NG_HD uint64_t ngram_kenlm_combine(uint64_t key, int32_t older) {
  return (key * 8978948897894561157ull) ^ ((uint64_t)(uint32_t)(1u + (uint32_t)older) * 17894857484156487943ull);
}

// The entry with this key in order n's probing table, or null: linear probing from key % buckets; key 0 is an empty
// bucket (util/probing_hash_table.hh Find).
CTC_NG_HD const uint32_t *ngram_probe(const NgramView &m, int n, uint64_t key) {
  const uint32_t *t = m.probe[n - 1];
  const uint32_t buckets = m.buckets[n - 1];
  const uint32_t words = n < m.order ? 4 : 3;
  for (uint64_t b = key % buckets;; b = b + 1 == buckets ? 0 : b + 1) {
    const uint32_t *e = t + b * words;
    const uint64_t got = (uint64_t)e[0] | ((uint64_t)e[1] << 32);
    if (got == key) return e;
    if (got == 0) return nullptr;
  }
}

// The stored (prob, backoff) bits of the n-gram key[0..n) (text order) in either layout; false if it is not there.  A
// probing file's key starts as the newest word's id and folds in the older words, newest first.
CTC_NG_HD bool ngram_lookup(const NgramView &m, const int32_t *key, int n, uint32_t &prob, uint32_t &backoff) {
  if (m.layout == kNgramKenlmProbing) {
    uint64_t h = (uint32_t)key[n - 1];
    for (int i = n - 2; i >= 0; --i) h = ngram_kenlm_combine(h, key[i]);
    const uint32_t *e = ngram_probe(m, n, h);
    if (!e) return false;
    prob = e[2];
    backoff = n < m.order ? e[3] : 0u;
    return true;
  }
  const NgramEntry *e = ngram_find(m, key, n);
  if (!e) return false;
  prob = ngram_bits(e->prob);
  backoff = ngram_bits(e->backoff);
  return true;
}

// ---- a KenLM trie file searched where it is (lm/search_trie.hh TrieSearch, lm/trie.cc, lm/bhiksha.cc) ----

// The 64 bits of the trie region from bit `bit` on.  Two aligned 64-bit loads and a shift: the packed fields start at
// any bit and straddle words, and an unaligned 8-byte load is a fault on the device.  The region's zero padding keeps
// the second word inside it.
CTC_NG_HD uint64_t ngram_trie_read(const uint64_t *b, uint64_t bit) {
  const uint64_t i = bit >> 6;
  const unsigned s = (unsigned)(bit & 63);
  const uint64_t lo = b[i];
  return s ? (lo >> s) | (b[i + 1] << (64 - s)) : lo;
}

CTC_NG_HD uint64_t ngram_trie_field(const uint64_t *b, uint64_t bit, unsigned width) {
  return ngram_trie_read(b, bit) & ((1ull << width) - 1);
}

// The next pointer of entry i of order n < order: the start of its children's range in order n + 1.
CTC_NG_HD uint64_t ngram_trie_next(const uint64_t *b, const NgramTrieOrder &o, uint64_t i) {
  uint64_t v = ngram_trie_field(b, o.bit + i * o.total_bits + o.word_bits + o.quant_bits, o.inline_bits);
  if (o.n_offsets) {  // array trie: the last offset index whose value is <= i (the first is 0, so there is one)
    uint64_t lo = 1, hi = o.n_offsets;
    while (lo < hi) {
      const uint64_t mid = lo + (hi - lo) / 2;
      if (ngram_trie_read(b, o.offsets + 64 * mid) <= i) lo = mid + 1;
      else hi = mid;
    }
    v |= (lo - 1) << o.inline_bits;
  }
  return v;
}

// Searches order n's entries [lo, hi) (one node's children: word ids unique and increasing) for `word`.  On a match
// the (prob, backoff) bits KenLM's FullScore reads for the entry, and, below the highest order, [lo, hi) becomes the
// entry's children's range.  Entry indices fit 32 bits (the loader refuses larger orders): 64-bit ranges would make the
// read-out kernel spill.
CTC_NG_HD bool ngram_trie_step(const NgramView &m, int n, int32_t word, uint32_t &lo, uint32_t &hi, uint32_t &prob,
                               uint32_t &backoff) {
  const uint64_t *b = m.trie.bits;
  const NgramTrieOrder &o = m.trie.orders[n - 1];
  const uint64_t total = o.total_bits;
  uint32_t a = lo, z = hi, i = 0;
  bool found = false;
  while (a < z && !found) {
    i = a + (z - a) / 2;
    const uint64_t got = ngram_trie_field(b, o.bit + i * total, o.word_bits);
    found = got == (uint64_t)(uint32_t)word;
    if (got < (uint64_t)(uint32_t)word) a = i + 1;
    else z = i;
  }
  if (!found) return false;
  const uint64_t vb = o.bit + i * total + o.word_bits;
  if (o.prob_bits) {  // quantized: the backoff code first (below the highest order), then the probability code
    const unsigned bb = n < m.order ? o.backoff_bits : 0;
    prob = (uint32_t)ngram_trie_read(b, o.prob_bins + 32 * ngram_trie_field(b, vb + bb, o.prob_bits));
    backoff = bb ? (uint32_t)ngram_trie_read(b, o.backoff_bins + 32 * ngram_trie_field(b, vb, bb)) : 0x80000000u;
  } else {  // the sign bit is not stored; the backoff follows the probability's 31 bits
    prob = (uint32_t)ngram_trie_read(b, vb) | 0x80000000u;
    backoff = n < m.order ? (uint32_t)ngram_trie_read(b, vb + 31) : 0x80000000u;
  }
  if (n < m.order) {
    lo = (uint32_t)ngram_trie_next(b, o, i);
    hi = (uint32_t)ngram_trie_next(b, o, i + 1);
  }
  return true;
}

// KenLM GenericModel::FullScore(in, w, out).prob: log10 p(w | in's history).  Only the search depends on the layout.
// A probing file's probabilities carry KenLM's independent-left flag in their sign bit: they are read as Prob() reads
// them (sign set; the highest order's as stored), and a set flag ends the search, as in KenLM's ResumeScore.  A trie
// is walked from w's unigram record, one older history word per order, each search within the last match's children.
CTC_NG_HD float ngram_score(const NgramView &m, const NgramState &in, int32_t w, NgramState &out) {
  const bool probing = m.layout == kNgramKenlmProbing;
  const bool trie = m.layout == kNgramKenlmTrie;
  float prob = m.uni_prob[w];
  bool stop = probing && (ngram_bits(prob) >> 31);
  if (probing) prob = ngram_float(ngram_bits(prob) | 0x80000000u);
  out.backoff[0] = m.uni_backoff[w];
  out.len = ngram_has_extension(out.backoff[0]) ? 1 : 0;
  out.words[0] = w;
  int matched = 1;
  int32_t key[kNgramMaxOrder];
  uint32_t lo = 0, hi = 0;  // trie: the children of the longest match so far
  if (trie && in.len > 0) {
    const uint64_t u = m.trie.orders[0].bit + 128 * (uint64_t)w + 64;  // (the `next` field of w's unigram record)
    lo = (uint32_t)ngram_trie_read(m.trie.bits, u);
    hi = (uint32_t)ngram_trie_read(m.trie.bits, u + 128);
  }
  for (int j = 0; j < in.len && !stop; ++j) {  // the n-gram of the last j + 1 history words and w
    const int n = j + 2;
    uint32_t p, bo;
    if (trie) {
      if (!ngram_trie_step(m, n, in.words[j], lo, hi, p, bo)) break;
    } else {
      for (int i = 0; i <= j; ++i) key[i] = in.words[j - i];
      key[j + 1] = w;
      if (!ngram_lookup(m, key, n, p, bo)) break;
    }
    if (probing) {
      stop = p >> 31;
      if (n < m.order) p |= 0x80000000u;
    }
    prob = ngram_float(p);
    matched = n;
    if (n < m.order) {
      out.backoff[j + 1] = ngram_float(bo);
      if (ngram_has_extension(ngram_float(bo))) out.len = n;
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

// ---- the reference's label-to-word front end (scorer.cpp:95-194, decoder_utils.cpp:83-120) over flat tables ----

// One unigram of the spelling table (open addressing); len < 0 marks an empty slot.
struct NgramWordSlot {
  uint32_t hash, off;  // FNV-1a of the spelling, its offset in the spelling bytes
  int32_t len, id;     // spelling length in bytes, KenLM word id
};

// Read-only view of the front end's tables, built once per model (ngram_build_front): the decoder's labels as one byte
// blob, and a lookup from a word's bytes to its id (0 for a word the model does not have, as KenLM's index()).
struct NgramFront {
  int space_id = -1;            // the " " label, -1 if none
  int is_character_based = 1;
  int32_t bos = 0, eos = 0;     // ids of "<s>" / "</s>"
  const unsigned char *label_bytes = nullptr;  // label l: label_bytes[label_off[l] .. label_off[l + 1])
  const int32_t *label_off = nullptr;          // [labels + 1]
  const unsigned char *word_bytes = nullptr;   // the unigrams' spellings
  const NgramWordSlot *words = nullptr;        // [word_mask + 1], a power of two at least twice the unigram count
  uint32_t word_mask = 0;
};

CTC_NG_HD uint32_t ngram_fnv(uint32_t h, unsigned char c) { return (h ^ c) * 16777619u; }
constexpr uint32_t kNgramFnvBasis = 2166136261u;

// A byte position in the string a label row spells: byte o of label tok[k]; k == n is the end.  Positions are kept
// normalised (o inside its label, empty labels skipped), so two equal positions compare equal.
struct NgramPos { int k, o; };

CTC_NG_HD int ngram_label_len(const NgramFront &f, int32_t l) { return f.label_off[l + 1] - f.label_off[l]; }
CTC_NG_HD NgramPos ngram_norm(const NgramFront &f, const int32_t *tok, int n, NgramPos c) {
  while (c.k < n && c.o >= ngram_label_len(f, tok[c.k])) { ++c.k; c.o = 0; }
  return c;
}
CTC_NG_HD unsigned char ngram_byte(const NgramFront &f, const int32_t *tok, NgramPos c) {
  return f.label_bytes[f.label_off[tok[c.k]] + c.o];
}
CTC_NG_HD NgramPos ngram_next(const NgramFront &f, const int32_t *tok, int n, NgramPos c) {
  ++c.o;
  return ngram_norm(f, tok, n, c);
}
CTC_NG_HD bool ngram_same(NgramPos a, NgramPos b) { return a.k == b.k && a.o == b.o; }

// The id of the word spelled by the bytes [a, b) of the row (Scorer's ext_scorer index(), 0 if the model lacks it).
// The bytes are walked twice, once for the hash and once per candidate, so no word buffer is needed.
CTC_NG_HD int32_t ngram_word_id(const NgramFront &f, const int32_t *tok, int n, NgramPos a, NgramPos b) {
  uint32_t h = kNgramFnvBasis;
  int32_t len = 0;
  for (NgramPos c = a; !ngram_same(c, b); c = ngram_next(f, tok, n, c)) {
    h = ngram_fnv(h, ngram_byte(f, tok, c));
    ++len;
  }
  for (uint32_t s = h & f.word_mask;; s = (s + 1) & f.word_mask) {
    const NgramWordSlot &w = f.words[s];
    if (w.len < 0) return 0;
    if (w.hash != h || w.len != len) continue;
    NgramPos c = a;
    int32_t i = 0;
    for (; i < len && ngram_byte(f, tok, c) == f.word_bytes[w.off + i]; ++i) c = ngram_next(f, tok, n, c);
    if (i == len) return w.id;
  }
}

// Scorer::get_log_cond_prob(Scorer::make_ngram(prefix)) of the prefix spelled by tok[0..n): the last max_order words
// (split on the space label; one label per word for a character-based model), "<s>"-padded in front when the prefix has
// fewer.
CTC_NG_HD double ngram_prefix_cond(const NgramView &m, const NgramFront &f, const int32_t *tok, int n) {
  int32_t ids[kNgramMaxOrder];
  int got = 0, i = n;
  for (int o = 0; o < m.order; ++o) {
    int j;
    if (f.is_character_based) {
      j = i > 0 ? i - 1 : 0;
    } else {
      j = i;
      while (j > 0 && tok[j - 1] != f.space_id) --j;
    }
    // the word is labels [j, i); a character-based model's is the one label i - 1 (none at the start)
    const NgramPos a = ngram_norm(f, tok, n, NgramPos{j, 0}), b = ngram_norm(f, tok, n, NgramPos{i, 0});
    ids[m.order - 1 - got++] = ngram_word_id(f, tok, n, a, b);
    if (j == 0) {
      for (int k = 0; k < m.order - o - 1; ++k) ids[m.order - 1 - got++] = m.bos;
      break;
    }
    i = f.is_character_based ? j : j - 1;
  }
  return ngram_cond_ids(m, ids + m.order - got, got);
}

// Scorer::get_sent_log_prob(Scorer::split_labels(prefix)) of tok[0..n): the labels' concatenated string split on ' '
// bytes with split_str's rule (empty pieces dropped), or into UTF-8 characters for a character-based model
// (split_utf8_str); "<s>"-padded, "</s>" appended, every max_order window scored from the null context and summed in
// double from left to right.  The sentence is streamed through a window of max_order ids.
CTC_NG_HD double ngram_sentence(const NgramView &m, const NgramFront &f, const int32_t *tok, int n) {
  const NgramPos end{n, 0};
  NgramPos c = ngram_norm(f, tok, n, NgramPos{0, 0});
  bool any_word = n > 0;  // split_utf8_str gives one word, possibly empty, for any non-empty prefix
  if (!f.is_character_based) {
    any_word = false;
    for (NgramPos q = c; !ngram_same(q, end) && !any_word; q = ngram_next(f, tok, n, q)) any_word = ngram_byte(f, tok, q) != ' ';
  }
  int pads = any_word ? m.order - 1 : m.order;
  bool empty_word = f.is_character_based && n > 0 && ngram_same(c, end), eos_done = false;
  int32_t win[kNgramMaxOrder];  // the last max_order ids of the sentence so far
  int cnt = 0;
  double score = 0.0;
  while (true) {  // one id of the sentence per pass (one inlined lookup for the whole sentence)
    int32_t id;
    if (pads > 0) {
      id = m.bos;
      --pads;
    } else if (empty_word) {
      id = ngram_word_id(f, tok, n, c, c);
      empty_word = false;
    } else {
      if (!f.is_character_based)
        while (!ngram_same(c, end) && ngram_byte(f, tok, c) == ' ') c = ngram_next(f, tok, n, c);
      if (!ngram_same(c, end)) {
        const NgramPos a = c;
        c = ngram_next(f, tok, n, c);
        if (f.is_character_based)
          while (!ngram_same(c, end) && (ngram_byte(f, tok, c) & 0xc0) == 0x80) c = ngram_next(f, tok, n, c);
        else
          while (!ngram_same(c, end) && ngram_byte(f, tok, c) != ' ') c = ngram_next(f, tok, n, c);
        id = ngram_word_id(f, tok, n, a, c);
      } else if (!eos_done) {
        id = f.eos;
        eos_done = true;
      } else {
        break;
      }
    }
    if (cnt == m.order) {
      for (int k = 1; k < m.order; ++k) win[k - 1] = win[k];
      win[m.order - 1] = id;
    } else {
      win[cnt++] = id;
    }
    if (cnt == m.order) score += ngram_cond_ids(m, win, m.order);
  }
  return score;
}

// ---- the read-out rescoring (reference DecoderState::decode, ctc_beam_search_decoder.cpp:173-208) ----
// Every double operation rounds as in the x86-64 host build, which has no FMA: on the device the multiplies, adds and
// subtracts are written as _rn intrinsics, which nvcc never contracts.
#if defined(__CUDA_ARCH__)
#define CTC_NG_DMUL(a, b) __dmul_rn((a), (b))
#define CTC_NG_DADD(a, b) __dadd_rn((a), (b))
#define CTC_NG_DSUB(a, b) __dsub_rn((a), (b))
#else
#define CTC_NG_DMUL(a, b) ((a) * (b))
#define CTC_NG_DADD(a, b) ((a) + (b))
#define CTC_NG_DSUB(a, b) ((a) - (b))
#endif

// The reported score of one result row.  score: what the finalize kernel wrote (minus the raw prefix score); len: the
// row's length; last_word: a word-based row whose last label is not the space, so that its unfinished last word is
// scored: float(cond * alpha), then float(s + beta) added to the raw score in float.  Then approx_ctc =
// double(raw) - len * beta - sent * alpha, reported as -double(float(approx_ctc)) (decoder_utils.cpp:68, binding.cpp:91).
CTC_NG_HD float lm_readout_score(float score, int len, bool last_word, double cond, double sent, double alpha,
                                 double beta) {
  float ext = -score;
  if (last_word) {
    float s = (float)CTC_NG_DMUL(cond, alpha);
    s = (float)CTC_NG_DADD((double)s, beta);
    ext = ext + s;
  }
  double approx = (double)ext;
  approx = CTC_NG_DSUB(approx, CTC_NG_DMUL((double)len, beta));
  approx = CTC_NG_DSUB(approx, CTC_NG_DMUL(sent, alpha));
  const float approx_f = (float)approx;
  return (float)(-(double)approx_f);
}

// lm_readout_score of the row tok[0..len) with an ARPA model: both terms from the front end above.
CTC_NG_HD float ngram_readout_row(const NgramView &m, const NgramFront &f, const int32_t *tok, int len, float score,
                                  double alpha, double beta) {
  const bool last_word = !f.is_character_based && len > 0 && tok[len - 1] != f.space_id;
  const double cond = last_word ? ngram_prefix_cond(m, f, tok, len) : 0.0;
  return lm_readout_score(score, len, last_word, cond, ngram_sentence(m, f, tok, len), alpha, beta);
}

}  // namespace ctc

#undef CTC_NG_DMUL
#undef CTC_NG_DADD
#undef CTC_NG_DSUB
#undef CTC_NG_HD

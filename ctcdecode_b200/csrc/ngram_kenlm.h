// KenLM binary files ("mmap lm http://kheafield.com/code format version 5", written by KenLM's build_binary) for the
// n-gram scorer, and load_ngram_file, the one loader entry that takes ARPA text or a binary file.
//
// What is read (KenLM lm/binary_format.cc, vocab.cc, search_hashed.cc, trie.cc, bhiksha.cc, quantize.cc):
//   * the header: the Sanity block (magic, test floats and integers of this endianness and these type sizes), the fixed
//     parameters (order, probing multiplier, model type, has-vocabulary flag, search version) and the n-gram counts;
//   * the vocabulary strings at the end of the file, in word-id order with "<unk>" first: word id = position, so the
//     file's own vocabulary hash table is never read;
//   * PROBING (type 0): the unigram array is split into uni_prob / uni_backoff, and the tables of orders 2..N are kept
//     byte for byte (NgramModel::probing) and searched as they are (ngram_lm.h ngram_probe): their keys are 64-bit
//     hashes of word ids, from which the n-grams cannot be recovered;
//   * TRIE, QUANT_TRIE, ARRAY_TRIE, QUANT_ARRAY_TRIE (types 2-5): the search region (quantization bins, unigram
//     records, Bhiksha offset arrays, bit-packed orders) is kept byte for byte (NgramModel::trie_bits) with a
//     descriptor per order, and searched as it is (ngram_lm.h ngram_trie_step), after one validation pass
//     (trie_validate) that makes every search end inside the region.  The file already holds the entries build_binary
//     filled in for pruned suffixes, so nothing is added.
// Refused, with the reason (all before anything reaches the device): a truncated file or header, the "incomplete" magic,
// a version other than 5, other test values, REST_PROBING (type 1, build_binary -r), an unknown model type or search
// version, order 1 or above kNgramMaxOrder, no vocabulary strings or a word count that disagrees with the header, no
// <s> or </s>, region sizes that disagree with the file's length, a probing table with no empty bucket (its search
// would never end), trie word ids out of range or out of order, and trie pointers that decrease or point past their
// array.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include "ngram_arpa.h"

namespace ctc {

namespace kenlm_detail {

constexpr char kMagicPrefix[] = "mmap lm http://kheafield.com/code";
constexpr char kMagicVersion[] = "mmap lm http://kheafield.com/code format version";
constexpr char kMagicIncomplete[] = "mmap lm http://kheafield.com/code incomplete\n";
// The Sanity block: the magic with its two NULs padded to 56 bytes, 0.0f 1.0f -0.5f, the word indices 1 and 2^32 - 1,
// 4 bytes of padding, the uint64 1.
constexpr size_t kSanityBytes = 88;
// FixedWidthParameters: order (u8), probing multiplier (f32 at 4), model type (i32 at 8), has vocabulary (u8 at 12),
// search version (u32 at 16).
constexpr size_t kFixedBytes = 20;
enum { kProbing = 0, kRestProbing = 1, kTrie = 2, kQuantTrie = 3, kArrayTrie = 4, kQuantArrayTrie = 5 };

inline uint64_t align8(uint64_t x) { return (x + 7) / 8 * 8; }

inline uint8_t required_bits(uint64_t v) {  // bits to store integers up to v (util/bit_packing.cc RequiredBits)
  if (!v) return 0;
  uint8_t r = 1;
  while (v >>= 1) ++r;
  return r;
}

// Buckets of a probing table of `entries` (util/probing_hash_table.hh Size with DivMod), in KenLM's float arithmetic.
inline uint64_t probing_buckets(uint64_t entries, float multiplier) {
  return std::max(entries + 1, (uint64_t)(multiplier * (float)entries));
}

struct File {
  std::vector<unsigned char> b;
  template <class T> T at(uint64_t off) const {
    T v;
    memcpy(&v, b.data() + off, sizeof(T));
    return v;
  }
};

// Pointer compression of the array tries (lm/bhiksha.cc): how many high bits of a next pointer move to the offset array.
inline uint8_t chop_bits(uint64_t max_offset, uint64_t max_next, uint8_t configured) {
  const uint8_t required = required_bits(max_next);
  uint8_t best = 0;
  int64_t lowest = std::numeric_limits<int64_t>::max();
  for (uint8_t chop = 0; chop <= std::min(required, configured); ++chop) {
    const int64_t change = (int64_t)((max_next >> (required - chop)) * 64 - max_offset * (uint64_t)chop);
    if (change < lowest) { lowest = change; best = chop; }
  }
  return best;
}

// One bit-packed trie order: entry i has its word id at bit i * total of `base`, then its value (quant bits), then,
// for a middle order, the low bits of its next pointer.
struct PackedOrder {
  uint64_t base = 0, entries = 0;
  uint8_t word_bits = 0, quant_bits = 0, inline_bits = 0, total_bits = 0;
  // array tries: the offset array (file offset, count) whose index gives a next pointer's high bits
  uint64_t offsets = 0, n_offsets = 0;
};

// TrieSearch::Size's pieces for one middle order (trie.cc BitPackedMiddle::Size, bhiksha.cc).
inline uint64_t middle_size(bool array, uint8_t bhiksha_bits, uint8_t quant_bits, uint64_t entries, uint64_t max_vocab,
                            uint64_t max_next, PackedOrder *o, uint64_t base) {
  uint64_t bhiksha = 0;
  uint8_t inline_bits = required_bits(max_next);
  uint64_t n_offsets = 0;
  if (array) {
    const uint8_t chop = chop_bits(entries + 1, max_next, bhiksha_bits);
    n_offsets = (max_next >> (required_bits(max_next) - chop)) + 1;
    bhiksha = 8 * (1 + n_offsets) + 7;
    inline_bits = (uint8_t)(required_bits(max_next) - chop);
  }
  const uint8_t total = (uint8_t)(required_bits(max_vocab) + quant_bits + inline_bits);
  if (o) {
    o->base = base + bhiksha;
    o->entries = entries;
    o->word_bits = required_bits(max_vocab);
    o->quant_bits = quant_bits;
    o->inline_bits = inline_bits;
    o->total_bits = total;
    o->offsets = align8(base) + 8;  // (8-byte aligned in the file, after an 8-byte header)
    o->n_offsets = n_offsets;
  }
  return bhiksha + ((1 + entries) * total + 7) / 8 + 8;
}

inline uint64_t longest_size(uint8_t quant_bits, uint64_t entries, uint64_t max_vocab, PackedOrder *o, uint64_t base) {
  const uint8_t total = (uint8_t)(required_bits(max_vocab) + quant_bits);
  if (o) {
    o->base = base;
    o->entries = entries;
    o->word_bits = required_bits(max_vocab);
    o->quant_bits = quant_bits;
    o->total_bits = total;
  }
  return ((1 + entries) * total + 7) / 8 + 8;
}

// The pointers of order q over [i, ...) read in increasing index order (the unigram records' `next` for q == 1).  An
// array trie's high bits come from a walk along the offset array; with its first value 0 and its values in order that
// is the same index the search's binary search (ngram_trie_next) finds.
struct PointerWalk {
  const uint64_t *b;
  const NgramTrieOrder &o;
  bool unigrams;
  uint64_t k = 0;
  uint64_t at(uint64_t i) {
    if (unigrams) return ngram_trie_read(b, o.bit + 128 * i + 64);
    uint64_t v = ngram_trie_field(b, o.bit + i * o.total_bits + o.word_bits + o.quant_bits, o.inline_bits);
    if (o.n_offsets) {
      while (k + 1 < o.n_offsets && ngram_trie_read(b, o.offsets + 64 * (k + 1)) <= i) ++k;
      v |= k << o.inline_bits;
    }
    return v;
  }
};

// One pass over the trie from the unigrams down, through the nodes a search can reach: every node's child range lies
// within the next order's array and ranges follow each other (pointers never decrease), and the word ids of a node are
// in the vocabulary and increasing.  A search in a trie that passes stays in bounds and finds what a full-key table
// would.  Reads the region sequentially and allocates nothing.  Returns "" or the reason.
inline std::string trie_validate(const NgramModel &m, uint64_t bound) {
  const uint64_t *b = m.trie_bits.data();
  const int order = m.order;
  uint64_t lo = 0, hi = bound;  // the parents (order n - 1) reachable from the unigrams
  for (int n = 2; n <= order; ++n) {
    const NgramTrieOrder &parent = m.trie_orders[n - 2], &o = m.trie_orders[n - 1];
    uint64_t c_lo, c_hi;
    {
      PointerWalk walk{b, parent, n == 2};
      c_lo = c_hi = walk.at(lo);
      for (uint64_t p = lo + 1; p <= hi; ++p) {
        const uint64_t v = walk.at(p);
        if (v < c_hi) return "a trie pointer of order " + std::to_string(n - 1) + " decreases";
        c_hi = v;
      }
      if (c_hi > o.entries) return "a trie pointer of order " + std::to_string(n - 1) + " points past its array";
    }
    if (o.offsets) {
      if (o.n_offsets == 0 || ngram_trie_read(b, o.offsets) != 0) return "array-compressed pointers do not start at 0";
      for (uint64_t j = 1; j < o.n_offsets; ++j)
        if (ngram_trie_read(b, o.offsets + 64 * j) < ngram_trie_read(b, o.offsets + 64 * (j - 1)))
          return "array-compressed pointers out of order";
    }
    PointerWalk walk{b, parent, n == 2};
    uint64_t c = walk.at(lo);
    for (uint64_t p = lo; p < hi; ++p) {
      const uint64_t end = walk.at(p + 1);
      for (uint64_t first = c, prev_word = 0; c < end; ++c) {
        const uint64_t w = ngram_trie_field(b, o.bit + c * o.total_bits, o.word_bits);
        if (w >= bound) return "a trie word id of order " + std::to_string(n) + " is outside the vocabulary";
        if (c > first && w <= prev_word) return "trie words of order " + std::to_string(n) + " out of order";
        prev_word = w;
      }
    }
    lo = c_lo;
    hi = c_hi;
  }
  return "";
}

}  // namespace kenlm_detail

// Fills m from the KenLM binary file at path.  Returns "" on success, else the reason the file is refused.
static inline std::string load_kenlm_binary(const char *path, NgramModel &m) {
  using namespace kenlm_detail;
  File f;
  {
    FILE *fp = fopen(path, "rb");
    if (!fp) return "cannot open the file";
    unsigned char buf[1 << 16];
    size_t got;
    while ((got = fread(buf, 1, sizeof(buf), fp)) > 0) f.b.insert(f.b.end(), buf, buf + got);
    fclose(fp);
  }
  const uint64_t size = f.b.size();
  const std::string kb = "KenLM binary file: ";
  if (size >= strlen(kMagicIncomplete) && !memcmp(f.b.data(), kMagicIncomplete, strlen(kMagicIncomplete)))
    return kb + "the file did not finish building (\"incomplete\" magic)";
  if (size >= strlen(kMagicVersion) && !memcmp(f.b.data(), kMagicVersion, strlen(kMagicVersion))) {
    const char *v = reinterpret_cast<const char *>(f.b.data()) + strlen(kMagicVersion);
    const size_t room = std::min<uint64_t>(size - strlen(kMagicVersion), 8);
    const std::string digits(v, room);
    char *end = nullptr;
    const long version = strtol(digits.c_str(), &end, 10);
    if (end != digits.c_str() && version != 5)
      return kb + "format version " + std::to_string(version) + ", only version 5 is read";
  }
  if (size <= kSanityBytes + kFixedBytes)
    return kb + "truncated: " + std::to_string(size) + " bytes, too short for a header";
  {
    unsigned char want[kSanityBytes] = {0};
    memcpy(want, "mmap lm http://kheafield.com/code format version 5\n", 51);
    const float fl[3] = {0.0f, 1.0f, -0.5f};
    const uint32_t wi[3] = {1u, 0xffffffffu, 0u};
    const uint64_t one = 1;
    memcpy(want + 56, fl, 12);
    memcpy(want + 68, wi, 12);
    memcpy(want + 80, &one, 8);
    if (memcmp(want, f.b.data(), 51))
      return kb + "unrecognised header (not a version 5 binary)";
    if (memcmp(want, f.b.data(), kSanityBytes))
      return kb + "the header's test values do not match (built with another endianness or other type sizes)";
  }
  const int order = f.at<uint8_t>(kSanityBytes);
  const float multiplier = f.at<float>(kSanityBytes + 4);
  const int32_t type = f.at<int32_t>(kSanityBytes + 8);
  const bool has_vocabulary = f.at<uint8_t>(kSanityBytes + 12) != 0;
  const uint32_t search_version = f.at<uint32_t>(kSanityBytes + 16);
  if (type == kRestProbing) return kb + "REST_PROBING models (build_binary -r) are not supported";
  if (type < 0 || type > kQuantArrayTrie) return kb + "unknown model type " + std::to_string(type);
  const bool probing = type == kProbing;
  if (search_version != (probing ? 0u : 1u))
    return kb + "search version " + std::to_string(search_version) + " of model type " + std::to_string(type);
  if (order < 2) return kb + "order " + std::to_string(order) + ": at least a bigram model is needed";
  if (order > kNgramMaxOrder)
    return kb + "order " + std::to_string(order) + " is above " + std::to_string(kNgramMaxOrder);
  if (probing && !(multiplier >= 1.0f)) return kb + "probing multiplier below 1";
  const uint64_t header = align8(kSanityBytes + kFixedBytes + 8 * (uint64_t)order);
  if (size < header) return kb + "truncated: the header's counts are cut off";
  std::vector<uint64_t> counts(order);
  for (int n = 0; n < order; ++n) counts[n] = f.at<uint64_t>(kSanityBytes + kFixedBytes + 8 * n);
  if (!has_vocabulary) return kb + "the file has no vocabulary strings (build it without build_binary -s)";
  for (uint64_t c : counts)
    if (c >= (1ull << 40)) return kb + "an n-gram count of " + std::to_string(c) + " is implausible";

  // ---- region sizes from the counts (GenericModel::Size), checked against the file's length ----
  const uint64_t vocab_at = header;
  const uint64_t vocab_bytes = probing ? 8 + probing_buckets(counts[0], multiplier) * 12 : 8 + 8 * counts[0];
  const uint64_t search_at = vocab_at + vocab_bytes;
  uint64_t at = search_at;
  uint64_t uni_at = 0, probe_at[kNgramMaxOrder] = {}, buckets[kNgramMaxOrder] = {};
  // tries
  const bool quant = type == kQuantTrie || type == kQuantArrayTrie;
  const bool array = type == kArrayTrie || type == kQuantArrayTrie;
  uint8_t prob_bits = 0, backoff_bits = 0, bhiksha_bits = 0;
  PackedOrder packed[kNgramMaxOrder];
  if (probing) {
    uni_at = at;
    at += (counts[0] + 1) * 8;
    for (int n = 2; n <= order; ++n) {
      buckets[n - 1] = probing_buckets(counts[n - 1], multiplier);
      if (buckets[n - 1] > 0xffffffffull)  // (NgramView holds 32-bit bucket counts)
        return kb + "the " + std::to_string(n) + "-gram probing table has 2^32 buckets or more";
      probe_at[n - 1] = at;
      at += buckets[n - 1] * (n < order ? 16 : 12);
    }
  } else {
    if (quant) {
      if (size < search_at + 3) return kb + "truncated: the quantization header is cut off";
      const uint8_t version = f.at<uint8_t>(search_at);
      prob_bits = f.at<uint8_t>(search_at + 1);
      backoff_bits = f.at<uint8_t>(search_at + 2);
      if (version != 2) return kb + "quantization version " + std::to_string(version);
      if (prob_bits < 1 || prob_bits > 25 || backoff_bits < 1 || backoff_bits > 25)
        return kb + "quantization bits out of range";
      at += (uint64_t)(order - 2) * (((1ull << backoff_bits) + (1ull << prob_bits)) * 4) + (1ull << prob_bits) * 4 + 8;
    }
    uni_at = at;
    at += (counts[0] + 2) * 16;
    if (array && order > 2) {
      if (size < at + 2) return kb + "truncated: the pointer compression header is cut off";
      if (f.at<uint8_t>(at) != 0) return kb + "pointer compression version " + std::to_string(f.at<uint8_t>(at));
      bhiksha_bits = f.at<uint8_t>(at + 1);
    }
    for (int n = 2; n <= order; ++n)  // (the search keeps entry indices in 32 bits)
      if (counts[n - 1] >= (1ull << 32))
        return kb + "the " + std::to_string(n) + "-gram trie array has 2^32 entries or more";
    const uint8_t middle_bits = quant ? (uint8_t)(prob_bits + backoff_bits) : 63;
    for (int n = 2; n < order; ++n)
      at += middle_size(array, bhiksha_bits, middle_bits, counts[n - 1], counts[0], counts[n], &packed[n - 1], at);
    at += longest_size(quant ? prob_bits : 31, counts[order - 1], counts[0], &packed[order - 1], at);
  }
  if (size < at)
    return kb + "truncated: " + std::to_string(size) + " bytes, the counts need " + std::to_string(at) +
           " before the vocabulary strings";

  // ---- the vocabulary strings: "<unk>" first, then every word in id order, each NUL-terminated ----
  const uint64_t bound = probing ? f.at<uint32_t>(vocab_at + 4) : f.at<uint64_t>(vocab_at) + 1;
  if (probing && f.at<uint32_t>(vocab_at) != 0)
    return kb + "probing vocabulary version " + std::to_string(f.at<uint32_t>(vocab_at));
  if (bound != counts[0] && bound != counts[0] + 1)
    return kb + "the vocabulary has " + std::to_string(bound) + " words, the header counts " +
           std::to_string(counts[0]) + " unigrams";
  if (size - at < 6 || memcmp(f.b.data() + at, "<unk>", 6)) return kb + "no vocabulary strings after the n-grams";
  if (f.b.back() != 0) return kb + "truncated: the last vocabulary string is cut off";
  m.vocabulary.clear();
  m.word_id.clear();
  for (uint64_t p = at; p < size;) {
    const unsigned char *s = f.b.data() + p;
    const size_t len = strlen(reinterpret_cast<const char *>(s));
    m.vocabulary.emplace_back(reinterpret_cast<const char *>(s), len);
    p += len + 1;
  }
  if (m.vocabulary.size() != bound)
    return kb + "the file has " + std::to_string(m.vocabulary.size()) + " vocabulary strings, the header says " +
           std::to_string(bound);
  for (size_t id = 1; id < m.vocabulary.size(); ++id)
    if (!m.word_id.emplace(m.vocabulary[id], (int32_t)id).second)
      return kb + "duplicate word \"" + m.vocabulary[id] + "\"";
  if (!m.word_id.count("<s>")) return kb + "no <s> in the vocabulary";
  if (!m.word_id.count("</s>")) return kb + "no </s> in the vocabulary";
  m.order = order;

  if (probing) {
    m.layout = kNgramKenlmProbing;
    m.uni_prob.resize(bound);
    m.uni_backoff.resize(bound);
    for (uint64_t i = 0; i < bound; ++i) {
      m.uni_prob[i] = f.at<float>(uni_at + 8 * i);  // raw: the sign bit is KenLM's independent-left flag
      m.uni_backoff[i] = f.at<float>(uni_at + 8 * i + 4);
    }
    for (int n = 2; n <= order; ++n) {
      const uint64_t stride = n < order ? 16 : 12, bytes = buckets[n - 1] * stride;
      bool empty = false;
      for (uint64_t b = 0; b < buckets[n - 1] && !empty; ++b)
        empty = f.at<uint64_t>(probe_at[n - 1] + b * stride) == 0;
      if (!empty) return kb + "the " + std::to_string(n) + "-gram probing table has no empty bucket";
      m.probing[n - 1].assign((bytes + 7) / 8, 0);
      memcpy(m.probing[n - 1].data(), f.b.data() + probe_at[n - 1], bytes);
      m.buckets[n - 1] = (uint32_t)buckets[n - 1];
    }
  } else {
    // the search region, byte for byte: quantization header and bins, unigram records, and per order the offset array
    // (array tries) and the bit-packed entries
    m.layout = kNgramKenlmTrie;
    const uint64_t region = at - search_at;
    m.trie_bits.assign((region + 7) / 8 + 1, 0);
    memcpy(m.trie_bits.data(), f.b.data() + search_at, region);
    m.trie_orders.assign(order, NgramTrieOrder());
    m.trie_orders[0].bit = (uni_at - search_at) * 8;
    m.trie_orders[0].entries = bound;
    m.uni_prob.resize(bound);
    m.uni_backoff.resize(bound);
    for (uint64_t i = 0; i < bound; ++i) {
      m.uni_prob[i] = f.at<float>(uni_at + 16 * i);
      m.uni_backoff[i] = f.at<float>(uni_at + 16 * i + 4);
    }
    const uint64_t per_order = ((1ull << prob_bits) + (1ull << backoff_bits)) * 4;
    for (int n = 2; n <= order; ++n) {
      const PackedOrder &p = packed[n - 1];
      NgramTrieOrder &o = m.trie_orders[n - 1];
      o.bit = (p.base - search_at) * 8;
      o.entries = p.entries;
      o.word_bits = p.word_bits;
      o.quant_bits = p.quant_bits;
      o.inline_bits = p.inline_bits;
      o.total_bits = p.total_bits;
      if (array && n < order) {
        o.offsets = (p.offsets - search_at) * 8;
        o.n_offsets = p.n_offsets;
      }
      if (quant) {  // the bins after the 8-byte quantization header: per middle order prob then backoff, then the longest's
        o.prob_bits = prob_bits;
        o.backoff_bits = backoff_bits;
        o.prob_bins = (8 + (n - 2) * per_order) * 8;
        o.backoff_bins = o.prob_bins + (1ull << prob_bits) * 32;
      }
    }
    if (const std::string why = trie_validate(m, bound); !why.empty()) return kb + why;
  }
  m.is_character_based = ngram_character_based(m.vocabulary);
  ngram_build_front(m);
  return "";
}

// ARPA text or a KenLM binary file, told apart by the first bytes.  Returns "" on success, else the reason.
static inline std::string load_ngram_file(const char *path, NgramModel &m) {
  char head[sizeof(kenlm_detail::kMagicPrefix) - 1] = {0};
  size_t got = 0;
  if (FILE *fp = fopen(path, "rb")) {
    got = fread(head, 1, sizeof(head), fp);
    fclose(fp);
  }
  if (got == sizeof(head) && !memcmp(head, kenlm_detail::kMagicPrefix, sizeof(head))) return load_kenlm_binary(path, m);
  return load_arpa(path, m);
}

}  // namespace ctc

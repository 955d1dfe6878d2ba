// The per-utterance CTC prefix beam-search program: ONE CTA PER UTTERANCE, beams in shared memory.
//
// Replaces the reference's DecoderState::next / DecoderState::decode
// (reference ctc_beam_search_decoder.cpp:56-211), PathTrie (path_trie.cpp:38-163) and the
// std::nth_element prune (ctc_beam_search_decoder.cpp:149-160, decoder_utils.cpp:122-132).
// It is NOT a translation of that code.  The reference materialises beam x vocab trie nodes per
// frame, DFS-walks the whole trie and deletes all but beam_size of them; this program relies on
// the set-semantics of the algorithm (SURVEY.md Appendix A: every float field receives at most two
// commutative log_sum_exp contributions per frame, and unselected candidates leave no trace):
//
//   * the beam lives in shared-memory slot arrays (node id, last char, p_blank, p_nonblank, score);
//   * the beam x pruned-vocab candidates are never materialised -- a candidate's score is one
//     float add, recomputed on the fly;
//   * only candidates that survive the cut become nodes of a per-utterance arena in global memory
//     (16 bytes: parent, char, lpc, timestep).  The arena is WRITE-ONLY inside the frame loop: it is
//     read again only by the final backtrace (and by the rare "revive" slow path);
//   * what the reference finds by walking child vectors -- "which children of a beam member already
//     exist in the trie?" (path_trie.cpp:39-57) -- is kept in shared memory: every member knows the
//     slot of its parent if the parent is in the beam, and the only other existing children are
//     DEAD ANCHORS: dead nodes whose parent is in the beam and that still have a beam member below
//     them.  There are never more of those than beam members, so a K-entry table holds them, with
//     their lpc / timestep, so "timesteps" keeps the reference's arg-max-while-parent-in-beam
//     semantics (path_trie.cpp:41-46) including revival of dead interior nodes (path_trie.cpp:50-56);
//   * removal (path_trie.cpp:144-163) needs no cascade: a dead node is in the reference's trie iff
//     some member's nearest anchor is that node, which is a per-frame recount in shared memory;
//   * the top-beam_size cut is an exact radix select over 48-bit keys (ordered float score,
//     then smaller char first == prefix_compare) with shared-memory histograms.
//
// The source is written as barrier-separated parallel regions (CTC_PAR { ... } CTC_BARRIER();) so
// the very same text also compiles as a sequential single-threaded emulation for CPU logic tests
// (tests/native/emulate_cta.cpp, test infrastructure only -- the product never runs it).
#pragma once
#include <cfloat>
#include <cstdint>

#include "glibc_math.cuh"
#include "ngram_lm.h"

// CTC_PAR { ... }                 a parallel region over the NT threads of the CTA (variable `tid`)
// CTC_WARPS { ... CTC_LANES { ... } ... }   a warp-structured region: code directly inside CTC_WARPS is
//     warp-uniform (variable `warp`); CTC_LANES blocks run per lane (variables `lane`, `LX`); values that
//     cross a warp collective (ballot) live in CTC_LV arrays indexed by LX (one element per lane in the
//     emulation, a single register on the device).
#if defined(CTC_EMULATE)
// The emulation runs the "threads" of a region one after the other.  A region is only correct on the device if its
// result does not depend on that order, so the order is a test knob (ctc::g_emu_order, CTC_EMU_ORDER): bit 0 walks the
// warps of a region from the last to the first, bit 1 the lanes of a CTC_LANES block, bit 2 swaps the two halves of a
// CTC_HALVES region (two pieces of work that run concurrently on different warps of the device).
namespace ctc { static int g_emu_order = 0; constexpr int kLW = 32; }
#define CTC_PAR                                                                                                  \
  for (int tid_i_ = 0, tid = (::ctc::g_emu_order & 1) ? NT - 32 : 0; tid_i_ < NT;                                 \
       ++tid_i_, tid = (::ctc::g_emu_order & 1) ? ((NT / 32 - 1 - tid_i_ / 32) * 32 + (tid_i_ & 31)) : tid_i_)
#define CTC_WARPS                                                                                                \
  for (int warp_i_ = 0, warp = (::ctc::g_emu_order & 1) ? NT / 32 - 1 : 0; warp_i_ < NT / 32;                     \
       ++warp_i_, warp = (::ctc::g_emu_order & 1) ? NT / 32 - 1 - warp_i_ : warp_i_)
#define CTC_LANES                                                                                                \
  for (int lane_i_ = 0, lane = (::ctc::g_emu_order & 2) ? 31 : 0, LX = lane; lane_i_ < 32;                        \
       ++lane_i_, lane = (::ctc::g_emu_order & 2) ? 31 - lane_i_ : lane_i_, LX = lane)
#define CTC_HALVES for (int half_i_ = 0, half = (::ctc::g_emu_order & 4) ? 1 : 0; half_i_ < 2; ++half_i_, half ^= 1)
#define CTC_BARRIER() ((void)0)
#define CTC_SYNCWARP() ((void)0)
#define CTC_FN static inline
#define CTC_MFN inline
#else
#define CTC_PAR for (int tid = (int)threadIdx.x, once_ = 1; once_; once_ = 0)
#define CTC_WARPS for (int warp = (int)(threadIdx.x >> 5), once_w_ = 1; once_w_; once_w_ = 0)
#define CTC_LANES for (int lane = (int)(threadIdx.x & 31), LX = 0, once_l_ = 1; once_l_; once_l_ = 0)
#define CTC_HALVES for (int half = 0; half < 2; ++half)
#define CTC_BARRIER() __syncthreads()
#define CTC_SYNCWARP() __syncwarp()
#define CTC_FN __device__ __forceinline__
#define CTC_MFN __device__ __forceinline__
namespace ctc { constexpr int kLW = 1; }
#endif
#define CTC_LV(type, name) type name[::ctc::kLW]

namespace ctc {

// ---- status / flag bits reported per utterance (include/ctcdecode_b200.h mirrors these) --------
enum : int {
  FLAG_TIE_PRUNE = 1,   // comparator-equivalent prefixes straddled the beam cut (reference: unspecified)
  FLAG_TIE_FINAL = 2,   // comparator-equivalent prefixes adjacent in the final order
  FLAG_TIE_VOCAB = 4,   // equal probabilities straddled the cutoff_top_n / cutoff_prob cut
  FLAG_ERR_ARENA = 256, // node arena / anchor table exhausted (cannot happen with the documented sizing)
};

constexpr float kNInf = -FLT_MAX;  // reference NUM_FLT_INF negated (decoder_utils.h:12)
constexpr int kNBins = 256;
constexpr int kRowTrailer = 3;  // trailing floats of a pruned row: blank log-prob (no FLT_MIN), meta, max non-blank
constexpr int kNewFlag = 1 << 30;
// packed dictionary arc (lm_host.h pack_dictionary): the target state in the low bits, plus
constexpr int kDictFinal = 1 << 30;        // the target is a final state: the child restarts at the start state
constexpr int kDictSpace = 1 << 29;        // the state the child ends up in has an arc for the space label
constexpr int kDictStateMask = (1 << 29) - 1;  // in-frame marker: "parent slot refers to this frame's NEW occupant"

// Trie node in the global arena: what the final backtrace needs (reference path_trie.cpp:109-126), one 32-byte
// sector.  `jump` is the ancestor kJump levels further up the last multiple of kJump in depth: for a node of depth
// d >= 1 the ancestor of depth ((d - 1) / kJump) * kJump.  The backtrace of a prefix of length L is then L / kJump
// dependent hops along the jump pointers plus kJump hops inside each stretch, all stretches in parallel, instead of
// L dependent DRAM round trips (finalize_cta_run).
constexpr int kJump = 16;
struct alignas(32) Node {
  int parent;  // node index, -1 for the root
  int chr;     // character, -1 for the root
  float lpc;   // reference PathTrie::log_prob_c
  int ts;      // reference PathTrie::timestep
  int jump;    // node index of the checkpoint ancestor (unused for the root)
  int pad_[3];
};
// a new node's jump pointer from its parent's (node id, depth, jump)
CTC_HD int jump_of_child(int parent_node, int parent_depth, int parent_jump) {
  return (parent_depth % kJump == 0) ? parent_node : parent_jump;
}

// Per-utterance persistent state (global memory; survives between chunks of a streaming decode).
// Layout in ints: [0]=M (beam count) [1]=nnodes [2]=abs_t [3]=flags, then 12 slot arrays of K ints
// (node, chr, depth, bprev, nbprev, score, lpc, ts, pslot, anch, dstate, jump; floats by bit pattern) and the
// dead-anchor table, 6 arrays of 2*KP ints (dnode, dchr, dpslot, dlpc, dts, ddstate), KP = K rounded up to 32.
// dstate / ddstate (dictionary state of the scorer path) are 0 without a scorer.
constexpr int kStateHeader = 4;
constexpr int kSlotArrays = 12;
constexpr int kAnchorArrays = 6;
// KP: slots per slot array.  Beam sizes up to 256 round up to 32 / 64 / 128 / 256 -- the sizes the beam kernel is
// instantiated for with KP as a compile-time constant -- larger ones to a multiple of 32.
CTC_HD int kp_of(int K) { return K <= 32 ? 32 : K <= 64 ? 64 : K <= 128 ? 128 : K <= 256 ? 256 : (K + 31) / 32 * 32; }
CTC_HD long long state_ints(int K) { return kStateHeader + (long long)kSlotArrays * K + (long long)kAnchorArrays * 2 * kp_of(K); }

// ---- shared memory carve-up (bytes) ---------------------------------------------------------------
// Three parts: a fixed-size head (offsets are compile-time constants), the SLOT BLOCK -- every array whose length
// is a multiple of KP = beam size rounded up to 32, at offset kSmemHead + unit * KP * 4, so that with KP a
// template constant (beam_cta_run<..., KPT>) every slot-array address folds into the immediate field of the
// shared-memory instruction -- and a tail whose sizes depend on the pruned vocabulary / tile / thread count.
enum : int {  // head, bytes
  H_MBAR = 0, H_EXPTAB = 16, H_LOGTAB = H_EXPTAB + 32 * 8, H_HIST = H_LOGTAB + 32 * 8,
  H_WCNT = H_HIST + 2 * 256 * 4,  // 8 x 32 ints: per-warp list counts [0,32) / selected counts [32,64), and from 128
                                  // the per-warp score range of the new beam: [parity][min | max][warp]
  H_CTL = H_WCNT + 8 * 32 * 4, kSmemHead = H_CTL + 32 * 4 + 16 * 8
};
static_assert(kSmemHead % 16 == 0, "slot block alignment");
enum : int {  // slot block, in units of KP ints
  U_NODE = 0, U_CHR, U_DEPTH, U_BPREV, U_NBPREV, U_SCORE, U_LPC, U_TS,
  U_PSLOT,                // 2 units: double buffered links of the beam of frame t / t+1
  U_ANCH = U_PSLOT + 2,   // 2 units
  U_DSTATE = U_ANCH + 2, U_LMSP,
  U_DDSTATE,              // 2 units
  U_BNEW = U_DDSTATE + 2, U_NBNEW, U_SNEW, U_EVICT, U_SEL, U_SEL2, U_FREEL, U_FREEL2,
  U_NEWINFO,              // 11 units
  U_TIE = U_NEWINFO + 11, // 2 units
  U_DNODE = U_TIE + 2, U_DCHR = U_DNODE + 2, U_DPSLOT = U_DCHR + 2, U_DLPC = U_DPSLOT + 2, U_DTS = U_DLPC + 2,
  U_DREV = U_DTS + 2,     // dead-anchor table: 2 units each
  U_CNT2 = U_DREV + 2,    // 3 units
  U_AMAP = U_CNT2 + 3, U_SLOT2Q,
  U_STASH,                // 7 units: node, chr, lpc, ts, dstate, depth, jump of the members evicted in this frame
  U_EFREE = U_STASH + 7,  // 2 units
  U_RVWORK = U_EFREE + 2, // 3 units
  U_NODEN = U_RVWORK + 3, // node id / depth / jump pointer of a member committed by the barrier-free back half of a
  U_DEPTHN,               // frame, installed into U_NODE / U_DEPTH / U_JUMP by the slot owner at the start of the next
  U_JUMPN,                // frame (U_NODEN: -1 = nothing pending)
  U_JUMP,                 // jump pointer of the member's node (Node::jump)
  U_CODE,                 // 0xFFFF - (chr + 1) of the member as the frame started: the tie-break half of its 48-bit key,
                          // read by the barrier-free back half while slot owners already overwrite U_CHR
  U_SLOT_UNITS
};
CTC_HD int slot_off(int unit, int KP) { return kSmemHead + unit * KP * 4; }

struct SmemLayout {
  int evcnt, mask, mask2, rmask, dmask, rank, tile_lp, tile_idx, clk, cli;  // tail offsets
  int total;
  int KP, W, WC, NW, seg;
};
CTC_HD int align_up(int x, int a) { return (x + a - 1) / a * a; }
// budget_kb: shared memory one CTA may take so that the intended number of CTAs fits an SM (227 KB, 1 KB reserved
// per CTA): 111 = two per SM (default), 74 = three (plan.h picks it from the batch size).  Only the
// candidate-list segments give way; a segment that overflows costs that frame the grid-walking fallback.
CTC_HD SmemLayout make_layout(int K, int V, int NP, int tile_frames, bool sorted, int NT, bool lm = false,
                              int budget_kb = 111) {
  SmemLayout L;
  const int KP = kp_of(K);
  const int W = (NP + 31) / 32;
  const int NW = NT / 32;
  L.KP = KP;
  L.W = W;
  L.NW = NW;
  L.WC = (V + 31) / 32;
  int o = slot_off(U_SLOT_UNITS, KP);
  L.evcnt = o;     o += (KP / 32) * 4;
  // "existing child" masks: [KP][W] bits over pruned ranks (scorer path), [KP][WC] bits over CHARACTERS otherwise (the
  // masks of frame t+1 are built while frame t commits, when the frame's ranks are not known yet); rmask: ranks
  const int MWd = lm ? W : (L.WC > W ? L.WC : W);
  L.mask = o;      o += KP * MWd * 4;
  L.mask2 = o;     o += KP * MWd * 4;
  L.rmask = o;     o += KP * W * 4;
  L.dmask = o;     o += lm ? KP * L.WC * 4 : 0;   // scorer path: [KP][WC] dictionary arc bits
  L.rank = o;      o += sorted ? 2 * align_up(V * 2, 16) : 0;   // two rank tables: frame t+1's is built during frame t
  o = align_up(o, 128);
  L.tile_lp = o;   o += 2 * tile_frames * NP * 4;
  L.tile_idx = o;  o += sorted ? 2 * tile_frames * NP * 2 : 0;
  o = align_up(o, 16);
  // candidate-list segment per warp: room for every candidate of the members a warp owns, capped at 64 KB in
  // total -- and at what the budget leaves, if that is at least 8 KB
  int seg = ((K + NW - 1) / NW) * (NP - kRowTrailer);
  {
    int cap_bytes = budget_kb * 1024 - o - 64;
    if (cap_bytes > 64 * 1024) cap_bytes = 64 * 1024;
    if (cap_bytes < NW * 32 * 8) {  // not even minimal segments fit beside the intended number of CTAs per SM: one CTA
      cap_bytes = 227 * 1024 - o - 64;
      if (cap_bytes > 64 * 1024) cap_bytes = 64 * 1024;
    }
    if (seg > cap_bytes / 8 / NW) seg = cap_bytes / 8 / NW;
  }
  if (seg < 32) seg = 32;
  L.seg = seg;
  L.clk = o;       o += NW * seg * 4;
  L.cli = o;       o += NW * seg * 4;
  L.total = align_up(o, 16);
  return L;
}

// One language model of a scorer decode, with its weights: the LM slot a beam CTA decodes with.  BeamParams derives from
// it (after BeamCommon), so these fields of the kernel parameters are the call's model; a decode over several models (or weights) gives
// each CTA a slot of BeamParams::lm_slots instead (beam_program.cuh, lm_slot).  Everything else of the scorer path
// (space_id, dict_wc, lm_char) is call-wide.
struct LmSlot {
  const int *dict_next;             // [n_states][V]: -1 = no arc, else next state | kDictFinal | kDictSpace
  const uint32_t *dict_mask;        // [n_states][dict_wc]: bit c = the state has an arc for character c
  int dict_start;
  double beta;                      // Scorer::beta
  double lm_alpha;                  // Scorer::alpha: a term is float(cond_log_prob * alpha), as the host computes it
  // device n-gram scorer only
  NgramView ngram;                  // the model's tables in device memory
  const int *word_of_state;         // word-based: [n_states] the word a dictionary state completes with a space
  const int *label_word;            // character-based: [V] the word id of each label
  int lm_hist_n;                    // order - 1
  NgramFront front;                 // the read-out's front-end tables (labels' bytes, unigram spellings)
};

// The kernel parameters every decode has, at the start of BeamParams (the kernels without a scorer read nothing else).
struct BeamCommon {
  const float *lp;        // [B][T][NP] pruned float32 log-probs from the prune kernel
  const uint16_t *idx;    // [B][T][NP] character of each pruned entry, 0xFFFF = unused (sorted mode only)
  const int *seq_lens;    // [B] or nullptr
  int T, V, NP, K, blank;
  int t0, nframes;        // this launch consumes rows [t0, t0 + nframes) of each utterance (nframes <= 0: all T rows)
  int tile_frames;        // frames per staged tile
  SmemLayout L;           // shared-memory carve-up (make_layout), filled in by the launcher
  Node *arena;            // offline: base of B arenas
  long long arena_stride; // nodes per utterance
  int *state;             // offline: base of B state blocks (state_ints(K) ints each, see above)
  long long state_stride; // ints per utterance
  Node *const *arena_ptrs;  // streaming: per-utterance arena (overrides arena/arena_stride)
  int *const *state_ptrs;   // streaming: per-utterance state block
  const int *arena_caps;    // streaming: per-utterance arena capacity (nodes)
  int arena_cap;            // offline capacity per utterance
  int fresh;                // 1: start from the root state instead of loading `state`
  int force_fallback;       // test knob: run the grid-walking select path every frame
  int no_fast;              // test knob: never take the barrier-free back half of a frame
  float heur_bias;          // test knob: added to the checked heuristic bound (> 0 makes it fail its check often)
  const unsigned char *finalize;  // [B] or nullptr (= finalize all)
  int backtrace;          // 1: an index-order kernel without a scorer runs finalize_cta_run after its last frame itself
  int *out_tokens, *out_timesteps;  // [B][K][out_T]
  float *out_scores;                // [B][K]
  int *out_lens;                    // [B][K]
  int *n_results;                   // [B]
  int out_T;
  int *flags;  // [B], OR-ed
  long long *timing;  // optional [B][16]: cycles thread 0 spent between consecutive barriers, per region
};

struct BeamParams : BeamCommon, LmSlot {
  // ---- scorer path (word-based LM + dictionary, reference ctc_beam_search_decoder.cpp:74-82,93-95,120-137 and
  //      path_trie.cpp:59-96); everything below, and the LmSlot fields, are unused (0 / nullptr) when no scorer is
  //      attached
  int dict_wc;                      // words per mask row, ceil(V / 32)
  int space_id;                     // label of " ", -2 if there is none (reference :34-40)
  float *lm_arena;                 // [B][arena_stride]: per node float(cond_log_prob(make_ngram(node)) * alpha)
  int *dstate_arena;                // [B][arena_stride]: per node dictionary state
  // The exchange with the host's Scorer hook: two blocks per utterance in device-mapped pinned host memory, each
  // starting on its own 128-byte line (lm_nl_stride / lm_up_stride ints apart, lm_host.h exchange_strides):
  //   newlist  (device -> host)  [0] = number of entries, [1] = frames finished ("done" flag, persistent mode),
  //                              from [4]: 16-byte entries (node, parent, chr, needs_lm) per node created this frame
  //   lm_upd   (host -> device)  [0] = frames answered ("go" flag, persistent mode), [1] = number of pairs,
  //                              from [2]: (node, float bits of its LM term) pairs for the nodes of the last list
  int *newlist;
  const int *lm_upd;
  int lm_nl_stride, lm_up_stride;
  // persistent scorer mode: ONE launch for the whole utterance; after every frame the CTA publishes its new-node
  // list, raises the done flag and warp 0 polls the go flag's line until the host has answered.
  int lm_persistent;
  int lm_hs_last;                   // also hand shake after the LAST frame of the launch (streaming: a next chunk follows)
  float *const *lm_arena_ptrs;      // streaming: per-stream LM / dictionary-state arrays (else lm_arena + b * stride)
  int *const *dstate_ptrs;
  // character-based language models (reference scorer.cpp:148-161, ctc_beam_search_decoder.cpp:120-137 with
  // is_character_based()): no dictionary, and EVERY appended character takes an LM term -- which depends on the child,
  // so each node carries a row of V terms, float(cond_log_prob(prefix + c) * alpha), filled by the host when the node
  // is created: lm_row[(node) * V + c].  The update block then holds (node, V floats) entries.
  int lm_char;
  float *lm_row;                    // [B][arena_stride][V]
  float *const *lm_row_ptrs;        // streaming
  int *hs_abort;                    // [1] mapped host memory: host asks the kernel to stop waiting
  void (*emu_handshake)(void *ctx, int b);  // CPU emulation only: the host side of the handshake, called in place
  void *emu_ctx;
  // device n-gram scorer (an ARPA scorer, ngram_lm.h): the CTA computes the LM terms of the nodes it creates itself, so
  // there are no exchange blocks and no handshake (lm_persistent = 0, newlist / lm_upd unused)
  int lm_dev;
  int *lm_hist;                     // [B][arena_stride][lm_hist_stride] the node's last order - 1 LM word ids, oldest first
  // Per-CTA LM slots.  CTA g's slot index is s = lm_slot_of[g], or g / sweep_B without lm_slot_of (0 without either).
  // Its model and weights are lm_slots[s] (or the call's, the LmSlot fields above, without lm_slots), except that
  // lm_ab[s] = (alpha, beta) replaces the weights when lm_ab is set.
  //   sweep of the LM weights (ctcdec_decode_batch_lm_sweep_async): CTA g decodes input row g % sweep_B (lp, idx,
  //     seq_lens) with the call's model and the pair lm_ab[g / sweep_B]; everything else is indexed by g.  The slots
  //     of a sweep differ in their weights only, so its table holds just those, 16 bytes a pair.
  //   several models (ctcdec_decode_batch_lm_mixed_async): CTA g decodes input row g with lm_slots[lm_slot_of[g]].
  //     A CTA keeps its own lm_hist_n histories per node, lm_hist_stride ints apart: the slots' largest lm_hist_n
  //     (0: lm_hist_n).
  int sweep_B;
  const double *lm_ab;              // [P][2]
  const LmSlot *lm_slots;           // [S]
  const unsigned char *lm_slot_of;  // [B]
  int lm_hist_stride;
};

// control words: 32 ints in L.ctl
enum {
  C_M = 0, C_NNODES, C_FLAGS, C_NSEL, C_NFREE, C_NTIE, C_NREV, C_NPAIRS, C_ABOVE, C_BIN, C_CNT, C_KMIN, C_KMAX,
  C_SMAX, C_NEFREE, C_NETAKEN, C_NRVWORK, C_OVF, C_ANYREF, C_NLIVE, C_SMIN, C_NCAND,
  // second copies, used by frames of odd parity in kernels whose frames have no barrier between reading and
  // resetting these words (beam_program.cuh, "merged front / barrier-free back half")
  C_OVF_B, C_ANYREF_B, C_NPAIRS_B,
  // scorer kernels: the CTA's (alpha, beta) as two doubles in words [C_AB, C_AB + 4) (8-byte aligned: H_CTL is)
  C_AB = 26
};

// ---- small helpers --------------------------------------------------------------------------------
CTC_FN uint32_t ord_f(float x) {  // monotone float -> uint32 (larger float => larger key)
  uint32_t u = f_bits(x);
  return u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}
CTC_FN float unord_f(uint32_t o) { return bits_f((o & 0x80000000u) ? (o ^ 0x80000000u) : ~o); }
// prefix_compare as a key: score descending, then character ascending (decoder_utils.cpp:122-132)
CTC_FN uint64_t key64(float score, int chr) {
  return ((uint64_t)ord_f(score) << 16) | (uint64_t)(0xFFFF - (chr + 1));
}

#if defined(CTC_EMULATE)
template <class T> static inline T atom_add(T *p, T v) { T o = *p; *p = o + v; return o; }
static inline int atom_exch(int *p, int v) { int o = *p; *p = v; return o; }
static inline unsigned atom_sub_u(unsigned *p, unsigned v) { unsigned o = *p; *p = o - v; return o; }
static inline int atom_or(int *p, int v) { int o = *p; *p = o | v; return o; }
static inline unsigned atom_or(unsigned *p, unsigned v) { unsigned o = *p; *p = o | v; return o; }
template <class T> static inline T ld_cg(const T *p) { return *p; }
static inline void atom_max_i(int *p, int v) { if (v > *p) *p = v; }
#else
template <class T> CTC_FN T atom_add(T *p, T v) { return atomicAdd(p, v); }
CTC_FN int atom_exch(int *p, int v) { return atomicExch(p, v); }
CTC_FN unsigned atom_sub_u(unsigned *p, unsigned v) { return atomicSub(p, v); }
CTC_FN int atom_or(int *p, int v) { return atomicOr(p, v); }
CTC_FN unsigned atom_or(unsigned *p, unsigned v) { return atomicOr(p, v); }
template <class T> CTC_FN T ld_cg(const T *p) { return __ldcg(p); }
CTC_FN void atom_max_i(int *p, int v) { atomicMax(p, v); }
#endif

#if defined(CTC_EMULATE)
static inline unsigned ctc_ballot(const int (&pred)[kLW]) {
  unsigned b = 0;
  for (int l = 0; l < 32; ++l) b |= (pred[l] ? 1u : 0u) << l;
  return b;
}
static inline int ctc_popc(unsigned x) { return __builtin_popcount(x); }
static inline int ctc_ffs(unsigned x) { return __builtin_ffs((int)x); }
#else
CTC_FN unsigned ctc_ballot(const int (&pred)[kLW]) { return __ballot_sync(0xffffffffu, pred[0]); }
CTC_FN int ctc_popc(unsigned x) { return __popc(x); }
CTC_FN int ctc_ffs(unsigned x) { return __ffs((int)x); }
#endif
CTC_FN unsigned ctc_lt_mask(int lane) { return (1u << lane) - 1u; }
// position of the q-th (0-based) set bit of x; x has more than q bits set
CTC_FN int ctc_nth_bit(unsigned x, int q) {
#if defined(CTC_EMULATE)
  for (int b = 0; b < 32; ++b)
    if ((x >> b) & 1u) { if (q == 0) return b; --q; }
  return 0;
#else
  return (int)__fns(x, 0, q + 1);
#endif
}
// warp-wide maximum of one value per lane
#if defined(CTC_EMULATE)
static inline unsigned ctc_warp_max(const unsigned (&v)[kLW]) {
  unsigned m = 0;
  for (int l = 0; l < 32; ++l) m = v[l] > m ? v[l] : m;
  return m;
}
static inline unsigned ctc_warp_min(const unsigned (&v)[kLW]) {
  unsigned m = 0xFFFFFFFFu;
  for (int l = 0; l < 32; ++l) m = v[l] < m ? v[l] : m;
  return m;
}
#else
CTC_FN unsigned ctc_warp_max(const unsigned (&v)[kLW]) { return __reduce_max_sync(0xffffffffu, v[0]); }
CTC_FN unsigned ctc_warp_min(const unsigned (&v)[kLW]) { return __reduce_min_sync(0xffffffffu, v[0]); }
#endif

// one lane's 64-bit value to the whole warp
#if defined(CTC_EMULATE)
static inline uint64_t ctc_shfl64(const uint64_t (&v)[kLW], int src) { return v[src]; }
#else
CTC_FN uint64_t ctc_shfl64(const uint64_t (&v)[kLW], int src) {
  const unsigned lo = __shfl_sync(0xffffffffu, (unsigned)v[0], src), hi = __shfl_sync(0xffffffffu, (unsigned)(v[0] >> 32), src);
  return ((uint64_t)hi << 32) | lo;
}
#endif

// log_sum_exp<float> (reference decoder_utils.h:47-54) with the 32-entry expf / 16-entry logf tables
// staged in shared memory (a __constant__ table indexed per thread would serialise divergent reads).
CTC_FN float lse_smem(float x, float y, const uint64_t *exptab, const double *logtab) {
  if (x <= -FLT_MAX) return y;
  if (y <= -FLT_MAX) return x;
  const float m = x > y ? x : y;
  const float d = f_add(x > y ? y : x, -m);
  if (!(d >= -17.0f)) return f_add(0.0f, m);  // 1.0f + expf(d) == 1.0f, logf(1.0f) == 0
  const float s = f_add(1.0f, expf_glibc_t(d, exptab));
  return f_add(logf_glibc_t(s, logtab), m);
}

// Everything a region needs, by value (pointers into shared memory / this utterance's global state).
template <bool SORTED, bool LM>
struct Cta {
  // shared: beam slots
  int *s_node, *s_chr, *s_depth, *s_ts, *s_pslot, *s_anch, *s_dstate;
  float *s_bprev, *s_nbprev, *s_score, *s_lpc, *s_bnew, *s_nbnew, *s_snew, *s_lmsp;
  uint32_t *s_mask, *s_rmask;
  // shared: dead-anchor table (2*KP entries; dpslot < 0 = free)
  int *s_dnode, *s_dchr, *s_dpslot, *s_dts, *s_drev, *s_ddstate;
  float *s_dlpc;
  // shared: scratch
  int *s_evict, *s_sel, *s_sel2, *s_free, *s_free2, *s_newinfo, *s_tie, *s_cnt2, *s_amap, *s_efree,
      *s_rvwork, *s_hist, *s_ctl, *s_cli, *s_wcnt, *s_evcnt, *s_slot2q, *s_stash;
  uint32_t *s_clk;
  int16_t *s_rank;  // [V]
  const uint64_t *s_exptab;
  const double *s_logtab;
  // per frame
  const float *lp;      // [NP]
  const uint16_t *idx;  // [NP] (sorted mode)
  // global
  Node *nodes;
  int K, KP, V, NP, W, blank;
  int WS;      // words per member of s_mask
  bool mch;    // s_mask is indexed by character (kernels without a scorer), not by pruned rank
  // scorer path, per frame: prune everything under min_cutoff once the beam is full (reference :74-82,93-95)
  const int *dict_next;
  uint32_t *s_dmask;    // [KP][WC]: which characters the dictionary lets follow each member
  int WC;
  int space_id;
  const double *s_ab;      // this CTA's (alpha, beta) in s_ctl: its LM slot's, or its pair of a sweep
  bool lm_full;
  float lm_cutoff;
  bool lm_char;            // character-based model: no dictionary, an LM term per (member, character)
  const float *lm_row;     // this utterance's [node][V] terms

  CTC_MFN int chr_at(int r) const { return SORTED ? (int)idx[r] : r; }
  CTC_MFN int rank_of(int c) const { return SORTED ? (int)s_rank[c] : c; }
  // `if (full_beam && log_prob_c + prefix->score < min_cutoff) break;`  (reference :93-95)
  CTC_MFN bool dict_ok(int i, int c) const { return (s_dmask[i * WC + (c >> 5)] >> (c & 31)) & 1u; }
  CTC_MFN bool lm_cut(float l, float score) const { return LM && lm_full && f_add(l, score) < lm_cutoff; }
  // language model term when the appended character is the space (reference :120-137): log_p += score; log_p += beta
  CTC_MFN float lm_apply(float log_p, int i) const {
    const float a = f_add(log_p, s_lmsp[i]);
    return (float)d_add((double)a, s_ab[1]);
  }
  // does appending character ch to member i take a language-model term?  (reference :120: the space of a word-based
  // model, every character of a character-based one)
  CTC_MFN bool lm_scored(int ch) const { return ch == space_id || lm_char; }
  // the term itself: word-based -- the member's "prefix + space" term; character-based -- the row of the member's node
  CTC_MFN float lm_apply_c(float log_p, int i, int ch) const {
    const float term = lm_char ? ld_cg(&lm_row[(size_t)s_node[i] * V + ch]) : s_lmsp[i];
    const float a = f_add(log_p, term);
    return (float)d_add((double)a, s_ab[1]);
  }

  // Score of candidate (beam slot i) + (pruned entry r); false if it is not a new-prefix candidate.
  // (reference ctc_beam_search_decoder.cpp:108-118 with nb_cur == -inf => lse(-inf, log_p) = log_p)
  CTC_MFN bool cand(int i, int r, float &sc, int &c) const {
    c = chr_at(r);
    if (c == blank) return false;
    {  // that child is itself a beam member
      const int mb = mch ? c : r;
      if ((s_mask[i * WS + (mb >> 5)] >> (mb & 31)) & 1u) return false;
    }
    const float l = lp[r];
    if (LM) {
      if (lm_cut(l, s_score[i])) return false;
      // a child that does not exist yet needs a dictionary arc (reference path_trie.cpp:59-70); an existing dead
      // child (rmask) is found before the dictionary is consulted (path_trie.cpp:39-57)
      if (!lm_char && !((s_rmask[i * W + (r >> 5)] >> (r & 31)) & 1u) && !dict_ok(i, c)) return false;
    }
    if (c == s_chr[i]) {
      const float b = s_bprev[i];
      sc = (b > kNInf) ? f_add(l, b) : kNInf;
    } else {
      sc = f_add(l, s_score[i]);
    }
    if (LM && lm_scored(c)) sc = lm_apply_c(sc, i, c);
    return true;
  }
};

}  // namespace ctc

// The CTA program itself: barrier-separated parallel regions over the structures of beam_core.cuh.
// Included by ctc_kernels.cu (device build) and tests/native/emulate_cta.cpp (CTC_EMULATE, test only).
#pragma once
#include "beam_core.cuh"
#if defined(CTC_EMULATE)
#include <cstdio>   // (the emulation's histogram check)
#include <cstdlib>
#endif

// compile-time switches of the barrier-free back half (tools/build_variants.sh builds A/B variants with -D...).
// The frame loop is bound by its INSTRUCTION FOOTPRINT: each of these features is a win on paper but adds code to the
// loop, and they made the kernel slower in proportion to the code they added.  They are OFF by default and kept,
// tested, for A/B measurements.  (Moving the rarely taken general back half out of line with __noinline__ is worse
// still: the ABI call forces the slot-array pointers and the frame's scalars through local memory.)
#ifndef CTC_OPT_FAST2
#define CTC_OPT_FAST2 0     // rank the keys of a shared K-th-key bin instead of taking the general back half
#endif
#ifndef CTC_OPT_HEADOFF
#define CTC_OPT_HEADOFF 0   // a grid-walking warp computes the next frame's key range while the owners commit
#endif
#ifndef CTC_OPT_BITSCAN
#define CTC_OPT_BITSCAN 0   // histogram suffix sums from eight ballots instead of five dependent shuffles
#endif
#ifndef CTC_OPT_CH
#define CTC_OPT_CH 1        // 32-entry chunks of a list segment the barrier-free back half accepts
#endif
#ifndef CTC_OPT_ROWS2
#define CTC_OPT_ROWS2 0     // grid walk: the two-rows-per-iteration / two-column-group variants of the row loop
#endif
#ifndef CTC_OPT_EXPECT
#define CTC_OPT_EXPECT 0    // branch-probability hints on the rare paths
#endif
#if CTC_OPT_EXPECT && !defined(CTC_EMULATE)
#define CTC_LIKELY(x) __builtin_expect(!!(x), 1)
#define CTC_UNLIKELY(x) __builtin_expect(!!(x), 0)
#else
#define CTC_LIKELY(x) (x)
#define CTC_UNLIKELY(x) (x)
#endif

namespace ctc {

// ---- device n-gram scorer (BeamParams::lm_dev): the LM terms of a node, computed by the thread that creates it -----
// A node keeps the last order - 1 LM word ids of its prefix (oldest first, "<s>"-padded like Scorer::make_ngram).  A
// child through the space label shifts in the word its parent's dictionary state completes; in a character-based model
// every child shifts in its character's word id; any other child keeps its parent's history.  The terms are those the
// host hooks give (lm_host.h lm_after_frame / lm_char_row): float(cond_log_prob * alpha) of history + the node's word
// (word-based, when a space can follow the node) or of history + each label (character-based, the node's row).
// m: the CTA's LM slot (its model); alpha: the CTA's weight (the slot's, or its pair of a sweep).  hist: the CTA's
// histories, m.lm_hist_n ints per node.
CTC_FN float lm_dev_term(const LmSlot &m, double alpha, int *ids, int word) {
  ids[m.lm_hist_n] = word;
  return (float)(ngram_cond_ids(m.ngram, ids, m.lm_hist_n + 1) * alpha);
}

CTC_FN void lm_dev_root_term(const LmSlot *mp, double alpha, float *lm_row, int c) {
  const LmSlot &m = *mp;
  int ids[kNgramMaxOrder];
  for (int k = 0; k < m.lm_hist_n; ++k) ids[k] = m.ngram.bos;
  lm_row[c] = lm_dev_term(m, alpha, ids, m.label_word[c]);
}

CTC_FN void lm_dev_node(const BeamParams &p, const LmSlot *mp, double alpha, int *hist, float *lm_arena, float *lm_row,
                        int nid, int par, int ch, int par_state, int arc, int dst) {
  const LmSlot &m = *mp;
  const int H = m.lm_hist_n;
  int ids[kNgramMaxOrder];
  const int *hp = hist + (size_t)par * H;
  const bool shift = p.lm_char || ch == p.space_id;
  for (int k = 0; k < H; ++k) ids[k] = shift ? (k + 1 < H ? hp[k + 1] : 0) : hp[k];
  if (shift) ids[H - 1] = p.lm_char ? m.label_word[ch] : m.word_of_state[par_state];
  for (int k = 0; k < H; ++k) hist[(size_t)nid * H + k] = ids[k];
  if (p.lm_char) {
    for (int c = 0; c < p.V; ++c) lm_row[(size_t)nid * p.V + c] = lm_dev_term(m, alpha, ids, m.label_word[c]);
  } else if (arc & kDictSpace) {
    lm_arena[nid] = lm_dev_term(m, alpha, ids, m.word_of_state[dst]);
  }
}

// The LM slot of beam CTA b (BeamParams::lm_slots): its index, and its model -- a slot of the table, or the call's
// model in the kernel parameters (a __grid_constant__ parameter: its address is taken without a local copy).
CTC_FN int lm_slot_index(const BeamParams &p, int b) {
  return p.lm_slot_of ? (int)p.lm_slot_of[b] : p.sweep_B ? b / p.sweep_B : 0;
}
CTC_FN const LmSlot *lm_slot(const BeamParams &p, int s) {
  return p.lm_slots ? p.lm_slots + s : static_cast<const LmSlot *>(&p);
}

#if defined(CTC_EMULATE) && defined(CTC_STATS)
struct EmuStats { long long frames, passes, walk_iters, anchors_live, evicted, anchors_new, rv_hops, created, revived,
                  hist_adds, tie_frames, sel_all_frames, rv_frames, rows, rows_skipped, cl_entries, rewalks, fb_frames, ovf_first, heur_fail,
                  fast_frames, nf_anchor, nf_notfull, nf_seg, nf_pass, nf_pass_cnt, fast2_frames; };
static EmuStats g_stats;
#define CTC_STAT(x) (x)
#else
#define CTC_STAT(x) ((void)0)
#endif

// one count into a radix histogram of kNBins ints.  A key outside the range the bins were laid over would index past
// the histogram -- on the device an out-of-bounds shared-memory atomic -- so the CPU emulation checks every bin and
// stops the decode with a message.
#if defined(CTC_EMULATE)
static inline void emu_hist_add(int *hist, unsigned long long bin, const char *file, int line) {
  if (bin >= (unsigned long long)kNBins) {
    fprintf(stderr, "%s:%d: radix histogram bin %llu out of range [0, %d)\n", file, line, bin, kNBins);
    abort();
  }
  ++hist[bin];
}
#define CTC_HIST_ADD(hist, bin) emu_hist_add((hist), (bin), __FILE__, __LINE__)
#else
#define CTC_HIST_ADD(hist, bin) atom_add(&(hist)[(int)(bin)], 1)
#endif

#if defined(CTC_EMULATE)
#define CTC_TICK(id) ((void)0)
#define CTC_BARRIER_T(id) CTC_BARRIER()
#else
// a barrier that also accounts, per warp, the cycles between leaving the previous such barrier and arriving at
// this one (TIMING instantiations only): shows which warp each region waits for
#define CTC_BARRIER_T(id)                                                   \
  do {                                                                      \
    if (TIMING && (threadIdx.x & 31) == 0) s_wbusy[(id) * 32 + (threadIdx.x >> 5)] += clock64() - w_last; \
    __syncthreads();                                                        \
    if (TIMING) w_last = clock64();                                         \
  } while (0)
// per-region cycle accounting by thread 0 (TIMING instantiations only; tools/region_timing.py)
#define CTC_TICK(id)                                                        \
  do {                                                                      \
    if (TIMING && threadIdx.x == 0) {                                       \
      const long long now_ = clock64();                                     \
      s_tick[id] += now_ - s_tick[15];                                      \
      s_tick[15] = now_;                                                    \
    }                                                                       \
  } while (0)
#endif

#if !defined(CTC_EMULATE)
// ---- TMA (cp.async.bulk) + mbarrier plumbing for the staged [tile_frames x NP] log-prob tiles -------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n"
      " bra WAIT_%=;\n DONE_%=:\n}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
#endif

// One pass of the radix select ends here: given the histogram of keys in [lo, lo + width) binned by
// (key - lo) >> shift, find the bin holding the need-th largest key.  Executed by warp 0 (device) /
// once (emulation).  Writes ctl: C_BIN, C_ABOVE(+=), C_CNT.
template <int NT>
CTC_FN void scan_find_bin(const int *hist, int need, int *s_ctl, int tid) {
#if defined(CTC_EMULATE)
  if (tid != 0) return;
  int a = 0;
  for (int bb = kNBins - 1; bb >= 0; --bb) {
    if (a + hist[bb] >= need) {
      s_ctl[C_BIN] = bb;
      s_ctl[C_ABOVE] += a;
      s_ctl[C_CNT] = hist[bb];
      return;
    }
    a += hist[bb];
  }
  s_ctl[C_BIN] = 0;  // unreachable when the invariants hold
  s_ctl[C_CNT] = hist[0];
#else
  if (tid >= 32) return;
  constexpr int PER = kNBins / 32;
  const int top = kNBins - 1 - PER * tid;  // this lane owns bins top, top-1, ..., top-PER+1
  int h[PER];
  int sum = 0;
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    h[q] = hist[top - q];
    sum += h[q];
  }
  int incl = sum;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, d);
    if (tid >= d) incl += v;
  }
  const unsigned ball = __ballot_sync(0xffffffffu, incl >= need);
  const int owner = ball ? (__ffs(ball) - 1) : 31;
  if (tid == owner) {
    int a = incl - sum;
    int bin = top - PER + 1, cnt = h[PER - 1];
    bool found = false;
#pragma unroll
    for (int q = 0; q < PER; ++q) {
      if (!found) {
        if (a + h[q] >= need) {
          bin = top - q;
          cnt = h[q];
          found = true;
        } else {
          a += h[q];
        }
      }
    }
    s_ctl[C_BIN] = bin;
    s_ctl[C_ABOVE] += a;
    s_ctl[C_CNT] = cnt;
  }
#endif
}

// Same search, executed redundantly by EVERY warp (device) so that no barrier / broadcast is needed afterwards.
CTC_FN void scan_bin_all(const int *hist, int need, int &bin, int &above, int &cnt) {
#if defined(CTC_EMULATE)
  int a = 0;
  for (int bb = kNBins - 1; bb >= 0; --bb) {
    if (a + hist[bb] >= need) { bin = bb; above = a; cnt = hist[bb]; return; }
    a += hist[bb];
  }
  bin = 0; above = a - hist[0]; cnt = hist[0];  // unreachable when the invariants hold
#else
  // lane l owns the 8 consecutive bins [8 l, 8 l + 8) (two 16-byte loads): sums them, the 32 lane totals go through
  // a 5-step suffix scan (lanes above = higher keys), a ballot finds the lane the need-th key falls into, that
  // lane's 8 bins are walked from the top, and three shuffles broadcast the answer.
  static_assert(kNBins == 256, "8 bins per lane");
  const int lane = (int)(threadIdx.x & 31);
  const int4 ha = *reinterpret_cast<const int4 *>(hist + 8 * lane), hb = *reinterpret_cast<const int4 *>(hist + 8 * lane + 4);
  const int h[8] = {ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w};
  const int tot = ((h[0] + h[1]) + (h[2] + h[3])) + ((h[4] + h[5]) + (h[6] + h[7]));
  // sfx = the sum of tot over lanes >= this lane.  The lane totals are small (a beam plus a few candidates over 256
  // bins), so the suffix sums are assembled from eight INDEPENDENT ballots, one per bit of tot, instead of a chain of
  // five dependent shuffles; a lane total above 255 (degenerate key distributions) takes the shuffle scan.
  int sfx;
  if (CTC_OPT_BITSCAN && __ballot_sync(0xffffffffu, tot > 255) == 0u) {
    const unsigned ge = 0xFFFFFFFFu << lane;
    sfx = 0;
#pragma unroll
    for (int pbit = 0; pbit < 8; ++pbit)
      sfx += __popc(__ballot_sync(0xffffffffu, (tot >> pbit) & 1) & ge) << pbit;
  } else {
    sfx = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int v = __shfl_down_sync(0xffffffffu, sfx, d);
      if (lane + d < 32) sfx += v;
    }
  }
  const unsigned ball = __ballot_sync(0xffffffffu, sfx >= need);  // lanes <= target
  const int target = ball ? 31 - __clz((int)ball) : 0;
  // walk this lane's bins from the top (only the target lane's result is used)
  int a = sfx - tot, q_hit = 0, a_hit = a, c_hit = h[0];
  bool found = false;
#pragma unroll
  for (int q = 7; q >= 0; --q) {
    const bool hit = !found && (a + h[q] >= need);
    if (hit) { q_hit = q; a_hit = a; c_hit = h[q]; found = true; }
    a += h[q];
  }
  if (!found) a_hit = a - h[0];  // unreachable when the invariants hold (mirrors the sequential version)
  bin = __shfl_sync(0xffffffffu, 8 * lane + q_hit, target);
  above = __shfl_sync(0xffffffffu, a_hit, target);
  cnt = __shfl_sync(0xffffffffu, c_hit, target);
#endif
}

// 32-bit block max / min into a shared word (device: hardware warp redux + one atomic per warp).
CTC_FN void red_max_u32(unsigned *dst, unsigned v) {
#if defined(CTC_EMULATE)
  if (v > *dst) *dst = v;
#else
  v = __reduce_max_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) atomicMax(dst, v);
#endif
}
CTC_FN void red_min_u32(unsigned *dst, unsigned v) {
#if defined(CTC_EMULATE)
  if (v < *dst) *dst = v;
#else
  v = __reduce_min_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) atomicMin(dst, v);
#endif
}

// Per-warp minimum / maximum of a key into dst[warp] / dst[32 + warp] (plain stores, no contention); whoever needs
// the block-wide range reduces the NW pairs (warp_range_load).  Every thread of the CTA must call it.
CTC_FN void warp_range_store(int *dst, unsigned mn, unsigned mx, int tid) {
#if defined(CTC_EMULATE)
  unsigned *d = (unsigned *)dst;
  const int w = tid >> 5;
  if ((tid & 31) == 0) { d[w] = 0xFFFFFFFFu; d[32 + w] = 0u; }
  if (mn < d[w]) d[w] = mn;
  if (mx > d[32 + w]) d[32 + w] = mx;
#else
  mn = __reduce_min_sync(0xffffffffu, mn);
  mx = __reduce_max_sync(0xffffffffu, mx);
  // every lane stores (same value, same word: one broadcast write).  Not `if (lane == 0)`: nvcc 12.9 folded
  // (tid >> 5) * 4 into tid >> 3 under that predicate and then reused the address where all lanes run.
  dst[tid >> 5] = (int)mn;
  dst[32 + (tid >> 5)] = (int)mx;
#endif
}
template <int NW>
CTC_FN void warp_range_load(const int *src, unsigned &mn, unsigned &mx) {
  mn = 0xFFFFFFFFu; mx = 0u;
#pragma unroll
  for (int w = 0; w < NW; ++w) {
    const unsigned a = (unsigned)src[w], b = (unsigned)src[32 + w];
    mn = a < mn ? a : mn;
    mx = b > mx ? b : mx;
  }
}

CTC_FN Node load_node(const Node *p) {
#if defined(CTC_EMULATE)
  return *p;
#else
  const int4 a = __ldcg(reinterpret_cast<const int4 *>(p));  // nodes are written by this CTA: read through L2
  Node n;
  n.parent = a.x; n.chr = a.y; n.lpc = __int_as_float(a.z); n.ts = a.w;
  n.jump = __ldcg(&p->jump);  // (same 32-byte sector)
  return n;
#endif
}
CTC_FN void store_node(Node *p, const Node &n) {
#if defined(CTC_EMULATE)
  *p = n;
#else
  // st.global.cg: the arena is write-only here (no L1 allocation), and a GLOBAL store cannot alias the shared-memory
  // slot arrays (a generic one could, and makes the compiler reload them after every node store)
  __stcg(reinterpret_cast<int4 *>(p), make_int4(n.parent, n.chr, __float_as_int(n.lpc), n.ts));
  __stcg(&p->jump, n.jump);
#endif
}
// 16-byte entry of the new-node list the scorer path hands to the host (device-mapped host memory: one store)
struct alignas(16) Entry16 { int a, b, c, d; };
CTC_FN void store_entry16(int *dst, const Entry16 &e) {
#if defined(CTC_EMULATE)
  dst[0] = e.a; dst[1] = e.b; dst[2] = e.c; dst[3] = e.d;
#else
  *reinterpret_cast<int4 *>(dst) = make_int4(e.a, e.b, e.c, e.d);
#endif
}
CTC_FN void flush_lpc_ts(Node *p, float lpc, int ts) {
#if defined(CTC_EMULATE)
  p->lpc = lpc; p->ts = ts;
#else
  __stcg(reinterpret_cast<int2 *>(&p->lpc), make_int2(__float_as_int(lpc), ts));
#endif
}

template <int NT>
CTC_FN void finalize_cta_run(const BeamParams &p, const int b, unsigned char *smem);

// ======================================================================================================
//  beam_cta_run: consume frames [0, Tb) of utterance b, leave the beam state in global memory.
// ======================================================================================================
// KPT: beam size rounded up to 32 as a compile-time constant (0 = taken from p.K at run time); with KPT > 0 every
// slot-array address is an immediate offset.  TIMING: per-region cycle counters (tools/region_timing.py).
template <int NT, bool SORTED, bool LM, int KPT = 0, bool TIMING = false>
CTC_FN void beam_cta_run(const BeamParams &p, const int b, unsigned char *smem) {
  const int K = p.K, V = p.V, NP = p.NP, F = p.tile_frames;
  const SmemLayout &L = p.L;  // computed by the host (plan.h): constant-bank reads, nothing to recompute per frame
  constexpr int NW = NT / 32;
  const int KP = KPT > 0 ? KPT : L.KP;
  const int W = L.W, KP2 = 2 * KP, SEG = L.seg;
  // MERGED (kernels without a scorer): a frame is TWO barrier-separated regions on the common path.
  //   front: the members' terms (region R1) and the grid walk (region G) run side by side -- on different warps where
  //          the CTA has more warps than the beam has 32-slot blocks (WB0 = first grid-walking warp, NB of them),
  //          one after the other inside each warp otherwise.  That needs the "existing child" masks before the frame
  //          starts: indexed by CHARACTER they depend on the beam's links only, so the commit of frame t-1
  //          builds them (double buffered by frame parity, like the first radix histogram and the words of s_ctl
  //          that are read right after a barrier and reset in the same region).
  //   back:  FASTB -- every warp redundantly finds the K-th key and classifies ALL members / list entries into
  //          ballot words it keeps in registers, so the slot owners commit the new beam without another barrier.
  //          Frames that need more (dead anchors in the table, beam not full, a second radix pass, ties, list
  //          overflow) take the general back half below, unchanged.
  // (cut-vocabulary kernels CAN run the two-region frame -- masks by character, rank table built a frame ahead; the
  //  code is below and passes the same tests -- but on config 4 (beam 200: all eight warps own slots, so every
  //  warp repeats the whole classification) it is slower than the five-region frame)
  constexpr bool MERGED = !LM && !SORTED;
  constexpr int KPW = KPT / 32;
  constexpr bool FASTB = MERGED && KPT > 0 && KPT <= NT && KPW <= 8;
  constexpr int WB0 = (MERGED && KPT > 0 && KPW < NW) ? KPW : 0;
  constexpr int NB = NW - WB0;
  constexpr int CH = CTC_OPT_CH;  // 32-entry chunks of a list segment the barrier-free back half looks at (the second one rarely)
  // FAST2: a frame whose K-th key shares its histogram bin with other keys stays in the barrier-free back half when
  // that bin holds at most 32 keys: every warp ranks them among themselves (64 scratch words per warp: the
  // general path's selection lists, unused in such a frame)
  constexpr bool FAST2 = CTC_OPT_FAST2 && FASTB && 4 * KPT >= NW * 64;

  Cta<SORTED, LM> c;
#define CTC_SLOT(type, unit) ((type *)(smem + slot_off(unit, KP)))
  c.s_node = CTC_SLOT(int, U_NODE);        c.s_chr = CTC_SLOT(int, U_CHR);
  c.s_depth = CTC_SLOT(int, U_DEPTH);      c.s_bprev = CTC_SLOT(float, U_BPREV);
  c.s_nbprev = CTC_SLOT(float, U_NBPREV);  c.s_score = CTC_SLOT(float, U_SCORE);
  c.s_lpc = CTC_SLOT(float, U_LPC);        c.s_ts = CTC_SLOT(int, U_TS);
  c.s_pslot = CTC_SLOT(int, U_PSLOT);      c.s_anch = CTC_SLOT(int, U_ANCH);
  c.s_dstate = CTC_SLOT(int, U_DSTATE);    c.s_lmsp = CTC_SLOT(float, U_LMSP);
  c.s_ddstate = CTC_SLOT(int, U_DDSTATE);
  c.s_bnew = CTC_SLOT(float, U_BNEW);      c.s_nbnew = CTC_SLOT(float, U_NBNEW);
  c.s_snew = CTC_SLOT(float, U_SNEW);      c.s_mask = (uint32_t *)(smem + L.mask);
  c.s_rmask = (uint32_t *)(smem + L.rmask);  c.s_evict = CTC_SLOT(int, U_EVICT);
  c.s_sel = CTC_SLOT(int, U_SEL);          c.s_sel2 = CTC_SLOT(int, U_SEL2);
  c.s_free = CTC_SLOT(int, U_FREEL);       c.s_free2 = CTC_SLOT(int, U_FREEL2);
  c.s_newinfo = CTC_SLOT(int, U_NEWINFO);  c.s_tie = CTC_SLOT(int, U_TIE);
  c.s_dnode = CTC_SLOT(int, U_DNODE);      c.s_dchr = CTC_SLOT(int, U_DCHR);
  c.s_dpslot = CTC_SLOT(int, U_DPSLOT);    c.s_dlpc = CTC_SLOT(float, U_DLPC);
  c.s_dts = CTC_SLOT(int, U_DTS);          c.s_drev = CTC_SLOT(int, U_DREV);
  c.s_cnt2 = CTC_SLOT(int, U_CNT2);        c.s_amap = CTC_SLOT(int, U_AMAP);
  c.s_efree = CTC_SLOT(int, U_EFREE);
  c.s_rvwork = CTC_SLOT(int, U_RVWORK);    c.s_hist = (int *)(smem + H_HIST);
  c.s_rank = (int16_t *)(smem + L.rank);   c.s_ctl = (int *)(smem + H_CTL);
  c.s_clk = (uint32_t *)(smem + L.clk);    c.s_cli = (int *)(smem + L.cli);
  c.s_wcnt = (int *)(smem + H_WCNT);       c.s_evcnt = (int *)(smem + L.evcnt);
  c.s_slot2q = CTC_SLOT(int, U_SLOT2Q);    c.s_stash = CTC_SLOT(int, U_STASH);
  int *const pslot_base = CTC_SLOT(int, U_PSLOT), *const anch_base = CTC_SLOT(int, U_ANCH);
  int *const s_nodeN = CTC_SLOT(int, U_NODEN), *const s_depthN = CTC_SLOT(int, U_DEPTHN);
  int *const s_jumpN = CTC_SLOT(int, U_JUMPN), *const s_jump = CTC_SLOT(int, U_JUMP);
  int *const s_code = CTC_SLOT(int, U_CODE);
  const int WS = MERGED ? (L.WC > W ? L.WC : W) : W;  // words per member of the "existing child" masks
  const int VR = SORTED ? align_up(V * 2, 16) / 2 : 0;  // entries of one rank table
  int16_t *const rank_base = (int16_t *)(smem + L.rank);
  uint32_t *const mask_buf0 = (uint32_t *)(smem + L.mask), *const mask_buf1 = (uint32_t *)(smem + L.mask2);
  int cur = 0;  // which half of the double-buffered link arrays describes the current beam
  int par = 0;  // frame parity: which C_CMIN / C_CMAX pair holds the current beam's score range
  c.s_exptab = (uint64_t *)(smem + H_EXPTAB);
  c.s_logtab = (double *)(smem + H_LOGTAB);
  c.K = K; c.KP = KP; c.V = V; c.NP = NP; c.W = W; c.blank = p.blank;
  c.WS = WS; c.mch = MERGED;
  c.s_dmask = (uint32_t *)(smem + L.dmask); c.WC = L.WC;
  // the CTA's LM slot: its model, read where a node or member needs it, and its (alpha, beta) -- the slot's, or its pair
  // of a sweep -- read once, at the start, into s_ab; in a sweep also the input row of this CTA
  const int bi = LM && p.sweep_B ? b % p.sweep_B : b;
  const int lm_si = LM ? lm_slot_index(p, b) : 0;
  const LmSlot *const lm = LM ? lm_slot(p, lm_si) : nullptr;
  // (inside the frame loop the slot is found again where a node needs it: no pointer stays live across frames)
  auto cta_slot = [&]() { return lm_slot(p, lm_slot_index(p, b)); };
  const double *const lm_pair = LM && p.lm_ab ? p.lm_ab + 2 * lm_si : nullptr;
  c.dict_next = LM ? lm->dict_next : nullptr; c.space_id = p.space_id; c.lm_full = false; c.lm_cutoff = kNInf;
  c.s_ab = (const double *)(smem + H_CTL + C_AB * 4);
  c.lm_char = LM && p.lm_char != 0; c.lm_row = nullptr;
  int *const s_ctl = c.s_ctl;
#if !defined(CTC_EMULATE)
  long long *const s_tick = (long long *)(smem + H_CTL + 32 * 4);
  if (TIMING && threadIdx.x == 0) {
    for (int x = 0; x < 15; ++x) s_tick[x] = 0;
    s_tick[15] = clock64();
  }
  long long *const s_wbusy = (long long *)(smem + L.total);  // [16][32], TIMING launches add 4 KB for it
  long long w_last = 0;
  if (TIMING) {
    for (int x = threadIdx.x; x < 16 * 32; x += NT) s_wbusy[x] = 0;
    w_last = clock64();
  }
#endif

  Node *const nodes = p.arena_ptrs ? p.arena_ptrs[b] : p.arena + (long long)b * p.arena_stride;
  int *const st = p.state_ptrs ? p.state_ptrs[b] : p.state + (long long)b * p.state_stride;
  const int arena_cap = p.arena_caps ? p.arena_caps[b] : p.arena_cap;
  c.nodes = nodes;
  float *const lm_arena = !LM ? nullptr : p.lm_arena_ptrs ? p.lm_arena_ptrs[b] : p.lm_arena + (long long)b * p.arena_stride;
  int *const dstate_arena = !LM ? nullptr : p.dstate_ptrs ? p.dstate_ptrs[b] : p.dstate_arena + (long long)b * p.arena_stride;
  float *const lm_row = !(LM && p.lm_char) ? nullptr
                        : p.lm_row_ptrs ? p.lm_row_ptrs[b] : p.lm_row + (size_t)b * (size_t)p.arena_stride * (size_t)V;
  c.lm_row = lm_row;
  int *const newlist = LM && !p.lm_dev ? p.newlist + (long long)b * p.lm_nl_stride : nullptr;
  const int *const lm_upd = LM && !p.lm_dev ? p.lm_upd + (long long)b * p.lm_up_stride : nullptr;
  // (a streaming state keeps its histories behind its LM terms, in the same allocation: lm_arena[arena_cap ...])
  int *const lm_hist = !(LM && p.lm_dev) ? nullptr
                       : p.lm_arena_ptrs ? reinterpret_cast<int *>(lm_arena + arena_cap)
                                         : p.lm_hist + (size_t)b * (size_t)p.arena_stride *
                                                           (size_t)(p.lm_hist_stride ? p.lm_hist_stride : p.lm_hist_n);
  int *const s_upd = CTC_SLOT(int, U_NEWINFO);  // staging for the host's answer (free outside R4c..R5: 10 * KP ints)
  // the host's answer: (node, term) pairs -- or, for a character-based model, (node, V terms) entries that are too many
  // for the staging area and are copied from the mapped block straight into the node rows
  auto lm_scatter_updates = [&](int tid) {
    if (!(LM && p.lm_char)) {
      const int nu = s_upd[1];
      for (int q = tid; q < nu; q += NT) lm_arena[s_upd[2 + 2 * q]] = bits_f((uint32_t)s_upd[3 + 2 * q]);
    } else {
      const volatile int *blk = lm_upd;
      int nu = s_upd[1];
      if (nu > K) nu = K;
      const int es = 1 + V;
      for (int x = tid; x < nu * V; x += NT) {
        const int q = x / V, cch = x - q * V;
        const int node = blk[2 + q * es];
        lm_row[(size_t)node * V + cch] = bits_f((uint32_t)blk[2 + q * es + 1 + cch]);
      }
    }
  };
  // Fetch the host's (node, LM term) pairs into s_upd; wait_for > 0: first poll the block's go flag until it
  // reaches wait_for.  One warp, whole 128-byte lines per request: the block lives in host memory and every
  // request is a PCIe round trip (tools/micro/sysmem_pingpong.cu measures one handshake).
  auto lm_fetch_updates = [&](int wait_for) {
#if defined(CTC_EMULATE)
    (void)wait_for;
    const int words = p.lm_char ? 2 : 2 + 2 * lm_upd[1];  // (the rows of a character-based model are not staged)
    for (int w = 0; w < words; ++w) s_upd[w] = lm_upd[w];
#else
    if (threadIdx.x < 32) {
      const int lane = (int)threadIdx.x;
      const volatile int *blk = lm_upd;
      int v = 0;
      bool seen = false;  // the poll that saw the flag also brought the first 64-byte line of the block
      if (wait_for > 0) {
        const long long deadline = clock64() + 20000000000ll;  // ~10 s: never hang the GPU on a dead host
        unsigned it = 0;
        for (;;) {
          v = blk[lane];
          if (__shfl_sync(0xffffffffu, v, 0) >= wait_for) { seen = true; break; }
          if ((++it & 255u) == 0u) {
            int bad = 0;
            if (lane == 0) bad = (*(volatile int *)p.hs_abort != 0 || clock64() > deadline) ? 1 : 0;
            if (__shfl_sync(0xffffffffu, bad, 0)) {
              if (lane == 0) s_ctl[C_FLAGS] |= FLAG_ERR_ARENA;
              break;
            }
          }
        }
      }
      // The host writes the pairs first and the flag last (release), and the flag shares its 64-byte line with the
      // count and the first seven pairs: a read of that line that shows the flag shows them too (one coherent line
      // read; stores to a line become visible in program order).  Only a longer answer -- or a character model's
      // rows -- costs a second PCIe round trip, behind a fence.
      int cnt = __shfl_sync(0xffffffffu, v, 1);
      if (!(seen && !p.lm_char && cnt >= 0 && cnt <= 7)) {
        if (wait_for > 0) __threadfence_system();  // acquire: the payload loads below stay behind the flag load
        v = blk[lane];
        cnt = __shfl_sync(0xffffffffu, v, 1);
      }
      if (cnt > K) cnt = K;
      s_upd[lane] = lane == 1 ? cnt : v;
      if (!p.lm_char)
        for (int w = 32 + lane; w < 2 + 2 * cnt; w += 32) s_upd[w] = blk[w];
    }
#endif
  };
  int Tb = p.seq_lens ? p.seq_lens[bi] : p.T;  // reference binding.cpp:64-65 clamps to T
  if (Tb > p.T) Tb = p.T;
  const int t0 = p.nframes > 0 ? p.t0 : 0;
  Tb -= t0;
  if (p.nframes > 0 && Tb > p.nframes) Tb = p.nframes;
  if (Tb < 0) Tb = 0;
  const int fresh = p.fresh;
  const int abs_t0 = fresh ? 0 : st[2];
  int *const st_slots = st + kStateHeader;
  int *const st_anchors = st_slots + kSlotArrays * K;

  if (LM && !p.lm_dev) {
    // scores the host's Scorer hook computed for the nodes created by the previous launch
    CTC_PAR {
      if (tid == 0) newlist[0] = 0;
    }
    lm_fetch_updates(0);
    CTC_BARRIER();
    CTC_PAR { lm_scatter_updates(tid); }
    CTC_BARRIER();
  }
  // ---- region: stage tables, load (or create) the beam state --------------------------------------
  CTC_PAR {
    for (int i = tid; i < 32; i += NT) {
      ((uint64_t *)c.s_exptab)[i] = kExp2fTab[i];
      ((double *)c.s_logtab)[i] = kLogfTab[i];
    }
    for (int j = tid; j < KP; j += NT) {
      int node = 0, chr = -1, depth = 0, ts = 0, pslot = -1, anch = -1, dstate = LM ? lm->dict_start : 0, jump = -1;
      float bprev = kNInf, nbprev = kNInf, score = kNInf, lpc = kNInf;
      if (fresh) {
        if (j == 0) { bprev = 0.0f; score = 0.0f; }  // reference ctc_beam_search_decoder.cpp:43
      } else if (j < K) {
        const int *s = st_slots;
        node = s[j]; chr = s[K + j]; depth = s[2 * K + j]; bprev = bits_f((uint32_t)s[3 * K + j]);
        nbprev = bits_f((uint32_t)s[4 * K + j]); score = bits_f((uint32_t)s[5 * K + j]);
        lpc = bits_f((uint32_t)s[6 * K + j]); ts = s[7 * K + j]; pslot = s[8 * K + j]; anch = s[9 * K + j];
        dstate = s[10 * K + j]; jump = s[11 * K + j];
      }
      c.s_node[j] = node; c.s_chr[j] = chr; c.s_depth[j] = depth; c.s_bprev[j] = bprev; c.s_nbprev[j] = nbprev;
      c.s_score[j] = score; c.s_lpc[j] = lpc; c.s_ts[j] = ts; c.s_pslot[j] = pslot; c.s_anch[j] = anch;
      c.s_dstate[j] = dstate; s_jump[j] = jump;
      if (LM) for (int w = 0; w < L.WC; ++w) c.s_dmask[j * L.WC + w] = lm->dict_mask[(long long)dstate * L.WC + w];
      c.s_lmsp[j] = (LM && !fresh && j < st[0]) ? ld_cg(&lm_arena[node]) : 0.0f;
      c.s_evict[j] = 0;
      s_nodeN[j] = -1;
    }
    for (int a = tid; a < KP2; a += NT) {
      int dnode = 0, dchr = 0, dpslot = -1, dts = 0, ddstate = 0;
      float dlpc = kNInf;
      if (!fresh) {
        dnode = st_anchors[a]; dchr = st_anchors[KP2 + a]; dpslot = st_anchors[2 * KP2 + a];
        dlpc = bits_f((uint32_t)st_anchors[3 * KP2 + a]); dts = st_anchors[4 * KP2 + a];
        ddstate = st_anchors[5 * KP2 + a];
      }
      c.s_dnode[a] = dnode; c.s_dchr[a] = dchr; c.s_dpslot[a] = dpslot; c.s_dlpc[a] = dlpc; c.s_dts[a] = dts;
      c.s_ddstate[a] = ddstate;
      c.s_drev[a] = 0;
    }
    for (int x = tid; x < 3 * KP; x += NT) c.s_cnt2[x] = 0;
    for (int x = tid; x < KP * WS; x += NT) { mask_buf0[x] = 0u; mask_buf1[x] = 0u; }
    for (int x = tid; x < KP * W; x += NT) c.s_rmask[x] = 0u;
    for (int x = tid; x < 2 * kNBins; x += NT) c.s_hist[x] = 0;
    if (SORTED) for (int v = tid; v < 2 * VR; v += NT) rank_base[v] = (int16_t)-1;
    if (tid == 0) {
      for (int x = 0; x < 32; ++x) s_ctl[x] = 0;
      s_ctl[C_M] = fresh ? 1 : st[0];
      s_ctl[C_NNODES] = fresh ? 1 : st[1];
      s_ctl[C_FLAGS] = fresh ? 0 : st[3];
      if (LM) {
        double *const ab = (double *)(s_ctl + C_AB);
        ab[0] = lm_pair ? lm_pair[0] : lm->lm_alpha;
        ab[1] = lm_pair ? lm_pair[1] : lm->beta;
      }
      s_ctl[C_KMIN] = (int)0xFFFFFFFFu;
      s_ctl[C_SMIN] = (int)0xFFFFFFFFu;
      if (fresh) {  // root node (reference path_trie.cpp:11-30)
        Node root; root.parent = -1; root.chr = -1; root.lpc = kNInf; root.ts = 0; root.jump = -1;
        store_node(&nodes[0], root);
        if (LM) { dstate_arena[0] = lm->dict_start; lm_arena[0] = 0.0f; }
      }
    }
    // device n-gram scorer, before the first frame of an utterance or stream: the root's history (the "<s>" padding
    // of Scorer::make_ngram) and, for a character-based model, its row of LM terms
    if (LM && p.lm_dev && abs_t0 == 0) {
      for (int k = tid; k < lm->lm_hist_n; k += NT) lm_hist[k] = lm->ngram.bos;
      if (p.lm_char)
        for (int x = tid; x < V; x += NT) lm_dev_root_term(lm, lm_pair ? lm_pair[0] : lm->lm_alpha, lm_row, x);
    }
  }
#if !defined(CTC_EMULATE)
  uint64_t *const mbar = (uint64_t *)(smem + H_MBAR);
  float *const tile_lp = (float *)(smem + L.tile_lp);
  uint16_t *const tile_idx = (uint16_t *)(smem + L.tile_idx);
  const float *const g_lp = p.lp + ((size_t)bi * p.T + t0) * NP;
  const uint16_t *const g_idx = SORTED ? p.idx + ((size_t)bi * p.T + t0) * NP : nullptr;
  if (threadIdx.x == 0) {
    mbar_init(&mbar[0], 1);
    mbar_init(&mbar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  auto issue_tile = [&](int tile) {
    const int stage = tile & 1, f0 = tile * F;
    const int nf = (Tb - f0 < F) ? (Tb - f0) : F;
    const uint32_t bytes_lp = (uint32_t)nf * NP * 4u, bytes_idx = SORTED ? (uint32_t)nf * NP * 2u : 0u;
    mbar_expect_tx(&mbar[stage], bytes_lp + bytes_idx);
    bulk_g2s(tile_lp + (size_t)stage * F * NP, g_lp + (size_t)f0 * NP, bytes_lp, &mbar[stage]);
    if (SORTED) bulk_g2s(tile_idx + (size_t)stage * F * NP, g_idx + (size_t)f0 * NP, bytes_idx, &mbar[stage]);
  };
#endif
  CTC_BARRIER();
#if !defined(CTC_EMULATE)
  if (threadIdx.x == 0 && Tb > 0) issue_tile(0);
#endif

  int M = s_ctl[C_M];
  // number of dead anchors currently in the table (0 almost always: lets the frame loop skip their sweeps), and the
  // score range of the beam (kept up to date by region R5: the radix range of a frame is known before region R1)
  CTC_PAR {
    int cntv = 0;
    for (int a = tid; a < KP2; a += NT) cntv += (c.s_dpslot[a] >= 0) ? 1 : 0;
    if (cntv) atom_add(&s_ctl[C_NLIVE], cntv);
    unsigned smin = 0xFFFFFFFFu, smax = 0u;
    for (int j = tid; j < M; j += NT) {
      const unsigned o = ord_f(c.s_score[j]);
      smin = o < smin ? o : smin;
      smax = o > smax ? o : smax;
    }
    warp_range_store(c.s_wcnt + 128, smin, smax, tid);
    if (MERGED) {
      // "existing child" masks of the first frame (afterwards every commit builds those of the next frame): member j
      // whose parent sits in beam slot i masks grid cell (i, chr[j])  (reference path_trie.cpp:39-57)
      int np = 0;
      for (int j = tid; j < M; j += NT) {
        const int i = c.s_pslot[j], ch = c.s_chr[j];
        if (i >= 0 && ch >= 0) { atom_or(&mask_buf0[i * WS + (ch >> 5)], 1u << (ch & 31)); ++np; }
      }
      // (the pair count: with a per-frame vocabulary cut only children whose character the frame keeps count, so
      //  those kernels count in region R1)
      if (np && !SORTED) atom_add(&s_ctl[C_NPAIRS], np);
    }
  }
  CTC_BARRIER();
  int nlive = s_ctl[C_NLIVE];
  const bool head_offload = CTC_OPT_HEADOFF && WB0 > 0 && !(p.no_fast & 2);  // (test knob bit 1: every warp computes the head itself)
  bool head_ready = false;       // FASTB: the head block of the coming frame has been written (see the fast back half)
  int nnodes = s_ctl[C_NNODES];  // MERGED: the node count travels in a register across barrier-free commits;
  bool nn_stale = false;         // s_ctl[C_NNODES] is brought up to date before a general back half needs it
  CTC_BARRIER();

  // "is the parent designation q (a beam slot, possibly tagged kNewFlag) alive after this frame?"
#define CTC_PARENT_ALIVE(q) ((((q) & kNewFlag) != 0) || c.s_evict[(q)] == 0)

  // =================================== the frame loop ===============================================
#if !defined(CTC_EMULATE)
  int tile = 0, ft = 0;
#endif
  for (int t = 0; t < Tb; ++t) {
    const int t_abs = abs_t0 + t;
#if defined(CTC_EMULATE)
    c.lp = p.lp + ((size_t)bi * p.T + t0 + t) * NP;
    c.idx = SORTED ? p.idx + ((size_t)bi * p.T + t0 + t) * NP : nullptr;
#else
    {
      if (ft == F) { ft = 0; ++tile; }
      if (ft == 0) {
        mbar_wait(&mbar[tile & 1], (uint32_t)((tile >> 1) & 1));
        // stage (tile+1)&1 was last read in frame t-1, which every thread has left (closing barrier)
        if (threadIdx.x == 0 && (tile + 1) * F < Tb) issue_tile(tile + 1);
      }
      c.lp = tile_lp + ((size_t)(tile & 1) * F + ft) * NP;
      c.idx = SORTED ? tile_idx + ((size_t)(tile & 1) * F + ft) * NP : nullptr;
      ++ft;
    }
#endif
    // row trailer written by the prune kernel: [NP-2] = n | (rank_of_blank + 1) << 16, [NP-1] = max
    // non-blank log-prob of the frame
    CTC_TICK(0);  // tile wait
    const uint32_t meta = f_bits(c.lp[NP - 2]);
    const int n = (int)(meta & 0xFFFFu);
    const int rblank = (int)(meta >> 16) - 1;
    const float lpmax = c.lp[NP - 1];

    if (SORTED) c.s_rank = rank_base + (MERGED ? par : 0) * VR;
    if (SORTED && (!MERGED || t == 0)) {
      // rank of every kept character.  MERGED kernels build the table of frame t + 1 during frame t (below); only
      // the first frame of a launch builds its own.
      CTC_PAR {
        for (int r = tid; r < n; r += NT) c.s_rank[c.idx[r]] = (int16_t)r;
      }
      CTC_BARRIER();
      CTC_TICK(1);
    }
    // score-key range [lo32, top32] of everything that can still be selected in this frame, and the shift that
    // maps it onto the radix bins.  Without a scorer it follows from the beam as it stands and the frame's row, so
    // members can bin themselves in region R1 and region G starts right after the barrier:
    //   every new member score >= blank term = lp_blank + old score >= lp_blank + (lowest old score)   [beam full]
    //   every key <= (highest old score) + (largest log-prob of the row) + 2 ln 2  (two nested log_sum_exp of at
    //   most three such terms; 1.5 > 2 ln 2 + rounding)
    unsigned lo32 = 0u, top32 = 0u;
    unsigned lo_valid = 0u;   // the proven lower bound (lo32 may be the checked heuristic one, SORTED kernels)
    bool heuristic = false;
    int shift32 = 0;  // smallest shift with ((top32 - lo32) >> shift32) < kNBins
    auto set_shift = [&]() {
      const unsigned wm = top32 - lo32;
#if defined(CTC_EMULATE)
      const int bits = wm ? 32 - __builtin_clz(wm) : 0;
#else
      const int bits = 32 - __clz((int)wm);
#endif
      shift32 = bits > 8 ? bits - 8 : 0;
    };
    // the range of a frame from its row and the score range [cmin_o, cmax_o] (monotone keys) of the beam it starts from
    auto head_of = [&](const float *row, unsigned cmin_o, unsigned cmax_o, bool full, unsigned &lo, unsigned &top,
                       unsigned &lov, bool &heur) {
      const uint32_t meta_r = f_bits(row[NP - 2]);
      const int rblank_r = (int)(meta_r >> 16) - 1;
      const float lpmax_r = row[NP - 1];
      const float cmin = unord_f(cmin_o), cmax = unord_f(cmax_o);
      float lpm = lpmax_r;
      lo = 0u; heur = false;
      if (rblank_r >= 0) {
        const float lpb = row[rblank_r];
        if (full) lo = ord_f(f_add(lpb, cmin));
        lpm = lpb > lpm ? lpb : lpm;
      }
      top = ord_f(f_add(f_add(cmax, lpm), 1.5f));
      // (a frame that keeps no character at all, cutoff_top_n = 0: -FLT_MAX + -FLT_MAX rounds to -inf, below the
      // members' -FLT_MAX scores)
      if (top < ord_f(kNInf)) top = ord_f(kNInf);
      lov = lo;
      if (full && !p.force_fallback) {
        // A second, usually much tighter bound (where the vocabulary is cut per frame the blank is often not among
        // the kept characters and the bound above is void): every row's best candidate scores at least
        // (lowest beam score) + (largest non-blank log-prob of the row), so normally K keys reach that value.
        // Masked cells and the repeated-character rule can break the count, therefore this bound is CHECKED after
        // the grid walk (histogram total >= K); if it fails, kernels for a cut vocabulary walk the grid again with
        // the proven bound, index-order kernels (where that is a 3-in-1000-frames event) take the grid-walking select.
        const unsigned lo_h = ord_f(f_add(f_add(cmin, lpmax_r), p.heur_bias));
        if (lo_h > lo && lo_h <= top) { lo = lo_h; heur = true; }
      }
      if (top < lo) top = lo;
    };
    if (!LM) {
      if (FASTB && head_ready) {
        // left behind by a grid-walking warp of the previous frame while the slot owners committed the beam
        const int *hb = c.s_wcnt + 64 + 8 * par;
        lo32 = (unsigned)hb[0]; top32 = (unsigned)hb[1]; lo_valid = (unsigned)hb[2]; heuristic = hb[3] != 0;
      } else {
        unsigned cmin_o, cmax_o;
        // (only warps that own slots leave a range: with the beam size a compile-time constant that is the first KPW)
        warp_range_load<(KPT > 0 && KPT <= NT) ? KPW : NW>(c.s_wcnt + 128 + 64 * par, cmin_o, cmax_o);
        head_of(c.lp, cmin_o, cmax_o, M == K, lo32, top32, lo_valid, heuristic);
      }
      head_ready = false;
      set_shift();
    }
    if (LM) {
      // min_cutoff = worst beam score + blank_prob - max(0, beta); active once the beam is full
      // (reference ctc_beam_search_decoder.cpp:74-82: the sorted beam's last element is its minimum)
      CTC_PAR {
        unsigned smin = 0xFFFFFFFFu;
        for (int j = tid; j < M; j += NT) { const unsigned o = ord_f(c.s_score[j]); smin = o < smin ? o : smin; }
#if defined(CTC_EMULATE)
        red_min_u32((unsigned *)&s_ctl[C_SMIN], smin);
#else
        if (tid < ((M + 31) & ~31)) red_min_u32((unsigned *)&s_ctl[C_SMIN], smin);
#endif
      }
      CTC_BARRIER();
      const float worst = unord_f((unsigned)s_ctl[C_SMIN]);
      const double mx0 = c.s_ab[1] > 0.0 ? c.s_ab[1] : 0.0;
      c.lm_full = (M == K);
      c.lm_cutoff = (float)d_add((double)f_add(worst, c.lp[NP - 3]), -mx0);
    }

    // ---- frame-parity views (MERGED kernels; parity 0 everywhere else) and what is known before the frame starts
    const int hpar = MERGED ? par : 0;
    int *const hist0 = c.s_hist + hpar * kNBins;  // first radix histogram of this frame
    const int ovf_w = (MERGED && par) ? C_OVF_B : C_OVF, ovf_nx = (MERGED && !par) ? C_OVF_B : C_OVF;
    const int anyref_w = (MERGED && par) ? C_ANYREF_B : C_ANYREF, anyref_nx = (MERGED && !par) ? C_ANYREF_B : C_ANYREF;
    const int npairs_w = (MERGED && par) ? C_NPAIRS_B : C_NPAIRS, npairs_nx = (MERGED && !par) ? C_NPAIRS_B : C_NPAIRS;
    uint32_t *const mask_next = par ? mask_buf0 : mask_buf1;  // MERGED: "existing child" masks of frame t + 1
    if (MERGED) c.s_mask = par ? mask_buf1 : mask_buf0;
    (void)ovf_nx; (void)anyref_nx; (void)mask_next;
    const int n_nb = n - (rblank >= 0 ? 1 : 0);
    // how many prefixes exist after this frame: the members plus every grid cell that is a new candidate.  With a
    // scorer the dictionary / cutoff decide that per cell, so the count is taken after the grid walk instead.
    // (MERGED: the pair count came with the beam; otherwise region R1 counts it, see below)
    // (cut-vocabulary kernels: only children whose character the frame keeps are pairs, region R1 counts them and
    //  select_all is known after the front; the grid walk bins its candidates regardless)
    long long total = (MERGED && !SORTED) ? (long long)M * (n_nb + 1) - s_ctl[npairs_w] : 0;
    bool select_all = MERGED && !SORTED && total <= (long long)K;  // reference :149 `prefixes.size() >= beam_size`
    const int G = (n + 31) >> 5;                        // 32-wide column groups of the candidate grid

    // ---- region R1: every member's blank / repeat / extension-from-parent terms, merged with
    //      log_sum_exp; dead anchors take their lpc / timestep update.  All in shared memory.
    // (reference ctc_beam_search_decoder.cpp:97-118,138-139; path_trie.cpp:39-57,129-137)
    auto members_region = [&](const int tid) {
      if (tid == 0) {
        s_ctl[C_NREV] = 0;  // (not with the other counters in R5: slow threads may still be reading them there --
        s_ctl[C_NSEL] = 0;  //  C_NSEL is read right after the classification's barrier, the last one before R5)
        if (MERGED) {
          s_ctl[npairs_nx] = 0;  // (the commit of this frame counts the pairs of the next one into it)
          if (nn_stale) s_ctl[C_NNODES] = nnodes;
        }
      }
      if (MERGED)  // the other histogram: scanned by the previous frame, first used again by the next one
        for (int x = tid; x < kNBins; x += NT) c.s_hist[(hpar ^ 1) * kNBins + x] = 0;
      if (MERGED && SORTED) {  // the other rank table (last read by the previous frame's members): the back half refills it
        int *const rn = reinterpret_cast<int *>(rank_base + (par ^ 1) * VR);
        for (int x = tid; x < VR / 2; x += NT) rn[x] = -1;
      }
      unsigned kmin = 0xFFFFFFFFu, kmax = 0u, smax = 0u;
      int npairs = 0;
      for (int j0 = 0; j0 < M; j0 += NT) {
        const int j = j0 + tid;
        if (j < M) {
          if (FASTB) {  // a member committed by the barrier-free back half of the previous frame moves in
            const int pn = s_nodeN[j];
            if (pn >= 0) { c.s_node[j] = pn; c.s_depth[j] = s_depthN[j]; s_jump[j] = s_jumpN[j]; s_nodeN[j] = -1; }
          }
          const float sc = c.s_score[j];
          const int ch = c.s_chr[j];
          if (FAST2) s_code[j] = 0xFFFF - (ch + 1);
          const float bnew = (rblank >= 0 && !c.lm_cut(c.lp[rblank], sc)) ? f_add(c.lp[rblank], sc) : kNInf;
          float rep = kNInf, ext = kNInf;
          const int rr = (ch >= 0) ? c.rank_of(ch) : -1;
          if (rr >= 0) {
            const float l = c.lp[rr];
            if (!c.lm_cut(l, sc)) rep = f_add(l, c.s_nbprev[j]);
            const int i = c.s_pslot[j];
            if (i >= 0 && !c.lm_cut(l, c.s_score[i])) {  // parent is a beam member: an existing child of it
              if (c.s_lpc[j] < l) { c.s_lpc[j] = l; c.s_ts[j] = t_abs; }  // path_trie.cpp:41-46
              if (ch == c.s_chr[i]) {
                const float pb = c.s_bprev[i];
                ext = (pb > kNInf) ? f_add(l, pb) : kNInf;
              } else {
                ext = f_add(l, c.s_score[i]);
              }
              if (LM && c.lm_scored(ch)) ext = c.lm_apply_c(ext, i, ch);
              // (MERGED: the mask bit -- and in index order the pair count -- were set when the beam was committed)
              if (!MERGED) atom_or(&c.s_mask[i * W + (rr >> 5)], 1u << (rr & 31));
              if (!MERGED || SORTED) ++npairs;
            }
          }
          CTC_TICK(12);  // members: loads and terms
          const float nb = lse_smem(rep, ext, c.s_exptab, c.s_logtab);
          const float sn = lse_smem(bnew, nb, c.s_exptab, c.s_logtab);
          CTC_TICK(13);  // members: two log_sum_exp
          c.s_bnew[j] = bnew; c.s_nbnew[j] = nb; c.s_snew[j] = sn;
          const unsigned o = ord_f(sn);
          if (!LM) {
            // first radix pass: the member bins itself (the histograms were cleared by region R5)
            if (o >= lo32) CTC_HIST_ADD(hist0, (o - lo32) >> shift32);
          } else {
            kmin = o < kmin ? o : kmin;
            kmax = o > kmax ? o : kmax;
          }
        }
      }
      if (LM) {
        // the largest key each member's grid row can reach before beta: its score + the frame's best non-blank
        // log-prob + the row's largest LM term when that is positive (alpha < 0, or a backoff weight > 0).  (A loop
        // of its own: inside the one above it costs the index-order scorer kernel a spill.)
        for (int j = tid; j < M; j += NT) {
          float tm = 0.0f;
          if (!c.lm_char) {
            tm = c.s_lmsp[j] > tm ? c.s_lmsp[j] : tm;
          } else {
            const float *const row = c.lm_row + (size_t)c.s_node[j] * V;
            for (int r = 0; r < n; ++r) { const float x = ld_cg(&row[c.chr_at(r)]); tm = x > tm ? x : tm; }
          }
          float u = f_add(c.s_score[j], lpmax);
          if (tm > 0.0f) u = f_add(u, tm);
          const unsigned os = ord_f(u);
          smax = os > smax ? os : smax;
        }
      }
      if (npairs) atom_add(&s_ctl[MERGED ? npairs_w : (int)C_NPAIRS], npairs);
      if (nlive > 0) {
        for (int a = tid; a < KP2; a += NT) {
          const int i = c.s_dpslot[a];
          if (i >= 0) {  // dead node whose parent is in the beam: an existing (dead) child of slot i
            const int rr = c.rank_of(c.s_dchr[a]);
            if (rr >= 0 && !c.lm_cut(c.lp[rr], c.s_score[i])) {
              const float l = c.lp[rr];
              if (c.s_dlpc[a] < l) { c.s_dlpc[a] = l; c.s_dts[a] = t_abs; }
              atom_or(&c.s_rmask[i * W + (rr >> 5)], 1u << (rr & 31));
            }
          }
        }
      }
      if (LM) {  // with a scorer the range is taken from the new member scores and the rows' bounds (the LM term is not
                 // bounded above)
#if defined(CTC_EMULATE)
        red_min_u32((unsigned *)&s_ctl[C_KMIN], kmin);
        red_max_u32((unsigned *)&s_ctl[C_KMAX], kmax);
        red_max_u32((unsigned *)&s_ctl[C_SMAX], smax);
#else
        if (tid < ((M + 31) & ~31)) {  // whole warps that own at least one member
          red_min_u32((unsigned *)&s_ctl[C_KMIN], kmin);
          red_max_u32((unsigned *)&s_ctl[C_KMAX], kmax);
          red_max_u32((unsigned *)&s_ctl[C_SMAX], smax);
        }
#endif
      }
    };
    // ---- region G: the ONE walk over the beam x pruned-vocab grid.  A warp owns a beam member per
    //      iteration (member values are warp-broadcast), lanes own the characters.  Candidates whose score
    //      key reaches lo32 (the worst member's key once the beam is full) are appended to the warp's
    //      candidate-list segment -- ballot + popc, no atomics, deterministic -- and counted into the
    //      first radix histogram.  Everything after this region works on the list.
    // If a list segment overflows (the beam is filling up, or most member scores collapsed because the blank /
    // their own character was cut from the frame, so that lo32 filters nothing), every candidate has still been
    // counted in the first histogram: the bin holding the K-th key is known, lo32 moves up to that bin's lower edge
    // and the grid is walked ONCE more with lists that now only take what can still be selected.  Only if that
    // overflows too does the frame take the grid-walking fallback.
    bool rebin = LM;  // members are binned inside region G (scorer path; or the tightened second walk, SORTED only)
    bool have_scan = false;  // the first histogram has already been scanned (pre_bin / pre_above / pre_cnt)
    int pre_bin = 0, pre_above = 0, pre_cnt = 0;
    // "does member i already have a child by character ch in the beam?" for masks indexed by character (ch >= 0)
    auto mbit = [&](int i, int ch) -> bool { return (c.s_mask[i * WS + (ch >> 5)] >> (ch & 31)) & 1u; };
    constexpr bool MCS = MERGED && SORTED;  // the lanes of a column group hold arbitrary characters: per-lane mask words
    auto grid_walk = [&](const int warp, const bool rebin) {
      int cnt = 0;
      uint32_t *const segk = c.s_clk + warp * SEG;
      int *const segi = c.s_cli + warp * SEG;
      if (rebin && !select_all) {  // (without a scorer the members binned themselves in region R1)
        CTC_LANES {
          for (int j = warp * 32 + lane; j < M; j += NT) {
            const unsigned k = ord_f(c.s_snew[j]);
            if (k >= lo32) CTC_HIST_ADD(hist0, (k - lo32) >> shift32);
          }
        }
      }
      // ---- the dominant column first.  In a frame with one likely non-blank character (log-prob lpmax, runner-up
      //      lpmax2 at least 1 below) that column is walked column-wise -- lane = row, 32 rows per step -- and left
      //      out of the row walk, whose skip test then uses lpmax2: in such frames EVERY row passes the lpmax test
      //      (each row's extension by the likely character is a candidate that counts) but only the top rows have
      //      anything else to offer.
      int rstar = -1;         // rank of the most likely non-blank kept character (column-first frames only)
      float lp_rows = lpmax;  // largest log-prob the row walk can still meet
      if (!LM && n > 0) {
        float lp2 = kNInf;
        int r1 = -1;
        if (SORTED) {  // rows are sorted by probability: the first two non-blank ranks
          r1 = (rblank == 0) ? 1 : 0;
          int r2 = r1 + 1;
          if (r2 == rblank) ++r2;
          if (r1 >= n) r1 = -1;
          else if (r2 < n) lp2 = c.lp[r2];
        } else if (n <= 32) {
          CTC_LV(unsigned, key);
          CTC_LV(unsigned, key2);
          CTC_LANES { key[LX] = (lane < n && lane != rblank) ? ord_f(c.lp[lane]) : 0u; }
          const unsigned m1 = ctc_warp_max(key);
          CTC_LV(int, ism);
          CTC_LANES { ism[LX] = (key[LX] == m1 && m1 != 0u) ? 1 : 0; }
          const unsigned bm = ctc_ballot(ism);
          r1 = bm ? ctc_ffs(bm) - 1 : -1;
          CTC_LANES { key2[LX] = (lane == r1) ? 0u : key[LX]; }
          const unsigned m2 = ctc_warp_max(key2);
          if (m2 != 0u) lp2 = unord_f(m2);
        }
        if (r1 >= 0 && f_add(c.lp[r1], -lp2) >= 1.0f) { rstar = r1; lp_rows = lp2; }
      }
      if (rstar >= 0) {
        const int chs = c.chr_at(rstar);
        const float ls = c.lp[rstar];
        for (int i0 = (warp - WB0) * 32; i0 < M; i0 += NB * 32) {
          CTC_LV(int, pred);
          CTC_LV(uint32_t, kk);
          CTC_LANES {
            const int i = i0 + lane;
            pred[LX] = 0;
            kk[LX] = 0u;
            if (i < M) {
              const bool rep = (chs == c.s_chr[i]);
              const float b = c.s_bprev[i];
              float sc = f_add(ls, rep ? b : c.s_score[i]);
              if (rep && !(b > kNInf)) sc = kNInf;
              const unsigned k = ord_f(sc);
              const int mb = MERGED ? chs : rstar;  // (masks by character / by rank)
              const bool ok = !((c.s_mask[i * WS + (mb >> 5)] >> (mb & 31)) & 1u) && (k >= lo32);
              pred[LX] = ok ? 1 : 0;
              kk[LX] = k;
              if (ok && !select_all) CTC_HIST_ADD(hist0, (k - lo32) >> shift32);
            }
          }
          const unsigned bal = ctc_ballot(pred);
          CTC_LANES {
            if (pred[LX]) {
              const int pos = cnt + ctc_popc(bal & ctc_lt_mask(lane));
              if (pos < SEG) { segk[pos] = kk[LX]; segi[pos] = ((i0 + lane) << 16) | rstar; }
            }
          }
          cnt += ctc_popc(bal);
          CTC_STAT(g_stats.cl_entries += ctc_popc(bal));
        }
      }
      // rows (members) are tested 32 at a time: lane l of the w-th grid-walking warp looks at row base + w + NB * l.  A row whose best
      // possible candidate (score + max non-blank log-prob) stays under lo32 contributes nothing; on config 2
      // that removes 80 % of the rows.
#pragma unroll 1
      for (int base = 0; base < M; base += 32 * NB) {
        CTC_LV(int, rowok);
        CTC_LANES {
          const int i = base + (warp - WB0) + NB * lane;
          rowok[LX] = 0;
          if (i < M) {
            CTC_STAT(g_stats.rows++);
            rowok[LX] = (LM || ord_f(f_add(c.s_score[i], lp_rows)) >= lo32) ? 1 : 0;
            CTC_STAT(g_stats.rows_skipped += !rowok[LX]);
          }
        }
        unsigned rows = ctc_ballot(rowok);
        // per-lane column constants of group 0 (the only group when n <= 32)
        CTC_LV(int, colc);
        CTC_LV(float, colv);
        CTC_LANES {
          colc[LX] = -2;  // not a candidate column (beyond n, or the blank)
          colv[LX] = 0.0f;
          if (rows && lane < n && lane != rstar) {  // (the dominant column has been walked already)
            const int ch = c.chr_at(lane);
            if (ch != c.blank) { colc[LX] = ch; colv[LX] = c.lp[lane]; }
          }
        }
        // two rows per iteration when the grid is one group wide: two independent load -> add -> key ->
        // ballot chains in flight instead of one
        while (CTC_OPT_ROWS2 && !LM && G == 1 && (rows & (rows - 1u))) {
          const int rl1 = ctc_ffs(rows) - 1;
          rows &= rows - 1u;
          const int rl2 = ctc_ffs(rows) - 1;
          rows &= rows - 1u;
          const int i1 = base + (warp - WB0) + NB * rl1, i2 = base + (warp - WB0) + NB * rl2;
          const float sc1 = c.s_score[i1], b1 = c.s_bprev[i1], sc2 = c.s_score[i2], b2 = c.s_bprev[i2];
          const int ch1 = c.s_chr[i1], ch2 = c.s_chr[i2];
          const uint32_t mw1 = MCS ? 0u : c.s_mask[i1 * WS], mw2 = MCS ? 0u : c.s_mask[i2 * WS];
          CTC_LV(int, pred1);
          CTC_LV(int, pred2);
          CTC_LV(uint32_t, kk1);
          CTC_LV(uint32_t, kk2);
          CTC_LANES {
            const int ch = colc[LX];
            const float l = colv[LX];
            const bool rep1 = (ch == ch1), rep2 = (ch == ch2);
            float s1 = f_add(l, rep1 ? b1 : sc1), s2 = f_add(l, rep2 ? b2 : sc2);
            if (rep1 && !(b1 > kNInf)) s1 = kNInf;
            if (rep2 && !(b2 > kNInf)) s2 = kNInf;
            const unsigned k1 = ord_f(s1), k2 = ord_f(s2);
            const bool m1 = MCS ? (ch >= 0 && mbit(i1, ch)) : (((mw1 >> lane) & 1u) != 0u);
            const bool m2 = MCS ? (ch >= 0 && mbit(i2, ch)) : (((mw2 >> lane) & 1u) != 0u);
            const bool ok1 = (ch >= 0) && !m1 && (k1 >= lo32);
            const bool ok2 = (ch >= 0) && !m2 && (k2 >= lo32);
            pred1[LX] = ok1 ? 1 : 0; kk1[LX] = k1;
            pred2[LX] = ok2 ? 1 : 0; kk2[LX] = k2;
            if (!select_all) {
              if (ok1) CTC_HIST_ADD(hist0, (k1 - lo32) >> shift32);
              if (ok2) CTC_HIST_ADD(hist0, (k2 - lo32) >> shift32);
            }
          }
          const unsigned bal1 = ctc_ballot(pred1), bal2 = ctc_ballot(pred2);
          const int n1 = ctc_popc(bal1);
          CTC_LANES {
            if (pred1[LX]) {
              const int pos = cnt + ctc_popc(bal1 & ctc_lt_mask(lane));
              if (pos < SEG) { segk[pos] = kk1[LX]; segi[pos] = (i1 << 16) | lane; }
            }
            if (pred2[LX]) {
              const int pos = cnt + n1 + ctc_popc(bal2 & ctc_lt_mask(lane));
              if (pos < SEG) { segk[pos] = kk2[LX]; segi[pos] = (i2 << 16) | lane; }
            }
          }
          cnt += n1 + ctc_popc(bal2);
          CTC_STAT(g_stats.cl_entries += n1 + ctc_popc(bal2));
        }
        if (CTC_OPT_ROWS2 && !LM && G == 2) {
          // two column groups (33..64 kept characters): both groups of a row in one go
          CTC_LV(int, colc2);
          CTC_LV(float, colv2);
          CTC_LANES {
            colc2[LX] = -2;
            colv2[LX] = 0.0f;
            if (rows && 32 + lane < n) {
              const int ch = c.chr_at(32 + lane);
              if (ch != c.blank) { colc2[LX] = ch; colv2[LX] = c.lp[32 + lane]; }
            }
          }
          while (rows) {
            const int rl = ctc_ffs(rows) - 1;
            rows &= rows - 1u;
            const int i = base + (warp - WB0) + NB * rl;
            const float sc_i = c.s_score[i], b_i = c.s_bprev[i];
            const int ch_i = c.s_chr[i];
            const uint32_t mwa = MCS ? 0u : c.s_mask[i * WS], mwb = MCS ? 0u : c.s_mask[i * WS + 1];
            CTC_LV(int, pred1);
            CTC_LV(int, pred2);
            CTC_LV(uint32_t, kk1);
            CTC_LV(uint32_t, kk2);
            CTC_LANES {
              const int cha = colc[LX], chb = colc2[LX];
              const bool repa = (cha == ch_i), repb = (chb == ch_i);
              float s1 = f_add(colv[LX], repa ? b_i : sc_i), s2 = f_add(colv2[LX], repb ? b_i : sc_i);
              if (repa && !(b_i > kNInf)) s1 = kNInf;
              if (repb && !(b_i > kNInf)) s2 = kNInf;
              const unsigned k1 = ord_f(s1), k2 = ord_f(s2);
              const bool ma = MCS ? (cha >= 0 && mbit(i, cha)) : (((mwa >> lane) & 1u) != 0u);
              const bool mb2 = MCS ? (chb >= 0 && mbit(i, chb)) : (((mwb >> lane) & 1u) != 0u);
              const bool ok1 = (cha >= 0) && !ma && (k1 >= lo32);
              const bool ok2 = (chb >= 0) && !mb2 && (k2 >= lo32);
              pred1[LX] = ok1 ? 1 : 0; kk1[LX] = k1;
              pred2[LX] = ok2 ? 1 : 0; kk2[LX] = k2;
              if (!select_all) {
                if (ok1) CTC_HIST_ADD(hist0, (k1 - lo32) >> shift32);
                if (ok2) CTC_HIST_ADD(hist0, (k2 - lo32) >> shift32);
              }
            }
            const unsigned bal1 = ctc_ballot(pred1), bal2 = ctc_ballot(pred2);
            const int n1 = ctc_popc(bal1);
            CTC_LANES {
              if (pred1[LX]) {
                const int pos = cnt + ctc_popc(bal1 & ctc_lt_mask(lane));
                if (pos < SEG) { segk[pos] = kk1[LX]; segi[pos] = (i << 16) | lane; }
              }
              if (pred2[LX]) {
                const int pos = cnt + n1 + ctc_popc(bal2 & ctc_lt_mask(lane));
                if (pos < SEG) { segk[pos] = kk2[LX]; segi[pos] = (i << 16) | (32 + lane); }
              }
            }
            cnt += n1 + ctc_popc(bal2);
            CTC_STAT(g_stats.cl_entries += n1 + ctc_popc(bal2));
          }
        }
        if (LM && G == 1) {
          // scorer path, one column group: two rows per iteration and no divergent branch, so that the two dependent
          // chains (shared-memory loads -> dictionary bit -> LM term in double -> key -> histogram -> ballot) overlap
          // -- with two warps per scheduler nothing else hides their latency
          while (rows) {
            const int rl1 = ctc_ffs(rows) - 1;
            rows &= rows - 1u;
            const bool two = rows != 0u;
            const int rl2 = two ? ctc_ffs(rows) - 1 : rl1;
            if (two) rows &= rows - 1u;
            const int i1 = base + (warp - WB0) + NB * rl1, i2 = base + (warp - WB0) + NB * rl2;
            const float sc_1 = c.s_score[i1], b_1 = c.s_bprev[i1], sc_2 = c.s_score[i2], b_2 = c.s_bprev[i2];
            const int ch_1 = c.s_chr[i1], ch_2 = c.s_chr[i2];
            const uint32_t mw1 = c.s_mask[i1 * WS], mw2 = c.s_mask[i2 * WS];
            const uint32_t rm1 = c.s_rmask[i1 * W], rm2 = c.s_rmask[i2 * W];
            CTC_LV(int, pred1);
            CTC_LV(int, pred2);
            CTC_LV(uint32_t, kk1);
            CTC_LV(uint32_t, kk2);
            CTC_LANES {
              const int ch = colc[LX];
              const float l = colv[LX];
              const bool valid = ch >= 0;
              const int chs = valid ? ch : 0;
              const bool rep1 = (ch == ch_1), rep2 = (ch == ch_2);
              float s1 = f_add(l, rep1 ? b_1 : sc_1), s2 = f_add(l, rep2 ? b_2 : sc_2);
              if (rep1 && !(b_1 > kNInf)) s1 = kNInf;
              if (rep2 && !(b_2 > kNInf)) s2 = kNInf;
              const bool okl1 = !c.lm_cut(l, sc_1) && (c.lm_char || ((rm1 >> lane) & 1u) || c.dict_ok(i1, chs));
              const bool okl2 = !c.lm_cut(l, sc_2) && (c.lm_char || ((rm2 >> lane) & 1u) || c.dict_ok(i2, chs));
              const float t1 = c.lm_apply_c(s1, i1, chs), t2 = c.lm_apply_c(s2, i2, chs);
              const bool scored = c.lm_scored(ch);
              s1 = scored ? t1 : s1;
              s2 = scored ? t2 : s2;
              const unsigned k1 = ord_f(s1), k2 = ord_f(s2);
              const bool ok1 = valid && !((mw1 >> lane) & 1u) && (k1 >= lo32) && okl1;
              const bool ok2 = two && valid && !((mw2 >> lane) & 1u) && (k2 >= lo32) && okl2;
              pred1[LX] = ok1 ? 1 : 0; kk1[LX] = k1;
              pred2[LX] = ok2 ? 1 : 0; kk2[LX] = k2;
              if (!select_all) {
                if (ok1) CTC_HIST_ADD(hist0, (k1 - lo32) >> shift32);
                if (ok2) CTC_HIST_ADD(hist0, (k2 - lo32) >> shift32);
              }
            }
            const unsigned bal1 = ctc_ballot(pred1), bal2 = ctc_ballot(pred2);
            const int n1 = ctc_popc(bal1);
            CTC_LANES {
              if (pred1[LX]) {
                const int pos = cnt + ctc_popc(bal1 & ctc_lt_mask(lane));
                if (pos < SEG) { segk[pos] = kk1[LX]; segi[pos] = (i1 << 16) | lane; }
              }
              if (pred2[LX]) {
                const int pos = cnt + n1 + ctc_popc(bal2 & ctc_lt_mask(lane));
                if (pos < SEG) { segk[pos] = kk2[LX]; segi[pos] = (i2 << 16) | lane; }
              }
            }
            cnt += n1 + ctc_popc(bal2);
            CTC_STAT(g_stats.cl_entries += n1 + ctc_popc(bal2));
          }
        }
        while (rows) {
          const int rl = ctc_ffs(rows) - 1;
          rows &= rows - 1u;
          const int i = base + (warp - WB0) + NB * rl;
          const float sc_i = c.s_score[i], b_i = c.s_bprev[i];
          const int ch_i = c.s_chr[i];
          for (int g = 0; g < G; ++g) {
            const uint32_t mw = MCS ? 0u : c.s_mask[i * WS + g];
            const uint32_t rmw = LM ? c.s_rmask[i * W + g] : 0u;
            CTC_LV(int, pred);
            CTC_LV(uint32_t, kk);
            CTC_LANES {
              int ch = colc[LX];
              float l = colv[LX];
              if (g > 0) {  // further groups: load the column on the fly (few rows get here)
                const int r = g * 32 + lane;
                ch = -2;
                l = 0.0f;
                if (r < n) {
                  const int c2 = c.chr_at(r);
                  if (c2 != c.blank) { ch = c2; l = c.lp[r]; }
                }
              }
              const bool rep = (ch == ch_i);
              float sc = f_add(l, rep ? b_i : sc_i);
              if (rep && !(b_i > kNInf)) sc = kNInf;
              bool okl = true;
              if (LM && ch >= 0) {  // cutoff, dictionary arc (unless the child already exists, dead), LM term
                okl = !c.lm_cut(l, sc_i) && (c.lm_char || ((rmw >> lane) & 1u) || c.dict_ok(i, ch));
                if (c.lm_scored(ch)) sc = c.lm_apply_c(sc, i, ch);
              }
              const unsigned k = ord_f(sc);
              const bool mk = MCS ? (ch >= 0 && mbit(i, ch)) : (((mw >> lane) & 1u) != 0u);
              const bool ok = (ch >= 0) && !mk && (k >= lo32) && okl;
              pred[LX] = ok ? 1 : 0;
              kk[LX] = k;
              if (ok && !select_all) CTC_HIST_ADD(hist0, (k - lo32) >> shift32);
            }
            const unsigned bal = ctc_ballot(pred);
            if (bal) {
              CTC_LANES {
                if (pred[LX]) {
                  const int pos = cnt + ctc_popc(bal & ctc_lt_mask(lane));
                  if (pos < SEG) { segk[pos] = kk[LX]; segi[pos] = (i << 16) | (g * 32 + lane); }
                }
              }
              cnt += ctc_popc(bal);
              CTC_STAT(g_stats.cl_entries += ctc_popc(bal));
            }
          }
        }
      }
      CTC_LANES {
        if (lane == 0) {
          if (cnt > SEG) atom_or(&s_ctl[ovf_w], 1);
          c.s_wcnt[warp] = cnt < SEG ? cnt : SEG;
        }
      }
    };
    CTC_TICK(1);  // head (SORTED kernels: + rank table)
    if (!MERGED) {
      CTC_PAR { members_region(tid); }
      CTC_BARRIER_T(2);
      CTC_TICK(2);  // R1
      total = (long long)M * (n_nb + 1) - s_ctl[C_NPAIRS];
      select_all = !LM && total <= (long long)K;
      if (LM) {
        lo32 = (!select_all && M == K) ? (unsigned)s_ctl[C_KMIN] : 0u;
        top32 = (unsigned)s_ctl[C_KMAX];
        // a scored candidate gains its LM term and beta, either of which can be positive: its key is at most its row's
        // bound from region R1 (score + best log-prob + the row's largest positive term) plus max(0, beta).  Every
        // step rounds monotonically, so no key the grid walk bins lies above top32 (it would index past the histogram).
        const double bmax = c.s_ab[1] > 0.0 ? c.s_ab[1] : 0.0;
        const unsigned o = ord_f((float)d_add((double)unord_f((unsigned)s_ctl[C_SMAX]), bmax));
        top32 = o > top32 ? o : top32;
        set_shift();
      }
    }
    for (int attempt = 0;; ++attempt) {
      if (MERGED && attempt == 0) {
        // ---- the front of the frame: members (R1) and grid walk (G) in ONE region; nothing the one writes is read
        //      by the other.  (The emulation runs the halves in either order, CTC_EMU_ORDER bit 2.)
        CTC_HALVES {
          if (half == 0) {
            CTC_PAR { members_region(tid); }
          } else {
            CTC_WARPS {
              if (warp >= WB0) grid_walk(warp, false);
              else { CTC_LANES { if (lane == 0) c.s_wcnt[warp] = 0; } }
            }
          }
        }
        CTC_BARRIER_T(3);
        CTC_TICK(2);  // front: R1 | G
        if (SORTED) {  // (the pairs of this frame were counted by the members' region)
          total = (long long)M * (n_nb + 1) - s_ctl[npairs_w];
          select_all = total <= (long long)K;
        }
      } else {
        if (MERGED) {
          // the tightened second walk of a MERGED kernel: the members re-bin themselves (every thread), the
          // grid-walking warps walk
          CTC_PAR {
            if (!select_all)
              for (int j = tid; j < M; j += NT) {
                const unsigned k = ord_f(c.s_snew[j]);
                if (k >= lo32) CTC_HIST_ADD(hist0, (k - lo32) >> shift32);
              }
          }
        }
        CTC_WARPS {
          if (warp >= WB0) grid_walk(warp, MERGED ? false : rebin);
          else { CTC_LANES { if (lane == 0) c.s_wcnt[warp] = 0; } }
        }
        CTC_BARRIER_T(3);
      }
      // (only where the vocabulary is cut per frame: there the blank / a member's character can drop out of a frame
      // and take the lower bound with it; an index-order kernel keeps its single straight-line walk)
      if (!SORTED || LM || attempt > 0 || select_all || p.force_fallback) break;
      {
        const bool ovf = s_ctl[ovf_w] != 0;
        if (!ovf && !heuristic) break;
        scan_bin_all(hist0, K, pre_bin, pre_above, pre_cnt);
        unsigned lo_new;
        if (pre_above + pre_cnt < K) {
          lo_new = lo_valid;                 // the heuristic bound cut too deep: walk again with the proven one
          CTC_STAT(g_stats.heur_fail++);
        } else if (ovf) {
          lo_new = lo32 + ((unsigned)pre_bin << shift32);
          if (lo_new == lo32) break;         // nothing to gain: grid-walking fallback
        } else {
          have_scan = true;                  // bound holds, lists fit: the select continues from this scan
          break;
        }
        CTC_BARRIER();  // every warp has scanned the histogram
        CTC_PAR {
          for (int x = tid; x < kNBins; x += NT) hist0[x] = 0;
          if (tid == 0) s_ctl[ovf_w] = 0;
        }
        CTC_BARRIER();
        lo32 = lo_new;
        heuristic = false;
        set_shift();
        rebin = true;
        CTC_STAT(g_stats.rewalks++);
      }
    }
    // ---- cut-vocabulary MERGED kernels: the rank table of frame t + 1 (its row is already staged; at a tile boundary
    //      the tile was requested a whole tile ago), into the table the members' region of this frame cleared
    if (MERGED && SORTED && t + 1 < Tb) {
#if defined(CTC_EMULATE)
      const float *nrow = p.lp + ((size_t)bi * p.T + t0 + t + 1) * NP;
      const uint16_t *nidx = p.idx + ((size_t)bi * p.T + t0 + t + 1) * NP;
#else
      int ft2 = ft, tile2 = tile;
      if (ft2 == F) { ft2 = 0; ++tile2; mbar_wait(&mbar[tile2 & 1], (uint32_t)((tile2 >> 1) & 1)); }
      const float *nrow = tile_lp + ((size_t)(tile2 & 1) * F + ft2) * NP;
      const uint16_t *nidx = tile_idx + ((size_t)(tile2 & 1) * F + ft2) * NP;
#endif
      const int n_next = (int)(f_bits(nrow[NP - 2]) & 0xFFFFu);
      int16_t *const rn = rank_base + (par ^ 1) * VR;
      CTC_PAR {
        for (int r = tid; r < n_next; r += NT) rn[nidx[r]] = (int16_t)r;
      }
    }
    CTC_TICK(3);  // G
    bool fallback = s_ctl[ovf_w] != 0 || p.force_fallback;  // a segment overflowed (twice): redo on the grid
    CTC_STAT(g_stats.fb_frames += fallback);

    // ================= the barrier-free back half (FASTB kernels, common frame) ===========================
    // Taken when: the beam is full, no dead anchor is in the table, no list overflowed and every list segment fits
    // one ballot, and ONE radix pass settles the cut (the bin of the K-th key holds selected keys only -- which also
    // checks the heuristic bound).  Every warp scans the histogram, then classifies ALL members and ALL list
    // entries itself: evw[] / selw[] end up identical in every warp's registers, so slot owners can rank their slot
    // among the evicted ones and pick their candidate without any exchange.  What a slot owner reads of OTHER
    // slots in this region is not written in it: new scores (s_snew), list entries, the old beam's links, and
    // node id / depth of a parent -- a new member's own node id / depth therefore wait in s_nodeN / s_depthN until
    // the next frame's region R1.
    int *const npslot = pslot_base + (cur ^ 1) * KP, *const nanch = anch_base + (cur ^ 1) * KP;
    int nrev = 0;
    bool fastb = false;
    unsigned thr_hi = 0u, thr_code = 0u;
    if (FASTB) {
      fastb = !(p.no_fast & 1) && !fallback && nlive == 0 && M == K && !select_all;
      CTC_STAT(g_stats.nf_anchor += (nlive != 0));
      CTC_STAT(g_stats.nf_notfull += (M != K || select_all));
      if (fastb) {
#pragma unroll
        for (int q = 0; q < NB; ++q) fastb = fastb && c.s_wcnt[WB0 + q] <= 32 * CH;
        CTC_STAT(g_stats.nf_seg += !fastb);
      }
      bool inbin = false;  // the K-th key shares its bin: rank the bin's keys (FAST2)
      if (fastb) {
        scan_bin_all(hist0, K, pre_bin, pre_above, pre_cnt);
        have_scan = true;
        fastb = (pre_above + pre_cnt == K);
        if (FAST2 && !fastb && pre_above + pre_cnt > K && pre_cnt <= 32 && !(p.no_fast & 4)) { fastb = true; inbin = true; }
        CTC_STAT(g_stats.nf_pass += !fastb);
        CTC_STAT(g_stats.nf_pass_cnt += fastb ? 0 : pre_cnt);
      }
      // selected <=> 48-bit key >= (thr_hi, thr_code): score key, then smaller character first.  One radix pass:
      // the lower edge of the K-th key's bin, any character.
      thr_hi = lo32 + ((unsigned)pre_bin << shift32);
      thr_code = 0u;
      if (CTC_UNLIKELY(FAST2 && fastb && inbin)) {
        // ---- the bin [thr_hi, thr_hi + 2^shift32) holds pre_cnt <= 32 keys of which K - pre_above are selected: every
        //      warp gathers them (members' keys need their character, list entries the character of their column)
        //      into a scratch row of its own and ranks them by counting; the key of rank K - pre_above - 1 is the
        //      threshold.  Two equal keys there (comparator-equal prefixes at the cut: the reference's choice is
        //      unspecified) leave the frame to the general back half and its tie handling.
        const int need = K - pre_above;
        const unsigned bw = 1u << shift32;
        bool ok2 = true;
        unsigned t_hi = thr_hi, t_code = 0u;
        CTC_WARPS {
          uint64_t *const scr2 = reinterpret_cast<uint64_t *>(c.s_sel) + warp * 32;
          int n = 0;
#pragma unroll
          for (int blk = 0; blk < KPW; ++blk) {
            CTC_LV(int, inb);
            CTC_LV(uint64_t, kk);
            CTC_LANES {
              const int j = blk * 32 + lane;
              inb[LX] = 0; kk[LX] = 0ull;
              if (j < K) {
                const unsigned k = ord_f(c.s_snew[j]);
                if (k >= thr_hi && k - thr_hi < bw) { inb[LX] = 1; kk[LX] = ((uint64_t)k << 16) | (uint64_t)(unsigned)s_code[j]; }
              }
            }
            const unsigned bl = ctc_ballot(inb);
            CTC_LANES { if (inb[LX]) { const int pos = n + ctc_popc(bl & ctc_lt_mask(lane)); if (pos < 32) scr2[pos] = kk[LX]; } }
            n += ctc_popc(bl);
          }
#pragma unroll
          for (int q = 0; q < NB; ++q) {
            const int cn = c.s_wcnt[WB0 + q];
#pragma unroll
            for (int h = 0; h < CH; ++h) {
              if (h > 0 && cn <= 32 * h) break;
              CTC_LV(int, inb);
              CTC_LV(uint64_t, kk);
              CTC_LANES {
                const int e = 32 * h + lane;
                inb[LX] = 0; kk[LX] = 0ull;
                if (e < cn) {
                  const unsigned k = c.s_clk[(WB0 + q) * SEG + e];
                  if (k >= thr_hi && k - thr_hi < bw) {
                    const int r = c.s_cli[(WB0 + q) * SEG + e] & 0xFFFF;
                    inb[LX] = 1; kk[LX] = ((uint64_t)k << 16) | (uint64_t)(0xFFFF - (c.chr_at(r) + 1));
                  }
                }
              }
              const unsigned bl = ctc_ballot(inb);
              CTC_LANES { if (inb[LX]) { const int pos = n + ctc_popc(bl & ctc_lt_mask(lane)); if (pos < 32) scr2[pos] = kk[LX]; } }
              n += ctc_popc(bl);
            }
          }
          CTC_SYNCWARP();
          CTC_LV(int, hit);
          CTC_LV(uint64_t, mykey);
          CTC_LANES {
            hit[LX] = 0; mykey[LX] = 0ull;
            if (n == pre_cnt && lane < n) {
              const uint64_t mk = scr2[lane];
              int rank = 0, eq = 0;
              for (int i = 0; i < n; ++i) {
                const uint64_t o = scr2[i];
                rank += (o > mk) ? 1 : 0;
                eq += (o == mk) ? 1 : 0;
              }
              mykey[LX] = mk;
              hit[LX] = (rank == need - 1 && eq == 1) ? 1 : 0;
            }
          }
          const unsigned hb = ctc_ballot(hit);
          if (ctc_popc(hb) != 1) {
            ok2 = false;
          } else {
            const uint64_t tk = ctc_shfl64(mykey, ctc_ffs(hb) - 1);
            t_hi = (unsigned)(tk >> 16); t_code = (unsigned)(tk & 0xFFFFull);
          }
          CTC_SYNCWARP();  // (the scratch rows alias the general path's lists: every lane is done reading)
        }
        if (ok2) { thr_hi = t_hi; thr_code = t_code; }
        else { fastb = false; CTC_STAT(g_stats.nf_pass++); }
        CTC_STAT(g_stats.fast2_frames += ok2);
      }
    }
    if (CTC_LIKELY(FASTB && fastb)) {
      CTC_STAT(g_stats.passes++);
      CTC_STAT(g_stats.fast_frames++);
      // is the key (k, character ch) selected?  (the character is only looked at for a key equal to the threshold's)
      // (thr_code != 0 only in a frame that ranked a shared bin -- uniform, so the code is not even loaded otherwise)
      const bool two = FAST2 && thr_code != 0u;
      CTC_TICK(14);  // fast back half: checks + histogram scan
      int nsel_f = 0;
      CTC_WARPS {
        unsigned evw[KPW > 0 ? KPW : 1];
#pragma unroll
        for (int blk = 0; blk < KPW; ++blk) {
          CTC_LV(int, ev);
          CTC_LANES {
            const int j = blk * 32 + lane;
            ev[LX] = 0;
            if (j < K) {
              const unsigned k = ord_f(c.s_snew[j]);
              ev[LX] = (k > thr_hi || (k == thr_hi && (!two || (unsigned)s_code[j] >= thr_code))) ? 0 : 1;
            }
          }
          evw[blk] = ctc_ballot(ev);
        }
        // this warp's word of the evicted-slot bitmap, the number of evicted slots below its first slot, and the total
        // (= the number of selected candidates: the beam is full)
        unsigned mine = evw[0];
        int base_w = 0, nsel = 0;
#pragma unroll
        for (int bq = 0; bq < KPW; ++bq) {
          mine = (bq == warp) ? evw[bq] : mine;
          base_w += (bq < warp) ? ctc_popc(evw[bq]) : 0;
          nsel += ctc_popc(evw[bq]);
        }
        if (warp >= KPW) mine = 0u;
        const int cnt_w = ctc_popc(mine);
        // The r-th selected list entry (segments in warp order, entries in list order) moves into the r-th evicted
        // slot.  Each slot-owning warp copies the entries its own slots take -- ranks [base_w, base_w + cnt_w) -- into
        // a scratch row of its own, so nothing but a __syncwarp lies between classification and commit.
        int *const scr = c.s_newinfo + (warp < KPW ? warp : 0) * 64;
        if (cnt_w > 0) {
          int acc = 0;
#pragma unroll 1
          for (int q = 0; q < NB; ++q) {
            const int cn = c.s_wcnt[WB0 + q];
#pragma unroll
            for (int h = 0; h < CH; ++h) {
              if (h > 0 && cn <= 32 * h) break;  // (warp-uniform)
              CTC_LV(int, sl);
              CTC_LV(uint32_t, kv);
              CTC_LANES {
                const int e = 32 * h + lane;
                kv[LX] = e < cn ? c.s_clk[(WB0 + q) * SEG + e] : 0u;
                sl[LX] = 0;
                if (e < cn)
                  sl[LX] = (kv[LX] > thr_hi ||
                            (kv[LX] == thr_hi &&
                             (!two || (unsigned)(0xFFFF - (c.chr_at(c.s_cli[(WB0 + q) * SEG + e] & 0xFFFF) + 1)) >= thr_code))) ? 1 : 0;
              }
              const unsigned sb = ctc_ballot(sl);
              CTC_LANES {
                if (sl[LX]) {
                  const int rk = acc + ctc_popc(sb & ctc_lt_mask(lane)) - base_w;
                  if (rk >= 0 && rk < cnt_w) {
                    scr[2 * rk] = c.s_cli[(WB0 + q) * SEG + 32 * h + lane];
                    scr[2 * rk + 1] = (int)kv[LX];
                  }
                }
              }
              acc += ctc_popc(sb);
            }
          }
          if (acc != nsel) { CTC_LANES { if (lane == 0) s_ctl[C_FLAGS] |= FLAG_ERR_ARENA; } }  // cannot happen
          CTC_SYNCWARP();
        }
        if (head_offload && warp == WB0 && t + 1 < Tb) {
          // ---- this warp owns no slots: while the owners commit, it works out the NEXT frame's key range.  The
          //      new beam's score range follows from what was just classified (kept members' new scores, selected
          //      candidates' keys), the next row is already staged (at a tile boundary the tile was requested a
          //      whole tile ago) -- so the head of frame t + 1 costs the slot owners nothing.
          CTC_LV(unsigned, kmn);
          CTC_LV(unsigned, kmx);
          CTC_LANES {
            kmn[LX] = 0xFFFFFFFFu; kmx[LX] = 0u;
#pragma unroll
            for (int blk = 0; blk < KPW; ++blk) {
              const int j = blk * 32 + lane;
              if (j < K) {
                const unsigned k = ord_f(c.s_snew[j]);
                if (k > thr_hi || (k == thr_hi && (!two || (unsigned)s_code[j] >= thr_code))) { kmn[LX] = k < kmn[LX] ? k : kmn[LX]; kmx[LX] = k > kmx[LX] ? k : kmx[LX]; }
              }
            }
#pragma unroll
            for (int q = 0; q < NB; ++q) {
#pragma unroll
              for (int h = 0; h < CH; ++h) {
                if (32 * h + lane < c.s_wcnt[WB0 + q]) {
                  const unsigned k = c.s_clk[(WB0 + q) * SEG + 32 * h + lane];
                  if (k > thr_hi || (k == thr_hi && (!two || (unsigned)(0xFFFF - (c.chr_at(c.s_cli[(WB0 + q) * SEG + 32 * h + lane] & 0xFFFF) + 1)) >= thr_code))) {
                    kmn[LX] = k < kmn[LX] ? k : kmn[LX]; kmx[LX] = k > kmx[LX] ? k : kmx[LX];
                  }
                }
              }
            }
          }
          const unsigned nmin = ctc_warp_min(kmn), nmax = ctc_warp_max(kmx);
#if defined(CTC_EMULATE)
          const float *nrow = p.lp + ((size_t)bi * p.T + t0 + t + 1) * NP;
#else
          int ft2 = ft, tile2 = tile;
          if (ft2 == F) { ft2 = 0; ++tile2; mbar_wait(&mbar[tile2 & 1], (uint32_t)((tile2 >> 1) & 1)); }
          const float *nrow = tile_lp + ((size_t)(tile2 & 1) * F + ft2) * NP;
#endif
          unsigned hlo, htop, hlov;
          bool hheur;
          head_of(nrow, nmin, nmax, true, hlo, htop, hlov, hheur);
          CTC_LANES {
            if (lane == 0) {
              int *hb = c.s_wcnt + 64 + 8 * (par ^ 1);
              hb[0] = (int)hlo; hb[1] = (int)htop; hb[2] = (int)hlov; hb[3] = hheur ? 1 : 0;
            }
          }
        }
        CTC_TICK(6);  // fast back half: evicted / selected ballots, scratch rows
        // is beam slot x evicted in this frame?  (x < KP.  The bitmap is packed into 64-bit scalars and picked by
        // selects on the bits of x: an indexed evw[x >> 5] would put the array into local memory)
        const uint64_t w01 = (uint64_t)evw[0] | (KPW > 1 ? (uint64_t)evw[KPW > 1 ? 1 : 0] << 32 : 0ull);
        const uint64_t w23 = KPW > 2 ? ((uint64_t)evw[KPW > 2 ? 2 : 0] | (KPW > 3 ? (uint64_t)evw[KPW > 3 ? 3 : 0] << 32 : 0ull)) : 0ull;
        const uint64_t w45 = KPW > 4 ? ((uint64_t)evw[KPW > 4 ? 4 : 0] | (KPW > 5 ? (uint64_t)evw[KPW > 5 ? 5 : 0] << 32 : 0ull)) : 0ull;
        const uint64_t w67 = KPW > 6 ? ((uint64_t)evw[KPW > 6 ? 6 : 0] | (KPW > 7 ? (uint64_t)evw[KPW > 7 ? 7 : 0] << 32 : 0ull)) : 0ull;
        auto evbit = [&](int x) -> bool {
          uint64_t a = (KPW > 2 && (x & 64)) ? w23 : w01;
          if (KPW > 4) {
            const uint64_t b = (x & 64) ? w67 : w45;
            a = (x & 128) ? b : a;
          }
          return (a >> (x & 63)) & 1ull;
        };
        CTC_LV(unsigned, cmin);
        CTC_LV(unsigned, cmax);
        CTC_LV(int, pair);
        CTC_LANES {
          cmin[LX] = 0xFFFFFFFFu; cmax[LX] = 0u; pair[LX] = 0;
          const int j = warp * 32 + lane;
          if (warp < KPW && j < K) {
            int newp = -1, res = -1, start = 0, ch_mine;
            bool resolved = false;
            const bool ev = (mine >> lane) & 1u;
            if (!ev) {
              // the member stays: roll cur -> prev (reference path_trie.cpp:129-137)
              c.s_bprev[j] = c.s_bnew[j];
              c.s_nbprev[j] = c.s_nbnew[j];
              const float sn = c.s_snew[j];
              c.s_score[j] = sn;
              cmin[LX] = cmax[LX] = ord_f(sn);
              ch_mine = c.s_chr[j];
              const int pq = c.s_pslot[j];
              if (pq >= 0) {
                if (!evbit(pq)) { newp = pq; resolved = true; }
                start = pq;
              } else {
                const int a = c.s_anch[j];
                if (a < 0) { resolved = true; }
                else {
                  const int q = c.s_dpslot[a];
                  if (!evbit(q)) { res = a; resolved = true; }
                  start = q;
                }
              }
            } else {
              // evicted: write back lpc / timestep, remember what a dead anchor made of this node would need ...
              CTC_STAT(g_stats.evicted++);
              flush_lpc_ts(&nodes[c.s_node[j]], c.s_lpc[j], c.s_ts[j]);
              c.s_stash[j] = c.s_node[j]; c.s_stash[KP + j] = c.s_chr[j];
              c.s_stash[2 * KP + j] = (int)f_bits(c.s_lpc[j]); c.s_stash[3 * KP + j] = c.s_ts[j];
              c.s_stash[4 * KP + j] = 0;
              // ... and take the q-th selected candidate, q = rank of this slot among the evicted ones
              // (reference path_trie.cpp:97-105 create); its score is the list key
              const int qloc = ctc_popc(mine & ctc_lt_mask(lane));  // rank among this warp's evicted slots
              const int id = scr[2 * qloc];
              const float sc = unord_f((uint32_t)scr[2 * qloc + 1]);
              const int par_slot = id >> 16, r = id & 0xFFFF;
              const int ch = c.chr_at(r);
              const float lpc = c.lp[r];
              CTC_STAT(g_stats.created++);
              // node ids follow the rank of the slot among the evicted slots: no atomic, and the arena is filled the
              // same way on every run
              int nid = nnodes + base_w + qloc;
              if (nid >= arena_cap) {  // cannot happen with capacity 1 + K * frames; never write out of bounds
                s_ctl[C_FLAGS] |= FLAG_ERR_ARENA;
                nid = arena_cap - 1;
              }
              const int pnode = c.s_node[par_slot], pdepth = c.s_depth[par_slot];
              Node nn; nn.parent = pnode; nn.chr = ch; nn.lpc = lpc; nn.ts = t_abs;
              nn.jump = jump_of_child(pnode, pdepth, s_jump[par_slot]);
              store_node(&nodes[nid], nn);
              s_nodeN[j] = nid; s_depthN[j] = pdepth + 1; s_jumpN[j] = nn.jump;
              c.s_chr[j] = ch;
              c.s_bprev[j] = kNInf; c.s_nbprev[j] = sc; c.s_score[j] = sc;  // score = lse(-inf, nb)
              cmin[LX] = cmax[LX] = ord_f(sc);
              c.s_lpc[j] = lpc; c.s_ts[j] = t_abs;
              ch_mine = ch;
              start = par_slot;
              if (!evbit(start)) { newp = start; resolved = true; }
            }
            if (!resolved) {
              int cs = start;  // an old slot evicted in this frame
              while (true) {
                CTC_STAT(g_stats.walk_iters++);
                const int pq = c.s_pslot[cs];
                if (pq >= 0) {
                  if (!evbit(pq)) { res = KP2 + cs; break; }
                  cs = pq;
                  continue;
                }
                const int a = c.s_anch[cs];
                if (a < 0) { res = -1; break; }
                const int q = c.s_dpslot[a];
                if (!evbit(q)) { res = a; break; }
                cs = q;
              }
            }
            if (res >= 0) { atom_add(&c.s_cnt2[res], 1); s_ctl[anyref_w] = 1; }
            npslot[j] = newp;
            nanch[j] = res;
            c.s_evict[j] = ev ? 1 : 0;
            if (newp >= 0) {  // the "existing child" mask of the next frame (ch_mine >= 0: only the root has none)
              atom_or(&mask_next[newp * WS + (ch_mine >> 5)], 1u << (ch_mine & 31));
              pair[LX] = SORTED ? 0 : 1;  // (cut-vocabulary kernels count pairs per frame, in region R1)
            }
          }
        }
        CTC_TICK(7);  // fast back half: slot owners commit
        // what the next frame needs before its first region: pair count, score range of the new beam
        const unsigned pb = ctc_ballot(pair);
        if (!(head_offload && t + 1 < Tb)) {  // (otherwise a grid-walking warp has the next frame's range from the ballots)
          const unsigned mn = ctc_warp_min(cmin), mx = ctc_warp_max(cmax);
          CTC_LANES {
            c.s_wcnt[128 + 64 * (par ^ 1) + warp] = (int)mn;        // (every lane stores the same word, see
            c.s_wcnt[128 + 64 * (par ^ 1) + 32 + warp] = (int)mx;   //  warp_range_store)
          }
        }
        CTC_LANES {
          if (lane == 0 && pb) atom_add(&s_ctl[npairs_nx], ctc_popc(pb));
#pragma unroll 1
          for (int x = warp * 32 + lane; x < KP * WS; x += NT) c.s_mask[x] = 0u;  // this frame's masks: used up
          if (warp == NW - 1 && lane == 0) { s_ctl[ovf_nx] = 0; s_ctl[anyref_nx] = 0; }
        }
        nsel_f = nsel;  // (the same in every warp)
      }
      nnodes += nsel_f;
      nn_stale = true;
      head_ready = head_offload && t + 1 < Tb;
    } else {
    // ================= the general back half ===============================================================
#if defined(CTC_OPT_BLOAT) && !defined(CTC_EMULATE)
    if (p.no_fast == 0x7fffff01) {  // (never: a measurement build carries the block twice)
#include "beam_general_back_half.inc"
    }
#endif
#include "beam_general_back_half.inc"
    }  // general back half
    CTC_BARRIER_T(8);
    CTC_TICK(8);  // R5
    if (MERGED && !fastb) { nnodes = s_ctl[C_NNODES]; nn_stale = false; }
    const int M_new = select_all ? (int)total : K;
    const bool anchors_active = nlive > 0 || nrev > 0 || s_ctl[anyref_w] != 0;
    int nlive_next = 0;

    if (CTC_UNLIKELY(anchors_active)) {
      // ---- region R5b: dead anchors nobody hangs below any more leave the trie (that IS the reference's
      //      remove()); anchors whose parent left the beam stop being anchors.
      CTC_PAR {
        for (int a = tid; a < KP2; a += NT) {
          const int q = c.s_dpslot[a];
          if (q >= 0) {
            const bool keep = CTC_PARENT_ALIVE(q) && c.s_cnt2[a] > 0 && !c.s_drev[a];
            if (!keep) {
              if (!c.s_drev[a]) flush_lpc_ts(&nodes[c.s_dnode[a]], c.s_dlpc[a], c.s_dts[a]);
              c.s_dpslot[a] = -1;
            } else {
              CTC_STAT(g_stats.anchors_live++);
              atom_add(&s_ctl[C_NLIVE], 1);
            }
          }
          if (c.s_dpslot[a] < 0) c.s_efree[atom_add(&s_ctl[C_NEFREE], 1)] = a;
        }
      }
      CTC_BARRIER();
      CTC_TICK(9);  // R5b

      // ---- region R5c: members evicted now that still have beam members below them and whose parent
      //      stays become dead anchors (reference: exists_ = false, node stays in the trie)
      CTC_PAR {
        const int nefree = s_ctl[C_NEFREE];
        for (int e = tid; e < M; e += NT) {
          if (c.s_evict[e] && c.s_cnt2[KP2 + e] > 0) {
            const int k = atom_add(&s_ctl[C_NETAKEN], 1);
            int a = 0;
            if (k < nefree) a = c.s_efree[k];
            else s_ctl[C_FLAGS] |= FLAG_ERR_ARENA;
            CTC_STAT(g_stats.anchors_new++);
            atom_add(&s_ctl[C_NLIVE], 1);
            c.s_dnode[a] = c.s_stash[e]; c.s_dchr[a] = c.s_stash[KP + e]; c.s_dpslot[a] = c.s_pslot[e];
            c.s_dlpc[a] = bits_f((uint32_t)c.s_stash[2 * KP + e]); c.s_dts[a] = c.s_stash[3 * KP + e];
            c.s_ddstate[a] = c.s_stash[4 * KP + e];
            c.s_amap[e] = a;
          }
        }
      }
      CTC_BARRIER();
      CTC_TICK(10);  // R5c
      nlive_next = s_ctl[C_NLIVE];
      // ---- region R5d: provisional anchor codes become table indices; in-frame tags are dropped
      CTC_PAR {
        for (int j = tid; j < M_new; j += NT) {
          const int ra = nanch[j];
          if (ra >= KP2) nanch[j] = c.s_amap[ra - KP2];
        }
        for (int a = tid; a < KP2; a += NT) {
          const int q = c.s_dpslot[a];
          if (q >= 0) c.s_dpslot[a] = q & ~kNewFlag;
          c.s_drev[a] = 0;
        }
        for (int x = tid; x < 3 * KP; x += NT) c.s_cnt2[x] = 0;
        if (tid == 0) { s_ctl[C_NEFREE] = 0; s_ctl[C_NETAKEN] = 0; }
      }
      CTC_BARRIER();
    }
    CTC_TICK(11);  // R5d
    cur ^= 1;
    par ^= 1;
    c.s_pslot = pslot_base + cur * KP;
    c.s_anch = anch_base + cur * KP;
    nlive = nlive_next;
    M = M_new;
    if (LM && p.lm_persistent && (t + 1 < Tb || p.lm_hs_last)) {
      // ---- scorer path, persistent mode: hand the new nodes to the host, wait for their LM terms -----------
#if defined(CTC_EMULATE)
      p.emu_handshake(p.emu_ctx, b);
#else
      if (threadIdx.x == 0) {
        __threadfence_system();  // the new-node list (written before the barriers above) before the flag
        *(volatile int *)&newlist[1] = t0 + t + 1;
      }
#endif
      lm_fetch_updates(t0 + t + 1);
      CTC_BARRIER();
      CTC_TICK(12);  // handshake: fence, flag, wait for the host, fetch its answer
      CTC_PAR {
        lm_scatter_updates(tid);  // into the per-node array (read again when a node is revived or a launch starts)
        // ... and into the slots of the members the pairs are about, straight from the staged answer: continuing members
        // keep their term, so nothing waits for the array in global memory
        if (!p.lm_char) {
          const int nu = s_upd[1];
          for (int j = tid; j < M; j += NT) {
            const int node = c.s_node[j];
            for (int q = 0; q < nu; ++q)
              if (s_upd[2 + 2 * q] == node) c.s_lmsp[j] = bits_f((uint32_t)s_upd[3 + 2 * q]);
          }
        }
      }
      CTC_BARRIER();
      CTC_TICK(13);  // LM terms in
    }
    CTC_STAT(g_stats.frames++);
    CTC_STAT(g_stats.sel_all_frames += select_all);
  }
#undef CTC_PARENT_ALIVE

  // ---- region: store the beam state (streaming continues from here; the finalize kernel reads it) and
  //      bring the arena's lpc / timestep up to date for everything still held in shared memory
  CTC_PAR {
    int *s = st_slots;
    for (int j = tid; j < K; j += NT) {
      if (FASTB && s_nodeN[j] >= 0) { c.s_node[j] = s_nodeN[j]; c.s_depth[j] = s_depthN[j]; s_jump[j] = s_jumpN[j]; s_nodeN[j] = -1; }
      s[j] = c.s_node[j]; s[K + j] = c.s_chr[j]; s[2 * K + j] = c.s_depth[j];
      s[3 * K + j] = (int)f_bits(c.s_bprev[j]); s[4 * K + j] = (int)f_bits(c.s_nbprev[j]);
      s[5 * K + j] = (int)f_bits(c.s_score[j]); s[6 * K + j] = (int)f_bits(c.s_lpc[j]); s[7 * K + j] = c.s_ts[j];
      s[8 * K + j] = c.s_pslot[j]; s[9 * K + j] = c.s_anch[j]; s[10 * K + j] = c.s_dstate[j]; s[11 * K + j] = s_jump[j];
      if (j < M) flush_lpc_ts(&nodes[c.s_node[j]], c.s_lpc[j], c.s_ts[j]);
    }
    for (int a = tid; a < KP2; a += NT) {
      st_anchors[a] = c.s_dnode[a]; st_anchors[KP2 + a] = c.s_dchr[a]; st_anchors[2 * KP2 + a] = c.s_dpslot[a];
      st_anchors[3 * KP2 + a] = (int)f_bits(c.s_dlpc[a]); st_anchors[4 * KP2 + a] = c.s_dts[a];
      st_anchors[5 * KP2 + a] = c.s_ddstate[a];
      if (c.s_dpslot[a] >= 0) flush_lpc_ts(&nodes[c.s_dnode[a]], c.s_dlpc[a], c.s_dts[a]);
    }
    if (tid == 0) {
      st[0] = M; st[1] = MERGED ? nnodes : s_ctl[C_NNODES]; st[2] = abs_t0 + Tb; st[3] = s_ctl[C_FLAGS];
    }
  }
#if !defined(CTC_EMULATE)
  if (TIMING && p.timing) {  // [B][16] region cycles of thread 0, then [B][16][32] busy cycles per region and warp
    if (threadIdx.x == 0)
      for (int x = 0; x < 16; ++x) p.timing[(size_t)b * 16 + x] = s_tick[x];
    __syncthreads();
    for (int x = threadIdx.x; x < 16 * 32; x += NT)
      p.timing[(size_t)gridDim.x * 16 + (size_t)b * 16 * 32 + x] = s_wbusy[x];
  }
#endif
  if (MERGED && p.backtrace) {
    // the backtrace of this utterance, by this CTA, while other CTAs still run their frames: no finalize launch, and
    // only the last CTA's backtrace is left exposed.  It reads the state block stored above and takes the slot block
    // of shared memory (the head keeps the tile barriers and the timing counters; the host checks the size).
    CTC_BARRIER();
    finalize_cta_run<NT>(p, b, smem + kSmemHead);
  }
}

// ======================================================================================================
//  finalize_cta_run: DecoderState::decode + get_beam_search_result + the write-back of binding.cpp
//  (reference ctc_beam_search_decoder.cpp:164-211, decoder_utils.cpp:48-73, path_trie.cpp:109-126,
//   binding.cpp:79-99).  Sorts the <= K members by (score desc, char asc), walks each prefix up the
//   trie, writes only [:len] of each row; rows >= n_results are left untouched like the reference.
//
//  The walk is a pointer chase through an arena of hundreds of megabytes: every hop is a DRAM round trip.  Instead
//  of len dependent hops per prefix, a thread per prefix follows the JUMP pointers (Node::jump: the ancestor at the
//  last multiple of kJump in depth) and records up to R checkpoints; then every (prefix, checkpoint) pair is an
//  independent stretch of at most kJump hops, spread over all threads.  Rounds repeat until every prefix reached
//  the root: len / kJump + kJump dependent hops instead of len.
// ======================================================================================================
CTC_HD int finalize_rounds_cap(int K) {  // checkpoints per prefix and round: whatever 32 KB of shared memory hold
  int R = 8192 / (K > 0 ? K : 1);
  return R < 1 ? 1 : (R > 16 ? 16 : R);
}
CTC_HD size_t finalize_smem_bytes(int K) {
  // keys [K] u64, order [K], flag, cur node [K], cur depth [K], checkpoint count [K], checkpoints [K][R]
  return (size_t)K * 8 + (size_t)K * 4 * 4 + (size_t)K * finalize_rounds_cap(K) * 4 + 64;
}
// Does a one-launch offline decode run the backtrace in the beam kernel's epilogue (BeamParams::backtrace)?  Index-order
// kernels without a scorer do, in the shared memory behind the layout's head (the slot block alone is larger).
CTC_HD bool cta_backtrace(bool sorted, int K, const SmemLayout &L) {
  return !sorted && kSmemHead + finalize_smem_bytes(K) <= (size_t)L.total;
}
template <int NT>
CTC_FN void finalize_cta_run(const BeamParams &p, const int b, unsigned char *smem) {
  const int K = p.K;
  const Node *const nodes = p.arena_ptrs ? p.arena_ptrs[b] : p.arena + (long long)b * p.arena_stride;
  int *const st = p.state_ptrs ? p.state_ptrs[b] : p.state + (long long)b * p.state_stride;
  if (p.finalize && !p.finalize[b]) return;
  const int M = st[0];
  const int *s = st + kStateHeader;
  const int R = finalize_rounds_cap(K);
  uint64_t *s_key = (uint64_t *)smem;             // [K]
  int *s_order = (int *)(smem + (size_t)K * 8);   // [K]
  int *s_cur = s_order + K, *s_dep = s_cur + K, *s_ncp = s_dep + K;  // [K] each, by output row
  int *s_cp = s_ncp + K;                          // [K][R] checkpoint node ids
  int *s_flag = s_cp + (size_t)K * R;             // [0] tie flag, [1] deepest prefix
  CTC_PAR {
    for (int j = tid; j < M; j += NT) s_key[j] = key64(bits_f((uint32_t)s[5 * K + j]), s[K + j]);
    if (tid == 0) { s_flag[0] = 0; s_flag[1] = 0; }
  }
  CTC_BARRIER();
  CTC_PAR {
    for (int j = tid; j < M; j += NT) {
      const uint64_t k = s_key[j];
      int rk = 0, tie = 0;
      for (int x = 0; x < M; ++x) {
        const uint64_t kx = s_key[x];
        rk += (kx > k || (kx == k && x < j)) ? 1 : 0;
        tie |= (kx == k && x != j) ? 1 : 0;
      }
      s_order[rk] = j;
      if (tie) s_flag[0] = 1;  // benign race: all writers store 1
    }
  }
  CTC_BARRIER();
  CTC_PAR {
    int dmax = 0;
    for (int q = tid; q < M; q += NT) {
      const int j = s_order[q];
      const int depth = s[2 * K + j];
      const float score = bits_f((uint32_t)s[5 * K + j]);
      p.out_scores[(size_t)b * K + q] = (float)(-(double)score);  // decoder_utils.cpp:68, binding.cpp:91
      p.out_lens[(size_t)b * K + q] = depth;
      s_cur[q] = s[j];
      s_dep[q] = depth;
      dmax = depth > dmax ? depth : dmax;
    }
    if (dmax > 0) atom_max_i(&s_flag[1], dmax);
    if (tid == 0) {
      p.n_results[b] = M;
      int f = st[3] | (s_flag[0] ? FLAG_TIE_FINAL : 0);
      atom_or(&p.flags[b], f);
    }
  }
  CTC_BARRIER();
  const int rounds = ((s_flag[1] + kJump - 1) / kJump + R - 1) / R;  // a prefix of depth d has ceil(d / kJump) checkpoints
  for (int rd = 0; rd < rounds; ++rd) {
    // (a) one thread per prefix: up to R checkpoints along the jump pointers
    CTC_PAR {
      for (int q = tid; q < M; q += NT) {
        int nid = s_cur[q], d = s_dep[q], k = 0;
        while (k < R && d > 0) {
          s_cp[(size_t)q * R + k] = nid;
          nid = ld_cg(&nodes[nid].jump);
          d = ((d - 1) / kJump) * kJump;
          ++k;
        }
        s_ncp[q] = k;
        s_cur[q] = nid;  // (s_dep[q] is advanced after the stretches below have read it)
      }
    }
    CTC_BARRIER();
    // (b) every (prefix, checkpoint) pair: the stretch of at most kJump nodes below the checkpoint's jump target.
    // Each thread walks U stretches in lockstep, so that a CTA of fewer than 1024 threads (the beam kernel's own
    // backtrace) keeps as many independent hops in flight as the 1024-thread finalize kernel.
    constexpr int U = NT >= 1024 ? 1 : 1024 / NT;
    CTC_PAR {
      for (int it0 = tid; it0 < M * R; it0 += U * NT) {
        int nid[U], d[U], dend[U];
        size_t row[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int it = it0 + u * NT;
          const int q = it / R, k = it - q * R;
          d[u] = 0; dend[u] = 0; nid[u] = 0; row[u] = 0;
          if (it >= M * R || k >= s_ncp[q]) continue;
          const int d0 = s_dep[q];
          d[u] = (k == 0) ? d0 : ((d0 - 1) / kJump) * kJump - (k - 1) * kJump;  // depth of the k-th checkpoint
          dend[u] = ((d[u] - 1) / kJump) * kJump;
          nid[u] = s_cp[(size_t)q * R + k];
          row[u] = ((size_t)b * K + q) * (size_t)p.out_T;
        }
        for (int h = 0; h < kJump; ++h) {
#pragma unroll
          for (int u = 0; u < U; ++u) {
            if (d[u] <= dend[u]) continue;
            const Node nd = load_node(&nodes[nid[u]]);
            if (d[u] - 1 < p.out_T) {
              p.out_tokens[row[u] + d[u] - 1] = nd.chr;
              p.out_timesteps[row[u] + d[u] - 1] = nd.ts;
            }
            nid[u] = nd.parent;
            --d[u];
          }
        }
      }
    }
    CTC_BARRIER();
    CTC_PAR {
      for (int q = tid; q < M; q += NT) {
        int d = s_dep[q];
        for (int k = 0; k < s_ncp[q]; ++k) d = ((d - 1) / kJump) * kJump;
        s_dep[q] = d;
      }
    }
    CTC_BARRIER();
  }
}

// ======================================================================================================
//  committed_cta_run: the committed prefix of one stream -- the path from the root to the lowest common ancestor
//  (LCA) of the current beam members.  A node's (char, timestep) changes only while its parent is a beam member
//  (reference path_trie.cpp:38-46) and every future member descends from a current one, so no node on that path
//  changes, dies or is revived again: its tokens and timesteps start every row any later read-out of the stream
//  returns.  Trie paths are unique, so the LCA's depth is the longest common prefix of the rows a finalize of the same
//  state writes.  Reads the state block and the arena only.
//
//  The search runs top-down over the jump pointers (Node::jump): every member descends to its ancestor at the
//  deepest multiple of kJump not below the shallowest member, then all step one jump at a time until their ancestors
//  agree (at depth 0 all are the root); the last 15 levels above that are resolved by stepping parents in lockstep.
//  About (depth - LCA depth) / kJump + 2 * kJump dependent hops per member, all members in parallel.  The path
//  [since, LCA depth) is then written like finalize writes a row: jump checkpoints, stretches in parallel.
// ======================================================================================================
constexpr int kCommitCp = 256;  // checkpoints of the write-out per round
CTC_HD size_t committed_smem_bytes(int K) { return (size_t)K * 3 * 4 + (size_t)kCommitCp * 4 + 64; }
// Steps (a) and (b): returns the LCA depth D; with M > 0 the LCA's node id is left in ((int *)smem)[K] (s_hi[0]).
template <int NT>
CTC_FN int members_lca(const Node *nodes, const int *st, int K, unsigned char *smem) {
  const int M = st[0];
  const int *s = st + kStateHeader;
  int *s_cur = (int *)smem;       // [K] each member's ancestor at the current aligned depth
  int *s_hi = s_cur + K;          // [K] its ancestor one step above that (a checkpoint, or the member's own node)
  int *s_hd = s_hi + K;           // [K] depth of s_hi
  int *s_cp = s_hd + K;           // [kCommitCp] write-out checkpoints
  int *s_ctl = s_cp + kCommitCp;  // [0] -(shallowest member depth), [1] disagreement, [2..4] write-out cursor
  CTC_PAR {
    if (tid == 0) { s_ctl[0] = -0x7fffffff; s_ctl[1] = 0; }
  }
  CTC_BARRIER();
  CTC_PAR {
    for (int j = tid; j < M; j += NT) atom_max_i(&s_ctl[0], -s[2 * K + j]);
  }
  CTC_BARRIER();
  const int dmin = M > 0 ? -s_ctl[0] : 0;
  int A = dmin / kJump * kJump;
  CTC_PAR {
    for (int j = tid; j < M; j += NT) {
      int nid = s[j], d = s[2 * K + j], hi = nid, hd = d;
      while (d > A) {
        hi = nid; hd = d;
        nid = ld_cg(&nodes[nid].jump);
        d = (d - 1) / kJump * kJump;
      }
      s_cur[j] = nid; s_hi[j] = hi; s_hd[j] = hd;
    }
  }
  CTC_BARRIER();
  // (a) the deepest aligned depth A at which every member has the same ancestor
  for (;;) {
    CTC_PAR {
      for (int j = tid; j < M; j += NT)
        if (s_cur[j] != s_cur[0]) s_ctl[1] = 1;  // benign race: all writers store 1
    }
    CTC_BARRIER();
    const int split = s_ctl[1];
    CTC_BARRIER();  // (everyone has read the flag before it is cleared)
    if (!split || A == 0) break;
    CTC_PAR {
      for (int j = tid; j < M; j += NT) {
        s_hi[j] = s_cur[j]; s_hd[j] = A;
        s_cur[j] = ld_cg(&nodes[s_cur[j]].jump);
      }
      if (tid == 0) s_ctl[1] = 0;
    }
    A -= kJump;
    CTC_BARRIER();
  }
  // (b) the LCA lies in [A, U]: every member's ancestor at depth U, then parents in lockstep until they agree
  const int U = dmin < A + kJump - 1 ? dmin : A + kJump - 1;
  CTC_PAR {
    for (int j = tid; j < M; j += NT) {
      int nid = s_hi[j];
      for (int d = s_hd[j]; d > U; --d) nid = ld_cg(&nodes[nid].parent);
      s_hi[j] = nid;
    }
    if (tid == 0) s_ctl[1] = 0;
  }
  CTC_BARRIER();
  int D = U;
  while (D > A) {
    CTC_PAR {
      for (int j = tid; j < M; j += NT)
        if (s_hi[j] != s_hi[0]) s_ctl[1] = 1;
    }
    CTC_BARRIER();
    const int split = s_ctl[1];
    CTC_BARRIER();
    if (!split) break;
    CTC_PAR {
      for (int j = tid; j < M; j += NT) s_hi[j] = ld_cg(&nodes[s_hi[j]].parent);
      if (tid == 0) s_ctl[1] = 0;
    }
    --D;
    CTC_BARRIER();
  }
  return D;
}

// since: positions already read out (the previous call's result); outside [0, LCA depth] it is taken as 0.
// Writes *committed = LCA depth and columns [0, min(depth - since, cap)) of out_tok / out_ts (positions since..).
template <int NT>
CTC_FN void committed_cta_run(const Node *nodes, const int *st, int K, int since, int *committed, int *out_tok,
                              int *out_ts, int cap, unsigned char *smem) {
  const int M = st[0];
  const int D = members_lca<NT>(nodes, st, K, smem);
  int *s_hi = (int *)smem + K;
  int *s_cp = s_hi + 2 * K;
  int *s_ctl = s_cp + kCommitCp;
  // (c) write positions [s0, min(D, s0 + cap)) of the path root -> LCA; node of depth d holds position d - 1
  const int s0 = (since >= 0 && since <= D) ? since : 0;
  CTC_PAR {
    if (tid == 0) { *committed = D; s_ctl[2] = M > 0 ? s_hi[0] : 0; s_ctl[3] = D; }
  }
  CTC_BARRIER();
  int dcur = D;
  while (dcur > s0) {
    CTC_PAR {
      if (tid == 0) {
        int nid = s_ctl[2], d = s_ctl[3], n = 0;
        while (n < kCommitCp && d > s0) {
          s_cp[n++] = nid;
          nid = ld_cg(&nodes[nid].jump);
          d = (d - 1) / kJump * kJump;
        }
        s_ctl[2] = nid; s_ctl[3] = d; s_ctl[4] = n;
      }
    }
    CTC_BARRIER();
    const int dnext = s_ctl[3], n = s_ctl[4];
    CTC_PAR {
      for (int k = tid; k < n; k += NT) {
        int d = k == 0 ? dcur : (dcur - 1) / kJump * kJump - (k - 1) * kJump;  // depth of the k-th checkpoint
        int dend = (d - 1) / kJump * kJump;
        dend = dend > s0 ? dend : s0;
        int nid = s_cp[k];
        for (; d > dend; --d) {
          const Node nd = load_node(&nodes[nid]);
          const int col = d - 1 - s0;
          if (col < cap) { out_tok[col] = nd.chr; out_ts[col] = nd.ts; }
          nid = nd.parent;
        }
      }
    }
    CTC_BARRIER();
    dcur = dnext;
  }
}

}  // namespace ctc

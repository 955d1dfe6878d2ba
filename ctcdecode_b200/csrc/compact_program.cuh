// Compaction of a streaming state's node arena: one CTA per stream, run between chunks (ctcdec_stream_compact).
//
// The beam kernel appends every node it creates and frees none, so a stream's arena grows with its length.  What any
// later launch, finalize or committed-prefix call reads is a subset of R = the ancestors-or-self of the current beam
// members (state block slots 0 .. M-1): the beam kernel reads the members' nodes and walks parents only from a member
// up to one of its dead anchors (the revive slow path), and every occupied dead anchor is an ancestor of a member;
// finalize and committed_cta_run walk from the members to the root.  Everything outside R is unobservable.
//
// Two programs, with the host in between to size the new arrays:
//   compact_mark_cta_run    map[n] = the node's new id, or -1 if n is not in R; returns |R| in *kept.  The new ids
//                           are the ranks of the old ids in R: the root stays 0 and a parent stays below its children.
//   compact_gather_cta_run  copies the nodes of R into the new arena (parent and jump renumbered; chr, lpc, ts as they
//                           are), with their LM terms, histories, dictionary states and rows of a character-based
//                           model, and rewrites the words of the state block that hold node ids: the members' node and
//                           jump slots, the occupied dead anchors' node, and the node count.
//
// Both are written as barrier-separated regions (beam_core.cuh), so the same text runs in the CPU emulation.
#pragma once
#include "beam_program.cuh"

namespace ctc {

// shared memory of compact_mark_cta_run: members_lca's, then a count per thread
CTC_HD size_t compact_smem_bytes(int K, int NT) { return committed_smem_bytes(K) + (size_t)NT * 4; }

// map: [cap] ints of scratch, cap = the arena's capacity.  Marking: the root -> LCA path in parallel stretches of at
// most kJump nodes below the jump checkpoints (as committed_cta_run writes it out), then every member's tail walks
// parents until it meets a marked node.  Nothing walks above the LCA twice, so the dependent hops are about (depth - LCA depth) per member plus
// LCA depth / kJump on one thread.
template <int NT>
CTC_FN void compact_mark_cta_run(const Node *nodes, const int *st, int K, int cap, int *map, int *kept,
                                 unsigned char *smem) {
  const int M = st[0], n = st[1] < cap ? st[1] : cap;  // (st[1] <= cap: the beam kernel never passes the capacity)
  const int *s = st + kStateHeader;
  const int KP2 = 2 * kp_of(K);
  const int *const dnode = s + kSlotArrays * K, *const dpslot = dnode + 2 * KP2;
  CTC_PAR {
    for (int i = tid; i < n; i += NT) map[i] = 0;
  }
  // (members_lca starts with a barrier: the cleared map is visible before anything is marked)
  const int D = members_lca<NT>(nodes, st, K, smem);
  const int *const s_hi = (const int *)smem + K;
  int *const s_cp = (int *)smem + 3 * K;
  int *const s_ctl = s_cp + kCommitCp;
  int *const s_cnt = (int *)(smem + committed_smem_bytes(K));
  CTC_PAR {
    if (tid == 0) { map[0] = 1; s_ctl[2] = M > 0 ? s_hi[0] : 0; s_ctl[3] = D; }
  }
  CTC_BARRIER();
  for (int dcur = D; dcur > 0;) {
    CTC_PAR {
      if (tid == 0) {
        int nid = s_ctl[2], d = s_ctl[3], c = 0;
        while (c < kCommitCp && d > 0) {
          s_cp[c++] = nid;
          nid = ld_cg(&nodes[nid].jump);
          d = (d - 1) / kJump * kJump;
        }
        s_ctl[2] = nid; s_ctl[3] = d; s_ctl[4] = c;
      }
    }
    CTC_BARRIER();
    const int dnext = s_ctl[3], c = s_ctl[4];
    CTC_PAR {
      for (int k = tid; k < c; k += NT) {
        int d = k == 0 ? dcur : (dcur - 1) / kJump * kJump - (k - 1) * kJump;  // depth of the k-th checkpoint
        const int dend = (d - 1) / kJump * kJump;
        for (int nid = s_cp[k]; d > dend; --d) {
          map[nid] = 1;
          nid = ld_cg(&nodes[nid].parent);
        }
      }
    }
    CTC_BARRIER();
    dcur = dnext;
  }
  // the members' tails; the root -> LCA path is marked, so every walk ends there at the latest
  CTC_PAR {
    for (int j = tid; j < M; j += NT)
      for (int nid = s[j]; !map[nid]; nid = ld_cg(&nodes[nid].parent)) map[nid] = 1;
  }
  CTC_BARRIER();
  // the occupied dead anchors: ancestors of members, so already marked (the emulation checks it); seeds all the same
  CTC_PAR {
    for (int a = tid; a < KP2; a += NT) {
      if (dpslot[a] < 0) continue;
#if defined(CTC_EMULATE)
      if (!map[dnode[a]]) {
        fprintf(stderr, "compact: dead anchor %d (node %d) is not an ancestor of a member\n", a, dnode[a]);
        abort();
      }
#endif
      for (int nid = dnode[a]; !map[nid]; nid = ld_cg(&nodes[nid].parent)) map[nid] = 1;
    }
  }
  CTC_BARRIER();
  // new ids: an exclusive prefix sum of the marks, each thread over a contiguous range of ids
  const int per = (n + NT - 1) / NT;
  CTC_PAR {
    const int i1 = (tid + 1) * per < n ? (tid + 1) * per : n;
    int c = 0;
    for (int i = tid * per; i < i1; ++i) c += map[i];
    s_cnt[tid] = c;
  }
  CTC_BARRIER();
  CTC_PAR {
    if (tid == 0) {
      int o = 0;
      for (int t = 0; t < NT; ++t) { const int c = s_cnt[t]; s_cnt[t] = o; o += c; }
      *kept = o;
    }
  }
  CTC_BARRIER();
  CTC_PAR {
    const int i1 = (tid + 1) * per < n ? (tid + 1) * per : n;
    int o = s_cnt[tid];
    for (int i = tid * per; i < i1; ++i) map[i] = map[i] ? o++ : -1;
  }
}

// One stream's old and new arrays.  The LM arrays follow the streaming layout (ctc_api.cu StreamState): lm holds cap
// terms, then cap x H history ids; row (character-based model) cap x V terms.  lm / dst / row are NULL without a
// scorer, row also for a word-based model.
struct CompactJob {
  const Node *arena;
  Node *arena_new;
  int *state;
  const int *map;
  const float *lm;
  float *lm_new;
  const int *dst;
  int *dst_new;
  const float *row;
  float *row_new;
  int K, cap, cap_new, H, V, kept;
};

template <int NT>
CTC_FN void compact_gather_cta_run(const CompactJob &j) {
  const int K = j.K, H = j.H, V = j.V;
  int *const st = j.state;
  const int n = st[1] < j.cap ? st[1] : j.cap, M = st[0];
  const int *const hist = j.lm ? reinterpret_cast<const int *>(j.lm + j.cap) : nullptr;
  int *const hist_new = j.lm ? reinterpret_cast<int *>(j.lm_new + j.cap_new) : nullptr;
  CTC_PAR {
    for (int i = tid; i < n; i += NT) {
      const int m = j.map[i];
      if (m < 0) continue;
      Node nd = load_node(&j.arena[i]);
      nd.parent = nd.parent >= 0 ? j.map[nd.parent] : -1;
      nd.jump = nd.jump >= 0 ? j.map[nd.jump] : -1;
      store_node(&j.arena_new[m], nd);
      if (j.lm) {
        j.lm_new[m] = j.lm[i];
        j.dst_new[m] = j.dst[i];
        for (int k = 0; k < H; ++k) hist_new[(size_t)m * H + k] = hist[(size_t)i * H + k];
      }
      if (j.row)
        for (int c = 0; c < V; ++c) j.row_new[(size_t)m * V + c] = j.row[(size_t)i * V + c];
    }
  }
  CTC_BARRIER();  // (everyone has read st[1])
  int *const s = st + kStateHeader;
  const int KP2 = 2 * kp_of(K);
  int *const dnode = s + kSlotArrays * K;
  const int *const dpslot = dnode + 2 * KP2;
  CTC_PAR {
    for (int q = tid; q < M; q += NT) {
      s[q] = j.map[s[q]];
      const int jp = s[11 * K + q];
      s[11 * K + q] = jp >= 0 ? j.map[jp] : -1;
    }
    for (int a = tid; a < KP2; a += NT)
      if (dpslot[a] >= 0) dnode[a] = j.map[dnode[a]];
    if (tid == 0) st[1] = j.kept;
  }
}

}  // namespace ctc

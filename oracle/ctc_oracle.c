/*
 * TEST INFRASTRUCTURE ONLY -- CPU oracle for the CTC prefix beam-search hot path.
 *
 * This file is the checker, never the product: only tests/, __graft_entry__.smoke() and
 * bench.py's cpu_baseline / --impl reference legs may load it.  Nothing under ctcdecode_b200/
 * may import, link or execute it; the product path fails loudly without its CUDA library.
 *
 * It is a plain-C restatement of the reference algorithm (parlance/ctcdecode @ c90ad94), one
 * function per reference function, citing the file:line it follows.  Arithmetic goes through
 * the host libm (expf/logf/log/exp) exactly as the reference's `std::log/std::exp` calls do, and
 * the file is compiled with -ffp-contract=off like the reference's plain -O3 x86-64 build
 * (setup.py:57), so float32 scores are bit-identical to the reference on the same machine.
 *
 * Parity pinning: tests/test_oracle.py compares this file against oracle/_ref
 * (the unmodified reference sources compiled by oracle/Makefile) bit-for-bit, and
 * tests/golden/ holds outputs of that reference build for the reference's own fixtures
 * (tests/test_decode.py:13-32) and for seeded synthetic inputs.
 *
 * Only the no-LM path (ext_scorer == nullptr) is restated; the Scorer/KenLM hook is exercised
 * through oracle/_ref.
 *
 * The one place the reference is unspecified -- comparator-equivalent prefixes (equal float
 * score AND equal last character) straddling the beam cut or adjacent in the final order, and
 * equal probabilities straddling the cutoff_top_n cut, which the reference resolves through
 * libstdc++ introsort/introselect internals -- is resolved here deterministically (first in
 * trie DFS order wins) and reported through tie_flags.
 *
 * At a beam-cut tie the reference keeps SOME r of the m comparator-equal prefixes that straddle
 * the cut; which r is all its choice decides (the order of the kept prefixes changes no
 * arithmetic: a node's per-frame sums have at most two terms and log_sum_exp is symmetric).
 * ctc_oracle_decode_choices() takes one choice per such tie event -- an index into the r-subsets
 * of the m members, 0 = the first r in DFS order, the default -- and reports every event, so a
 * caller can enumerate every output the reference may produce.  Equal probabilities at the
 * vocabulary cut keep the lowest indices (as the CUDA program does); they take no choice.
 */
#include <float.h>
#include <limits.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NUM_FLT_INF FLT_MAX /* decoder_utils.h:12 */
#define NUM_FLT_MIN FLT_MIN /* decoder_utils.h:13 */

#define TIE_PRUNE 1 /* equivalent prefixes straddled the top-beam_size cut at some frame */
#define TIE_FINAL 2 /* equivalent prefixes adjacent in the final ordering               */
#define TIE_VOCAB 4 /* equal probabilities straddled the cutoff_top_n / cutoff_prob cut  */

/* ---- log_sum_exp<T>  (decoder_utils.h:47-54) ------------------------------------------- */
static float lse_f(float x, float y) {
  if (x <= -FLT_MAX) return y;
  if (y <= -FLT_MAX) return x;
  float xmax = x > y ? x : y; /* std::max(x, y) */
  return logf(expf(x - xmax) + expf(y - xmax)) + xmax;
}
static double lse_d(double x, double y) {
  if (x <= -DBL_MAX) return y;
  if (y <= -DBL_MAX) return x;
  double xmax = x > y ? x : y;
  return log(exp(x - xmax) + exp(y - xmax)) + xmax;
}

/* ---- PathTrie  (path_trie.h:45-67, path_trie.cpp:11-30) --------------------------------- */
typedef struct Node {
  float log_prob_b_prev, log_prob_nb_prev, log_prob_b_cur, log_prob_nb_cur;
  float log_prob_c, score, approx_ctc;
  int character, timestep;
  struct Node *parent;
  int exists;
  int n_children, cap_children;
  struct Node **children; /* insertion order, like vector<pair<int,PathTrie*>> children_ */
} Node;

static void node_init(Node *n) {
  n->log_prob_b_prev = n->log_prob_nb_prev = -NUM_FLT_INF;
  n->log_prob_b_cur = n->log_prob_nb_cur = -NUM_FLT_INF;
  n->log_prob_c = -NUM_FLT_INF;
  n->score = -NUM_FLT_INF;
  n->approx_ctc = 0.0f;
  n->character = -1; /* ROOT_ */
  n->timestep = 0;
  n->parent = NULL;
  n->exists = 1;
  n->n_children = n->cap_children = 0;
  n->children = NULL;
}

static void node_free_subtree(Node *n) { /* ~PathTrie, path_trie.cpp:32-36 */
  for (int i = 0; i < n->n_children; ++i) {
    node_free_subtree(n->children[i]);
    free(n->children[i]);
  }
  free(n->children);
}

/* PathTrie::get_path_trie without dictionary  (path_trie.cpp:38-57, 97-106) */
static Node *node_get_child(Node *self, int new_char, int new_timestep, float cur_log_prob_c) {
  for (int i = 0; i < self->n_children; ++i) {
    Node *c = self->children[i];
    if (c->character == new_char) {
      if (c->log_prob_c < cur_log_prob_c) {
        c->log_prob_c = cur_log_prob_c;
        c->timestep = new_timestep;
      }
      if (!c->exists) {
        c->exists = 1;
        c->log_prob_b_prev = c->log_prob_nb_prev = -NUM_FLT_INF;
        c->log_prob_b_cur = c->log_prob_nb_cur = -NUM_FLT_INF;
      }
      return c;
    }
  }
  Node *n = (Node *)malloc(sizeof(Node));
  node_init(n);
  n->character = new_char;
  n->timestep = new_timestep;
  n->parent = self;
  n->log_prob_c = cur_log_prob_c;
  if (self->n_children == self->cap_children) {
    self->cap_children = self->cap_children ? 2 * self->cap_children : 4;
    self->children = (Node **)realloc(self->children, sizeof(Node *) * self->cap_children);
  }
  self->children[self->n_children++] = n;
  return n;
}

/* PathTrie::remove  (path_trie.cpp:144-163) */
static void node_remove(Node *self) {
  self->exists = 0;
  if (self->n_children == 0) {
    Node *p = self->parent;
    for (int i = 0; i < p->n_children; ++i) {
      if (p->children[i]->character == self->character) {
        memmove(&p->children[i], &p->children[i + 1], sizeof(Node *) * (p->n_children - i - 1));
        p->n_children--;
        break;
      }
    }
    if (p->n_children == 0 && !p->exists) node_remove(p);
    free(self->children);
    free(self);
  }
}

typedef struct {
  Node **v;
  int n, cap;
} NodeVec;
static void vec_push(NodeVec *v, Node *n) {
  if (v->n == v->cap) {
    v->cap = v->cap ? 2 * v->cap : 256;
    v->v = (Node **)realloc(v->v, sizeof(Node *) * v->cap);
  }
  v->v[v->n++] = n;
}

/* PathTrie::iterate_to_vec  (path_trie.cpp:128-142); recursion depth <= prefix length */
static void node_iterate_to_vec(Node *self, NodeVec *out) {
  if (self->exists) {
    self->log_prob_b_prev = self->log_prob_b_cur;
    self->log_prob_nb_prev = self->log_prob_nb_cur;
    self->log_prob_b_cur = -NUM_FLT_INF;
    self->log_prob_nb_cur = -NUM_FLT_INF;
    self->score = lse_f(self->log_prob_b_prev, self->log_prob_nb_prev);
    vec_push(out, self);
  }
  for (int i = 0; i < self->n_children; ++i) node_iterate_to_vec(self->children[i], out);
}

/* prefix_compare  (decoder_utils.cpp:122-132): returns 1 if x orders strictly before y */
static int prefix_compare(const Node *x, const Node *y) {
  if (x->score == y->score) {
    if (x->character == y->character) return 0;
    return x->character < y->character;
  }
  return x->score > y->score;
}

/* stable merge sort under prefix_compare (ties keep input = DFS order) */
static void merge_sort_nodes(Node **a, Node **tmp, int n) {
  if (n < 2) return;
  int h = n / 2;
  merge_sort_nodes(a, tmp, h);
  merge_sort_nodes(a + h, tmp, n - h);
  int i = 0, j = h, k = 0;
  while (i < h && j < n) tmp[k++] = prefix_compare(a[j], a[i]) ? a[j++] : a[i++];
  while (i < h) tmp[k++] = a[i++];
  while (j < n) tmp[k++] = a[j++];
  memcpy(a, tmp, sizeof(Node *) * n);
}

static int prefix_equiv(const Node *x, const Node *y) { return !prefix_compare(x, y) && !prefix_compare(y, x); }

/* C(n, k), saturating at ULLONG_MAX */
static unsigned long long binom(int n, int k) {
  if (k < 0 || k > n) return 0;
  if (k > n - k) k = n - k;
  unsigned long long r = 1;
  for (int i = 1; i <= k; ++i) { /* r = C(n-k+i-1, i-1) -> C(n-k+i, i), exact at every step */
    unsigned __int128 t = (unsigned __int128)r * (unsigned)(n - k + i) / (unsigned)i;
    if (t > ULLONG_MAX) return ULLONG_MAX;
    r = (unsigned long long)t;
  }
  return r;
}

/* Reorder a[0..m) so that the r-subset of rank `choice` (lexicographic order of index sets: rank 0 = {0..r-1}) comes
 * first, each part keeping its relative order.  Uses tmp[0..m) only: the kept part goes there, the dropped part is
 * compacted in place (its write index never passes the read index). */
static void keep_subset(Node **a, Node **tmp, int m, int r, unsigned long long choice) {
  int k = r, nk = 0, nd = 0;
  for (int i = 0; i < m; ++i) {
    unsigned long long with_i = k > 0 ? binom(m - i - 1, k - 1) : 0;
    if (k > 0 && choice < with_i) {
      tmp[nk++] = a[i];
      --k;
    } else {
      choice -= with_i;
      a[nd++] = a[i];
    }
  }
  memmove(a + nk, a, sizeof(Node *) * nd);
  memcpy(a, tmp, sizeof(Node *) * nk);
}

/* ---- get_pruned_log_probs  (decoder_utils.cpp:10-45) ------------------------------------ */
typedef struct {
  int idx;
  double p;
} ProbIdx;
static int prob_desc(const void *a, const void *b) { /* pair_comp_second_rev + index tie-break */
  const ProbIdx *x = (const ProbIdx *)a, *y = (const ProbIdx *)b;
  if (x->p > y->p) return -1;
  if (x->p < y->p) return 1;
  return x->idx - y->idx;
}
static int get_pruned_log_probs(const double *prob_step, int V, double cutoff_prob, size_t cutoff_top_n,
                                int log_input, ProbIdx *work, int *out_idx, float *out_lp, int *tie) {
  double log_cutoff_prob = log(cutoff_prob);
  for (int i = 0; i < V; ++i) {
    work[i].idx = i;
    work[i].p = prob_step[i];
  }
  size_t cutoff_len = (size_t)V;
  if (log_cutoff_prob < 0.0 || cutoff_top_n < cutoff_len) {
    qsort(work, V, sizeof(ProbIdx), prob_desc);
    if (log_cutoff_prob < 0.0) {
      double cum_prob = 0.0;
      cutoff_len = 0;
      for (int i = 0; i < V; ++i) {
        cum_prob = lse_d(cum_prob, log_input ? work[i].p : log(work[i].p));
        cutoff_len += 1;
        if (cum_prob >= cutoff_prob || cutoff_len >= cutoff_top_n) break;
      }
    } else {
      cutoff_len = cutoff_top_n;
    }
    if (cutoff_len < (size_t)V && cutoff_len > 0 && work[cutoff_len - 1].p == work[cutoff_len].p)
      *tie |= TIE_VOCAB;
  }
  for (size_t i = 0; i < cutoff_len; ++i) {
    out_idx[i] = work[i].idx;
    out_lp[i] = (float)(log_input ? work[i].p : log(work[i].p + NUM_FLT_MIN));
  }
  return (int)cutoff_len;
}

/* ---- DecoderState  (ctc_beam_search_decoder.h:73-124, .cpp:17-53) ------------------------- */
typedef struct {
  int abs_time_step;
  int beam_size, V, blank_id, log_input;
  size_t cutoff_top_n;
  double cutoff_prob;
  Node root;
  NodeVec prefixes;
  int tie_flags;
  /* what kind of ties straddled the beam cut (tools/tie_report.py): frames where the tied prefixes are -FLT_MAX
   * "junk" (SURVEY.md quirk Q6) / carry a finite score, and the first such frame */
  int tie_junk_frames, tie_finite_frames, tie_first_frame;
  /* beam-cut tie control (ctc_oracle_decode_choices): the kept subset at the i-th tie event is tie_choice[i] (0 when
   * i >= n_tie_choice); each event is logged as (frame, m, r, junk) into tie_events[4 * i] while i < max_tie_events */
  const long long *tie_choice;
  int n_tie_choice;
  int *tie_events;
  int max_tie_events, n_tie_events;
  /* scratch */
  ProbIdx *work;
  int *pr_idx;
  float *pr_lp;
  double *row;
  Node **tmp;
  int tmp_cap;
} OracleState;

void *ctc_oracle_state_new(int V, int beam_size, double cutoff_prob, int cutoff_top_n, int blank_id,
                           int log_input) {
  OracleState *s = (OracleState *)calloc(1, sizeof(OracleState));
  s->V = V;
  s->beam_size = beam_size;
  s->cutoff_prob = cutoff_prob;
  s->cutoff_top_n = (size_t)cutoff_top_n;
  s->blank_id = blank_id;
  s->log_input = log_input;
  node_init(&s->root);
  s->root.score = s->root.log_prob_b_prev = 0.0f; /* ctc_beam_search_decoder.cpp:43 */
  vec_push(&s->prefixes, &s->root);
  s->work = (ProbIdx *)malloc(sizeof(ProbIdx) * V);
  s->pr_idx = (int *)malloc(sizeof(int) * V);
  s->pr_lp = (float *)malloc(sizeof(float) * V);
  s->row = (double *)malloc(sizeof(double) * V);
  return s;
}

void ctc_oracle_state_free(void *h) {
  OracleState *s = (OracleState *)h;
  node_free_subtree(&s->root);
  free(s->prefixes.v);
  free(s->work);
  free(s->pr_idx);
  free(s->pr_lp);
  free(s->row);
  free(s->tmp);
  free(s);
}

/* DecoderState::next, ext_scorer == nullptr  (ctc_beam_search_decoder.cpp:56-162).
 * probs: [num_time_steps, V] float32, widened to double like binding.cpp:69-70. */
void ctc_oracle_state_next(void *h, const float *probs, int num_time_steps) {
  OracleState *s = (OracleState *)h;
  const int V = s->V;
  for (int time_step = 0; time_step < num_time_steps; ++time_step, ++s->abs_time_step) {
    for (int i = 0; i < V; ++i) s->row[i] = (double)probs[(size_t)time_step * V + i];
    int n_pruned = get_pruned_log_probs(s->row, V, s->cutoff_prob, s->cutoff_top_n, s->log_input, s->work,
                                        s->pr_idx, s->pr_lp, &s->tie_flags);
    for (int index = 0; index < n_pruned; ++index) { /* loop over chars, :87 */
      int c = s->pr_idx[index];
      float log_prob_c = s->pr_lp[index];
      for (int i = 0; i < s->prefixes.n && i < s->beam_size; ++i) { /* :91 */
        Node *prefix = s->prefixes.v[i];
        if (c == s->blank_id) { /* :97-101 */
          prefix->log_prob_b_cur = lse_f(prefix->log_prob_b_cur, log_prob_c + prefix->score);
          continue;
        }
        if (c == prefix->character) { /* :103-106 */
          prefix->log_prob_nb_cur = lse_f(prefix->log_prob_nb_cur, log_prob_c + prefix->log_prob_nb_prev);
        }
        Node *prefix_new = node_get_child(prefix, c, s->abs_time_step, log_prob_c); /* :108 */
        float log_p = -NUM_FLT_INF;
        if (c == prefix->character && prefix->log_prob_b_prev > -NUM_FLT_INF) { /* :112-117 */
          log_p = log_prob_c + prefix->log_prob_b_prev;
        } else if (c != prefix->character) {
          log_p = log_prob_c + prefix->score;
        }
        prefix_new->log_prob_nb_cur = lse_f(prefix_new->log_prob_nb_cur, log_p); /* :138-139 */
      }
    }
    s->prefixes.n = 0;
    node_iterate_to_vec(&s->root, &s->prefixes); /* :145-147 */
    if (s->prefixes.n >= s->beam_size) {          /* :149-160 (nth_element + remove) */
      if (s->tmp_cap < s->prefixes.n) {
        s->tmp_cap = 2 * s->prefixes.n;
        s->tmp = (Node **)realloc(s->tmp, sizeof(Node *) * s->tmp_cap);
      }
      merge_sort_nodes(s->prefixes.v, s->tmp, s->prefixes.n);
      if (s->prefixes.n > s->beam_size) {
        Node **v = s->prefixes.v;
        const int K = s->beam_size;
        if (prefix_equiv(v[K - 1], v[K])) {
          if (!(s->tie_flags & TIE_PRUNE)) s->tie_first_frame = s->abs_time_step;
          s->tie_flags |= TIE_PRUNE;
          int junk = v[K]->score <= -NUM_FLT_INF;
          if (junk) s->tie_junk_frames++;
          else s->tie_finite_frames++;
          /* the tie event: the maximal run [lo, hi) of prefixes equivalent to v[K], in DFS order (stable sort) */
          int lo = K - 1, hi = K + 1;
          while (lo > 0 && prefix_equiv(v[lo - 1], v[K])) --lo;
          while (hi < s->prefixes.n && prefix_equiv(v[hi], v[K])) ++hi;
          int e = s->n_tie_events++;
          if (e < s->max_tie_events) {
            int *ev = s->tie_events + 4 * (size_t)e;
            ev[0] = s->abs_time_step;
            ev[1] = hi - lo;
            ev[2] = K - lo;
            ev[3] = junk;
          }
          long long choice = e < s->n_tie_choice ? s->tie_choice[e] : 0;
          if (choice > 0) keep_subset(v + lo, s->tmp, hi - lo, K - lo, (unsigned long long)choice);
        }
      }
      for (int i = s->beam_size; i < s->prefixes.n; ++i) node_remove(s->prefixes.v[i]);
      s->prefixes.n = s->beam_size;
    }
  }
}

/* DecoderState::decode + get_beam_search_result + get_path_vec, no scorer
 * (ctc_beam_search_decoder.cpp:164-211, decoder_utils.cpp:48-73, path_trie.cpp:109-126) and the
 * write-back of binding.cpp:79-99: only [:len] of each row is written.  Returns n_results. */
int ctc_oracle_state_decode(void *h, int row_stride, int *out_tokens, int *out_timesteps, float *out_scores,
                            int *out_lens, int *tie_flags) {
  OracleState *s = (OracleState *)h;
  int n = s->prefixes.n < s->beam_size ? s->prefixes.n : s->beam_size;
  Node **copy = (Node **)malloc(sizeof(Node *) * (n + 1));
  Node **tmp = (Node **)malloc(sizeof(Node *) * (n + 1));
  memcpy(copy, s->prefixes.v, sizeof(Node *) * n);
  merge_sort_nodes(copy, tmp, n); /* :187-190 then decoder_utils.cpp:59: same comparator w/o scorer */
  for (int i = 0; i + 1 < n; ++i)
    if (!prefix_compare(copy[i], copy[i + 1]) && !prefix_compare(copy[i + 1], copy[i])) s->tie_flags |= TIE_FINAL;
  for (int p = 0; p < n; ++p) {
    copy[p]->approx_ctc = copy[p]->score; /* :194-208 */
    int len = 0;
    for (Node *q = copy[p]; q->character != -1; q = q->parent) ++len;
    int k = len;
    for (Node *q = copy[p]; q->character != -1; q = q->parent) {
      --k;
      out_tokens[(size_t)p * row_stride + k] = q->character;
      out_timesteps[(size_t)p * row_stride + k] = q->timestep;
    }
    out_scores[p] = (float)(-(double)copy[p]->approx_ctc); /* decoder_utils.cpp:68, binding.cpp:91 */
    out_lens[p] = len;
  }
  if (tie_flags) *tie_flags = s->tie_flags;
  free(copy);
  free(tmp);
  return n;
}

/* out[0..2] = frames with a -FLT_MAX tie at the beam cut, frames with a finite-score tie, first tie frame (or -1) */
void ctc_oracle_state_tie_stats(void *h, int *out) {
  OracleState *s = (OracleState *)h;
  out[0] = s->tie_junk_frames;
  out[1] = s->tie_finite_frames;
  out[2] = (s->tie_flags & TIE_PRUNE) ? s->tie_first_frame : -1;
}

/* ctc_beam_search_decoder_batch, serial  (ctc_beam_search_decoder.cpp:213-227, 245-285) with the
 * marshalling of binding.cpp:59-99.  Outputs: tokens/timesteps [B,beam,T], scores/lens [B,beam]. */
int ctc_oracle_decode_batch(const float *probs, const int *seq_lens, int B, int T, int V, int beam_size,
                            double cutoff_prob, int cutoff_top_n, int blank_id, int log_input, int *out_tokens,
                            int *out_timesteps, float *out_scores, int *out_lens, int *n_results,
                            int *tie_flags) {
  for (int b = 0; b < B; ++b) {
    int len = seq_lens ? seq_lens[b] : T;
    if (len > T) len = T; /* binding.cpp:64-65 */
    if (len < 0) len = 0;
    void *st = ctc_oracle_state_new(V, beam_size, cutoff_prob, cutoff_top_n, blank_id, log_input);
    ctc_oracle_state_next(st, probs + (size_t)b * T * V, len);
    int tf = 0;
    int n = ctc_oracle_state_decode(st, T, out_tokens + (size_t)b * beam_size * T,
                                    out_timesteps + (size_t)b * beam_size * T, out_scores + (size_t)b * beam_size,
                                    out_lens + (size_t)b * beam_size, &tf);
    if (n_results) n_results[b] = n;
    if (tie_flags) tie_flags[b] = tf;
    ctc_oracle_state_free(st);
  }
  return 1;
}

/* One utterance (len frames of a [T, V] row block) with the beam-cut tie choices `choice[0..n_choice)` (further events:
 * choice 0, i.e. exactly ctc_oracle_decode_batch's result).  Every tie event met is written as (frame, m, r, junk) to
 * events[4 * i] for i < max_events; *n_events = how many were met.  Outputs as one utterance of the batch entry. */
int ctc_oracle_decode_choices(const float *probs, int len, int T, int V, int beam_size, double cutoff_prob,
                              int cutoff_top_n, int blank_id, int log_input, const long long *choice, int n_choice,
                              int *events, int max_events, int *n_events, int *out_tokens, int *out_timesteps,
                              float *out_scores, int *out_lens, int *tie_flags) {
  if (len > T) len = T;
  if (len < 0) len = 0;
  OracleState *st = (OracleState *)ctc_oracle_state_new(V, beam_size, cutoff_prob, cutoff_top_n, blank_id, log_input);
  st->tie_choice = choice;
  st->n_tie_choice = n_choice;
  st->tie_events = events;
  st->max_tie_events = max_events;
  ctc_oracle_state_next(st, probs, len);
  int n = ctc_oracle_state_decode(st, T, out_tokens, out_timesteps, out_scores, out_lens, tie_flags);
  *n_events = st->n_tie_events;
  ctc_oracle_state_free(st);
  return n;
}

/* libm probes used by the exhaustive device-vs-host float checks in tests/ (Appendix B of SURVEY.md) */
void ctc_oracle_expf_array(const float *x, float *y, long n) {
  for (long i = 0; i < n; ++i) y[i] = expf(x[i]);
}
void ctc_oracle_logf_array(const float *x, float *y, long n) {
  for (long i = 0; i < n; ++i) y[i] = logf(x[i]);
}
void ctc_oracle_lse_array(const float *x, const float *y, float *z, long n) {
  for (long i = 0; i < n; ++i) z[i] = lse_f(x[i], y[i]);
}
/* double probes (the cum_prob chain of decoder_utils.cpp:26-31): which 0 exp(x), 1 log(x), 2 log_sum_exp<double>(x, x2) */
void ctc_oracle_f64_array(int which, const double *x, const double *x2, double *y, long n) {
  for (long i = 0; i < n; ++i) y[i] = which == 0 ? exp(x[i]) : which == 1 ? log(x[i]) : lse_d(x[i], x2[i]);
}
void ctc_oracle_logprob_array(const float *p, float *y, long n) { /* decoder_utils.cpp:40-43 */
  for (long i = 0; i < n; ++i) y[i] = (float)log((double)p[i] + NUM_FLT_MIN);
}

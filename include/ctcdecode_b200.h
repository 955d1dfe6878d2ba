/*
 * ctcdecode_b200 -- C ABI of the H100-native (sm_90a) CTC prefix beam-search decoder.
 *
 * This is the drop-in boundary for ONE path of parlance/ctcdecode: the batched beam search that the
 * reference reaches through its pybind module `ctcdecode._ext.ctc_decode` (reference
 * ctcdecode/src/binding.cpp:290-303).  Every entry point below names the reference interface it
 * replaces.  Plain pointers and sizes only -- no torch / pybind types -- so the same library binds
 * from the reference's own __init__.py (ctypes), from C++ (binding.cpp) or from anything with an FFI.
 * INTEGRATION.md shows the reference-side stubs.
 *
 * Conventions
 *   - every function returns CTCDEC_OK (0) or a negative CTCDEC_E_* code; ctcdec_last_error() gives
 *     the message for the calling thread.  Nothing aborts the process (the reference's
 *     VALID_CHECK -> LOG(FATAL) does, decoder_utils.h:17-23).
 *   - tensors are dense, row-major, caller-allocated, exactly shaped like the reference's:
 *       probs      float32 [B, T, V]          (probabilities, or log-probabilities if log_input)
 *       seq_lens   int32   [B] or NULL         (NULL = T for every utterance; values clamped to
 *                                               [0, T] like reference binding.cpp:64-65)
 *       tokens     int32   [B, beam, T]        (reference `output`;  only [b, p, :lens[b,p]] written)
 *       timesteps  int32   [B, beam, T]        (only [b, p, :lens[b,p]] written)
 *       scores     float32 [B, beam]           (rows p < n_results[b] written)
 *       lens       int32   [B, beam]           (reference `out_seq_len`; rows p < n_results[b] written)
 *     plus two outputs the reference does not have (both may be NULL):
 *       n_results  int32   [B]   how many beams utterance b produced (reference: results.size())
 *       flags      int32   [B]   CTCDEC_FLAG_* bits; the TIE bits mark utterances where the
 *                                reference's own result is unspecified (equal score AND equal last
 *                                character straddling a cut -- std::nth_element / std::sort internals)
 *   - "device" entry points take device pointers and a CUDA stream and never synchronise (except the scorer
 *     path's ctcdec_decode_batch_lm_device, whose language model is answered by the host during the call); "host"
 *     entry points take host pointers, stage through pinned memory and return when results are in
 *     the caller's buffers (what the reference's CPU-tensor API looks like to its caller).
 */
#ifndef CTCDECODE_B200_H_
#define CTCDECODE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTCDEC_OK 0
#define CTCDEC_E_INVALID (-1)   /* bad argument (shape, range, NULL)                                  */
#define CTCDEC_E_UNSUPPORTED (-2) /* configuration outside what the kernels implement (says which)    */
#define CTCDEC_E_CUDA (-3)      /* a CUDA runtime call failed                                         */
#define CTCDEC_E_WORKSPACE (-4) /* workspace too small                                                */
#define CTCDEC_E_NO_DEVICE (-5) /* no CUDA device / wrong architecture: there is NO CPU fallback      */
#define CTCDEC_E_INTERNAL (-6)  /* a kernel raised CTCDEC_FLAG_ERR_ARENA: results are not valid (host entry points) */

#define CTCDEC_FLAG_TIE_PRUNE 1
#define CTCDEC_FLAG_TIE_FINAL 2
#define CTCDEC_FLAG_TIE_VOCAB 4
#define CTCDEC_FLAG_ERR_ARENA 256

/* Decoder parameters: the arguments of the reference's ctc_beam_search_decoder_batch
 * (ctc_beam_search_decoder.h:63-72) / paddle_beam_decode (binding.cpp:103-120) that shape the search.
 * `num_processes` has no equivalent: the batch is a CUDA grid, one CTA per utterance.
 *
 * Accepted shapes: a beam CTA keeps the whole beam and its candidate lists in the 227 KB of shared memory an H100 CTA
 * can have, so the largest beam falls as the (pruned) vocabulary grows.  Largest beam without a scorer, batches of
 * up to 264 utterances (tests/test_plan_envelope.py has every vocabulary, mode and batch plan):
 *   nothing cut (cutoff_top_n >= V): 736 up to V = 29, 672 at V = 64, 544 at 256, 320 at 1024, 128 at 1500, 64 at
 *     4096; beams 1-32 take V <= 10845, beam 100 V <= 3389, beam 200 V <= 1469;
 *   top-40 cut (the default) or cutoff_prob < 1: 736 up to V = 29 (704 at V = 29 with cutoff_prob), 576 at 256, 352
 *     at 1024, 288 at 1500, 128 at 4096, 32 at 16384; beams 1-32 take V <= 16384 (the vocabulary-sort limit), beam
 *     100 V <= 4896, beam 200 V <= 2048.
 * With a scorer: nothing cut 704 at V = 29, 512 at 256, 256 at 1024 (V <= 9053 for beams 1-32); top-40 cut 704 at
 * V = 29, 608 at 256, 480 at 1024.  Every shape outside returns CTCDEC_E_UNSUPPORTED with the reason (the shared memory
 * the layout needs, or the sort limit), at plan time: nothing is launched.  The hard bounds beam_size <= 4096 and
 * vocab_size <= 65534 are never reached. */
typedef struct ctcdec_config {
  int vocab_size;      /* V = len(labels)                                   */
  int beam_size;       /* beam_width                                         */
  int blank_id;        /* index of the CTC blank                             */
  int log_input;       /* 0: probs are probabilities, 1: log-probabilities   */
  int cutoff_top_n;    /* reference default 40                               */
  double cutoff_prob;  /* reference default 1.0                              */
} ctcdec_config;

const char *ctcdec_version(void);
const char *ctcdec_last_error(void);

/* Number of CUDA devices usable by this library (compute capability 9.0); 0 if none. */
int ctcdec_device_count(void);

/* Bytes of device scratch ctcdec_decode_batch_device needs for a [B, T, V] batch. */
int ctcdec_workspace_bytes(const ctcdec_config *cfg, int B, int T, size_t *bytes);

/* Replaces: beam_decode / paddle_beam_decode -> ctc_beam_search_decoder_batch with ext_scorer == NULL
 * (reference binding.cpp:35-120, ctc_beam_search_decoder.cpp:245-285).  All pointers are DEVICE
 * pointers on the current device; work is enqueued on `stream` (a cudaStream_t) and not synchronised. */
int ctcdec_decode_batch_device(const ctcdec_config *cfg, const float *probs, const int32_t *seq_lens, int B, int T,
                               int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                               int32_t *n_results, int32_t *flags, void *workspace, size_t workspace_bytes,
                               void *stream);

/* The step BEFORE the path, fused (SURVEY.md section 8f row 3): the acoustic model's raw LOGITS [B, T, V] on the
 * device, in float32 / float16 / bfloat16.  The reference makes callers soft-max on their side and then re-takes the
 * logarithm per frame (README.md:54-57, decoder_utils.cpp:40-43); here the scan kernel computes the float32
 * log-softmax of each frame on the fly and decodes as with log_probs_input (cfg->log_input is ignored): one HBM
 * read of the logits, no probability tensor.  If log_probs_out is not NULL the [B, T, V] float32 log-softmax rows
 * the decode used are written there; the reference, fed those values with log_probs_input=True, gives bit-identical
 * results (that is how the parity test for this entry point works).  Everything else as above. */
#define CTCDEC_DTYPE_F32 0
#define CTCDEC_DTYPE_F16 1
#define CTCDEC_DTYPE_BF16 2
int ctcdec_decode_batch_device_logits(const ctcdec_config *cfg, const void *logits, int dtype, const int32_t *seq_lens,
                                      int B, int T, int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                      int32_t *n_results, int32_t *flags, float *log_probs_out, void *workspace,
                                      size_t workspace_bytes, void *stream);

/* The step AFTER the path (SURVEY.md section 8f row 4): compact the dense [B, beam, T] results of
 * ctcdec_decode_batch_device (of which only [b, p, :lens[b, p]] is meaningful, reference binding.cpp:79-99) into a
 * ragged layout on the device.  offsets [B * beam + 1] (int64): exclusive prefix sum of the row lengths, rows
 * p >= n_results[b] counting 0, offsets[B * beam] = total; packed_tokens / packed_timesteps [capacity]: rows whose
 * end exceeds `capacity` are not written (compare offsets[B * beam] with capacity).  All DEVICE pointers; enqueued
 * on `stream`. */
int ctcdec_pack_results_device(const int32_t *tokens, const int32_t *timesteps, const int32_t *lens,
                               const int32_t *n_results, int B, int K, int T, int64_t *offsets,
                               int32_t *packed_tokens, int32_t *packed_timesteps, size_t capacity, void *stream);

/* Same operation with HOST buffers shaped exactly like the reference's CPU tensors
 * (reference __init__.py:77-86).  The batch is cut into up to 8 groups of utterances, each on its own stream, so
 * that the upload, the kernels and the download of different groups overlap; small results are staged through
 * pinned memory.  Pinned caller buffers keep every copy asynchronous (pageable ones work, more slowly).
 * Environment (tuning / test knobs, all optional): CTCDEC_HOST_CHUNK=n utterances per group; CTCDEC_NT=128|160|192|256|
 * 512|1024 threads per utterance; CTCDEC_NO_FAST=1|2 the general back half of a frame everywhere / no head hand-over; CTCDEC_GENERIC_KP=1 the run-time-beam-size kernel; CTCDEC_FORCE_FALLBACK=1 the
 * grid-walking select on every frame; CTCDEC_SEG=n / CTCDEC_HEUR_BIAS=x small candidate lists / a failing heuristic
 * bound (tests/test_gpu_parity.py drives every select path with them). */
int ctcdec_decode_batch_host(const ctcdec_config *cfg, const float *probs, const int32_t *seq_lens, int B, int T,
                             int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens, int32_t *n_results,
                             int32_t *flags, int device);

/* The same call spread over several GPUs of the box from ONE host thread of the caller: the batch is cut into
 * contiguous shards, one per device in `devices` (NULL / n_devices <= 0: every usable device), each shard runs
 * ctcdec_decode_batch_host on its own device from its own worker thread (per-device streams and buffers; utterances are
 * independent, so nothing crosses between GPUs -- the reference's ThreadPool fan-out over utterances,
 * ctc_beam_search_decoder.cpp:245-285, at box scale).  This is what decoder.decode(cpu_probs) of a large batch uses. */
int ctcdec_decode_batch_host_multi(const ctcdec_config *cfg, const float *probs, const int32_t *seq_lens, int B, int T,
                                   int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                   int32_t *n_results, int32_t *flags, const int *devices, int n_devices);

/* ---- scorer path: language model (+ dictionary for word-based models) (reference Scorer, scorer.h:41-110) ---
 *
 * The language model itself stays on the HOST behind a hook the integrator supplies -- the reference side wraps its
 * own Scorer / KenLM (INTEGRATION.md); this library contains no KenLM.  Both hooks take a prefix as label ids:
 *   cond_log_prob(ctx, labels, n)  = Scorer::get_log_cond_prob(Scorer::make_ngram(prefix))   (scorer.cpp:74-93,163-194)
 *                                    i.e. the natural-log probability of the prefix's last word given the words
 *                                    before it (up to max_order, "<s>"-padded); OOV -> -1000
 *   sent_log_prob(ctx, labels, n)  = Scorer::get_sent_log_prob(Scorer::split_labels(prefix))  (scorer.cpp:95-146)
 * The hooks must be pure and thread-safe: the library calls them concurrently from a few worker threads of its own
 * (each utterance is served by one worker), like the reference calls its Scorer from the thread pool of
 * ctc_beam_search_decoder_batch (ctc_beam_search_decoder.cpp:228-247). */
typedef struct ctcdec_scorer_hooks {
  void *ctx;
  double (*cond_log_prob)(void *ctx, const int32_t *labels, int n);
  double (*sent_log_prob)(void *ctx, const int32_t *labels, int n);
} ctcdec_scorer_hooks;

/* Replaces: paddle_get_scorer (binding.cpp:143-150).  `labels` are the decoder's labels (UTF-8), `words` the
 * language model's vocabulary (what KenLM's EnumerateVocab reports, scorer.cpp:55-72): every word spellable with the
 * labels goes into the dictionary, followed by the space label (scorer.cpp:196-230, decoder_utils.cpp:164-193).
 * is_character_based != 0 (Scorer::is_character_based(): every word of the model is one UTF-8 character,
 * scorer.cpp:63-71): no dictionary (`words` is ignored, ctcdec_scorer_dict_size() is 0), no " " label needed, and the
 * hook is asked about EVERY appended character -- cond_log_prob gets the prefix's last (up to) max_order labels, the
 * new character last (ctc_beam_search_decoder.cpp:120-137 with prefix_to_score = prefix_new, scorer.cpp:172-174); at
 * read-out no last-word term is added (:174).  The device keeps one row of n_labels terms per trie node for such a
 * model: batch x (1 + beam x frames) x n_labels x 4 bytes, CTCDEC_E_UNSUPPORTED beyond 64 GiB. */
int ctcdec_scorer_create(const ctcdec_scorer_hooks *hooks, double alpha, double beta, const char *const *labels,
                         int n_labels, const char *const *words, int n_words, int max_order, int is_character_based,
                         void **scorer);
/* The same scorer from an ARPA text file or a KenLM binary file (told apart by the file's first bytes), with no hook to
 * supply: the library reads the n-gram tables itself and its
 * own hooks reproduce the reference Scorer over KenLM (Scorer::get_log_cond_prob / get_sent_log_prob, scorer.cpp:74-120)
 * bit for bit: the longest matching n-gram, KenLM's float sum of context backoffs in KenLM's order, "<s>" padding scored
 * as words, any out-of-vocabulary word -1000.  Word-based or character-based is read from the vocabulary as
 * scorer.cpp:61-71 does; max_order is the file's order; the dictionary is built from the unigrams.  Every entry point
 * that takes a scorer takes this one, and the accessors below behave as for a hook scorer.  The n-gram tables go to the
 * device once per device, and the beam kernel computes the LM terms of the trie nodes it creates itself: the offline
 * entries and ctcdec_decode_stream_host run without the per-frame host handshake (one launch per batch or chunk), and
 * the device keeps the last max_order - 1 word ids of every node, batch x (1 + beam x frames) x (max_order - 1) x 4
 * bytes (CTCDEC_E_UNSUPPORTED beyond 64 GiB).  The blocking entries rescore their results on the host, through this
 * scorer's hooks; ctcdec_decode_batch_lm_device_async and ctcdec_decode_stream_device rescore them on the device with
 * the same label-to-word front end over tables of the labels' bytes and the unigrams' spellings.
 * KenLM binary files (format version 5, as build_binary writes them): PROBING files keep their own hash tables, which
 * go to the device byte for byte and are searched there as KenLM searches them; TRIE, QUANT_TRIE, ARRAY_TRIE and
 * QUANT_ARRAY_TRIE files keep their search data (bit-packed word ids, values and next pointers, Bhiksha offset arrays,
 * quantization bins) byte for byte too, and the device walks the trie as KenLM's TrieSearch does, reading the values
 * KenLM reads (dequantized with the file's own bins).  The word ids are the file's.
 * Refused with CTCDEC_E_UNSUPPORTED, the reason in ctcdec_last_error(), anything the tables cannot reproduce exactly:
 * ARPA text: non-ARPA input, order 1 or above 6, counts that disagree with the sections, a malformed line, a duplicate
 * entry, an n-gram word missing from the unigrams, no <s> or </s>, an n-gram whose context is missing, a positive
 * log-prob, a NaN or +inf log-prob, a non-finite backoff.  A binary file (the reason says "KenLM binary"): a truncated
 * file or header, an unfinished build, a version other than 5, other endianness or type sizes, REST_PROBING, an
 * unknown model type or search version, order 1 or above 6, no vocabulary strings or a word count that disagrees
 * with the header, no <s> or </s>, region sizes that disagree with the file's length, a probing table with no empty
 * bucket, trie word ids or pointers out of range or out of order.  A file that cannot be opened is
 * CTCDEC_E_INVALID. */
int ctcdec_scorer_create_arpa(const char *path, double alpha, double beta, const char *const *labels, int n_labels,
                              void **scorer);
/* Diagnostic: *bytes = the bytes of a scorer from ctcdec_scorer_create_arpa's n-gram data that go to each device it
 * decodes on: the unigrams and the orders >= 2 (ARPA text: 32-byte entries, two or more slots per n-gram; a probing
 * file: its own tables; a trie file: its search data), not the dictionary or the front end's tables.  Needs no device.
 * A hook scorer is CTCDEC_E_UNSUPPORTED. */
int ctcdec_scorer_table_bytes(const void *scorer, size_t *bytes);
/* Diagnostic: the scorer's hooks on one label-id prefix -- cond_log_prob and sent_log_prob of ctcdec_scorer_hooks, for a
 * hook scorer or an ARPA scorer.  Labels must lie in [0, n_labels). */
int ctcdec_scorer_cond_log_prob(const void *scorer, const int32_t *labels, int n, double *out);
int ctcdec_scorer_sent_log_prob(const void *scorer, const int32_t *labels, int n, double *out);
/* Diagnostic: the read-out rescoring of [B, K] result rows in HOST buffers, as the decodes apply it (reference
 * DecoderState::decode, ctc_beam_search_decoder.cpp:173-208).  tokens [B, K, row_stride], lens [B, K], n_results [B]:
 * rows p < min(n_results[b], K) are rescored in scores [B, K] (which hold minus the raw prefix scores, as the finalize
 * kernel writes them), the others are left alone.  device < 0: on the host, through the scorer's hooks (any scorer);
 * device >= 0: by the read-out kernel on that device (a scorer from ctcdec_scorer_create_arpa only, else
 * CTCDEC_E_UNSUPPORTED).  Labels must lie in [0, n_labels) and lengths in [0, row_stride]. */
int ctcdec_scorer_rescore_rows(void *scorer, const int32_t *tokens, const int32_t *lens, const int32_t *n_results,
                               float *scores, int B, int K, int row_stride, int device);
/* Replaces: paddle_release_scorer, is_character_based, get_max_order, get_dict_size, reset_params
 * (binding.cpp:267-287). */
int ctcdec_scorer_destroy(void *scorer);
int ctcdec_scorer_is_character_based(const void *scorer);
int ctcdec_scorer_max_order(const void *scorer);
int ctcdec_scorer_dict_size(const void *scorer);
int ctcdec_scorer_reset_params(void *scorer, double alpha, double beta);

/* Replaces: paddle_beam_decode_lm -> beam_decode -> ctc_beam_search_decoder_batch with a scorer
 * (binding.cpp:122-140, ctc_beam_search_decoder.cpp:56-211).  HOST buffers, shaped like ctcdec_decode_batch_host.
 * The beam search runs on `device` in ONE kernel launch; after every frame each utterance's CTA hands the trie
 * nodes it created to the host through device-mapped pinned memory and waits for their LM terms (hook calls).
 * Environment: CTCDEC_LM_PER_FRAME=1 selects the older protocol (one launch per frame), CTCDEC_LM_THREADS=n the
 * number of host workers (default min(8, cores): more do not help, the frame is bound by the PCIe round trip). */
int ctcdec_decode_batch_lm_host(const ctcdec_config *cfg, void *scorer, const float *probs, const int32_t *seq_lens,
                                int B, int T, int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                int32_t *n_results, int32_t *flags, int device);

/* Bytes of device scratch ctcdec_decode_batch_lm_device needs for a [B, T, V] batch with this scorer: the regions of
 * ctcdec_workspace_bytes' plan, then the LM term and the dictionary state of every trie node (2 x batch x (1 + beam x
 * T) x 4 bytes, each 256-byte aligned), for a character-based model the per-node rows of LM terms (batch x (1 + beam x
 * T) x V x 4, CTCDEC_E_UNSUPPORTED beyond 64 GiB), for a scorer from ctcdec_scorer_create_arpa the per-node LM
 * histories (batch x (1 + beam x T) x (max_order - 1) x 4, CTCDEC_E_UNSUPPORTED beyond 64 GiB), and a device copy of
 * seq_lens.  Checks the scorer and the shape
 * like the decode does: the same refusals, no device needed. */
int ctcdec_lm_workspace_bytes(const ctcdec_config *cfg, const void *scorer, int B, int T, size_t *bytes);

/* ctcdec_decode_batch_lm_host with the input and the results on the DEVICE (the current device), in the caller's
 * workspace.  Extension: the reference's scorer path decodes CPU tensors only.
 *   input      [B, T, V] device buffer.  dtype -1: float32 probabilities, or log-probabilities if cfg->log_input;
 *              CTCDEC_DTYPE_F32 / F16 / BF16: raw logits, log-softmaxed per frame by the scan kernel as in
 *              ctcdec_decode_batch_device_logits (cfg->log_input is ignored; log_probs_out, optional, receives the
 *              float32 log-softmax rows the decode used).
 *   seq_lens   HOST int32 [B] or NULL: the host answers each utterance's per-frame handshake and must know its length.
 *   tokens / timesteps [B, beam, T], scores / lens [B, beam], n_results / flags [B]: device buffers, n_results and
 *              flags required (B > 0).  Rows p >= n_results[b] are left untouched.  scores hold the reported (approx_ctc)
 *              scores, as with the host entry.
 * BLOCKING, unlike the other device entry points: the host answers the beam kernel's per-frame handshake during the
 * call, which returns when every output is in place.  The prune and beam kernels go onto `stream` after the work
 * already queued there; the handshake's 8 s no-progress limit starts once that work has finished.  A stream that is
 * being captured into a CUDA graph is refused with CTCDEC_E_UNSUPPORTED before anything is enqueued.  The plan is the
 * host entry's (the same accepted shapes); CTCDEC_LM_PER_FRAME=1 selects one launch per frame here too.  A set
 * CTCDEC_FLAG_ERR_ARENA returns CTCDEC_E_INTERNAL, as with the host entry points.  Calls on one device serialise. */
int ctcdec_decode_batch_lm_device(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                                  const int32_t *seq_lens, int B, int T, int32_t *tokens, int32_t *timesteps,
                                  float *scores, int32_t *lens, int32_t *n_results, int32_t *flags,
                                  float *log_probs_out, void *workspace, size_t workspace_bytes, void *stream);

/* ctcdec_decode_batch_lm_device for a scorer from ctcdec_scorer_create_arpa, WITHOUT waiting: the same arguments, outputs
 * and workspace (ctcdec_lm_workspace_bytes), except that seq_lens is a DEVICE int32 [B] buffer (or NULL).  The prune,
 * beam and finalize kernels and the read-out kernel (the reference's approx_ctc rescoring, computed on the device from
 * the scorer's tables) are enqueued on `stream` after the work already queued there, and the call returns; the results
 * are in place when the stream gets past them.  After its checks the call allocates nothing, copies nothing to or
 * from pageable or pinned host memory and never synchronises, except on its first use of a scorer on a device, which
 * uploads the scorer's tables and raises the kernels' shared-memory limits.
 *   CUDA graphs: the call can be captured.  Decode once outside the capture first (same scorer, device and shapes): a
 *              call made during capture that would have to upload the tables or raise a kernel's limit returns
 *              CTCDEC_E_UNSUPPORTED instead; the capture stays valid (a refusal over a kernel's limit may leave part of
 *              the decode in the graph, which the caller then discards).  alpha and beta are read when the work is
 *              enqueued, so a graph replays the values it captured: capture again after ctcdec_scorer_reset_params.
 *   Errors of the kernels show in flags only: a set CTCDEC_FLAG_ERR_ARENA means the utterance's results are not valid
 *              (as with ctcdec_decode_stream_device).
 * A hook scorer returns CTCDEC_E_UNSUPPORTED (its language model runs on the host during the decode: use
 * ctcdec_decode_batch_lm_device).  The workspace and outputs must not be reused before the stream has finished with
 * them.  Enqueueing on one device serialises, the kernels of different streams overlap. */
int ctcdec_decode_batch_lm_device_async(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                                        const int32_t *seq_lens, int B, int T, int32_t *tokens, int32_t *timesteps,
                                        float *scores, int32_t *lens, int32_t *n_results, int32_t *flags,
                                        float *log_probs_out, void *workspace, size_t workspace_bytes, void *stream);

/* Bytes of device scratch ctcdec_decode_batch_lm_sweep_async needs for P (alpha, beta) pairs over a [B, T, V] batch:
 * ctcdec_lm_workspace_bytes(cfg, scorer, P x B, T), less the pruned rows of (P - 1) x B utterances (the input is scanned
 * once: B x T x NP x 4 bytes, and B x T x NP x 2 more when the vocabulary is cut, each region 256-byte aligned; NP is
 * the pruned row length, min(V, cutoff_top_n) + 3 -- V + 3 without a cut -- rounded up to a multiple of 8), plus the
 * pairs' table (16 x P bytes, 256-byte aligned).  The 64 GiB limits of the per-node rows and histories apply to the
 * P x B utterances.  The same refusals as ctcdec_lm_workspace_bytes, no device needed; also CTCDEC_E_INVALID for
 * P < 1 and CTCDEC_E_UNSUPPORTED for a hook scorer. */
int ctcdec_lm_sweep_workspace_bytes(const ctcdec_config *cfg, const void *scorer, int B, int T, int P, size_t *bytes);

/* Extension: a sweep of the language-model weights.  Decodes one batch under P pairs (alphas[p], betas[p]), host
 * double[P] arrays, in one enqueue: the vocabulary scan runs once over the B input utterances, then one beam CTA per
 * (pair, utterance).  Slice p of every output is exactly what ctcdec_decode_batch_lm_device_async returns for the same
 * batch after ctcdec_scorer_reset_params(scorer, alphas[p], betas[p]): each value goes through float32, as reset_params
 * stores it (reference Scorer::reset_params(float, float)), so the baseline is reset_params, not a scorer created with
 * the unrounded doubles.  The scorer's own alpha and beta are neither read nor changed.
 *   Arguments as ctcdec_decode_batch_lm_device_async (seq_lens a DEVICE int32 [B] buffer or NULL, log_probs_out
 *              [B, T, V], written once), except the outputs, all contiguous device buffers with a leading pair axis:
 *              tokens / timesteps [P, B, beam, T], scores / lens [P, B, beam], n_results / flags [P, B].  Slice p is
 *              laid out as a B-utterance decode writes it.  flags[p, b] carries the vocabulary scan's
 *              CTCDEC_FLAG_TIE_VOCAB bit of utterance b and the beam and finalize bits of its own decode.
 *   Workspace: ctcdec_lm_sweep_workspace_bytes.  The beam kernel runs with the block size a B-utterance decode gets:
 *              the 128- and 256-thread kernels may order comparator-equal results (CTCDEC_FLAG_TIE_FINAL) differently.
 *   CUDA graphs: as ctcdec_decode_batch_lm_device_async -- decode once outside the capture first.  After its checks the
 *              call copies nothing from pageable or pinned host memory: the pairs travel in kernel launch parameters,
 *              so a graph replays the pairs it captured.
 *   Errors of the kernels show in flags only: a set CTCDEC_FLAG_ERR_ARENA means that (pair, utterance)'s results are
 *              not valid.
 * A scorer from ctcdec_scorer_create_arpa only (word- or character-based, ARPA text or a KenLM binary); a hook scorer
 * returns CTCDEC_E_UNSUPPORTED (its terms float(cond_log_prob x alpha) are computed on the host), P < 1 or NULL alphas /
 * betas CTCDEC_E_INVALID. */
int ctcdec_decode_batch_lm_sweep_async(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                                       const int32_t *seq_lens, int B, int T, const double *alphas,
                                       const double *betas, int P, int32_t *tokens, int32_t *timesteps, float *scores,
                                       int32_t *lens, int32_t *n_results, int32_t *flags, float *log_probs_out,
                                       void *workspace, size_t workspace_bytes, void *stream);

/* The most language models one ctcdec_decode_batch_lm_mixed_async call takes: their LM slots (model tables, dictionary,
 * order and weights) travel in the parameters of one kernel launch. */
#define CTCDEC_LM_MIXED_MAX_MODELS 16

/* Bytes of device scratch ctcdec_decode_batch_lm_mixed_async needs for S scorers over a [B, T, V] batch.  When all S
 * pointers are one scorer, exactly ctcdec_lm_workspace_bytes(cfg, scorers[0], B, T).  Otherwise
 * ctcdec_lm_workspace_bytes(cfg, m, B, T) for the scorer m of the largest order (the per-node LM histories take the
 * largest order - 1 ids per node), less its 256 bytes of alignment slack, plus the slot table (256 bytes per scorer,
 * 256-byte aligned), the utterances' slot indices (B bytes, 256-byte aligned) and the 256 bytes of slack.  The refusals
 * of ctcdec_decode_batch_lm_mixed_async's checks of scorers and S, no device needed. */
int ctcdec_lm_mixed_workspace_bytes(const ctcdec_config *cfg, void *const *scorers, int S, int B, int T, size_t *bytes);

/* Extension: decode a batch whose utterances need different language models, in one enqueue.  Utterance b is decoded
 * with the model and weights of scorers[lm_index[b]]: every output of it, flags included, is bit for bit what
 * ctcdec_decode_batch_lm_device_async with that scorer gives for it -- against the sub-batch of that scorer's utterances
 * whenever both calls get the same beam-kernel block size, which holds up to 264 utterances; above that the two block
 * sizes may order comparator-equal rows (CTCDEC_FLAG_TIE_FINAL) differently.  Each scorer's alpha and beta are read
 * when the call is made.  Every beam CTA finds its model through its LM slot; the read-out rescores each row with its
 * utterance's model, front end and weights.  A call whose scorers are all one object is
 * ctcdec_decode_batch_lm_device_async.
 *   scorers [S]: scorers from ctcdec_scorer_create_arpa (ARPA text or any KenLM binary it takes; layout, order and
 *              weights may differ), 1 <= S <= CTCDEC_LM_MIXED_MAX_MODELS, all built for the decoder's labels (string
 *              for string) and all word-based or all character-based.
 *   lm_index   HOST int32 [B], each in [0, S): checked on the host.
 *   Everything else as ctcdec_decode_batch_lm_device_async: seq_lens a DEVICE int32 [B] buffer or NULL, device outputs,
 *              no waiting, capturable into a CUDA graph after one decode with these scorers outside the capture (the
 *              slots and indices travel in kernel launch parameters, so a graph replays the models and weights it
 *              captured).  Workspace: ctcdec_lm_mixed_workspace_bytes.
 * Refused: NULL scorers, S < 1 or S > CTCDEC_LM_MIXED_MAX_MODELS, NULL lm_index (B > 0) or an index outside [0, S), or
 * scorers built for different labels: CTCDEC_E_INVALID; a hook scorer beside any other scorer, or word-based beside
 * character-based models: CTCDEC_E_UNSUPPORTED. */
int ctcdec_decode_batch_lm_mixed_async(const ctcdec_config *cfg, void *const *scorers, int S, const int32_t *lm_index,
                                       const void *input, int dtype, const int32_t *seq_lens, int B, int T,
                                       int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                       int32_t *n_results, int32_t *flags, float *log_probs_out, void *workspace,
                                       size_t workspace_bytes, void *stream);

/* ---- streaming (OnlineCTCBeamDecoder) ------------------------------------------------------------- */

/* Replaces: paddle_get_decoder_state (binding.cpp:246-261).  The state (beam + trie + absolute frame
 * counter, reference ctc_beam_search_decoder.h:73-124) lives in device memory of `device`. */
int ctcdec_state_create(const ctcdec_config *cfg, int device, void **state);
/* The same with a word-based scorer (the `void *scorer` argument of paddle_get_decoder_state, binding.cpp:246-261).
 * The scorer is BORROWED and must outlive the state (reference ctc_beam_search_decoder.cpp:31); scorer == NULL is
 * ctcdec_state_create.  Chunks of such states are decoded by ctcdec_decode_stream_host: one persistent launch per
 * chunk with the per-frame hook handshake of ctcdec_decode_batch_lm_host, scores re-computed at eos like
 * DecoderState::decode (ctc_beam_search_decoder.cpp:164-211). */
int ctcdec_state_create_lm(const ctcdec_config *cfg, void *scorer, int device, void **state);
/* Replaces: paddle_release_state (binding.cpp:263-265). */
int ctcdec_state_destroy(void *state);
/* Frames consumed so far (reference DecoderState::abs_time_step). */
int ctcdec_state_frames(const void *state, int *frames);

/* Replaces: beam_decode_with_given_state / paddle_beam_decode_with_given_state ->
 * ctc_beam_search_decoder_batch_with_states (binding.cpp:153-241, ctc_beam_search_decoder.cpp:288-317).
 * probs [B, T, V] and seq_lens are HOST buffers holding the next chunk of every stream; states[b] is
 * advanced by min(seq_lens[b], T) frames; for streams with is_eos[b] != 0 the current beams are written
 * to tokens/timesteps [B, beam, out_T] (rows of other streams untouched), scores/lens [B, beam].
 * out_T must be >= the longest prefix (the number of frames consumed is always enough).
 * The states of one call share the decoder configuration and the device.  Their scorers are one object (or none), or,
 * as the reference's per-state Scorer allows, different scorers from ctcdec_scorer_create_arpa -- at most
 * CTCDEC_LM_MIXED_MAX_MODELS of them, all word-based or all character-based, built for the same labels: each stream
 * then decodes with its own scorer's model, and its eos read-out uses that scorer's alpha and beta as they are when the
 * call is made.  Refused: a different configuration or device, states with a scorer beside states without one, a hook
 * scorer beside another scorer, word-based beside character-based models, more than CTCDEC_LM_MIXED_MAX_MODELS
 * scorers (CTCDEC_E_UNSUPPORTED); scorers built for different labels (CTCDEC_E_INVALID). */
int ctcdec_decode_stream_host(const float *probs, const int32_t *seq_lens, int B, int T, void *const *states,
                              const uint8_t *is_eos, int32_t *tokens, int32_t *timesteps, int out_T, float *scores,
                              int32_t *lens, int32_t *n_results, int32_t *flags);

/* Bytes of device scratch one ctcdec_decode_stream_device call of B streams and T frames needs (the pruned rows of
 * the chunk and the per-call tables of stream pointers). */
int ctcdec_stream_workspace_bytes(const ctcdec_config *cfg, int B, int T, size_t *bytes);
/* The same for the B states of a call (B >= 1, checked as ctcdec_decode_stream_device checks them): exactly
 * ctcdec_stream_workspace_bytes when their scorers are one object (or none); for states of S > 1 different scorers
 * that plus their LM slots, al256(B) + al256(256 x S) bytes (al256: rounded up to a multiple of 256). */
int ctcdec_stream_states_workspace_bytes(void *const *states, int B, int T, size_t *bytes);

/* ctcdec_decode_stream_host with the chunk and the results on the DEVICE, enqueued on `stream` (a cudaStream_t of the
 * states' device, which must be the current device).  Extension: the reference decodes CPU tensors only.
 *   probs      [B, T, V] device buffer.  dtype -1: float32 probabilities, or log-probabilities if cfg->log_input;
 *              CTCDEC_DTYPE_F32 / F16 / BF16: raw logits, log-softmaxed per frame by the scan kernel as in
 *              ctcdec_decode_batch_device_logits (cfg->log_input is ignored).
 *   seq_lens   HOST int32 [B] or NULL; is_eos and states are host arrays too.  The host therefore knows every
 *              stream's frame count: ctcdec_state_frames is exact as soon as the call returns.
 *   tokens / timesteps [B, beam, out_T], scores / lens [B, beam]: device buffers, written for eos streams only (rows
 *              p < n_results[b]); out_T must be >= frames consumed after this chunk by every eos stream (checked).
 *   n_results / flags [B]: device buffers, required.  Every entry is written: n_results 0 for streams not at eos,
 *              flags the CTCDEC_FLAG_* bits of this chunk (and of the finalize for eos streams).  A set
 *              CTCDEC_FLAG_ERR_ARENA means the stream's results are not valid; this call cannot report it as an error
 *              code without waiting for the kernels.
 * The call does not wait for the device, with one exception: when a stream's node arena must grow (1 + beam x frames
 * nodes, capacity doubling from 256 frames: about log2(frames / 256) times per stream) the old arena is copied on
 * `stream` and the host waits for that copy before freeing it.  States with a scorer from ctcdec_scorer_create_arpa are
 * decoded here too (the first call uploads the scorer's tables): the beam kernel computes the LM terms, and at eos the
 * read-out kernel rescores the eos streams' rows on the device (alpha and beta as they are when the call is made).
 * States with a hook scorer return CTCDEC_E_UNSUPPORTED (their beam kernel needs the per-frame host handshake of
 * ctcdec_decode_stream_host).  The workspace and the outputs
 * must not be reused before the work on `stream` is done, as with ctcdec_decode_batch_device.
 * Device-path calls record an event on each state; ctcdec_decode_stream_host waits for it on its own stream, a later
 * device-path call on another stream waits for it too, and ctcdec_state_destroy synchronises it before freeing. */
int ctcdec_decode_stream_device(const void *probs, int dtype, const int32_t *seq_lens, int B, int T,
                                void *const *states, const uint8_t *is_eos, int32_t *tokens, int32_t *timesteps,
                                int out_T, float *scores, int32_t *lens, int32_t *n_results, int32_t *flags,
                                void *workspace, size_t workspace_bytes, void *stream);

/* Extension: the COMMITTED prefix of every stream -- the part of the transcript no later chunk can change.  It is the
 * trie path from the root to the lowest common ancestor of the stream's current beam members: the longest common
 * prefix of the rows an eos read-out would return now, which also starts every row of any later read-out, tokens and
 * timesteps alike (DESIGN.md, "Streaming on the device").
 *   committed  device int32 [B]: the committed depth (never decreases from chunk to chunk);
 *   since      device int32 [B] or NULL (= 0): positions the caller already has, normally the previous call's
 *              committed[b].  A value outside [0, committed depth] is taken as 0;
 *   tokens / timesteps  device int32 [B, cap]: row b receives positions [since[b], committed[b]) from column 0;
 *              columns at or beyond cap are not written (compare committed - since with cap).
 * Reads the states only, so any state works, including one with a scorer advanced by ctcdec_decode_stream_host.
 * Enqueued on `stream` (the states' device must be the current device); does not wait for the device. */
int ctcdec_stream_committed_device(void *const *states, int B, const int32_t *since, int32_t *committed,
                                   int32_t *tokens, int32_t *timesteps, int cap, void *stream);

/* Extension: compaction of streaming states.  A state's node arena only grows while it decodes (up to beam nodes per
 * frame); everything a later chunk, eos read-out or ctcdec_stream_committed_device can read lies on the paths from
 * the root to the current beam members.  This call keeps exactly those nodes, renumbered in their old order (the
 * root stays 0, a parent below its children), with their LM terms, histories, dictionary states and rows, rewrites the
 * node ids in each state block and frees the old arrays.  Every later output of a compacted stream equals, bit for
 * bit, that of the same stream never compacted (DESIGN.md, "Streaming on the device").
 *   nodes_kept  host int64 [B] or NULL: the nodes each state holds now.
 * Capacity after the call: max(1 + beam x 256, kept + beam x 256) nodes; decoding grows it again as it needs, by the
 * nodes kept plus beam x frames consumed since.
 * The states may come from different configurations and scorers but must live on one device, the current one.
 * Ordered after the states' pending device-path work on `stream`; the call waits for the device twice (to size the
 * new arrays, and before freeing the old ones) and returns when it is done.  Refused before anything is enqueued:
 * NULL or duplicate states (CTCDEC_E_INVALID), states with a hook scorer (CTCDEC_E_UNSUPPORTED: the host mirror of
 * their trie is indexed by node id), states of several devices, and a stream being captured into a CUDA graph
 * (CTCDEC_E_UNSUPPORTED).  An allocation failure leaves every state as it was. */
int ctcdec_stream_compact(void *const *states, int B, int64_t *nodes_kept, void *stream);
/* Extension: the device memory a streaming state holds: its node arena, state block and scorer arrays. */
int ctcdec_state_device_bytes(const void *state, size_t *bytes);

/* ---- measurement hook (bench.py) --------------------------------------------------------------------
 * With profiling enabled on the calling thread, ctcdec_decode_batch_device records CUDA events on its stream
 * around each of its kernels; ctcdec_profile_read waits for the last decode of this thread and returns
 * the device time in milliseconds of {prune/log scan, beam search, finalize}.  When nothing is cut from the
 * vocabulary (cutoff_prob = 1 and cutoff_top_n >= vocab_size) the beam kernel runs the backtrace itself: there
 * is no finalize kernel, its time is reported as 0, and the beam search time includes the backtrace. */
int ctcdec_profile_enable(int on);
int ctcdec_profile_read(float *ms3);
/* Diagnostic: if device_buffer (int64 [B][16] followed by int64 [B][16][32], device memory) is non-NULL, every
 * following ctcdec_decode_batch_device call of this thread runs the instrumented build of the beam kernel:
 * thread 0 of each CTA records the clock cycles it spent in each barrier-delimited region of the frame loop,
 * and every warp the cycles it was busy before each of the main barriers (tools/region_timing.py).  Built for
 * 256-thread launches with beam sizes 65..256 and for the scorer path; other shapes return CTCDEC_E_UNSUPPORTED. */
int ctcdec_profile_region_cycles(void *device_buffer);

/* The device entry points leave their results on the GPU; this brings the meaningful part of the two big tensors to the
 * host the way ctcdec_decode_batch_host does: columns [0, max_len) of every row ([rows][row_stride] int32 on both
 * sides, rows = batch x beam), two strided DMA copies on `stream`, synchronised before returning.  Page-locked
 * destinations make it run at PCIe speed (reference binding.cpp:79-99 writes only [:len] of a row, too). */
int ctcdec_rows_to_host(const int32_t *d_tokens, const int32_t *d_timesteps, long long rows, int row_stride, int max_len,
                        int32_t *tokens, int32_t *timesteps, void *stream);

/* ---- diagnostics used by the tests (device self-check of the bit-exact libm restatements) ----------- */
/* y[i] = f(x[i]) computed ON THE DEVICE; which: 0 expf, 1 logf, 2 float(log(double(x) + FLT_MIN)),
 * 3 log_sum_exp(x[i], x2[i]).  Host pointers. */
int ctcdec_selftest_math(int which, const float *x, const float *x2, float *y, size_t n, int device);
/* the double chain of the vocabulary cut (reference decoder_utils.cpp:26-31): which 0 exp(x) for x <= 0 (arguments under
 * -40 give 0.0, see glibc_math.cuh), 1 log(x) for normal positive x, 2 log_sum_exp<double>(x[i], x2[i]). */
int ctcdec_selftest_math_f64(int which, const double *x, const double *x2, double *y, size_t n, int device);

#ifdef __cplusplus
}
#endif
#endif /* CTCDECODE_B200_H_ */

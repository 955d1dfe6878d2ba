// C ABI of ctcdecode_b200 (include/ctcdecode_b200.h): kernel wrappers, launch logic, workspace carve-up,
// host-buffer entry points and the device-resident streaming state.  sm_90a only; there is no CPU path.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <atomic>
#include <chrono>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ctcdecode_b200.h"
#include "beam_program.cuh"
#include "compact_program.cuh"
#include "plan.h"
#include "lm_host.h"
#include "prune_program.cuh"
#include "pack_program.cuh"

namespace ctc {

// ---------------------------------------------------------------------------------------------------
//  kernels
// ---------------------------------------------------------------------------------------------------
// two co-resident CTAs per SM (one for NT = 1024, three for NT = 128): 128 registers per thread up to NT = 256, 64 at NT = 512.
// A config-2 batch of 256 utterances is 1.73 CTAs per SM, and the frame loop wants its registers.
// KPT: beam size rounded up to 32 as a compile-time constant (0 = generic), TIMING: per-region cycle counters.
// (__grid_constant__: a scorer CTA without a slot table reads the call's model through a pointer to the parameters)
template <int NT, bool SORTED, bool LM, int KPT, bool TIMING>
__global__ void __launch_bounds__(NT, (NT >= 1024 ? 1 : NT <= 128 ? 3 : 2)) beam_kernel(const __grid_constant__ BeamParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  beam_cta_run<NT, SORTED, LM, KPT, TIMING>(p, (int)blockIdx.x, smem);
}

template <int NT>
__global__ void __launch_bounds__(NT) finalize_kernel(const BeamParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  finalize_cta_run<NT>(p, (int)blockIdx.x, smem);
}

// committed prefix of a streaming state: one CTA per stream, the stream's arena / state pointers travel in the
// launch parameters (up to kCommitPerLaunch streams per launch), so the call needs no workspace
constexpr int kCommitPerLaunch = 192;
struct CommitArgs {
  const Node *arena[kCommitPerLaunch];
  const int *state[kCommitPerLaunch];
  int K, b0, cap;
  const int *since;
  int *committed, *tokens, *timesteps;
};
template <int NT>
__global__ void __launch_bounds__(NT) committed_kernel(const CommitArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int i = (int)blockIdx.x, b = a.b0 + i;
  committed_cta_run<NT>(a.arena[i], a.state[i], a.K, a.since ? a.since[b] : 0, &a.committed[b],
                        a.tokens + (size_t)b * a.cap, a.timesteps + (size_t)b * a.cap, a.cap, smem);
}

// arena compaction of streaming states (compact_program.cuh): one CTA per stream, the stream's arrays in the launch
// parameters, kCompactPerLaunch streams per launch
constexpr int kCompactPerLaunch = 32;
constexpr int kCompactNT = 256;
struct CompactMarkArgs {
  const Node *arena[kCompactPerLaunch];
  const int *state[kCompactPerLaunch];
  int *map[kCompactPerLaunch];
  int K[kCompactPerLaunch], cap[kCompactPerLaunch];
  int *kept;
};
__global__ void __launch_bounds__(kCompactNT) compact_mark_kernel(const CompactMarkArgs a) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int i = (int)blockIdx.x;
  compact_mark_cta_run<kCompactNT>(a.arena[i], a.state[i], a.K[i], a.cap[i], a.map[i], &a.kept[i], smem);
}
struct CompactGatherArgs {
  CompactJob job[kCompactPerLaunch];
};
static_assert(sizeof(CompactGatherArgs) <= 4096, "the jobs must fit the kernel parameters");
__global__ void __launch_bounds__(kCompactNT) compact_gather_kernel(const CompactGatherArgs a) {
  compact_gather_cta_run<kCompactNT>(a.job[blockIdx.x]);
}

// The per-call tables of a streaming chunk (each stream's arena, state block, capacity, eos flag, scorer arrays and
// chunk length), in device memory.  A kernel writes them from its launch parameters, kTabPerLaunch streams per
// launch: the call needs no host staging buffer that would have to outlive an asynchronous copy.
struct StreamTabLayout { size_t arenas, states, caps, fin, lmar, dst, rows, lens, total; };
static StreamTabLayout stream_tab_layout(int B) {
  const size_t p = al256((size_t)B * 8), i = al256((size_t)B * 4);
  StreamTabLayout t;
  t.arenas = 0; t.states = p; t.caps = 2 * p; t.fin = t.caps + i; t.lmar = t.fin + al256((size_t)B);
  t.dst = t.lmar + p; t.rows = t.dst + p; t.lens = t.rows + p; t.total = t.lens + i;
  return t;
}
constexpr int kTabPerLaunch = 64;
struct StreamTabArgs {
  unsigned char *tab;
  StreamTabLayout L;
  int b0, n;
  Node *arena[kTabPerLaunch];
  int *state[kTabPerLaunch];
  float *lmar[kTabPerLaunch];
  int *dst[kTabPerLaunch];
  float *rows[kTabPerLaunch];
  int cap[kTabPerLaunch], len[kTabPerLaunch];
  unsigned char fin[kTabPerLaunch];
};
__global__ void stream_table_kernel(const StreamTabArgs a) {
  const int i = (int)threadIdx.x;
  if (i >= a.n) return;
  const int b = a.b0 + i;
  reinterpret_cast<Node **>(a.tab + a.L.arenas)[b] = a.arena[i];
  reinterpret_cast<int **>(a.tab + a.L.states)[b] = a.state[i];
  reinterpret_cast<int *>(a.tab + a.L.caps)[b] = a.cap[i];
  a.tab[a.L.fin + b] = a.fin[i];
  reinterpret_cast<float **>(a.tab + a.L.lmar)[b] = a.lmar[i];
  reinterpret_cast<int **>(a.tab + a.L.dst)[b] = a.dst[i];
  reinterpret_cast<float **>(a.tab + a.L.rows)[b] = a.rows[i];
  reinterpret_cast<int *>(a.tab + a.L.lens)[b] = a.len[i];
}

// The (alpha, beta) pairs of a sweep (ctcdec_decode_batch_lm_sweep_async) into the workspace, from the launch parameters
// (kTabPerLaunch pairs per launch), so that the call copies nothing from host memory and a graph replays the pairs it
// captured.
struct SweepPairArgs {
  double *tab;
  int p0, n;
  double ab[2 * kTabPerLaunch];
};
__global__ void sweep_pairs_kernel(const SweepPairArgs a) {
  const int i = (int)threadIdx.x;
  if (i >= a.n) return;
  a.tab[2 * (a.p0 + i)] = a.ab[2 * i];
  a.tab[2 * (a.p0 + i) + 1] = a.ab[2 * i + 1];
}

// The LM slots of a decode over several models (ctcdec_decode_batch_lm_mixed_async) and each utterance's slot index
// into the workspace, from the launch parameters: the call copies nothing from host memory, and a graph replays the
// models and weights it captured.  All slots travel in one launch (kMaxLmSlots of them: CTCDEC_LM_MIXED_MAX_MODELS),
// the indices kSlotIndexPerLaunch per launch.
constexpr int kMaxLmSlots = CTCDEC_LM_MIXED_MAX_MODELS;
constexpr size_t kLmSlotBytes = 256;  // workspace bytes per slot (ctcdec_lm_mixed_workspace_bytes)
static_assert(sizeof(LmSlot) <= kLmSlotBytes, "an LM slot outgrew its workspace share");
struct LmSlotArgs {
  LmSlot *tab;
  int S;
  LmSlot slot[kMaxLmSlots];
};
static_assert(sizeof(LmSlotArgs) <= 4096, "the slots must fit the kernel parameters");
__global__ void lm_slots_kernel(const LmSlotArgs a) {
  if ((int)threadIdx.x < a.S) a.tab[threadIdx.x] = a.slot[threadIdx.x];
}
constexpr int kSlotIndexPerLaunch = 4000;
struct SlotIndexArgs {
  unsigned char *tab;
  int b0, n;
  unsigned char index[kSlotIndexPerLaunch];
};
__global__ void lm_slot_index_kernel(const SlotIndexArgs a) {
  for (int i = (int)threadIdx.x; i < a.n; i += (int)blockDim.x) a.tab[a.b0 + i] = a.index[i];
}

// Sweep: the prune scan's flags of the B input rows (slice 0 of flags [P][B]) into the other P - 1 slices, before the
// beam and finalize kernels OR in each CTA's own bits.
__global__ void sweep_flags_kernel(int32_t *flags, int B, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[B + i] = flags[i % B];
}

// Read-out of an ARPA scorer's results (ngram_readout_row, reference DecoderState::decode): one thread per [B, K] result
// row, rows p >= n_results[b] skipped, scores rescored in place.  Each row is a serial chain of hash probes (about
// words x order of them).  Rows take their utterance's LM slot in the per-row instantiations (compile-time choices:
// what a row loads stays live across its walks, and the single-model instantiation is kept free of that):
//   kReadSweep: row r takes the pair ab[r / (pair_B x K)] instead of alpha / beta (the model is m, f);
//   kReadSlots: row r of utterance b takes model, front end and weights of slots[slot_of[b]].
constexpr int kReadoutThreads = 128;
enum { kReadOne = 0, kReadSweep = 1, kReadSlots = 2 };
template <int MODE>
__global__ void __launch_bounds__(kReadoutThreads) lm_readout_kernel(const NgramView m, const NgramFront f, double alpha,
                                                                     double beta, const double *ab, int pair_B,
                                                                     const LmSlot *slots, const unsigned char *slot_of,
                                                                     const int32_t *tokens,
                                                                     const int32_t *lens, const int32_t *n_results,
                                                                     float *scores, int B, int K, int row_stride) {
  const long long r = (long long)blockIdx.x * kReadoutThreads + threadIdx.x;
  if (r >= (long long)B * K) return;
  const int b = (int)(r / K), p = (int)(r % K);
  if (p >= n_results[b]) return;
  if (MODE == kReadSlots) {
    const LmSlot &sl = slots[slot_of[b]];
    scores[r] = ngram_readout_row(sl.ngram, sl.front, tokens + r * row_stride, lens[r], scores[r], sl.lm_alpha, sl.beta);
    return;
  }
  if (MODE == kReadSweep) {
    const int q = b / pair_B;
    alpha = ab[2 * q];
    beta = ab[2 * q + 1];
  }
  scores[r] = ngram_readout_row(m, f, tokens + r * row_stride, lens[r], scores[r], alpha, beta);
}

__global__ void selftest_math_f64_kernel(int which, const double *x, const double *x2, double *y, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    y[i] = which == 0 ? exp_glibc_nonpos(x[i]) : which == 1 ? log_glibc(x[i]) : lse_d(x[i], x2[i]);
}

__global__ void selftest_math_kernel(int which, const float *x, const float *x2, float *y, size_t n) {
  __shared__ uint64_t exptab[32];
  __shared__ double logftab[32];
  __shared__ double logtab[256];
  for (int i = threadIdx.x; i < 32; i += blockDim.x) { exptab[i] = kExp2fTab[i]; logftab[i] = kLogfTab[i]; }
  for (int i = threadIdx.x; i < 256; i += blockDim.x) logtab[i] = kLogTab[i];
  __syncthreads();
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float r;
    if (which == 0) r = expf_glibc_t(x[i], exptab);
    else if (which == 1) r = logf_glibc_t(x[i], logftab);
    else if (which == 2) r = logprob_glibc_t(x[i], logtab);
    else r = lse_smem(x[i], x2[i], exptab, logftab);
    y[i] = r;
  }
}

// ---------------------------------------------------------------------------------------------------
//  errors
// ---------------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static int fail(int code, const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CU(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return fail(CTCDEC_E_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
  } while (0)

// utterances the calling thread is about to have in flight together (host entry point: all its groups)
static thread_local int g_batch_in_flight = 0;

// set while ctcdec_decode_batch_lm_device_async enqueues into a stream that is being captured: a kernel whose dynamic
// shared-memory limit has not been raised on this device yet is refused instead of raised
static thread_local bool g_capturing = false;
static const char kCaptureFirst[] = "decode once outside the capture first";

// the kernels raise CTCDEC_FLAG_ERR_ARENA for an utterance whose node arena / anchor table ran out or whose scorer
// handshake was abandoned: its results are not valid, so the host entry points fail instead of returning them
static int check_error_flags(const int *flags, int B) {
  for (int b = 0; b < B; ++b)
    if (flags[b] & FLAG_ERR_ARENA)
      return fail(CTCDEC_E_INTERNAL, "utterance %d: the beam kernel reported an internal error (node arena / anchor table "
                  "exhausted or scorer handshake abandoned); results are not valid", b);
  return CTCDEC_OK;
}

// lm: a scorer is attached (pl->L is then the scorer kernel's layout)
static int make_plan(const ctcdec_config *cfg, int B, int T, Plan *pl, bool lm = false) {
  char msg[256];
  int nt = 0;
  if (const char *e = getenv("CTCDEC_NT")) nt = atoi(e);  // tuning knob: threads per CTA of the beam kernel
  const int rc = make_plan_core(cfg, B, T, pl, msg, sizeof(msg), nt, g_batch_in_flight, lm);
  if (rc) return fail(rc, "%s", msg);
  return CTCDEC_OK;
}

// Raises kernel Kern's dynamic shared-memory limit on the current device to `bytes`, once per device and size:
// cudaFuncSetAttribute on a kernel that is running waits for it, which would serialise the utterance groups the host
// entry point pipelines.  A limit that is not raised yet is refused while a stream is being captured.  (Keyed on the
// kernel itself: every beam_kernel instance has the same function type.)
template <auto Kern>
static int raise_smem_limit(size_t bytes, const char *what) {
  if (bytes <= 48 * 1024) return CTCDEC_OK;
  static std::atomic<int> limit[64];
  static std::mutex limit_mu;
  int dev = 0;
  CU(cudaGetDevice(&dev));
  if ((int)bytes > limit[dev & 63].load(std::memory_order_acquire)) {
    if (g_capturing) return fail(CTCDEC_E_UNSUPPORTED, "%s kernel not prepared on device %d: %s", what, dev, kCaptureFirst);
    std::lock_guard<std::mutex> lk(limit_mu);  // (check again under the lock: two host threads, same device)
    if ((int)bytes > limit[dev & 63].load(std::memory_order_acquire)) {
      CU(cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
      limit[dev & 63].store((int)bytes, std::memory_order_release);
    }
  }
  return CTCDEC_OK;
}

template <int NT, bool SORTED, bool LM, int KPT, bool TIMING>
static int launch_beam_k(const BeamParams &bp, int B, cudaStream_t s) {
  const int smem_bytes = bp.L.total + (TIMING ? 4096 : 0);  // TIMING: [16][32] per-warp counters behind the layout
  int rc = raise_smem_limit<beam_kernel<NT, SORTED, LM, KPT, TIMING>>(smem_bytes, "beam");
  if (rc) return rc;
  beam_kernel<NT, SORTED, LM, KPT, TIMING><<<B, NT, smem_bytes, s>>>(bp);
  CU(cudaGetLastError());
  return CTCDEC_OK;
}

// Instantiations: without a scorer the usual block sizes (128 / 256 threads) come specialised for beam sizes up to
// 32 / 64 / 128 / 256 slots (every slot-array address an immediate) besides the generic kernel; the scorer path,
// whose frame time is the host handshake, and the tuning-knob block sizes use the generic kernel only.  The
// per-region cycle counters (diagnostic) exist for the 256-thread kernels of beam 65..256 and for the scorer path.
template <int NT, bool SORTED>
static int launch_beam_ns(const BeamParams &bp, int B, cudaStream_t s) {
  const bool lm = bp.dict_next != nullptr, timing = bp.timing != nullptr;
  const int KP = bp.L.KP;
  if (lm) {
    if (timing) {
      if constexpr (NT <= 256) return launch_beam_k<NT, SORTED, true, 0, true>(bp, B, s);
      else return fail(CTCDEC_E_UNSUPPORTED, "region timing is built for 128 / 256 threads only");
    }
    return launch_beam_k<NT, SORTED, true, 0, false>(bp, B, s);
  }
  if (timing) {
    if constexpr (NT == 256) {
      if (KP == 128) return launch_beam_k<NT, SORTED, false, 128, true>(bp, B, s);
      if (KP == 256) return launch_beam_k<NT, SORTED, false, 256, true>(bp, B, s);
    }
    return fail(CTCDEC_E_UNSUPPORTED, "region timing is built for 256 threads and beam sizes 65..256 only");
  }
  if constexpr (NT <= 256) {
    if (KP == 32) return launch_beam_k<NT, SORTED, false, 32, false>(bp, B, s);
    if (KP == 64) return launch_beam_k<NT, SORTED, false, 64, false>(bp, B, s);
    if (KP == 128) return launch_beam_k<NT, SORTED, false, 128, false>(bp, B, s);
    if (KP == 256) return launch_beam_k<NT, SORTED, false, 256, false>(bp, B, s);
  }
  return launch_beam_k<NT, SORTED, false, 0, false>(bp, B, s);
}

static int launch_beam(const BeamParams &bp_in, const Plan &pl, int B, cudaStream_t s) {
  BeamParams bp = bp_in;
  bp.L = pl.L;
  if (const char *e = getenv("CTCDEC_HEUR_BIAS")) bp.heur_bias = (float)atof(e);  // test knob: make the checked bound fail
  if (const char *e = getenv("CTCDEC_NO_FAST")) bp.no_fast = atoi(e);  // test knob: 1 = general back half in every frame, 2 = no head offload
  if (const char *e = getenv("CTCDEC_SEG")) bp.L.seg = std::max(1, std::min(bp.L.seg, atoi(e)));  // test knob: small list segments
  const bool generic = getenv("CTCDEC_GENERIC_KP") != nullptr;  // test knob: force the run-time-KP kernel
  if (generic && !bp.timing && !bp.dict_next) {
    switch (pl.NT) {
      case 128: return pl.sorted ? launch_beam_k<128, true, false, 0, false>(bp, B, s) : launch_beam_k<128, false, false, 0, false>(bp, B, s);
      case 256: return pl.sorted ? launch_beam_k<256, true, false, 0, false>(bp, B, s) : launch_beam_k<256, false, false, 0, false>(bp, B, s);
      default: break;
    }
  }
  switch (pl.NT) {
    case 128: return pl.sorted ? launch_beam_ns<128, true>(bp, B, s) : launch_beam_ns<128, false>(bp, B, s);
    case 160: return pl.sorted ? launch_beam_ns<160, true>(bp, B, s) : launch_beam_ns<160, false>(bp, B, s);
    case 192: return pl.sorted ? launch_beam_ns<192, true>(bp, B, s) : launch_beam_ns<192, false>(bp, B, s);
    case 256: return pl.sorted ? launch_beam_ns<256, true>(bp, B, s) : launch_beam_ns<256, false>(bp, B, s);
    case 1024: return pl.sorted ? launch_beam_ns<1024, true>(bp, B, s) : launch_beam_ns<1024, false>(bp, B, s);
    default: return pl.sorted ? launch_beam_ns<512, true>(bp, B, s) : launch_beam_ns<512, false>(bp, B, s);
  }
}

struct PruneInput {
  const void *data;   // probabilities / log-probabilities (kind IN_F32) or logits
  int kind;           // IN_F32, IN_LOGITS_F32, IN_LOGITS_F16, IN_LOGITS_BF16
  float *lsm_out;     // optional: the float32 log-softmax rows (logits kinds)
  bool blank_prob = false;  // scorer path: also emit the row trailer [NP-3] (the reference's blank_prob)
};

template <bool SORTED, int KPL, bool LOGITS>
static int launch_prune_k(const PruneParams &pp, int grid, int threads, size_t smem, cudaStream_t s) {
  const int rc = raise_smem_limit<prune_kernel<SORTED, KPL, LOGITS>>(smem, "prune");
  if (rc) return rc;
  prune_kernel<SORTED, KPL, LOGITS><<<grid, threads, smem, s>>>(pp);
  return CTCDEC_OK;
}

// the prune scan of B utterances into the pruned rows and characters of the plan's workspace ws
static int launch_prune(const ctcdec_config *cfg, const Plan &pl, const PruneInput &in, const int *seq_lens, int B,
                        int T, unsigned char *ws, int *flags, cudaStream_t s) {
  float *const lp = reinterpret_cast<float *>(ws + pl.off_lp);
  uint16_t *const idx = pl.sorted ? reinterpret_cast<uint16_t *>(ws + pl.off_idx) : nullptr;
  PruneParams pp;
  memset(&pp, 0, sizeof(pp));
  const bool logits = in.kind != IN_F32;
  pp.probs = logits ? nullptr : static_cast<const float *>(in.data);
  pp.logits = logits ? in.data : nullptr;
  pp.in_kind = in.kind; pp.lsm_out = logits ? in.lsm_out : nullptr;
  pp.seq_lens = seq_lens; pp.B = B; pp.T = T; pp.V = cfg->vocab_size; pp.NP = pl.NP;
  pp.blank = cfg->blank_id; pp.log_input = logits ? 1 : cfg->log_input; pp.top_n = cfg->cutoff_top_n;
  pp.cp_active = pl.cp_active; pp.cutoff_prob = cfg->cutoff_prob; pp.P = pl.P;
  {
    const double cp = cfg->cutoff_prob, band = 1e-9 * (1.0 + std::fabs(cp));
    pp.cp_s_fire = std::expm1(cp); pp.cp_s_lo = std::expm1(cp - band); pp.cp_s_hi = std::expm1(cp + band);
  } pp.lp = lp; pp.idx = idx;
  pp.flags = flags;
  pp.want_blank_prob = in.blank_prob ? 1 : 0;
  const int V = cfg->vocab_size;
  pp.Vpad = (V + 3) / 4 * 4;
  const long long frames = (long long)B * T;
  if (frames == 0) return CTCDEC_OK;
  int rc = CTCDEC_OK;
  const PruneShape ps = prune_shape(pl, V, logits);
  const int wpc = ps.wpc;
  const size_t smem = ps.smem;
  if (!pl.sorted) {
    const int grid = (int)std::min<long long>((frames + wpc - 1) / wpc, kNumSMs * 16);
    rc = logits ? launch_prune_k<false, 0, true>(pp, grid, wpc * 32, smem, s)
                : launch_prune_k<false, 0, false>(pp, grid, wpc * 32, smem, s);
  } else {
    const int grid = (int)std::min<long long>((frames + wpc - 1) / wpc, kNumSMs * 8);
    if (V <= 256)
      rc = logits ? launch_prune_k<true, 8, true>(pp, grid, wpc * 32, smem, s) : launch_prune_k<true, 8, false>(pp, grid, wpc * 32, smem, s);
    else if (V <= 1024)
      rc = logits ? launch_prune_k<true, 32, true>(pp, grid, wpc * 32, smem, s) : launch_prune_k<true, 32, false>(pp, grid, wpc * 32, smem, s);
    else
      rc = logits ? launch_prune_k<true, 0, true>(pp, grid, wpc * 32, smem, s) : launch_prune_k<true, 0, false>(pp, grid, wpc * 32, smem, s);
  }
  if (rc) return rc;
  CU(cudaGetLastError());
  return CTCDEC_OK;
}

static int launch_finalize(const BeamParams &bp, int B, cudaStream_t s) {
  const size_t smem = finalize_smem_bytes(bp.K);
  const int rc = raise_smem_limit<finalize_kernel<1024>>(smem, "finalize");
  if (rc) return rc;
  // 1024 threads: the backtrace is a latency-bound pointer chase, its only resource is chains in flight
  finalize_kernel<1024><<<B, 1024, smem, s>>>(bp);
  CU(cudaGetLastError());
  return CTCDEC_OK;
}

// sm_90a code runs on compute capability 9.0 devices only
static bool is_sm90(int dev) {
  int major = 0, minor = 0;
  return cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) == cudaSuccess &&
         cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) == cudaSuccess && major == 9 && minor == 0;
}

static int check_device() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail(CTCDEC_E_NO_DEVICE, "no CUDA device: %s (this library has no CPU fallback)", cudaGetErrorString(e));
  if (!is_sm90(dev)) return fail(CTCDEC_E_NO_DEVICE, "device %d is not compute capability 9.0; the kernels are built for sm_90a only", dev);
  return CTCDEC_OK;
}

// makes `device` (an index of the per-device cache and locks) the current device and checks it
static int use_device(int device) {
  if (device < 0 || device >= 64) return fail(CTCDEC_E_INVALID, "device %d out of range", device);
  if (cudaSetDevice(device) != cudaSuccess)
    return fail(CTCDEC_E_NO_DEVICE, "cudaSetDevice(%d) failed (this library has no CPU fallback)", device);
  return check_device();
}

// the current device, checked, for the entry points that run on the caller's device and use its cache or lock
static int current_device(int *device) {
  const int rc = check_device();
  if (rc) return rc;
  CU(cudaGetDevice(device));
  if (*device >= 64) return fail(CTCDEC_E_INVALID, "device %d out of range", *device);
  return CTCDEC_OK;
}

// dtype -1 (probabilities, where the entry point takes them) or a CTCDEC_DTYPE_* of logits -> the prune input kind
static int input_kind(int dtype, bool probs, int *kind) {
  if ((dtype != -1 || !probs) && dtype != CTCDEC_DTYPE_F32 && dtype != CTCDEC_DTYPE_F16 && dtype != CTCDEC_DTYPE_BF16)
    return probs ? fail(CTCDEC_E_INVALID, "dtype %d is not -1 (probabilities) or one of CTCDEC_DTYPE_F32 / F16 / BF16", dtype)
                 : fail(CTCDEC_E_INVALID, "dtype %d is not one of CTCDEC_DTYPE_F32 / F16 / BF16", dtype);
  *kind = dtype == -1 ? IN_F32 : dtype == CTCDEC_DTYPE_F32 ? IN_LOGITS_F32
        : dtype == CTCDEC_DTYPE_F16 ? IN_LOGITS_F16 : IN_LOGITS_BF16;
  return CTCDEC_OK;
}

// the 256-byte aligned start of a workspace; the sizes the library asks for include the 256 bytes this may skip
static unsigned char *align256(void *p) {
  return reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(p) + 255) / 256 * 256);
}

// ---------------------------------------------------------------------------------------------------
//  per-device cache for the host-buffer entry points (stream + grow-only device buffers)
// ---------------------------------------------------------------------------------------------------
constexpr int kHostChunks = 8;  // utterance groups (streams) the host-buffer entry point pipelines over
// device buffers: the input rows, the seq_lens of ctcdec_decode_batch_host, the token / timestep rows, the small
// outputs (small_out), the workspace, the per-call tables of a streaming chunk
enum CacheSlot { kBufInput, kBufSeqLens, kBufTokens, kBufTimesteps, kBufSmall, kBufWork, kBufStreamTab, kBufSlots };
// pinned host memory: the hook scorer's exchange blocks (new-node lists, LM updates, abort flag), the small outputs,
// the staged token / timestep rows
enum PinSlot { kPinNewList, kPinUpdates, kPinAbort, kPinSmall, kPinRows, kPinSlots };
struct DevCache {
  cudaStream_t stream = nullptr;
  cudaStream_t cs[kHostChunks] = {};
  void *buf[kBufSlots] = {};
  size_t cap[kBufSlots] = {};
  void *pin[kPinSlots] = {};
  size_t pcap[kPinSlots] = {};
  cudaEvent_t beam_ev = nullptr;  // scorer path: recorded just before the persistent beam launch
};
static DevCache g_cache[64];
static std::mutex g_mu[64];  // one per device: threads driving different GPUs from one process do not serialise

static int ensure(DevCache &c, int slot, size_t bytes) {
  if (bytes <= c.cap[slot]) return CTCDEC_OK;
  if (c.buf[slot]) CU(cudaFree(c.buf[slot]));
  c.buf[slot] = nullptr;
  c.cap[slot] = 0;
  const size_t want = bytes + bytes / 8;
  CU(cudaMalloc(&c.buf[slot], want));
  c.cap[slot] = want;
  return CTCDEC_OK;
}

// optional per-kernel timing of the device entry point (bench.py roofline leg)
struct Profile {
  bool on = false;
  bool valid = false;
  bool fused_finalize = false;  // the beam kernel ran the backtrace itself: ev[2] and ev[3] bracket no kernel
  long long *timing = nullptr;  // device buffer [B][16] for per-region cycle counts (diagnostic)
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
};
static thread_local Profile g_prof;

static int ensure_pinned(DevCache &c, int slot, size_t bytes) {
  if (bytes <= c.pcap[slot]) return CTCDEC_OK;
  if (c.pin[slot]) CU(cudaFreeHost(c.pin[slot]));
  c.pin[slot] = nullptr;
  c.pcap[slot] = 0;
  CU(cudaMallocHost(&c.pin[slot], bytes + bytes / 8));
  c.pcap[slot] = bytes + bytes / 8;
  return CTCDEC_OK;
}

// Result rows on their way back to the caller.  A device-to-host copy into PAGEABLE memory goes through the driver's
// small bounce buffers and faults the caller's freshly allocated pages in from the copying thread; when the caller's
// arrays are not page-locked the rows are therefore copied compactly
// ([rows][max_len]) into pinned staging memory of the library's own and spread into the caller's [rows][row_stride]
// arrays by a few host threads.  Page-locked (or registered) destinations get the DMA directly.
static bool host_ptr_is_pinned(const void *p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost || a.type == cudaMemoryTypeManaged;
}
constexpr size_t kMaxRowStaging = (size_t)512 << 20;  // beyond this the rows go straight to the caller's pages
static void spread_rows(const int *stage_tok, const int *stage_ts, int32_t *tokens, int32_t *timesteps, size_t rows,
                        int max_len, int row_stride) {
  unsigned nt = std::thread::hardware_concurrency();
  nt = nt == 0 ? 1 : (nt > 8 ? 8 : nt);
  const size_t bytes = rows * (size_t)max_len * 8;
  if (bytes < ((size_t)1 << 20)) nt = 1;
  auto work = [&](unsigned w) {
    const size_t r0 = rows * w / nt, r1 = rows * (w + 1) / nt;
    for (size_t r = r0; r < r1; ++r) {
      memcpy(tokens + r * row_stride, stage_tok + r * max_len, (size_t)max_len * 4);
      memcpy(timesteps + r * row_stride, stage_ts + r * max_len, (size_t)max_len * 4);
    }
  };
  std::vector<std::thread> pool;
  for (unsigned w = 1; w < nt; ++w) pool.emplace_back(work, w);
  work(0);
  for (auto &th : pool) th.join();
}

// rows of `bytes` go through the staging when the caller's arrays are pageable and the staging stays small enough
static bool stage_rows(const void *tokens, const void *timesteps, size_t bytes) {
  return bytes <= kMaxRowStaging && !(host_ptr_is_pinned(tokens) && host_ptr_is_pinned(timesteps));
}

// Enqueues columns [0, max_len) of `rows` token / timestep rows of row_stride columns from the device: compactly into
// the staging ([rows][max_len] each, for spread_rows once s has finished) if stage_tok is given, else by DMA into the
// caller's arrays.
static int enqueue_rows(const int32_t *d_tok, const int32_t *d_ts, int32_t *tokens, int32_t *timesteps,
                        int32_t *stage_tok, int32_t *stage_ts, size_t rows, int max_len, int row_stride, cudaStream_t s) {
  const size_t src_pitch = (size_t)row_stride * 4, pitch = (size_t)(stage_tok ? max_len : row_stride) * 4;
  CU(cudaMemcpy2DAsync(stage_tok ? stage_tok : tokens, pitch, d_tok, src_pitch, (size_t)max_len * 4, rows,
                       cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpy2DAsync(stage_ts ? stage_ts : timesteps, pitch, d_ts, src_pitch, (size_t)max_len * 4, rows,
                       cudaMemcpyDeviceToHost, s));
  return CTCDEC_OK;
}

// The [B, K] scores and lens and the [B] n_results and flags of a decode.  In the cache (slot kBufSmall, and its pinned
// staging kPinSmall) they share one block, laid out by small_out, with flags = n_results + B.
struct SmallOut { float *scores; int32_t *lens, *n_results, *flags; };
static size_t small_bytes(int B, int K) { return (size_t)B * K * 4 * 2 + (size_t)B * 8 + 1024; }
static SmallOut small_out(void *p, int B, int K) {
  const size_t n_bk = (size_t)B * K;
  SmallOut o;
  o.scores = static_cast<float *>(p);
  o.lens = reinterpret_cast<int32_t *>(static_cast<char *>(p) + al256(n_bk * 4));
  o.n_results = reinterpret_cast<int32_t *>(static_cast<char *>(p) + 2 * al256(n_bk * 4));
  o.flags = o.n_results + B;
  return o;
}

// Enqueues the copy of utterances [b0, b0 + nb) of the small outputs d into the pinned staging h (pinned: a copy into
// pageable memory would block the calling thread until the work before it has finished).
static int read_small(const SmallOut &h, const SmallOut &d, int K, int b0, int nb, cudaStream_t s) {
  const size_t ko = (size_t)b0 * K, bytes = (size_t)nb * K * 4;
  CU(cudaMemcpyAsync(h.scores + ko, d.scores + ko, bytes, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(h.lens + ko, d.lens + ko, bytes, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(h.n_results + b0, d.n_results + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpyAsync(h.flags + b0, d.flags + b0, (size_t)nb * 4, cudaMemcpyDeviceToHost, s));
  return CTCDEC_OK;
}

// Rows p < n_results[b] of the staged scores and lens into the caller's [B, K] arrays, for the utterances in `mask`
// (all if NULL).  The other rows stay as the caller left them: the finalize kernel does not write them, and the device
// buffers are reused between calls (reference binding.cpp:79-99 writes results.size() rows).
static void copy_result_rows(const SmallOut &h, int B, int K, const uint8_t *mask, float *scores, int32_t *lens) {
  for (int b = 0; b < B; ++b) {
    if (mask && !mask[b]) continue;
    const size_t nr = (size_t)std::max(0, std::min(h.n_results[b], K));
    memcpy(scores + (size_t)b * K, h.scores + (size_t)b * K, nr * 4);
    memcpy(lens + (size_t)b * K, h.lens + (size_t)b * K, nr * 4);
  }
}

// The longest result of utterances [b0, b0 + nb) (those in `mask`, if given).  Only rows p < n_results[b] count: the
// lens of the others are whatever the caller's arrays held (the reference's Python zero-fills out_seq_len).
static int max_result_len(const SmallOut &h, int K, int b0, int nb, const uint8_t *mask) {
  int max_len = 0;
  for (int b = b0; b < b0 + nb; ++b)
    if (!mask || mask[b])
      for (int p = 0; p < h.n_results[b] && p < K; ++p) max_len = std::max(max_len, h.lens[(size_t)b * K + p]);
  return max_len;
}

// completion of device-path work (ctcdec_decode_stream_device / ctcdec_stream_committed_device) on a state; one event
// per call, shared by the call's states
struct StreamEvent {
  cudaEvent_t ev = nullptr;
  ~StreamEvent() { if (ev) cudaEventDestroy(ev); }
};

// Frames of room a streaming arena has beyond what its nodes need: at creation, and after a compaction (capacity
// max(1 + beam x 256, kept + beam x 256) nodes)
constexpr int kArenaSlackFrames = 256;

// streaming state object
struct StreamState {
  std::shared_ptr<StreamEvent> last;  // the last device-path call that used this state (or null)
  ctcdec_config cfg;
  int device;
  Node *arena;
  int arena_cap;
  int *state;
  int frames;
  // node accounting: the arena holds at most node_base + beam x since nodes (node_base: nodes kept by the last
  // compaction, 1 before any; since: frames consumed after it)
  long long node_base = 1, since = 0;
  // scorer path (ctcdec_state_create_lm): the borrowed scorer (reference DecoderState::ext_scorer,
  // ctc_beam_search_decoder.cpp:31), per-node LM terms / dictionary states, the host mirror of the trie
  HostScorer *sc = nullptr;
  float *lm_arena = nullptr;
  int *dstate = nullptr;
  float *lm_row = nullptr;  // character-based model: [arena_cap][V] per-node rows of LM terms
  // ARPA scorer: order - 1, and lm_arena holds [arena_cap] terms, then [arena_cap][order - 1] LM word ids per node
  int lm_hist_n = 0;
  TrieMirror mirror;
};

static int ensure_dict_on_device(HostScorer *sc, int device) {
  if (sc->d_next && sc->device != device) {
    cudaSetDevice(sc->device); cudaFree(sc->d_next); cudaFree(sc->d_mask); sc->d_next = nullptr; cudaSetDevice(device);
  }
  if (!sc->d_next) {
    CU(cudaMalloc(&sc->d_next, sc->dict.packed.size() * 4));
    CU(cudaMalloc(&sc->d_mask, sc->dict.mask.size() * 4));
    CU(cudaMemcpy(sc->d_next, sc->dict.packed.data(), sc->dict.packed.size() * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(sc->d_mask, sc->dict.mask.data(), sc->dict.mask.size() * 4, cudaMemcpyHostToDevice));
    sc->device = device;
  }
  return CTCDEC_OK;
}

// The tables of an n-gram scorer (ARPA or KenLM binary) and the kernel's word-id arrays in device memory, uploaded once
// per device.
static int ensure_ngram_on_device(HostScorer *sc, int device) {
  if (sc->d_ngram && sc->ngram_device != device) {
    cudaSetDevice(sc->ngram_device); cudaFree(sc->d_ngram); sc->d_ngram = nullptr; cudaSetDevice(device);
  }
  if (sc->d_ngram) return CTCDEC_OK;
  const NgramModel &m = *sc->ngram;
  std::vector<std::pair<const void *, size_t>> parts;
  parts.emplace_back(m.uni_prob.data(), m.uni_prob.size() * 4);
  parts.emplace_back(m.uni_backoff.data(), m.uni_backoff.size() * 4);
  if (m.layout == kNgramKenlmTrie) {  // a KenLM trie file's search region, byte for byte, and its order descriptors
    parts.emplace_back(m.trie_bits.data(), m.trie_bits.size() * 8);
    parts.emplace_back(m.trie_orders.data(), m.trie_orders.size() * sizeof(NgramTrieOrder));
  } else {
    for (int n = 2; n <= m.order; ++n) {
      if (m.layout == kNgramKenlmProbing)  // a KenLM probing file's tables, byte for byte
        parts.emplace_back(m.probing[n - 1].data(), m.probing[n - 1].size() * 8);
      else
        parts.emplace_back(m.tables[n - 1].data(), m.tables[n - 1].size() * sizeof(NgramEntry));
    }
  }
  parts.emplace_back(sc->word_of_state.data(), sc->word_of_state.size() * 4);
  parts.emplace_back(sc->label_word.data(), sc->label_word.size() * 4);
  parts.emplace_back(m.label_bytes.data(), m.label_bytes.size());
  parts.emplace_back(m.label_off.data(), m.label_off.size() * 4);
  parts.emplace_back(m.word_bytes.data(), m.word_bytes.size());
  parts.emplace_back(m.words.data(), m.words.size() * sizeof(NgramWordSlot));
  std::vector<size_t> off;
  size_t total = 0;
  for (const auto &pt : parts) { off.push_back(total); total += al256(pt.second); }
  std::vector<unsigned char> staged(total);
  for (size_t i = 0; i < parts.size(); ++i)
    if (parts[i].second) memcpy(staged.data() + off[i], parts[i].first, parts[i].second);
  unsigned char *d = nullptr;
  CU(cudaMalloc(&d, total));
  const cudaError_t e = cudaMemcpy(d, staged.data(), total, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { cudaFree(d); return fail(CTCDEC_E_CUDA, "n-gram tables upload: %s", cudaGetErrorString(e)); }
  NgramView v = m.view();
  size_t i = 0;
  v.uni_prob = reinterpret_cast<const float *>(d + off[i++]);
  v.uni_backoff = reinterpret_cast<const float *>(d + off[i++]);
  if (m.layout == kNgramKenlmTrie) {
    v.trie.bits = reinterpret_cast<const uint64_t *>(d + off[i++]);
    v.trie.orders = reinterpret_cast<const NgramTrieOrder *>(d + off[i++]);
  } else {
    for (int n = 2; n <= m.order; ++n) {
      if (m.layout == kNgramKenlmProbing) v.probe[n - 1] = reinterpret_cast<const uint32_t *>(d + off[i++]);
      else v.table[n - 1] = reinterpret_cast<const NgramEntry *>(d + off[i++]);
    }
  }
  sc->d_word_of_state = reinterpret_cast<int *>(d + off[i++]);
  sc->d_label_word = reinterpret_cast<int *>(d + off[i++]);
  NgramFront f = m.front();
  f.label_bytes = d + off[i++];
  f.label_off = reinterpret_cast<const int32_t *>(d + off[i++]);
  f.word_bytes = d + off[i++];
  f.words = reinterpret_cast<const NgramWordSlot *>(d + off[i++]);
  sc->d_view = v;
  sc->d_front = f;
  sc->d_ngram = d;
  sc->ngram_device = device;
  return CTCDEC_OK;
}

// Enqueues the read-out of an ARPA scorer's [B, K] result rows (row_stride columns each) on s; the scorer's tables must
// be on the current device.  alpha and beta are the scorer's values now, or, for a sweep, the device table ab [P][2]
// with pair_B utterances per pair.
// For a decode over several models, slots / slot_of are the device tables of the LM slots and of each utterance's slot
// (sc is then unused).
static int launch_readout(const HostScorer *sc, const int32_t *tokens, const int32_t *lens, const int32_t *n_results,
                          float *scores, int B, int K, int row_stride, cudaStream_t s, const double *ab = nullptr,
                          int pair_B = 0, const LmSlot *slots = nullptr, const unsigned char *slot_of = nullptr) {
  const long long rows = (long long)B * K;
  if (rows == 0) return CTCDEC_OK;
  const unsigned grid = (unsigned)((rows + kReadoutThreads - 1) / kReadoutThreads);
  if (slots)
    lm_readout_kernel<kReadSlots><<<grid, kReadoutThreads, 0, s>>>(NgramView(), NgramFront(), 0.0, 0.0, nullptr, 1,
                                                                   slots, slot_of, tokens, lens, n_results, scores, B,
                                                                   K, row_stride);
  else if (ab)
    lm_readout_kernel<kReadSweep><<<grid, kReadoutThreads, 0, s>>>(sc->d_view, sc->d_front, 0.0, 0.0, ab, pair_B,
                                                                   nullptr, nullptr, tokens, lens, n_results, scores,
                                                                   B, K, row_stride);
  else
    lm_readout_kernel<kReadOne><<<grid, kReadoutThreads, 0, s>>>(sc->d_view, sc->d_front, sc->alpha, sc->beta, nullptr,
                                                                 1, nullptr, nullptr, tokens, lens, n_results, scores,
                                                                 B, K, row_stride);
  CU(cudaGetLastError());
  return CTCDEC_OK;
}

// Host side of the per-frame handshake of a persistent scorer-path launch (beam_program.cuh, "persistent mode"):
// workers own every nt-th utterance (and one hook cache each, so nothing is locked); utterance b is answered
// need[b] times.  Returns non-zero when the kernel stopped making progress (the caller raises the abort flag).
struct HandshakeStats { long long hooks = 0, created = 0; unsigned workers = 0; };
static int serve_handshakes(HostScorer *sc, int B, int K, const int *need, TrieMirror *const *mirrors,
                            int *h_newlist, int *h_upd, HandshakeStats *stats) {
  int nls = 0, ups = 0;
  exchange_strides(K, exchange_row_len(*sc), &nls, &ups);
  unsigned nt = std::thread::hardware_concurrency();
  if (const char *e = getenv("CTCDEC_LM_THREADS")) nt = (unsigned)atoi(e);
  // the frame is bound by the PCIe round trip of its flags, not by the workers, and many busy-polling workers starve
  // each other's hyper-threads: at most 8
  nt = nt == 0 ? 1 : (nt > 8 ? 8 : nt);
  if ((unsigned)B < nt) nt = (unsigned)B;
  if (sc->cond_caches.size() < nt) sc->cond_caches.resize(nt);
  std::atomic<int> failed{0};
  std::atomic<long long> n_hook{0}, n_new{0};
  auto worker = [&](unsigned w) {
    std::vector<int> scratch;
    HostScorer::CondCache &cache = sc->cond_caches[w];
    int remaining = 0;
    for (int b = (int)w; b < B; b += (int)nt) remaining += need[b] > 0 ? 1 : 0;
    std::vector<int> served(B, 0);
    auto last_progress = std::chrono::steady_clock::now();
    long long hooks = 0, created = 0;
    unsigned idle = 0;
    while (remaining > 0 && !failed.load(std::memory_order_relaxed)) {
      bool progress = false;
      for (int b = (int)w; b < B; b += (int)nt) {
        if (served[b] >= need[b]) continue;
        int *nl = h_newlist + (size_t)b * nls, *up = h_upd + (size_t)b * ups;
        const int d = reinterpret_cast<std::atomic<int> *>(&nl[1])->load(std::memory_order_acquire);  // "done"
        if (d <= served[b]) continue;
        hooks += lm_after_frame(*sc, cache, *mirrors[b], nl, up, scratch);
        created += nl[0];
        reinterpret_cast<std::atomic<int> *>(&up[0])->store(d, std::memory_order_release);            // "go"
        served[b] = d;
        if (d >= need[b]) --remaining;
        progress = true;
      }
      if (!progress) {
#if defined(__x86_64__) || defined(__i386__)
        __builtin_ia32_pause();  // (a spinning worker must not starve the hyper-thread that runs another worker's hooks)
#endif
      }
      if (progress) { idle = 0; last_progress = std::chrono::steady_clock::now(); }
      else if ((++idle & 0xFFFF) == 0 &&
               std::chrono::duration<double>(std::chrono::steady_clock::now() - last_progress).count() > 8.0)
        failed.store(1);  // the kernel stopped making progress (fault or lost launch): stop waiting
    }
    n_hook += hooks; n_new += created;
  };
  std::vector<std::thread> pool;
  for (unsigned w = 1; w < nt; ++w) pool.emplace_back(worker, w);
  worker(0);
  for (auto &th : pool) th.join();
  if (stats) { stats->hooks = n_hook; stats->created = n_new; stats->workers = nt; }
  return failed.load();
}

// the caller's outputs of a decode (device memory)
struct DecodeOut {
  int32_t *tokens, *timesteps;  // [B, K, out_T]
  float *scores;                // [B, K]
  int32_t *lens;                // [B, K]
  int32_t *n_results, *flags;   // [B]
};

// The kernel parameters every decode shares: the pruned rows in the plan's workspace ws, the outputs and the knobs.
// The caller adds the arenas and states (one flat region, or the per-stream tables), tile_frames, fresh and a scorer.
static BeamParams beam_params(const ctcdec_config &cfg, const Plan &pl, const unsigned char *ws, const int *seq_lens,
                              int T, const DecodeOut &o, int out_T) {
  BeamParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.lp = reinterpret_cast<const float *>(ws + pl.off_lp);
  bp.idx = pl.sorted ? reinterpret_cast<const uint16_t *>(ws + pl.off_idx) : nullptr;
  bp.seq_lens = seq_lens; bp.T = T; bp.V = cfg.vocab_size; bp.NP = pl.NP; bp.K = cfg.beam_size; bp.blank = cfg.blank_id;
  bp.out_tokens = o.tokens; bp.out_timesteps = o.timesteps; bp.out_scores = o.scores; bp.out_lens = o.lens;
  bp.n_results = o.n_results; bp.out_T = out_T; bp.flags = o.flags;
  bp.timing = g_prof.timing;
  bp.force_fallback = getenv("CTCDEC_FORCE_FALLBACK") ? 1 : 0;  // test knob
  return bp;
}

// the flat arenas and states of an offline decode, in the plan's workspace ws
static void flat_arenas(BeamParams &bp, const Plan &pl, unsigned char *ws) {
  bp.arena = reinterpret_cast<Node *>(ws + pl.off_arena); bp.arena_stride = pl.arena_stride;
  bp.state = reinterpret_cast<int *>(ws + pl.off_state); bp.state_stride = pl.state_stride;
  bp.arena_cap = (int)pl.arena_stride;
}

// The scorer's model and weights as an LM slot (beam_core.cuh): its dictionary must be on the device, and for an n-gram
// scorer its tables too.
static LmSlot scorer_slot(const HostScorer &sc) {
  LmSlot m;
  m.dict_next = sc.d_next; m.dict_mask = sc.d_mask; m.dict_start = sc.dict.start; m.beta = sc.beta;
  m.lm_alpha = 0.0; m.word_of_state = nullptr; m.label_word = nullptr; m.lm_hist_n = 0;
  if (sc.ngram) {
    m.lm_alpha = sc.alpha; m.ngram = sc.d_view; m.front = sc.d_front;
    m.word_of_state = sc.d_word_of_state; m.label_word = sc.d_label_word; m.lm_hist_n = sc.max_order - 1;
  }
  return m;
}

// The LM slots of S scorers (each with its alpha and beta as they are now) into the device table slots, and the slot
// index of each of B utterances or streams into slot_of, enqueued on s from kernel launch parameters.
static int upload_slots(HostScorer *const *scs, int S, const unsigned char *index, int B, LmSlot *slots,
                        unsigned char *slot_of, cudaStream_t s) {
  LmSlotArgs a;
  memset(&a, 0, sizeof(a));
  a.tab = slots; a.S = S;
  for (int i = 0; i < S; ++i) a.slot[i] = scorer_slot(*scs[i]);
  lm_slots_kernel<<<1, kMaxLmSlots, 0, s>>>(a);
  CU(cudaGetLastError());
  for (int b0 = 0; b0 < B; b0 += kSlotIndexPerLaunch) {
    SlotIndexArgs x;
    x.tab = slot_of; x.b0 = b0; x.n = std::min(kSlotIndexPerLaunch, B - b0);
    memcpy(x.index, index + b0, (size_t)x.n);
    lm_slot_index_kernel<<<1, 256, 0, s>>>(x);
    CU(cudaGetLastError());
  }
  return CTCDEC_OK;
}

// The scorer's part of the kernel parameters (its dictionary must be on the device): the dictionary and the word
// bonus, and for an n-gram scorer, whose tables must be on the device too, the model the beam kernel scores with.
static void attach_scorer(BeamParams &bp, const HostScorer &sc) {
  static_cast<LmSlot &>(bp) = scorer_slot(sc);
  bp.dict_wc = sc.dict.wc; bp.space_id = sc.space_id; bp.lm_char = sc.is_character_based ? 1 : 0;
  bp.lm_dev = sc.ngram ? 1 : 0;
}

// The pinned exchange blocks of a hook scorer's handshake (beam_core.cuh) for B utterances, in the cache c, and the
// kernel parameters that point at them: headers cleared, abort flag down, and for a character-based model the root's
// row of LM terms in the update block of each utterance in `at_root` (all if NULL), the first entry its CTA picks up.
static int prepare_exchange(DevCache &c, HostScorer &sc, int B, const uint8_t *at_root, BeamParams &bp) {
  int nls = 0, ups = 0;
  exchange_strides(bp.K, exchange_row_len(sc), &nls, &ups);
  int rc = ensure_pinned(c, kPinNewList, (size_t)B * nls * 4);
  if (rc || (rc = ensure_pinned(c, kPinUpdates, (size_t)B * ups * 4)) || (rc = ensure_pinned(c, kPinAbort, 256))) return rc;
  int *h_newlist = (int *)c.pin[kPinNewList], *h_upd = (int *)c.pin[kPinUpdates];
  for (int b = 0; b < B; ++b) { memset(h_newlist + (size_t)b * nls, 0, 16); memset(h_upd + (size_t)b * ups, 0, 8); }
  if (sc.is_character_based) {  // (computed once, copied to the others)
    const int *root = nullptr;
    std::vector<int> scratch;
    for (int b = 0; b < B; ++b) {
      if (at_root && !at_root[b]) continue;
      int *up = h_upd + (size_t)b * ups;
      if (root) memcpy(up, root, (size_t)(3 + bp.V) * 4);
      else { lm_char_root_entry(sc, sc.cond_caches[0], up, scratch); root = up; }
    }
  }
  *static_cast<int *>(c.pin[kPinAbort]) = 0;
  // The per-frame exchange with the host goes through pinned, device-mapped host memory (unified addressing): the
  // kernel reads the few LM updates and writes the new-node list straight over PCIe, with no memcpy calls.
  bp.newlist = h_newlist; bp.lm_upd = h_upd; bp.lm_nl_stride = nls; bp.lm_up_stride = ups;
  return CTCDEC_OK;
}

// One persistent launch of the beam kernel with a hook scorer (after prepare_exchange), served by serve_handshakes until
// utterance b has been answered answers[b] frames, and synchronised.  After each frame a CTA publishes its new nodes in
// mapped host memory, raises its done flag and polls its go flag; CTAs never wait on each other, so the scheme needs no
// co-residency, and a kernel-side deadline and the abort flag bound every wait.  `what` names the path in errors.
static int run_handshake(const BeamParams &bp_in, const Plan &pl, int B, HostScorer *sc, DevCache &c, const int *answers,
                         TrieMirror *const *mirrors, HandshakeStats *stats, const char *what, cudaStream_t s) {
  BeamParams bp = bp_in;
  auto *const hs_abort = static_cast<std::atomic<int> *>(c.pin[kPinAbort]);
  bp.lm_persistent = 1; bp.hs_abort = static_cast<int *>(c.pin[kPinAbort]);
  if (!c.beam_ev) CU(cudaEventCreateWithFlags(&c.beam_ev, cudaEventDisableTiming));
  CU(cudaEventRecord(c.beam_ev, s));
  const int rc = launch_beam(bp, pl, B, s);
  if (rc) return rc;
  // the handshake gives up after 8 s without progress: start its clock once the work queued on s before the beam
  // kernel (the caller's, on a stream of the caller's) has finished
  const cudaError_t ew = cudaEventSynchronize(c.beam_ev);
  if (ew != cudaSuccess) {
    hs_abort->store(1, std::memory_order_release);
    return fail(CTCDEC_E_CUDA, "work queued before the beam kernel (%s): %s", what, cudaGetErrorString(ew));
  }
  const int failed = serve_handshakes(sc, B, bp.K, answers, mirrors, (int *)c.pin[kPinNewList],
                                      (int *)c.pin[kPinUpdates], stats);
  if (failed) hs_abort->store(1, std::memory_order_release);
  const cudaError_t e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return fail(CTCDEC_E_CUDA, "beam kernel (%s): %s", what, cudaGetErrorString(e));
  if (failed) return fail(CTCDEC_E_CUDA, "beam kernel (%s) stopped answering the per-frame handshake", what);
  return CTCDEC_OK;
}

// the caller's workspace, 256-byte aligned, which must hold `need` bytes (need includes the 256 the alignment may skip)
static int workspace_start(void *workspace, size_t workspace_bytes, size_t need, unsigned char **ws) {
  if (!workspace || workspace_bytes < need)
    return fail(CTCDEC_E_WORKSPACE, "workspace of %zu bytes given, %zu needed", workspace_bytes, need);
  *ws = align256(workspace);
  return CTCDEC_OK;
}

}  // namespace ctc

using namespace ctc;

extern "C" {

const char *ctcdec_version(void) { return "ctcdecode_b200 0.1 (sm_90a)"; }
const char *ctcdec_last_error(void) { return g_err; }

int ctcdec_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  int ok = 0;
  for (int d = 0; d < n; ++d)
    if (is_sm90(d)) ++ok;
  return ok;
}

int ctcdec_workspace_bytes(const ctcdec_config *cfg, int B, int T, size_t *bytes) {
  Plan pl;
  int rc = make_plan(cfg, B, T, &pl);
  if (rc) return rc;
  if (!bytes) return fail(CTCDEC_E_INVALID, "bytes is NULL");
  *bytes = pl.total + 256;
  return CTCDEC_OK;
}

static int decode_device_impl(const ctcdec_config *cfg, const PruneInput &in, const int32_t *seq_lens, int B, int T,
                              int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                              int32_t *n_results, int32_t *flags, void *workspace, size_t workspace_bytes,
                              void *stream) {
  Plan pl;
  int rc = make_plan(cfg, B, T, &pl);
  if (rc) return rc;
  if ((rc = check_device())) return rc;
  if (B == 0) return CTCDEC_OK;
  if (!in.data && T > 0) return fail(CTCDEC_E_INVALID, "probs is NULL");
  if (!tokens || !timesteps || !scores || !lens) return fail(CTCDEC_E_INVALID, "an output pointer is NULL");
  unsigned char *ws = nullptr;
  if ((rc = workspace_start(workspace, workspace_bytes, pl.total + 256, &ws))) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (!flags || !n_results) return fail(CTCDEC_E_INVALID, "n_results and flags device buffers are required by the device entry point");
  CU(cudaMemsetAsync(flags, 0, (size_t)B * 4, s));  // (OR-accumulated by the prune and finalize kernels)

  const bool prof = g_prof.on;
  if (prof) {
    for (int i = 0; i < 4; ++i)
      if (!g_prof.ev[i]) CU(cudaEventCreate(&g_prof.ev[i]));
    g_prof.valid = false;
    CU(cudaEventRecord(g_prof.ev[0], s));
  }
  if ((rc = launch_prune(cfg, pl, in, seq_lens, B, T, ws, flags, s))) return rc;
  if (prof) CU(cudaEventRecord(g_prof.ev[1], s));

  BeamParams bp = beam_params(*cfg, pl, ws, seq_lens, T, DecodeOut{tokens, timesteps, scores, lens, n_results, flags}, T);
  flat_arenas(bp, pl, ws);
  bp.tile_frames = pl.F; bp.fresh = 1;
  bp.backtrace = cta_backtrace(pl.sorted, bp.K, pl.L);
  if ((rc = launch_beam(bp, pl, B, s))) return rc;
  if (prof) CU(cudaEventRecord(g_prof.ev[2], s));
  if (!bp.backtrace && (rc = launch_finalize(bp, B, s))) return rc;
  if (prof) {
    CU(cudaEventRecord(g_prof.ev[3], s));
    g_prof.valid = true;
    g_prof.fused_finalize = bp.backtrace != 0;
  }
  return CTCDEC_OK;
}

int ctcdec_decode_batch_device(const ctcdec_config *cfg, const float *probs, const int32_t *seq_lens, int B, int T,
                               int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                               int32_t *n_results, int32_t *flags, void *workspace, size_t workspace_bytes,
                               void *stream) {
  return decode_device_impl(cfg, PruneInput{probs, IN_F32, nullptr}, seq_lens, B, T, tokens, timesteps, scores, lens,
                            n_results, flags, workspace, workspace_bytes, stream);
}

int ctcdec_decode_batch_device_logits(const ctcdec_config *cfg, const void *logits, int dtype, const int32_t *seq_lens,
                                      int B, int T, int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                      int32_t *n_results, int32_t *flags, float *log_probs_out, void *workspace,
                                      size_t workspace_bytes, void *stream) {
  int kind = 0;
  const int rc = input_kind(dtype, false, &kind);
  if (rc) return rc;
  return decode_device_impl(cfg, PruneInput{logits, kind, log_probs_out}, seq_lens, B, T, tokens, timesteps, scores,
                            lens, n_results, flags, workspace, workspace_bytes, stream);
}

int ctcdec_pack_results_device(const int32_t *tokens, const int32_t *timesteps, const int32_t *lens,
                               const int32_t *n_results, int B, int K, int T, int64_t *offsets,
                               int32_t *packed_tokens, int32_t *packed_timesteps, size_t capacity, void *stream) {
  if (B < 0 || K < 1 || T < 0) return fail(CTCDEC_E_INVALID, "bad shape B=%d beam=%d T=%d", B, K, T);
  if (!tokens || !timesteps || !lens || !n_results || !offsets || (capacity > 0 && (!packed_tokens || !packed_timesteps)))
    return fail(CTCDEC_E_INVALID, "NULL argument");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  static_assert(sizeof(long long) == sizeof(int64_t), "offsets are 64-bit");
  pack_offsets_kernel<<<1, 1024, 0, s>>>(lens, n_results, B, K, reinterpret_cast<long long *>(offsets));
  CU(cudaGetLastError());
  const long long rows = (long long)B * K;
  if (rows > 0 && capacity > 0) {
    const int grid = (int)std::min<long long>((rows + 7) / 8, kNumSMs * 8);
    pack_rows_kernel<<<grid, 256, 0, s>>>(tokens, timesteps, lens, n_results, B, K, T,
                                          reinterpret_cast<const long long *>(offsets), packed_tokens,
                                          packed_timesteps, (long long)capacity);
    CU(cudaGetLastError());
  }
  return CTCDEC_OK;
}

int ctcdec_profile_enable(int on) {
  g_prof.on = on != 0;
  g_prof.valid = false;
  return CTCDEC_OK;
}

int ctcdec_profile_region_cycles(void *device_buffer) {
  g_prof.timing = static_cast<long long *>(device_buffer);
  return CTCDEC_OK;
}

int ctcdec_profile_read(float *ms) {
  if (!ms) return fail(CTCDEC_E_INVALID, "ms is NULL");
  if (!g_prof.valid) return fail(CTCDEC_E_INVALID, "no profiled decode on this thread");
  CU(cudaEventSynchronize(g_prof.ev[3]));
  for (int i = 0; i < 3; ++i) CU(cudaEventElapsedTime(&ms[i], g_prof.ev[i], g_prof.ev[i + 1]));
  if (g_prof.fused_finalize) ms[2] = 0.0f;
  return CTCDEC_OK;
}

int ctcdec_decode_batch_host(const ctcdec_config *cfg, const float *probs, const int32_t *seq_lens, int B, int T,
                             int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens, int32_t *n_results,
                             int32_t *flags, int device) {
  Plan pl;
  int rc = make_plan(cfg, B, T, &pl);
  if (rc || (rc = use_device(device))) return rc;
  if (B == 0) return CTCDEC_OK;
  std::lock_guard<std::mutex> lock(g_mu[device]);
  DevCache &c = g_cache[device];
  const int V = cfg->vocab_size, K = cfg->beam_size;
  // The batch is cut into up to kHostChunks groups of utterances, each with its own stream: upload, kernels and
  // download of different groups overlap (an utterance is T serial frames whatever the batch size, so a group's
  // kernels take as long as the whole batch's would; only the PCIe legs of the first / last group stay exposed,
  // and for batches of several waves the downloads hide under the next group's kernels).
  int chunk = std::max(64, (B + kHostChunks - 1) / kHostChunks);
  if (const char *e = getenv("CTCDEC_HOST_CHUNK")) chunk = std::max(1, atoi(e));  // tuning knob: utterances per group
  const int C = std::min(kHostChunks, (B + chunk - 1) / chunk);
  chunk = (B + C - 1) / C;
  for (int i = 0; i < C; ++i)
    if (!c.cs[i]) CU(cudaStreamCreateWithFlags(&c.cs[i], cudaStreamNonBlocking));
  struct InFlight { InFlight(int n) { g_batch_in_flight = n; } ~InFlight() { g_batch_in_flight = 0; } } in_flight(B);
  Plan plc;
  if ((rc = make_plan(cfg, chunk, T, &plc))) return rc;
  const size_t ws_stride = al256(plc.total + 512);
  const size_t n_probs = (size_t)B * T * V, n_out = (size_t)B * K * T;
  if ((rc = ensure(c, kBufInput, n_probs * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufSeqLens, (size_t)B * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufTokens, n_out * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufTimesteps, n_out * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufSmall, small_bytes(B, K)))) return rc;
  if ((rc = ensure(c, kBufWork, ws_stride * C))) return rc;
  if ((rc = ensure_pinned(c, kPinSmall, small_bytes(B, K)))) return rc;
  float *d_probs = (float *)c.buf[kBufInput];
  int *d_lens_in = seq_lens ? (int *)c.buf[kBufSeqLens] : nullptr;
  int *d_tok = (int *)c.buf[kBufTokens], *d_ts = (int *)c.buf[kBufTimesteps];
  const SmallOut d = small_out(c.buf[kBufSmall], B, K), h = small_out(c.pin[kPinSmall], B, K);
  const bool staged = n_out > 0 && stage_rows(tokens, timesteps, n_out * 8);
  if (staged && (rc = ensure_pinned(c, kPinRows, n_out * 8))) return rc;
  int *const stage_tok = staged ? static_cast<int *>(c.pin[kPinRows]) : nullptr;
  int *const stage_ts = staged ? stage_tok + n_out : nullptr;
  int chunk_len[kHostChunks] = {};
  for (int i = 0; i < C; ++i) {
    const int b0 = i * chunk, nb = std::min(chunk, B - b0);
    cudaStream_t s = c.cs[i];
    const size_t po = (size_t)b0 * T * V, oo = (size_t)b0 * K * T, ko = (size_t)b0 * K;
    if (n_probs) CU(cudaMemcpyAsync(d_probs + po, probs + po, (size_t)nb * T * V * 4, cudaMemcpyHostToDevice, s));
    if (seq_lens) CU(cudaMemcpyAsync(d_lens_in + b0, seq_lens + b0, (size_t)nb * 4, cudaMemcpyHostToDevice, s));
    rc = ctcdec_decode_batch_device(cfg, d_probs + po, seq_lens ? d_lens_in + b0 : nullptr, nb, T, d_tok + oo, d_ts + oo,
                                    d.scores + ko, d.lens + ko, d.n_results + b0, d.flags + b0,
                                    (char *)c.buf[kBufWork] + ws_stride * i, ws_stride, s);
    // small results first: lens tell how many columns of the big tensors carry data
    if (rc || (rc = read_small(h, d, K, b0, nb, s))) return rc;
  }
  for (int i = 0; i < C; ++i) {
    const int b0 = i * chunk, nb = std::min(chunk, B - b0);
    cudaStream_t s = c.cs[i];
    CU(cudaStreamSynchronize(s));
    chunk_len[i] = std::min(max_result_len(h, K, b0, nb, nullptr), T);
    const size_t oo = (size_t)b0 * K * T;
    if (chunk_len[i] > 0 && (rc = enqueue_rows(d_tok + oo, d_ts + oo, tokens + oo, timesteps + oo,
                                               staged ? stage_tok + oo : nullptr, staged ? stage_ts + oo : nullptr,
                                               (size_t)nb * K, chunk_len[i], T, s)))
      return rc;
  }
  copy_result_rows(h, B, K, nullptr, scores, lens);
  for (int i = 0; i < C; ++i) {
    CU(cudaStreamSynchronize(c.cs[i]));
    if (staged && chunk_len[i] > 0) {  // (the later groups' rows are still on their way meanwhile)
      const int b0 = i * chunk, nb = std::min(chunk, B - b0);
      const size_t oo = (size_t)b0 * K * T;
      spread_rows(stage_tok + oo, stage_ts + oo, tokens + oo, timesteps + oo, (size_t)nb * K, chunk_len[i], T);
    }
  }
  if (n_results) memcpy(n_results, h.n_results, (size_t)B * 4);
  if (flags) memcpy(flags, h.flags, (size_t)B * 4);
  return check_error_flags(h.flags, B);
}

int ctcdec_decode_batch_host_multi(const ctcdec_config *cfg, const float *probs, const int32_t *seq_lens, int B, int T,
                                   int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                   int32_t *n_results, int32_t *flags, const int *devices, int n_devices) {
  if (!cfg) return fail(CTCDEC_E_INVALID, "cfg is NULL");
  if (B < 0 || T < 0) return fail(CTCDEC_E_INVALID, "negative batch (%d) or time (%d)", B, T);
  std::vector<int> devs;
  if (devices && n_devices > 0) {
    devs.assign(devices, devices + n_devices);
  } else {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) n = 0;
    for (int d = 0; d < n && d < 64; ++d)
      if (is_sm90(d)) devs.push_back(d);
  }
  if (devs.empty()) return fail(CTCDEC_E_NO_DEVICE, "no usable CUDA device (this library has no CPU fallback)");
  const int nd = (int)std::min<size_t>(devs.size(), (size_t)std::max(B, 1));
  if (nd == 1)
    return ctcdec_decode_batch_host(cfg, probs, seq_lens, B, T, tokens, timesteps, scores, lens, n_results, flags, devs[0]);
  const int V = cfg->vocab_size, K = cfg->beam_size;
  std::vector<int> rcs(nd, CTCDEC_OK);
  std::vector<std::string> errs(nd);
  std::vector<std::thread> pool;
  const int per = (B + nd - 1) / nd;
  for (int i = 0; i < nd; ++i) {
    const int b0 = std::min(B, i * per), nb = std::min(per, B - b0);
    if (nb <= 0) continue;
    pool.emplace_back([&, i, b0, nb]() {
      const size_t po = (size_t)b0 * T * V, oo = (size_t)b0 * K * T, ko = (size_t)b0 * K;
      rcs[i] = ctcdec_decode_batch_host(cfg, probs ? probs + po : nullptr, seq_lens ? seq_lens + b0 : nullptr, nb, T,
                                        tokens + oo, timesteps + oo, scores + ko, lens + ko,
                                        n_results ? n_results + b0 : nullptr, flags ? flags + b0 : nullptr, devs[i]);
      if (rcs[i]) errs[i] = g_err;  // (the message lives in the worker's thread-local buffer)
    });
  }
  for (auto &th : pool) th.join();
  for (int i = 0; i < nd; ++i)
    if (rcs[i]) return fail(rcs[i], "device %d: %s", devs[i], errs[i].c_str());
  return CTCDEC_OK;
}

// ---------------------------------------------------------------------------------------------------
//  streaming
// ---------------------------------------------------------------------------------------------------
static int state_init_device(StreamState *st) {
  // the root-only beam (reference ctc_beam_search_decoder.cpp:42-44), in the layout of beam_core.cuh
  const int K = st->cfg.beam_size, KP2 = 2 * kp_of(K);
  const long long n = state_ints(K);
  std::unique_ptr<int[]> h(new int[n]);
  for (long long i = 0; i < n; ++i) h[i] = 0;
  h[0] = 1; h[1] = 1; h[2] = 0; h[3] = 0;
  int *s = h.get() + kStateHeader;
  const float ninf = -FLT_MAX, zero = 0.0f;
  for (int j = 0; j < K; ++j) {
    s[j] = 0; s[K + j] = -1; s[2 * K + j] = 0;
    memcpy(&s[3 * K + j], j == 0 ? &zero : &ninf, 4);
    memcpy(&s[4 * K + j], &ninf, 4);
    memcpy(&s[5 * K + j], j == 0 ? &zero : &ninf, 4);
    memcpy(&s[6 * K + j], &ninf, 4);
    s[7 * K + j] = 0; s[8 * K + j] = -1; s[9 * K + j] = -1; s[10 * K + j] = 0; s[11 * K + j] = -1;
  }
  int *a = s + kSlotArrays * K;
  for (int e = 0; e < KP2; ++e) {
    a[e] = 0; a[KP2 + e] = 0; a[2 * KP2 + e] = -1;
    memcpy(&a[3 * KP2 + e], &ninf, 4);
    a[4 * KP2 + e] = 0; a[5 * KP2 + e] = 0;
  }
  CU(cudaMemcpy(st->state, h.get(), n * 4, cudaMemcpyHostToDevice));
  Node root;
  memset(&root, 0, sizeof(root));
  root.parent = -1; root.chr = -1; root.lpc = -FLT_MAX; root.ts = 0; root.jump = -1;
  CU(cudaMemcpy(st->arena, &root, sizeof(Node), cudaMemcpyHostToDevice));
  return CTCDEC_OK;
}

// lm: the state will decode with a scorer, whose beam kernel layout is checked instead (at one stream, the widest
// block size the plan picks for the configuration: every batch of such states fits then)
static int state_create(const ctcdec_config *cfg, int device, bool lm, void **state) {
  Plan pl;
  int rc = make_plan(cfg, 1, 1, &pl, lm);
  if (rc) return rc;
  if (!state) return fail(CTCDEC_E_INVALID, "state is NULL");
  if ((rc = use_device(device))) return rc;
  StreamState *st = new StreamState();
  st->cfg = *cfg; st->device = device; st->frames = 0; st->arena = nullptr; st->state = nullptr;
  st->arena_cap = 1 + cfg->beam_size * kArenaSlackFrames;
  if (cudaMalloc(&st->arena, (size_t)st->arena_cap * sizeof(Node)) != cudaSuccess ||
      cudaMalloc(&st->state, (size_t)state_ints(cfg->beam_size) * 4) != cudaSuccess) {
    if (st->arena) cudaFree(st->arena);
    delete st;
    return fail(CTCDEC_E_CUDA, "cudaMalloc failed for the streaming state");
  }
  if ((rc = state_init_device(st))) { cudaFree(st->arena); cudaFree(st->state); delete st; return rc; }
  *state = st;
  return CTCDEC_OK;
}

int ctcdec_state_create(const ctcdec_config *cfg, int device, void **state) { return state_create(cfg, device, false, state); }

int ctcdec_state_create_lm(const ctcdec_config *cfg, void *scorer, int device, void **state) {
  if (!scorer) return ctcdec_state_create(cfg, device, state);
  HostScorer *sc = static_cast<HostScorer *>(scorer);
  if (cfg && (int)sc->labels.size() != cfg->vocab_size)
    return fail(CTCDEC_E_INVALID, "scorer was built for %zu labels, decoder has %d", sc->labels.size(), cfg->vocab_size);
  int rc = state_create(cfg, device, true, state);
  if (rc) return rc;
  StreamState *st = static_cast<StreamState *>(*state);
  st->lm_hist_n = sc->ngram ? sc->max_order - 1 : 0;
  // node 0 (the root): dictionary start state (0) and LM term 0, reference path_trie.cpp:11-30 / :165-174
  if (cudaMalloc(&st->lm_arena, (size_t)st->arena_cap * (1 + st->lm_hist_n) * 4) != cudaSuccess ||
      cudaMalloc(&st->dstate, (size_t)st->arena_cap * 4) != cudaSuccess ||
      cudaMemset(st->lm_arena, 0, 4) != cudaSuccess || cudaMemset(st->dstate, 0, 4) != cudaSuccess) {
    ctcdec_state_destroy(st);
    *state = nullptr;
    return fail(CTCDEC_E_CUDA, "cudaMalloc failed for the streaming state (scorer arrays)");
  }
  if (sc->is_character_based &&
      cudaMalloc(&st->lm_row, (size_t)st->arena_cap * sc->labels.size() * 4) != cudaSuccess) {
    ctcdec_state_destroy(st);
    *state = nullptr;
    return fail(CTCDEC_E_CUDA, "cudaMalloc failed for the streaming state (rows of a character-based model)");
  }
  st->sc = sc;
  st->mirror.reserve((size_t)st->arena_cap);
  return CTCDEC_OK;
}

int ctcdec_state_destroy(void *state) {
  if (!state) return CTCDEC_OK;
  StreamState *st = static_cast<StreamState *>(state);
  cudaSetDevice(st->device);
  if (st->last) cudaEventSynchronize(st->last->ev);  // device-path work may still read or write the state
  cudaFree(st->arena);
  cudaFree(st->state);
  if (st->lm_arena) cudaFree(st->lm_arena);
  if (st->dstate) cudaFree(st->dstate);
  if (st->lm_row) cudaFree(st->lm_row);
  delete st;
  return CTCDEC_OK;
}

int ctcdec_state_frames(const void *state, int *frames) {
  if (!state || !frames) return fail(CTCDEC_E_INVALID, "NULL argument");
  *frames = static_cast<const StreamState *>(state)->frames;
  return CTCDEC_OK;
}

// Two scorers of one call that are not the same object: both n-gram scorers from ctcdec_scorer_create_arpa, of one kind
// and built for the same labels (each utterance or stream then decodes with its own through its LM slot).  i: the
// index named in the message.
static int check_scorer_pair(const HostScorer *a, const HostScorer *b, const char *what, int i) {
  if (!a->ngram || !b->ngram)
    return fail(CTCDEC_E_UNSUPPORTED, "a hook scorer cannot share a call with another scorer: its terms come from the "
                "host's per-frame handshake");
  if (a->is_character_based != b->is_character_based)
    return fail(CTCDEC_E_UNSUPPORTED, "%s %d and 0 of one call are not both word-based or both character-based", what,
                i);
  if (a->labels != b->labels) return fail(CTCDEC_E_INVALID, "%s %d and 0 were built for different labels", what, i);
  return CTCDEC_OK;
}

// The distinct scorers of a call's states (scs, at most kMaxLmSlots of them) and the index of each stream's among them.
static void stream_scorers(void *const *states, int B, std::vector<HostScorer *> *scs,
                           std::vector<unsigned char> *slot_of) {
  scs->clear();
  slot_of->assign((size_t)B, 0);
  for (int b = 0; b < B; ++b) {
    HostScorer *sc = static_cast<const StreamState *>(states[b])->sc;
    size_t i = 0;
    while (i < scs->size() && (*scs)[i] != sc) ++i;
    if (i == scs->size()) scs->push_back(sc);
    (*slot_of)[b] = (unsigned char)i;
  }
}

// all states of one call: non-NULL, distinct, same configuration and device; their scorers one object (or none), or
// n-gram scorers that check_scorer_pair lets share a call, at most kMaxLmSlots different ones
static int check_states(void *const *states, int B) {
  if (!states) return fail(CTCDEC_E_INVALID, "states is NULL");
  for (int b = 0; b < B; ++b)
    if (!states[b]) return fail(CTCDEC_E_INVALID, "states[%d] is NULL", b);
  const StreamState *s0 = static_cast<const StreamState *>(states[0]);
  std::vector<const HostScorer *> seen(1, s0->sc);
  for (int b = 1; b < B; ++b) {
    const StreamState *sb = static_cast<const StreamState *>(states[b]);
    if (memcmp(&sb->cfg, &s0->cfg, sizeof(s0->cfg)) != 0 || sb->device != s0->device)
      return fail(CTCDEC_E_UNSUPPORTED, "all states of one call must come from the same decoder configuration and device");
    if (sb->sc != s0->sc) {
      if (!sb->sc || !s0->sc)
        return fail(CTCDEC_E_UNSUPPORTED, "states with a scorer and states without one cannot share a call");
      int rc = check_scorer_pair(s0->sc, sb->sc, "the scorers of states", b);
      if (rc) return rc;
      if (std::find(seen.begin(), seen.end(), sb->sc) == seen.end()) seen.push_back(sb->sc);
      if ((int)seen.size() > kMaxLmSlots)
        return fail(CTCDEC_E_UNSUPPORTED, "the states of one call use more than %d different scorers "
                    "(CTCDEC_LM_MIXED_MAX_MODELS)", kMaxLmSlots);
    }
    for (int a = 0; a < b; ++a)
      if (states[a] == states[b]) return fail(CTCDEC_E_INVALID, "states[%d] and states[%d] are the same object", a, b);
  }
  return CTCDEC_OK;
}

// Device bytes of the LM slots of a streaming call whose states use several scorers (0 for one scorer or none): the
// streams' slot indices, then one slot per scorer, each region 256-byte aligned.
static size_t stream_slot_bytes(void *const *states, int B) {
  std::vector<HostScorer *> scs;
  std::vector<unsigned char> slot_of;
  stream_scorers(states, B, &scs, &slot_of);
  return scs.size() > 1 ? al256((size_t)B) + al256(scs.size() * kLmSlotBytes) : 0;
}

// order work on stream s after the pending device-path calls of these states
static int wait_device_work(void *const *states, int B, cudaStream_t s) {
  const StreamEvent *prev = nullptr;
  for (int b = 0; b < B; ++b) {
    const StreamEvent *e = static_cast<StreamState *>(states[b])->last.get();
    if (e && e != prev) CU(cudaStreamWaitEvent(s, e->ev, 0));
    prev = e;
  }
  return CTCDEC_OK;
}

static int record_device_work(void *const *states, int B, cudaStream_t s) {
  auto e = std::make_shared<StreamEvent>();
  CU(cudaEventCreateWithFlags(&e->ev, cudaEventDisableTiming));
  CU(cudaEventRecord(e->ev, s));
  for (int b = 0; b < B; ++b) static_cast<StreamState *>(states[b])->last = e;
  return CTCDEC_OK;
}

// Grow each arena so that node_base + K * (frames since the last compaction, this chunk included) nodes fit: for a
// state never compacted, 1 + K * (frames consumed after this chunk).  Doubling keeps this to about
// log2(frames / 256) times per stream; the copy runs on s (after the stream's earlier work) and the host waits for
// it before the old arrays are freed.
static int grow_arenas(void *const *states, int B, const int *clen, cudaStream_t s) {
  for (int b = 0; b < B; ++b) {
    StreamState *sb = static_cast<StreamState *>(states[b]);
    const int K = sb->cfg.beam_size, V = sb->cfg.vocab_size;
    const long long need = sb->node_base + (long long)K * (sb->since + clen[b]);
    if (need <= sb->arena_cap) continue;
    long long cap = std::max<long long>(need, 2ll * sb->arena_cap);
    if (cap > 0x7fffffffll / 2) return fail(CTCDEC_E_UNSUPPORTED, "stream too long for the node arena");
    Node *na = nullptr;
    CU(cudaMalloc(&na, (size_t)cap * sizeof(Node)));
    const long long used = std::min<long long>(sb->arena_cap, sb->node_base + (long long)K * sb->since);
    CU(cudaMemcpyAsync(na, sb->arena, (size_t)used * sizeof(Node), cudaMemcpyDeviceToDevice, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaFree(sb->arena));
    sb->arena = na;
    if (sb->sc) {
      float *nl = nullptr;
      int *nd = nullptr;
      CU(cudaMalloc(&nl, (size_t)cap * (1 + sb->lm_hist_n) * 4));
      CU(cudaMalloc(&nd, (size_t)cap * 4));
      CU(cudaMemcpyAsync(nl, sb->lm_arena, (size_t)used * 4, cudaMemcpyDeviceToDevice, s));
      if (sb->lm_hist_n)  // the LM histories, behind the terms
        CU(cudaMemcpyAsync(nl + cap, sb->lm_arena + sb->arena_cap, (size_t)used * sb->lm_hist_n * 4,
                           cudaMemcpyDeviceToDevice, s));
      CU(cudaMemcpyAsync(nd, sb->dstate, (size_t)used * 4, cudaMemcpyDeviceToDevice, s));
      CU(cudaStreamSynchronize(s));
      CU(cudaFree(sb->lm_arena));
      CU(cudaFree(sb->dstate));
      sb->lm_arena = nl;
      sb->dstate = nd;
      if (sb->lm_row) {
        float *nr = nullptr;
        CU(cudaMalloc(&nr, (size_t)cap * V * 4));
        CU(cudaMemcpyAsync(nr, sb->lm_row, (size_t)used * V * 4, cudaMemcpyDeviceToDevice, s));
        CU(cudaStreamSynchronize(s));
        CU(cudaFree(sb->lm_row));
        sb->lm_row = nr;
      }
    }
    sb->arena_cap = (int)cap;
  }
  return CTCDEC_OK;
}

// Device buffers of one chunk step.
struct ChunkBuffers {
  const void *chunk;  // [B, T, V]: probabilities / log-probabilities (kind IN_F32) or logits
  int kind;
  unsigned char *ws;  // the plan's pruned rows and characters (a workspace laid out by the plan, up to off_arena)
  unsigned char *tab; // stream_tab_layout(B).total bytes
  unsigned char *slot_tab;  // states of several scorers: stream_slot_bytes bytes for their slot indices and LM slots,
                            // else NULL
  DecodeOut out;
  int out_T;
};

// One chunk step of a streaming decode, enqueued on s; shared by ctcdec_decode_stream_host (which stages the chunk
// and the results around it) and ctcdec_decode_stream_device.  Grows the arenas, writes the per-call tables, runs the
// prune scan, the beam kernel (for states with a scorer: the persistent launch with the per-frame host handshake,
// which needs the pinned exchange buffers of `c` and returns synchronised) and, if a stream is at eos, the finalize
// kernel; advances every state's frame counter.  n_results / flags are cleared first; flags then collect the prune's
// and the finalize's bits.
static int stream_chunk_step(const ctcdec_config &cfg, Plan &pl, void *const *states, int B, int T,
                             const int32_t *seq_lens, const uint8_t *is_eos, const ChunkBuffers &io, DevCache *c,
                             cudaStream_t s) {
  int rc = CTCDEC_OK;
  bool any_eos = false;
  std::vector<int> clen(B);
  std::vector<uint8_t> at_root(B);  // streams that have not seen a frame yet
  for (int b = 0; b < B; ++b) {
    clen[b] = std::max(0, std::min(seq_lens ? seq_lens[b] : T, T));
    any_eos |= is_eos[b] != 0;
    at_root[b] = static_cast<StreamState *>(states[b])->frames == 0;
  }
  if ((rc = grow_arenas(states, B, clen.data(), s))) return rc;
  HostScorer *const sc = static_cast<StreamState *>(states[0])->sc;
  const int device = static_cast<StreamState *>(states[0])->device;
  std::vector<HostScorer *> scs;
  std::vector<unsigned char> slot_of;
  stream_scorers(states, B, &scs, &slot_of);
  for (HostScorer *si : scs)
    if (si && ((rc = ensure_dict_on_device(si, device)) || (si->ngram && (rc = ensure_ngram_on_device(si, device)))))
      return rc;
  const StreamTabLayout L = stream_tab_layout(B);
  for (int b0 = 0; b0 < B; b0 += kTabPerLaunch) {
    StreamTabArgs a;
    memset(&a, 0, sizeof(a));
    a.tab = io.tab; a.L = L; a.b0 = b0; a.n = std::min(kTabPerLaunch, B - b0);
    for (int i = 0; i < a.n; ++i) {
      StreamState *sb = static_cast<StreamState *>(states[b0 + i]);
      a.arena[i] = sb->arena; a.state[i] = sb->state; a.cap[i] = sb->arena_cap; a.fin[i] = is_eos[b0 + i] ? 1 : 0;
      a.lmar[i] = sb->lm_arena; a.dst[i] = sb->dstate; a.rows[i] = sb->lm_row; a.len[i] = clen[b0 + i];
    }
    stream_table_kernel<<<1, kTabPerLaunch, 0, s>>>(a);
    CU(cudaGetLastError());
  }
  const int *d_len = seq_lens ? reinterpret_cast<const int *>(io.tab + L.lens) : nullptr;
  CU(cudaMemsetAsync(io.out.flags, 0, (size_t)B * 4, s));
  CU(cudaMemsetAsync(io.out.n_results, 0, (size_t)B * 4, s));
  if (T > 0 && (rc = launch_prune(&cfg, pl, PruneInput{io.chunk, io.kind, nullptr, sc != nullptr}, d_len, B, T, io.ws,
                                  io.out.flags, s)))
    return rc;
  BeamParams bp = beam_params(cfg, pl, io.ws, d_len, T, io.out, io.out_T);
  bp.tile_frames = pl.F;
  bp.arena_ptrs = (Node *const *)(io.tab + L.arenas); bp.state_ptrs = (int *const *)(io.tab + L.states);
  bp.arena_caps = (const int *)(io.tab + L.caps);
  bp.finalize = io.tab + L.fin;
  bp.fresh = 0;
  if (sc && T > 0) {
    attach_scorer(bp, *sc);
    bp.lm_arena_ptrs = (float *const *)(io.tab + L.lmar);
    bp.dstate_ptrs = (int *const *)(io.tab + L.dst);
    if (sc->is_character_based) bp.lm_row_ptrs = (float *const *)(io.tab + L.rows);
  }
  if (scs.size() > 1) {
    // streams of several scorers: stream b decodes with the LM slot of its own scorer, its weights as they are now
    // (each stream keeps its own order - 1 histories behind its LM terms)
    unsigned char *const d_slot_of = io.slot_tab;
    LmSlot *const slots = reinterpret_cast<LmSlot *>(io.slot_tab + al256((size_t)B));
    if ((rc = upload_slots(scs.data(), (int)scs.size(), slot_of.data(), B, slots, d_slot_of, s))) return rc;
    bp.lm_slots = slots; bp.lm_slot_of = d_slot_of;
  }
  if (sc && !sc->ngram && T > 0) {
    // hook scorer: one persistent launch per chunk, hand shake after EVERY frame (the frame after the chunk's last
    // one, in the next call, needs the LM terms of the nodes created now).  An n-gram scorer needs none: the beam
    // kernel computes the LM terms itself.
    if ((rc = prepare_exchange(*c, *sc, B, at_root.data(), bp))) return rc;
    bp.lm_hs_last = 1;
    std::vector<TrieMirror *> mirrors(B);
    for (int b = 0; b < B; ++b) mirrors[b] = &static_cast<StreamState *>(states[b])->mirror;
    if ((rc = run_handshake(bp, pl, B, sc, *c, clen.data(), mirrors.data(), nullptr, "scorer path, streaming", s)))
      return rc;
  } else if (T > 0 && (rc = launch_beam(bp, pl, B, s))) {
    return rc;
  }
  for (int b = 0; b < B; ++b) {
    StreamState *sb = static_cast<StreamState *>(states[b]);
    sb->frames += clen[b];
    sb->since += clen[b];
  }
  if (any_eos && (rc = launch_finalize(bp, B, s))) return rc;
  return CTCDEC_OK;
}

int ctcdec_decode_stream_host(const float *probs, const int32_t *seq_lens, int B, int T, void *const *states,
                              const uint8_t *is_eos, int32_t *tokens, int32_t *timesteps, int out_T, float *scores,
                              int32_t *lens, int32_t *n_results, int32_t *flags) {
  if (B <= 0) return B == 0 ? CTCDEC_OK : fail(CTCDEC_E_INVALID, "negative batch");
  if (!states || !is_eos) return fail(CTCDEC_E_INVALID, "states / is_eos is NULL");
  int rc = check_states(states, B);
  if (rc) return rc;
  StreamState *s0 = static_cast<StreamState *>(states[0]);
  const ctcdec_config cfg = s0->cfg;
  Plan pl;
  if ((rc = make_plan(&cfg, B, T, &pl, s0->sc != nullptr))) return rc;
  const int device = s0->device;
  if ((rc = use_device(device))) return rc;
  std::lock_guard<std::mutex> lock(g_mu[device]);
  DevCache &c = g_cache[device];
  if (!c.stream) CU(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
  cudaStream_t s = c.stream;
  if ((rc = wait_device_work(states, B, s))) return rc;
  const int V = cfg.vocab_size, K = cfg.beam_size;
  bool any_eos = false;
  for (int b = 0; b < B; ++b) any_eos |= is_eos[b] != 0;
  if (any_eos && (!tokens || !timesteps || !scores || !lens)) return fail(CTCDEC_E_INVALID, "an output pointer is NULL");
  if (any_eos && out_T < 0) return fail(CTCDEC_E_INVALID, "out_T < 0");
  const size_t n_probs = (size_t)B * T * V, n_out = any_eos ? (size_t)B * K * (size_t)out_T : 0;
  HostScorer *const sc = s0->sc;
  if ((rc = ensure(c, kBufInput, n_probs * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufTokens, n_out * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufTimesteps, n_out * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufSmall, small_bytes(B, K)))) return rc;
  if ((rc = ensure(c, kBufWork, pl.off_arena + 512))) return rc;  // only the lp / idx part of the plan is used
  const size_t slot_bytes = stream_slot_bytes(states, B);
  if ((rc = ensure(c, kBufStreamTab, stream_tab_layout(B).total + slot_bytes + 256))) return rc;
  float *d_probs = (float *)c.buf[kBufInput];
  int *d_tok = (int *)c.buf[kBufTokens], *d_ts = (int *)c.buf[kBufTimesteps];
  const SmallOut d = small_out(c.buf[kBufSmall], B, K);
  if (n_probs) CU(cudaMemcpyAsync(d_probs, probs, n_probs * 4, cudaMemcpyHostToDevice, s));
  ChunkBuffers io;
  io.chunk = d_probs; io.kind = IN_F32;
  io.ws = align256(c.buf[kBufWork]);
  io.tab = (unsigned char *)c.buf[kBufStreamTab];
  io.slot_tab = slot_bytes ? io.tab + stream_tab_layout(B).total : nullptr;
  io.out = DecodeOut{d_tok, d_ts, d.scores, d.lens, d.n_results, d.flags};
  io.out_T = out_T;
  if ((rc = stream_chunk_step(cfg, pl, states, B, T, seq_lens, is_eos, io, &c, s))) return rc;
  if (any_eos) {
    if ((rc = ensure_pinned(c, kPinSmall, small_bytes(B, K)))) return rc;
    const SmallOut h = small_out(c.pin[kPinSmall], B, K);
    if ((rc = read_small(h, d, K, 0, B, s))) return rc;
    CU(cudaStreamSynchronize(s));
    copy_result_rows(h, B, K, is_eos, scores, lens);
    const int max_len = max_result_len(h, K, 0, B, is_eos);
    if (max_len > out_T) return fail(CTCDEC_E_INVALID, "out_T (%d) smaller than the longest prefix (%d)", out_T, max_len);
    if (max_len > 0) {
      // copy per finalized stream so rows of non-eos streams stay untouched
      for (int b = 0; b < B; ++b) {
        if (!is_eos[b] || h.n_results[b] == 0) continue;
        const size_t off = (size_t)b * K * out_T;
        if ((rc = enqueue_rows(d_tok + off, d_ts + off, tokens + off, timesteps + off, nullptr, nullptr,
                               (size_t)h.n_results[b], max_len, out_T, s)))
          return rc;
      }
    }
    CU(cudaStreamSynchronize(s));
    if (sc) {  // reported scores of the finished streams: approx_ctc (reference ctc_beam_search_decoder.cpp:173-208),
               // each with its own scorer
      std::vector<HostScorer *> scs;
      std::vector<unsigned char> slot_of;
      stream_scorers(states, B, &scs, &slot_of);
      std::vector<int> nres_eos(B);
      for (size_t i = 0; i < scs.size(); ++i) {
        for (int b = 0; b < B; ++b) nres_eos[b] = is_eos[b] && slot_of[b] == i ? h.n_results[b] : 0;
        lm_rescore_batch(*scs[i], B, K, out_T, nres_eos.data(), tokens, lens, scores);
      }
    }
    if (n_results) memcpy(n_results, h.n_results, (size_t)B * 4);
    if (flags) memcpy(flags, h.flags, (size_t)B * 4);
    if ((rc = check_error_flags(h.flags, B))) return rc;
  } else {
    CU(cudaStreamSynchronize(s));
    if (n_results) memset(n_results, 0, (size_t)B * 4);
  }
  return CTCDEC_OK;
}

// device scratch of ctcdec_decode_stream_device: the plan's pruned rows / characters, then the per-call tables, then
// for states of several scorers their LM slots (slot_bytes, stream_slot_bytes)
static size_t stream_workspace_bytes(const Plan &pl, int B, size_t slot_bytes = 0) {
  return al256(pl.off_arena) + stream_tab_layout(B).total + slot_bytes + 256;
}

int ctcdec_stream_workspace_bytes(const ctcdec_config *cfg, int B, int T, size_t *bytes) {
  Plan pl;
  int rc = make_plan(cfg, B, T, &pl);
  if (rc) return rc;
  if (!bytes) return fail(CTCDEC_E_INVALID, "bytes is NULL");
  *bytes = stream_workspace_bytes(pl, B);
  return CTCDEC_OK;
}

int ctcdec_stream_states_workspace_bytes(void *const *states, int B, int T, size_t *bytes) {
  if (B <= 0) return fail(CTCDEC_E_INVALID, "batch %d: the states decide the workspace, at least one is needed", B);
  int rc = check_states(states, B);
  if (rc) return rc;
  const StreamState *s0 = static_cast<const StreamState *>(states[0]);
  Plan pl;
  if ((rc = make_plan(&s0->cfg, B, T, &pl))) return rc;
  if (!bytes) return fail(CTCDEC_E_INVALID, "bytes is NULL");
  *bytes = stream_workspace_bytes(pl, B, stream_slot_bytes(states, B));
  return CTCDEC_OK;
}

// the states' device must be the current one: the caller's stream and buffers belong to it
static int check_current_device(const StreamState *s0) {
  int dev = -1;
  const int rc = current_device(&dev);
  if (rc) return rc;
  if (dev != s0->device) return fail(CTCDEC_E_INVALID, "the states live on device %d, the current device is %d", s0->device, dev);
  return CTCDEC_OK;
}

int ctcdec_decode_stream_device(const void *probs, int dtype, const int32_t *seq_lens, int B, int T,
                                void *const *states, const uint8_t *is_eos, int32_t *tokens, int32_t *timesteps,
                                int out_T, float *scores, int32_t *lens, int32_t *n_results, int32_t *flags,
                                void *workspace, size_t workspace_bytes, void *stream) {
  if (B <= 0) return B == 0 ? CTCDEC_OK : fail(CTCDEC_E_INVALID, "negative batch");
  int kind = 0;
  int rc = input_kind(dtype, true, &kind);
  if (rc) return rc;
  if (!states || !is_eos) return fail(CTCDEC_E_INVALID, "states / is_eos is NULL");
  if ((rc = check_states(states, B))) return rc;
  StreamState *s0 = static_cast<StreamState *>(states[0]);
  HostScorer *const sc = s0->sc;
  if (sc && !sc->ngram)
    return fail(CTCDEC_E_UNSUPPORTED, "states with a scorer need the per-frame host handshake: use ctcdec_decode_stream_host");
  const ctcdec_config cfg = s0->cfg;
  Plan pl;
  if ((rc = make_plan(&cfg, B, T, &pl, sc != nullptr))) return rc;
  if (!probs && T > 0) return fail(CTCDEC_E_INVALID, "probs is NULL");
  if (!n_results || !flags) return fail(CTCDEC_E_INVALID, "n_results and flags device buffers are required");
  bool any_eos = false;
  for (int b = 0; b < B; ++b) {
    if (!is_eos[b]) continue;
    any_eos = true;
    const int len = std::max(0, std::min(seq_lens ? seq_lens[b] : T, T));
    const int need = static_cast<StreamState *>(states[b])->frames + len;
    if (out_T < need) return fail(CTCDEC_E_INVALID, "out_T (%d) smaller than stream %d's frames after this chunk (%d)", out_T, b, need);
  }
  if (any_eos && (!tokens || !timesteps || !scores || !lens)) return fail(CTCDEC_E_INVALID, "an output pointer is NULL");
  if ((rc = check_current_device(s0))) return rc;
  unsigned char *ws = nullptr;
  const size_t slot_bytes = stream_slot_bytes(states, B);
  if ((rc = workspace_start(workspace, workspace_bytes, stream_workspace_bytes(pl, B, slot_bytes), &ws))) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  std::lock_guard<std::mutex> lock(g_mu[s0->device]);
  if ((rc = wait_device_work(states, B, s))) return rc;
  ChunkBuffers io;
  io.chunk = probs; io.kind = kind;
  io.ws = ws;
  io.tab = ws + al256(pl.off_arena);
  io.slot_tab = slot_bytes ? io.tab + stream_tab_layout(B).total : nullptr;
  io.out = DecodeOut{tokens, timesteps, scores, lens, n_results, flags};
  io.out_T = out_T;
  if ((rc = stream_chunk_step(cfg, pl, states, B, T, seq_lens, is_eos, io, nullptr, s))) return rc;
  if (sc && any_eos) {  // the eos streams' reported scores (the other streams' n_results are 0: their rows are skipped)
    if ((rc = ensure_ngram_on_device(sc, s0->device))) return rc;
    if (slot_bytes) {  // each stream's rows with its own scorer's slot (written by the chunk step, also with T = 0)
      const LmSlot *slots = reinterpret_cast<const LmSlot *>(io.slot_tab + al256((size_t)B));
      rc = launch_readout(nullptr, tokens, lens, n_results, scores, B, cfg.beam_size, out_T, s, nullptr, 0, slots,
                          io.slot_tab);
    } else {
      rc = launch_readout(sc, tokens, lens, n_results, scores, B, cfg.beam_size, out_T, s);
    }
    if (rc) return rc;
  }
  return record_device_work(states, B, s);
}

int ctcdec_stream_committed_device(void *const *states, int B, const int32_t *since, int32_t *committed,
                                   int32_t *tokens, int32_t *timesteps, int cap, void *stream) {
  if (B <= 0) return B == 0 ? CTCDEC_OK : fail(CTCDEC_E_INVALID, "negative batch");
  if (!committed) return fail(CTCDEC_E_INVALID, "committed is NULL");
  if (cap < 0) return fail(CTCDEC_E_INVALID, "cap %d < 0", cap);
  if (cap > 0 && (!tokens || !timesteps)) return fail(CTCDEC_E_INVALID, "tokens / timesteps is NULL");
  int rc = check_states(states, B);
  if (rc) return rc;
  StreamState *s0 = static_cast<StreamState *>(states[0]);
  if ((rc = check_current_device(s0))) return rc;
  const int K = s0->cfg.beam_size;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  std::lock_guard<std::mutex> lock(g_mu[s0->device]);
  if ((rc = wait_device_work(states, B, s))) return rc;
  const size_t smem = committed_smem_bytes(K);
  if ((rc = raise_smem_limit<committed_kernel<128>>(smem, "committed-prefix"))) return rc;
  for (int b0 = 0; b0 < B; b0 += kCommitPerLaunch) {
    CommitArgs a;
    memset(&a, 0, sizeof(a));
    const int n = std::min(kCommitPerLaunch, B - b0);
    for (int i = 0; i < n; ++i) {
      const StreamState *sb = static_cast<const StreamState *>(states[b0 + i]);
      a.arena[i] = sb->arena; a.state[i] = sb->state;
    }
    a.K = K; a.b0 = b0; a.cap = cap; a.since = since; a.committed = committed; a.tokens = tokens; a.timesteps = timesteps;
    committed_kernel<128><<<n, 128, smem, s>>>(a);
    CU(cudaGetLastError());
  }
  return record_device_work(states, B, s);
}

// Device bytes of one state's arrays of `cap` nodes: arena, and with a scorer the LM terms and histories, dictionary
// states and a character-based model's rows.
static size_t state_arena_bytes(const StreamState *st, long long cap) {
  size_t n = (size_t)cap * sizeof(Node);
  if (st->sc) n += (size_t)cap * (1 + st->lm_hist_n) * 4 + (size_t)cap * 4;
  if (st->lm_row) n += (size_t)cap * st->cfg.vocab_size * 4;
  return n;
}

int ctcdec_state_device_bytes(const void *state, size_t *bytes) {
  if (!state || !bytes) return fail(CTCDEC_E_INVALID, "NULL argument");
  const StreamState *st = static_cast<const StreamState *>(state);
  *bytes = state_arena_bytes(st, st->arena_cap) + (size_t)state_ints(st->cfg.beam_size) * 4;
  return CTCDEC_OK;
}

int ctcdec_stream_compact(void *const *states, int B, int64_t *nodes_kept, void *stream) {
  if (B <= 0) return B == 0 ? CTCDEC_OK : fail(CTCDEC_E_INVALID, "negative batch");
  if (!states) return fail(CTCDEC_E_INVALID, "states is NULL");
  for (int b = 0; b < B; ++b) {
    if (!states[b]) return fail(CTCDEC_E_INVALID, "states[%d] is NULL", b);
    for (int a = 0; a < b; ++a)
      if (states[a] == states[b]) return fail(CTCDEC_E_INVALID, "states[%d] and states[%d] are the same object", a, b);
  }
  StreamState *s0 = static_cast<StreamState *>(states[0]);
  for (int b = 0; b < B; ++b) {
    const StreamState *sb = static_cast<const StreamState *>(states[b]);
    if (sb->device != s0->device) return fail(CTCDEC_E_UNSUPPORTED, "all states of one call must live on one device");
    if (sb->sc && !sb->sc->ngram)
      return fail(CTCDEC_E_UNSUPPORTED, "states[%d] has a hook scorer: the host's mirror of its trie is indexed by node "
                  "id, so its arena cannot be compacted", b);
  }
  int rc = check_current_device(s0);
  if (rc) return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  CU(cudaStreamIsCapturing(s, &capturing));
  if (capturing != cudaStreamCaptureStatusNone)
    return fail(CTCDEC_E_UNSUPPORTED, "ctcdec_stream_compact cannot be captured into a CUDA graph: it waits for the "
                "device and allocates the compacted arrays");
  size_t smem = 0, map_ints = 0;
  for (int b = 0; b < B; ++b) {
    const StreamState *sb = static_cast<const StreamState *>(states[b]);
    smem = std::max(smem, compact_smem_bytes(sb->cfg.beam_size, kCompactNT));
    map_ints += (size_t)sb->arena_cap;
  }
  if ((rc = raise_smem_limit<compact_mark_kernel>(smem, "compaction"))) return rc;
  std::lock_guard<std::mutex> lock(g_mu[s0->device]);
  if ((rc = wait_device_work(states, B, s))) return rc;
  // scratch: every stream's id map (at most arena_cap nodes each), then the kept counts
  int *scratch = nullptr;
  CU(cudaMalloc(&scratch, (map_ints + B) * 4));
  std::unique_ptr<int, cudaError_t (*)(void *)> scratch_owner(scratch, cudaFree);
  int *const d_kept = scratch + map_ints;
  std::vector<int *> maps(B);
  size_t o = 0;
  for (int b = 0; b < B; o += static_cast<StreamState *>(states[b])->arena_cap, ++b) maps[b] = scratch + o;
  for (int b0 = 0; b0 < B; b0 += kCompactPerLaunch) {
    CompactMarkArgs a;
    memset(&a, 0, sizeof(a));
    const int n = std::min(kCompactPerLaunch, B - b0);
    for (int i = 0; i < n; ++i) {
      const StreamState *sb = static_cast<const StreamState *>(states[b0 + i]);
      a.arena[i] = sb->arena; a.state[i] = sb->state; a.map[i] = maps[b0 + i]; a.K[i] = sb->cfg.beam_size;
      a.cap[i] = sb->arena_cap;
    }
    a.kept = d_kept + b0;
    compact_mark_kernel<<<n, kCompactNT, smem, s>>>(a);
    CU(cudaGetLastError());
  }
  std::vector<int> kept(B);
  CU(cudaMemcpyAsync(kept.data(), d_kept, (size_t)B * 4, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  // the compacted arrays; on a failure here nothing has changed yet
  struct Fresh { Node *arena = nullptr; float *lm = nullptr, *row = nullptr; int *dst = nullptr; long long cap = 0; };
  std::vector<Fresh> nw(B);
  auto free_fresh = [&](bool which_new) {
    for (int b = 0; b < B; ++b) {
      StreamState *sb = static_cast<StreamState *>(states[b]);
      if (which_new) { cudaFree(nw[b].arena); cudaFree(nw[b].lm); cudaFree(nw[b].dst); cudaFree(nw[b].row); }
      else { cudaFree(sb->arena); cudaFree(sb->lm_arena); cudaFree(sb->dstate); cudaFree(sb->lm_row); }
    }
  };
  for (int b = 0; b < B; ++b) {
    const StreamState *sb = static_cast<const StreamState *>(states[b]);
    const long long K = sb->cfg.beam_size;
    Fresh &f = nw[b];
    f.cap = std::max<long long>(1 + K * kArenaSlackFrames, kept[b] + K * kArenaSlackFrames);
    bool ok = cudaMalloc(&f.arena, (size_t)f.cap * sizeof(Node)) == cudaSuccess;
    if (ok && sb->sc)
      ok = cudaMalloc(&f.lm, (size_t)f.cap * (1 + sb->lm_hist_n) * 4) == cudaSuccess &&
           cudaMalloc(&f.dst, (size_t)f.cap * 4) == cudaSuccess;
    if (ok && sb->lm_row) ok = cudaMalloc(&f.row, (size_t)f.cap * sb->cfg.vocab_size * 4) == cudaSuccess;
    if (!ok) {
      cudaGetLastError();
      free_fresh(true);
      return fail(CTCDEC_E_CUDA, "cudaMalloc failed for the compacted arrays of stream %d; the states are unchanged", b);
    }
  }
  for (int b0 = 0; b0 < B; b0 += kCompactPerLaunch) {
    CompactGatherArgs a;
    memset(&a, 0, sizeof(a));
    const int n = std::min(kCompactPerLaunch, B - b0);
    for (int i = 0; i < n; ++i) {
      const StreamState *sb = static_cast<const StreamState *>(states[b0 + i]);
      const Fresh &f = nw[b0 + i];
      CompactJob &j = a.job[i];
      j.arena = sb->arena; j.arena_new = f.arena; j.state = sb->state; j.map = maps[b0 + i];
      j.lm = sb->lm_arena; j.lm_new = f.lm; j.dst = sb->dstate; j.dst_new = f.dst; j.row = sb->lm_row; j.row_new = f.row;
      j.K = sb->cfg.beam_size; j.cap = sb->arena_cap; j.cap_new = (int)f.cap; j.H = sb->lm_hist_n;
      j.V = sb->cfg.vocab_size; j.kept = kept[b0 + i];
    }
    compact_gather_kernel<<<n, kCompactNT, 0, s>>>(a);
    CU(cudaGetLastError());
  }
  if ((rc = record_device_work(states, B, s))) return rc;
  CU(cudaStreamSynchronize(s));
  free_fresh(false);
  for (int b = 0; b < B; ++b) {
    StreamState *sb = static_cast<StreamState *>(states[b]);
    const Fresh &f = nw[b];
    sb->arena = f.arena; sb->lm_arena = f.lm; sb->dstate = f.dst; sb->lm_row = f.row; sb->arena_cap = (int)f.cap;
    sb->node_base = kept[b];
    sb->since = 0;
    if (nodes_kept) nodes_kept[b] = kept[b];
  }
  return CTCDEC_OK;
}

// ---------------------------------------------------------------------------------------------------
//  scorer path
// ---------------------------------------------------------------------------------------------------
int ctcdec_scorer_create(const ctcdec_scorer_hooks *hooks, double alpha, double beta, const char *const *labels,
                         int n_labels, const char *const *words, int n_words, int max_order, int is_character_based,
                         void **scorer) {
  if (!hooks || !hooks->cond_log_prob || !hooks->sent_log_prob) return fail(CTCDEC_E_INVALID, "scorer hooks are NULL");
  if (!labels || n_labels < 1 || (!words && n_words > 0) || n_words < 0 || !scorer)
    return fail(CTCDEC_E_INVALID, "bad labels / words / scorer argument");
  if (max_order < 1) return fail(CTCDEC_E_INVALID, "max_order %d < 1", max_order);
  HostScorer *sc = new HostScorer();
  sc->hooks = *hooks; sc->alpha = alpha; sc->beta = beta; sc->max_order = max_order;
  sc->is_character_based = is_character_based ? 1 : 0;
  sc->space_id = -2;
  for (int i = 0; i < n_labels; ++i) {
    sc->labels.emplace_back(labels[i] ? labels[i] : "");
    if (sc->labels.back() == " ") sc->space_id = i;  // reference ctc_beam_search_decoder.cpp:34-40
  }
  if (sc->is_character_based) {
    // no dictionary, every appended character is scored (reference scorer.cpp:50-53, ctc_beam_search_decoder.cpp:46, :120-137)
    sc->dict = accept_all_dictionary(n_labels);
    *scorer = sc;
    return CTCDEC_OK;
  }
  if (sc->space_id < 0) {
    delete sc;
    return fail(CTCDEC_E_UNSUPPORTED, "a word-based scorer needs a \" \" label to end words with");
  }
  std::vector<std::string> w;
  for (int i = 0; i < n_words; ++i) w.emplace_back(words[i] ? words[i] : "");
  sc->dict = build_dictionary(sc->labels, sc->space_id, w);
  pack_dictionary(sc->dict, sc->space_id);
  *scorer = sc;
  return CTCDEC_OK;
}

int ctcdec_scorer_create_arpa(const char *path, double alpha, double beta, const char *const *labels, int n_labels,
                              void **scorer) {
  if (!path || !labels || n_labels < 1 || !scorer) return fail(CTCDEC_E_INVALID, "bad path / labels / scorer argument");
  if (FILE *probe = fopen(path, "rb")) fclose(probe);
  else return fail(CTCDEC_E_INVALID, "cannot open the language model %s", path);
  std::shared_ptr<NgramModel> m = std::make_shared<NgramModel>();
  for (int i = 0; i < n_labels; ++i) {
    m->labels.emplace_back(labels[i] ? labels[i] : "");
    if (m->labels.back() == " ") m->space_id = i;  // reference Scorer::set_char_map (scorer.cpp:148-161)
  }
  const std::string why = load_ngram_file(path, *m);
  if (!why.empty()) return fail(CTCDEC_E_UNSUPPORTED, "language model %s refused: %s", path, why.c_str());
  std::vector<const char *> words;
  for (const std::string &w : m->vocabulary) words.push_back(w.c_str());
  const ctcdec_scorer_hooks hooks = {m.get(), ngram_hook_cond, ngram_hook_sent};
  const int rc = ctcdec_scorer_create(&hooks, alpha, beta, labels, n_labels, words.data(), (int)words.size(), m->order,
                                      m->is_character_based, scorer);
  if (rc != CTCDEC_OK) return rc;
  HostScorer *sc = static_cast<HostScorer *>(*scorer);
  sc->ngram = m;
  lm_dev_word_ids(*sc);
  return CTCDEC_OK;
}

int ctcdec_scorer_table_bytes(const void *scorer, size_t *bytes) {
  if (!scorer || !bytes) return fail(CTCDEC_E_INVALID, "bad scorer / bytes argument");
  const HostScorer *sc = static_cast<const HostScorer *>(scorer);
  if (!sc->ngram) return fail(CTCDEC_E_UNSUPPORTED, "table_bytes takes a scorer from ctcdec_scorer_create_arpa only");
  *bytes = sc->ngram->table_bytes();
  return CTCDEC_OK;
}

static int scorer_hook_call(const void *scorer, const int32_t *labels, int n, double *out, bool sent) {
  if (!scorer || (!labels && n > 0) || n < 0 || !out) return fail(CTCDEC_E_INVALID, "bad scorer / labels / out argument");
  const HostScorer *sc = static_cast<const HostScorer *>(scorer);
  for (int i = 0; i < n; ++i)
    if (labels[i] < 0 || labels[i] >= (int)sc->labels.size())
      return fail(CTCDEC_E_INVALID, "label %d at position %d is outside [0, %d)", labels[i], i, (int)sc->labels.size());
  *out = (sent ? sc->hooks.sent_log_prob : sc->hooks.cond_log_prob)(sc->hooks.ctx, labels, n);
  return CTCDEC_OK;
}
int ctcdec_scorer_cond_log_prob(const void *scorer, const int32_t *labels, int n, double *out) {
  return scorer_hook_call(scorer, labels, n, out, false);
}
int ctcdec_scorer_sent_log_prob(const void *scorer, const int32_t *labels, int n, double *out) {
  return scorer_hook_call(scorer, labels, n, out, true);
}

int ctcdec_scorer_destroy(void *scorer) {
  if (!scorer) return CTCDEC_OK;
  HostScorer *sc = static_cast<HostScorer *>(scorer);
  if (sc->d_next) { cudaSetDevice(sc->device); cudaFree(sc->d_next); cudaFree(sc->d_mask); }
  if (sc->d_ngram) { cudaSetDevice(sc->ngram_device); cudaFree(sc->d_ngram); }
  delete sc;
  return CTCDEC_OK;
}
int ctcdec_scorer_is_character_based(const void *scorer) { return scorer ? static_cast<const HostScorer *>(scorer)->is_character_based : 0; }
int ctcdec_scorer_max_order(const void *scorer) { return scorer ? static_cast<const HostScorer *>(scorer)->max_order : 0; }
int ctcdec_scorer_dict_size(const void *scorer) { return scorer ? static_cast<const HostScorer *>(scorer)->dict.n_words : 0; }  // (0 for a character-based model: reference Scorer::dict_size_ stays 0)
int ctcdec_scorer_reset_params(void *scorer, double alpha, double beta) {
  if (!scorer) return fail(CTCDEC_E_INVALID, "scorer is NULL");
  HostScorer *sc = static_cast<HostScorer *>(scorer);
  sc->alpha = (double)(float)alpha;  // reference Scorer::reset_params(float, float) (scorer.cpp:122-125): both values
  sc->beta = (double)(float)beta;    // pass through float32 (the constructor takes doubles)
  return CTCDEC_OK;
}

// ARPA scorer: the device keeps the last order - 1 LM word ids of every trie node, batch x (1 + beam x frames) x
// (order - 1) ints
static int lm_hist_bytes(const HostScorer *sc, const Plan &pl, int B, size_t *bytes) {
  *bytes = sc->ngram ? (size_t)B * pl.arena_stride * (size_t)(sc->max_order - 1) * 4 : 0;
  if (*bytes > ((size_t)64 << 30))
    return fail(CTCDEC_E_UNSUPPORTED, "n-gram scorer: %zu bytes of per-node LM histories (batch x (1 + beam x frames) x "
                "(order - 1) x 4)", *bytes);
  return CTCDEC_OK;
}

// character-based model: the device keeps a row of V LM terms per trie node, batch x (1 + beam x frames) x V floats
static int lm_row_bytes(const HostScorer *sc, const Plan &pl, int B, size_t *bytes) {
  *bytes = sc->is_character_based ? (size_t)B * pl.arena_stride * sc->labels.size() * 4 : 0;
  if (*bytes > ((size_t)64 << 30))
    return fail(CTCDEC_E_UNSUPPORTED, "character-based model: %zu bytes of per-node rows (batch x (1 + beam x frames) x labels x 4)", *bytes);
  return CTCDEC_OK;
}

// Device buffers of one offline scorer decode: the library's own (ctcdec_decode_batch_lm_host, per-device cache) or
// the caller's outputs and workspace (ctcdec_decode_batch_lm_device).
struct LmBuffers {
  PruneInput in;                 // the [B, T, V] input rows
  const int *seq_lens;           // device copy of seq_lens, or NULL
  unsigned char *ws;             // the plan's regions (256-byte aligned)
  float *lm_arena;               // [B][arena_stride] LM term of each trie node
  int *dstate;                   // [B][arena_stride] dictionary state of each trie node
  float *lm_row;                 // character-based model: [B][arena_stride][V] rows of LM terms, else NULL
  int *lm_hist;                  // ARPA scorer: [B][arena_stride][order - 1] LM word ids of each trie node, else NULL
  DecodeOut out;                 // (scores: the raw prefix scores, which the caller rescores)
  // sweep of the LM weights (ARPA scorer): P pairs (alpha, beta) in the device table lm_ab [P][2]; the per-node arrays
  // and the outputs above then hold P x B utterances (pair-major), the input rows B
  int P = 1;
  const double *lm_ab = nullptr;
  // several models (ctcdec_decode_batch_lm_mixed_async): the device tables of the LM slots and of each utterance's
  // slot; lm_hist holds the slots' largest order - 1 ids per node
  const LmSlot *lm_slots = nullptr;
  const unsigned char *lm_slot_of = nullptr;
  int lm_hist_stride = 0;
};

// One offline scorer decode from the point where the input is on the device, enqueued on s; shared by both scorer
// entry points, which stage around it (ctcdec_decode_batch_lm_host) or not (ctcdec_decode_batch_lm_device).  Uploads
// the dictionary, prepares the pinned exchange blocks of `c`, runs the prune scan, the beam kernel (persistent with
// the per-frame host handshake, or one launch per frame with CTCDEC_LM_PER_FRAME) and enqueues the finalize kernel.
// An ARPA scorer (ctcdec_scorer_create_arpa) skips the exchange: its tables go to the device and the one beam launch
// computes the LM terms itself.  seq_lens: the host array (the handshake serves need[b] frames of utterance b).  The
// caller holds g_mu[device].
static int lm_batch_step(const ctcdec_config *cfg, const Plan &pl, HostScorer *sc, DevCache &c, int device,
                         const int32_t *seq_lens, int B, int T, const LmBuffers &io, cudaStream_t s) {
  const int K = cfg->beam_size;
  int rc = ensure_dict_on_device(sc, device);
  if (rc || (sc->ngram && (rc = ensure_ngram_on_device(sc, device)))) return rc;
  const int G = io.P * B;  // beam CTAs
  CU(cudaMemsetAsync(io.out.flags, 0, (size_t)G * 4, s));
  if ((rc = launch_prune(cfg, pl, io.in, io.seq_lens, B, T, io.ws, io.out.flags, s))) return rc;
  if (io.P > 1) {
    const long long n = (long long)(io.P - 1) * B;
    sweep_flags_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(io.out.flags, B, n);
    CU(cudaGetLastError());
  }

  BeamParams bp = beam_params(*cfg, pl, io.ws, io.seq_lens, T, io.out, T);
  flat_arenas(bp, pl, io.ws);
  bp.tile_frames = 1; bp.fresh = 1;
  attach_scorer(bp, *sc);
  bp.lm_arena = io.lm_arena; bp.dstate_arena = io.dstate; bp.lm_row = io.lm_row;
  if (sc->ngram) {
    // ARPA scorer: the beam kernel computes the LM terms itself, so ONE launch decodes the batch, with no exchange
    // blocks, host workers or handshake
    bp.lm_hist = io.lm_hist;
    bp.sweep_B = io.lm_ab ? B : 0; bp.lm_ab = io.lm_ab;
    bp.lm_slots = io.lm_slots; bp.lm_slot_of = io.lm_slot_of; bp.lm_hist_stride = io.lm_hist_stride;
    if ((rc = launch_beam(bp, pl, G, s))) return rc;
    return launch_finalize(bp, G, s);
  }
  if ((rc = prepare_exchange(c, *sc, B, nullptr, bp))) return rc;
  int *const h_newlist = (int *)c.pin[kPinNewList], *const h_upd = (int *)c.pin[kPinUpdates];
  std::vector<int> need(B);
  int tmax = 0;
  for (int b = 0; b < B; ++b) {
    need[b] = std::max(0, std::min(seq_lens ? seq_lens[b] : T, T));
    tmax = std::max(tmax, need[b]);
  }
  std::vector<TrieMirror> mirror(B);
  for (int b = 0; b < B; ++b) mirror[b].reserve((size_t)1 + (size_t)K * need[b]);
  const bool lm_timing = getenv("CTCDEC_LM_TIMING") != nullptr;
  if (getenv("CTCDEC_LM_PER_FRAME") == nullptr) {
    // ---- persistent mode (default): ONE launch decodes every utterance start to end; host workers (each owning
    // every nt-th utterance, with its own hook cache) answer each frame with the LM terms.
    const auto c0 = std::chrono::steady_clock::now();
    std::vector<TrieMirror *> mirrors(B);
    std::vector<int> answers(B);
    for (int b = 0; b < B; ++b) { mirrors[b] = &mirror[b]; answers[b] = std::max(0, need[b] - 1); }
    HandshakeStats hst;
    if ((rc = run_handshake(bp, pl, B, sc, c, answers.data(), mirrors.data(), &hst, "scorer path", s))) return rc;
    if (lm_timing)
      fprintf(stderr, "[ctcdec lm] persistent: frames %d, %u host workers, kernel+handshakes %.1f ms (%lld hook calls, %lld new nodes)\n",
              tmax, hst.workers, std::chrono::duration<double>(std::chrono::steady_clock::now() - c0).count() * 1e3,
              hst.hooks, hst.created);
  } else {
    // one frame per launch (bp.tile_frames = 1, as in persistent mode): the plan's layout, whose tile holds pl.F rows
    std::vector<int> scratch;
    double t_gpu = 0.0, t_hook = 0.0;
    long long n_hook = 0, n_new = 0;
    for (int t = 0; t < std::max(tmax, 1); ++t) {
      const auto c0 = std::chrono::steady_clock::now();
      bp.t0 = t; bp.nframes = 1; bp.fresh = (t == 0) ? 1 : 0;
      if ((rc = launch_beam(bp, pl, B, s))) return rc;
      CU(cudaStreamSynchronize(s));
      const auto c1 = std::chrono::steady_clock::now();
      for (int b = 0; b < B; ++b) {
        int *const nl = h_newlist + (size_t)b * bp.lm_nl_stride;
        n_hook += lm_after_frame(*sc, sc->cond_caches[0], mirror[b], nl, h_upd + (size_t)b * bp.lm_up_stride, scratch);
        n_new += nl[0];
      }
      const auto c2 = std::chrono::steady_clock::now();
      t_gpu += std::chrono::duration<double>(c1 - c0).count();
      t_hook += std::chrono::duration<double>(c2 - c1).count();
    }
    if (lm_timing)
      fprintf(stderr, "[ctcdec lm] frames %d: launch+copy+sync %.1f ms, host mirror+hooks %.1f ms (%lld hook calls, %lld new nodes)\n",
              tmax, t_gpu * 1e3, t_hook * 1e3, n_hook, n_new);
  }
  return launch_finalize(bp, B, s);
}

// Device scratch of a scorer decode (the caller's workspace, or the per-device cache's for ctcdec_decode_batch_lm_host):
// the plan's regions, then the per-node LM terms and dictionary states, for a character-based model the per-node rows
// of LM terms, for an ARPA scorer the per-node LM histories, and the device copy of seq_lens.
struct LmWorkspace { size_t lm_arena, dstate, rows, hist, lens, total; };
static int lm_workspace(const HostScorer *sc, const Plan &pl, int B, LmWorkspace *w) {
  size_t row_bytes = 0, hist_bytes = 0;
  int rc = lm_row_bytes(sc, pl, B, &row_bytes);
  if (rc || (rc = lm_hist_bytes(sc, pl, B, &hist_bytes))) return rc;
  const size_t node_bytes = al256((size_t)B * pl.arena_stride * 4);
  w->lm_arena = pl.total;
  w->dstate = w->lm_arena + node_bytes;
  w->rows = w->dstate + node_bytes;
  w->hist = w->rows + al256(row_bytes);
  w->lens = w->hist + al256(hist_bytes);
  w->total = w->lens + al256((size_t)B * 4);
  return CTCDEC_OK;
}

// the buffers of a scorer decode in a workspace laid out by lm_workspace (ws: its aligned start); the caller sets seq_lens
static LmBuffers lm_buffers(const HostScorer &sc, const LmWorkspace &w, unsigned char *ws, const PruneInput &in,
                            const DecodeOut &out) {
  LmBuffers io;
  io.in = in;
  io.seq_lens = nullptr;
  io.ws = ws;
  io.lm_arena = reinterpret_cast<float *>(ws + w.lm_arena);
  io.dstate = reinterpret_cast<int *>(ws + w.dstate);
  io.lm_row = sc.is_character_based ? reinterpret_cast<float *>(ws + w.rows) : nullptr;
  io.lm_hist = sc.ngram ? reinterpret_cast<int *>(ws + w.hist) : nullptr;
  io.out = out;
  return io;
}

int ctcdec_decode_batch_lm_host(const ctcdec_config *cfg, void *scorer, const float *probs, const int32_t *seq_lens,
                                int B, int T, int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                int32_t *n_results, int32_t *flags, int device) {
  if (!scorer) return fail(CTCDEC_E_INVALID, "scorer is NULL");
  const auto t_call0 = std::chrono::steady_clock::now();
  HostScorer *sc = static_cast<HostScorer *>(scorer);
  Plan pl;
  int rc = make_plan(cfg, B, T, &pl, true);
  if (rc) return rc;
  if ((int)sc->labels.size() != cfg->vocab_size) return fail(CTCDEC_E_INVALID, "scorer was built for %zu labels, decoder has %d", sc->labels.size(), cfg->vocab_size);
  if ((rc = use_device(device))) return rc;
  if (B == 0) return CTCDEC_OK;
  std::lock_guard<std::mutex> lock(g_mu[device]);
  DevCache &c = g_cache[device];
  if (!c.stream) CU(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
  cudaStream_t s = c.stream;
  const int V = cfg->vocab_size, K = cfg->beam_size;
  const size_t n_probs = (size_t)B * T * V, n_out = (size_t)B * K * T, n_bk = (size_t)B * K;
  LmWorkspace w;
  if ((rc = lm_workspace(sc, pl, B, &w))) return rc;
  if ((rc = ensure(c, kBufInput, n_probs * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufTokens, n_out * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufTimesteps, n_out * 4 + 256))) return rc;
  if ((rc = ensure(c, kBufSmall, small_bytes(B, K)))) return rc;
  if ((rc = ensure(c, kBufWork, w.total + 256))) return rc;
  float *d_probs = (float *)c.buf[kBufInput];
  int *d_tok = (int *)c.buf[kBufTokens], *d_ts = (int *)c.buf[kBufTimesteps];
  const SmallOut d = small_out(c.buf[kBufSmall], B, K);
  LmBuffers io = lm_buffers(*sc, w, align256(c.buf[kBufWork]), PruneInput{d_probs, IN_F32, nullptr, true},
                            DecodeOut{d_tok, d_ts, d.scores, d.lens, d.n_results, d.flags});
  if (n_probs) CU(cudaMemcpyAsync(d_probs, probs, n_probs * 4, cudaMemcpyHostToDevice, s));
  if (seq_lens) {
    io.seq_lens = reinterpret_cast<int *>(io.ws + w.lens);
    CU(cudaMemcpyAsync((int *)io.seq_lens, seq_lens, (size_t)B * 4, cudaMemcpyHostToDevice, s));
  }
  if ((rc = lm_batch_step(cfg, pl, sc, c, device, seq_lens, B, T, io, s))) return rc;
  const bool lm_timing = getenv("CTCDEC_LM_TIMING") != nullptr;
  const auto t_fin0 = std::chrono::steady_clock::now();
  if ((rc = ensure_pinned(c, kPinSmall, small_bytes(B, K)))) return rc;
  const SmallOut h = small_out(c.pin[kPinSmall], B, K);
  if ((rc = read_small(h, d, K, 0, B, s))) return rc;
  CU(cudaStreamSynchronize(s));
  copy_result_rows(h, B, K, nullptr, scores, lens);
  const int max_len = std::min(max_result_len(h, K, 0, B, nullptr), T);
  if (max_len > 0) {
    const size_t st_bytes = n_bk * (size_t)max_len * 8;
    const bool staged = stage_rows(tokens, timesteps, st_bytes);
    if (staged && (rc = ensure_pinned(c, kPinRows, st_bytes))) return rc;
    int32_t *const stage_tok = staged ? static_cast<int32_t *>(c.pin[kPinRows]) : nullptr;
    int32_t *const stage_ts = staged ? stage_tok + n_bk * (size_t)max_len : nullptr;
    if ((rc = enqueue_rows(d_tok, d_ts, tokens, timesteps, stage_tok, stage_ts, n_bk, max_len, T, s))) return rc;
    CU(cudaStreamSynchronize(s));
    if (staged) spread_rows(stage_tok, stage_ts, tokens, timesteps, n_bk, max_len, T);
  }
  const auto t_fin1 = std::chrono::steady_clock::now();
  lm_rescore_batch(*sc, B, K, T, h.n_results, tokens, lens, scores);  // reported scores: approx_ctc (reference :194-208)
  if (lm_timing)
    fprintf(stderr, "[ctcdec lm] finalize + copies back %.1f ms, read-out rescoring (sentence hook) %.1f ms, whole call %.1f ms\n",
            std::chrono::duration<double>(t_fin1 - t_fin0).count() * 1e3,
            std::chrono::duration<double>(std::chrono::steady_clock::now() - t_fin1).count() * 1e3,
            std::chrono::duration<double>(std::chrono::steady_clock::now() - t_call0).count() * 1e3);
  if (n_results) memcpy(n_results, h.n_results, (size_t)B * 4);
  if (flags) memcpy(flags, h.flags, (size_t)B * 4);
  return check_error_flags(h.flags, B);
}

// the checks both scorer device functions make before anything else: the scorer, the plan with a scorer, the labels
static int lm_device_plan(const ctcdec_config *cfg, const void *scorer, int B, int T, Plan *pl, LmWorkspace *w) {
  if (!scorer) return fail(CTCDEC_E_INVALID, "scorer is NULL");
  const HostScorer *sc = static_cast<const HostScorer *>(scorer);
  int rc = make_plan(cfg, B, T, pl, true);
  if (rc) return rc;
  if ((int)sc->labels.size() != cfg->vocab_size)
    return fail(CTCDEC_E_INVALID, "scorer was built for %zu labels, decoder has %d", sc->labels.size(), cfg->vocab_size);
  return lm_workspace(sc, *pl, B, w);
}

int ctcdec_lm_workspace_bytes(const ctcdec_config *cfg, const void *scorer, int B, int T, size_t *bytes) {
  Plan pl;
  LmWorkspace w;
  const int rc = lm_device_plan(cfg, scorer, B, T, &pl, &w);
  if (rc) return rc;
  if (!bytes) return fail(CTCDEC_E_INVALID, "bytes is NULL");
  *bytes = w.total + 256;
  return CTCDEC_OK;
}

// A sweep of P (alpha, beta) pairs over B utterances: the launch plan of a B-utterance decode (its block size: the
// 128- and 256-thread kernels can order comparator-equal results differently, and slice p must equal that decode bit
// for bit; with a scorer both keep two CTAs per SM), the arenas, states and per-node arrays of P x B beam CTAs, the
// pruned rows of the B input utterances (scanned once), and the device table of the pairs at w->total (*bytes: the
// whole workspace the caller provides).
static int lm_sweep_plan(const ctcdec_config *cfg, const void *scorer, int B, int T, int P, Plan *pl, LmWorkspace *w,
                         size_t *bytes) {
  if (P < 1) return fail(CTCDEC_E_INVALID, "%d (alpha, beta) pairs: a sweep needs at least one", P);
  if (B > 0 && (long long)P * B > 0x7fffffffll)
    return fail(CTCDEC_E_UNSUPPORTED, "%d pairs x batch %d: too many beam CTAs", P, B);
  if (scorer && !static_cast<const HostScorer *>(scorer)->ngram)
    return fail(CTCDEC_E_UNSUPPORTED, "a sweep takes a scorer from ctcdec_scorer_create_arpa only: a hook scorer's "
                "terms float(cond_log_prob x alpha) are computed on the host");
  int rc = lm_device_plan(cfg, scorer, B, T, pl, w);
  if (rc) return rc;
  plan_regions(pl, B, P * B, T);
  if ((rc = lm_workspace(static_cast<const HostScorer *>(scorer), *pl, P * B, w))) return rc;
  *bytes = w->total + al256((size_t)P * 16) + 256;
  return CTCDEC_OK;
}

int ctcdec_lm_sweep_workspace_bytes(const ctcdec_config *cfg, const void *scorer, int B, int T, int P, size_t *bytes) {
  Plan pl;
  LmWorkspace w;
  size_t need = 0;
  const int rc = lm_sweep_plan(cfg, scorer, B, T, P, &pl, &w, &need);
  if (rc) return rc;
  if (!bytes) return fail(CTCDEC_E_INVALID, "bytes is NULL");
  *bytes = need;
  return CTCDEC_OK;
}

// The checks the two device entries of the scorer path share once their plan is made, the current device, and the split
// of the caller's workspace (which must hold `need` bytes) into *io.  B == 0 returns CTCDEC_OK before the workspace.
static int lm_device_args(const HostScorer &sc, const LmWorkspace &w, const void *input, int kind, float *log_probs_out,
                          int B, int T, const DecodeOut &o, void *workspace, size_t workspace_bytes, size_t need,
                          int *device, LmBuffers *io) {
  if (B > 0 && (!o.n_results || !o.flags)) return fail(CTCDEC_E_INVALID, "n_results and flags device buffers are required");
  if (B > 0 && (!o.scores || !o.lens || (T > 0 && (!input || !o.tokens || !o.timesteps))))
    return fail(CTCDEC_E_INVALID, "the input or an output pointer is NULL");
  int rc = current_device(device);
  if (rc || B == 0) return rc;
  unsigned char *ws = nullptr;
  if ((rc = workspace_start(workspace, workspace_bytes, need, &ws))) return rc;
  *io = lm_buffers(sc, w, ws, PruneInput{input, kind, kind == IN_F32 ? nullptr : log_probs_out, true}, o);
  return CTCDEC_OK;
}

int ctcdec_decode_batch_lm_device(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                                  const int32_t *seq_lens, int B, int T, int32_t *tokens, int32_t *timesteps,
                                  float *scores, int32_t *lens, int32_t *n_results, int32_t *flags,
                                  float *log_probs_out, void *workspace, size_t workspace_bytes, void *stream) {
  if (!scorer) return fail(CTCDEC_E_INVALID, "scorer is NULL");
  int kind = 0;
  int rc = input_kind(dtype, true, &kind);
  if (rc) return rc;
  Plan pl;
  LmWorkspace w;
  if ((rc = lm_device_plan(cfg, scorer, B, T, &pl, &w))) return rc;
  HostScorer *sc = static_cast<HostScorer *>(scorer);
  int device = 0;
  LmBuffers io;
  if ((rc = lm_device_args(*sc, w, input, kind, log_probs_out, B, T,
                           DecodeOut{tokens, timesteps, scores, lens, n_results, flags}, workspace, workspace_bytes,
                           w.total + 256, &device, &io)) || B == 0)
    return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  // the host answers the beam kernel's per-frame handshake while the call runs: a captured graph could not replay that
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  CU(cudaStreamIsCapturing(s, &capturing));
  if (capturing != cudaStreamCaptureStatusNone)
    return fail(CTCDEC_E_UNSUPPORTED, "the scorer path cannot be captured into a CUDA graph (the host answers the beam "
                "kernel's per-frame handshake during the call)");
  const int K = cfg->beam_size;
  const size_t n_bk = (size_t)B * K;
  std::lock_guard<std::mutex> lock(g_mu[device]);
  DevCache &c = g_cache[device];
  if (seq_lens) {
    io.seq_lens = reinterpret_cast<int *>(io.ws + w.lens);
    CU(cudaMemcpyAsync((int *)io.seq_lens, seq_lens, (size_t)B * 4, cudaMemcpyHostToDevice, s));
  }
  if ((rc = lm_batch_step(cfg, pl, sc, c, device, seq_lens, B, T, io, s))) return rc;
  // Read-out: the finalize kernel wrote the rows in place; the reported scores are the reference's approx_ctc, which
  // needs the sentence hook on each row's labels, so columns [0, max_len) of the rows come to pinned staging
  if ((rc = ensure_pinned(c, kPinSmall, small_bytes(B, K)))) return rc;
  const SmallOut h = small_out(c.pin[kPinSmall], B, K);
  if ((rc = read_small(h, SmallOut{scores, lens, n_results, flags}, K, 0, B, s))) return rc;
  CU(cudaStreamSynchronize(s));
  const int max_len = std::min(max_result_len(h, K, 0, B, nullptr), T);
  static const int32_t no_rows = 0;
  const int32_t *stage_tok = &no_rows;
  if (max_len > 0) {
    if ((rc = ensure_pinned(c, kPinRows, n_bk * (size_t)max_len * 4))) return rc;
    int32_t *const st = static_cast<int32_t *>(c.pin[kPinRows]);
    CU(cudaMemcpy2DAsync(st, (size_t)max_len * 4, tokens, (size_t)T * 4, (size_t)max_len * 4, n_bk, cudaMemcpyDeviceToHost, s));
    CU(cudaStreamSynchronize(s));
    stage_tok = st;
  }
  lm_rescore_batch(*sc, B, K, max_len, h.n_results, stage_tok, h.lens, h.scores);
  // (rows p >= n_results[b] go back as they were read: the caller's values, unchanged)
  CU(cudaMemcpyAsync(scores, h.scores, n_bk * 4, cudaMemcpyHostToDevice, s));
  CU(cudaStreamSynchronize(s));
  return check_error_flags(h.flags, B);
}

// the utterances' slot indices (checked to lie in [0, S)) as bytes
static std::vector<unsigned char> lm_index_bytes(const int32_t *lm_index, int B) {
  std::vector<unsigned char> v((size_t)B);
  for (int b = 0; b < B; ++b) v[b] = (unsigned char)lm_index[b];
  return v;
}

// A decode over several models (ctcdec_decode_batch_lm_mixed_async): the host arrays of the call.
struct MixedCall {
  void *const *scorers;
  int S;
  const int32_t *lm_index;
};

// The checks of a decode over several models and its workspace: the plan of a B-utterance decode with a scorer, the
// workspace of the scorer with the largest order (*rep: its per-node histories have the stride every slot fits in),
// then the S slots and the B slot indices at w->total (*bytes: the whole workspace the caller provides).  *single: all
// scorers are one object, which decodes as ctcdec_decode_batch_lm_device_async does, in its workspace.
static int lm_mixed_plan(const ctcdec_config *cfg, void *const *scorers, int S, int B, int T, Plan *pl, LmWorkspace *w,
                         size_t *bytes, HostScorer **rep, bool *single) {
  if (!scorers) return fail(CTCDEC_E_INVALID, "scorers is NULL");
  if (S < 1 || S > kMaxLmSlots)
    return fail(CTCDEC_E_INVALID, "%d scorers: a call takes 1 to %d (CTCDEC_LM_MIXED_MAX_MODELS)", S, kMaxLmSlots);
  for (int i = 0; i < S; ++i)
    if (!scorers[i]) return fail(CTCDEC_E_INVALID, "scorers[%d] is NULL", i);
  const HostScorer *s0 = static_cast<const HostScorer *>(scorers[0]);
  *rep = static_cast<HostScorer *>(scorers[0]);
  *single = true;
  for (int i = 1; i < S; ++i) {
    HostScorer *si = static_cast<HostScorer *>(scorers[i]);
    if (si == s0) continue;
    *single = false;
    const int rc = check_scorer_pair(s0, si, "scorers", i);
    if (rc) return rc;
    if (si->max_order > (*rep)->max_order) *rep = si;
  }
  int rc = lm_device_plan(cfg, *rep, B, T, pl, w);
  if (rc) return rc;
  *bytes = *single ? w->total + 256 : w->total + al256((size_t)S * kLmSlotBytes) + al256((size_t)B) + 256;
  return CTCDEC_OK;
}

int ctcdec_lm_mixed_workspace_bytes(const ctcdec_config *cfg, void *const *scorers, int S, int B, int T,
                                    size_t *bytes) {
  Plan pl;
  LmWorkspace w;
  size_t need = 0;
  HostScorer *rep = nullptr;
  bool single = false;
  const int rc = lm_mixed_plan(cfg, scorers, S, B, T, &pl, &w, &need, &rep, &single);
  if (rc) return rc;
  if (!bytes) return fail(CTCDEC_E_INVALID, "bytes is NULL");
  *bytes = need;
  return CTCDEC_OK;
}

// ctcdec_decode_batch_lm_device_async (P = 0: the scorer's alpha and beta), ctcdec_decode_batch_lm_sweep_async (P >= 1
// host pairs: outputs [P, B, ...]) and ctcdec_decode_batch_lm_mixed_async (mx: utterance b with
// mx->scorers[mx->lm_index[b]]; scorer NULL).
static int lm_decode_async(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                           const int32_t *seq_lens, int B, int T, const double *alphas, const double *betas, int P,
                           int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens, int32_t *n_results,
                           int32_t *flags, float *log_probs_out, void *workspace, size_t workspace_bytes, void *stream,
                           const MixedCall *mx = nullptr) {
  HostScorer *rep = nullptr;
  bool single = true;
  Plan pl;
  LmWorkspace w;
  size_t need_bytes = 0;
  int rc = CTCDEC_OK;
  if (mx) {
    if ((rc = lm_mixed_plan(cfg, mx->scorers, mx->S, B, T, &pl, &w, &need_bytes, &rep, &single))) return rc;
    if (B > 0 && !mx->lm_index) return fail(CTCDEC_E_INVALID, "lm_index (host int32[B]) is NULL");
    for (int b = 0; b < B; ++b)
      if (mx->lm_index[b] < 0 || mx->lm_index[b] >= mx->S)
        return fail(CTCDEC_E_INVALID, "lm_index[%d] = %d outside [0, %d)", b, mx->lm_index[b], mx->S);
    if (single) {
      scorer = mx->scorers[0];
      mx = nullptr;
    }
  }
  if (!scorer && !mx) return fail(CTCDEC_E_INVALID, "scorer is NULL");
  int kind = 0;
  if ((rc = input_kind(dtype, true, &kind))) return rc;
  const bool sweep = P > 0;
  if (!mx) {
    rc = sweep ? lm_sweep_plan(cfg, scorer, B, T, P, &pl, &w, &need_bytes) : lm_device_plan(cfg, scorer, B, T, &pl, &w);
    if (rc) return rc;
    if (!sweep) need_bytes = w.total + 256;
  }
  HostScorer *sc = mx ? rep : static_cast<HostScorer *>(scorer);
  if (!sc->ngram)
    return fail(CTCDEC_E_UNSUPPORTED, "the asynchronous scorer decode takes a scorer from ctcdec_scorer_create_arpa only: "
                "a hook scorer needs the host during the call (use ctcdec_decode_batch_lm_device)");
  if (sweep && (!alphas || !betas)) return fail(CTCDEC_E_INVALID, "alphas and betas (host double[P]) are required");
  int device = 0;
  LmBuffers io;
  if ((rc = lm_device_args(*sc, w, input, kind, log_probs_out, B, T,
                           DecodeOut{tokens, timesteps, scores, lens, n_results, flags}, workspace, workspace_bytes,
                           need_bytes, &device, &io)) || B == 0)
    return rc;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
  CU(cudaStreamIsCapturing(s, &capturing));
  std::lock_guard<std::mutex> lock(g_mu[device]);
  // nothing that allocates, uploads or synchronises may run while the stream is captured: the scorer's tables must be
  // on this device already (the first decode puts them there)
  const int n_sc = mx ? mx->S : 1;
  for (int i = 0; i < n_sc; ++i) {
    HostScorer *si = mx ? static_cast<HostScorer *>(mx->scorers[i]) : sc;
    if (capturing != cudaStreamCaptureStatusNone &&
        !(si->d_next && si->device == device && si->d_ngram && si->ngram_device == device))
      return fail(CTCDEC_E_UNSUPPORTED, "the scorer's tables are not on device %d yet: %s", device, kCaptureFirst);
    if (mx && ((rc = ensure_dict_on_device(si, device)) || (rc = ensure_ngram_on_device(si, device)))) return rc;
  }
  struct CaptureGuard {
    explicit CaptureGuard(bool on) { g_capturing = on; }
    ~CaptureGuard() { g_capturing = false; }
  } guard(capturing != cudaStreamCaptureStatusNone);
  io.seq_lens = seq_lens;
  if (sweep) {
    // each pair through float32, as ctcdec_scorer_reset_params stores them
    double *tab = reinterpret_cast<double *>(io.ws + w.total);
    for (int p0 = 0; p0 < P; p0 += kTabPerLaunch) {
      SweepPairArgs a;
      a.tab = tab; a.p0 = p0; a.n = std::min(kTabPerLaunch, P - p0);
      for (int i = 0; i < a.n; ++i) {
        a.ab[2 * i] = (double)(float)alphas[p0 + i];
        a.ab[2 * i + 1] = (double)(float)betas[p0 + i];
      }
      sweep_pairs_kernel<<<1, kTabPerLaunch, 0, s>>>(a);
      CU(cudaGetLastError());
    }
    io.P = P; io.lm_ab = tab;
  }
  if (mx) {
    // the slots: each scorer's model with its alpha and beta as they are now
    LmSlot *const slots = reinterpret_cast<LmSlot *>(io.ws + w.total);
    unsigned char *const slot_of = io.ws + w.total + al256((size_t)mx->S * kLmSlotBytes);
    const std::vector<unsigned char> index = lm_index_bytes(mx->lm_index, B);
    if ((rc = upload_slots(reinterpret_cast<HostScorer *const *>(mx->scorers), mx->S, index.data(), B, slots, slot_of,
                           s)))
      return rc;
    io.lm_slots = slots; io.lm_slot_of = slot_of; io.lm_hist_stride = rep->max_order - 1;
  }
  // (the host lengths only serve the hook scorers' handshake: the ARPA branch of the step reads the device copy)
  if ((rc = lm_batch_step(cfg, pl, sc, g_cache[device], device, nullptr, B, T, io, s))) return rc;
  return launch_readout(sc, tokens, lens, n_results, scores, io.P * B, cfg->beam_size, T, s, io.lm_ab, B, io.lm_slots,
                        io.lm_slot_of);
}

int ctcdec_decode_batch_lm_device_async(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                                        const int32_t *seq_lens, int B, int T, int32_t *tokens, int32_t *timesteps,
                                        float *scores, int32_t *lens, int32_t *n_results, int32_t *flags,
                                        float *log_probs_out, void *workspace, size_t workspace_bytes, void *stream) {
  return lm_decode_async(cfg, scorer, input, dtype, seq_lens, B, T, nullptr, nullptr, 0, tokens, timesteps, scores,
                         lens, n_results, flags, log_probs_out, workspace, workspace_bytes, stream);
}

int ctcdec_decode_batch_lm_sweep_async(const ctcdec_config *cfg, void *scorer, const void *input, int dtype,
                                       const int32_t *seq_lens, int B, int T, const double *alphas,
                                       const double *betas, int P, int32_t *tokens, int32_t *timesteps, float *scores,
                                       int32_t *lens, int32_t *n_results, int32_t *flags, float *log_probs_out,
                                       void *workspace, size_t workspace_bytes, void *stream) {
  if (P < 1) return fail(CTCDEC_E_INVALID, "%d (alpha, beta) pairs: a sweep needs at least one", P);
  return lm_decode_async(cfg, scorer, input, dtype, seq_lens, B, T, alphas, betas, P, tokens, timesteps, scores, lens,
                         n_results, flags, log_probs_out, workspace, workspace_bytes, stream);
}

int ctcdec_decode_batch_lm_mixed_async(const ctcdec_config *cfg, void *const *scorers, int S, const int32_t *lm_index,
                                       const void *input, int dtype, const int32_t *seq_lens, int B, int T,
                                       int32_t *tokens, int32_t *timesteps, float *scores, int32_t *lens,
                                       int32_t *n_results, int32_t *flags, float *log_probs_out, void *workspace,
                                       size_t workspace_bytes, void *stream) {
  const MixedCall mx{scorers, S, lm_index};
  return lm_decode_async(cfg, nullptr, input, dtype, seq_lens, B, T, nullptr, nullptr, 0, tokens, timesteps, scores,
                         lens, n_results, flags, log_probs_out, workspace, workspace_bytes, stream, &mx);
}

// Diagnostic: the read-out of [B, K] host rows, on the host (lm_rescore_batch through the scorer's hooks) or by the
// read-out kernel on `device` (ARPA scorers).
int ctcdec_scorer_rescore_rows(void *scorer, const int32_t *tokens, const int32_t *lens, const int32_t *n_results,
                               float *scores, int B, int K, int row_stride, int device) {
  if (!scorer) return fail(CTCDEC_E_INVALID, "scorer is NULL");
  if (B < 0 || K < 1 || row_stride < 0) return fail(CTCDEC_E_INVALID, "bad shape B=%d K=%d row_stride=%d", B, K, row_stride);
  if (B > 0 && (!lens || !n_results || !scores || (row_stride > 0 && !tokens)))
    return fail(CTCDEC_E_INVALID, "NULL argument");
  HostScorer *sc = static_cast<HostScorer *>(scorer);
  const int V = (int)sc->labels.size();
  for (int b = 0; b < B; ++b)
    for (int p = 0; p < n_results[b] && p < K; ++p) {
      const size_t r = (size_t)b * K + p;
      if (lens[r] < 0 || lens[r] > row_stride)
        return fail(CTCDEC_E_INVALID, "row (%d, %d): length %d outside [0, %d]", b, p, lens[r], row_stride);
      for (int i = 0; i < lens[r]; ++i)
        if (tokens[r * row_stride + i] < 0 || tokens[r * row_stride + i] >= V)
          return fail(CTCDEC_E_INVALID, "row (%d, %d): label %d outside [0, %d)", b, p, tokens[r * row_stride + i], V);
    }
  if (device < 0) {
    lm_rescore_batch(*sc, B, K, row_stride, n_results, tokens, lens, scores);
    return CTCDEC_OK;
  }
  if (!sc->ngram) return fail(CTCDEC_E_UNSUPPORTED, "the read-out kernel takes a scorer from ctcdec_scorer_create_arpa only");
  int rc = use_device(device);
  if (rc) return rc;
  if (B == 0) return CTCDEC_OK;
  std::lock_guard<std::mutex> lock(g_mu[device]);
  if ((rc = ensure_ngram_on_device(sc, device))) return rc;
  const size_t rows = (size_t)B * K, tok_bytes = rows * row_stride * 4;
  unsigned char *d = nullptr;
  const size_t o_lens = al256(tok_bytes), o_nres = o_lens + al256(rows * 4), o_sc = o_nres + al256((size_t)B * 4);
  CU(cudaMalloc(&d, o_sc + rows * 4));
  std::unique_ptr<unsigned char, decltype(&cudaFree)> hold(d, &cudaFree);
  if (tok_bytes) CU(cudaMemcpy(d, tokens, tok_bytes, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d + o_lens, lens, rows * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d + o_nres, n_results, (size_t)B * 4, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d + o_sc, scores, rows * 4, cudaMemcpyHostToDevice));
  if ((rc = launch_readout(sc, reinterpret_cast<int32_t *>(d), reinterpret_cast<int32_t *>(d + o_lens),
                           reinterpret_cast<int32_t *>(d + o_nres), reinterpret_cast<float *>(d + o_sc), B, K,
                           row_stride, nullptr)))
    return rc;
  CU(cudaMemcpy(scores, d + o_sc, rows * 4, cudaMemcpyDeviceToHost));
  return CTCDEC_OK;
}

int ctcdec_rows_to_host(const int32_t *d_tokens, const int32_t *d_timesteps, long long rows, int row_stride, int max_len,
                        int32_t *tokens, int32_t *timesteps, void *stream) {
  if (rows < 0 || row_stride < 0 || max_len < 0 || max_len > row_stride) return fail(CTCDEC_E_INVALID, "bad rows / row_stride / max_len");
  if (rows == 0 || max_len == 0) return CTCDEC_OK;
  if (!d_tokens || !d_timesteps || !tokens || !timesteps) return fail(CTCDEC_E_INVALID, "NULL pointer");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t pitch = (size_t)row_stride * 4, width = (size_t)max_len * 4;
  CU(cudaMemcpy2DAsync(tokens, pitch, d_tokens, pitch, width, (size_t)rows, cudaMemcpyDeviceToHost, s));
  CU(cudaMemcpy2DAsync(timesteps, pitch, d_timesteps, pitch, width, (size_t)rows, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return CTCDEC_OK;
}

int ctcdec_selftest_math_f64(int which, const double *x, const double *x2, double *y, size_t n, int device) {
  if (which < 0 || which > 2 || !x || !y || (which == 2 && !x2)) return fail(CTCDEC_E_INVALID, "bad selftest arguments");
  int rc = use_device(device);
  if (rc) return rc;
  if (n == 0) return CTCDEC_OK;
  double *dx = nullptr, *dx2 = nullptr, *dy = nullptr;
  CU(cudaMalloc(&dx, n * 8));
  CU(cudaMalloc(&dy, n * 8));
  if (which == 2) CU(cudaMalloc(&dx2, n * 8));
  CU(cudaMemcpy(dx, x, n * 8, cudaMemcpyHostToDevice));
  if (which == 2) CU(cudaMemcpy(dx2, x2, n * 8, cudaMemcpyHostToDevice));
  selftest_math_f64_kernel<<<kNumSMs * 8, 256>>>(which, dx, dx2, dy, n);
  CU(cudaGetLastError());
  CU(cudaMemcpy(y, dy, n * 8, cudaMemcpyDeviceToHost));
  cudaFree(dx); cudaFree(dy);
  if (dx2) cudaFree(dx2);
  return CTCDEC_OK;
}

int ctcdec_selftest_math(int which, const float *x, const float *x2, float *y, size_t n, int device) {
  if (which < 0 || which > 3 || !x || !y || (which == 3 && !x2)) return fail(CTCDEC_E_INVALID, "bad selftest arguments");
  int rc = use_device(device);
  if (rc) return rc;
  if (n == 0) return CTCDEC_OK;
  float *dx = nullptr, *dx2 = nullptr, *dy = nullptr;
  CU(cudaMalloc(&dx, n * 4));
  CU(cudaMalloc(&dy, n * 4));
  if (which == 3) CU(cudaMalloc(&dx2, n * 4));
  CU(cudaMemcpy(dx, x, n * 4, cudaMemcpyHostToDevice));
  if (which == 3) CU(cudaMemcpy(dx2, x2, n * 4, cudaMemcpyHostToDevice));
  selftest_math_kernel<<<kNumSMs * 8, 256>>>(which, dx, dx2, dy, n);
  CU(cudaGetLastError());
  CU(cudaMemcpy(y, dy, n * 4, cudaMemcpyDeviceToHost));
  cudaFree(dx); cudaFree(dy);
  if (dx2) cudaFree(dx2);
  return CTCDEC_OK;
}

}  // extern "C"

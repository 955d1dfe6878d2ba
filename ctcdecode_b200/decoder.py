"""Host-side mirror of the reference's Python interface for the beam-search path.

Same class names, constructor arguments, argument meaning and return tuple as the reference's
``ctcdecode/__init__.py`` (CTCBeamDecoder :6-140, OnlineCTCBeamDecoder :143-250, DecoderState :253-272), so
``decoder.decode(output)`` keeps working; the work itself goes through the C ABI of
include/ctcdecode_b200.h into the sm_90a kernels.  There is no CPU fallback: without the CUDA library or
without an H100 the calls raise.

Differences from the reference, all additive:
  * ``probs`` may live on the GPU; it is then decoded in place, with or without a scorer (the reference does
    ``probs.cpu()`` first, __init__.py:77).  Results are CPU tensors like the reference's unless
    ``device_outputs=True``.  ``decode_logits`` takes the acoustic model's raw logits instead, also with a scorer.
  * ``num_processes`` is accepted and ignored: the batch is a CUDA grid (one CTA per utterance).
  * ``decoder.last_flags`` / ``decoder.last_n_results`` expose the per-utterance tie flags and beam counts
    of the last call (the reference has no equivalent; see include/ctcdecode_b200.h).
  * ``model_path`` (word-based KenLM models): the language model stays on the host behind a hook; the real Scorer
    comes from a provider library (``scorer_provider=`` / CTCDECODE_B200_SCORER_PROVIDER, see scorer.py and
    INTEGRATION.md; providers/ builds one from the reference's own Scorer + KenLM).  ``scorer_provider="device"``
    needs no provider: the library reads the ARPA or KenLM binary file itself (REST_PROBING binaries excepted) and
    reproduces the reference Scorer bit for bit.  CUDA probabilities and logits
    stay on the GPU with a scorer too (ctcdec_decode_batch_lm_device); that call returns when the results are in place,
    because the host answers the beam kernel's per-frame LM handshake while it runs.  The online decoder takes a
    scorer too (device-resident states, one persistent launch per chunk).  Character-based models are detected like
    the reference does (every word of the model is one UTF-8 character) and decoded without a dictionary.
  * ``non_blocking=True`` (with ``device_outputs=True``, and ``scorer_provider="device"`` when there is a language
    model): a CUDA decode with the device scorer is only enqueued on the current stream, read-out rescoring included
    (ctcdec_decode_batch_lm_device_async / ctcdec_decode_stream_device), so it can run behind the acoustic model and
    be captured into a CUDA graph (decode once before capturing; a graph replays the alpha / beta it captured).  The
    call may return before the results exist, and a kernel error shows only as CTCDEC_FLAG_ERR_ARENA in
    ``last_flags``, a CUDA tensor.  ``OnlineCTCBeamDecoder`` then decodes CUDA chunks and ``decode_logits`` with the
    device scorer on the GPU as well.
  * ``decode_sweep(x, alphas, betas)`` (device scorer): one batch under P (alpha, beta) pairs in one enqueue, results
    with a leading pair axis, each slice equal to ``decode`` after ``reset_params`` with that pair.
  * ``decode_mixed(x, lm_index, decoders)`` (device scorer): one batch whose utterances need different language models
    (per customer, domain or language) in one enqueue: utterance b is decoded with the model and weights of
    ``decoders[lm_index[b]]``, bit for bit as that decoder's ``decode`` gives it; up to 16 models, all word-based or all
    character-based, built for the same labels.
  * the [batch, beam, T] result tensors are PAGE-LOCKED CPU tensors (torch's caching host allocator, so a decode loop
    reuses the same blocks) up to CTCDECODE_B200_PIN_OUTPUT_BYTES per tensor (default 1 GiB), pageable beyond: a fresh
    pageable [256, 100, 1000] int32 pair costs page faults on every call, several times the decode itself.
  * ``OnlineCTCBeamDecoder.decode`` / ``decode_logits`` take ``DecoderState``s of different device-scorer decoders
    (``scorer_provider="device"``, same configuration and labels, up to 16 models) in one call, as the reference's
    ``decode`` takes states of different decoders: each stream decodes with its own decoder's model and weights.
  * ``OnlineCTCBeamDecoder``: CUDA chunks (without a scorer, or with ``non_blocking=True``) are decoded in place on the
    current stream, raw logits go
    through ``decode_logits``, ``device_outputs=True`` leaves the results on the GPU, and ``committed_prefix`` reports
    the part of each stream's transcript no later chunk can change.
  * ``device="all"`` (or no device and a CPU batch of more than 4 x 132 utterances on a multi-GPU box): the host batch
    is sharded over every visible GPU by one call (ctcdec_decode_batch_host_multi).
"""
import ctypes
import os

import torch

from . import _native

_PIN_CAP = int(os.environ.get("CTCDECODE_B200_PIN_OUTPUT_BYTES", str(1 << 30)))


def _host_empty(*shape, dtype=torch.int32):
    """Uninitialised CPU result tensor: page-locked when it is big enough to matter and small enough to afford (the
    rows then arrive by DMA straight from the GPU, and torch's caching host allocator recycles the block in a loop)."""
    n = torch.empty(0, dtype=dtype).element_size()
    for d in shape:
        n *= int(d)
    if (1 << 16) <= n <= _PIN_CAP and torch.cuda.is_available():
        try:
            return torch.empty(*shape, dtype=dtype, pin_memory=True)
        except RuntimeError:
            pass
    return torch.empty(*shape, dtype=dtype)


def convert_to_string(tokens, vocabulary, seq_len):
    """Label ids -> text for one beam: the helper the reference's README suggests callers write themselves
    (README.md:99-109), e.g. convert_to_string(beam_results[0][0], labels, out_lens[0][0])."""
    n = int(seq_len)
    return "".join(vocabulary[int(x)] for x in tokens[:n])


def _cfg(decoder):
    return _native.Config(decoder._num_labels, decoder._beam_width, decoder._blank_id, decoder._log_probs,
                          decoder._cutoff_top_n_value(), float(decoder._cutoff_prob))


class _Base(object):
    def _init_common(self, labels, model_path, alpha, beta, cutoff_top_n, cutoff_prob, beam_width, num_processes,
                     blank_id, log_probs_input, device, scorer_provider=None, non_blocking=False):
        if non_blocking and not self._device_outputs:
            raise ValueError("non_blocking=True needs device_outputs=True: the results stay on the GPU")
        if non_blocking and model_path and \
                (scorer_provider or os.environ.get("CTCDECODE_B200_SCORER_PROVIDER")) != "device":
            raise ValueError('non_blocking=True with a language model needs scorer_provider="device": a hook scorer '
                             "answers the decode on the host")
        self._non_blocking = bool(non_blocking)
        self._beam_width = int(beam_width)
        self._scorer = None
        self._num_processes = num_processes
        self._labels = list(labels)
        self._num_labels = len(self._labels)
        self._blank_id = int(blank_id)
        self._log_probs = 1 if log_probs_input else 0
        self._cutoff_prob = cutoff_prob
        self._device = device
        self.last_flags = None
        self.last_n_results = None
        _native.load()
        if model_path:
            from .scorer import make_scorer
            self._scorer = make_scorer(self._labels, model_path, alpha, beta, scorer_provider)

    def _device_index(self, probs=None):
        if probs is not None and probs.is_cuda:
            return probs.device.index if probs.device.index is not None else torch.cuda.current_device()
        if self._device is not None and self._device != "all":
            return torch.device(self._device).index or 0
        return 0

    def _use_all_gpus(self, B):
        """CPU input: device="all" spreads the batch over every visible GPU; with no device given that happens once
        the batch is more than two waves of one GPU (> 4 x 132 utterances, 132 SMs) and there is more than one GPU."""
        if self._device == "all":
            return torch.cuda.device_count() > 1
        return self._device is None and B > 4 * 132 and torch.cuda.device_count() > 1

    def character_based(self):
        return self._scorer.is_character_based() if self._scorer else None

    def max_order(self):
        return self._scorer.max_order() if self._scorer else None

    def dict_size(self):
        return self._scorer.dict_size() if self._scorer else None


class CTCBeamDecoder(_Base):
    """Drop-in for the reference CTCBeamDecoder (reference ctcdecode/__init__.py:6-140)."""

    def __init__(self, labels, model_path=None, alpha=0, beta=0, cutoff_top_n=40, cutoff_prob=1.0, beam_width=100,
                 num_processes=4, blank_id=0, log_probs_input=False, device=None, device_outputs=False,
                 scorer_provider=None, non_blocking=False):
        self.cutoff_top_n = cutoff_top_n  # public attribute name kept from the reference (:39)
        self._device_outputs = device_outputs
        self._ws = None
        self._init_common(labels, model_path, alpha, beta, cutoff_top_n, cutoff_prob, beam_width, num_processes,
                          blank_id, log_probs_input, device, scorer_provider, non_blocking)

    def _cutoff_top_n_value(self):
        return int(self.cutoff_top_n)

    def decode(self, probs, seq_lens=None):
        """probs: [B, T, V] float tensor (CPU or CUDA); seq_lens: optional [B] ints.
        Returns (beam_results [B, beam, T] int32, beam_scores [B, beam] float32, timesteps [B, beam, T] int32,
        out_lens [B, beam] int32) exactly like reference __init__.py:53-123: only [b, p, :out_lens[b, p]] of
        beam_results / timesteps is meaningful, the rest is uninitialised."""
        lib = _native.load()
        if probs.dim() != 3:
            raise ValueError("probs must be [batch, time, labels], got %s" % (tuple(probs.shape),))
        B, T, V = probs.shape
        if V != self._num_labels:
            raise ValueError("probs has %d labels, decoder was built with %d" % (V, self._num_labels))
        cfg = _cfg(self)
        K = self._beam_width
        if probs.is_cuda:
            return self._decode_device(lib, cfg, probs, seq_lens, B, T, K)
        dev_index = self._device_index(probs)
        probs = probs.cpu().float().contiguous()
        if seq_lens is not None:
            seq_lens = seq_lens.cpu().int().contiguous()
        output = _host_empty(B, K, T)
        timesteps = _host_empty(B, K, T)
        scores = torch.empty(B, K, dtype=torch.float32)
        out_seq_len = torch.zeros(B, K, dtype=torch.int32)
        n_results = torch.zeros(B, dtype=torch.int32)
        flags = torch.zeros(B, dtype=torch.int32)
        if self._scorer is not None:  # reference __init__.py:87-104 paddle_beam_decode_lm
            _native.check(lib.ctcdec_decode_batch_lm_host(
                ctypes.byref(cfg), self._scorer.handle, probs.data_ptr(),
                seq_lens.data_ptr() if seq_lens is not None else None, B, T, output.data_ptr(), timesteps.data_ptr(),
                scores.data_ptr(), out_seq_len.data_ptr(), n_results.data_ptr(), flags.data_ptr(), dev_index))
        elif self._use_all_gpus(B):
            # one host batch over every GPU of the box (contiguous shards, a worker thread per device, nothing
            # crosses between GPUs): the reference's ThreadPool fan-out over utterances at box scale
            _native.check(lib.ctcdec_decode_batch_host_multi(
                ctypes.byref(cfg), probs.data_ptr(), seq_lens.data_ptr() if seq_lens is not None else None, B, T,
                output.data_ptr(), timesteps.data_ptr(), scores.data_ptr(), out_seq_len.data_ptr(),
                n_results.data_ptr(), flags.data_ptr(), None, 0))
        else:
            _native.check(lib.ctcdec_decode_batch_host(
                ctypes.byref(cfg), probs.data_ptr(), seq_lens.data_ptr() if seq_lens is not None else None, B, T,
                output.data_ptr(), timesteps.data_ptr(), scores.data_ptr(), out_seq_len.data_ptr(),
                n_results.data_ptr(), flags.data_ptr(), dev_index))
        self.last_flags, self.last_n_results = flags, n_results
        return output, scores, timesteps, out_seq_len

    def decode_logits(self, logits, seq_lens=None, return_log_probs=False):
        """Extension (SURVEY.md section 8f row 3, "the step before"): decode the acoustic model's raw LOGITS, a CUDA
        tensor [B, T, V] in float32 / float16 / bfloat16, without the caller-side softmax the reference asks for
        (README.md:54-57): the scan kernel computes each frame's float32 log-softmax on the fly and decodes as with
        log_probs_input=True.  Returns the usual four tensors, plus -- with return_log_probs -- the float32
        log-softmax the decode used (feeding that to the reference with log_probs_input=True reproduces the result
        bit for bit).  With a scorer the language model is applied as in decode (the call then waits for the device)."""
        lib = _native.load()
        if logits.dim() != 3 or not logits.is_cuda:
            raise ValueError("logits must be a CUDA tensor [batch, time, labels]")
        dtypes = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
        if logits.dtype not in dtypes:
            raise ValueError("logits must be float32, float16 or bfloat16, got %s" % logits.dtype)
        B, T, V = logits.shape
        if V != self._num_labels:
            raise ValueError("logits has %d labels, decoder was built with %d" % (V, self._num_labels))
        lsm = torch.empty(B, T, V, dtype=torch.float32, device=logits.device) if return_log_probs else None
        res = self._decode_device(lib, _cfg(self), logits.contiguous(), seq_lens, B, T, self._beam_width,
                                  logits_dtype=dtypes[logits.dtype], lsm_out=lsm)
        return res + (lsm,) if return_log_probs else res

    def pack_results(self, beam_results, timesteps, out_lens, n_results=None):
        """Extension (SURVEY.md section 8f row 4, "the step after"): compact dense CUDA results [B, beam, T] (from a
        decoder built with device_outputs=True) into a ragged layout on the device.  Returns (offsets int64
        [B * beam + 1], tokens int32 [total], timesteps int32 [total]); row r = b * beam + p is
        tokens[offsets[r]:offsets[r + 1]].  n_results defaults to the last decode's."""
        lib = _native.load()
        if not (beam_results.is_cuda and timesteps.is_cuda and out_lens.is_cuda):
            raise ValueError("pack_results takes the CUDA tensors of a device_outputs=True decode")
        n_results = self.last_n_results if n_results is None else n_results
        dev = beam_results.device
        n_results = n_results.to(device=dev, dtype=torch.int32).contiguous()
        B, K, T = beam_results.shape
        beam_results, timesteps, out_lens = beam_results.contiguous(), timesteps.contiguous(), out_lens.contiguous()
        offsets = torch.empty(B * K + 1, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(lib.ctcdec_pack_results_device(
                beam_results.data_ptr(), timesteps.data_ptr(), out_lens.data_ptr(), n_results.data_ptr(), B, K, T,
                offsets.data_ptr(), None, None, 0, stream))
            total = int(offsets[-1])
            tok = torch.empty(total, dtype=torch.int32, device=dev)
            ts = torch.empty(total, dtype=torch.int32, device=dev)
            _native.check(lib.ctcdec_pack_results_device(
                beam_results.data_ptr(), timesteps.data_ptr(), out_lens.data_ptr(), n_results.data_ptr(), B, K, T,
                offsets.data_ptr(), tok.data_ptr(), ts.data_ptr(), total, stream))
        return offsets, tok, ts

    def _decode_device(self, lib, cfg, probs, seq_lens, B, T, K, logits_dtype=None, lsm_out=None):
        dev = probs.device
        scorer = self._scorer.handle if self._scorer is not None else None
        if logits_dtype is None:
            probs = probs.float().contiguous()
        lm_async = scorer and self._non_blocking
        if seq_lens is not None:
            # (the blocking scorer path answers every utterance's per-frame handshake on the host: its lengths stay there)
            seq_lens = seq_lens.to(device="cpu" if scorer and not lm_async else dev, dtype=torch.int32).contiguous()
        nbytes = ctypes.c_size_t(0)
        if scorer:
            _native.check(lib.ctcdec_lm_workspace_bytes(ctypes.byref(cfg), scorer, B, T, ctypes.byref(nbytes)))
        else:
            _native.check(lib.ctcdec_workspace_bytes(ctypes.byref(cfg), B, T, ctypes.byref(nbytes)))
        if self._ws is None or self._ws.numel() < nbytes.value or self._ws.device != dev:
            self._ws = None
            self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        output = torch.empty(B, K, T, dtype=torch.int32, device=dev)
        timesteps = torch.empty(B, K, T, dtype=torch.int32, device=dev)
        scores = torch.empty(B, K, dtype=torch.float32, device=dev)
        out_seq_len = torch.zeros(B, K, dtype=torch.int32, device=dev)
        n_results = torch.zeros(B, dtype=torch.int32, device=dev)
        flags = torch.zeros(B, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            if scorer:
                # blocking: returns when the results are in place (the host serves a hook scorer during the call and
                # rescores the results); non_blocking: enqueued on the stream, read-out included
                fn = lib.ctcdec_decode_batch_lm_device_async if lm_async else lib.ctcdec_decode_batch_lm_device
                _native.check(fn(
                    ctypes.byref(cfg), scorer, probs.data_ptr(), -1 if logits_dtype is None else logits_dtype,
                    seq_lens.data_ptr() if seq_lens is not None else None, B, T, output.data_ptr(),
                    timesteps.data_ptr(), scores.data_ptr(), out_seq_len.data_ptr(), n_results.data_ptr(),
                    flags.data_ptr(), lsm_out.data_ptr() if lsm_out is not None else None, self._ws.data_ptr(),
                    self._ws.numel(), stream))
            elif logits_dtype is None:
                _native.check(lib.ctcdec_decode_batch_device(
                    ctypes.byref(cfg), probs.data_ptr(), seq_lens.data_ptr() if seq_lens is not None else None, B, T,
                    output.data_ptr(), timesteps.data_ptr(), scores.data_ptr(), out_seq_len.data_ptr(),
                    n_results.data_ptr(), flags.data_ptr(), self._ws.data_ptr(), self._ws.numel(), stream))
            else:
                _native.check(lib.ctcdec_decode_batch_device_logits(
                    ctypes.byref(cfg), probs.data_ptr(), logits_dtype,
                    seq_lens.data_ptr() if seq_lens is not None else None, B, T, output.data_ptr(),
                    timesteps.data_ptr(), scores.data_ptr(), out_seq_len.data_ptr(), n_results.data_ptr(),
                    flags.data_ptr(), lsm_out.data_ptr() if lsm_out is not None else None, self._ws.data_ptr(),
                    self._ws.numel(), stream))
        self.last_flags, self.last_n_results = flags, n_results
        if self._device_outputs:
            return output, scores, timesteps, out_seq_len
        # reference semantics: CPU tensors.  Only columns < max(out_lens) carry data.
        lens_cpu = out_seq_len.cpu()
        max_len = int(lens_cpu.max()) if lens_cpu.numel() else 0
        out_cpu = _host_empty(B, K, T)
        ts_cpu = _host_empty(B, K, T)
        if max_len > 0:  # two strided DMA copies straight into the result tensors
            with torch.cuda.device(dev):
                _native.check(lib.ctcdec_rows_to_host(output.data_ptr(), timesteps.data_ptr(), B * K, T, max_len,
                                                      out_cpu.data_ptr(), ts_cpu.data_ptr(),
                                                      torch.cuda.current_stream(dev).cuda_stream))
        self.last_flags, self.last_n_results = flags.cpu(), n_results.cpu()
        return out_cpu, scores.cpu(), ts_cpu, lens_cpu

    def reset_params(self, alpha, beta):
        if self._scorer is not None:  # reference __init__.py:134-136
            self._scorer.reset_params(alpha, beta)

    def decode_sweep(self, x, alphas, betas, seq_lens=None, logits=False):
        """Extension: decode one batch under P language-model weight pairs (alphas[p], betas[p]) in one enqueue
        (ctcdec_decode_batch_lm_sweep_async), e.g. to tune alpha and beta on a dev set; a grid is the caller's
        itertools.product.  x: [B, T, V] probabilities (log-probabilities with log_probs_input), CPU or CUDA, or with
        logits=True raw float32 / float16 / bfloat16 CUDA logits as in decode_logits.  Returns the four tensors of
        decode with a leading pair axis -- beam_results / timesteps [P, B, beam, T], beam_scores / out_lens [P, B, beam]
        -- and sets last_flags / last_n_results [P, B].  Slice p equals decode after reset_params(alphas[p], betas[p])
        (both rounded to float32, as reset_params does); the decoder's own alpha and beta stay as they are.  CPU input
        is uploaded and the call waits; CUDA input follows device_outputs / non_blocking as decode does.  Needs the
        device scorer (scorer_provider="device")."""
        from .scorer import ArpaScorer
        if not isinstance(self._scorer, ArpaScorer):
            raise ValueError('decode_sweep needs a language model with scorer_provider="device": the sweep runs the '
                             "device n-gram scorer")
        alphas = [float(a) for a in alphas]
        betas = [float(b) for b in betas]
        if len(alphas) != len(betas) or not alphas:
            raise ValueError("alphas and betas must be non-empty and of equal length, got %d and %d"
                             % (len(alphas), len(betas)))
        if x.dim() != 3:
            raise ValueError("x must be [batch, time, labels], got %s" % (tuple(x.shape),))
        B, T, V = x.shape
        if V != self._num_labels:
            raise ValueError("x has %d labels, decoder was built with %d" % (V, self._num_labels))
        dtype = -1
        if logits:
            dtypes = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
            if not x.is_cuda or x.dtype not in dtypes:
                raise ValueError("logits must be a float32, float16 or bfloat16 CUDA tensor")
            dtype = dtypes[x.dtype]
            x = x.contiguous()
        host = not x.is_cuda
        dev = x.device if not host else torch.device("cuda", self._device_index())
        if dtype == -1:
            x = x.to(device=dev, dtype=torch.float32).contiguous()
        if seq_lens is not None:
            seq_lens = seq_lens.to(device=dev, dtype=torch.int32).contiguous()
        lib = _native.load()
        cfg = _cfg(self)
        K, P = self._beam_width, len(alphas)
        scorer = self._scorer.handle
        nbytes = ctypes.c_size_t(0)
        _native.check(lib.ctcdec_lm_sweep_workspace_bytes(ctypes.byref(cfg), scorer, B, T, P, ctypes.byref(nbytes)))
        if self._ws is None or self._ws.numel() < nbytes.value or self._ws.device != dev:
            self._ws = None
            self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        output = torch.empty(P, B, K, T, dtype=torch.int32, device=dev)
        timesteps = torch.empty(P, B, K, T, dtype=torch.int32, device=dev)
        scores = torch.empty(P, B, K, dtype=torch.float32, device=dev)
        out_seq_len = torch.zeros(P, B, K, dtype=torch.int32, device=dev)
        n_results = torch.zeros(P, B, dtype=torch.int32, device=dev)
        flags = torch.zeros(P, B, dtype=torch.int32, device=dev)
        a = (ctypes.c_double * P)(*alphas)
        b = (ctypes.c_double * P)(*betas)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(lib.ctcdec_decode_batch_lm_sweep_async(
                ctypes.byref(cfg), scorer, x.data_ptr(), dtype, seq_lens.data_ptr() if seq_lens is not None else None,
                B, T, a, b, P, output.data_ptr(), timesteps.data_ptr(), scores.data_ptr(), out_seq_len.data_ptr(),
                n_results.data_ptr(), flags.data_ptr(), None, self._ws.data_ptr(), self._ws.numel(), stream))
        self.last_flags, self.last_n_results = flags, n_results
        if self._device_outputs and not host:
            if not self._non_blocking:
                torch.cuda.current_stream(dev).synchronize()
                self._check_flags(flags)
            return output, scores, timesteps, out_seq_len
        torch.cuda.current_stream(dev).synchronize()
        self._check_flags(flags)
        self.last_flags, self.last_n_results = flags.cpu(), n_results.cpu()
        return output.cpu(), scores.cpu(), timesteps.cpu(), out_seq_len.cpu()

    def decode_mixed(self, x, lm_index, decoders, seq_lens=None, logits=False):
        """Extension: decode one batch whose utterances need different language models in one enqueue
        (ctcdec_decode_batch_lm_mixed_async): utterance b with the model and weights of decoders[lm_index[b]], each a
        CTCBeamDecoder built with scorer_provider="device" (ARPA text or a KenLM binary; order, layout, alpha and beta may
        differ), all word-based or all character-based and built for this decoder's labels.  At most
        CTCDEC_LM_MIXED_MAX_MODELS (16) decoders.  This decoder's configuration (beam, cut, blank, log input) applies
        to the whole batch.  x and seq_lens as in decode_sweep: [B, T, V] probabilities, CPU or CUDA, or with
        logits=True raw float32 / float16 / bfloat16 CUDA logits.  Returns decode's four tensors and sets last_flags /
        last_n_results; utterance b's results equal decoders[lm_index[b]].decode's (with this configuration) bit for
        bit.  CPU input is uploaded and the call waits; CUDA input follows device_outputs / non_blocking as decode."""
        from .scorer import ArpaScorer
        decoders = list(decoders)
        if not decoders:
            raise ValueError("decoders must not be empty")
        for i, d in enumerate(decoders):
            if not isinstance(getattr(d, "_scorer", None), ArpaScorer):
                raise ValueError('decoders[%d] has no language model with scorer_provider="device": a mixed decode '
                                 "runs the device n-gram scorer" % i)
            if list(d._labels) != self._labels:
                raise ValueError("decoders[%d] was built for other labels than this decoder" % i)
        if x.dim() != 3:
            raise ValueError("x must be [batch, time, labels], got %s" % (tuple(x.shape),))
        B, T, V = x.shape
        if V != self._num_labels:
            raise ValueError("x has %d labels, decoder was built with %d" % (V, self._num_labels))
        lm_index = torch.as_tensor(lm_index).to(device="cpu", dtype=torch.int32).contiguous()
        if lm_index.shape != (B,):
            raise ValueError("lm_index must be [batch], got %s" % (tuple(lm_index.shape),))
        dtype = -1
        if logits:
            dtypes = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
            if not x.is_cuda or x.dtype not in dtypes:
                raise ValueError("logits must be a float32, float16 or bfloat16 CUDA tensor")
            dtype = dtypes[x.dtype]
            x = x.contiguous()
        host = not x.is_cuda
        dev = x.device if not host else torch.device("cuda", self._device_index())
        if dtype == -1:
            x = x.to(device=dev, dtype=torch.float32).contiguous()
        if seq_lens is not None:
            seq_lens = seq_lens.to(device=dev, dtype=torch.int32).contiguous()
        lib = _native.load()
        cfg = _cfg(self)
        K, S = self._beam_width, len(decoders)
        scorers = (ctypes.c_void_p * S)(*[d._scorer.handle for d in decoders])
        nbytes = ctypes.c_size_t(0)
        _native.check(lib.ctcdec_lm_mixed_workspace_bytes(ctypes.byref(cfg), scorers, S, B, T, ctypes.byref(nbytes)))
        if self._ws is None or self._ws.numel() < nbytes.value or self._ws.device != dev:
            self._ws = None
            self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        output = torch.empty(B, K, T, dtype=torch.int32, device=dev)
        timesteps = torch.empty(B, K, T, dtype=torch.int32, device=dev)
        scores = torch.empty(B, K, dtype=torch.float32, device=dev)
        out_seq_len = torch.zeros(B, K, dtype=torch.int32, device=dev)
        n_results = torch.zeros(B, dtype=torch.int32, device=dev)
        flags = torch.zeros(B, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(lib.ctcdec_decode_batch_lm_mixed_async(
                ctypes.byref(cfg), scorers, S, lm_index.data_ptr(), x.data_ptr(), dtype,
                seq_lens.data_ptr() if seq_lens is not None else None, B, T, output.data_ptr(), timesteps.data_ptr(),
                scores.data_ptr(), out_seq_len.data_ptr(), n_results.data_ptr(), flags.data_ptr(), None,
                self._ws.data_ptr(), self._ws.numel(), stream))
        self.last_flags, self.last_n_results = flags, n_results
        if self._device_outputs and not host:
            if not self._non_blocking:
                torch.cuda.current_stream(dev).synchronize()
                self._check_flags(flags)
            return output, scores, timesteps, out_seq_len
        torch.cuda.current_stream(dev).synchronize()
        self._check_flags(flags)
        self.last_flags, self.last_n_results = flags.cpu(), n_results.cpu()
        return output.cpu(), scores.cpu(), timesteps.cpu(), out_seq_len.cpu()

    @staticmethod
    def _check_flags(flags):
        bad = (flags & _native.FLAG_ERR_ARENA).nonzero()
        if bad.numel():
            where = "utterance %d" % int(bad[0][0]) if flags.dim() == 1 else \
                "pair %d, utterance %d" % tuple(int(v) for v in bad[0])
            raise _native.NativeError("%s: the beam kernel reported an internal error; results are not valid" % where)


class OnlineCTCBeamDecoder(_Base):
    """Drop-in for the reference OnlineCTCBeamDecoder (reference ctcdecode/__init__.py:143-250); the per-stream
    DecoderState (beam, trie, absolute frame counter) lives in GPU memory between chunks."""

    def __init__(self, labels, model_path=None, alpha=0, beta=0, cutoff_top_n=40, cutoff_prob=1.0, beam_width=100,
                 num_processes=4, blank_id=0, log_probs_input=False, device=None, scorer_provider=None,
                 device_outputs=False, non_blocking=False):
        self._cutoff_top_n = cutoff_top_n  # private name kept from the reference (:175)
        self._device_outputs = device_outputs
        self._ws = None
        self._init_common(labels, model_path, alpha, beta, cutoff_top_n, cutoff_prob, beam_width, num_processes,
                          blank_id, log_probs_input, device, scorer_provider=scorer_provider,
                          non_blocking=non_blocking)

    def _cutoff_top_n_value(self):
        return int(self._cutoff_top_n)

    def decode(self, probs, states, is_eos_s, seq_lens=None):
        """Feeds one chunk per stream.  Returns (beam_results, beam_scores, timesteps, out_lens) like reference
        __init__.py:189-238: beam_results / timesteps are [B, n_beams, max_len] (both [B, 0, 0] while no stream
        has reached eos), beam_scores / out_lens are [B, beam].

        A CUDA chunk (without a scorer, or with non_blocking=True) is decoded in place on the current stream
        (ctcdec_decode_stream_device).
        With device_outputs=True the results stay on the GPU and the call does not wait for it: beam_results /
        timesteps are [B, beam, out_T] (out_T: the most frames an eos stream has consumed; [B, 0, 0] without eos),
        only [b, p, :out_lens[b, p]] of rows p < last_n_results[b] of eos streams being meaningful."""
        lib = _native.load()
        if probs.dim() != 3:
            raise ValueError("probs must be [batch, time, labels], got %s" % (tuple(probs.shape),))
        if probs.is_cuda and (self._scorer is None or self._non_blocking):
            return self._decode_device(lib, probs, states, is_eos_s, seq_lens, -1)
        probs = probs.cpu().float().contiguous()
        B, T, V = probs.shape
        self._check_chunk(B, V, states, is_eos_s)
        if seq_lens is not None:
            seq_lens = seq_lens.cpu().int().contiguous()
        K = self._beam_width
        scores = torch.empty(B, K, dtype=torch.float32)
        out_seq_len = torch.zeros(B, K, dtype=torch.int32)
        n_results = torch.zeros(B, dtype=torch.int32)
        flags = torch.zeros(B, dtype=torch.int32)
        handles = (ctypes.c_void_p * B)(*[s.state for s in states])
        eos = (ctypes.c_uint8 * B)(*[1 if e else 0 for e in is_eos_s])
        any_eos = any(bool(e) for e in is_eos_s)
        out_T = 0
        if any_eos:
            for b, s in enumerate(states):
                if is_eos_s[b]:
                    fr = ctypes.c_int(0)
                    _native.check(lib.ctcdec_state_frames(s.state, ctypes.byref(fr)))
                    ln = T if seq_lens is None else max(0, min(int(seq_lens[b]), T))
                    out_T = max(out_T, fr.value + ln)
        tokens = torch.zeros(B, K, max(out_T, 1), dtype=torch.int32)
        timesteps = torch.zeros(B, K, max(out_T, 1), dtype=torch.int32)
        _native.check(lib.ctcdec_decode_stream_host(
            probs.data_ptr(), seq_lens.data_ptr() if seq_lens is not None else None, B, T, handles, eos,
            tokens.data_ptr(), timesteps.data_ptr(), max(out_T, 1), scores.data_ptr(), out_seq_len.data_ptr(),
            n_results.data_ptr(), flags.data_ptr()))
        self.last_flags, self.last_n_results = flags, n_results
        if not any_eos:
            empty = torch.zeros(B, 0, 0, dtype=torch.int32)
            return empty, scores, empty.clone(), out_seq_len
        max_res = int(n_results.max())
        max_len = int(out_seq_len.max())
        # reference binding.cpp:181-205: tensors sized [B, max_result_size, max_output_tokens_size]
        return (tokens[:, :max_res, :max_len].contiguous(), scores, timesteps[:, :max_res, :max_len].contiguous(),
                out_seq_len)

    def decode_logits(self, logits, states, is_eos_s, seq_lens=None):
        """Extension: decode's CUDA path for the acoustic model's raw LOGITS, a CUDA tensor [B, T, V] in float32 /
        float16 / bfloat16; each frame's float32 log-softmax is taken on the fly (as CTCBeamDecoder.decode_logits
        does), so chunks decode exactly like the concatenated logits would offline."""
        lib = _native.load()
        if self._scorer is not None and not self._non_blocking:
            raise NotImplementedError("ctcdecode_b200: decode_logits with a scorer needs non_blocking=True "
                                      "(and scorer_provider=\"device\")")
        if logits.dim() != 3 or not logits.is_cuda:
            raise ValueError("logits must be a CUDA tensor [batch, time, labels]")
        dtypes = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
        if logits.dtype not in dtypes:
            raise ValueError("logits must be float32, float16 or bfloat16, got %s" % logits.dtype)
        return self._decode_device(lib, logits, states, is_eos_s, seq_lens, dtypes[logits.dtype])

    def _check_chunk(self, B, V, states, is_eos_s):
        if V != self._num_labels:
            raise ValueError("probs has %d labels, decoder was built with %d" % (V, self._num_labels))
        if len(states) != B or len(is_eos_s) != B:
            raise ValueError("need one state and one is_eos flag per batch item")

    @staticmethod
    def _frames(lib, states):
        out = []
        for s in states:
            fr = ctypes.c_int(0)
            _native.check(lib.ctcdec_state_frames(s.state, ctypes.byref(fr)))
            out.append(fr.value)
        return out

    @staticmethod
    def _states_device(states, dev):
        for s in states:
            if s.device != dev.index:
                raise ValueError("a state lives on cuda:%d, the chunk on %s" % (s.device, dev))

    def _decode_device(self, lib, x, states, is_eos_s, seq_lens, dtype):
        B, T, V = x.shape
        self._check_chunk(B, V, states, is_eos_s)
        dev = x.device
        self._states_device(states, dev)
        x = (x.float() if dtype < 0 else x).contiguous()
        # seq_lens, is_eos and the frame counts stay on the host: the output sizes follow without reading the device
        lens_h = [T] * B if seq_lens is None else [max(0, min(int(v), T)) for v in seq_lens.cpu().tolist()]
        sl = None if seq_lens is None else torch.tensor(lens_h, dtype=torch.int32)
        eos = [bool(e) for e in is_eos_s]
        eos_b = [b for b in range(B) if eos[b]]
        frames = self._frames(lib, [states[b] for b in eos_b])
        out_T = max([frames[i] + lens_h[b] for i, b in enumerate(eos_b)], default=0)
        K = self._beam_width
        cfg = _cfg(self)
        nbytes = ctypes.c_size_t(0)
        handles = (ctypes.c_void_p * B)(*[s.state for s in states])
        # (states of several device-scorer decoders need room for their LM slots as well)
        if B:
            _native.check(lib.ctcdec_stream_states_workspace_bytes(handles, B, T, ctypes.byref(nbytes)))
        else:
            _native.check(lib.ctcdec_stream_workspace_bytes(ctypes.byref(cfg), B, T, ctypes.byref(nbytes)))
        if self._ws is None or self._ws.numel() < nbytes.value or self._ws.device != dev:
            self._ws = None
            self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        tokens = torch.zeros(B, K, max(out_T, 1), dtype=torch.int32, device=dev)
        timesteps = torch.zeros(B, K, max(out_T, 1), dtype=torch.int32, device=dev)
        scores = torch.zeros(B, K, dtype=torch.float32, device=dev)
        out_seq_len = torch.zeros(B, K, dtype=torch.int32, device=dev)
        n_results = torch.zeros(B, dtype=torch.int32, device=dev)
        flags = torch.zeros(B, dtype=torch.int32, device=dev)
        eos_arr = (ctypes.c_uint8 * B)(*[1 if e else 0 for e in eos])
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(lib.ctcdec_decode_stream_device(
                x.data_ptr(), dtype, sl.data_ptr() if sl is not None else None, B, T, handles, eos_arr,
                tokens.data_ptr(), timesteps.data_ptr(), max(out_T, 1), scores.data_ptr(), out_seq_len.data_ptr(),
                n_results.data_ptr(), flags.data_ptr(), self._ws.data_ptr(), self._ws.numel(), stream))
        if self._device_outputs:
            self.last_flags, self.last_n_results = flags, n_results
            if not any(eos):
                empty = torch.zeros(B, 0, 0, dtype=torch.int32, device=dev)
                return empty, scores, empty.clone(), out_seq_len
            return tokens[:, :, :out_T], scores, timesteps[:, :, :out_T], out_seq_len
        # the host path's return values: CPU tensors, [B, max_res, max_len] (flags are not reported without eos)
        n_results, lens_cpu = n_results.cpu(), out_seq_len.cpu()
        flags = flags.cpu() if any(eos) else torch.zeros(B, dtype=torch.int32)
        self.last_flags, self.last_n_results = flags, n_results
        if (flags & _native.FLAG_ERR_ARENA).any():
            raise _native.NativeError("ctcdecode_b200: the beam kernel reported an internal error (node arena "
                                      "exhausted); results are not valid")
        if not any(eos):
            empty = torch.zeros(B, 0, 0, dtype=torch.int32)
            return empty, scores.cpu(), empty.clone(), lens_cpu
        max_res, max_len = int(n_results.max()), int(lens_cpu.max())
        return (tokens[:, :max_res, :max_len].cpu(), scores.cpu(), timesteps[:, :max_res, :max_len].cpu(), lens_cpu)

    def committed_prefix(self, states, since=None):
        """Extension: the part of each stream's transcript that no later chunk can change -- the path from the trie
        root to the lowest common ancestor of the stream's beam members (ctcdec_stream_committed_device).  Its tokens
        and timesteps start every row any later decode of the stream returns.  since: int32 [B] positions the caller
        already has (normally the previous call's `committed`), None = 0; a value beyond the committed depth reads
        from 0.  Returns (tokens [B, D], timesteps [B, D], n_new [B], committed [B]): row b holds the n_new[b] new
        positions from column 0, D = max(n_new).  CUDA tensors with device_outputs=True, CPU tensors otherwise; the
        call waits for the device once, to size D."""
        lib = _native.load()
        B = len(states)
        if B == 0:
            z = torch.zeros(0, dtype=torch.int32)
            return z.view(0, 0), z.view(0, 0), z, z
        devs = {s.device for s in states}
        if len(devs) != 1:
            raise ValueError("all states must live on one device, got %s" % sorted(devs))
        dev = torch.device("cuda", devs.pop())
        cap = max(max(self._frames(lib, states)), 1)  # committed <= frames consumed: nothing is cut off
        tok = torch.empty(B, cap, dtype=torch.int32, device=dev)
        ts = torch.empty(B, cap, dtype=torch.int32, device=dev)
        committed = torch.empty(B, dtype=torch.int32, device=dev)
        if since is not None:
            since = torch.as_tensor(since).to(device=dev, dtype=torch.int32).contiguous()
            if since.shape != (B,):
                raise ValueError("since must be [batch]")
        handles = (ctypes.c_void_p * B)(*[s.state for s in states])
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(lib.ctcdec_stream_committed_device(
                handles, B, since.data_ptr() if since is not None else None, committed.data_ptr(), tok.data_ptr(),
                ts.data_ptr(), cap, stream))
        start = torch.zeros_like(committed) if since is None else \
            torch.where((since >= 0) & (since <= committed), since, torch.zeros_like(since))
        n_new = committed - start
        D = int(n_new.max())
        tok, ts = tok[:, :D], ts[:, :D]
        if self._device_outputs:
            return tok, ts, n_new, committed
        return tok.cpu(), ts.cpu(), n_new.cpu(), committed.cpu()

    def compact(self, states):
        """Extension: frees the parts of each stream's trie that no later call can read (ctcdec_stream_compact).  A
        stream's node arena otherwise grows by up to beam_width nodes per frame for as long as the stream lives; after
        this call it holds only the paths from the root to the current beam members, and every later result of the
        stream is bit for bit what it would have been without the call.  A server calls it every so many chunks, like
        committed_prefix.  Waits for the device.  States of a hook scorer (scorer_provider other than "device") are
        refused.  Returns the nodes each state holds now: int64 CPU tensor [B]."""
        lib = _native.load()
        B = len(states)
        kept = torch.zeros(B, dtype=torch.int64)
        if B == 0:
            return kept
        devs = {s.device for s in states}
        if len(devs) != 1:
            raise ValueError("all states must live on one device, got %s" % sorted(devs))
        dev = torch.device("cuda", devs.pop())
        handles = (ctypes.c_void_p * B)(*[s.state for s in states])
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(lib.ctcdec_stream_compact(handles, B, kept.data_ptr(), stream))
        return kept

    def reset_state(state):  # noqa: N805 -- signature kept from the reference (:249), which lacks `self`
        state.release()


class DecoderState(object):
    """One stream's decoding state (reference ctcdecode/__init__.py:253-272); device resident."""

    def __init__(self, decoder):
        lib = _native.load()
        cfg = _cfg(decoder)
        handle = ctypes.c_void_p()
        # the scorer is borrowed by the state (reference ctc_beam_search_decoder.cpp:31): keep the decoder alive
        self._decoder = decoder
        scorer = decoder._scorer.handle if decoder._scorer else None
        self.device = decoder._device_index()
        _native.check(lib.ctcdec_state_create_lm(ctypes.byref(cfg), scorer, self.device, ctypes.byref(handle)))
        self.state = handle.value

    def device_bytes(self):
        """Extension: the device memory this state holds (node arena, state block, scorer arrays), in bytes."""
        n = ctypes.c_size_t(0)
        _native.check(_native.load().ctcdec_state_device_bytes(self.state, ctypes.byref(n)))
        return n.value

    def release(self):
        if getattr(self, "state", None):
            _native.load().ctcdec_state_destroy(self.state)
            self.state = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

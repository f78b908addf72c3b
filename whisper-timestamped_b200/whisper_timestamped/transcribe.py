"""Public API of the drop-in: transcribe_timestamped() / transcribe().

Same signature, option checks and return value as the reference
(/root/reference/whisper_timestamped/transcribe.py:79-357), but organised for a batched GPU engine:

  1. every audio "stream" (the whole file, or independent fixed-length cuts when `chunks=` is given)
     advances through upstream's seek loop; each round the next window of EVERY active stream is
     decoded in ONE engine batch (encoder + greedy decoder on the GPU, cross-attention rows of the
     alignment heads written straight into the alignment buffer — no forward hooks, no per-token
     device->host copies: replaces T.py:783-793, 849-881);
  2. as soon as a decode batch is consumed, the hook state machine of the reference is replayed offline
     (windows.py) on its windows to find the segments, and all of them are aligned in one batch on the GPU
     (alignment.py: attention post-processing + DTW); the batch's alignment rows are then freed;
  3. words, confidences and post-processing follow T.py:912-1002 and 313-357.
"""
import io
import logging
import sys
from typing import List, Optional

import numpy as np

from . import vad as V
from . import words as W
from .tokenizer import LANGUAGES, TO_LANGUAGE_CODE, get_tokenizer
from .writers import filtered_keys, flatten, remove_keys, write_csv, write_tsv  # T.py:2298-2323, 3183-3199
from .windows import (HOP_LENGTH, N_FRAMES, SAMPLE_RATE, WindowRecord, make_decode_setup, plan_window_alignment,
                      slice_window_segments)

logger = logging.getLogger("whisper_timestamped")

AUDIO_TIME_PER_TOKEN = 0.02
USE_EFFICIENT_BY_DEFAULT = True
TRUST_WHISPER_TIMESTAMP_BY_DEFAULT = True
DISFLUENCY_MARK = "[*]"


def should_use_space(language):
    return norm_language(language) not in ["zh", "ja", "th", "lo", "my", "yue"]


def norm_language(language):
    if language is None:
        return "en"
    return TO_LANGUAGE_CODE.get(language.lower(), language)


class _File:
    """One recording of a call: its audio, its language, tokenizer and decode setup, the streams it is transcribed as
    (the whole recording, or its cuts with `chunks=`) and where its stdout goes."""

    def __init__(self, audio, out):
        self.audio = audio
        self.out = out
        self.vad_spans = self.convert_timestamps = None
        self.language = self.language_probs = None
        self.tokenizer = self.setup = None
        self.use_space = True
        self.streams = []


class _Stream:
    """One independently transcribed piece of audio: upstream's seek loop state."""

    def __init__(self, index, file, mel_handle, content_frames, time_shift, initial_prompt_tokens):
        self.index = index
        self.file = file
        self.mel = mel_handle
        self.content_frames = content_frames
        self.time_shift = time_shift               # seconds added to every time of this stream
        self.seek = 0
        self.all_tokens = list(initial_prompt_tokens)
        self.n_initial_prompt = len(initial_prompt_tokens)
        self.prompt_reset_since = 0
        self.segments = []                          # upstream-style segment dicts
        self.records: List[WindowRecord] = []       # every decoded window, in order
        self.kept = []                              # per record: was it kept (not skipped as silence)

    @property
    def active(self):
        return self.seek < self.content_frames

    def next_job(self):
        size = min(N_FRAMES, self.content_frames - self.seek)
        prompt = self.file.setup.initial_tokens(self.all_tokens[self.prompt_reset_since:])
        return dict(stream=self.index, mel=self.mel, seek=self.seek, segment_size=size, prompt=prompt,
                    language=self.file.language)

    def consume(self, rec: WindowRecord, tokenizer, no_speech_threshold, logprob_threshold,
                condition_on_previous_text):
        self.records.append(rec)
        if no_speech_threshold is not None:
            skip = rec.no_speech_prob > no_speech_threshold
            if logprob_threshold is not None and rec.avg_logprob > logprob_threshold:
                skip = False
            if skip:
                self.kept.append(False)
                self.seek += rec.segment_size
                return
        self.kept.append(True)
        segs, advance = slice_window_segments(rec, tokenizer)
        self.seek += advance
        for s in segs:
            s["id"] = len(self.segments)
            self.segments.append(s)
            self.all_tokens.extend(s["tokens"])
        if not condition_on_previous_text or rec.temperature > 0.5:
            self.prompt_reset_since = len(self.all_tokens)


def top_layers_heads(n_layer, n_head, k):
    """`word_alignment_most_top_layers=k`: every head of the top k decoder layers (k clipped at the number of layers),
    layer-major — the order of the reference's reshape to [k*H, T, F] (T.py:1542-1543)."""
    assert k > 0, "word_alignment_most_top_layers must be a strictly positive number"
    return [(l, h) for l in range(max(0, n_layer - k), n_layer) for h in range(n_head)]


def shared_setup_key(setup):
    """What a greedy decode batch takes from its DecodeSetup: the decode session's key, the token masks, and the
    <|startoftranscript|> and <|nospeech|> tokens of the prefill.  All of it is the same for every language of one model,
    so windows of recordings in different languages can share a batch: the language lives in each window's prompt."""
    tok = setup.tokenizer
    return (setup.n_ctx, setup.sample_len, setup.suppress_tokens, setup.blank_tokens, setup.max_initial_timestamp_index,
            setup.temperature, setup.beam_size, setup.best_of, tok.sot, tok.eot, tok.no_speech, tok.no_timestamps,
            tok.timestamp_begin)


def decode_with_fallback(eng, jobs, setup, temperatures, tokenizer, compression_ratio_threshold, logprob_threshold,
                         no_speech_threshold):
    """Upstream `decode_with_fallback` (reached by the reference through model.transcribe, T.py:904 / 1068, options
    T.py:111-113) for a BATCH of windows: every window is decoded at the first temperature (beam search or greedy at
    0, best-of-n sampling above); the windows whose result is too repetitive or too unlikely — and not silence — are
    decoded again, together, at the next temperature; the last attempt stands."""
    from .windows import needs_fallback
    final = [None] * len(jobs)
    pending = list(range(len(jobs)))
    for k, t in enumerate(temperatures):
        recs = eng.decode_windows([jobs[i] for i in pending], setup.at_temperature(t))
        again = []
        for i, rec in zip(pending, recs):
            final[i] = rec
            if k + 1 < len(temperatures) and needs_fallback(rec, tokenizer, compression_ratio_threshold, logprob_threshold,
                                                            no_speech_threshold):
                again.append(i)
        pending = again
        if not pending:
            break
    return final


def transcribe_timestamped(
    model,
    audio,
    language=None,
    task="transcribe",
    remove_punctuation_from_words=False,
    compute_word_confidence=True,
    include_punctuation_in_confidence=False,
    refine_whisper_precision=0.5,
    min_word_duration=0.02,
    plot_word_alignment=False,
    word_alignment_most_top_layers=None,
    remove_empty_words=False,
    use_backend_timestamps=False,
    seed=1234,
    vad=False,
    detect_disfluencies=False,
    trust_whisper_timestamps=TRUST_WHISPER_TIMESTAMP_BY_DEFAULT,
    naive_approach=False,
    temperature=0.0 if USE_EFFICIENT_BY_DEFAULT else (0.0, 0.2, 0.4, 0.6, 0.8, 1.0),
    best_of=None,
    beam_size=None,
    patience=None,
    length_penalty=None,
    compression_ratio_threshold=2.4,
    logprob_threshold=-1.0,
    no_speech_threshold=0.6,
    fp16=None,
    condition_on_previous_text=True,
    initial_prompt=None,
    suppress_tokens="-1",
    sample_len=None,
    verbose=False,
    *,
    chunks=None,
    engine=None,
    continuous_batching=False,
):
    """Drop-in for whisper_timestamped.transcribe (reference T.py:79-357).

    `audio` may also be a list or tuple of recordings (paths, arrays or tensors): the call then returns one result per
    recording, in input order, each equal to what `transcribe(model, that_audio, **options)` returns; stdout is what those
    calls print, one recording after the other.  In the one-pass strategy without `vad`, the windows of all recordings
    share the decode batches (each recording keeps its own language, prompt chain and post-processing); otherwise the
    recordings run one after the other, each reseeded with `seed` as separate calls are.

    Extra keyword-only arguments (not in the reference):
      chunks: None = upstream semantics (one sequential stream over the whole file).  A number of
              seconds = cut the audio at fixed boundaries and transcribe every cut as an independent
              file (condition_on_previous_text is forced off across cuts); all cuts are decoded in the
              same GPU batches.  This is the data-parallel mode BASELINE.json's north_star names.
      engine: inject a decode/alignment engine (tests); default = the model's CUDA engine.
      continuous_batching: let the engine admit a stream's next window into the running decode batch as soon as its
              previous window finishes, instead of decoding in rounds that wait for their slowest window.  Same
              results.  Off by default: on the bench workload 20 % of the windows run to the 224-token limit and their
              follow-up windows belong to the chunks that are already the longest, so there is little to gain; it pays
              when windows end early and unevenly.
    """
    options = {k: v for k, v in locals().items() if k not in ("model", "audio")}
    multi = isinstance(audio, (list, tuple))
    if multi and chunks is not None:
        raise NotImplementedError("chunks= with a list of audios is not built: pass the recordings one by one")
    # ---- option checks, as T.py:223-261
    assert refine_whisper_precision >= 0 and refine_whisper_precision / AUDIO_TIME_PER_TOKEN == round(
        refine_whisper_precision / AUDIO_TIME_PER_TOKEN), \
        f"refine_whisper_precision must be a positive multiple of {AUDIO_TIME_PER_TOKEN}"
    refine_nframes = round(refine_whisper_precision / AUDIO_TIME_PER_TOKEN)
    assert min_word_duration >= 0, "min_word_duration must be a positive number"
    assert word_alignment_most_top_layers is None or word_alignment_most_top_layers > 0, \
        "word_alignment_most_top_layers must be a strictly positive number"
    if isinstance(temperature, (list, tuple)) and len(temperature) == 1:
        temperature = temperature[0]
    if isinstance(temperature, (list, tuple)):
        naive_approach = True
    elif temperature > 0 and best_of is not None and best_of > 1:
        naive_approach = True
    if beam_size is not None:
        naive_approach = True
    if use_backend_timestamps:
        naive_approach = True
    if isinstance(model, str):
        from .model import load_model
        model = load_model(model)
    if use_backend_timestamps:
        raise NotImplementedError("use_backend_timestamps (upstream whisper.timing / HF token timestamps) is not built in "
                                  "this H100 drop-in")
    if not naive_approach and temperature != 0:
        raise NotImplementedError(
            "a scalar temperature > 0 inside the one-pass strategy (sampling under the attention hooks) is not built; "
            "pass naive_approach=True, best_of > 1 or a temperature tuple (two-pass strategy, SURVEY.md §8 rows A14/A15)")
    if not trust_whisper_timestamps and not naive_approach:
        raise NotImplementedError("trust_whisper_timestamps=False is only built for the two-pass strategy (naive_approach=True)")
    if plot_word_alignment:
        raise NotImplementedError("plot_word_alignment is out of scope of the hot path")
    vad = V.check_vad_method(vad)          # explicit (start, end) lists only; detector names raise NotImplementedError
    if multi and (naive_approach or vad is not None):
        # one recording after the other through the single-file path, which reseeds below as separate calls do
        return [transcribe_timestamped(model, a, **options) for a in audio]
    if seed is not None:                   # T.py:223-225: sampling (temperature > 0) draws from torch's global generator
        import torch
        torch.manual_seed(seed)

    eng = engine if engine is not None else model.engine()
    if hasattr(eng, "release"):
        eng.release()                      # alignment buffers of a previous call
    dims = model.dims
    # alignment heads of this call: every head of the top k layers (T.py:259, 401, 892, 1542-1548), else the model's own
    if word_alignment_most_top_layers is not None:
        if not hasattr(eng, "set_alignment_heads"):
            raise NotImplementedError("word_alignment_most_top_layers: this engine cannot change its alignment heads")
        eng.set_alignment_heads(top_layers_heads(dims.n_text_layer, dims.n_text_head, word_alignment_most_top_layers))
    elif hasattr(eng, "set_alignment_heads"):
        eng.set_alignment_heads(None)
    is_multilingual = model.is_multilingual
    num_languages = model.num_languages

    # ---- audio -> log-mel on the device, per stream (upstream pads 30 s and floors at the stream max).  A list call
    # buffers each recording's stdout and prints it at the end, in input order
    files = [_File(eng.load_audio(a), io.StringIO() if multi else sys.stdout) for a in (audio if multi else [audio])]
    if not files:
        return []
    for f in files:
        if vad is not None:                # T.py:294-296: the model only sees the glued speech
            f.audio, f.vad_spans, f.convert_timestamps = V.remove_non_speech(f.audio, vad)
        n_samples = int(f.audio.shape[-1])
        if chunks is None:
            f.cuts = [(0, n_samples)]
        else:
            step = int(round(float(chunks) * SAMPLE_RATE))
            assert step > 0
            f.cuts = [(s, min(s + step, n_samples)) for s in range(0, max(n_samples, 1), step)]
            condition_on_previous_text = False
        f.mels = [eng.log_mel(f.audio[s:e]) for (s, e) in f.cuts]
        if not naive_approach:
            f.audio = None                 # only the two-pass strategy goes back to the samples

    # ---- language (T.py:811-820 + upstream detection on the first window of each file)
    if language is None and not is_multilingual:
        language = "en"
    language_detected = language is None
    if language_detected:
        tok0 = get_tokenizer(True, num_languages=num_languages)
        # stdout as the reference + upstream produce it (T.py:817-820, 844-846, 1030-1032, 1073-1075; upstream
        # prints the result whenever verbose is not None).  With a VAD the inner call runs with verbose=False (T.py:286).
        inner_verbose = verbose if (vad is None or verbose is not True) else False
        if inner_verbose:
            for f in files:
                print("Detecting language using up to the first 30 seconds. Use `--language` to specify the language",
                      file=f.out)
        first = [f.mels[0] for f in files]
        if hasattr(eng, "detect_languages"):
            found = eng.detect_languages(first, tok0)
        else:
            found = [eng.detect_language(m, tok0) for m in first]
        for f, (lang, probs) in zip(files, found):
            f.language, f.language_probs = lang, probs
            if inner_verbose is not None:
                print(f"Detected language: {LANGUAGES[f.language].title()}", file=f.out)
                f.out.flush()
    temperatures = [float(t) for t in temperature] if isinstance(temperature, (list, tuple)) else [float(temperature)]
    streams = []
    for f in files:
        lang = f.language if language_detected else language
        lang = lang.lower() if lang else lang
        if lang not in LANGUAGES and lang in TO_LANGUAGE_CODE:
            lang = TO_LANGUAGE_CODE[lang]
        f.language = lang
        f.tokenizer = get_tokenizer(is_multilingual, num_languages=num_languages, language=lang, task=task)
        f.setup = make_decode_setup(f.tokenizer, dims.n_text_ctx, sample_len=sample_len, suppress_tokens=suppress_tokens,
                                    temperature=temperatures[0], beam_size=beam_size, patience=patience, best_of=best_of,
                                    length_penalty=length_penalty)
        f.use_space = should_use_space(lang)
        initial_prompt_tokens = f.tokenizer.encode(" " + initial_prompt.strip()) if initial_prompt is not None else []
        for (s, e), mel in zip(f.cuts, f.mels):
            content_frames = eng.mel_frames(mel) - N_FRAMES
            f.streams.append(_Stream(len(streams), f, mel, content_frames, s / SAMPLE_RATE, initial_prompt_tokens))
            streams.append(f.streams[-1])
    # the engine decodes windows of every file in shared batches under one setup: the files' setups may only differ in
    # what their prompts carry (the language)
    setup, tokenizer = files[0].setup, files[0].tokenizer
    assert all(shared_setup_key(f.setup) == shared_setup_key(setup) for f in files), \
        "the recordings of one call need decode setups that can share a batch"

    consumed = []         # (stream, window idx, prompt of the stream's next window or None) not yet aligned
    aligned = {}          # (stream idx, window idx) -> (plans, info, [(plan, request, jumps, disfluency starts)])

    def align_consumed():
        """One-pass strategy: plan and align the windows consumed since the last call (one decode batch, or one
        collection of continuous batching), then free their alignment rows.  A window's plan needs only its own tokens
        and the next window's prompt, which consume() has produced; the jumps stay on the host until the words are
        assembled at the end."""
        if naive_approach or not consumed:
            consumed.clear()
            return
        pending, items = [], []
        for st, wi, nxt in consumed:
            rec = st.records[wi]
            reqs = {}

            def yields_words(plan, reqs=reqs, f=st.file):
                # T.py:540-559: `ws` is empty when there is nothing between the timestamps or every word is a
                # special token; this only depends on the tokens, so it is known before the DTW runs
                req = None
                if len(plan.tokens) > 1:
                    req = W.prepare_alignment(plan.tokens, plan.n_rows, f.tokenizer, use_space=f.use_space,
                                              refine_nframes=refine_nframes,
                                              remove_punctuation_from_words=remove_punctuation_from_words,
                                              unfinished_decoding=plan.unfinished)
                reqs[id(plan)] = req
                if req is None:
                    return False
                kept = req.words[1:] if req.unfinished else req.words[1:-1]
                return any(not w.startswith("<|") for w in kept)

            plans, info = plan_window_alignment(rec, st.file.setup, nxt, yields_words)
            aligned[(st.index, wi)] = (plans, info, [])
            for plan in plans:
                req = reqs[id(plan)]
                for msg in (req.warnings if req is not None else []):
                    logger.warning(msg)
                if req is not None and rec.max_duration and req.f0 >= rec.max_duration:
                    logger.warning("Got start time outside of audio boundary")
                if req is None:
                    aligned[(st.index, wi)][2].append((plan, None, None, None))
                    continue
                pending.append((st.index, wi, plan, req))
                items.append(dict(window=rec.qk_window, row0=plan.row0, last_row=plan.row0 + req.row_offset_last,
                                  T=req.T, f0=req.f0, F=req.F, max_dur=rec.max_duration or 0))
        lefts_list = None
        if items and detect_disfluencies:
            jumps_list, lefts_list = eng.align(items, disfluencies=True)
        else:
            jumps_list = eng.align(items) if items else []
        for (si, wi, plan, req), j, l_ in zip(pending, jumps_list, lefts_list or [None] * len(jumps_list)):
            aligned[(si, wi)][2].append((plan, req, j, l_))
        if hasattr(eng, "free_alignment_rows"):
            eng.free_alignment_rows([st.records[wi].qk_window for st, wi, _ in consumed])
        consumed.clear()

    # ---- decode: the next window of every active stream in one GPU batch
    def consume(job, rec):
        st = streams[job["stream"]]
        if language_detected and st is st.file.streams[0] and not st.records:
            rec.mel_from_language_detection = True        # first window of the file, see WindowRecord.max_duration
        st.consume(rec, st.file.tokenizer, no_speech_threshold, logprob_threshold, condition_on_previous_text)
        nxt = st.next_job() if st.active else None
        consumed.append((st, len(st.records) - 1, nxt["prompt"] if nxt is not None else None))
        return nxt

    plain_greedy = len(temperatures) == 1 and temperatures[0] == 0 and setup.beam_size is None
    if plain_greedy and hasattr(eng, "decode_stream") and continuous_batching:
        # continuous batching: a stream's next window is admitted into the decode batch as soon as its previous one
        # finishes (no round barrier); per stream the windows are still decoded strictly in upstream's order
        eng.decode_stream([st.next_job() for st in streams if st.active], setup, consume, collected=align_consumed)
    else:
        # one decode batch at a time (the engine's batch size), so that only one batch of alignment rows is alive
        limit = eng.batch_limit(setup) if hasattr(eng, "batch_limit") and not naive_approach else None
        while True:
            jobs = [st.next_job() for st in streams if st.active]
            if not jobs:
                break
            for i in range(0, len(jobs), limit or len(jobs)):
                part = jobs[i:i + limit] if limit else jobs
                records = decode_with_fallback(eng, part, setup, temperatures, tokenizer, compression_ratio_threshold,
                                               logprob_threshold, no_speech_threshold)
                for job, rec in zip(part, records):
                    consume(job, rec)
                align_consumed()
    align_consumed()
    finish = dict(naive_approach=naive_approach, chunks=chunks, vad=vad, verbose=verbose, refine_nframes=refine_nframes,
                  refine_whisper_precision=refine_whisper_precision, trust_whisper_timestamps=trust_whisper_timestamps,
                  remove_punctuation_from_words=remove_punctuation_from_words,
                  compute_word_confidence=compute_word_confidence,
                  include_punctuation_in_confidence=include_punctuation_in_confidence,
                  detect_disfluencies=detect_disfluencies, no_speech_threshold=no_speech_threshold,
                  logprob_threshold=logprob_threshold, remove_empty_words=remove_empty_words,
                  min_word_duration=min_word_duration)
    results = [_file_result(f, eng, aligned, **finish) for f in files]
    if hasattr(eng, "release"):
        eng.release()
    if not multi:
        return results[0]
    for f in files:
        sys.stdout.write(f.out.getvalue())
    sys.stdout.flush()
    return results


def _file_result(f, eng, aligned, *, naive_approach, chunks, vad, verbose, refine_nframes, refine_whisper_precision,
                 trust_whisper_timestamps, remove_punctuation_from_words, compute_word_confidence,
                 include_punctuation_in_confidence, detect_disfluencies, no_speech_threshold, logprob_threshold,
                 remove_empty_words, min_word_duration):
    """The result of one recording from its decoded windows and their alignments (T.py:712-1002, 313-357)."""
    tokenizer, setup, language, use_space, streams = f.tokenizer, f.setup, f.language, f.use_space, f.streams
    audio, language_probs, vad_spans, convert_timestamps = f.audio, f.language_probs, f.vad_spans, f.convert_timestamps
    if naive_approach:
        # ---- two-pass strategy (T.py:1004-1338): pass 1 above was plain decoding; pass 2 re-runs the decoder teacher-forced
        # on every segment's own audio window and aligns all of its tokens at once
        assert chunks is None, "the two-pass strategy works on one sequential stream (chunks=None)"
        from . import naive as NV
        st = streams[0]
        all_segments = list(st.segments)
        all_words = NV.second_pass(eng, audio, all_segments, tokenizer, language, use_space=use_space,
                                   refine_nframes=refine_nframes, trust_whisper_timestamps=trust_whisper_timestamps,
                                   remove_punctuation_from_words=remove_punctuation_from_words,
                                   compute_word_confidence=compute_word_confidence,
                                   include_punctuation_in_confidence=include_punctuation_in_confidence,
                                   min_word_duration=0.0, detect_disfluencies=detect_disfluencies,
                                   verbose=bool(verbose) and vad is None)
        for w in all_words:
            w["_stream"] = 0
        text_parts = [tokenizer.decode(st.all_tokens[st.n_initial_prompt:])]
    else:
        # ---- per stream: words, confidences, compile (T.py:712-771, 912-1002)
        all_segments, all_words = [], []
        text_parts = []
        for st in streams:
            seg_words = []        # words of every flushed segment of this stream, in order
            seg_logprobs = []     # log-probs of the text tokens of the same segments
            seg_avglogprob = []
            seg_tokens = []       # the token list each flushed segment ended up with
            for wi, rec in enumerate(st.records):
                plans, info, done = aligned[(st.index, wi)]
                ws_of_window, kept_plans = [], []
                for (plan, req, jumps, lefts) in done:
                    ws = W.words_from_jumps(req, jumps, lefts, tokenizer=tokenizer) if req is not None else []
                    assert ws, "plan_window_alignment only keeps segments that yield words"
                    ws_of_window.append(ws)
                    kept_plans.append(plan)
                # chunk-level log-probs and the silence rule (T.py:712-748)
                should_skip = False
                if compute_word_confidence or no_speech_threshold is not None:
                    should_skip = (rec.no_speech_prob > no_speech_threshold) if no_speech_threshold is not None else False
                    lp = np.array(rec.logprobs, dtype=np.float32)
                    n = len(lp)
                    last_unfinished = bool(kept_plans) and kept_plans[-1].unfinished and plans and plans[-1] is kept_plans[-1] \
                        and info["final_unfinished"]
                    if last_unfinished:
                        fallback = kept_plans[-1].appended_token
                        chosen_last = rec.tokens[n - 1] if n - 1 < len(rec.tokens) else tokenizer.eot
                        if fallback != chosen_last:
                            lp[-1] = rec.last_row_logprobs(fallback)
                        ws_of_window[-1][-1]["avg_logprob_reliable"] = kept_plans[-1].last_token_reliable
                        n += 1
                    elif info["reached"] and ws_of_window:
                        ws_of_window[-1][-1]["avg_logprob_reliable"] = (setup.temperature == 0)
                    assert np.all(np.isfinite(lp)), "Got infinite logprob"
                    avg_logprob = float(lp.sum(dtype=np.float32)) / n if n else 0.0
                    if logprob_threshold is not None and avg_logprob > logprob_threshold:
                        should_skip = False
                if should_skip:
                    continue                       # upstream skipped this window too (no segments)
                for plan, ws in zip(kept_plans, ws_of_window):
                    seg_words.append(ws)
                    seg_tokens.append(list(plan.tokens))
                    if compute_word_confidence:
                        a = plan.row0 + 1          # skip the start timestamp
                        b = plan.row0 + len(plan.tokens) - (0 if (plan.unfinished and plan is kept_plans[-1] and info["final_unfinished"]) else 1)
                        seg_logprobs.append(lp[a:b])
                        seg_avglogprob.append(avg_logprob)
                    else:
                        seg_logprobs.append(None)
                        seg_avglogprob.append(None)

            whisper_segments = [s for s in st.segments if s["text"]] if any(not s["text"] for s in st.segments) \
                else list(st.segments)
            l1, l2 = len(whisper_segments), len(seg_words)
            assert l1 == l2 or l1 == 0, \
                f"Inconsistent number of segments: whisper_segments ({l1}) != timestamped_word_segments ({l2})"
            special0 = min(tokenizer.sot, tokenizer.eot)

            def strip_special(toks):
                toks = list(toks)
                while toks and toks[0] >= special0:
                    toks = toks[1:]
                while toks and toks[-1] >= special0:
                    toks = toks[:-1]
                return toks

            for i, (segment, ws, lps, avglp, flushed) in enumerate(zip(whisper_segments, seg_words, seg_logprobs,
                                                                        seg_avglogprob, seg_tokens)):
                # T.py:941-957: the tokens the state machine flushed vs the tokens upstream kept
                ours, theirs = strip_special(flushed), strip_special(segment["tokens"])
                if ours != theirs:
                    if len(ours) == len(theirs) + 1:
                        logger.warning(f"An additional token was added on segment {i}")
                    elif len(theirs) == 0:
                        logger.warning(f"Whisper has empty segment {i}")
                        assert segment["end"] == segment["start"], f"Fatal Error: Got empty segment {i} with non-zero duration"
                        segment["tokens"] = ours
                        segment["text"] = tokenizer.decode(ours)
                    else:
                        assert len(ours) < len(theirs) and ours == theirs[:len(ours)], \
                            f"Fatal Error: Got inconsistent text for segment {i}:\n{ours}\n!=\n{theirs}"
                        segment["tokens"] = list(flushed)
                        segment["text"] = tokenizer.decode(segment["tokens"])
                        logger.warning(f"Text had to be shortned on segment {i}")
                    ws[-1]["avg_logprob_reliable"] = False
                offset = segment["seek"] * HOP_LENGTH / SAMPLE_RATE
                for w in ws:
                    w["start"] += offset
                    w["end"] += offset
                    w["idx_segment"] = len(all_segments) + i      # index in the FILTERED list, used on the full list (as T.py:963 / 329-331)
                if compute_word_confidence:
                    if ws[-1].get("avg_logprob_reliable", True):
                        if abs(segment["avg_logprob"] - avglp) >= 1e-2:
                            logger.warning(f"Recomputed different logprob for segment {i}: {avglp} != {segment['avg_logprob']}")
                    if include_punctuation_in_confidence:
                        segment["confidence"] = W.round_confidence(float(np.exp(lps.mean(dtype=np.float32))))
                    nopunc = []
                    i_end = 0
                    for w in ws:
                        i_start = i_end
                        pieces = w["tokens"]
                        i_end += len(pieces)
                        assert i_end <= len(lps), f"Fatal Error: Got out-of-bound index for segment {i}: {i_end} > {len(lps)}"
                        if include_punctuation_in_confidence:
                            wl = lps[i_start:i_end]
                        else:
                            while len(pieces) > 1 and len(pieces[-1]) and pieces[-1][-1] in W.PUNCTUATION:
                                pieces = pieces[:-1]
                            wl = lps[i_start:i_start + len(pieces)]
                            nopunc.append(wl)
                        w["confidence"] = W.round_confidence(float(np.exp(wl.mean(dtype=np.float32))) if len(wl) else 0.0)
                    if i_end not in (len(lps), len(lps) - 1):
                        logger.warning(f"Got inconsistent length for segment {i} ({len(lps)} != {i_end}). Some words have been ignored.")
                    if not include_punctuation_in_confidence:
                        cat = np.concatenate(nopunc) if nopunc else np.zeros(0, np.float32)
                        segment["confidence"] = W.round_confidence(float(np.exp(cat.mean(dtype=np.float32))))
                for w in ws:
                    w["_stream"] = st.index
                all_words.extend(ws)
            # stream time shift (independent cuts) is applied after the per-window offsets
            if st.time_shift:
                for w in (w for ws in seg_words for w in ws):
                    w["start"] = W.round_timestamp(w["start"] + st.time_shift)
                    w["end"] = W.round_timestamp(w["end"] + st.time_shift)
                for s in st.segments:
                    s["start"] += st.time_shift
                    s["end"] += st.time_shift
                    s["seek"] += int(round(st.time_shift * SAMPLE_RATE / HOP_LENGTH))
            all_segments.extend(st.segments)              # empty-text segments stay in the output, like the reference
            text_parts.append(tokenizer.decode(st.all_tokens[st.n_initial_prompt:]))

    transcription = dict(text="".join(text_parts), segments=all_segments, language=language)
    if language_probs:
        transcription["language_probs"] = language_probs
    words = all_words

    # ---- post-processing, as T.py:313-357
    if remove_empty_words:
        transcription, words = W.remove_last_null_duration_words(transcription, words, recompute_text=True)
    # independent cuts are post-processed independently (each is "the reference run on that cut alone")
    for idx in sorted({w["_stream"] for w in words}):
        W.ensure_increasing_positions([w for w in words if w["_stream"] == idx],
                                      min_duration=min_word_duration if trust_whisper_timestamps else 0)
    segs = transcription["segments"]
    for word in words:
        if verbose and not naive_approach and vad is None:        # T.py:323-324
            print_timestamped(word, f.out)
        word.pop("tokens", None)
        word.pop("tokens_indices", None)
        word.pop("avg_logprob_reliable", None)
        word.pop("_stream", None)
        idx = word.pop("idx_segment")
        assert idx < len(segs), f"Fatal error: Got unexpected segment index {idx} >= {len(segs)}"
        seg = segs[idx]
        if "words" in seg:
            seg["words"].append(word)
        else:
            seg["words"] = [word]
            if refine_whisper_precision:
                seg["start"] = word["start"]
        if refine_whisper_precision:
            seg["end"] = word["end"]
    if chunks is not None:
        for i, seg in enumerate(segs):        # independent cuts: ids / seeks are those of the whole recording
            seg["id"] = i
    if vad is not None:
        # back to the time axis of the original audio (T.py:341-355)
        for seg in segs:
            for word in seg.get("words", []):
                word["start"], word["end"] = convert_timestamps(word["start"], word["end"])
                if verbose:                                        # T.py:346-347
                    print_timestamped(word, f.out)
            if refine_whisper_precision and len(seg.get("words", [])):
                seg["start"] = seg["words"][0]["start"]
                seg["end"] = seg["words"][-1]["end"]
            else:
                seg["start"], seg["end"] = convert_timestamps(seg["start"], seg["end"])
        transcription["speech_activity"] = [{"start": s, "end": e} for (s, e) in vad_spans]
    return transcription


def print_timestamped(w, file=None):
    """`[mm:ss.mmm --> mm:ss.mmm] text` on stdout (T.py:1363-1368), or on `file`."""
    from .make_subtitles import format_timestamp
    file = file if file is not None else sys.stdout
    line = f"[{format_timestamp(w['start'])} --> {format_timestamp(w['end'])}] {w['text']}\n"
    file.write(line.encode(sys.getdefaultencoding(), errors="replace").decode())
    file.flush()


transcribe = transcribe_timestamped


# ---- command line (the reference's `whisper_timestamped` console script, T.py:2964-3182)
OUTPUT_FORMATS = ["txt", "vtt", "srt", "tsv", "csv", "json"]


def _str2bool(s):
    """"True" / "False" (as openai-whisper's str2bool)."""
    if s in ("True", "False"):
        return s == "True"
    raise ValueError(f"Expected one of {{'True', 'False'}}, got {s}")


def _optional(cast):
    return lambda s: None if s == "None" else cast(s)


def _output_formats(s):
    if s == "all":
        return list(OUTPUT_FORMATS)
    formats = s.split(",")
    for fmt in formats:
        if fmt not in OUTPUT_FORMATS:
            raise ValueError(f"Expected one of {OUTPUT_FORMATS}, got {fmt}")
    return formats


def _vad_option(s):
    """An explicit list of (start, end) seconds is parsed; any other value goes to transcribe() as given."""
    import ast
    return ast.literal_eval(s) if s.lstrip().startswith(("[", "(")) else s


def parse_cli_args(argv=None):
    """argv -> (audio files, load_model arguments, transcribe options, output settings), with the reference's options,
    defaults and conversions (the shortcuts --accurate / --efficient, a temperature tuple from
    --temperature_increment_on_fallback, the renamed --naive / --punctuations_with_words / --compute_confidence /
    --recompute_all_timestamps)."""
    import argparse

    from . import __version__
    parser = argparse.ArgumentParser(description="Transcribe audio files with whisper and compute word timestamps",
                                     formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("-v", "--version", action="version", version=__version__, help="show version and exit")
    parser.add_argument("audio", nargs="+", help="audio file(s) to transcribe")
    parser.add_argument("--model", default="small", help="Whisper model: an official name, a checkpoint path, or "
                                                         "synthetic:<name> for seeded synthetic weights")
    parser.add_argument("--model_dir", default=None, type=str, help="where checkpoints are looked up (~/.cache/whisper)")
    parser.add_argument("--device", default=None, help="CUDA device (the current one by default)")
    parser.add_argument("--backend", default="openai-whisper", choices=["openai-whisper", "transformers"], type=str,
                        help="model backend")
    parser.add_argument("--output_dir", "-o", default=None, type=str, help="directory to save the outputs")
    parser.add_argument("--output_format", "-f", default="all", type=_output_formats,
                        help=f"comma-separated output formats among {', '.join(OUTPUT_FORMATS)}, or all")
    parser.add_argument("--task", default="transcribe", choices=["transcribe", "translate"], type=str,
                        help="X->X speech recognition or X->English translation")
    parser.add_argument("--language", default=None,
                        choices=sorted(LANGUAGES) + sorted(k.title() for k in TO_LANGUAGE_CODE),
                        help="language spoken in the audio; detected per file when not given")
    parser.add_argument("--vad", default=False, type=_vad_option,
                        help="voice activity detection: False, or a list of (start, end) speech timestamps in seconds")
    parser.add_argument("--detect_disfluencies", default=False, type=_str2bool, help="mark disfluencies as [*] words")
    parser.add_argument("--recompute_all_timestamps", default=not TRUST_WHISPER_TIMESTAMP_BY_DEFAULT, type=_str2bool,
                        help="do not rely on Whisper's segment timestamps")
    parser.add_argument("--punctuations_with_words", default=True, type=_str2bool,
                        help="whether to include punctuations in the words")
    parser.add_argument("--temperature", default=0.0, type=float, help="temperature to use for sampling")
    parser.add_argument("--best_of", default=None if USE_EFFICIENT_BY_DEFAULT else 5, type=_optional(int),
                        help="number of candidates when sampling with non-zero temperature")
    parser.add_argument("--beam_size", default=None if USE_EFFICIENT_BY_DEFAULT else 5, type=_optional(int),
                        help="number of beams in beam search, only applicable when temperature is zero")
    parser.add_argument("--patience", default=None, type=float, help="patience of beam decoding")
    parser.add_argument("--length_penalty", default=None, type=float, help="token length penalty coefficient (alpha)")
    parser.add_argument("--suppress_tokens", default="-1", type=str,
                        help="comma-separated token ids to suppress; '-1' suppresses most special characters")
    parser.add_argument("--initial_prompt", default=None, type=str, help="text prompt for the first window of each file")
    parser.add_argument("--condition_on_previous_text", default=True, type=_str2bool,
                        help="prompt each window with the text of the previous ones")
    parser.add_argument("--fp16", default=None, type=_str2bool, help="accepted for compatibility")
    parser.add_argument("--temperature_increment_on_fallback", default=0.0 if USE_EFFICIENT_BY_DEFAULT else 0.2,
                        type=_optional(float), help="temperature step of the fallback when a decoding fails the thresholds")
    parser.add_argument("--compression_ratio_threshold", default=2.4, type=_optional(float),
                        help="gzip compression ratio above which a decoding has failed")
    parser.add_argument("--logprob_threshold", default=-1.0, type=_optional(float),
                        help="average log-probability below which a decoding has failed")
    parser.add_argument("--no_speech_threshold", default=0.6, type=_optional(float),
                        help="<|nospeech|> probability above which a failed window counts as silence")
    parser.add_argument("--threads", default=0, type=_optional(int), help="torch CPU threads")
    parser.add_argument("--compute_confidence", default=True, type=_str2bool, help="compute word confidence scores")
    parser.add_argument("--verbose", default=False, type=_str2bool, help="print the words as they are timestamped")
    parser.add_argument("--plot", default=False, action="store_true", help="plot word alignments")
    parser.add_argument("--debug", default=False, action="store_true", help="debug logging of the word alignment")

    def shortcut(values):
        class Shortcut(argparse.Action):
            def __init__(self, option_strings, dest, **kwargs):
                super().__init__(option_strings, dest, nargs=0, **kwargs)

            def __call__(self, parser, namespace, _values, option_string=None):
                for k, v in values.items():
                    setattr(namespace, k, v)
        return Shortcut

    parser.add_argument("--accurate", action=shortcut(dict(best_of=5, beam_size=5, temperature_increment_on_fallback=0.2)),
                        help="openai-whisper's defaults: best_of=5, beam_size=5, temperature_increment_on_fallback=0.2")
    parser.add_argument("--efficient", action=shortcut(dict(best_of=None, beam_size=None,
                                                            temperature_increment_on_fallback=None)),
                        help="no beam search and no sampling fallback")
    parser.add_argument("--naive", default=False, action="store_true",
                        help="two-pass strategy: transcribe, then align the words in a second decoder pass")
    args = vars(parser.parse_args(argv))
    args.pop("accurate", None)
    args.pop("efficient", None)

    temperature = args.pop("temperature")
    increment = args.pop("temperature_increment_on_fallback")
    if increment:
        temperature = tuple(float(t) for t in np.arange(temperature, 1.0 + 1e-6, increment))
    else:
        temperature = [temperature]
    files = args.pop("audio")
    model_args = dict(name=args.pop("model"), device=args.pop("device"), download_root=args.pop("model_dir"),
                      backend=args.pop("backend"))
    output = dict(output_dir=args.pop("output_dir"), output_format=args.pop("output_format"),
                  threads=args.pop("threads"), debug=args.pop("debug"))
    args["plot_word_alignment"] = args.pop("plot")
    args["naive_approach"] = args.pop("naive")
    args["remove_punctuation_from_words"] = not args.pop("punctuations_with_words")
    args["compute_word_confidence"] = args.pop("compute_confidence")
    args["trust_whisper_timestamps"] = not args.pop("recompute_all_timestamps")
    args["temperature"] = temperature
    return files, model_args, args, output


def write_outputs(result, outname, formats):
    """The files the reference's command line writes for one result: `<outname>.words.json` and the txt / vtt / srt /
    csv / tsv files of the segments and (`.words.*`) of the words."""
    import json
    from . import writers as WR
    if "json" in formats:
        with open(outname + ".words.json", "w", encoding="utf-8") as f:
            json.dump(result, f, indent=2, ensure_ascii=False)
    if "txt" in formats:
        with open(outname + ".txt", "w", encoding="utf-8") as f:
            WR.write_txt(result["segments"], file=f)
    for fmt, write in (("vtt", WR.write_vtt), ("srt", WR.write_srt)):
        if fmt in formats:
            with open(f"{outname}.{fmt}", "w", encoding="utf-8") as f:
                write(remove_keys(result["segments"], "words"), file=f)
            with open(f"{outname}.words.{fmt}", "w", encoding="utf-8") as f:
                write(flatten(result["segments"], "words"), file=f)
    for fmt, write in (("csv", write_csv), ("tsv", write_tsv)):
        if fmt in formats:
            with open(f"{outname}.{fmt}", "w", encoding="utf-8") as f:
                write(result["segments"], file=f)
            with open(f"{outname}.words.{fmt}", "w", encoding="utf-8") as f:
                write(flatten(result["segments"], "words"), file=f)


def cli(argv=None):
    """`python -m whisper_timestamped.transcribe audio [audio ...] [options]`: every file in ONE transcribe() call (their
    windows share the GPU decode batches), then the reference's outputs per file under `<output_dir>/<basename>`, or
    without --output_dir (and without --verbose) the result of each file as JSON on stdout."""
    import json
    import os
    files, model_args, options, output = parse_cli_args(argv)
    if output["threads"]:
        import torch
        torch.set_num_threads(output["threads"])
    from .model import load_model
    model = load_model(**model_args)
    logging.basicConfig()
    if output["debug"]:
        logger.setLevel(logging.DEBUG)
    out_dir = output["output_dir"]
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
    results = transcribe_timestamped(model, list(files), **options)
    for path, result in zip(files, results):
        if out_dir:
            write_outputs(result, os.path.join(out_dir, os.path.basename(path)), output["output_format"])
        elif not options["verbose"]:
            json.dump(filtered_keys(result), sys.stdout, indent=2, ensure_ascii=False)


if __name__ == "__main__":
    cli()

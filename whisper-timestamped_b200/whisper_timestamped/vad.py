"""Explicit-list voice activity: `vad=[(start, end), ...]` of transcribe() (SURVEY.md §8f row 2).

What the reference does with such a list (/root/reference/whisper_timestamped/transcribe.py): `check_vad_method`
(T.py:1870-1913) validates the pairs, `get_vad_segments` (T.py:1944-1947, 2056-2083) turns them into sample spans with
no dilatation, `remove_non_speech` (T.py:2085-2156) glues the speech spans together, the model runs on the glued
audio, and `do_convert_timestamps` (T.py:2158-2200) maps every word / segment time back to the original time axis
(T.py:341-352); the spans are reported as `speech_activity` (T.py:354-355).

The model-based detectors (silero, auditok) need packages / torch.hub downloads that do not exist offline; they raise
NotImplementedError here.  Pure host logic + tensor slicing — no kernel involved.
"""
SAMPLE_RATE = 16000


def check_vad_method(method):
    """None / False -> None; an iterable of (start, end) pairs -> list of tuples; detector names are not built."""
    if method in (None, False, "False", "false", "None", "none"):
        return None
    if not isinstance(method, (str, bool)) and hasattr(method, "__iter__"):
        pairs = []
        for pair in method:
            assert len(pair) == 2, f"Got unexpected element {pair} in the list of VAD segments. Expect (start, end) pairs"
            pairs.append(tuple(pair))
        return pairs
    raise NotImplementedError(
        f"vad={method!r}: only an explicit list of (start, end) speech timestamps is built in the H100 drop-in "
        "(silero / auditok models are not available offline)")


def speech_spans_in_samples(pairs, n_samples, sample_rate=SAMPLE_RATE):
    """Sample spans of the listed speech intervals (rounded like the reference; no dilatation for explicit lists)."""
    return [(round(s * sample_rate), round(e * sample_rate)) for (s, e) in pairs]


def remove_non_speech(audio, pairs, sample_rate=SAMPLE_RATE):
    """audio: 1-D tensor (any device).  Returns (glued speech audio, spans in seconds, converter(t, t2=None))."""
    import torch
    spans = speech_spans_in_samples(pairs, int(audio.shape[-1]), sample_rate)
    if not spans:
        spans = [(0, int(audio.shape[-1]))]            # avoid_empty_speech=True (T.py:296)
    glued = torch.cat([audio[..., s:e] for (s, e) in spans], dim=-1)
    spans_sec = [(float(s) / sample_rate, float(e) / sample_rate) for (s, e) in spans]
    return glued, spans_sec, (lambda t, t2=None: convert_timestamps(spans_sec, t, t2))


def _clamp(x, lo, hi):
    return max(lo, min(hi, x))


def convert_timestamps(spans, t, t2=None):
    """Time(s) on the glued axis -> original axis.  When a pair straddles a cut the candidate that best preserves the
    duration wins; results are rounded to 10 ms."""
    assert len(spans)
    removed = 0          # silence dropped before the current span
    glued_end = 0        # end of the current span on the glued axis
    prev_end = 0
    candidates = []
    for (a, b) in spans:
        glued_end = glued_end + (b - a)
        removed += a - prev_end
        prev_end = b
        first_in = t <= glued_end
        second_in = first_in if t2 is None else t2 <= glued_end
        if first_in or second_in:
            candidates.append([_clamp(removed + t, a, b), _clamp(removed + t2, a, b) if t2 is not None else None])
            if first_in and second_in:
                break
    if not candidates:
        candidates.append([removed + t, removed + t2 if t2 is not None else None])
    if len(candidates) > 1:
        candidates = sorted(candidates, key=lambda c: abs(abs(t2 - t) - abs(c[1] - c[0])))
    best = candidates[0]
    if t2 is None:
        return round(best[0], 2)
    return [round(x, 2) for x in best]

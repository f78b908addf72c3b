"""Host-only helpers the reference's command line uses to write a result dict to text formats
(/root/reference/whisper_timestamped/transcribe.py:2298-2323 `flatten`, `remove_keys`, `write_csv`; 3183-3199
`filtered_keys`), and the txt / srt / vtt writers it takes from openai-whisper (`get_writer(fmt).write_result` with
`highlight_words=False` and no line width or count, T.py:2982-2999).  Every layout is pinned byte for byte by the files
the reference's command line wrote, tests/expected/punctuations_* (replayed by tests/test_subtitles.py and
tests/test_cli_writers.py).
"""
import csv

KEPT_KEYS = ("text", "segments", "words", "language", "start", "end", "confidence", "language_probs", "speech_activity")


def flatten(list_of_lists, key=None):
    """All items of all sub-lists; with `key`, of `sublist[key]` (missing key = nothing)."""
    for sub in list_of_lists:
        yield from (sub.get(key, []) if key else sub)


def remove_keys(list_of_dicts, key):
    """The dicts without `key`."""
    for d in list_of_dicts:
        yield {k: v for k, v in d.items() if k != key}


def write_csv(transcript, file, sep=",", text_first=True, format_timestamps=None, header=False):
    """One row per segment (or word): text, start, end — or start, end, text with `text_first=False`."""
    fmt = format_timestamps if format_timestamps is not None else (lambda x: x)
    out = csv.writer(file, delimiter=sep)
    if header is True:
        header = ["text", "start", "end"] if text_first else ["start", "end", "text"]
    if header:
        out.writerow(header)
    for item in transcript:
        text, start, end = item["text"].strip(), fmt(item["start"]), fmt(item["end"])
        out.writerow([text, start, end] if text_first else [start, end, text])


def write_tsv(transcript, file):
    """start / end in integer milliseconds, tab separated, with a header (T.py:2976)."""
    write_csv(transcript, file, sep="\t", header=True, text_first=False, format_timestamps=lambda x: round(1000 * x))


def filtered_keys(result, keys=KEPT_KEYS):
    """The part of a result the command line prints to stdout: only `keys`, floats rounded to 2 decimals
    (`language_probs` values untouched)."""
    if isinstance(result, dict):
        return {k: (v if k == "language_probs" else filtered_keys(v, keys)) for k, v in result.items() if k in keys}
    if isinstance(result, list):
        return [filtered_keys(v, keys) for v in result]
    if isinstance(result, float):
        return round(result, 2)
    return result


def write_txt(transcript, file):
    """One line per segment: its stripped text."""
    for segment in transcript:
        print(segment["text"].strip(), file=file, flush=True)


def write_srt(transcript, file):
    """SubRip cues numbered from 1, `hh:mm:ss,mmm` times, `-->` in the text written `->`."""
    from .make_subtitles import write_srt as cues
    cues(list(transcript), file=file)


def write_vtt(transcript, file):
    """WebVTT cues, `[hh:]mm:ss.mmm` times.  The `.vtt` and `.words.vtt` files of the reference's command line start
    with the `WEBVTT` header twice; the same bytes are written here."""
    from .make_subtitles import write_vtt as cues
    print("WEBVTT\n", file=file)
    cues(list(transcript), file=file)

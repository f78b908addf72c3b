"""The command line's host-only parts: the txt / srt / vtt writers against the files the reference's own command line
wrote (tests/expected/punctuations_{yes,no}, copied by tests/golden/make_cli_writer_vectors.py), byte for byte, and the
mapping of argv to transcribe() options on invocations taken from the reference's CLI tests."""
import io
import json
import os

import pytest

from whisper_timestamped import writers as WR
from whisper_timestamped.transcribe import parse_cli_args, write_outputs

HERE = os.path.dirname(os.path.abspath(__file__))
G = os.path.join(HERE, "golden", "subtitles")
FOLDERS = ["punctuations_yes", "punctuations_no"]
STEMS = ["punctuations.mp3", "bonjour.wav"]


def _expected(folder, stem, ext):
    with open(os.path.join(G, f"{folder}_{stem}.{ext}"), "rb") as f:
        return f.read()


def _written(write, items):
    buf = io.StringIO()
    write(items, file=buf)
    return buf.getvalue().encode("utf-8")


@pytest.mark.parametrize("stem", STEMS)
@pytest.mark.parametrize("folder", FOLDERS)
def test_txt_srt_vtt_writers_match_reference_cli_outputs(folder, stem):
    result = json.load(open(os.path.join(G, f"{folder}_{stem}.words.json"), encoding="utf-8"))
    segs = result["segments"]
    assert _written(WR.write_txt, segs) == _expected(folder, stem, "txt")
    assert _written(WR.write_srt, WR.remove_keys(segs, "words")) == _expected(folder, stem, "srt")
    assert _written(WR.write_srt, WR.flatten(segs, "words")) == _expected(folder, stem, "words.srt")
    assert _written(WR.write_vtt, WR.remove_keys(segs, "words")) == _expected(folder, stem, "vtt")
    assert _written(WR.write_vtt, WR.flatten(segs, "words")) == _expected(folder, stem, "words.vtt")
    assert _expected(folder, stem, "words.vtt").startswith(b"WEBVTT\n\nWEBVTT\n\n")


@pytest.mark.parametrize("stem", STEMS)
@pytest.mark.parametrize("folder", FOLDERS)
def test_write_outputs_writes_every_reference_file(tmp_path, folder, stem):
    result = json.load(open(os.path.join(G, f"{folder}_{stem}.words.json"), encoding="utf-8"))
    out = str(tmp_path / stem)
    write_outputs(result, out, ["txt", "vtt", "srt", "tsv", "csv", "json"])
    for ext in ("txt", "srt", "vtt", "csv", "tsv", "words.srt", "words.vtt", "words.csv", "words.tsv"):
        got = open(f"{out}.{ext}", "rb").read()
        assert got.replace(b"\r\n", b"\n") == _expected(folder, stem, ext).replace(b"\r\n", b"\n"), ext
    assert json.load(open(out + ".words.json", encoding="utf-8")) == result
    os.makedirs(tmp_path / "some")
    write_outputs(result, str(tmp_path / "some" / stem), ["json", "srt"])
    assert sorted(os.listdir(tmp_path / "some")) == [f"{stem}.{e}" for e in ("srt", "words.json", "words.srt")]


DEFAULTS = dict(task="transcribe", language=None, vad=False, detect_disfluencies=False, best_of=None, beam_size=None,
                patience=None, length_penalty=None, suppress_tokens="-1", initial_prompt=None,
                condition_on_previous_text=True, fp16=None, compression_ratio_threshold=2.4, logprob_threshold=-1.0,
                no_speech_threshold=0.6, verbose=False, plot_word_alignment=False, naive_approach=False,
                remove_punctuation_from_words=False, compute_word_confidence=True, trust_whisper_timestamps=True,
                temperature=[0.0])


@pytest.mark.parametrize("argv, changed", [
    (["--model", "small", "--language", "en", "--accurate"],
     dict(language="en", best_of=5, beam_size=5, temperature=(0.0, 0.2, 0.4, 0.6, 0.8, 1.0))),
    (["--model", "small", "--language", "en", "--efficient", "--naive"], dict(language="en", naive_approach=True)),
    (["--model", "small", "--language", "en", "--temperature", "0.2", "--efficient"], dict(language="en", temperature=[0.2])),
    (["--model", "medium.en", "--efficient", "--punctuations", "False"], dict(remove_punctuation_from_words=True)),
    (["--model", "tiny", "--recompute_all_timestamps", "True"], dict(trust_whisper_timestamps=False)),
    (["--model", "small", "--language", "English", "--condition", "False", "--temperature", "0.1", "--efficient"],
     dict(language="English", condition_on_previous_text=False, temperature=[0.1])),
    (["--model", "tiny", "--compute_confidence", "False", "--vad", "[(0.5, 3.0), (4, 9.5)]", "--plot"],
     dict(compute_word_confidence=False, vad=[(0.5, 3.0), (4, 9.5)], plot_word_alignment=True)),
])
def test_argv_to_transcribe_options(argv, changed):
    files, model_args, options, output = parse_cli_args(["a.wav", "dir/b.wav"] + argv)
    assert files == ["a.wav", "dir/b.wav"]
    assert model_args == dict(name=argv[1], device=None, download_root=None, backend="openai-whisper")
    temperature = options.pop("temperature")
    expected = dict(DEFAULTS, **changed)
    want_t = expected.pop("temperature")
    assert type(temperature) is type(want_t) and temperature == pytest.approx(want_t)
    assert options == expected
    assert output == dict(output_dir=None, output_format=["txt", "vtt", "srt", "tsv", "csv", "json"], threads=0,
                          debug=False)


def test_argv_output_settings_and_model():
    files, model_args, options, output = parse_cli_args(
        ["x.wav", "--model", "synthetic:tiny", "--model_dir", "/m", "--backend", "transformers", "-o", "out",
         "-f", "json,srt", "--threads", "3", "--debug", "--verbose", "True"])
    assert model_args == dict(name="synthetic:tiny", device=None, download_root="/m", backend="transformers")
    assert output == dict(output_dir="out", output_format=["json", "srt"], threads=3, debug=True)
    assert options["verbose"] is True
    with pytest.raises(SystemExit):
        parse_cli_args(["x.wav", "-f", "json,doc"])
    with pytest.raises(SystemExit):
        parse_cli_args([])

"""transcribe(model, [audio, ...]) and the command line on the GPU: one call over several recordings against the unmodified
reference run on each recording alone (tests/golden/multi/*.json), with the GPU tolerances of tests/test_gpu_model.py,
in decode rounds and with continuous batching; the windows of different recordings must share decode batches."""
import glob
import json
import os
import subprocess
import sys
import wave

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MULTI = sorted(glob.glob(os.path.join(HERE, "golden", "multi", "*.json")))
_MODELS = {}

pytestmark = pytest.mark.gpu


def _load(g):
    import whisper_timestamped as wt
    key = (g["model"], g["model_seed"], json.dumps(g["model_kwargs"], sort_keys=True))
    if key not in _MODELS:
        _MODELS.clear()
        torch.cuda.empty_cache()
        _MODELS[key] = wt.load_model(f"synthetic:{g['model']}", device="cuda:0", synthetic_seed=g["model_seed"],
                                     synthetic_kwargs=g["model_kwargs"])
    return _MODELS[key]


def _record_batches(eng):
    """Wraps the engine's decode drivers: the stream ids of the windows of every decode batch (rounds), or of the
    windows a continuous-batching run starts with, go to the returned list."""
    seen = []
    dw, ds = eng.decode_windows, eng.decode_stream

    def decode_windows(jobs, setup):
        seen.append([j["stream"] for j in jobs])
        return dw(jobs, setup)

    def decode_stream(jobs, setup, feed, collected=None):
        seen.append([j["stream"] for j in jobs])
        return ds(jobs, setup, feed, collected=collected)

    eng.decode_windows, eng.decode_stream = decode_windows, decode_stream
    return seen


@pytest.mark.parametrize("continuous", [False, True], ids=["rounds", "continuous"])
@pytest.mark.parametrize("path", MULTI, ids=[os.path.basename(p)[:-5] for p in MULTI])
def test_one_call_over_files_matches_reference_per_file(path, continuous):
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from test_host_e2e import CaptureWarnings, compare, norm_warnings
    g = json.load(open(path))
    gm = _load(g)
    eng = CudaEngine(gm)
    seen = _record_batches(eng)
    with CaptureWarnings() as cap:
        res = wt.transcribe(gm, [synthetic_speech(*a) for a in g["audios"]], engine=eng, continuous_batching=continuous,
                            **g["transcribe_kwargs"])
    assert len(res) == len(g["files"])
    for r, item in zip(res, g["files"]):
        compare(r, item["result"], conf_tol=2e-3, time_tol=0.0, prob_tol=1e-3)
    assert norm_warnings(cap.messages) == norm_warnings([m for item in g["files"] for m in item["warnings"]])
    kw = g["transcribe_kwargs"]
    if not (kw.get("temperature") or 0) > 0:
        # one-pass strategy: the first windows of all files are decoded together
        assert any(len(set(b)) > 1 for b in seen), seen


def _write_wav(path, audio):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes((np.clip(audio, -1, 1) * 32767).astype(np.int16).tobytes())


def test_cli_writes_the_list_call_results(tmp_path):
    import whisper_timestamped as wt
    from whisper_timestamped import writers as WR
    from whisper_timestamped.synthetic_audio import synthetic_speech
    paths = []
    for k, (dur, seed) in enumerate([(12.0, 5), (40.0, 6), (4.0, 7)]):
        p = tmp_path / f"rec{k}.wav"
        _write_wav(p, synthetic_speech(dur, seed))
        paths.append(str(p))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "whisper-timestamped_b200"),
                                                       os.environ.get("PYTHONPATH", "")]))
    out = tmp_path / "out"
    cmd = [sys.executable, "-m", "whisper_timestamped.transcribe", *paths, "--model", "synthetic:tiny", "--language", "en"]
    subprocess.run(cmd + ["-o", str(out)], check=True, env=env, cwd=str(tmp_path))
    gm = wt.load_model("synthetic:tiny", device="cuda:0")
    results = wt.transcribe(gm, paths, language="en")
    for p, res in zip(paths, results):
        stem = os.path.join(str(out), os.path.basename(p))
        assert json.load(open(stem + ".words.json", encoding="utf-8")) == json.loads(json.dumps(res))
        segs = res["segments"]
        for ext, write, items in (("txt", WR.write_txt, segs),
                                  ("srt", WR.write_srt, WR.remove_keys(segs, "words")),
                                  ("words.srt", WR.write_srt, WR.flatten(segs, "words")),
                                  ("vtt", WR.write_vtt, WR.remove_keys(segs, "words")),
                                  ("words.vtt", WR.write_vtt, WR.flatten(segs, "words")),
                                  ("csv", WR.write_csv, segs),
                                  ("words.csv", WR.write_csv, WR.flatten(segs, "words")),
                                  ("tsv", WR.write_tsv, segs),
                                  ("words.tsv", WR.write_tsv, WR.flatten(segs, "words"))):
            want = tmp_path / "want"
            with open(want, "w", encoding="utf-8") as f:
                write(items, file=f)
            assert open(f"{stem}.{ext}", "rb").read() == open(want, "rb").read(), (p, ext)
    # stdout mode: filtered_keys of each file, as JSON, one after the other
    std = subprocess.run(cmd, check=True, env=env, cwd=str(tmp_path), capture_output=True, text=True).stdout
    want = "".join(json.dumps(WR.filtered_keys(json.loads(json.dumps(r))), indent=2, ensure_ascii=False) for r in results)
    assert std == want

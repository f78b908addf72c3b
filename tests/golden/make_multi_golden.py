"""Generates tests/golden/multi/<case>.json: goldens of `transcribe(model, [audio, ...])`.  For every case the UNMODIFIED
reference (/root/reference/whisper_timestamped, over the oracle's stand-ins, as tests/golden/make_e2e_golden.py) runs
once per file with the shared options, exactly as its command line loops over its files (T.py:3131-3139).  Build
container only; the JSON fixtures are committed.

    python tests/golden/make_multi_golden.py [case ...]

Each fixture holds the model recipe, the shared transcribe kwargs, the audio recipes (duration, seed) and per file the
reference's result, its warnings, its stdout when `verbose` is set, and the smallest top-2 gap of the product's greedy
decode of that file through the CPU stand-in (tests/golden/check_margins.py; not computed for sampling, nor for
large-v3, whose windows take minutes each through the float32 stand-in).

Language detection: the synthetic tiny model detects "hi" on every audio seed 0-49 at 8, 20, 35 and 50 s, so the
detection cases cannot mix two detected languages; they keep one language (a batch of several detected files, each
with its own detection mel and `language_probs`).
"""
import json
import os
import subprocess
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "multi")
BENCH_KW = {"ts_offset": 4.5, "eot_logit": 14.5}        # == bench.py SYNTH_KW

DETECT_FILES = [(20.0, 71), (35.0, 13), (8.0, 72), (50.0, 73)]
CASES = {
    # name: (model, model kwargs, [(duration, audio seed)], transcribe kwargs)
    # long files chain their prompts while the short ones finish: follow-up windows share batches with first windows
    "tiny_en": ("tiny", {}, [(3.3, 51), (95.0, 52), (12.0, 53), (61.0, 54), (7.0, 55), (40.0, 56)], {"language": "en"}),
    "tiny_detect": ("tiny", {}, DETECT_FILES, {}),
    "tiny_verbose_detect": ("tiny", {}, DETECT_FILES, {"verbose": True}),
    # sampling: every file starts from the same seeded generator state, as separate calls do
    "tiny_bestof": ("tiny", {}, [(20.0, 81), (35.0, 82)], {"language": "en", "temperature": 0.3, "best_of": 3}),
    # bench recipe: the 45-s audio of e2e_large_v3_45s and two more files
    "large_v3_bench": ("large-v3", BENCH_KW, [(45.0, 31), (12.0, 91), (70.0, 92)], {"language": "en"}),
}


def run_case(case):
    import importlib.util
    sys.path.insert(0, HERE)
    spec = importlib.util.spec_from_file_location("make_e2e_golden", os.path.join(HERE, "make_e2e_golden.py"))
    E = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(E)                    # the reference on the oracle's stand-ins
    mname, mkw, audios, tkw = CASES[case]
    model = E.build_model(mname, **mkw)
    files = []
    t0 = time.time()
    for dur, aseed in audios:
        res, warns = E.run_reference(model, E.sa.synthetic_speech(dur, seed=aseed), **tkw)
        item = {"audio": [dur, aseed], "result": res, "warnings": warns}
        if tkw.get("verbose") is not None:
            item["stdout"] = E.run_reference.stdout
        files.append(item)
        print(f"  {case} {dur}s/{aseed}: {len(res['segments'])} segments, {len(warns)} warnings, "
              f"{time.time() - t0:.0f}s", flush=True)
    out = {"case": case, "model": mname, "model_seed": 1234, "model_kwargs": mkw, "transcribe_kwargs": tkw,
           "audios": [list(a) for a in audios], "reference_version": E.ref.__version__,
           "cpu_seconds": round(time.time() - t0, 2), "files": files}
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, f"{case}.json")
    with open(path, "w") as f:
        json.dump(out, f, ensure_ascii=False)
        f.write("\n")
    return path


def add_margins(path):
    """Runs in its own process: the product package has the reference's import name."""
    sys.path.insert(0, HERE)
    import check_margins
    g = json.load(open(path))
    kw = g["transcribe_kwargs"]
    if (kw.get("temperature") or 0) > 0 or "large" in g["model"]:
        return
    for item in g["files"]:
        one = dict(g, audio=item["audio"])
        gap, w, r = check_margins.min_gap(one)
        item["min_top2_gap"] = {"gap": gap, "window": w, "row": r}
        print(f"  {g['case']} {item['audio']}: gap {gap:.2e} (window {w}, row {r})", flush=True)
    with open(path, "w") as f:
        json.dump(g, f, ensure_ascii=False)
        f.write("\n")


def main():
    if sys.argv[1:2] == ["--margins"]:
        add_margins(sys.argv[2])
        return
    for case in sys.argv[1:] or list(CASES):
        path = run_case(case)
        subprocess.run([sys.executable, __file__, "--margins", path], check=True)


if __name__ == "__main__":
    main()

"""Generates tests/golden/heads/*.json: the UNMODIFIED reference (whisper_timestamped, as make_e2e_golden.py loads it) on CPU with
`word_alignment_most_top_layers=k` (every head of the top k decoder layers) and with the default head set of a model
that has no alignment-head table (every head of the top half of the layers, upstream's default for a fine-tuned
`.pt`).  Same recipe and stand-ins as make_e2e_golden.py; the audio seeds are those of existing goldens, so tokens
and segments equal theirs and only word times and confidences differ.

    python tests/golden/make_heads_golden.py [case ...]
"""
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_e2e_golden as E  # noqa: E402

OUT = os.path.join(HERE, "heads")

# name: (model, model kwargs, audio (duration, seed), chunk seconds or None, table heads?, transcribe kwargs)
CASES = {
    "tiny_top2": ("tiny", {}, (75.0, 11), None, True, {"language": "en", "word_alignment_most_top_layers": 2}),
    # k above the number of layers: clipped to every head of every layer
    "tiny_top9": ("tiny", {}, (60.0, 113), None, True, {"language": "en", "condition_on_previous_text": False,
                                                         "word_alignment_most_top_layers": 9}),
    "tiny_top1_naive": ("tiny", {}, (75.0, 21), None, True, {"language": "en", "naive_approach": True,
                                                              "temperature": 0.0, "word_alignment_most_top_layers": 1}),
    "tiny_top2_disfluencies": ("tiny", {}, (60.0, 12), None, True, {"language": "en", "detect_disfluencies": True,
                                                                     "word_alignment_most_top_layers": 2}),
    "tiny_top2_chunks": ("tiny", {}, (100.0, 41), 30.0, True, {"language": "en", "word_alignment_most_top_layers": 2}),
    # a checkpoint without an alignment-head table: the top half of the layers (tiny: layers 2-3, 12 heads)
    "tiny_default_heads": ("tiny", {}, (75.0, 11), None, False, {"language": "en"}),
    # large-v3 shape without a table: 320 heads
    "large_v3_default_45s": ("large-v3", E.BENCH_KW, (45.0, 31), None, False, {"language": "en"}),
    # the first 5 minutes of the bench workload, per 30-s cut, top 6 layers (120 heads)
    "large_v3_top6_bench300": ("large-v3", E.BENCH_KW, (300.0, 1234), 30.0, True,
                               {"language": "en", "word_alignment_most_top_layers": 6}),
}


def build_model(name, table, **kw):
    if table:
        return E.build_model(name, **kw)
    dims = E.zoo.DIMS[name]
    model = E.whisper.Whisper(E.whisper.ModelDimensions(**dims.asdict()))   # keeps upstream's top-half default
    model.load_state_dict(E.zoo.synthetic_state_dict(dims, seed=1234, **kw))
    return model.eval()


def main():
    os.makedirs(OUT, exist_ok=True)
    for case in sys.argv[1:] or list(CASES):
        mname, mkw, (dur, aseed), chunk_s, table, tkw = CASES[case]
        model = build_model(mname, table, **mkw)
        audio = E.sa.synthetic_speech(dur, seed=aseed)
        out = {"case": case, "model": mname, "model_seed": 1234, "model_kwargs": mkw, "audio": [dur, aseed],
               "table_heads": table, "transcribe_kwargs": tkw, "reference_version": E.ref.__version__}
        t0 = time.time()
        if chunk_s is None:
            res, warns = E.run_reference(model, audio, **tkw)
            out.update(warnings=warns, result=res)
        else:
            step = int(round(chunk_s * 16000))
            cuts = []
            for s in range(0, len(audio), step):
                res, warns = E.run_reference(model, audio[s:s + step], condition_on_previous_text=False, **tkw)
                cuts.append({"offset": s / 16000.0, "result": res, "warnings": warns})
            out.update(chunks=chunk_s, cuts=cuts)
        out["cpu_seconds"] = round(time.time() - t0, 2)
        with open(os.path.join(OUT, f"{case}.json"), "w") as f:
            json.dump(out, f, indent=1, ensure_ascii=False)
        print(f"{case}: {out['cpu_seconds']}s", flush=True)
        del model


if __name__ == "__main__":
    main()

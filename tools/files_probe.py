"""Many recordings: one transcribe() call per file vs ONE list call (windows of all files in shared decode batches), in
decode rounds and with continuous batching.  Workload: N seeded synthetic files of mixed durations (default 64 files of
3-120 s) on large-v3 with the bench recipe.  The arms alternate in one process (--reps rounds); each arm's wall time is
taken between device synchronisations.  Prints one JSON line: per arm the best and median seconds, audio-seconds/s,
windows and decode batches; whether tokens and word times are identical across the arms; GPU name and power limit.

    python tools/files_probe.py [--files 64] [--min-s 3] [--max-s 120] [--reps 2] [--model synthetic:large-v3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "whisper-timestamped_b200"))
BENCH_KW = {"ts_offset": 4.5, "eot_logit": 14.5}        # == bench.py SYNTH_KW


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        power = float(q.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        power = None
    return name, power


def fingerprint(results):
    """Tokens and word times of every file, in order."""
    return [[(s["tokens"], [(w["start"], w["end"]) for w in s.get("words", [])]) for s in r["segments"]] for r in results]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="synthetic:large-v3")
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--min-s", type=float, default=3.0)
    ap.add_argument("--max-s", type=float, default=120.0)
    ap.add_argument("--seed", type=int, default=2024)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.synthetic_audio import synthetic_speech
    model = wt.load_model(args.model, device="cuda:0",
                          synthetic_kwargs=BENCH_KW if args.model.startswith("synthetic:") else None)
    rng = np.random.default_rng(args.seed)
    durations = rng.uniform(args.min_s, args.max_s, args.files).round(1)
    audios = [synthetic_speech(float(d), seed=args.seed + k) for k, d in enumerate(durations)]
    total_s = float(durations.sum())
    eng = CudaEngine(model)
    counts = {}
    dw, ds = eng.decode_windows, eng.decode_stream

    def decode_windows(jobs, setup):
        counts["batches"] += 1
        counts["windows"] += len(jobs)
        return dw(jobs, setup)

    def decode_stream(jobs, setup, feed, collected=None):
        def fed(job, rec):
            counts["windows"] += 1
            return feed(job, rec)

        def coll():
            counts["batches"] += 1          # collections: windows finished together
            if collected is not None:
                collected()
        return ds(jobs, setup, fed, collected=coll)

    eng.decode_windows, eng.decode_stream = decode_windows, decode_stream
    kw = dict(language="en", engine=eng)
    arms = {
        "per_file": lambda: [wt.transcribe(model, a, continuous_batching=False, **kw) for a in audios],
        "list_rounds": lambda: wt.transcribe(model, audios, continuous_batching=False, **kw),
        "list_continuous": lambda: wt.transcribe(model, audios, continuous_batching=True, **kw),
    }
    times = {k: [] for k in arms}
    stats, prints = {}, {}
    for rep in range(args.reps + 1):                 # rep 0 warms up (graphs, sessions, allocator)
        for name, run in arms.items():
            counts.update(batches=0, windows=0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = run()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if rep:
                times[name].append(dt)
            stats[name] = dict(counts)
            prints[name] = fingerprint(res)
    gpu, power = gpu_info()
    out = dict(probe="files", model=args.model, files=args.files, audio_s=round(total_s, 1),
               durations_s=[args.min_s, args.max_s], reps=args.reps, gpu=gpu, power_limit_w=power,
               identical=all(prints[k] == prints["per_file"] for k in prints), arms={})
    for name in arms:
        best = min(times[name])
        out["arms"][name] = dict(best_s=round(best, 3), median_s=round(float(np.median(times[name])), 3),
                                 audio_s_per_s=round(total_s / best, 1), **stats[name])
    print(json.dumps(out))


if __name__ == "__main__":
    main()

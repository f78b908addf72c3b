"""Alignment-head probe: large-v3 with the bench recipe on the first 10 minutes of the bench audio in 30-s chunks, at
N = 10 (the official heads), 120 (`word_alignment_most_top_layers=6`) and 320 (every head of the top half: the default
of a checkpoint without a table).  Per head set: audio-sec/s, stage_ms() per stage, peak allocated memory, the
auto-sized decode batch, and the time of both attention-prep row kernels (serial over heads, head-parallel) on the
same alignment batches, with CUDA events.  Writes JSON (card name and power limit read in the same run).

    python tools/heads_probe.py --minutes 10 --out /tmp/heads_probe.json
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
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:                                     # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=int, default=10)
    ap.add_argument("--sets", default="10,120,320")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import whisper_timestamped as wt
    from whisper_timestamped import alignment as A
    from whisper_timestamped import engine as E
    from whisper_timestamped import model_zoo as zoo
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from bench import SYNTH_KW
    m = wt.load_model("synthetic:large-v3", device="cuda", synthetic_kwargs=SYNTH_KW)
    audio = np.concatenate([synthetic_speech(300.0, seed=1234 + k) for k in range((args.minutes + 4) // 5)])
    audio = audio[:args.minutes * 60 * 16000]
    dur = len(audio) / 16000
    eng = m.engine()
    L, H = m.dims.n_text_layer, m.dims.n_text_head
    sets = {10: None, 120: [(l, h) for l in range(L - 6, L) for h in range(H)],
            320: zoo.default_alignment_heads(m.dims)}
    prep_ms = {}

    def timed_prep(qk, plan, cost=None, d_segs=None, kernel=0):
        for k in (1, 2):                                       # both row kernels on this batch, then the chosen one
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            A.attn_prep(qk, plan, kernel=k)
            b.record()
            prep_ms.setdefault(k, []).append((a, b))
        return A.attn_prep(qk, plan, cost, d_segs, kernel)

    out = {"card": card(), "audio_seconds": dur, "runs": []}
    for n in [int(x) for x in args.sets.split(",")]:
        heads = sets[n]
        kw = dict(word_alignment_most_top_layers=6) if n == 120 else {}
        orig = E.attn_prep
        E.attn_prep = timed_prep
        try:
            if n == 320:                                       # transcribe() resets the model's heads: keep 320
                m.heads = heads
            wt.transcribe(m, audio[:30 * 16000], language="en", chunks=30.0, **kw)      # warm-up
            prep_ms.clear()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            eng.profile = True
            eng.stage_ms()
            t0 = time.time()
            wt.transcribe(m, audio, language="en", chunks=30.0, **kw)
            torch.cuda.synchronize()
            dt = time.time() - t0
            stages = eng.stage_ms()
            eng.profile = False
        finally:
            E.attn_prep = orig
            m.heads = sorted(zoo.ALIGNMENT_HEADS["large-v3"])
        from whisper_timestamped.windows import make_decode_setup
        from whisper_timestamped.tokenizer import get_tokenizer
        setup = make_decode_setup(get_tokenizer(True, num_languages=m.num_languages, language="en"), m.dims.n_text_ctx)
        run = {"N": n, "audio_sec_per_s": round(dur / dt, 2), "wall_s": round(dt, 3),
               "stage_ms": {k: round(v, 2) for k, v in stages.items()},
               "max_memory_allocated": torch.cuda.max_memory_allocated(), "batch_limit": eng.batch_limit(setup),
               "prep_ms": {("serial" if k == 1 else "head_parallel"): round(sum(a.elapsed_time(b) for a, b in v), 3)
                           for k, v in prep_ms.items()}}
        print(json.dumps(run), flush=True)
        out["runs"].append(run)
    eng.set_alignment_heads(None)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()

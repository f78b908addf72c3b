"""Encoder probe: one AudioEncoder pass over B synthetic 30-s windows (large-v3 by default); prints the CUDA-event
time, or serves as the target of an ncu launch list:
  ncu --cache-control none --metrics gpu__time_duration.sum --csv ... python tools/encoder_probe.py --windows 32 --reps 1
--profile FILE: one more pass under torch.profiler (CUDA activities), its kernel table written to FILE."""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "whisper-timestamped_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="synthetic:large-v3")
    ap.add_argument("--windows", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    m = wt.load_model(args.model, device="cuda")
    eng = CudaEngine(m, max_batch=args.windows)
    mel = torch.randn(3000 * args.windows, m.dims.n_mels, device="cuda") * 0.3
    jobs = [dict(mel=mel, seek=3000 * i, segment_size=3000) for i in range(args.windows)]
    xa = eng.encode(jobs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        xa = eng.encode(jobs)
    e1.record()
    torch.cuda.synchronize()
    print(f"encode {args.windows} windows: {e0.elapsed_time(e1) / args.reps:.1f} ms  ({e0.elapsed_time(e1) / args.reps / args.windows:.2f} ms/window)")
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.encode(jobs)
            torch.cuda.synchronize()
        table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=20, max_name_column_width=60)
        with open(args.profile, "w") as f:
            f.write(table)
        print(table)


if __name__ == "__main__":
    main()

"""Decode-step probe: milliseconds per decode step of a model at a fixed number of active windows, for the two step
implementations that share the session state:
  graph    : the per-operator step (tensor-core skinny GEMMs, one kernel per operator) replayed as ONE CUDA graph
  lean_mma : the lean small-batch step (wts_decode_step_kernels, <= 32 active windows) replayed as ONE CUDA graph

  python tools/step_probe.py --active 128,32,16,8,4,1 --cap 128 --steps 24
  ncu ... python tools/step_probe.py --eager --steps 2        (plain launches, for an ncu launch list)
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "whisper-timestamped_b200"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="synthetic:large-v3")
    ap.add_argument("--cap", type=int, default=128)
    ap.add_argument("--active", type=str, default="128,32,16,8,4,1")
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--eager", action="store_true")
    ap.add_argument("--only", default="graph,lean_mma")
    args = ap.parse_args()
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.tokenizer import get_tokenizer
    from whisper_timestamped.windows import make_decode_setup

    m = wt.load_model(args.model, device="cuda")
    eng = CudaEngine(m, max_batch=args.cap, small_batch_rows=32)
    tok = get_tokenizer(m.is_multilingual, num_languages=m.num_languages, language="en", task="transcribe")
    setup = make_decode_setup(tok, m.dims.n_text_ctx)
    ses = eng._decoder_session(setup, args.cap)
    cap = ses["cap"]
    g = torch.Generator(device="cuda").manual_seed(1)
    for li in range(m.dims.n_text_layer):
        for name in ("ck", "cv"):
            t = ses["st8"][name][li]
            t.copy_((torch.randn(t.shape, device="cuda", generator=g) * 0.5).to(t.dtype))
        if ses["st8"]["ckal"][li] is not None:          # layers without alignment heads have no float32 K copy
            ses["st8"]["ckal"][li].normal_(0, 0.5, generator=g)
    ses["suppress"].zero_()
    ses["suppress"][tok.eot] = 1                 # keep every window alive for the whole probe
    ses["blank"].zero_()
    prompt = list(tok.sot_sequence)
    P = len(prompt)

    def reset(n_active):
        tokens = np.zeros((cap, m.dims.n_text_ctx + 1), dtype=np.int32)
        tokens[:, :P] = prompt
        tokens[:, P:P + 8] = 1000
        ses["tokens"].copy_(torch.from_numpy(tokens))
        ses["n_tokens"].copy_(torch.from_numpy(np.full(cap, P + 8, dtype=np.int32)))
        ses["n_prompt"].copy_(torch.from_numpy(np.full(cap, P, dtype=np.int32)))
        dn = np.ones(cap, dtype=np.int32)
        dn[:n_active] = 0
        ses["done"].copy_(torch.from_numpy(dn))

    out = {}
    for n_active in [int(a) for a in args.active.split(",")]:
        res = {}
        reset(n_active)
        if args.eager:
            for _ in range(args.steps):
                eng._step(ses)
            torch.cuda.synchronize()
            continue
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if "graph" in args.only:
            graph = eng._step_graph(ses)
            for _ in range(3):
                graph.replay()
            e0.record()
            for _ in range(args.steps):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            res["graph_ms_per_step"] = round(e0.elapsed_time(e1) / args.steps, 3)
        if "lean_mma" in args.only.split(",") and ses["steps"] is not None and n_active <= eng.small_batch_rows:
            reset(n_active)
            graph = eng._lean_graph(ses, n_active)
            for _ in range(3):
                graph.replay()
            e0.record()
            for _ in range(args.steps):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            res["lean_mma_ms_per_step"] = round(e0.elapsed_time(e1) / args.steps, 3)
        out[n_active] = res
        print(f"active {n_active:4d} / cap {cap}: {res}", flush=True)
    print(json.dumps({"model": args.model, "cap": cap, "steps": args.steps, "ms": out}))


if __name__ == "__main__":
    main()

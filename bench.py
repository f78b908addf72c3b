"""bench.py — measures the flagship workload and prints one JSON line per run.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--workload e2e|align] [--impl ours|reference]
                    [--dump-outputs DIR]

Workloads
  e2e   : (default) BASELINE.json metric — audio-seconds/second of whisper_timestamped.transcribe() for
          large-v3 on 1 h of synthetic 16 kHz audio cut into independent 30-s chunks (config 3), word
          timestamps + confidences on; N GPUs shard the chunks (strong scaling) and gather the JSON.
  align : SURVEY.md §8(d) alignment micro-benchmark — a batch of synthetic alignment problems
          (N=10 heads, qk ~ 3*N(0,1) + monotone ridge) through wts_attn_prep_batch +
          wts_dtw_batch; reports the DTW kernel's algorithmic GB/s against the HBM peak.

--dump-outputs DIR writes what the timed path returned in its last timed step as DIR/<name>.npy (float64, 64 MB at
most: a larger output is written as a fixed seeded sample), so that two builds can be compared output for output: the
inputs are seeded and identical from run to run.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "whisper-timestamped_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402


def measured_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            d = json.load(f)
        return {"hbm_gbs": float(d["hbm_gbs"]), "bf16_tflops": float(d["bf16_tflops"]),
                "bf16_tflops_sustained": float(d.get("bf16_tflops_sustained", d["bf16_tflops"])),
                "source": "measured"}
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "source": "data sheet (H100 SXM)"}


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.index = index
        self.samples = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "100",
                 "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            parts = [x.strip() for x in line.split(",")]
            if len(parts) >= 7:
                self.samples.append(parts)

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        for p in self.samples:
            try:
                sm.append(float(p[0]))
                mx = float(p[1])
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), p[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


# ----------------------------------------------------------------------------- align workload

def make_align_batch(nseg, T, F, N, seed, device, rows_per_window=216):
    """Synthetic alignment problems per SURVEY.md §8(d): qk ~ 3*N(0,1) + 6*exp(-((f - F*t/T)/8)^2)."""
    import torch
    rows_per_window = max(rows_per_window, T)
    per_win = rows_per_window // T
    nwin = (nseg + per_win - 1) // per_win
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    qk = torch.empty((nwin, N, rows_per_window, 1500), dtype=torch.float32, device=device)
    qk.normal_(0.0, 3.0, generator=g)
    items = []
    f0 = min(100, 1500 - F)
    tt = torch.arange(T, device=device, dtype=torch.float32)[:, None]
    ff = torch.arange(F, device=device, dtype=torch.float32)[None, :]
    ridge = 6.0 * torch.exp(-((ff - F * (tt + 0.5) / T) / 8.0) ** 2)
    for k in range(nseg):
        w, r = divmod(k, per_win)
        items.append((w, r * T, None, T, f0, F, 0))
    for r in range(per_win):
        qk[:, :, r * T:(r + 1) * T, f0:f0 + F] += ridge
    return qk, items


def bytes_dtw(T, F):
    # SURVEY.md §8(d): read f32 cost once + 1 direction byte per cell + backtrack reads + jumps
    return 5 * T * F + (T + F) + 4 * (T + 1)


def bytes_prep(N, T, F):
    return 4 * N * T * F + 4 * T * F


def dtw_kernel_name(nseg, T):
    """Which DTW kernel wts_dtw_batch_sized picks for a batch of nseg single-strip matrices (csrc/dtw.cu)."""
    lane_min = int(os.environ.get("WTS_DTW_LANE_MIN", "8192"))
    if lane_min > 0 and nseg >= lane_min and T <= 32:
        g = int(os.environ.get("WTS_DTW_LANE_G", "2"))
        nc = 2 if g == 4 else int(os.environ.get("WTS_DTW_LANE_NC", "4"))
        return "dtw_lane_kernel<%d,%d,%d>" % (8 if T <= 8 else 16 if T <= 16 else 24 if T <= 24 else 32, nc, g)
    return "dtw_small_kernel<32,1>" if T <= 31 else "dtw_warp_kernel<float>"


def run_align(args, rank, world):
    import torch
    from whisper_timestamped.alignment import plan_segments, attn_prep, dtw, dtw_descriptors, _segs_to_device
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    T, F, N, nseg = args.align_T, args.align_F, 10, args.align_batch
    qk, items = make_align_batch(nseg, T, F, N, 1234 + rank, dev)
    plan = plan_segments(items, nonpositive=True)
    d_segs = _segs_to_device(plan.segs, dev)
    cost = torch.empty(plan.cost_elems, dtype=torch.float32, device=dev)
    ws = (torch.empty(plan.dir_words, dtype=torch.int32, device=dev),
          torch.empty(plan.bnd_doubles, dtype=torch.float64, device=dev))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_prep, t_dtw = [], []
    d_segs_dtw = dtw_descriptors(plan, dev)          # descriptors are resident: the events bracket kernels only
    jumps_buf = torch.empty(plan.jumps_elems, dtype=torch.int32, device=dev)

    def step(record):
        ev[0].record()
        attn_prep(qk, plan, cost=cost, d_segs=d_segs)
        ev[1].record()
        out = dtw(cost, plan, workspace=ws, d_segs=d_segs_dtw, jumps=jumps_buf)
        ev[2].record()
        if record:
            torch.cuda.synchronize()
            t_prep.append(ev[0].elapsed_time(ev[1]))
            t_dtw.append(ev[1].elapsed_time(ev[2]))
        return out

    for _ in range(args.warmup):
        step(False)
    torch.cuda.synchronize()
    sampler = ClockSampler(dev.index or 0)
    if rank == 0:
        sampler.start()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = step(True)
    e1.record()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    total_ms = e0.elapsed_time(e1)
    clocks = sampler.stop() if rank == 0 else None
    # what the last timed step computed, copied out before the host-buffer loop below reuses the cost buffer
    dumped = (align_dump_arrays(out["jumps"], cost, nseg, T)
              if rank == 0 and args.dump_outputs and args.workload == "align" else None)
    # host-buffer e2e: qk slices are device-resident products of the decoder in the real pipeline, so the
    # host-facing e2e of this micro-workload = descriptors H2D + jumps D2H each step
    e2e_t = []
    for _ in range(max(1, min(3, args.steps))):
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        d = _segs_to_device(plan.segs, dev)
        attn_prep(qk, plan, cost=cost, d_segs=d)
        o = dtw(cost, plan, workspace=ws)
        jh = o["jumps"].cpu()
        e2e_t.append(time.perf_counter() - t1)
    ms_dtw = float(np.mean(t_dtw))
    ms_prep = float(np.mean(t_prep))
    alg = nseg * bytes_dtw(T, F)
    peaks = measured_peaks()
    achieved = alg / (ms_dtw * 1e-3) / 1e9
    res = {
        "ms_total": total_ms / args.steps, "ms_dtw": ms_dtw, "ms_prep": ms_prep, "wall_s": wall,
        "dtw_gbs": achieved, "prep_gbs": nseg * bytes_prep(N, T, F) / (ms_prep * 1e-3) / 1e9,
        "segments_per_s": nseg / (total_ms / args.steps * 1e-3), "clocks": clocks,
        "e2e_segments_per_s": nseg / float(np.median(e2e_t)),
        "h2d": int(plan.segs.nbytes), "d2h": int(plan.jumps_elems * 4),
        "peaks": peaks, "alg_bytes": alg, "jumps_checksum": int(out["jumps"].sum().item()),
        "outputs": dumped,
    }
    return res


def cpu_baseline_align(args):
    """Oracle (kind 'port') on a bounded sample of the same workload, single host thread."""
    import torch
    import oracle
    from oracle.prep import attn_cost
    T, F, N = args.align_T, args.align_F, 10
    n = 48
    g = torch.Generator().manual_seed(99)
    qk = torch.empty((N, T, 1500)).normal_(0, 3.0, generator=g).numpy()
    t0 = time.perf_counter()
    for _ in range(n):
        c = attn_cost(qk, 100, 100 + F)
        oracle.dtw_symmetric1(c)
    dt = time.perf_counter() - t0
    return {"value": n / dt, "unit": "segments/s", "cores": 1, "kind": "port",
            "sample": f"{n} segments T={T} F={F} N={N}: scipy median + torch CPU softmax/mean/norm + oracle DTW (C)"}


# ------------------------------------------------------------------------------- e2e workload

# Synthetic-weight recipe used by both arms (tools/recipe_scan.py): with these offsets greedy decoding of the
# synthetic large-v3 behaves like speech — ~80 % of the windows end with <|endoftext|>, ~75 sampled tokens and
# 3-4 closed segments per window (the zoo defaults were tuned on the tiny model and leave most large-v3 windows
# running into the 224-token limit).
RECIPES = {
    "default": {"ts_offset": 4.5, "eot_logit": 14.5},
    # denser text (VERDICT r1 #7: the reference's own goldens hold ~115 tokens per 30-s window, the default recipe ~45):
    # picked with tools/recipe_scan.py; reported as a second line (`--recipe dense`), never instead of the default
    "dense": {"ts_offset": 6.0, "eot_logit": 13.0},       # ~116 decoded tokens per window, 71 % end with <|endoftext|>
}
SYNTH_KW = dict(RECIPES["default"])


def _dist_setup():
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    return rank, world, local


def _pkg_module(name):
    """A pure-python module of the product package loaded BY FILE PATH (model_zoo, synthetic_audio): the reference arm
    needs the synthetic recipe but must never import the product package (that would load libwts.so)."""
    import importlib.util
    key = "wts_bench_" + name
    if key in sys.modules:
        return sys.modules[key]
    path = os.path.join(ROOT, "whisper-timestamped_b200", "whisper_timestamped", name + ".py")
    spec = importlib.util.spec_from_file_location(key, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[key] = mod
    spec.loader.exec_module(mod)
    return mod


def make_audio(seconds, seed=1234):
    synthetic_speech = _pkg_module("synthetic_audio").synthetic_speech
    # built in 5-minute pieces so the generator stays cheap; deterministic for every rank
    pieces = []
    t, k = 0.0, 0
    while t < seconds:
        d = min(300.0, seconds - t)
        pieces.append(synthetic_speech(d, seed=seed + k))
        t += d
        k += 1
    return np.concatenate(pieces)


def gemm_roofline(engine, peaks, reps=20):
    """Dominant kernel = gemm_tc_kernel.  Times the encoder MLP up-projection shape (the largest FLOP share)
    alone with CUDA events; algorithmic flops = 2*M*N*K (one float32-accurate product; the kernel issues three
    bf16 wgmmas per product)."""
    import torch
    from whisper_timestamped.model import SB16
    d = engine.dims
    D = d.n_audio_state
    M, N, K = 16 * 1500, 4 * D, D
    dev = engine.dev
    a = SB16(M, K, dev)
    a.t.normal_()
    blk = engine.w.enc[0]
    out = SB16(M, N, dev)
    for _ in range(3):
        engine.gemm(a, blk.fc1, M, N, K, bias=blk.fc1_b, act=1, out_sb=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        engine.gemm(a, blk.fc1, M, N, K, bias=blk.fc1_b, act=1, out_sb=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
    return {"bound": "tensor", "achieved": tf, "peak": peaks["bf16_tflops"], "unit": "TFLOP/s",
            "frac": tf / peaks["bf16_tflops"], "peak_source": peaks["source"],
            "kernel": "gemm_tc_kernel (bf16x3: 3 wgmmas per float32-accurate product; tensor-pipe work = 3x achieved)",
            "shape": [M, N, K], "ms": ms}


def run_e2e(args, rank, world, local):
    import torch
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    model = wt.load_model(f"synthetic:{args.model}", device=dev, synthetic_kwargs=SYNTH_KW)
    eng = CudaEngine(model, max_batch=args.max_batch)
    audio = make_audio(args.audio_seconds)
    from whisper_timestamped import sharding
    mine, offset, _ = sharding.shard_audio(audio, args.chunk_seconds, rank, world)
    host_audio = torch.from_numpy(mine).pin_memory()
    dev_audio = host_audio.to(dev)
    opts = dict(language="en", chunks=args.chunk_seconds, engine=eng)

    def one(audio_in):
        eng.release()
        res = wt.transcribe(model, audio_in, **opts)
        sharding.shift_segments(res["segments"], offset)
        return sharding.gather_results(res, rank, world)       # rank 0: the stitched whole-recording result

    def barrier():
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize(dev)

    for _ in range(args.warmup):
        res = one(dev_audio)
    eng.profile = True
    eng.stage_ms()
    sampler = ClockSampler(local)
    barrier()
    if rank == 0:
        sampler.start()
    launches0 = eng.launches
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(args.steps):
        res = one(dev_audio)
    e1.record()
    timed_res = res
    barrier()
    wall = time.perf_counter() - t0
    ms = e0.elapsed_time(e1)
    stages = eng.stage_ms()
    eng.profile = False
    if rank == 0 and os.environ.get("WTS_BENCH_VERBOSE"):
        print("decode batches (B, steps, ms, ms/step):", [(b, s_, round(m, 1), round(m / max(s_, 1), 2)) for (b, s_, m) in eng.batch_ms],
              file=sys.stderr)
    clocks = sampler.stop() if rank == 0 else None
    launches = eng.launches - launches0
    # e2e through the public API with HOST audio (H2D inside) and the result dict back on the host
    barrier()
    t1 = time.perf_counter()
    for _ in range(args.steps):
        res = one(host_audio)
    barrier()
    e2e_wall = time.perf_counter() - t1
    if world > 1:
        import torch.distributed as dist
        t = torch.tensor([ms, e2e_wall * 1e3], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms, e2e_ms = t.tolist()
    else:
        e2e_ms = e2e_wall * 1e3
    total_audio = float(len(audio)) / 16000.0
    ntok = sum(len(s["tokens"]) for s in res["segments"])
    nw = sum(len(s.get("words", [])) for s in res["segments"])
    out = {"ms_per_step": ms / args.steps, "value": total_audio / (ms / args.steps * 1e-3),
           "e2e_value": total_audio / (e2e_ms / args.steps * 1e-3), "stages_ms_per_step": {k: v / args.steps for k, v in stages.items()},
           "clocks": clocks, "launches": launches, "segments": len(res["segments"]), "tokens": ntok, "words": nw,
           "h2d": int(mine.nbytes), "d2h": int(len(json.dumps(res["segments"]))) if rank == 0 else 0, "wall_s": wall,
           "decode_steps": getattr(eng, "decode_steps_run", 0), "small_batch_steps": eng.small_batch_steps,
           "result": res if rank == 0 else None, "timed_result": timed_res if rank == 0 else None}
    if rank == 0 and not args.no_roofline:
        peaks = measured_peaks()
        out["roofline"] = gemm_roofline(eng, peaks)
    return out


def usable_cores():
    """Host cores this process may really use: affinity mask and cgroup CPU quota (a container can see 128 CPUs
    and own far fewer; oversubscribing torch's thread pool then makes the CPU arm pathologically slow)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(float(quota) / float(period))))
    except Exception:
        try:
            quota = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            period = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if quota > 0:
                n = min(n, max(1, quota // period))
        except Exception:
            pass
    return max(1, min(n, int(os.environ.get("WTS_CPU_THREADS", "64"))))


def _load_reference():
    """The UNMODIFIED reference as installed by `pip install --no-deps --target baseline/_ref` (DESIGN.md §2),
    imported under an alias over the oracle stand-ins for its two missing third-party dependencies."""
    ref_dir = os.path.join(ROOT, "baseline", "_ref", "whisper_timestamped")
    if not os.path.isdir(ref_dir):
        return None
    up = os.path.join(ROOT, "oracle", "upstream")
    if up not in sys.path:
        sys.path.insert(0, up)
    import importlib.util
    spec = importlib.util.spec_from_file_location("wts_reference_pkg", os.path.join(ref_dir, "__init__.py"),
                                                  submodule_search_locations=[ref_dir])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["wts_reference_pkg"] = mod
    spec.loader.exec_module(mod)
    return mod


def build_reference_model(model_name):
    """The oracle's stand-in for openai-whisper (oracle/upstream/whisper) carrying the same synthetic weights and the
    reference's alignment heads — what the unmodified reference is handed as `model`.  Touches nothing of the product."""
    import torch
    up = os.path.join(ROOT, "oracle", "upstream")
    if up not in sys.path:
        sys.path.insert(0, up)
    import whisper                                        # oracle stand-in
    zoo = _pkg_module("model_zoo")
    dims = zoo.DIMS[model_name]
    sd = zoo.synthetic_state_dict(dims, seed=1234, **SYNTH_KW)
    model = whisper.Whisper(whisper.ModelDimensions(**dims.asdict()))
    model.load_state_dict(sd)
    del sd
    mask = torch.zeros(dims.n_text_layer, dims.n_text_head, dtype=torch.bool)
    for l, h in zoo.ALIGNMENT_HEADS[model_name]:
        mask[l, h] = True
    model.register_buffer("alignment_heads", mask.to_sparse(), persistent=False)
    return model.eval()


def reference_chunks(args, timed, warm):
    """Runs the reference's CPU path (float32, batch 1, sequential windows, per-token hooks) on 30-s chunks of the SAME
    synthetic audio, all usable host cores: `warm` chunk indices untimed, then `timed` chunk indices timed one by one.
    kind "reference": the unmodified reference from baseline/_ref over the oracle stand-ins for openai-whisper and
    dtw-python (neither can be installed in this image); kind "port": baseline/_ref missing -> the oracle engine behind
    the drop-in's host logic.  Returns (kind, cores, per-chunk seconds, per-chunk results)."""
    import torch
    cores = usable_cores()
    torch.set_num_threads(cores)
    try:
        torch.set_num_interop_threads(1)
    except RuntimeError:
        pass
    step = int(args.chunk_seconds * 16000)
    need = max(list(timed) + list(warm)) + 1
    # the SAME audio as the GPU arm: make_audio() draws it in 300-s pieces, so whole pieces are generated and then cut
    # (a shorter request would consume the generator differently and give different audio)
    whole = min(args.audio_seconds, 300.0 * np.ceil(need * args.chunk_seconds / 300.0))
    audio = make_audio(whole)[: need * step]
    ref = _load_reference()
    if ref is not None:
        kind = "reference"
        model = build_reference_model(args.model)

        def run(piece):
            return ref.transcribe(model, piece, language="en", condition_on_previous_text=False)
    else:
        kind = "port"
        from types import SimpleNamespace
        from oracle.engine import OracleEngine, build_oracle_model
        from whisper_timestamped import model_zoo as zoo
        from whisper_timestamped.transcribe import transcribe_timestamped
        dims = zoo.DIMS[args.model]
        heads = zoo.ALIGNMENT_HEADS[args.model]
        om = build_oracle_model(dims, zoo.synthetic_state_dict(dims, seed=1234, **SYNTH_KW), heads)
        shim = SimpleNamespace(dims=dims, is_multilingual=om.is_multilingual, num_languages=om.num_languages)

        def run(piece):
            return transcribe_timestamped(shim, piece, language="en", condition_on_previous_text=False,
                                          engine=OracleEngine(om, heads))
    for c in warm:
        run(audio[c * step:(c + 1) * step])
    secs, results = [], []
    for c in timed:
        t0 = time.perf_counter()
        results.append(run(audio[c * step:(c + 1) * step]))
        secs.append(time.perf_counter() - t0)
    return kind, cores, secs, results


def cpu_baseline_e2e(args, timed=None, warm=None):
    n_chunks = max(1, int(args.audio_seconds // args.chunk_seconds))
    if timed is None:
        n = max(1, min(n_chunks, int(round(args.cpu_seconds / args.chunk_seconds))))
        timed = list(range(n))
        warm = [min(n, n_chunks - 1)]                    # one untimed chunk first: thread pools, allocator, lazy imports
    kind, cores, secs, results = reference_chunks(args, timed, warm)
    dt = float(sum(secs))
    ntok = sum(len(x["tokens"]) for r in results for x in r["segments"])
    how = ("unmodified reference (baseline/_ref) over the oracle stand-ins for openai-whisper/dtw-python" if kind == "reference"
           else "oracle engine (stand-in for openai-whisper + scipy/torch/oracle-DTW alignment)")
    return {"value": len(timed) * args.chunk_seconds / dt, "unit": "audio-sec/s", "cores": cores, "kind": kind, "wall_s": dt,
            "chunk_seconds_each": [round(x, 2) for x in secs],
            "sample": f"{len(timed)} x {args.chunk_seconds:.0f}-s chunks (indices {timed[0]}..{timed[-1]}) of the same synthetic audio after "
                      f"{len(warm)} untimed warm-up chunk(s), {args.model} float32 on CPU, {how}; {dt:.1f} s, {ntok} tokens",
            "_results": results, "_timed": list(timed)}


def parity_vs_reference(ours, ref_results, timed, chunk_seconds):
    """Our stitched result against the reference's own output on the same chunks (run on this box a moment ago)."""
    eq_tokens, eq_words, max_dt, max_dc, n_seg, n_words = True, True, 0.0, 0.0, 0, 0
    for c, r in zip(timed, ref_results):
        lo, hi = int(c * chunk_seconds * 100), int((c + 1) * chunk_seconds * 100)
        mine = [s for s in ours["segments"] if lo <= s["seek"] < hi]
        theirs = r["segments"]
        n_seg += len(theirs)
        if [s["tokens"] for s in mine] != [s["tokens"] for s in theirs]:
            eq_tokens = False
            continue
        for a, b in zip(mine, theirs):
            wa, wb = a.get("words", []), b.get("words", [])
            if [w["text"] for w in wa] != [w["text"] for w in wb]:
                eq_words = False
                continue
            for x, y in zip(wa, wb):
                n_words += 1
                max_dt = max(max_dt, abs(x["start"] - (y["start"] + c * chunk_seconds)), abs(x["end"] - (y["end"] + c * chunk_seconds)))
                max_dc = max(max_dc, abs(x["confidence"] - y["confidence"]))
    return {"chunks": len(timed), "segments": n_seg, "words": n_words, "tokens_equal": eq_tokens, "word_texts_equal": eq_words,
            "max_word_dt": round(max_dt, 6), "max_confidence_diff": round(max_dc, 6)}


DUMP_LIMIT = 64 << 20          # bytes of .npy data --dump-outputs may write


def _write_dump(out_dir, arrays):
    total = sum(a.nbytes for a in arrays.values())
    assert total <= DUMP_LIMIT, f"--dump-outputs: {total} bytes exceed {DUMP_LIMIT}"   # the callers sample to fit
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def _seeded_subset(n, keep):
    """Sorted indices of a fixed seeded sample of `keep` out of `n` items (all of them when keep >= n)."""
    if keep >= n:
        return np.arange(n)
    return np.sort(np.random.default_rng(0).choice(n, size=keep, replace=False))


def _e2e_arrays(segs, index):
    f64 = lambda x: np.asarray(x, dtype=np.float64)
    segs = [segs[i] for i in index]
    words = [w for s in segs for w in s.get("words", [])]
    return {
        "segment_index": f64(index),
        "tokens": f64([t for s in segs for t in s["tokens"]]),
        "segment_tokens": f64([len(s["tokens"]) for s in segs]),
        "segment_seek": f64([s["seek"] for s in segs]),
        "segment_times": f64([[s["start"], s["end"]] for s in segs]).reshape(-1, 2),
        "segment_scores": f64([[s["avg_logprob"], s["compression_ratio"], s["no_speech_prob"], s.get("confidence", np.nan),
                                s["temperature"]] for s in segs]).reshape(-1, 5),
        "segment_words": f64([len(s.get("words", [])) for s in segs]),
        "word_times": f64([[w["start"], w["end"]] for w in words]).reshape(-1, 2),
        "word_confidence": f64([w["confidence"] for w in words]),
    }


def dump_e2e_outputs(out_dir, res):
    """What transcribe() returned: the tokens, per-segment numbers and per-word times / confidences, in order.  When
    that exceeds DUMP_LIMIT, a fixed seeded sample of whole segments (their indices in `segment_index`)."""
    segs = res["segments"]
    keep = len(segs)
    arrays = _e2e_arrays(segs, _seeded_subset(len(segs), keep))
    while sum(a.nbytes for a in arrays.values()) > DUMP_LIMIT:
        keep = int(keep * 0.9)
        arrays = _e2e_arrays(segs, _seeded_subset(len(segs), keep))
    _write_dump(out_dir, arrays)


def align_dump_arrays(jumps, cost, nseg, T, n_sample=1 << 20):
    """The DTW jumps of every segment (a fixed seeded sample of segments when they exceed half of DUMP_LIMIT) and a
    fixed seeded sample of the cost matrices (the whole cost buffer exceeds the limit), as host float64 arrays."""
    import torch
    idx = _seeded_subset(cost.numel(), min(n_sample, cost.numel()))
    sample = cost[torch.from_numpy(idx).to(cost.device)].cpu().numpy()
    rows = jumps.cpu().numpy().astype(np.float64).reshape(nseg, T + 1)
    seg = _seeded_subset(nseg, (DUMP_LIMIT // 2) // (8 * (T + 1)))
    return {"jumps": rows[seg], "jumps_segment_index": seg.astype(np.float64),
            "cost_sample_index": idx.astype(np.float64), "cost_sample": sample.astype(np.float64)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workload", default="e2e", choices=["e2e", "align"])
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--audio-seconds", type=float, default=3600.0)
    ap.add_argument("--chunk-seconds", type=float, default=30.0)
    # 64 windows decoded together: the decoder state of 128 large-v3 windows (cross K/V, alignment-head K, self KV)
    # plus the encoder scratch of one batch does not fit the 80 GB of an H100
    ap.add_argument("--max-batch", type=int, default=64)
    ap.add_argument("--cpu-seconds", type=float, default=60.0)
    ap.add_argument("--align-batch", type=int, default=16384)
    ap.add_argument("--align-T", type=int, default=24)
    ap.add_argument("--align-F", type=int, default=300)
    ap.add_argument("--recipe", default="default", choices=sorted(RECIPES))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-roofline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step as DIR/<name>.npy (float64, 64 MB at most)")
    args = ap.parse_args()
    if args.dump_outputs and args.impl != "ours":
        ap.error("--dump-outputs writes what this project's timed path computed; it has no meaning with --impl reference")
    args.warmup = max(args.warmup, 3)
    SYNTH_KW.clear()
    SYNTH_KW.update(RECIPES[args.recipe])
    rank, world, local = _dist_setup()

    workload_name = (f"{args.model}, {args.audio_seconds:.0f} s synthetic 16 kHz audio in independent "
                     f"{args.chunk_seconds:.0f}-s chunks, greedy, word timestamps + confidences")
    metric_name = "audio-sec/s (RTF) large-v3 1h synthetic @1/2/4/8 H100; DTW GB/s vs HBM peak"
    # identical in both arms (the driver compares them): what is computed, not how
    e2e_config = {"workload": workload_name, "model": args.model, "audio_seconds": args.audio_seconds,
                  "chunk_seconds": args.chunk_seconds, "decoding": "greedy, temperature 0, chunks independent",
                  "weights": "synthetic seed 1234 " + json.dumps(SYNTH_KW, sort_keys=True), "audio": "synthetic seed 1234",
                  "l2": "weights + KV caches + activations far larger than L2; every step re-reads them from memory"}
    if args.impl == "reference":
        if rank != 0:
            return
        if args.workload == "align":
            cb = cpu_baseline_align(args)
            print(json.dumps({"impl": "reference", "metric": "alignment segments/s (prep+DTW); DTW GB/s vs HBM peak",
                              "value": cb["value"], "unit": cb["unit"], "n_gpus": args.gpus, "steps": args.steps,
                              "warmup": args.warmup, "higher_is_better": True, "ms_per_step": None, "scaling": "weak",
                              "vs_baseline": None, "cpu_baseline": cb, "data": "synthetic", "dtype": "f64 accumulate / f32 cost",
                              "config": {"workload": f"align: {args.align_batch} segments/GPU, T={args.align_T}, F={args.align_F}, N=10 heads"},
                              "e2e": {"value": cb["value"], "unit": cb["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
            return
        # one step of this arm = ONE 30-s chunk of the workload through the reference's transcribe() (the whole hour would take
        # ~20 min per step on host cores): W untimed chunks, then K timed chunks, all distinct, taken in order from the recording
        n_chunks = max(1, int(args.audio_seconds // args.chunk_seconds))
        K = max(1, min(args.steps, n_chunks))
        W = max(0, min(args.warmup, n_chunks - K))
        cb = cpu_baseline_e2e(args, timed=list(range(K)), warm=list(range(K, K + W)))
        cb.pop("_results"), cb.pop("_timed")
        print(json.dumps({"impl": "reference", "metric": metric_name, "value": cb["value"], "unit": cb["unit"],
                          "n_gpus": args.gpus, "steps": K, "warmup": W, "higher_is_better": True,
                          "ms_per_step": cb["wall_s"] * 1e3 / K, "scaling": "strong", "vs_baseline": None,
                          "step_unit": f"one {args.chunk_seconds:.0f}-s chunk through the reference's transcribe() on {cb['cores']} host cores",
                          "cpu_baseline": cb, "config": e2e_config, "data": "synthetic", "dtype": "f32", "gpu_launches": 0,
                          "e2e": {"value": cb["value"], "unit": cb["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return

    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl")

    if args.workload == "e2e":
        res = run_e2e(args, rank, world, local)
        if rank == 0:
            line = {
                "metric": metric_name,
                "value": res["value"], "unit": "audio-sec/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": res["ms_per_step"], "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                "dtype": "bf16x3 tensor-core GEMMs (float32-accurate), f32 elsewhere, f64 DTW accumulate",
                "data": "synthetic audio, synthetic (seeded) weights of the exact architecture (recipe %s)" % json.dumps(SYNTH_KW),
                "config": e2e_config,
                "workload_stats": {"max_batch": args.max_batch, "segments": res["segments"], "tokens": res["tokens"],
                                   "words": res["words"], "decode_steps": res["decode_steps"],
                                   "small_batch_steps": res["small_batch_steps"]},
                "e2e": {"value": res["e2e_value"], "unit": "audio-sec/s", "h2d_bytes_per_step": res["h2d"],
                        "d2h_bytes_per_step": res["d2h"]},
                "gpu_launches": res["launches"], "clocks": res["clocks"], "stages_ms_per_step": res["stages_ms_per_step"],
            }
            if "roofline" in res:
                line["roofline"] = res["roofline"]
            if world == 1 and not args.no_roofline:
                # second half of the metric ("DTW GB/s vs HBM peak"): the SURVEY §8(d) alignment micro-workload, measured
                # in the same run (what `--workload align` reports); never allowed to take the headline down with it
                try:
                    import torch
                    torch.cuda.empty_cache()
                    al = run_align(args, rank, world)
                    line["dtw_roofline"] = {
                        "bound": "hbm", "achieved": al["dtw_gbs"], "peak": al["peaks"]["hbm_gbs"], "unit": "GB/s",
                        "frac": al["dtw_gbs"] / al["peaks"]["hbm_gbs"],
                        "kernel": dtw_kernel_name(args.align_batch, args.align_T), "ms": al["ms_dtw"], "prep_gbs": al["prep_gbs"], "prep_ms": al["ms_prep"],
                        "workload": f"{args.align_batch} segments, T={args.align_T}, F={args.align_F}, N=10 heads"}
                except Exception as err:                                   # noqa: BLE001
                    line["dtw_roofline"] = {"error": f"{type(err).__name__}: {err}"[:200]}
            if args.dump_outputs:
                dump_e2e_outputs(args.dump_outputs, res["timed_result"])
            if not args.no_cpu_baseline:
                cb = cpu_baseline_e2e(args)
                # the reference's own output on those chunks (computed on this box a moment ago) vs ours
                line["parity_vs_reference"] = parity_vs_reference(res["result"], cb.pop("_results"), cb.pop("_timed"),
                                                                  args.chunk_seconds)
                line["cpu_baseline"] = cb
            print(json.dumps(line))
    else:
        res = run_align(args, rank, world)
        if rank == 0 and args.dump_outputs:
            _write_dump(args.dump_outputs, res["outputs"])
        vals = [res["segments_per_s"]]
        ms = [res["ms_total"]]
        if world > 1:
            import torch
            import torch.distributed as dist
            t = torch.tensor([res["ms_total"]], device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = [t.item()]
            vals = [args.align_batch * world / (ms[0] * 1e-3)]
        if rank == 0:
            peaks = res["peaks"]
            line = {
                "metric": "alignment segments/s (prep+DTW); DTW GB/s vs HBM peak", "value": vals[0], "unit": "segments/s",
                "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms[0],
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64 accumulate / f32 cost",
                "data": "synthetic",
                "config": {"workload": f"align: {args.align_batch} segments/GPU, T={args.align_T}, F={args.align_F}, N=10 heads",
                           "l2": "inputs (qk %.1f GB) larger than L2" % (args.align_batch * 10 * args.align_T * 1500 * 4 / 1e9)},
                "roofline": {"bound": "hbm", "achieved": res["dtw_gbs"], "peak": peaks["hbm_gbs"], "unit": "GB/s",
                             "frac": res["dtw_gbs"] / peaks["hbm_gbs"],
                             "peak_source": peaks["source"],
                             "kernel": dtw_kernel_name(args.align_batch, args.align_T), "ms": res["ms_dtw"]},
                "prep": {"gbs": res["prep_gbs"], "ms": res["ms_prep"]},
                "e2e": {"value": res["e2e_segments_per_s"], "unit": "segments/s", "h2d_bytes_per_step": res["h2d"],
                        "d2h_bytes_per_step": res["d2h"]},
                "gpu_launches": 3 * args.steps, "clocks": res["clocks"], "jumps_checksum": res["jumps_checksum"],
            }
            if not args.no_cpu_baseline:
                line["cpu_baseline"] = cpu_baseline_align(args)
            print(json.dumps(line))
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

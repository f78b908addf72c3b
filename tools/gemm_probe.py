"""GEMM probe.  Times wts_gemm on the encoder shapes and on the decode shapes.  Decode shapes are timed as a CUDA graph
of dependent launches (what the decode step does), so host launch cost does not pollute them.

  python tools/gemm_probe.py [big|skinny|encoder|all] [--windows 64] [--json OUT.json] [--compare OTHER.json]
                             [--pkg DIR]

`encoder`: every GEMM the large-v3 encoder and the cross-K/V projection issue for a batch of --windows 30-s windows
(operand layouts and epilogues as engine.encode / engine._cross_kv issue them), the bench's roofline shape, and a bf16
torch.matmul at the fc1 shape (the dense rate the card reaches; a third of it bounds the 3-term split-bf16 product).
`skinny`: every GEMM of a large-v3 decode step (qkv, out-projection with in-place residual, fc1 with GELU and SB16
output, fc2 with in-place residual, vocabulary projection with a row mask) at M = 1, 9, 64 (the 64-row instance of the
split-K kernel) and 65, 128 (the 128-row one), timed as a graph chain over distinct weight sets.
Each GEMM first runs once on seeded inputs and its output is digested on the device; --json writes the digests and
times, --compare checks them bit for bit against another build's --json (e.g. the parent commit's tree via --pkg)."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _digest(t):
    """Bit-exact fingerprint of a tensor's bytes (two position-weighted int64 sums, computed on the device)."""
    x = t.contiguous().view(-1).view(torch.int32).to(torch.int64)
    w = torch.arange(x.numel(), device=x.device, dtype=torch.int64) * 2 + 1
    return [int(x.sum().item()), int(((x * w) % 2305843009213693951).sum().item())]


def _time(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def encoder_shapes(eng, B, dev, results):
    from whisper_timestamped.model import SB16
    D, C, H, T, KPAD = 1280, 128, 20, 1500, 1504
    R = B * T
    gen = torch.Generator(device=dev)

    def sb(rows, cols, seed, ld=None):
        s = SB16(rows, cols, dev, ld=ld)
        gen.manual_seed(seed)
        s.t.normal_(generator=gen)
        return s

    def vec(n, seed):
        gen.manual_seed(seed)
        return torch.randn(n, device=dev, generator=gen)

    # (name, M, N, K, batch count, builder -> (call, output tensor))
    def qk():
        a, w, out = sb(R, D, 1), sb(2 * D, D, 2), SB16(R, 2 * D, dev)
        bias = vec(2 * D, 3)
        return (lambda: eng.gemm(a, w, R, 2 * D, D, bias=bias, out_sb=out)), out.t

    def vt():
        w, h, out = sb(D, D, 4), sb(R, D, 5), SB16(B * D, KPAD, dev)
        bias = vec(D, 6)
        return (lambda: eng.gemm(w, h, D, T, D, batch=(B, 1), b_b=(T * D, 0), bias=bias, bias_on_m=True, out_sb=out,
                                 ldo=KPAD, o_b=(D * KPAD, 0))), out.t

    def resid(K, seed):
        def make():
            a, w = sb(R, K, seed), sb(D, K, seed + 1)
            bias = vec(D, seed + 2)
            gen.manual_seed(seed + 3)
            x = torch.randn(R, D, device=dev, generator=gen)
            return (lambda: eng.gemm(a, w, R, D, K, bias=bias, residual=x, ldr=D, out_f32=x, ldc=D)), x
        return make

    def fc1(M):
        def make():
            a, w, out = sb(M, D, 10), sb(4 * D, D, 11), SB16(M, 4 * D, dev)
            bias = vec(4 * D, 12)
            return (lambda: eng.gemm(a, w, M, 4 * D, D, bias=bias, act=1, out_sb=out)), out.t
        return make

    def conv1():
        x0, w, h1 = sb(B * 3002, C, 13), sb(D, 3 * C, 14), SB16(B * 3001, D, dev)
        bias = vec(D, 15)
        return (lambda: eng.gemm(x0, w, 3000, D, 3 * C, lda=C, batch=(B, 1), a_b=(3002 * C, 0), bias=bias, act=1,
                                 out_sb=h1, ldo=D, o_b=(3001 * D, 0), o_off=D)), h1.t

    def conv2():
        h1, w = sb(B * 3001, D, 16), sb(D, 3 * D, 17)
        bias, pos = vec(D, 18), vec(T * D, 19).view(T, D)
        x = torch.empty((R, D), device=dev)
        return (lambda: eng.gemm(h1, w, T, D, 3 * D, lda=2 * D, batch=(B, 1), a_b=(3001 * D, 0), bias=bias, act=1,
                                 residual=pos, ldr=D, r_b=(0, 0), out_f32=x, ldc=D, c_b=(T * D, 0))), x

    def cross_kv():
        xa, w = sb(R, D, 20), sb(D, D, 21)
        bias = vec(D, 22)
        tmp = torch.empty((B, H, T, 64), device=dev)
        return (lambda: eng.gemm(xa, w, T, D, D, batch=(B, 1), a_b=(T * D, 0), bias=bias, out_f32=tmp, ldc=64,
                                 c_b=(H * T * 64, 0), head_dim=64, head_stride=T * 64)), tmp

    shapes = [("qk", R, 2 * D, D, qk), ("vT bias_on_m", B * D, T, D, vt), ("out +=x", R, D, D, resid(D, 7)),
              ("fc1 gelu sb16", R, 4 * D, D, fc1(R)), ("fc2 +=x", R, D, 4 * D, resid(4 * D, 23)),
              ("conv1 lda<K", B * 3000, D, 3 * C, conv1), ("conv2 lda<K", R, D, 3 * D, conv2),
              ("cross-kv heads", R, D, D, cross_kv), ("roofline fc1", 16 * T, 4 * D, D, fc1(16 * T))]
    for (name, M, N, K, make) in shapes:
        call, out = make()
        call()
        torch.cuda.synchronize()
        dig = _digest(out)
        ms = _time(call, 10)
        tf = 2.0 * M * N * K / ms / 1e9
        print(f"{name:15s} M={M:6d} N={N:5d} K={K:5d}: {ms:8.3f} ms  {tf:7.1f} TF/s(alg)", flush=True)
        results.append(dict(name=name, M=M, N=N, K=K, ms=ms, tflops=tf, digest=dig))
        del call, out
        torch.cuda.empty_cache()
    # the dense bf16 rate of this card at the fc1 shape (cuBLAS through torch.matmul; a yardstick, not a product path)
    M, N, K = R, 4 * D, D
    gen.manual_seed(30)
    a = torch.randn(M, K, device=dev, generator=gen).bfloat16()
    w = torch.randn(N, K, device=dev, generator=gen).bfloat16()
    c = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ms = _time(lambda: torch.matmul(a, w.T, out=c), 10)
    tf = 2.0 * M * N * K / ms / 1e9
    print(f"{'torch bf16 mm':15s} M={M:6d} N={N:5d} K={K:5d}: {ms:8.3f} ms  {tf:7.1f} TF/s  (/3 = {tf / 3:.1f})", flush=True)
    results.append(dict(name="torch.matmul bf16 (fc1 shape)", M=M, N=N, K=K, ms=ms, tflops=tf))


def decode_shapes(eng, dev, results):
    from whisper_timestamped.model import SB16
    D, V = 1280, 51866
    n_w = 24                          # distinct weight sets so the chain streams weights from HBM like the decode step
    gen = torch.Generator(device=dev)

    def sb(rows, cols, seed, std=1.0):
        s = SB16(rows, cols, dev)
        gen.manual_seed(seed)
        s.t.normal_(0.0, std, generator=gen)
        return s

    def randn(shape, seed):
        gen.manual_seed(seed)
        return torch.randn(shape, device=dev, generator=gen)

    # (name, N, K, epilogue), with the weights marked b_const as the engine's decode step issues them
    shapes = [("dec qkv", 3 * D, D, "bias"), ("dec out +=x", D, D, "residual"), ("dec fc1 gelu sb16", 4 * D, D, "gelu"),
              ("dec fc2 +=x", D, 4 * D, "residual"), ("dec vocab mask", V, D, "mask")]
    for (name, N, K, epi) in shapes:
        ws = [sb(N, K, 100 + i, 0.02) for i in range(n_w)]
        bias = randn(N, 1) if epi != "mask" else None
        for M in (1, 9, 64, 65, 128):
            a = sb(M, K, 2)
            mask = (torch.arange(M, device=dev) % 3 != 1).to(torch.int32) if epi == "mask" else None
            if epi == "gelu":
                out = SB16(M, N, dev)
                res, kw = out.t, dict(act=1, out_sb=out)
            else:
                res = randn((M, N), 3)
                kw = dict(out_f32=res, ldc=N, row_mask=mask)
                if epi == "residual":
                    kw.update(residual=res, ldr=N)

            def chain(weights=ws):
                for w in weights:
                    eng.gemm(a, w, M, N, K, bias=bias, b_const=True, **kw)
            chain(ws[:1])
            torch.cuda.synchronize()
            dig = _digest(res)
            chain()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream(device=dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                with torch.cuda.graph(graph, stream=s):
                    chain()
            torch.cuda.current_stream(dev).wait_stream(s)
            ms = _time(graph.replay, 10) / n_w
            print(f"{name:17s} M={M:3d} N={N:5d} K={K:4d}: {ms * 1e3:7.2f} us per GEMM in a graph chain "
                  f"(weights {4.0 * N * K / 1e6:.1f} MB -> {4.0 * N * K / ms / 1e9:.2f} TB/s)", flush=True)
            results.append(dict(name=f"{name} M={M}", M=M, N=N, K=K, ms=ms, digest=dig))
            del graph
        del ws
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="?", default="all", choices=["all", "big", "skinny", "encoder"])
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--json", default=None)
    ap.add_argument("--compare", default=None)
    ap.add_argument("--pkg", default=os.path.join(ROOT, "whisper-timestamped_b200"),
                    help="directory holding the whisper_timestamped package to probe")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.pkg))
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.model import SB16
    dev = torch.device("cuda:0")
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = dev, 0, 0
    which = args.which
    results = []
    if which in ("all", "big"):
        for (M, N, K, name) in [(24000, 5120, 1280, "enc fc1"), (24000, 1280, 5120, "enc fc2"), (24000, 1280, 1280, "enc out")]:
            a, b = SB16(M, K, dev), SB16(N, K, dev)
            a.t.normal_()
            b.t.normal_()
            out = SB16(M, N, dev)
            ms = _time(lambda: eng.gemm(a, b, M, N, K, out_sb=out), 20)
            print(f"{name:8s} M={M} N={N} K={K}: {ms * 1e3:9.1f} us  {2.0 * M * N * K / ms / 1e9:8.1f} TF/s(alg)", flush=True)
    if which in ("all", "encoder"):
        print(f"encoder + cross-K/V GEMMs, large-v3, {args.windows} windows", flush=True)
        encoder_shapes(eng, args.windows, dev, results)
    if which in ("all", "skinny"):
        print("decode-step GEMMs, large-v3", flush=True)
        decode_shapes(eng, dev, results)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(dev), windows=args.windows, results=results), f, indent=1)
    if args.compare:
        other = {r["name"]: r for r in json.load(open(args.compare))["results"] if "digest" in r}
        same = True
        for r in results:
            if "digest" in r and r["name"] in other:
                eq = r["digest"] == other[r["name"]]["digest"]
                same &= eq
                print(f"{r['name']:15s} outputs {'bit-identical' if eq else 'DIFFER'}; "
                      f"{other[r['name']]['ms'] / r['ms']:.2f}x the other build's speed", flush=True)
        if not same:
            sys.exit(1)


if __name__ == "__main__":
    main()

"""GEMM probe.  Times wts_gemm on the encoder shapes and on the decode shapes.  Decode shapes are timed as a CUDA graph
of dependent launches (what the decode step does), so host launch cost does not pollute them."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "whisper-timestamped_b200"))


def main():
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.model import SB16
    dev = torch.device("cuda:0")
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = dev, 0, 0
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("all", "big"):
        for (M, N, K, name) in [(24000, 5120, 1280, "enc fc1"), (24000, 1280, 5120, "enc fc2"), (24000, 1280, 1280, "enc out")]:
            a, b = SB16(M, K, dev), SB16(N, K, dev)
            a.t.normal_()
            b.t.normal_()
            out = SB16(M, N, dev)
            for _ in range(3):
                eng.gemm(a, b, M, N, K, out_sb=out)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 20
            torch.cuda.synchronize()
            e0.record()
            for _ in range(reps):
                eng.gemm(a, b, M, N, K, out_sb=out)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / reps
            print(f"{name:8s} M={M} N={N} K={K}: {ms * 1e3:9.1f} us  {2.0 * M * N * K / ms / 1e9:8.1f} TF/s(alg)", flush=True)
    if which in ("all", "skinny"):
        n_w = 24                      # distinct weight sets so the chain streams weights from HBM like the decode step
        for (M, N, K, name) in [(128, 1280, 1280, "dec out"), (128, 3840, 1280, "dec qkv"), (128, 5120, 1280, "dec fc1"),
                                (128, 1280, 5120, "dec fc2"), (8, 1280, 1280, "dec out b8"), (8, 5120, 1280, "dec fc1 b8")]:
            a = SB16(M, K, dev)
            a.t.normal_()
            ws = [SB16(N, K, dev) for _ in range(n_w)]
            for w in ws:
                w.t.normal_(0, 0.02)
            bias = torch.zeros(N, device=dev)
            x = torch.zeros(M, N, device=dev)
            out = SB16(M, N, dev)

            def chain():
                for w in ws:
                    if N == K:
                        eng.gemm(a, w, M, N, K, bias=bias, residual=x, ldr=N, out_f32=x, ldc=N)
                    else:
                        eng.gemm(a, w, M, N, K, bias=bias, act=1, out_sb=out)
            chain()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream(device=dev)
            s.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(s):
                with torch.cuda.graph(graph, stream=s):
                    chain()
            torch.cuda.current_stream(dev).wait_stream(s)
            for _ in range(3):
                graph.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(10):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / 10 / n_w * 1e3
            print(f"{name:11s} M={M} N={N} K={K}: {us:7.2f} us per GEMM in a graph chain "
                  f"(weights {4.0 * N * K / 1e6:.1f} MB -> {4.0 * N * K / us / 1e6:.2f} TB/s)", flush=True)


if __name__ == "__main__":
    main()

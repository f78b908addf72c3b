"""GPU parity of the model path (log-mel, encoder, batched greedy decoder, cross-attention capture)
and of the whole transcribe() against (a) the oracle CPU stand-in run on the same inputs and
(b) the committed golden outputs of the unmodified reference.  Tolerance for floating point values:
1e-3 absolute (BASELINE.json north_star); token sequences must be identical."""
import glob
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1e-3
BACKENDS = [int(x) for x in os.environ.get("WTS_TEST_BACKENDS", "1,0").split(",")]


def _models(name="tiny", **kw):
    import whisper_timestamped as wt
    from whisper_timestamped import model_zoo as zoo
    from oracle_engine import OracleEngine, build_oracle_model
    dims = zoo.DIMS[name]
    sd = zoo.synthetic_state_dict(dims, seed=1234, **kw)
    heads = zoo.ALIGNMENT_HEADS[name]
    om = build_oracle_model(dims, sd, heads)
    gm = wt.load_model(f"synthetic:{name}", device="cuda:0", synthetic_kwargs=kw)
    return gm, om, OracleEngine(om, heads, keep_logprobs=True)


@pytest.fixture(scope="module")
def tiny():
    return _models("tiny")


def _engine(gm, backend, **kw):
    from whisper_timestamped.engine import CudaEngine
    return CudaEngine(gm, gemm_backend=backend, **kw)


@pytest.mark.parametrize("backend", BACKENDS)
def test_gemm_backends_vs_torch(backend):
    """wts_gemm (SB16 operands) against a float64 torch matmul of the same SB16 values."""
    import whisper_timestamped as wt
    from whisper_timestamped.model import SB16
    from whisper_timestamped.engine import CudaEngine
    from types import SimpleNamespace
    dev = torch.device("cuda:0")
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = dev, backend, 0
    g = torch.Generator(device="cpu").manual_seed(5)
    for (M, N, K) in [(200, 300, 136), (1500, 384, 384), (5, 51865, 384), (128, 64, 1500), (33, 17, 72), (1500, 1500, 64)]:
        Kp = (K + 7) // 8 * 8                      # row pitch: SB16 rows must stay 16-byte aligned
        a = torch.randn(M, Kp, generator=g).to(dev)
        b = torch.randn(N, Kp, generator=g).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        res = torch.randn(M, N, generator=g).to(dev)
        A, Bm = SB16.from_f32(a), SB16.from_f32(b)
        out = torch.zeros(M, N, device=dev)
        osb = SB16(M, N, dev)
        eng.gemm(A, Bm, M, N, K, bias=bias, act=1, residual=res, ldr=N, out_f32=out, ldc=N, out_sb=osb)
        torch.cuda.synchronize()
        ref = torch.nn.functional.gelu(A.to_f32()[:, :K].double() @ Bm.to_f32()[:, :K].double().T + bias.double()) + res.double()
        err = (out.double() - ref).abs().max().item()
        scale = ref.abs().max().item()
        assert err <= 2e-4 * max(1.0, scale), (M, N, K, err, scale)
        assert (osb.to_f32().double() - ref).abs().max().item() <= 3e-4 * max(1.0, scale)


@pytest.mark.parametrize("backend", BACKENDS)
def test_gemm_skinny_inplace_residual(backend):
    """Decode-time shape: one M tile, x += A W^T + b in place (tensor-core path: gemm_tc_kernel, K split over a
    thread-block cluster and reduced through distributed shared memory)."""
    from whisper_timestamped.model import SB16
    from whisper_timestamped.engine import CudaEngine
    dev = torch.device("cuda:0")
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = dev, backend, 0
    g = torch.Generator(device="cpu").manual_seed(9)
    for (M, N, K) in [(20, 1280, 5120), (120, 1280, 1280), (3, 384, 1536), (128, 3840, 1280)]:
        a = torch.randn(M, K, generator=g).to(dev)
        b = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        x = torch.randn(M, N, generator=g).to(dev)
        A, Bm = SB16.from_f32(a), SB16.from_f32(b)
        ref = x.double() + A.to_f32().double() @ Bm.to_f32().double().T + bias.double()
        eng.gemm(A, Bm, M, N, K, bias=bias, residual=x, ldr=N, out_f32=x, ldc=N)
        torch.cuda.synchronize()
        err = (x.double() - ref).abs().max().item()
        assert err <= 2e-4 * max(1.0, ref.abs().max().item()), (M, N, K, err)


@pytest.mark.parametrize("backend", BACKENDS)
def test_gemm_skinny_split_general_epilogue(backend):
    """Decode-time GEMMs whose epilogue is NOT the in-place residual (bias, GELU, SB16 / float32 outputs), ragged N and
    K, 1..128 rows: the cluster reduction must be exact and leave no state behind (every shape runs three times)."""
    from whisper_timestamped.model import SB16
    from whisper_timestamped.engine import CudaEngine
    dev = torch.device("cuda:0")
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = dev, backend, 0
    g = torch.Generator(device="cpu").manual_seed(11)
    for (M, N, K) in [(128, 5120, 1280), (120, 3840, 1280), (7, 1280, 5120), (64, 1000, 1288), (128, 1284, 136), (1, 384, 384)]:
        a = torch.randn(M, K, generator=g).to(dev)
        b = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        res = torch.randn(M, N, generator=g).to(dev)
        A, Bm = SB16.from_f32(a), SB16.from_f32(b)
        lin = A.to_f32().double() @ Bm.to_f32().double().T + bias.double()
        for rep in range(3):
            out = torch.full((M, N), 7.0, device=dev)
            osb = SB16(M, N, dev)
            eng.gemm(A, Bm, M, N, K, bias=bias, act=1, out_sb=osb)                       # fc1-like
            eng.gemm(A, Bm, M, N, K, bias=bias, out_f32=out, ldc=N)                      # qkv-like
            out2 = torch.zeros(M, N, device=dev)
            eng.gemm(A, Bm, M, N, K, bias=bias, residual=res, ldr=N, out_f32=out2, ldc=N)  # residual, not in place
            torch.cuda.synchronize()
            scale = max(1.0, lin.abs().max().item())
            assert (osb.to_f32().double() - torch.nn.functional.gelu(lin)).abs().max().item() <= 3e-4 * scale, (M, N, K, rep)
            assert (out.double() - lin).abs().max().item() <= 2e-4 * scale, (M, N, K, rep)
            assert (out2.double() - (lin + res.double())).abs().max().item() <= 2e-4 * scale, (M, N, K, rep)


def test_gemm_skinny_row_mask():
    """row_mask: rows of finished windows are skipped (outputs untouched), the others are exact; the active rows are
    spread over the cluster CTAs, so odd counts and all-inactive batches are covered."""
    from whisper_timestamped.model import SB16
    from whisper_timestamped.engine import CudaEngine
    dev = torch.device("cuda:0")
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = dev, 0, 0
    g = torch.Generator(device="cpu").manual_seed(13)
    for (M, N, K, n_act) in [(128, 1280, 1280, 5), (128, 5120, 1280, 37), (64, 1000, 1288, 0), (128, 51866, 384, 3), (20, 1280, 5120, 20)]:
        a = torch.randn(M, K, generator=g).to(dev)
        b = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        x0 = torch.randn(M, N, generator=g).to(dev)
        mask = torch.zeros(M, dtype=torch.int32)
        mask[torch.randperm(M, generator=g)[:n_act]] = 1
        mask = mask.to(dev)
        A, Bm = SB16.from_f32(a), SB16.from_f32(b)
        lin = A.to_f32().double() @ Bm.to_f32().double().T + bias.double()
        x = x0.clone()
        eng.gemm(A, Bm, M, N, K, bias=bias, residual=x, ldr=N, out_f32=x, ldc=N, row_mask=mask)
        osb = SB16(M, N, dev)
        osb.t.fill_(2.0)
        eng.gemm(A, Bm, M, N, K, bias=bias, act=1, out_sb=osb, row_mask=mask)
        torch.cuda.synchronize()
        on = mask.bool()
        scale = max(1.0, lin.abs().max().item())
        assert torch.equal(x[~on], x0[~on]), (M, N, K)
        assert torch.all(osb.to_f32()[~on] == 4.0)
        if n_act:
            assert (x[on].double() - (x0[on].double() + lin[on])).abs().max().item() <= 2e-4 * scale
            assert (osb.to_f32()[on].double() - torch.nn.functional.gelu(lin[on])).abs().max().item() <= 3e-4 * scale


def test_cross_attention_f16_vs_torch():
    """wts_cross_attention_f16 (one pass, online softmax over fp16 K/V; float32 K for the alignment heads) against
    float64 torch on the same cache contents; inactive rows must be left untouched."""
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(21)
    B, H, ctx, n_slots, qk_rows = 3, 6, 1500, 2, 5
    D = H * 64
    head_slot = torch.tensor([-1, 0, -1, -1, 1, -1], dtype=torch.int32, device=dev)
    k32 = (torch.randn(B, H, ctx, 64, generator=g) * 0.7).to(dev)
    v32 = torch.randn(B, H, ctx, 64, generator=g).to(dev)
    k16, v16 = k32.half().contiguous(), v32.half().contiguous()
    kal = torch.stack([k32[:, 1], k32[:, 4]], dim=1).contiguous()
    R = 5
    q = (torch.randn(R, D, generator=g) * 0.8).to(dev)
    row_seq = torch.tensor([0, 2, 1, 1, 0], dtype=torch.int32, device=dev)
    qk_row = torch.tensor([0, 3, -1, 4, 2], dtype=torch.int32, device=dev)
    active = torch.tensor([1, 1, 1, 0, 1], dtype=torch.int32, device=dev)
    out = SB16(R, D, dev)
    out.t.fill_(3.0)
    qk_out = torch.full((B, n_slots, qk_rows, ctx), -77.0, device=dev)
    rc = nat.lib.wts_cross_attention_f16(q.data_ptr(), D, k16.data_ptr(), v16.data_ptr(), kal.data_ptr(), head_slot.data_ptr(),
                                         n_slots, ctx, row_seq.data_ptr(), R, H, out.ptr, out.ld, out.plane, qk_out.data_ptr(),
                                         qk_rows, qk_row.data_ptr(), active.data_ptr(), nat.stream_ptr(dev))
    nat.check(rc, "wts_cross_attention_f16")
    torch.cuda.synchronize()
    got = out.to_f32().double()
    expect_qk = torch.full_like(qk_out, -77.0).double()
    for r in range(R):
        if not active[r]:
            assert torch.all(got[r] == 3.0 + 3.0)       # untouched planes (hi = lo = 3)
            continue
        sq = int(row_seq[r])
        for h in range(H):
            slot = int(head_slot[h])
            K = (k32 if slot >= 0 else k16.float())[sq, h].double()
            s = K @ q[r, h * 64:(h + 1) * 64].double()
            y = torch.softmax(s, dim=0) @ v16[sq, h].double()
            assert (got[r, h * 64:(h + 1) * 64] - y).abs().max().item() <= 2e-5, (r, h)
            if slot >= 0 and int(qk_row[r]) >= 0:
                expect_qk[sq, slot, int(qk_row[r])] = s
    assert (qk_out.double() - expect_qk).abs().max().item() <= 2e-5


def test_enc_attention_fused_vs_torch():
    """wts_enc_attention (wgmma, scores on-chip) against float64 softmax(q k^T) v of the same SB16 values."""
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    dev = torch.device("cuda:0")
    g = torch.Generator(device="cpu").manual_seed(3)
    B, H, n_ctx, KP = 2, 3, 1500, 1504
    D = H * 64
    qk = SB16.from_f32((torch.randn(B * n_ctx, 2 * D, generator=g) * 0.6).to(dev))
    vt = SB16.from_f32(torch.randn(B * D, KP, generator=g).to(dev))
    out = SB16(B * n_ctx, D, dev)
    rc = nat.lib.wts_enc_attention(qk.ptr, 2 * D, qk.plane, vt.ptr, KP, vt.plane, B, H, D, n_ctx, out.ptr, D, out.plane,
                                   nat.stream_ptr(dev))
    nat.check(rc, "wts_enc_attention")
    torch.cuda.synchronize()
    qkf = qk.to_f32().double().reshape(B, n_ctx, 2, H, 64)
    q, k = qkf[:, :, 0].permute(0, 2, 1, 3), qkf[:, :, 1].permute(0, 2, 1, 3)          # [B,H,n,64]
    v = vt.to_f32().double().reshape(B, H, 64, KP)[..., :n_ctx].permute(0, 1, 3, 2)     # [B,H,n,64]
    ref = (torch.softmax(q @ k.transpose(-1, -2), dim=-1) @ v).permute(0, 2, 1, 3).reshape(B * n_ctx, D)
    err = (out.to_f32().double() - ref).abs().max().item()
    assert err <= 2e-4, err


@pytest.mark.parametrize("backend", BACKENDS[:1])
def test_log_mel_matches_oracle(tiny, backend):
    from whisper_timestamped.synthetic_audio import synthetic_speech
    gm, om, oe = tiny
    eng = _engine(gm, backend)
    for dur, seed in ((30.0, 1), (7.3, 2), (0.5, 3)):
        audio = synthetic_speech(dur, seed=seed)
        mel = eng.log_mel(eng.load_audio(audio)).cpu().numpy()           # [frames, n_mels]
        ref = oe.log_mel(torch.from_numpy(audio)).numpy().T
        assert mel.shape == ref.shape
        assert np.max(np.abs(mel - ref)) <= TOL, np.max(np.abs(mel - ref))


@pytest.mark.parametrize("backend", BACKENDS)
def test_encoder_matches_oracle(tiny, backend):
    from whisper_timestamped.synthetic_audio import synthetic_speech
    gm, om, oe = tiny
    eng = _engine(gm, backend)
    audio = synthetic_speech(40.0, seed=21)
    mel = eng.log_mel(eng.load_audio(audio))
    jobs = [dict(mel=mel, seek=0, segment_size=3000), dict(mel=mel, seek=2500, segment_size=1500)]
    xa = eng.encode(jobs).to_f32().cpu().numpy().reshape(2, 1500, -1)
    omel = oe.log_mel(torch.from_numpy(audio))
    import whisper
    for k, job in enumerate(jobs):
        seg = whisper.pad_or_trim(omel[:, job["seek"]: job["seek"] + job["segment_size"]], 3000)
        with torch.no_grad():
            ref = om.encoder(seg[None])[0].numpy()
        err = np.max(np.abs(xa[k] - ref))
        assert err <= TOL, (k, err)


@pytest.mark.parametrize("small_rows", [32, 0, 2])
@pytest.mark.parametrize("backend", BACKENDS)
def test_decode_windows_matches_oracle(tiny, backend, small_rows):
    """Same windows through the CUDA engine and the oracle engine: identical tokens, log-probs, no-speech
    probability and alignment-head cross-attention rows within 1e-3.  small_rows: 32 = every step by the lean small-
    batch kernels (wts_decode_step_kernels), 0 = every step by the per-operator tensor-core graph, 2 = that graph until
    only two windows are left, then the lean kernels (the paths share caches and token state)."""
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from whisper_timestamped.tokenizer import get_tokenizer
    from whisper_timestamped.windows import make_decode_setup
    gm, om, oe = tiny
    eng = _engine(gm, backend, keep_full_logprobs=True, small_batch_rows=small_rows)
    tok = get_tokenizer(True, num_languages=gm.num_languages, language="en", task="transcribe")
    setup = make_decode_setup(tok, gm.dims.n_text_ctx)
    audio = synthetic_speech(65.0, seed=33)
    gmel = eng.log_mel(eng.load_audio(audio))
    omel = oe.log_mel(torch.from_numpy(audio))
    prompt_long = setup.initial_tokens(list(range(1000, 1040)))
    specs = [(0, 3000, setup.initial_tokens([])), (3000, 3000, prompt_long), (6000, 500, setup.initial_tokens([]))]
    gj = [dict(mel=gmel, seek=s, segment_size=z, prompt=p) for (s, z, p) in specs]
    oj = [dict(mel=omel, seek=s, segment_size=z, prompt=p) for (s, z, p) in specs]
    grec = eng.decode_windows(gj, setup)
    orec = oe.decode_windows(oj, setup)
    for k, (a, b) in enumerate(zip(grec, orec)):
        assert a.tokens == b.tokens, (k, a.tokens[:20], b.tokens[:20])
        assert a.ended_by_eot == b.ended_by_eot
        assert abs(a.no_speech_prob - b.no_speech_prob) <= TOL
        assert np.max(np.abs(a.logprobs - b.logprobs)) <= TOL, (k, np.max(np.abs(a.logprobs - b.logprobs)))
        buf, bi = eng.window_index[a.qk_window]
        qk = eng.qk_buffers[buf][bi, :, : a.n_rows].cpu().numpy()
        ref = oe.qk[b.qk_window].numpy()
        assert qk.shape == ref.shape
        assert np.max(np.abs(qk - ref)) <= TOL, (k, np.max(np.abs(qk - ref)))
        full = eng.full_logprobs[buf][bi, : a.n_rows].cpu().numpy()
        oref = oe.full_logprobs[b.qk_window].numpy()
        finite = np.isfinite(oref)
        assert np.array_equal(finite, np.isfinite(full))
        assert np.max(np.abs(full[finite] - oref[finite])) <= TOL
        if a.last_row_logprobs is not None and not a.ended_by_eot:
            # window that ran into the decoding limit: the row the reference reads its fallback token from (T.py:529-538)
            for t in (tok.eot, tok.timestamp_begin + 700, 1234):
                want = float(oref[a.n_rows - 1, t])
                got = a.last_row_logprobs(t)
                assert (np.isinf(want) and np.isinf(got)) or abs(got - want) <= TOL
    if small_rows == 32:
        assert eng.small_batch_steps > 0
    elif small_rows == 0:
        assert eng.small_batch_steps == 0


# the `verbose` goldens pin what is printed (host logic, tests/test_host_e2e.py); their decoding paths are the ones of
# tiny_detect_lang / tiny_naive / tiny_vad_list, which run here
CASES = sorted(p for p in glob.glob(os.path.join(HERE, "golden", "e2e_*.json")) if "_verbose_" not in os.path.basename(p))
CHUNK_CASES = sorted(glob.glob(os.path.join(HERE, "golden", "chunks_*.json")))


def _is_big(path):
    return any(b in os.path.basename(path) for b in ("medium", "large"))


def _backends_for(path):
    # the SIMT validator backend (1) is only run at tiny / base dimensions; the configurations bench.py measures
    # (medium, large-v3) go through the tensor-core path that is actually timed
    return [0] if _is_big(path) else BACKENDS


_PARAMS = [pytest.param(p, b, id=f"{os.path.basename(p)[4:-5]}-b{b}") for p in CASES for b in _backends_for(p)]
_CHUNK_PARAMS = [pytest.param(p, b, id=f"{os.path.basename(p)[:-5]}-b{b}") for p in CHUNK_CASES for b in _backends_for(p)]
_MODELS = {}


def _load(g):
    """One resident model at a time (large-v3 weights are 12 GB in SB16 + float32)."""
    import whisper_timestamped as wt
    key = (g["model"], g["model_seed"], json.dumps(g["model_kwargs"], sort_keys=True))
    if key not in _MODELS:
        _MODELS.clear()
        torch.cuda.empty_cache()
        _MODELS[key] = wt.load_model(f"synthetic:{g['model']}", device="cuda:0", synthetic_seed=g["model_seed"],
                                     synthetic_kwargs=g["model_kwargs"])
    return _MODELS[key]


@pytest.mark.parametrize("path,backend", _PARAMS)
def test_transcribe_matches_reference_golden(path, backend):
    """whisper_timestamped.transcribe() on the GPU vs the unmodified reference's output (CPU fp32): identical tokens,
    segments, word times; confidences within 2e-3; the same warnings (e.g. the too-much-text truncation and its
    "Got inconsistent length" follow-up on the large-v3 bench recipe)."""
    import whisper_timestamped as wt
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from test_host_e2e import CaptureWarnings, compare, norm_warnings
    g = json.load(open(path))
    gm = _load(g)
    eng = _engine(gm, backend)
    audio = synthetic_speech(*g["audio"])
    with CaptureWarnings() as cap:
        res = wt.transcribe(gm, audio, engine=eng, **g["transcribe_kwargs"])
    compare(res, g["result"], conf_tol=2e-3, time_tol=0.0, prob_tol=1e-3)
    if "warnings" in g:
        assert norm_warnings(cap.messages) == norm_warnings(g["warnings"])


@pytest.mark.parametrize("path,backend", _CHUNK_PARAMS)
def test_chunks_mode_equals_reference_on_every_cut(path, backend):
    """transcribe(..., chunks=30) — the unit of work bench.py shards over GPUs — against the unmodified reference run
    independently on every 30-s cut (condition_on_previous_text=False), incl. the first 5 minutes of the bench audio
    on large-v3 with the bench recipe."""
    import whisper_timestamped as wt
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from test_host_e2e import CaptureWarnings, compare, norm_warnings, stitch_cuts
    g = json.load(open(path))
    gm = _load(g)
    eng = _engine(gm, backend)
    audio = synthetic_speech(*g["audio"])
    with CaptureWarnings() as cap:
        res = wt.transcribe(gm, audio, engine=eng, chunks=g["chunks"], **g["transcribe_kwargs"])
    ref, warns = stitch_cuts(g)
    compare(res, ref, conf_tol=2e-3, time_tol=1e-6, prob_tol=1e-3)
    assert norm_warnings(cap.messages) == norm_warnings(warns)


def test_continuous_batching_equals_rounds():
    """decode_stream (a stream's next window joins the running batch as soon as its previous one finishes) gives exactly
    what the round-based loop gives: chunk mode with follow-up windows, more streams than decode slots, and the
    sequential (single-stream) mode with prompt carry-over."""
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.synthetic_audio import synthetic_speech
    gm = wt.load_model("synthetic:tiny", device="cuda:0")
    audio = synthetic_speech(200.0, seed=51)
    for kw, max_batch in ((dict(language="en", chunks=30.0), 64), (dict(language="en", chunks=20.0), 4), (dict(language="en"), 64)):
        a = wt.transcribe(gm, audio, engine=CudaEngine(gm, max_batch=max_batch), continuous_batching=True, **kw)
        b = wt.transcribe(gm, audio, engine=CudaEngine(gm, max_batch=max_batch), continuous_batching=False, **kw)
        assert a["text"] == b["text"]
        assert len(a["segments"]) == len(b["segments"]) > 3
        for x, y in zip(a["segments"], b["segments"]):
            assert x["tokens"] == y["tokens"] and x["seek"] == y["seek"]
            assert abs(x["avg_logprob"] - y["avg_logprob"]) <= 1e-5
            wx, wy = x.get("words", []), y.get("words", [])
            assert [(w_["text"], w_["start"], w_["end"]) for w_ in wx] == [(w_["text"], w_["start"], w_["end"]) for w_ in wy]
            assert all(abs(p["confidence"] - q["confidence"]) <= 2e-3 for p, q in zip(wx, wy))


def test_alignment_rows_held_across_collections():
    """Alignment rows nobody has freed stay intact while later windows are decoded: only the first collection of
    decode_stream (and the first batch of decode_windows) gets the session's row buffer, every later one keeps a copy
    of its own.  Every window is aligned at the very end, and both paths give the same jumps."""
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from whisper_timestamped.tokenizer import get_tokenizer
    from whisper_timestamped.windows import make_decode_setup
    gm = wt.load_model("synthetic:tiny", device="cuda:0")
    tok = get_tokenizer(True, num_languages=gm.num_languages, language="en", task="transcribe")
    setup = make_decode_setup(tok, gm.dims.n_text_ctx)
    audio = synthetic_speech(200.0, seed=51)

    def aligned(eng, recs):
        qk_out = eng._session["qk_out"].data_ptr()
        assert [b.data_ptr() == qk_out for b in eng.qk_buffers] == [True] + [False] * (len(eng.qk_buffers) - 1)
        items = [dict(window=r.qk_window, row0=0, last_row=r.n_rows - 1, T=r.n_rows, f0=0, F=1500, max_dur=0) for r in recs]
        return eng.align(items)

    stream = CudaEngine(gm, max_batch=4)
    mel = stream.log_mel(stream.load_audio(audio))
    jobs = [dict(mel=mel, seek=s, segment_size=3000, prompt=setup.initial_tokens([])) for s in range(0, 20000, 2000)]
    got = {}
    stream.decode_stream(jobs, setup, lambda job, rec: got.__setitem__(job["seek"], rec))
    a = [got[j["seek"]] for j in jobs]
    rounds = CudaEngine(gm, max_batch=4)
    b = rounds.decode_windows(jobs, setup)
    assert len(stream.qk_buffers) > 2 and len(rounds.qk_buffers) == 3
    for k, (x, y, jx, jy) in enumerate(zip(a, b, aligned(stream, a), aligned(rounds, b))):
        assert x.tokens == y.tokens and x.n_rows == y.n_rows, k
        assert np.array_equal(jx, jy), k

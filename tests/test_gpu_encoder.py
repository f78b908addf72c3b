"""The audio half of the model, kernel by kernel, against float64 references of the same operations: log-mel
(`CudaEngine.log_mel`: `wts_frames`, the float32 DFT GEMM, `wts_power`, the filterbank GEMM, `wts_logmel_max`,
`wts_logmel_finish`), the encoder (`CudaEngine.encode`: `wts_window_gather`, the conv stem as GEMMs over overlapping
rows, the blocks with the fused `wts_enc_attention` or the unfused scores GEMM / `wts_softmax_rows` / P·V GEMM) and the
cross-K/V projection (`CudaEngine._cross_kv`) at every official width.

The references are pinned on the CPU: `ref_log_mel` to upstream's `log_mel_spectrogram` at 80 and 128 mels, and
`ref_encoder` to upstream's `AudioEncoder` run in float64 from the same state dict.  On the GPU, `ref_encoder` reads
exactly what the kernels read (the SB16 weight planes with the q/k scale folded in, the float32 LayerNorm parameters
and positional embedding, the SB16 value of every mel entry) and keeps every intermediate in float64.

Observed maxima on an NVIDIA H100 80GB HBM3 at a 700 W power limit are noted next to each bound; `pytest -s` prints
them (lines starting with ERR)."""
import gc
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from whisper_timestamped import model_zoo as zoo
from whisper_timestamped.model import mel_filterbank

import oracle_engine  # noqa: F401  (puts oracle/upstream on sys.path: `whisper` below is the oracle stand-in)

N_SAMPLES, N_AUDIO, KPAD = 480000, 1500, 1504

# name: (D, H, n_mels, alignment heads of the 2 decoder layers), the decode-step test's head sets: every width has a
# layer with a single head other than 0 and one with several heads including the last; `small` has a layer without
# alignment heads, `medium` puts the several-head layer first.
WIDTHS = {
    "tiny": (384, 6, 80, [(0, 4), (1, 0), (1, 3), (1, 5)]),
    "base": (512, 8, 80, [(0, 1), (1, 2), (1, 6), (1, 7)]),
    "small": (768, 12, 80, [(1, 0), (1, 5), (1, 11)]),
    "medium": (1024, 16, 80, [(0, 0), (0, 7), (0, 15), (1, 11)]),
    "large-v3": (1280, 20, 128, [(0, 7), (1, 0), (1, 13), (1, 19)]),
}

# Bounds: about 4x the largest error observed on an NVIDIA H100 80GB HBM3 at 700 W (`pytest -s` prints them).
# log-mel, in output units ((log10 + 4) / 4): `far` = entries more than 2 decades of power above the floor max - 8
# (observed 1.21e-5, 30 s of speech at 128 mels); `floor` = the floor the GPU used and the largest entry (observed
# 1.8e-7).  Entries within 2 decades of the floor are held to NEAR_K x the error upstream's own float32 path has on the
# same entries, plus `far` (observed at most 2.4x upstream's, 7.3 s of speech at 128 mels; 6.7e-5 at most, a 20-Hz tone).
MEL_TOL = dict(far=5e-5, floor=8e-7)
NEAR_K = 4.0
# encoder output (ln_post, SB16) per width and depth (0 = conv stem + ln_post, 2 = two blocks), every configuration;
# observed at depth 0 / 2:
#   tiny      4.34e-5 / 6.81e-5
#   base      5.44e-5 / 7.36e-5
#   small     5.87e-5 / 7.89e-5
#   medium    6.58e-5 / 1.02e-4
#   large-v3  7.96e-5 / 1.04e-4
ENC_TOL = {"tiny": {0: 1.8e-4, 2: 2.8e-4}, "base": {0: 2.2e-4, 2: 3.0e-4}, "small": {0: 2.4e-4, 2: 3.2e-4},
           "medium": {0: 2.7e-4, 2: 4.1e-4}, "large-v3": {0: 3.2e-4, 2: 4.2e-4}}
FULL_DEPTH_TOL = 5.1e-4  # 32-block large-v3 encoder, observed 1.27e-4
STEM_TOL = 5e-5          # conv1 (SB16 out) and conv2 + positional embedding (float32 out), relative to max(1, |ref|):
                         # observed 8.0e-6 and 1.29e-5
ATTN_TOL = 7e-5          # attention output (SB16): observed 1.56e-5 fused, 1.67e-5 unfused
SOFTMAX_TOL = 1e-5       # wts_softmax_rows probabilities: observed 2.4e-6, the 16 significant bits SB16 carries
F32_TOL = 1.3e-4         # float32 cross K/V before the fp16 rounding (the alignment heads' K, the last layer's V):
                         # observed 1.63e-5 (K) and 3.37e-5 (V), large-v3 at B = 64

def _dims(name, n_layer, n_text_layer=2):
    D, H, M, _ = WIDTHS[name]
    return zoo.ModelDimensions(n_mels=M, n_audio_ctx=N_AUDIO, n_audio_state=D, n_audio_head=H, n_audio_layer=n_layer,
                               n_vocab=51866 if M == 128 else 51865, n_text_ctx=448, n_text_state=D, n_text_head=H,
                               n_text_layer=n_text_layer)


def _report(tag, **errs):
    print(f"\nERR {tag} " + " ".join(f"{k}={v:.3e}" for k, v in errs.items()))


# ---------------------------------------------------------------------------------------------- float64 references
def ref_log10_mel(audio, n_mels, padding):
    """float64 log10 of the mel energies (clamped at 1e-10), time-major [frames, n_mels], before the max - 8 floor:
    reflect padding of 200 samples, periodic Hann window of 400, |rfft|^2, the last frame dropped, the Slaney
    filterbank (its float32 values, as upstream and the GPU multiply with)."""
    x = np.concatenate([np.asarray(audio, dtype=np.float64), np.zeros(padding)])
    x = np.pad(x, 200, mode="reflect")
    n_frames = (len(x) - 400) // 160
    win = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(400) / 400)
    fb = mel_filterbank(n_mels).astype(np.float64).T
    frames = np.lib.stride_tricks.sliding_window_view(x, 400)[::160]
    out = np.empty((n_frames, n_mels))
    for i in range(0, n_frames, 16384):                  # bounded memory for recordings of many minutes
        f = frames[i:min(i + 16384, n_frames)] * win
        out[i:i + len(f)] = (np.abs(np.fft.rfft(f, axis=-1)) ** 2) @ fb
    return np.log10(np.maximum(out, 1e-10))


def ref_log_mel(audio, n_mels, padding):
    """float64 log-mel [frames, n_mels]: `ref_log10_mel`, the max - 8 floor, then (x + 4) / 4."""
    lg = ref_log10_mel(audio, n_mels, padding)
    return (np.maximum(lg, lg.max() - 8.0) + 4.0) / 4.0


def _ln(x, g, b):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * g + b


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def ref_encoder(W, mel):
    """One window in float64: mel [3000, n_mels] (zero past the segment) -> encoder output [1500, D]."""
    x = F.pad(mel, (0, 0, 1, 1))                                              # conv1 padding: [3002, C]
    x = _gelu(x.unfold(0, 3, 1).transpose(1, 2).reshape(3000, -1) @ W["conv1"].T + W["conv1_b"])
    x = F.pad(x, (0, 0, 1, 0))                                                # conv2 reads rows 2t .. 2t + 2 of [3001, D]
    x = _gelu(x.unfold(0, 3, 2).transpose(1, 2).reshape(1500, -1) @ W["conv2"].T + W["conv2_b"]) + W["pos"]
    D, H = x.shape[1], W["H"]
    for L in W["layers"]:
        h = _ln(x, *L["ln1"])
        q, k = (h @ L["wqk"].T + L["bqk"]).split(D, -1)
        v = h @ L["wv"].T + L["bv"]
        q, k, v = (t.reshape(1500, H, 64).transpose(0, 1) for t in (q, k, v))
        att = (torch.softmax(q @ k.transpose(1, 2), -1) @ v).transpose(0, 1).reshape(1500, D)
        x = x + att @ L["wo"].T + L["bo"]
        x = x + _gelu(_ln(x, *L["ln2"]) @ L["w1"].T + L["b1"]) @ L["w2"].T + L["b2"]
    return _ln(x, *W["ln_post"])


def ref_weights_from_model(m):
    """float64 encoder weights exactly as the kernels read them: SB16 planes recombined (q/k scale folded in)."""
    w = m.w

    def f(sb):
        return sb.to_f32().double()

    def v(t):
        return t.double()
    layers = [dict(ln1=(v(b.attn.ln_g), v(b.attn.ln_b)), wqk=f(b.attn.qk), bqk=v(b.attn.qk_b), wv=f(b.attn.v),
                   bv=v(b.attn.v_b), wo=f(b.attn.out), bo=v(b.attn.out_b), ln2=(v(b.mlp_ln_g), v(b.mlp_ln_b)),
                   w1=f(b.fc1), b1=v(b.fc1_b), w2=f(b.fc2), b2=v(b.fc2_b)) for b in w.enc]
    return dict(H=m.dims.n_audio_head, conv1=f(w.conv1), conv1_b=v(w.conv1_b), conv2=f(w.conv2), conv2_b=v(w.conv2_b),
                pos=v(w.enc_pos), layers=layers, ln_post=(v(w.ln_post_g), v(w.ln_post_b)))


def ref_weights_from_state_dict(sd, dims):
    """The same weights from an openai-whisper state dict (float64, conv kernels tap-major, d_head^-1/4 folded into
    q and k)."""
    D, H, C = dims.n_audio_state, dims.n_audio_head, dims.n_mels
    s = (D // H) ** -0.25

    def g(k):
        return sd[k].double()
    layers = []
    for i in range(dims.n_audio_layer):
        p = f"encoder.blocks.{i}."
        layers.append(dict(
            ln1=(g(p + "attn_ln.weight"), g(p + "attn_ln.bias")),
            wqk=torch.cat([g(p + "attn.query.weight") * s, g(p + "attn.key.weight") * s]),
            bqk=torch.cat([g(p + "attn.query.bias") * s, torch.zeros(D, dtype=torch.float64)]),
            wv=g(p + "attn.value.weight"), bv=g(p + "attn.value.bias"),
            wo=g(p + "attn.out.weight"), bo=g(p + "attn.out.bias"),
            ln2=(g(p + "mlp_ln.weight"), g(p + "mlp_ln.bias")),
            w1=g(p + "mlp.0.weight"), b1=g(p + "mlp.0.bias"), w2=g(p + "mlp.2.weight"), b2=g(p + "mlp.2.bias")))
    return dict(H=H, conv1=g("encoder.conv1.weight").permute(0, 2, 1).reshape(D, 3 * C),
                conv1_b=g("encoder.conv1.bias"),
                conv2=g("encoder.conv2.weight").permute(0, 2, 1).reshape(D, 3 * D), conv2_b=g("encoder.conv2.bias"),
                pos=g("encoder.positional_embedding"), layers=layers,
                ln_post=(g("encoder.ln_post.weight"), g("encoder.ln_post.bias")))


def _sb16_value(x):
    """float64 value of the SB16 split of float32 x (hi = bf16(x), lo = bf16(x - hi)), as the GPU kernels write it."""
    hi, lo = _sb16_planes(x)
    return hi.double() + lo.double()


def _sb16_planes(x):
    x = x.float()
    hi = x.to(torch.bfloat16)
    return hi, (x - hi.float()).to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------- CPU pins
@pytest.mark.parametrize("n_mels", [80, 128])
def test_reference_log_mel_matches_upstream(n_mels):
    """CPU: `ref_log_mel` against upstream's float32 `log_mel_spectrogram`, with 30 s of padding and without, on
    speech-like audio and a tone: the difference is the float32 rounding of upstream."""
    import whisper
    from whisper_timestamped.synthetic_audio import synthetic_speech
    t = np.arange(16000 * 3) / 16000
    err = 0.0
    for audio in (synthetic_speech(7.3, seed=n_mels), (0.3 * np.sin(2 * np.pi * 440.0 * t)).astype(np.float32)):
        for padding in (N_SAMPLES, 0):
            want = whisper.log_mel_spectrogram(torch.from_numpy(audio), n_mels, padding=padding).numpy().T
            got = ref_log_mel(audio, n_mels, padding)
            assert got.shape == want.shape
            err = max(err, float(np.abs(got - want).max()))
    _report(f"ref_log_mel n_mels={n_mels}", err=err)
    assert err <= 1e-4, err                                  # observed 9.1e-6 (80 mels) and 2.3e-5 (128 mels)


@pytest.mark.parametrize("dims", [zoo.DIMS["tiny"], zoo.ModelDimensions(128, 1500, 128, 2, 2, 51866, 448, 128, 2, 2)],
                         ids=["tiny", "mel128"])
def test_reference_encoder_matches_upstream(dims, monkeypatch):
    """CPU: `ref_encoder` on weights taken from the state dict reproduces upstream's AudioEncoder run in float64 from
    the same state dict (float64 LayerNorm), for two windows of which one ends early (zero frames).  Upstream takes
    the softmax of the attention scores in float32 (`qk.float()`): that rounding is the whole difference."""
    from whisper.model import AudioEncoder, LayerNorm, disable_sdpa
    monkeypatch.setattr(LayerNorm, "forward", torch.nn.LayerNorm.forward)     # float64 LayerNorm (upstream: float32)
    dims = zoo.ModelDimensions(**{**dims.asdict(), "n_audio_layer": 2})
    sd = zoo.synthetic_state_dict(dims, seed=11)
    enc = AudioEncoder(dims.n_mels, dims.n_audio_ctx, dims.n_audio_state, dims.n_audio_head, dims.n_audio_layer)
    enc.load_state_dict({k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")})
    enc = enc.double()
    g = torch.Generator().manual_seed(5)
    mel = torch.rand((2, 3000, dims.n_mels), generator=g, dtype=torch.float64) * 3 - 1.5
    mel[1, 1700:] = 0.0
    with torch.no_grad(), disable_sdpa():
        want = enc(mel.transpose(1, 2))
    W = ref_weights_from_state_dict(sd, dims)
    err = max(float((ref_encoder(W, mel[b]) - want[b]).abs().max()) for b in range(2))
    _report(f"ref_encoder {dims.n_mels} mels D={dims.n_audio_state}", err=err)
    assert err <= 2e-6, err                                  # observed 4.9e-7 (tiny and mel128)


# ------------------------------------------------------------------------------------------- models and engines
_MODELS = {}


def _release():
    """Drop the cached model (an engine and its model reference each other: collect the cycle)."""
    _MODELS.clear()
    _REFS.clear()
    _MEL_ENGINES.clear()
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


@pytest.fixture(autouse=True, scope="module")
def _free_device_memory():
    gc.collect()                    # engines of earlier modules that only a reference cycle keeps alive
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield
    _release()


def _model(name, n_layer):
    """(model, float64 encoder weights from its SB16 planes): reduced-depth synthetic model of width `name` with
    `n_layer` encoder blocks and 2 decoder layers; one is cached at a time."""
    key = (name, n_layer)
    if key not in _MODELS:
        _release()
        from whisper_timestamped.model import WhisperB200
        dims = _dims(name, n_layer)
        sd = zoo.synthetic_state_dict(dims, seed=23 + n_layer)
        m = WhisperB200(dims, sd, "cuda", name=name, alignment_heads=WIDTHS[name][3])
        del sd
        _MODELS[key] = (m, ref_weights_from_model(m))
    return _MODELS[key]


def _engine(m, backend=0, conv_backend=None, fused=True):
    from whisper_timestamped.engine import CudaEngine
    eng = CudaEngine(m, gemm_backend=backend)
    eng.conv_backend = backend if conv_backend is None else conv_backend
    eng.fused_attention = fused
    return eng


def _bare_engine(backend):
    """An engine without a model, for the operators that take their operands as arguments."""
    from whisper_timestamped.engine import CudaEngine
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = torch.device("cuda:0"), backend, 0
    return eng


# ------------------------------------------------------------------------------------------------- log-mel on GPU
def _tone(freq, seconds, amp=0.5):
    return (amp * np.sin(2 * np.pi * freq * np.arange(int(seconds * 16000)) / 16000)).astype(np.float32)


def _audio(case):
    rng = np.random.default_rng(sum(map(ord, case)))
    from whisper_timestamped.synthetic_audio import synthetic_speech
    if case.startswith("len"):
        return (0.1 * rng.standard_normal(int(case[3:]))).astype(np.float32)
    if case == "30s":
        return synthetic_speech(30.0, seed=3)
    if case == "7.3s":
        return synthetic_speech(7.3, seed=4)
    if case == "20min":
        # low-level noise over 20 minutes, the loudest event (a 0.5-amplitude tone burst) in the last second
        x = (1e-3 * rng.standard_normal(20 * 60 * 16000)).astype(np.float32)
        x[-12000:-4000] += _tone(1234.5, 0.5)
        return x
    if case == "zeros":
        return np.zeros(5 * 16000, dtype=np.float32)
    if case == "quiet":
        return (1e-4 * rng.standard_normal(6 * 16000)).astype(np.float32)
    if case == "click":
        x = np.zeros(10 * 16000, dtype=np.float32)
        x[int(4.2 * 16000)] = 0.5
        return x
    if case == "dc":
        return np.full(5 * 16000, 0.3, dtype=np.float32)
    if case == "tone_low":
        return _tone(20.0, 4.0)
    if case == "tone_high":
        return _tone(7990.0, 4.0)
    raise KeyError(case)


# padding only: upstream's reflect pad needs more than 200 samples; 201 samples is the shortest segment the two-pass
# strategy sends without padding
MEL_CASES = {"len0": (True,), "len1": (True,), "len159": (True,), "len160": (True,), "len161": (True,),
             "len201": (True, False), "len361": (True, False), "30s": (True, False), "7.3s": (True, False),
             "20min": (True,), "zeros": (True, False), "quiet": (True, False), "click": (True, False),
             "dc": (True, False), "tone_low": (True, False), "tone_high": (True, False)}
_MEL_ENGINES = {}


def _mel_engine(n_mels):
    """An engine of a minimal model (D = 64, no encoder block) with the log-mel constants of `n_mels` bands."""
    if n_mels not in _MEL_ENGINES:
        from whisper_timestamped.model import WhisperB200
        dims = zoo.ModelDimensions(n_mels, N_AUDIO, 64, 1, 0, 51866 if n_mels == 128 else 51865, 448, 64, 1, 1)
        _MEL_ENGINES[n_mels] = _engine(WhisperB200(dims, zoo.synthetic_state_dict(dims, seed=1), "cuda"))
    return _MEL_ENGINES[n_mels]


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", [80, 128])
@pytest.mark.parametrize("case", list(MEL_CASES))
def test_log_mel_matches_float64(case, n_mels):
    """`CudaEngine.log_mel` against `ref_log_mel`.  Entries more than 2 decades of power above the floor are held to
    an absolute bound; entries within 2 decades of it (ill-conditioned in any float32 DFT) to a small multiple of the
    error upstream's float32 path has on the same entries.  The floor the GPU used (every entry the reference clamps
    deep below it) and the largest entry are held tightly: the floor shifts every entry."""
    import whisper
    eng = _mel_engine(n_mels)
    audio = _audio(case)
    errs = dict(far=0.0, near=0.0, near_upstream=0.0, floor=0.0)
    for pad in MEL_CASES[case]:
        padding = N_SAMPLES if pad else 0
        got = eng.log_mel(eng.load_audio(audio), pad_30s=pad).double().cpu().numpy()
        lg = ref_log10_mel(audio, n_mels, padding)
        floor = lg.max() - 8.0
        ref = (np.maximum(lg, floor) + 4.0) / 4.0
        assert got.shape == ref.shape, (got.shape, ref.shape)
        up = whisper.log_mel_spectrogram(torch.from_numpy(audio), n_mels, padding=padding).double().numpy().T
        if case == "zeros":
            assert bool((got == -1.5).all())
        if case == "quiet":
            assert lg.max() < 0.0                            # the negative branch of the max key
        e = np.abs(got - ref)
        near = lg < floor + 2.0
        e_far = float(e[~near].max()) if (~near).any() else 0.0
        e_near = float(e[near].max()) if near.any() else 0.0
        e_up = float(np.abs(up - ref)[near].max()) if near.any() else 0.0
        deep = lg < floor - 1.0
        e_floor = abs(float(got.max()) - float(ref.max()))
        if deep.any():
            g_floor = got[deep]
            assert bool((g_floor == g_floor[0]).all()), "entries below the floor differ"
            e_floor = max(e_floor, abs(float(g_floor[0]) - (floor + 4.0) / 4.0))
        for k, x in (("far", e_far), ("near", e_near), ("near_upstream", e_up), ("floor", e_floor)):
            errs[k] = max(errs[k], x)
        assert e_floor <= MEL_TOL["floor"], (pad, e_floor)
        assert e_far <= MEL_TOL["far"], (pad, e_far)
        assert e_near <= NEAR_K * e_up + MEL_TOL["far"], (pad, e_near, e_up)
    _report(f"log_mel {case} n_mels={n_mels}", **errs)


# ------------------------------------------------------------------------------------------ encoder operators
def _mel_pool(n_mels, lengths, seed):
    """Distinct log-mel-like tensors [n, n_mels] of the given lengths, each a view of a buffer whose rows after the
    content hold a sentinel (a gather that reads past the last content frame picks it up)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for n in lengths:
        buf = torch.full((n + 8, n_mels), 7.0, device="cuda")
        buf[:n] = torch.rand((n, n_mels), device="cuda", generator=g) * 3 - 1.5
        out.append(buf[:n])
    return out


def _window_specs(lengths, n, seed):
    """n (mel index, seek, segment_size) triples: sizes 1, 1499, 2999, 3000 and random ones, seeks at arbitrary frames,
    and windows that end on their mel's last content frame."""
    rng = np.random.default_rng(seed)
    specs = []
    for i in range(n):
        j = i % len(lengths)
        size = [3000, 1499, 1, 2999][i % 4] if i % 3 else int(rng.integers(2, 3000))
        size = min(size, lengths[j])
        seek = lengths[j] - size if i % 5 == 0 else int(rng.integers(0, lengths[j] - size + 1))
        specs.append((j, seek, size))
    return specs


def _gather(n_mels, mels, specs):
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    B = len(specs)
    ptrs = torch.tensor([mels[j].data_ptr() for j, _, _ in specs], dtype=torch.int64, device="cuda")
    seek = torch.tensor([s for _, s, _ in specs], dtype=torch.int32, device="cuda")
    size = torch.tensor([z for _, _, z in specs], dtype=torch.int32, device="cuda")
    x0 = SB16(B * 3002, n_mels, "cuda")
    x0.t.fill_(5.0)
    nat.check(nat.lib.wts_window_gather(ptrs.data_ptr(), n_mels, seek.data_ptr(), size.data_ptr(), B, x0.ptr, x0.plane,
                                        nat.stream_ptr("cuda")), "wts_window_gather")
    torch.cuda.synchronize()
    return x0


@pytest.mark.gpu
@pytest.mark.parametrize("n_mels", [80, 128])
def test_window_gather_exact(n_mels):
    """64 windows from three distinct mel tensors (one pointer per window): rows 0 and 3001 and every frame past the
    segment are exactly zero, every other row is exactly the SB16 split of the mel."""
    lengths = [3000, 4711, 9000]
    mels = _mel_pool(n_mels, lengths, seed=n_mels)
    specs = _window_specs(lengths, 64, seed=n_mels)
    assert {z for _, _, z in specs} >= {1, 1499, 2999, 3000}
    assert any(s + z == lengths[j] for j, s, z in specs)
    x0 = _gather(n_mels, mels, specs)
    planes = x0.t.view(2, 64, 3002, n_mels)
    for b, (j, seek, size) in enumerate(specs):
        want = torch.zeros((3002, n_mels), device="cuda")
        want[1:1 + size] = mels[j][seek:seek + size]
        hi, lo = _sb16_planes(want)
        assert torch.equal(planes[0, b], hi) and torch.equal(planes[1, b], lo), (b, seek, size)


def _stem(eng, w1, b1, w2, b2, pos, x0, B, C, D):
    """conv1 and conv2 exactly as `CudaEngine.encode` issues them: (h1 SB16 [B*3001, D], x float32 [B*1500, D])."""
    from whisper_timestamped.model import SB16
    h1 = SB16(B * 3001, D, "cuda")
    eng.gemm(x0, w1, 3000, D, 3 * C, lda=C, batch=(B, 1), a_b=(3002 * C, 0), bias=b1, act=1,
             out_sb=h1, ldo=D, o_b=(3001 * D, 0), o_off=D)
    x = torch.full((B * 1500, D), 9.0, device="cuda")
    eng.gemm(h1, w2, 1500, D, 3 * D, lda=2 * D, batch=(B, 1), a_b=(3001 * D, 0), bias=b2, act=1,
             residual=pos, ldr=D, r_b=(0, 0), out_f32=x, ldc=D, c_b=(1500 * D, 0))
    torch.cuda.synchronize()
    return h1, x


@pytest.mark.gpu
@pytest.mark.parametrize("backend", [0, 1])
@pytest.mark.parametrize("n_mels", [80, 128])
@pytest.mark.parametrize("name", list(WIDTHS))
def test_conv_stem_layout_of_encode(name, n_mels, backend):
    """conv1 (lda = C, K = 3C, GELU, SB16 out shifted by one row) and conv2 (lda = 2D, K = 3D, GELU, positional
    embedding as residual) on gathered windows, against float64 convolutions of the same SB16 values."""
    from whisper_timestamped.model import SB16
    D = WIDTHS[name][0]
    C = n_mels
    eng = _bare_engine(backend)
    g = torch.Generator(device="cuda").manual_seed(D + C + backend)
    lengths = [3000, 5000]
    mels = _mel_pool(C, lengths, seed=D)
    specs = [(0, 0, 3000), (1, 1234, 1777), (1, 2000, 3000)]
    B = len(specs)
    x0 = _gather(C, mels, specs)
    w1 = SB16.from_f32(torch.randn((D, 3 * C), device="cuda", generator=g) / math.sqrt(3 * C))
    w2 = SB16.from_f32(torch.randn((D, 3 * D), device="cuda", generator=g) / math.sqrt(3 * D))
    b1 = 0.1 * torch.randn(D, device="cuda", generator=g)
    b2 = 0.1 * torch.randn(D, device="cuda", generator=g)
    pos = zoo.sinusoids(N_AUDIO, D).float().cuda()
    h1, x = _stem(eng, w1, b1, w2, b2, pos, x0, B, C, D)
    W = dict(conv1=w1.to_f32().double(), conv1_b=b1.double(), conv2=w2.to_f32().double(), conv2_b=b2.double())
    xin = x0.to_f32().double().view(B, 3002, C)
    h1g = h1.to_f32().double().view(B, 3001, D)
    e1 = e2 = 0.0
    for b in range(B):
        r1 = _gelu(xin[b].unfold(0, 3, 1).transpose(1, 2).reshape(3000, -1) @ W["conv1"].T + W["conv1_b"])
        assert bool((h1g[b, 0] == 0).all())
        e1 = max(e1, float((h1g[b, 1:] - r1).abs().max()) / max(1.0, float(r1.abs().max())))
        # conv2 from the h1 the GPU wrote (its SB16 value), so the two GEMMs are checked separately
        r2 = _gelu(h1g[b].unfold(0, 3, 2).transpose(1, 2).reshape(1500, -1) @ W["conv2"].T + W["conv2_b"]) + pos.double()
        e2 = max(e2, float((x.view(B, 1500, D)[b].double() - r2).abs().max()) / max(1.0, float(r2.abs().max())))
    _report(f"stem {name} C={C} backend={backend}", conv1=e1, conv2=e2)
    assert e1 <= STEM_TOL and e2 <= STEM_TOL, (e1, e2)


def _attention_inputs(B, H, n_ctx, seed):
    """q|k (SB16 [B*n_ctx, 2D]) and V^T (SB16 [B*D, ld]) with score rows of every kind, per head (query index mod 5):
    0 random (scores ~ N(0, 1)); 1 peaked (q.k = +-30 on key 777 or key n_ctx - 5); 2 flat (q = 0); 3 the maximum and
    most of the mass in the partial last key tile (the last 92 keys get +12); 4 every score <= 0 (all shifted by -20),
    where keys past n_ctx read as zero would win."""
    from whisper_timestamped.model import SB16
    D = H * 64
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn((B, n_ctx, H, 64), device="cuda", generator=g) * 64 ** -0.25
    k = torch.randn((B, n_ctx, H, 64), device="cuda", generator=g) * 64 ** -0.25
    q[..., 61:] = 0.0
    k[..., 61:] = 0.0
    kind = torch.arange(n_ctx, device="cuda") % 5
    peak = min(777, n_ctx - 5)
    k[:, peak, :, 63] = 1.0
    k[:, max(0, n_ctx - 92):, :, 62] = 1.0
    k[..., 61] = 1.0
    sign = torch.where(torch.arange(n_ctx, device="cuda") % 2 == 0, 30.0, -30.0)
    q[:, kind == 1, :, 63] = sign[kind == 1][None, :, None]
    q[:, kind == 2] = 0.0
    q[:, kind == 3, :, 62] = 12.0
    q[:, kind == 4, :, 61] = -20.0
    qk = SB16.from_f32(torch.cat([q.reshape(B * n_ctx, D), k.reshape(B * n_ctx, D)], 1))
    ld = (n_ctx + 7) // 8 * 8
    vt = SB16.from_f32(torch.randn((B * D, ld), device="cuda", generator=g))
    return qk, vt, ld


def _check_attention(out, qk, vt, B, H, n_ctx, ld):
    """Largest error of the attention output (SB16 [B*n_ctx, D]) against float64 softmax(q k^T) v of the SB16
    operands, window by window."""
    D = H * 64
    got = out.to_f32().view(B, n_ctx, D)
    x = qk.to_f32().view(B, n_ctx, 2, H, 64)
    vt = vt.to_f32().view(B, H, 64, ld)
    err = 0.0
    for b in range(B):
        q, k = x[b, :, 0].double().transpose(0, 1), x[b, :, 1].double().transpose(0, 1)     # [H, n, 64]
        v = vt[b, :, :, :n_ctx].double().transpose(1, 2)                                   # [H, n, 64]
        ref = (torch.softmax(q @ k.transpose(1, 2), -1) @ v).transpose(0, 1).reshape(n_ctx, D)
        err = max(err, float((got[b].double() - ref).abs().max()))
    return err


@pytest.mark.gpu
@pytest.mark.parametrize("n_ctx", [1500, 1408, 100])
@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("H", [6, 8, 12, 16, 20])
def test_enc_attention_fused_score_rows(H, B, n_ctx):
    """wts_enc_attention against float64 softmax(q k^T) v of the same SB16 values, on peaked, flat, tail-heavy and
    all-negative score rows; n_ctx = 1500 (partial last key tile), 1408 (whole tiles) and 100 (one partial tile)."""
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    if n_ctx != 1500 and B == 64:
        pytest.skip("the other key counts run at B <= 3")
    D = H * 64
    qk, vt, ld = _attention_inputs(B, H, n_ctx, seed=100 * H + B + n_ctx)
    out = SB16(B * n_ctx, D, "cuda")
    nat.check(nat.lib.wts_enc_attention(qk.ptr, 2 * D, qk.plane, vt.ptr, ld, vt.plane, B, H, D, n_ctx, out.ptr, D,
                                        out.plane, nat.stream_ptr("cuda")), "wts_enc_attention")
    torch.cuda.synchronize()
    err = _check_attention(out, qk, vt, B, H, n_ctx, ld)
    _report(f"enc_attention H={H} B={B} n_ctx={n_ctx}", err=err)
    assert err <= ATTN_TOL, err


@pytest.mark.gpu
@pytest.mark.parametrize("backend", [0, 1])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("H", [6, 8, 12, 16, 20])
def test_enc_attention_unfused_score_rows(H, B, backend):
    """The unfused attention as `encode` issues it (WTS_FUSED_ATTN=0 and backend 1): scores GEMM into float32 rows of
    pitch 1504, wts_softmax_rows over n = 1500, P V GEMM; on the same score rows as the fused kernel."""
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    D, n = H * 64, N_AUDIO
    eng = _bare_engine(backend)
    qk, vt, ld = _attention_inputs(B, H, n, seed=7 * H + B)
    assert ld == KPAD                                            # V^T at the encoder's padded pitch
    S = torch.full((B * H * n, KPAD), float("nan"), device="cuda")
    P = SB16(B * H * n, KPAD, "cuda")
    att = SB16(B * n, D, "cuda")
    eng.gemm(qk, qk, n, n, 64, lda=2 * D, ldb=2 * D, b_off=D, batch=(B, H), a_b=(n * 2 * D, 64), b_b=(n * 2 * D, 64),
             out_f32=S, ldc=KPAD, c_b=(H * n * KPAD, n * KPAD))
    nat.check(nat.lib.wts_softmax_rows(S.data_ptr(), KPAD, B * H * n, n, P.ptr, KPAD, P.plane, nat.stream_ptr("cuda")),
              "wts_softmax_rows")
    eng.gemm(P, vt, n, 64, n, lda=KPAD, ldb=KPAD, batch=(B, H), a_b=(H * n * KPAD, n * KPAD), b_b=(D * KPAD, 64 * KPAD),
             out_sb=att, ldo=D, o_b=(n * D, 64))
    torch.cuda.synchronize()
    err = _check_attention(att, qk, vt, B, H, n, ld)
    _report(f"unfused attention H={H} B={B} backend={backend}", err=err)
    assert err <= ATTN_TOL, err


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 1500, 2048])
def test_softmax_rows(n):
    """wts_softmax_rows against float64 softmax: random, peaked (+30) and constant rows and rows holding -inf; the
    pitch padding past n (NaN) is never read and the output past n is never written."""
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    rows, ld = 9, n + 8
    g = torch.Generator(device="cuda").manual_seed(n)
    s = torch.randn((rows, ld), device="cuda", generator=g) * 4
    s[1, n // 2] = 30.0
    s[2, :n] = 0.5
    s[3, ::3] = -float("inf")
    s[3, n - 1] = 1.0
    s[4, : n - 1] = -float("inf")                      # one finite entry: probability 1
    s[5, 1::2] = -float("inf")
    s[6] *= 1e-3
    s[:, n:] = float("nan")
    out = SB16(rows, ld, "cuda")
    out.t.fill_(2.0)
    nat.check(nat.lib.wts_softmax_rows(s.data_ptr(), ld, rows, n, out.ptr, ld, out.plane, nat.stream_ptr("cuda")),
              "wts_softmax_rows")
    torch.cuda.synchronize()
    got = out.to_f32()
    want = torch.softmax(s[:, :n].double(), -1)
    err = float((got[:, :n].double() - want).abs().max())
    assert bool((got[:, n:] == 4.0).all())
    assert bool((got[3, :n][s[3, :n] == -float("inf")] == 0).all())
    _report(f"softmax_rows n={n}", err=err)
    assert err <= SOFTMAX_TOL, err


# ---------------------------------------------------------------------------------------- the whole encoder
_REFS = {}


def _encoder_pool(name, n_layer):
    """Mel tensors and 64 window specs of a width, and the float64 reference of each window (computed on the GPU, one
    window at a time, cached with the model)."""
    m, W = _model(name, n_layer)
    key = (name, n_layer)
    if _REFS.get("key") != key:
        _REFS.clear()
        n_mels = m.dims.n_mels
        lengths = [3000, 4711, 9000]
        mels = _mel_pool(n_mels, lengths, seed=len(name) + n_layer)
        specs = _window_specs(lengths, 64, seed=n_mels + n_layer)
        refs = []
        with torch.no_grad():
            for j, seek, size in specs:
                x = torch.zeros((3000, n_mels), dtype=torch.float64, device="cuda")
                x[:size] = _sb16_value(mels[j][seek:seek + size])
                refs.append(ref_encoder(W, x).float())     # float32 copy: the errors are far above its rounding
        _REFS.update(key=key, mels=mels, specs=specs, refs=refs)
    return m, _REFS["mels"], _REFS["specs"], _REFS["refs"]


def _encode(eng, mels, specs, idx):
    jobs = [dict(mel=mels[specs[i][0]], seek=specs[i][1], segment_size=specs[i][2]) for i in idx]
    xa = eng.encode(jobs)
    torch.cuda.synchronize()
    return xa.to_f32().view(len(idx), N_AUDIO, -1)


# index sets of the batches: every window of a smaller batch is also window i of the 64-window batch
BATCHES = {1: [5], 2: [0, 63], 17: list(range(26, 9, -1)), 64: list(range(64))}
# (gemm backend, conv backend, fused attention); the unfused paths keep B * H * 1500^2 scores, so they run at B = 2
CONFIGS = {"b0": (0, 0, True), "b0-unfused": (0, 0, False), "b1": (1, 1, False), "b0-conv1": (0, 1, True),
           "b1-conv0": (1, 0, False)}


@pytest.mark.gpu
@pytest.mark.parametrize("n_layer", [0, 2])
@pytest.mark.parametrize("name", list(WIDTHS))
def test_encoder_matches_float64(name, n_layer):
    """encode() of batches of 1, 2, 17 and 64 windows (three mel tensors, arbitrary seeks and sizes) against the
    float64 encoder, every window; depth 0 is the conv stem + ln_post alone.  Every window of a smaller batch is bit
    for bit the same window of the 64-window batch: each output is a fixed-order sum whatever the batch.  The other
    configurations (unfused attention, backend 1, conv backend differing from the main one) run at B = 2."""
    m, mels, specs, refs = _encoder_pool(name, n_layer)
    tol = ENC_TOL[name][n_layer]
    errs = {}
    eng = _engine(m)
    full = _encode(eng, mels, specs, BATCHES[64])
    for B, idx in BATCHES.items():
        got = full if B == 64 else _encode(eng, mels, specs, idx)
        for r, i in enumerate(idx):
            e = float((got[r] - refs[i]).abs().max())
            errs["b0"] = max(errs.get("b0", 0.0), e)
            assert e <= tol, ("b0", B, i, e)
            assert torch.equal(got[r], full[i]), ("batch invariance", B, i)
    del full, eng
    for cfg, (backend, conv, fused) in CONFIGS.items():
        if cfg == "b0":
            continue
        got = _encode(_engine(m, backend, conv, fused), mels, specs, BATCHES[2])
        for r, i in enumerate(BATCHES[2]):
            e = float((got[r] - refs[i]).abs().max())
            errs[cfg] = max(errs.get(cfg, 0.0), e)
            assert e <= tol, (cfg, i, e)
    _report(f"encoder {name} layers={n_layer}", **errs)


@pytest.mark.gpu
def test_full_depth_large_v3_encoder():
    """The 32-block synthetic large-v3 encoder on 2 windows (backend 0, fused attention) against float64."""
    name = "large-v3"
    m, W = _model(name, 32)
    n_mels = m.dims.n_mels
    mels = _mel_pool(n_mels, [3000, 4711], seed=32)
    specs = [(0, 0, 3000), (1, 1711, 3000)]
    got = _encode(_engine(m), mels, specs, [0, 1])
    err = 0.0
    with torch.no_grad():
        for r, (j, seek, size) in enumerate(specs):
            x = torch.zeros((3000, n_mels), dtype=torch.float64, device="cuda")
            x[:size] = _sb16_value(mels[j][seek:seek + size])
            err = max(err, float((got[r].double() - ref_encoder(W, x)).abs().max()))
    _release()
    _report("encoder large-v3 layers=32", err=err)
    assert err <= FULL_DEPTH_TOL, err


# ------------------------------------------------------------------------------------------------- cross-K/V
def _fp16_ulp(x16):
    """Spacing of float16 at the (float16) values x16, as float32."""
    _, e = torch.frexp(x16.float())
    ulp = torch.clamp(torch.pow(2.0, (e - 11).float()), min=2.0 ** -24)
    return torch.where(x16 == 0, torch.full_like(ulp, 2.0 ** -24), ulp)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 64])
@pytest.mark.parametrize("name", list(WIDTHS))
def test_cross_kv_from_encoder_output(name, B):
    """_cross_kv on an encode() output: fp16 K/V within one fp16 ulp of the float64 projection of the SB16 output
    rounded to fp16 (where |value| >= 1/4; below, fp16's spacing shrinks towards the float32 GEMM's own error, which
    is added), the float32 V of the last layer (left in the staging buffer) within the GEMM's error, the float32 K of each layer's alignment heads in its own slots, slots of windows past B (and
    the buffers of a layer without alignment heads) untouched."""
    m, mels, specs, _ = _encoder_pool(name, 2)
    eng = _engine(m)
    idx = BATCHES[64] if B == 64 else [7]
    jobs = [dict(mel=mels[specs[i][0]], seek=specs[i][1], segment_size=specs[i][2]) for i in idx]
    xa = eng.encode(jobs)
    cap = max(B, 3)
    st8 = eng._alloc_cross_state(cap)
    for li in range(m.dims.n_text_layer):
        st8["ck"][li].fill_(3.0)
        st8["cv"][li].fill_(3.0)
        if st8["ckal"][li] is not None:
            st8["ckal"][li].fill_(3.0)
    eng._cross_kv(xa, st8, B)
    torch.cuda.synchronize()
    D, H = m.dims.n_text_state, m.dims.n_text_head
    x = xa.to_f32().double().view(B, N_AUDIO, D)
    errs = dict(k16_ulps=0.0, v16_ulps=0.0, kal=0.0, v32=0.0)
    for li, blk in enumerate(m.w.dec):
        c = blk.cross
        wk, wv, bv = c.k.to_f32().double(), c.v.to_f32().double(), c.v_b.double()
        s0, n_l = eng.layer_slots[li]
        assert (st8["ckal"][li] is None) == (n_l == 0)
        V_last = torch.empty((B, H, N_AUDIO, 64), dtype=torch.float64, device="cuda")
        for b in range(B):
            K = (x[b] @ wk.T).view(N_AUDIO, H, 64).transpose(0, 1)                     # [H, 1500, 64]
            V = (x[b] @ wv.T + bv).view(N_AUDIO, H, 64).transpose(0, 1)
            V_last[b] = V
            for n, want, key in (("ck", K, "k16_ulps"), ("cv", V, "v16_ulps")):
                w16 = want.half()
                d = (st8[n][li][b].float() - w16.float()).abs()
                ulp = _fp16_ulp(w16)
                big = want.abs() >= 0.25                # there one fp16 ulp is 2^-12 or more, far above float32 error
                ulps = float((d[big] / ulp[big]).max())
                errs[key] = max(errs[key], ulps)
                assert ulps <= 1.0, (n, li, b, ulps)
                assert bool((d <= ulp + F32_TOL).all()), (n, li, b, float((d - ulp).max()))
            for h in range(H):
                s = int(eng.head_slot[li, h])
                if s >= 0:
                    e = float((st8["ckal"][li][b, s - s0].double() - K[h]).abs().max())
                    errs["kal"] = max(errs["kal"], e)
                    assert e <= F32_TOL, (li, b, h, e)
        if li == m.dims.n_text_layer - 1:
            e = float((st8["kvtmp"][:B].double() - V_last).abs().max())
            errs["v32"] = e
            assert e <= F32_TOL, ("v32", e)
        for n in ("ck", "cv", "ckal"):
            t = st8[n][li]
            if t is not None and cap > B:
                assert bool((t[B:] == 3.0).all()), (n, li, "a slot past B changed")
    _report(f"cross_kv {name} B={B}", **errs)

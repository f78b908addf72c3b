"""load_model() and the device-resident Whisper weights of the H100 drop-in.

Replaces `load_model` (/root/reference/whisper_timestamped/transcribe.py:2405-2544) for the
openai-whisper checkpoint format ({"dims": ..., "model_state_dict": ...}; key names as produced by
hf_to_whisper_states, T.py:2876-2907).  No network here: official names resolve to a local
`<download_root>/<name>.pt` if present; `synthetic:<name>` builds the seeded synthetic weights of
model_zoo.synthetic_state_dict (benchmarks / parity tests).

Weights are re-laid-out once for the kernels: every Linear/Conv weight becomes a K-major SB16
(split-bf16) matrix, q/k projections absorb the d_head^-1/4 scale, q|k|v (self) and k|v (cross)
projections are concatenated, conv kernels are flattened tap-major so the convolutions are plain GEMMs
over overlapping rows of the (zero-padded) input.
"""
import math
import os
from types import SimpleNamespace

import torch

from . import _native as nat
from . import model_zoo as zoo


class SB16:
    """A float32 matrix carried as two bfloat16 planes (hi, lo) — the GEMM operand format."""

    def __init__(self, rows, cols, device, ld=None):
        self.rows, self.cols = rows, cols
        self.ld = ld or cols
        self.t = torch.zeros((2, rows, self.ld), dtype=torch.bfloat16, device=device)

    @property
    def plane(self):
        return self.rows * self.ld

    @property
    def ptr(self):
        return self.t.data_ptr()

    @staticmethod
    def from_f32(x: torch.Tensor):
        x = x.contiguous().float()
        assert x.dim() == 2 and x.is_cuda
        out = SB16(x.shape[0], x.shape[1], x.device)
        nat.check(nat.lib.wts_to_sb16(nat.ptr(x), x.numel(), out.t[0].data_ptr(), out.t[1].data_ptr(),
                                      nat.stream_ptr(x.device)), "wts_to_sb16")
        return out

    def to_f32(self):
        return self.t[0].float() + self.t[1].float()


class WhisperB200:
    """What `load_model` returns: .dims, .device, .is_multilingual, .num_languages, .alignment_heads,
    .transcribe(audio, **opts), .engine()."""

    def __init__(self, dims: zoo.ModelDimensions, state_dict, device, name=None, alignment_heads=None):
        if not torch.cuda.is_available():
            raise nat.WtsError("whisper_timestamped (H100 drop-in) needs a CUDA device: there is no CPU fallback")
        self.dims = dims
        self.name = name
        self.device = torch.device(device if device is not None else "cuda")
        self.heads = list(alignment_heads) if alignment_heads is not None else zoo.default_alignment_heads(dims)
        mask = torch.zeros(dims.n_text_layer, dims.n_text_head, dtype=torch.bool)
        for l, h in self.heads:
            mask[l, h] = True
        self.alignment_heads = mask.to_sparse()
        # heads in the order `alignment_heads.indices().T` enumerates them (T.py:1545): layer-major
        self.heads = sorted(self.heads)
        self._engine = None
        self.w = self._prepare(state_dict)

    # ---- reference-facing properties (upstream Whisper)
    @property
    def is_multilingual(self):
        return self.dims.n_vocab >= 51865

    @property
    def num_languages(self):
        return self.dims.n_vocab - 51765 - int(self.is_multilingual)

    def engine(self):
        if self._engine is None:
            from .engine import CudaEngine
            self._engine = CudaEngine(self)
        return self._engine

    def transcribe(self, audio, **opts):
        from .transcribe import transcribe_timestamped
        return transcribe_timestamped(self, audio, **opts)

    # ---- weight preparation
    def _prepare(self, sd):
        dev = self.device
        d = self.dims

        def g(name):
            return sd[name].to(dev, dtype=torch.float32).contiguous()

        def lin(wt):
            return SB16.from_f32(wt)

        w = SimpleNamespace()
        C, da = d.n_mels, d.n_audio_state
        w.conv1 = lin(g("encoder.conv1.weight").permute(0, 2, 1).reshape(da, 3 * C))
        w.conv1_b = g("encoder.conv1.bias")
        w.conv2 = lin(g("encoder.conv2.weight").permute(0, 2, 1).reshape(da, 3 * da))
        w.conv2_b = g("encoder.conv2.bias")
        w.enc_pos = g("encoder.positional_embedding")

        def attn_block(prefix, dm, n_head, cross, decoder=False):
            scale = (dm // n_head) ** -0.25
            b = SimpleNamespace()
            b.ln_g, b.ln_b = g(prefix + "_ln.weight"), g(prefix + "_ln.bias")
            q, qb = g(prefix + ".query.weight") * scale, g(prefix + ".query.bias") * scale
            k = g(prefix + ".key.weight") * scale
            v, vb = g(prefix + ".value.weight"), g(prefix + ".value.bias")
            zeros = torch.zeros_like(qb)
            if cross:
                b.q, b.q_b = lin(q), qb
                b.k = lin(k)
                b.v, b.v_b = lin(v), vb
            else:
                b.qkv = lin(torch.cat([q, k, v], 0))
                b.qkv_b = torch.cat([qb, zeros, vb]).contiguous()
                if not decoder:             # encoder only: separate q|k and v projections (V is produced transposed)
                    b.qk = lin(torch.cat([q, k], 0))
                    b.qk_b = torch.cat([qb, zeros]).contiguous()
                    b.v, b.v_b = lin(v), vb
            b.out, b.out_b = lin(g(prefix + ".out.weight")), g(prefix + ".out.bias")
            return b

        def block(prefix, dm, n_head, cross):
            blk = SimpleNamespace()
            blk.attn = attn_block(prefix + ".attn", dm, n_head, False, decoder=cross)
            blk.cross = attn_block(prefix + ".cross_attn", dm, n_head, True) if cross else None
            blk.mlp_ln_g, blk.mlp_ln_b = g(prefix + ".mlp_ln.weight"), g(prefix + ".mlp_ln.bias")
            blk.fc1, blk.fc1_b = lin(g(prefix + ".mlp.0.weight")), g(prefix + ".mlp.0.bias")
            blk.fc2, blk.fc2_b = lin(g(prefix + ".mlp.2.weight")), g(prefix + ".mlp.2.bias")
            return blk

        w.enc = [block(f"encoder.blocks.{i}", da, d.n_audio_head, False) for i in range(d.n_audio_layer)]
        w.ln_post_g, w.ln_post_b = g("encoder.ln_post.weight"), g("encoder.ln_post.bias")
        dt = d.n_text_state
        w.emb = g("decoder.token_embedding.weight")
        w.emb_sb = lin(w.emb)
        w.dec_pos = g("decoder.positional_embedding")
        w.dec = [block(f"decoder.blocks.{i}", dt, d.n_text_head, True) for i in range(d.n_text_layer)]
        w.ln_g, w.ln_b = g("decoder.ln.weight"), g("decoder.ln.bias")
        # per decoder layer: slot of each head in the alignment buffer (-1 = not an alignment head)
        slots = torch.full((d.n_text_layer, d.n_text_head), -1, dtype=torch.int32)
        for s, (l, h) in enumerate(self.heads):
            slots[l, h] = s
        w.head_slot = slots.to(dev)
        # log-mel constants: DFT basis [2*208, 400] (cos | -sin) and the mel filterbank [n_mels, 208]
        n = torch.arange(400, dtype=torch.float64)
        k = torch.arange(201, dtype=torch.float64)[:, None]
        ang = 2 * math.pi * k * n / 400.0
        basis = torch.zeros(416, 400, dtype=torch.float64)
        basis[:201] = torch.cos(ang)
        basis[208:409] = -torch.sin(ang)
        w.dft = basis.float().to(dev).contiguous()
        fb = torch.zeros(C, 208, dtype=torch.float32)
        fb[:, :201] = torch.from_numpy(mel_filterbank(C))
        w.melfb = fb.to(dev).contiguous()
        torch.cuda.synchronize(dev)
        return w


def mel_filterbank(n_mels: int):
    """librosa-style Slaney mel filterbank (sr 16 kHz, n_fft 400) — what upstream ships as
    assets/mel_filters.npz and `whisper.log_mel_spectrogram` multiplies with (T.py:1213)."""
    import numpy as np

    def hz_to_mel(f):
        f = np.asarray(f, dtype=np.float64)
        f_sp = 200.0 / 3
        min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
        return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)

    def mel_to_hz(m):
        m = np.asarray(m, dtype=np.float64)
        f_sp = 200.0 / 3
        min_log_hz, min_log_mel, logstep = 1000.0, 1000.0 / f_sp, np.log(6.4) / 27.0
        return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)

    fftfreqs = np.linspace(0, 8000.0, 201)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(8000.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, 201))
    for i in range(n_mels):
        weights[i] = np.maximum(0, np.minimum(-ramps[i] / fdiff[i], ramps[i + 2] / fdiff[i + 1]))
    weights *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return weights.astype(np.float32)


def load_model(name, device=None, backend="openai-whisper", download_root=None, in_memory=False, *,
               synthetic_seed=1234, synthetic_kwargs=None):
    """Same positional signature as the reference (T.py:2405-2411).

    name: an official model name, a path to an openai-whisper `.pt` checkpoint, or `synthetic:<official name>`.
    """
    if backend not in ("openai-whisper", "openai"):
        raise ValueError(f"backend '{backend}' is not supported by the H100 drop-in (only 'openai-whisper')")
    if isinstance(name, str) and name.startswith("synthetic:"):
        base = name.split(":", 1)[1]
        if base not in zoo.DIMS:
            raise RuntimeError(f"Model {base} not found; available models = {sorted(zoo.DIMS)}")
        dims = zoo.DIMS[base]
        sd = zoo.synthetic_state_dict(dims, seed=synthetic_seed, **(synthetic_kwargs or {}))
        return WhisperB200(dims, sd, device, name=base, alignment_heads=zoo.ALIGNMENT_HEADS.get(base))
    path = None
    if os.path.isfile(name):
        path = name
    elif name in zoo.DIMS:
        root = download_root or os.path.join(os.path.expanduser("~"), ".cache", "whisper")
        cand = os.path.join(root, name + ".pt")
        if os.path.isfile(cand):
            path = cand
        else:
            raise RuntimeError(
                f"checkpoint for '{name}' not found at {cand} and this environment has no network; "
                f"put the openai-whisper checkpoint there or use load_model('synthetic:{name}')")
    else:
        raise RuntimeError(f"Model {name} not found; available models = {sorted(zoo.DIMS)}")
    ckpt = torch.load(path, map_location="cpu")
    dims = zoo.ModelDimensions(**ckpt["dims"])
    base = os.path.splitext(os.path.basename(path))[0]
    return WhisperB200(dims, ckpt["model_state_dict"], device, name=base,
                       alignment_heads=zoo.ALIGNMENT_HEADS.get(base))

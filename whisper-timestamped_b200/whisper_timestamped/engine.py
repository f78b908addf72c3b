"""CUDA engine: log-mel, batched encoder, batched greedy decoder and batched alignment on one H100.

Everything on the device goes through libwts (hand-written sm_90a kernels behind the C-ABI of
include/wts.h); PyTorch only owns the buffers and the stream.  Replaces, for whole batches of 30-s
windows at a time, what the reference drives one window and one token at a time through upstream
`model.transcribe` and its forward hooks (/root/reference/whisper_timestamped/transcribe.py:887-904):

  log_mel()         whisper.log_mel_spectrogram                       (T.py:1213 / upstream transcribe)
  decode_windows()  AudioEncoder.forward + DecodingTask._main_loop + hook_attention_weights (T.py:783-793)
                    + hook_output_logits (T.py:849-881); cross-attention rows of the alignment heads are
                    written by the attention kernel itself into the [window, head, row, frame] buffer the
                    alignment kernels read — no hook, no device->host copy per token.
  align()           the numerical part of perform_word_alignment (T.py:1510-1581, 1648-1652)
"""
import ctypes
import os

import numpy as np
import torch

from . import _native as nat
from .alignment import attn_prep, dtw, plan_segments, split_jumps
from .model import SB16
from .windows import N_FRAMES, WindowRecord

N_SAMPLES = 480000
N_CTX_AUDIO = 1500
KPAD = 1504      # key dimension of score rows, padded so SB16 rows stay 16-byte aligned


def _i32(x, dev):
    return torch.as_tensor(np.asarray(x, dtype=np.int32)).to(dev)


class CudaEngine:
    def __init__(self, model, max_batch=None, gemm_backend=None, keep_full_logprobs=False, small_batch_rows=None):
        self.m = model
        self.dev = model.device
        self.w = model.w
        self.dims = model.dims
        self.max_batch = max_batch or int(os.environ.get("WTS_MAX_BATCH", "64"))
        self.backend = int(os.environ.get("WTS_GEMM_BACKEND", "0")) if gemm_backend is None else gemm_backend
        # the conv GEMMs read overlapping rows (row stride < K); WTS_CONV_BACKEND picks their kernel separately
        self.conv_backend = int(os.environ.get("WTS_CONV_BACKEND", str(self.backend)))
        self.fused_attention = os.environ.get("WTS_FUSED_ATTN", "1") != "0"
        self.keep_full_logprobs = keep_full_logprobs
        self.qk_buffers = []            # one [B, N, rows, 1500] float32 tensor per decode_windows call
        self.window_index = []          # global window id -> (buffer idx, b)
        self.full_logprobs = []         # per call (only when keep_full_logprobs)
        self.launches = 0
        self.use_graph = os.environ.get("WTS_CUDA_GRAPH", "1") != "0"
        # at most this many sequences still decoding -> the small-batch kernels take over (0 = never, at most 32).
        # Default 8: the lean kernels with mma.sync phases stream the weights without the per-GEMM tile set-up, which
        # pays off at a few active windows; tools/step_probe.py times both sides of the cut-over
        self.small_batch_rows = min(32, int(os.environ.get("WTS_SMALL_BATCH_ROWS", "8")) if small_batch_rows is None
                                    else int(small_batch_rows))
        self.small_batch_steps = 0
        self.decode_steps_run = 0
        self._graphs = {}
        self.profile = False            # when set, phases are bracketed with CUDA events (stage_ms())
        self._events = []
        self.heads = None
        self.set_alignment_heads(model.heads)

    # ------------------------------------------------------------------ alignment heads
    def set_alignment_heads(self, heads=None):
        """Heads whose cross-attention rows the decoder exports for word alignment, as (layer, head) pairs (None: the
        model's own heads); they get slots in layer-major order, so the heads of layer l hold the contiguous slots
        [s0_l, s0_l + n_l).  The slot tables, the per-layer float32 K copies and the decode session (and its CUDA
        graphs) are rebuilt only when the set changes."""
        heads = sorted((int(l), int(h)) for l, h in (self.m.heads if heads is None else heads))
        if heads == self.heads:
            return
        d = self.dims
        L, H = d.n_text_layer, d.n_text_head
        assert heads and all(0 <= l < L and 0 <= h < H for l, h in heads), heads
        assert len(set(heads)) == len(heads), "duplicate alignment heads"
        slots = torch.full((L, H), -1, dtype=torch.int32)
        for s_, (l, h) in enumerate(heads):
            slots[l, h] = s_
        self.heads = heads
        self.head_slot = slots.to(self.dev)
        counts = [sum(1 for l, _ in heads if l == li) for li in range(L)]
        self.layer_slots = [(sum(counts[:li]), counts[li]) for li in range(L)]      # (s0_l, n_l)
        self._session = None
        self._tf_state = None

    # ------------------------------------------------------------------ phase timers
    class _Phase:
        def __init__(self, eng, name):
            self.eng, self.name = eng, name

        def __enter__(self):
            if self.eng.profile:
                self.a = torch.cuda.Event(enable_timing=True)
                self.b = torch.cuda.Event(enable_timing=True)
                self.a.record(torch.cuda.current_stream(self.eng.dev))

        def __exit__(self, *exc):
            if self.eng.profile:
                self.b.record(torch.cuda.current_stream(self.eng.dev))
                self.eng._events.append((self.name, self.a, self.b))

    def phase(self, name):
        return CudaEngine._Phase(self, name)

    def stage_ms(self, reset=True):
        torch.cuda.synchronize(self.dev)
        out = {}
        self.batch_ms = [(B, steps, self._events[i][1].elapsed_time(self._events[i][2]))
                         for (B, steps, i) in getattr(self, "batch_log", [])]
        self.batch_log = []
        for name, a, b in self._events:
            out[name] = out.get(name, 0.0) + a.elapsed_time(b)
        if reset:
            self._events = []
        return out

    # ------------------------------------------------------------------ helpers
    def _st(self):
        return nat.stream_ptr(self.dev)

    def gemm(self, a, b, M, N, K, *, lda=None, ldb=None, a_plane=None, b_plane=None, a_off=0, b_off=0,
             batch=(1, 1), a_b=(0, 0), b_b=(0, 0), alpha=1.0, bias=None, bias_on_m=False, act=0,
             residual=None, ldr=0, r_b=(0, 0), out_f32=None, ldc=0, c_b=(0, 0), c_off=0,
             out_sb=None, ldo=0, o_plane=0, o_b=(0, 0), o_off=0, head_dim=0, head_stride=0,
             a_f32=False, b_f32=False, backend=None, row_mask=None, b_const=False):
        """a/b: SB16 objects (or float32 tensors with a_f32/b_f32).  Offsets/strides in elements.  b_const: b is a model
        weight that no kernel of the stream writes, so a decode-time GEMM may start loading it before the previous
        kernel has completed."""
        g = nat.Gemm()
        if a_f32:
            g.a, g.lda, g.a_plane = a.data_ptr() + 4 * a_off, lda, 0
        else:
            g.a, g.lda, g.a_plane = a.ptr + 2 * a_off, lda or a.ld, a_plane if a_plane is not None else a.plane
        if b_f32:
            g.b, g.ldb, g.b_plane = b.data_ptr() + 4 * b_off, ldb, 0
        else:
            g.b, g.ldb, g.b_plane = b.ptr + 2 * b_off, ldb or b.ld, b_plane if b_plane is not None else b.plane
        g.a_bo, g.a_bi = a_b
        g.b_bo, g.b_bi = b_b
        g.M, g.N, g.K = M, N, K
        g.batch_outer, g.batch_inner = batch
        g.alpha = alpha
        g.bias = bias.data_ptr() if bias is not None else None
        g.bias_on_m = 1 if bias_on_m else 0
        g.act = act
        if residual is not None:
            g.residual, g.ldr = residual.data_ptr(), ldr
            g.r_bo, g.r_bi = r_b
        if out_f32 is not None:
            g.out_f32, g.ldc = out_f32.data_ptr() + 4 * c_off, ldc
            g.c_bo, g.c_bi = c_b
        if out_sb is not None:
            g.out_sb16, g.ldo, g.o_plane = out_sb.ptr + 2 * o_off, ldo or out_sb.ld, o_plane or out_sb.plane
            g.o_bo, g.o_bi = o_b
        g.head_dim, g.head_stride = head_dim, head_stride
        g.backend = self.backend if backend is None else backend
        g.a_is_f32, g.b_is_f32 = int(a_f32), int(b_f32)
        g.row_mask = row_mask.data_ptr() if row_mask is not None else None
        g.b_const = int(b_const)
        if a_f32 or b_f32:
            g.backend = 1
        nat.check(nat.lib.wts_gemm(ctypes.byref(g), self._st()), "wts_gemm")
        self.launches += 1

    def layernorm(self, x, gamma, beta, M, D, out_sb=None, out_f32=None):
        nat.check(nat.lib.wts_layernorm(x.data_ptr(), D, gamma.data_ptr(), beta.data_ptr(), M, D,
                                        out_sb.ptr if out_sb is not None else None,
                                        out_sb.ld if out_sb is not None else 0,
                                        out_sb.plane if out_sb is not None else 0,
                                        out_f32.data_ptr() if out_f32 is not None else None, D, self._st()),
                  "wts_layernorm")
        self.launches += 1

    # ------------------------------------------------------------------ audio / log-mel
    def load_audio(self, audio):
        if isinstance(audio, str):
            import wave
            with wave.open(audio, "rb") as wv:
                if wv.getframerate() != 16000 or wv.getnchannels() != 1 or wv.getsampwidth() != 2:
                    raise RuntimeError("only 16 kHz mono s16 .wav files can be read here (no ffmpeg in this environment)")
                data = wv.readframes(wv.getnframes())
            audio = np.frombuffer(data, np.int16).astype(np.float32) / 32768.0
        if isinstance(audio, np.ndarray):
            audio = torch.from_numpy(np.ascontiguousarray(audio, dtype=np.float32))
        assert isinstance(audio, torch.Tensor), f"Got unexpected audio of type {type(audio)}"
        audio = audio.float()
        if audio.device != self.dev:
            audio = (audio.pin_memory() if audio.device.type == "cpu" else audio).to(self.dev, non_blocking=True)
        return audio.contiguous()

    def log_mel(self, audio, pad_30s=True):
        """float32 time-major log-mel [frames, n_mels] of `audio` + 30 s of zero padding (upstream
        log_mel_spectrogram(audio, n_mels, padding=N_SAMPLES)); the -8 floor uses this stream's maximum.
        pad_30s=False: no padding (the per-segment mel of the two-pass strategy, T.py:1213)."""
        with self.phase("mel"):
            return self._log_mel(audio, N_SAMPLES if pad_30s else 0)

    def _log_mel(self, audio, padding=N_SAMPLES):
        dev, st = self.dev, self._st()
        n = int(audio.numel())
        total = n + padding
        nf = total // 160
        C = self.dims.n_mels
        frames = torch.empty((nf, 400), dtype=torch.float32, device=dev)
        nat.check(nat.lib.wts_frames(audio.data_ptr(), n, total, nf, frames.data_ptr(), 0, st), "wts_frames")
        y = torch.empty((nf, 416), dtype=torch.float32, device=dev)
        self.gemm(frames, self.w.dft, nf, 416, 400, lda=400, ldb=400, a_f32=True, b_f32=True, out_f32=y, ldc=416)
        p = torch.empty((nf, 208), dtype=torch.float32, device=dev)
        nat.check(nat.lib.wts_power(y.data_ptr(), 416, nf, p.data_ptr(), 208, 0, st), "wts_power")
        mel = torch.empty((nf, C), dtype=torch.float32, device=dev)
        self.gemm(p, self.w.melfb, nf, C, 208, lda=208, ldb=208, a_f32=True, b_f32=True, out_f32=mel, ldc=C)
        key = torch.full((1,), -2 ** 31, dtype=torch.int32, device=dev)
        nat.check(nat.lib.wts_logmel_max(mel.data_ptr(), nf * C, key.data_ptr(), st), "wts_logmel_max")
        out = torch.empty((nf, C), dtype=torch.float32, device=dev)
        nat.check(nat.lib.wts_logmel_finish(mel.data_ptr(), nf, C, key.data_ptr(), out.data_ptr(), st), "wts_logmel_finish")
        self.launches += 6
        return out

    def mel_frames(self, mel):
        return int(mel.shape[0])

    # ------------------------------------------------------------------ encoder
    def encode(self, jobs):
        """jobs -> (xa SB16 [B*1500, d]).  conv1/conv2 as GEMMs over overlapping rows, then the blocks."""
        d, dev, st, w = self.dims, self.dev, self._st(), self.w
        B, C, D, H = len(jobs), d.n_mels, d.n_audio_state, d.n_audio_head
        ptrs = torch.as_tensor(np.array([j["mel"].data_ptr() for j in jobs], dtype=np.int64)).to(dev)
        seek = _i32([j["seek"] for j in jobs], dev)
        size = _i32([j["segment_size"] for j in jobs], dev)
        x0 = SB16(B * 3002, C, dev)
        nat.check(nat.lib.wts_window_gather(ptrs.data_ptr(), C, seek.data_ptr(), size.data_ptr(), B, x0.ptr, x0.plane, st),
                  "wts_window_gather")
        # conv1 (k=3, pad 1) + GELU: row t of the GEMM's A operand = padded rows t..t+2 (K = 3C, lda = C)
        h1 = SB16(B * 3001, D, dev)            # row 0 of every window stays zero = conv2's left padding
        self.gemm(x0, w.conv1, 3000, D, 3 * C, lda=C, batch=(B, 1), a_b=(3002 * C, 0), bias=w.conv1_b, act=1,
                  out_sb=h1, ldo=D, o_b=(3001 * D, 0), o_off=D, backend=self.conv_backend)
        # conv2 (k=3, stride 2, pad 1) + GELU + positional embedding: A row t = padded rows 2t..2t+2
        x = torch.empty((B * 1500, D), dtype=torch.float32, device=dev)
        self.gemm(h1, w.conv2, 1500, D, 3 * D, lda=2 * D, batch=(B, 1), a_b=(3001 * D, 0), bias=w.conv2_b, act=1,
                  residual=w.enc_pos, ldr=D, r_b=(0, 0), out_f32=x, ldc=D, c_b=(1500 * D, 0), backend=self.conv_backend)
        R = B * 1500
        hs = SB16(R, D, dev)
        qk = SB16(R, 2 * D, dev)
        vt = SB16(B * D, KPAD, dev)
        fused = self.backend == 0 and self.fused_attention
        if not fused:
            S = torch.empty((B * H * 1500, KPAD), dtype=torch.float32, device=dev)
            P = SB16(B * H * 1500, KPAD, dev)
        att = SB16(R, D, dev)
        mid = SB16(R, 4 * D, dev)
        for blk in w.enc:
            a = blk.attn
            self.layernorm(x, a.ln_g, a.ln_b, R, D, out_sb=hs)
            self.gemm(hs, a.qk, R, 2 * D, D, bias=a.qk_b, out_sb=qk)
            # V^T per window: [D, 1500] = Wv [D, D] x h^T  (swapped operands, bias along M)
            self.gemm(a.v, hs, D, 1500, D, batch=(B, 1), b_b=(1500 * D, 0), bias=a.v_b, bias_on_m=True,
                      out_sb=vt, ldo=KPAD, o_b=(D * KPAD, 0))
            if fused:
                # softmax(q k^T) v on the tensor cores, scores never leave the SM
                nat.check(nat.lib.wts_enc_attention(qk.ptr, 2 * D, qk.plane, vt.ptr, KPAD, vt.plane, B, H, D, 1500,
                                                    att.ptr, D, att.plane, st), "wts_enc_attention")
                self.launches += 1
            else:
                # scores[b, h] = q_h k_h^T  (scale folded into the weights)
                self.gemm(qk, qk, 1500, 1500, 64, lda=2 * D, ldb=2 * D, b_off=D, batch=(B, H),
                          a_b=(1500 * 2 * D, 64), b_b=(1500 * 2 * D, 64), out_f32=S, ldc=KPAD,
                          c_b=(H * 1500 * KPAD, 1500 * KPAD))
                nat.check(nat.lib.wts_softmax_rows(S.data_ptr(), KPAD, B * H * 1500, 1500, P.ptr, KPAD, P.plane, st),
                          "wts_softmax_rows")
                self.launches += 1
                # out[b, :, h*64:(h+1)*64] = P[b, h] x V_h   (B operand = rows h*64.. of V^T)
                self.gemm(P, vt, 1500, 64, 1500, lda=KPAD, ldb=KPAD, batch=(B, H),
                          a_b=(H * 1500 * KPAD, 1500 * KPAD), b_b=(D * KPAD, 64 * KPAD), out_sb=att, ldo=D,
                          o_b=(1500 * D, 64))
            self.gemm(att, a.out, R, D, D, bias=a.out_b, residual=x, ldr=D, out_f32=x, ldc=D)
            self.layernorm(x, blk.mlp_ln_g, blk.mlp_ln_b, R, D, out_sb=hs)
            self.gemm(hs, blk.fc1, R, 4 * D, D, bias=blk.fc1_b, act=1, out_sb=mid)
            self.gemm(mid, blk.fc2, R, D, 4 * D, bias=blk.fc2_b, residual=x, ldr=D, out_f32=x, ldc=D)
        xa = SB16(R, D, dev)
        self.layernorm(x, w.ln_post_g, w.ln_post_b, R, D, out_sb=xa)
        return xa

    # ------------------------------------------------------------------ decoder
    def _decoder_rows(self, st8, x, R, row_seq, row_pos, qk_row, qk_buf, active=None):
        """One pass of all decoder blocks over R query rows (ragged batch)."""
        d, w, st = self.dims, self.w, self._st()
        D, H, L = d.n_text_state, d.n_text_head, d.n_text_layer
        hs, qkv, att, q, mid = st8["hs"], st8["qkv"], st8["att"], st8["q"], st8["mid"]
        n_slots = len(self.heads)
        for li, blk in enumerate(w.dec):
            a, c = blk.attn, blk.cross
            s0, n_l = self.layer_slots[li]
            kal = st8["ckal"][li]
            self.layernorm(x, a.ln_g, a.ln_b, R, D, out_sb=hs)
            self.gemm(hs, a.qkv, R, 3 * D, D, bias=a.qkv_b, out_f32=qkv, ldc=3 * D, row_mask=active, b_const=True)
            fused_append = active is not None          # decode step: one row per sequence, the attention CTA appends K/V
            if not fused_append:
                nat.check(nat.lib.wts_kv_append(qkv.data_ptr() + 4 * D, qkv.data_ptr() + 8 * D, 3 * D, row_seq.data_ptr(),
                                                row_pos.data_ptr(), R, H, d.n_text_ctx, st8["sk"][li].data_ptr(),
                                                st8["sv"][li].data_ptr(), H * d.n_text_ctx * 64, st), "wts_kv_append")
                self.launches += 1
            nat.check(nat.lib.wts_decoder_attention(2 if fused_append else 0, qkv.data_ptr(), 3 * D, st8["sk"][li].data_ptr(),
                                                    st8["sv"][li].data_ptr(), H * d.n_text_ctx * 64, d.n_text_ctx,
                                                    row_seq.data_ptr(), row_pos.data_ptr(), R, H, att.ptr, att.ld,
                                                    att.plane, None, None, 0, 0, None,
                                                    active.data_ptr() if active is not None else None, st),
                      "wts_decoder_attention")
            self.gemm(att, a.out, R, D, D, bias=a.out_b, residual=x, ldr=D, out_f32=x, ldc=D, row_mask=active,
                      b_const=True)
            self.layernorm(x, c.ln_g, c.ln_b, R, D, out_sb=hs)
            self.gemm(hs, c.q, R, D, D, bias=c.q_b, out_f32=q, ldc=D, row_mask=active, b_const=True)
            nat.check(nat.lib.wts_cross_attention_f16_layer(
                q.data_ptr(), D, st8["ck"][li].data_ptr(), st8["cv"][li].data_ptr(), kal.data_ptr() if kal is not None else None,
                self.head_slot[li].data_ptr(), n_slots, s0, n_l, N_CTX_AUDIO, row_seq.data_ptr(), R, H, att.ptr, att.ld,
                att.plane, qk_buf.data_ptr(), qk_buf.shape[2], qk_row.data_ptr(),
                active.data_ptr() if active is not None else None, st), "wts_cross_attention_f16_layer")
            self.gemm(att, c.out, R, D, D, bias=c.out_b, residual=x, ldr=D, out_f32=x, ldc=D, row_mask=active,
                      b_const=True)
            self.layernorm(x, blk.mlp_ln_g, blk.mlp_ln_b, R, D, out_sb=hs)
            self.gemm(hs, blk.fc1, R, 4 * D, D, bias=blk.fc1_b, act=1, out_sb=mid, row_mask=active, b_const=True)
            self.gemm(mid, blk.fc2, R, D, 4 * D, bias=blk.fc2_b, residual=x, ldr=D, out_f32=x, ldc=D, row_mask=active,
                      b_const=True)
            self.launches += 2

    def _alloc_decoder_state(self, B, R):
        """Decoder state of B sequences: the cross-attention K/V buffers, self-attention K/V caches and the activation
        buffers of R query rows."""
        d, dev = self.dims, self.dev
        D, H, L = d.n_text_state, d.n_text_head, d.n_text_layer
        f32 = dict(dtype=torch.float32, device=dev)
        st8 = self._alloc_cross_state(B)
        st8.update(hs=SB16(R, D, dev), att=SB16(R, D, dev), mid=SB16(R, 4 * D, dev),
                   qkv=torch.empty((R, 3 * D), **f32), q=torch.empty((R, D), **f32),
                   sk=[torch.zeros((B, H, d.n_text_ctx, 64), **f32) for _ in range(L)],
                   sv=[torch.zeros((B, H, d.n_text_ctx, 64), **f32) for _ in range(L)])
        return st8

    def _alloc_cross_state(self, B):
        """Cross-attention K/V buffers for B windows (also the staging area of windows admitted into a session)."""
        d, dev = self.dims, self.dev
        H, L = d.n_text_head, d.n_text_layer
        return dict(
            ck=[torch.empty((B, H, N_CTX_AUDIO, 64), dtype=torch.float16, device=dev) for _ in range(L)],
            cv=[torch.empty((B, H, N_CTX_AUDIO, 64), dtype=torch.float16, device=dev) for _ in range(L)],
            # float32 K of each layer's own alignment heads only (none: no buffer)
            ckal=[torch.empty((B, n_l, N_CTX_AUDIO, 64), dtype=torch.float32, device=dev) if n_l else None
                  for (_, n_l) in self.layer_slots],
            kvtmp=torch.empty((B, H, N_CTX_AUDIO, 64), dtype=torch.float32, device=dev))

    def _cross_kv(self, xa, st8, B):
        d = self.dims
        D, H = d.n_text_state, d.n_text_head
        for li, blk in enumerate(self.w.dec):
            c = blk.cross
            tmp = st8["kvtmp"]
            s0, n_l = self.layer_slots[li]
            for (wt, bias, dst, al) in ((c.k, None, st8["ck"][li], st8["ckal"][li]), (c.v, c.v_b, st8["cv"][li], None)):
                self.gemm(xa, wt, 1500, D, D, batch=(B, 1), a_b=(1500 * D, 0), bias=bias, out_f32=tmp, ldc=64,
                          c_b=(H * 1500 * 64, 0), head_dim=64, head_stride=1500 * 64)
                nat.check(nat.lib.wts_cross_kv_pack_layer(tmp.data_ptr(), dst.data_ptr(),
                                                          al.data_ptr() if al is not None else None,
                                                          self.head_slot[li].data_ptr(), s0, n_l, B, H, N_CTX_AUDIO,
                                                          self._st()), "wts_cross_kv_pack_layer")
                self.launches += 1

    def _final_logits(self, x_rows, n_rows, logits, hs=None, row_mask=None):
        """LN + tied-embedding projection of `n_rows` float32 rows -> logits [n_rows, V].  hs: the SB16 LN output (a
        fresh one when None; the decode step passes its own so that a captured graph allocates nothing)."""
        d, w = self.dims, self.w
        D, V = d.n_text_state, d.n_vocab
        if hs is None:
            hs = SB16(n_rows, D, self.dev)
        self.layernorm(x_rows, w.ln_g, w.ln_b, n_rows, D, out_sb=hs)
        self.gemm(hs, w.emb_sb, n_rows, V, D, out_f32=logits, ldc=V, row_mask=row_mask, b_const=True)

    def decode_windows(self, jobs, setup):
        if getattr(setup, "beam_size", None) is not None or setup.temperature > 0:
            # upstream decoding strategies (beam search / best-of-n sampling): one window at a time, n_group hypotheses
            return [self._decode_strategy(job, setup) for job in jobs]
        out = []
        limit = self.batch_limit(setup)
        for i in range(0, len(jobs), limit):
            out.extend(self._decode_batch(jobs[i:i + limit], setup))
        return out

    def window_bytes(self, sample_len):
        """Device bytes one window of a decode batch needs: its slot of the decode session (cross K/V, float32 K of the
        alignment heads, self-attention caches, alignment rows and the buffer they are collected into) and the encoder
        activations of the window."""
        d = self.dims
        L, H, D, n_ctx = d.n_text_layer, d.n_text_head, d.n_text_state, d.n_text_ctx
        N, ctx = len(self.heads), N_CTX_AUDIO
        cross = L * H * ctx * 64 * 2 * 2 + N * ctx * 64 * 4 + H * ctx * 64 * 4
        self_kv = 2 * L * H * n_ctx * 64 * 4
        rows = 2 * N * (sample_len + 1) * ctx * 4
        Da = d.n_audio_state
        encoder = 3002 * d.n_mels * 4 + 3001 * Da * 4 + ctx * Da * (4 + 4 + 8 + 4 + 16 + 4) + Da * KPAD * 4
        return cross + self_kv + rows + encoder

    def batch_limit(self, setup):
        """Windows per decode batch: WTS_MAX_BATCH (default 64), lowered when that many windows of this head set
        would not fit in 85 % of the device memory that is free when the first batch of the head set is sized (torch's
        unused cached blocks are returned first: fragments of them cannot hold a session's multi-GB buffers)."""
        key = (tuple(self.heads), setup.sample_len)
        lim = getattr(self, "_limits", {})
        if key not in lim:
            torch.cuda.empty_cache()
            free, _ = torch.cuda.mem_get_info(self.dev)
            ses = getattr(self, "_session", None)
            if ses is not None:                                    # the session of the same head set is reused
                free += ses["cap"] * self.window_bytes(setup.sample_len)
            lim[key] = max(1, min(self.max_batch, int(0.85 * free) // self.window_bytes(setup.sample_len)))
            self._limits = lim
        return lim[key]

    def _decoder_session(self, setup, need):
        """Persistent decode state for up to `max_batch` windows: KV caches, token buffers, the alignment buffer
        and ONE captured CUDA graph of a decode step.  Every batch reuses it (unused slots are marked done and
        skipped by the attention / select kernels), so the graph is captured once per engine, not per batch."""
        d, dev = self.dims, self.dev
        tok = setup.tokenizer
        V, D, n_ctx = d.n_vocab, d.n_text_state, d.n_text_ctx
        ses = getattr(self, "_session", None)
        cap = 4
        while cap < need:
            cap *= 2
        cap = min(cap, max(self.batch_limit(setup), need))
        if ses is not None and ses["cap"] >= need:
            cap = ses["cap"]                      # a smaller batch reuses the larger session (and its graph)
        key = (cap, setup.sample_len, tok.eot, tok.timestamp_begin, tok.no_timestamps, setup.max_initial_timestamp_index,
               self.keep_full_logprobs, self.small_batch_rows)
        if ses is not None and ses["key"] == key:
            return ses
        self._session = ses = None
        qk_rows = setup.sample_len + 1
        n_slots = len(self.heads)
        i32 = dict(dtype=torch.int32, device=dev)
        ses = dict(key=key, cap=cap, qk_rows=qk_rows, graph=None, per_step=0)
        ses["st8"] = self._alloc_decoder_state(cap, cap)
        ses["st8"]["hs_fin"] = SB16(cap, D, dev)
        ses["tokens"] = torch.zeros((cap, n_ctx + 1), **i32)
        ses["n_tokens"] = torch.ones(cap, **i32)
        ses["n_prompt"] = torch.ones(cap, **i32)
        ses["done"] = torch.ones(cap, **i32)
        ses["logprobs"] = torch.zeros((cap, qk_rows), dtype=torch.float32, device=dev)
        ses["no_speech"] = torch.zeros(cap, dtype=torch.float32, device=dev)
        ses["full"] = torch.empty((cap, qk_rows, V), dtype=torch.float32, device=dev) if self.keep_full_logprobs else None
        ses["qk_buf"] = torch.zeros((cap, max(1, n_slots), qk_rows, N_CTX_AUDIO), dtype=torch.float32, device=dev)
        # the alignment rows of a batch (or of a collection of continuous batching) are collected here (allocated once:
        # no multi-GB allocation per batch); while earlier rows still occupy it (not yet aligned and freed), the rows
        # get a copy of their own
        ses["qk_out"] = torch.zeros_like(ses["qk_buf"])
        ses["qk_out_idx"] = None
        ses["s_tok"] = torch.zeros(cap, **i32)
        ses["s_pos"] = torch.zeros(cap, **i32)
        ses["s_qkr"] = torch.zeros(cap, **i32)
        ses["s_act"] = torch.zeros(cap, **i32)
        ses["seq_ids"] = _i32(list(range(cap)), dev)
        ses["logits"] = torch.empty((cap, V), dtype=torch.float32, device=dev)
        ses["xs"] = torch.empty((cap, D), dtype=torch.float32, device=dev)
        ses["last_full"] = torch.zeros((cap, V), dtype=torch.float32, device=dev)   # filtered log-softmax row at the limit
        ses["suppress"] = torch.zeros(V, dtype=torch.uint8, device=dev)
        ses["blank"] = torch.zeros(V, dtype=torch.uint8, device=dev)
        ses["cfg"] = nat.DecodeCfg(n_vocab=V, eot=tok.eot, timestamp_begin=tok.timestamp_begin,
                                   no_timestamps=tok.no_timestamps,
                                   max_initial_ts=-1 if setup.max_initial_timestamp_index is None else setup.max_initial_timestamp_index,
                                   sample_len=setup.sample_len, n_ctx=n_ctx, tokens_ld=n_ctx + 1)
        ses["steps"] = self._steps_descriptor(ses) if self.small_batch_rows > 0 else None
        self._session = ses
        return ses

    def _steps_descriptor(self, ses):
        """Arguments of the lean small-batch decode step (wts_decode_step_kernels): SB16 weights + this session's caches,
        token state and scratch.  None when the model's dimensions or the device are outside what the kernels support
        (those sessions decode every step with the per-operator graph)."""
        d, w, dev = self.dims, self.w, self.dev
        D, H, L, V = d.n_text_state, d.n_text_head, d.n_text_layer, d.n_vocab
        if D % 128 != 0 or D > 1280 or D != 64 * H:
            return None
        # one CTA per SM, and a CTA keeps at most two 8-feature tasks of the K = 4 D matrix-vector product (FC2)
        if D // 8 > 2 * torch.cuda.get_device_properties(dev).multi_processor_count:
            return None
        st8, cap = ses["st8"], ses["cap"]
        layers = (nat.DecLayer * L)()
        for li, blk in enumerate(w.dec):
            a, c, y = blk.attn, blk.cross, layers[li]
            y.ln1_g, y.ln1_b, y.b_qkv, y.b_o = a.ln_g.data_ptr(), a.ln_b.data_ptr(), a.qkv_b.data_ptr(), a.out_b.data_ptr()
            y.ln2_g, y.ln2_b, y.b_cq, y.b_co = c.ln_g.data_ptr(), c.ln_b.data_ptr(), c.q_b.data_ptr(), c.out_b.data_ptr()
            y.ln3_g, y.ln3_b = blk.mlp_ln_g.data_ptr(), blk.mlp_ln_b.data_ptr()
            y.b_fc1, y.b_fc2 = blk.fc1_b.data_ptr(), blk.fc2_b.data_ptr()
            y.self_k, y.self_v = st8["sk"][li].data_ptr(), st8["sv"][li].data_ptr()
            y.cross_k16, y.cross_v16 = st8["ck"][li].data_ptr(), st8["cv"][li].data_ptr()
            kal = st8["ckal"][li]
            y.cross_k_align, y.head_slot = kal.data_ptr() if kal is not None else None, self.head_slot[li].data_ptr()
            y.align_s0, y.align_n = self.layer_slots[li]
            for name, sb in (("qkv", a.qkv), ("o", a.out), ("cq", c.q), ("co", c.out), ("fc1", blk.fc1), ("fc2", blk.fc2)):
                assert sb.ld == sb.cols
                setattr(y, "sb_" + name, sb.ptr)
                setattr(y, "pl_" + name, sb.plane)
        raw = np.frombuffer(bytes(layers), dtype=np.uint8).copy()
        f32 = dict(dtype=torch.float32, device=dev)
        keep = dict(layers=torch.from_numpy(raw).to(dev), x=torch.zeros((cap, D), **f32), qkv=torch.zeros((cap, 3 * D), **f32),
                    att=torch.zeros((cap, D), **f32), q=torch.zeros((cap, D), **f32), mid=torch.zeros((cap, 4 * D), **f32))
        p = nat.DecodeSteps()
        p.layers = keep["layers"].data_ptr()
        p.emb, p.pos, p.ln_g, p.ln_b = w.emb.data_ptr(), w.dec_pos.data_ptr(), w.ln_g.data_ptr(), w.ln_b.data_ptr()
        p.tokens, p.n_tokens, p.n_prompt, p.done = (ses[k].data_ptr() for k in ("tokens", "n_tokens", "n_prompt", "done"))
        p.logprobs, p.qk_buf = ses["logprobs"].data_ptr(), ses["qk_buf"].data_ptr()
        p.full = ses["full"].data_ptr() if ses["full"] is not None else None
        p.last_full = ses["last_full"].data_ptr()
        p.suppress, p.blank = ses["suppress"].data_ptr(), ses["blank"].data_ptr()
        p.x, p.qkv, p.att, p.q, p.mid = (keep[k].data_ptr() for k in ("x", "qkv", "att", "q", "mid"))
        p.logits = ses["logits"].data_ptr()
        p.emb_sb, p.emb_plane = w.emb_sb.ptr, w.emb_sb.plane
        p.cfg = ses["cfg"]
        p.n_layer, p.D, p.H, p.n_ctx, p.n_audio_ctx = L, D, H, d.n_text_ctx, N_CTX_AUDIO
        p.n_slots, p.cap, p.lp_ld, p.qk_rows = len(self.heads), cap, ses["qk_rows"], ses["qk_rows"]
        return dict(args=p, keep=keep, host_layers=layers, graphs={})

    def _capture(self, ses, run):
        """CUDA graph of `run()`, one decode step.  Every kernel must have run once outside capture (lazy module loading
        and cudaFuncSetAttribute are not capturable), so `run()` is called once first on the live token state, which is
        restored afterwards: that call is not a decode step of the caller.  The capture itself runs nothing."""
        dev = self.dev
        saved = {k: ses[k].clone() for k in ("tokens", "n_tokens", "done", "logprobs")}
        run()
        torch.cuda.synchronize(dev)
        for k, v in saved.items():
            ses[k].copy_(v)
        graph = torch.cuda.CUDAGraph()
        cap_stream = torch.cuda.Stream(device=dev)
        cap_stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(cap_stream):
            with torch.cuda.graph(graph, stream=cap_stream):
                run()
        torch.cuda.current_stream(dev).wait_stream(cap_stream)
        return graph

    def _lean_graph(self, ses, n_active):
        """CUDA graph of ONE decoder step as the chain of lean per-phase kernels (wts_decode_step_kernels), with grids
        sized for 4 / 8 / 16 / 32 active rows, the smallest that fits `n_active`; captured on first use."""
        sd = ses["steps"]
        rows = 4 if n_active <= 4 else 8 if n_active <= 8 else 16 if n_active <= 16 else 32
        if rows not in sd["graphs"]:
            p = sd["args"]

            def launch():
                p.max_rows = rows
                nat.check(nat.lib.wts_decode_step_kernels(ctypes.byref(p), ctypes.byref(sd["host_layers"]), self._st()),
                          "wts_decode_step_kernels")
            sd["graphs"][rows] = self._capture(ses, launch)
        return sd["graphs"][rows]

    def _step_graph(self, ses):
        """ONE captured CUDA graph of a per-operator decode step (captured on first use)."""
        if ses["graph"] is None:
            l0 = self.launches
            ses["graph"] = self._capture(ses, lambda: self._step(ses))
            ses["per_step"] = (self.launches - l0) // 2       # the warm-up step and the recorded one
            self.launches -= ses["per_step"]
        return ses["graph"]

    def _decode_chunk(self, ses, n_active, chunk, max_steps):
        """`chunk` decode steps of every slot still decoding: the lean small-batch graph when at most `small_batch_rows`
        windows are left, else the per-operator step (one graph, or plain launches for short decodes)."""
        if ses["steps"] is not None and n_active <= self.small_batch_rows:
            graph = self._lean_graph(ses, n_active)
            for _ in range(chunk):
                graph.replay()
            self.launches += chunk * (8 * self.dims.n_text_layer + 3)
            self.small_batch_steps += chunk
        else:
            graph = self._step_graph(ses) if (self.use_graph and max_steps > 4) else None
            for _ in range(chunk):
                if graph is not None:
                    graph.replay()
                    self.launches += ses["per_step"]
                else:
                    self._step(ses)
        self.decode_steps_run += chunk

    def _set_masks(self, ses, setup):
        """Token masks of the logit filters: suppressed tokens, and the tokens blanked at the first sampled position."""
        dev = self.dev
        ses["suppress"].zero_()
        ses["suppress"][torch.as_tensor(list(setup.suppress_tokens), dtype=torch.long, device=dev)] = 1
        ses["blank"].zero_()
        if setup.blank_tokens:
            ses["blank"][torch.as_tensor(list(setup.blank_tokens), dtype=torch.long, device=dev)] = 1

    def _prefill(self, ses, prompts, slots, tok, qk_last):
        """Every prompt token of every window in one ragged batch through the decoder (own activation buffers, the
        session's caches), then the final logits of each prompt's last row and of its <|startoftranscript|> row, and the
        <|nospeech|> probability at the latter.  slots: session slot of each prompt; qk_last: the last prompt row writes
        alignment row 0 of the session's qk buffer.  Returns (logits [2 n, V]: last rows, then SOT rows; no_speech [n])."""
        d, dev, st, w = self.dims, self.dev, self._st(), self.w
        D, V = d.n_text_state, d.n_vocab
        n = len(prompts)
        P = [len(p) for p in prompts]
        R0 = sum(P)
        row_seq = _i32([b for b, p in zip(slots, prompts) for _ in p], dev)
        row_pos = _i32([i for p in prompts for i in range(len(p))], dev)
        row_tok = _i32([t for p in prompts for t in p], dev)
        qk_row = _i32([0 if qk_last and i == len(p) - 1 else -1 for p in prompts for i in range(len(p))], dev)
        f32 = dict(dtype=torch.float32, device=dev)
        pre = dict(ses["st8"])
        pre.update(hs=SB16(R0, D, dev), att=SB16(R0, D, dev), mid=SB16(R0, 4 * D, dev),
                   qkv=torch.empty((R0, 3 * D), **f32), q=torch.empty((R0, D), **f32))
        x = torch.empty((R0, D), **f32)
        nat.check(nat.lib.wts_embed(row_tok.data_ptr(), row_pos.data_ptr(), w.emb.data_ptr(), w.dec_pos.data_ptr(), R0, D,
                                    x.data_ptr(), st), "wts_embed")
        self._decoder_rows(pre, x, R0, row_seq, row_pos, qk_row, ses["qk_buf"])
        ends = np.cumsum(P) - 1
        sot_rows = [int(ends[k] - P[k] + 1 + prompts[k].index(tok.sot)) for k in range(n)]
        sel = _i32(list(ends) + sot_rows, dev)
        xr = torch.empty((2 * n, D), **f32)
        nat.check(nat.lib.wts_gather_rows(x.data_ptr(), D, sel.data_ptr(), 2 * n, D, xr.data_ptr(), st), "wts_gather_rows")
        logits2 = torch.empty((2 * n, V), **f32)
        self._final_logits(xr, 2 * n, logits2)
        no_speech = torch.zeros(n, **f32)
        if tok.no_speech is not None:
            nat.check(nat.lib.wts_softmax_pick(logits2.data_ptr() + 4 * n * V, V, V, tok.no_speech, no_speech.data_ptr(), n, st),
                      "wts_softmax_pick")
        return logits2, no_speech

    def _select(self, ses, logits, rows):
        d = self.dims
        nat.check(nat.lib.wts_decode_select(logits.data_ptr(), d.n_vocab, ctypes.byref(ses["cfg"]), ses["suppress"].data_ptr(),
                                            ses["blank"].data_ptr(), ses["tokens"].data_ptr(), ses["n_tokens"].data_ptr(),
                                            ses["n_prompt"].data_ptr(), ses["done"].data_ptr(), ses["logprobs"].data_ptr(),
                                            ses["qk_rows"], ses["full"].data_ptr() if ses["full"] is not None else None,
                                            ses["last_full"].data_ptr(), rows, self._st()), "wts_decode_select")
        self.launches += 1

    def _step(self, ses):
        """One decode step for all `cap` slots (identical launch sequence every step: CUDA-graph friendly)."""
        self._step_logits(ses)
        self._select(ses, ses["logits"], ses["cap"])
        self.launches += 1

    def _step_logits(self, ses):
        """The forward part of a decode step: logits of the next position of every active slot (no choice made)."""
        d, w, st = self.dims, self.w, self._st()
        cap, D = ses["cap"], d.n_text_state
        nat.check(nat.lib.wts_step_inputs(ses["tokens"].data_ptr(), d.n_text_ctx + 1, ses["n_tokens"].data_ptr(),
                                          ses["n_prompt"].data_ptr(), ses["done"].data_ptr(), cap, ses["s_tok"].data_ptr(),
                                          ses["s_pos"].data_ptr(), ses["s_qkr"].data_ptr(), ses["s_act"].data_ptr(), st),
                  "wts_step_inputs")
        nat.check(nat.lib.wts_embed(ses["s_tok"].data_ptr(), ses["s_pos"].data_ptr(), w.emb.data_ptr(), w.dec_pos.data_ptr(),
                                    cap, D, ses["xs"].data_ptr(), st), "wts_embed")
        self._decoder_rows(ses["st8"], ses["xs"], cap, ses["seq_ids"], ses["s_pos"], ses["s_qkr"], ses["qk_buf"],
                           active=ses["s_act"])
        self._final_logits(ses["xs"], cap, ses["logits"], hs=ses["st8"]["hs_fin"], row_mask=ses["s_act"])
        self.launches += 1

    # ------------------------------------------------------------------ the life of a decode slot
    # Token state of slot b, as wts_step_inputs and wts_decode_select read it: tokens[b, :n_tokens[b]], of which the
    # first n_prompt[b] are the prompt; done[b] = 0 running, 1 ended by <|endoftext|>, 2 stopped at the decoding limit;
    # logprobs[b, r]: log-prob of the token chosen at row r.  A window is seeded into a slot (_seed, inside _admit),
    # decoded, and collected into a WindowRecord with its alignment rows (_collect).
    def _park(self, ses):
        """Every slot parked (one token, done): the step and select kernels skip it until a window is seeded into it."""
        ses["tokens"].zero_()
        ses["n_tokens"].fill_(1)
        ses["n_prompt"].fill_(1)
        ses["done"].fill_(1)
        ses["logprobs"].zero_()

    def _slot_index(self, slots):
        """Index of `slots` in the session's per-slot tensors: a slice (views, in-place copies) when they are 0..n-1,
        else a device index."""
        slots = list(slots)
        if slots == list(range(len(slots))):
            return slice(0, len(slots))
        return torch.as_tensor(slots, dtype=torch.long, device=self.dev)

    def _seed(self, ses, slots, prompts):
        """`prompts` written into `slots`, which are set running; the other slots keep their state."""
        sel = self._slot_index(slots)
        th = np.zeros((len(prompts), ses["tokens"].shape[1]), dtype=np.int32)
        for k, p in enumerate(prompts):
            th[k, :len(p)] = p
        nt = np.array([len(p) for p in prompts], dtype=np.int32)
        for key, rows in (("tokens", th), ("n_tokens", nt), ("n_prompt", nt)):
            rows = torch.from_numpy(rows)
            ses[key][sel] = rows if isinstance(sel, slice) else rows.to(self.dev)    # a slice view takes host rows
        ses["done"][sel] = 0
        ses["logprobs"][sel] = 0.0

    def _admit(self, ses, batch, setup):
        """Windows into decode slots, batch = [(slot, job)]: encoder, cross-attention K/V, token state, prompt prefill
        and the first sampled token; the windows' <|nospeech|> probabilities stay in ses["no_speech"].  Slots 0..n-1
        are written in place.  Other slots get their cross K/V through a staging buffer, and their first token is
        selected with every other slot parked (the select kernel works on slots 0..rows-1)."""
        st8 = ses["st8"]
        n = len(batch)
        slots = [s for s, _ in batch]
        sel = self._slot_index(slots)
        direct = isinstance(sel, slice)
        with self.phase("encoder"):
            xa = self.encode([j for _, j in batch])
        with self.phase("cross_kv"):
            if direct:
                self._cross_kv(xa, st8, n)
            else:
                tmp = self._alloc_cross_state(n)
                self._cross_kv(xa, tmp, n)
                for li in range(self.dims.n_text_layer):
                    for name in ("ck", "cv", "ckal"):
                        if st8[name][li] is not None:
                            st8[name][li].index_copy_(0, sel, tmp[name][li])
                del tmp
        del xa
        prompts = [list(j["prompt"]) for _, j in batch]
        self._seed(ses, slots, prompts)
        with self.phase("prefill"):
            logits2, no_speech = self._prefill(ses, prompts, slots, setup.tokenizer, qk_last=True)
            if direct:
                self._select(ses, logits2, n)
            else:
                cap = ses["cap"]
                ses["logits"].index_copy_(0, sel, logits2[:n])
                saved = ses["done"].clone()
                ses["done"].fill_(1)
                ses["done"].index_fill_(0, sel, 0)
                self._select(ses, ses["logits"], cap)
                mask = torch.zeros(cap, dtype=torch.bool, device=self.dev)
                mask[sel] = True
                ses["done"].copy_(torch.where(mask, ses["done"], saved))
                self.launches += 4
            ses["no_speech"][sel] = no_speech

    def _collect(self, ses, batch, setup):
        """Records of the windows decoded in batch = [(slot, job)], in that order.  Their alignment rows are kept as
        one buffer: the session's qk_out when no earlier rows occupy it, else a copy of their own."""
        dev = self.dev
        n = len(batch)
        sel = self._slot_index([s for s, _ in batch])
        tokens_h, n_tok_h, done_h, lp_h, ns_h = (ses[k][sel].cpu().numpy()
                                                 for k in ("tokens", "n_tokens", "done", "logprobs", "no_speech"))
        prompts = [list(j["prompt"]) for _, j in batch]
        n_new = n_tok_h - np.array([len(p) for p in prompts])          # sampled tokens of each window
        max_rows = int(n_new.max()) + 1
        qk_buf, held = ses["qk_buf"], ses["qk_out_idx"]
        if held is None or held >= len(self.qk_buffers) or self.qk_buffers[held] is None:
            rows = ses["qk_out"][:n]
            ses["qk_out_idx"] = len(self.qk_buffers)
        else:
            rows = torch.empty((n, qk_buf.shape[1], max_rows, N_CTX_AUDIO), dtype=torch.float32, device=dev)
        rows[:, :, :max_rows] = qk_buf[sel, :, :max_rows]
        first = self._keep_rows(rows)
        full = ses["full"]
        if full is not None:
            full = full[sel, :max_rows].clone()
            self.full_logprobs.append(full)
        limit = [k for k in range(n) if int(done_h[k]) == 2]
        last_full = {}
        if limit:       # windows that ran into the decoding limit: the reference may need chunk_logprobs[-1][fallback]
            lf = ses["last_full"][torch.as_tensor([batch[k][0] for k in limit], device=dev)].cpu()
            last_full = {k: lf[i] for i, k in enumerate(limit)}
        records = []
        for k, (_, job) in enumerate(batch):
            P, n_k = len(prompts[k]), int(n_new[k])
            ended = int(done_h[k]) == 1
            n_rows = n_k + 1 if ended else n_k
            last_lp = None
            if k in last_full:
                last_lp = (lambda t, row=last_full[k]: float(row[t]))
            elif full is not None:
                last_lp = (lambda t, kk=k, rr=n_rows - 1, ff=full: float(ff[kk, rr, t].item()))
            records.append(WindowRecord(seek=job["seek"], segment_size=job["segment_size"], prompt=prompts[k],
                                        tokens=tokens_h[k, P:P + n_k].tolist(), logprobs=lp_h[k, :n_rows].copy(),
                                        ended_by_eot=ended, no_speech_prob=float(ns_h[k]), qk_window=first + k,
                                        temperature=0.0, language=job.get("language", setup.tokenizer.language),
                                        last_row_logprobs=last_lp))
        return records

    @torch.no_grad()
    def _decode_batch(self, jobs, setup):
        B = len(jobs)
        ses = self._decoder_session(setup, B)
        assert B <= ses["cap"]
        self._park(ses)                            # slots >= B stay parked
        self._set_masks(ses, setup)
        batch = list(enumerate(jobs))
        self._admit(ses, batch, setup)
        max_steps = setup.sample_len - 1
        steps_done = 0
        done = ses["done"]
        n_active = B
        with self.phase("decode_steps"):
            while steps_done < max_steps and n_active > 0:
                chunk = min(8, max_steps - steps_done)
                self._decode_chunk(ses, n_active, chunk, max_steps)
                steps_done += chunk
                n_active = int((done == 0).sum().item())
        if self.profile:
            self.batch_log = getattr(self, "batch_log", [])
            self.batch_log.append((B, steps_done, len(self._events) - 1))
        return self._collect(ses, batch, setup)

    # ------------------------------------------------------------------ continuous batching
    @torch.no_grad()
    def decode_stream(self, jobs, setup, feed, collected=None):
        """Greedy decoding with CONTINUOUS batching: decode `jobs`; as soon as a window finishes its record goes to
        `feed(job, record)`, which may return the next window of that audio stream (upstream's seek loop: the follow-up
        window of a 30-s cut, or the next window of a long file) — it is encoded, prefilled and admitted into the freed
        slot while the other windows keep decoding.  The round-based `decode_windows` makes every round wait for its
        slowest window (a stuck one runs to the 224-token limit) before the follow-up windows even start.
        Same kernels, same per-window arithmetic as `decode_windows`; only the grouping of windows into steps differs.
        `collected()`, when given, is called after the records of each collection have been fed."""
        assert not self.keep_full_logprobs, "decode_stream keeps no per-row log-prob tables"
        queue = list(jobs)
        if not queue:
            return
        ses = self._decoder_session(setup, min(self.batch_limit(setup), len(queue)))
        cap = ses["cap"]
        self._park(ses)
        self._set_masks(ses, setup)
        slot_job = [None] * cap               # job decoded in each slot
        free = list(range(cap))
        max_steps = setup.sample_len - 1
        done = ses["done"]
        while queue or any(j is not None for j in slot_job):
            if queue and free:
                batch = []
                while queue and free:
                    batch.append((free.pop(0), queue.pop(0)))
                self._admit(ses, batch, setup)
                for b, job in batch:
                    slot_job[b] = job
            with self.phase("decode_steps"):
                n_active = int((done == 0).sum().item())
                if n_active > 0:
                    self._decode_chunk(ses, n_active, 8, max_steps)
            done_h = done.cpu().numpy()
            finished = [(b, slot_job[b]) for b in range(cap) if slot_job[b] is not None and int(done_h[b]) != 0]
            if finished:
                for (b, job), rec in zip(finished, self._collect(ses, finished, setup)):
                    slot_job[b] = None
                    nxt = feed(job, rec)
                    if nxt is not None:
                        queue.append(nxt)
                if collected is not None:
                    collected()
                free.extend(b for b, _ in finished)
                free.sort()

    # ------------------------------------------------------------------ beam search / sampling (upstream strategies)
    @torch.no_grad()
    def _decode_strategy(self, job, setup):
        """One window through upstream's BeamSearchDecoder (temperature 0, beam_size hypotheses) or GreedyDecoder at a
        temperature > 0 (best_of sampled hypotheses), MaximumLikelihoodRanker on top — what the reference reaches through
        model.transcribe() in its two-pass strategy (T.py:1068; options T.py:104-113).

        The forward of every step (all hypotheses = rows of the per-operator step: KV caches, attention, tensor-core
        GEMMs) and the logit filters + log-softmax (wts_filtered_logprobs) run on the device; the hypothesis
        bookkeeping is upstream's, on the host: top-(beam+1) candidates per row, de-duplicated per sequence, best
        beam_size kept, finished pool, patience; sampling draws from torch's global CPU generator exactly like the
        reference on CPU does (Categorical over the filtered rows).  KV-cache rows follow their source hypothesis."""
        d, dev, st = self.dims, self.dev, self._st()
        tok = setup.tokenizer
        G = setup.n_group
        beam = setup.beam_size
        T = float(setup.temperature)
        ses = self._decoder_session(setup, G)
        cap, st8 = ses["cap"], ses["st8"]
        V, L, n_ctx = d.n_vocab, d.n_text_layer, d.n_text_ctx
        f32 = dict(dtype=torch.float32, device=dev)
        with self.phase("encoder"):
            xa = self.encode([job])
        with self.phase("cross_kv"):
            self._cross_kv(xa, st8, 1)
            for li in range(L):                          # every hypothesis attends to the same audio
                for name in ("ck", "cv", "ckal"):
                    t = st8[name][li]
                    if G > 1 and t is not None:
                        t[1:G].copy_(t[0:1].expand(G - 1, *t.shape[1:]))
        del xa
        prompt = list(job["prompt"])
        P = len(prompt)
        self._park(ses)
        self._seed(ses, range(G), [prompt] * G)
        self._set_masks(ses, setup)
        # ---- prefill of hypothesis 0, then its self-attention cache is shared out
        with self.phase("prefill"):
            logits2, no_speech = self._prefill(ses, [prompt], [0], tok, qk_last=False)
            for li in range(L):
                for name in ("sk", "sv"):
                    t = st8[name][li]
                    if G > 1:
                        t[1:G, :, :P].copy_(t[0:1, :, :P].expand(G - 1, t.shape[1], P, t.shape[3]))
            ses["logits"][:G].copy_(logits2[0:1].expand(G, V))
            self.launches += 6
        # ---- upstream's main loop
        lp_dev = torch.empty((cap, V), **f32)
        seqs = [list(prompt) for _ in range(G)]
        sum_lp = torch.zeros(G, dtype=torch.float32)              # float32 arithmetic like upstream's tensor
        finished = {}                                              # beam search: sequence (tuple) -> cumulative log-prob
        max_candidates = round(beam * (setup.patience or 1.0)) if beam else 0
        with self.phase("decode_steps"):
            for i in range(setup.sample_len):
                nat.check(nat.lib.wts_filtered_logprobs(ses["logits"].data_ptr(), V, ctypes.byref(ses["cfg"]),
                                                        ses["suppress"].data_ptr(), ses["blank"].data_ptr(),
                                                        ses["tokens"].data_ptr(), ses["n_tokens"].data_ptr(),
                                                        ses["n_prompt"].data_ptr(), lp_dev.data_ptr(), G, st),
                          "wts_filtered_logprobs")
                self.launches += 1
                source = list(range(G))
                if beam:
                    vals, idxs = torch.topk(lp_dev[:G], beam + 1, dim=-1)
                    vals, idxs = vals.cpu(), idxs.cpu()
                    scores, sources = {}, {}
                    for j in range(G):
                        prefix = seqs[j]
                        for logprob, token in zip(vals[j], idxs[j]):
                            sequence = tuple(prefix + [int(token)])
                            scores[sequence] = (sum_lp[j] + logprob).item()
                            sources[sequence] = j
                    new_seqs, source, newly_finished = [], [], {}
                    for sequence in sorted(scores, key=scores.get, reverse=True):
                        if sequence[-1] == tok.eot:
                            newly_finished[sequence] = scores[sequence]
                        else:
                            sum_lp[len(new_seqs)] = scores[sequence]
                            new_seqs.append(list(sequence))
                            source.append(sources[sequence])
                            if len(new_seqs) == beam:
                                break
                    for seq in sorted(newly_finished, key=newly_finished.get, reverse=True):
                        if len(finished) >= max_candidates:
                            break
                        finished[seq] = newly_finished[seq]
                    seqs = new_seqs
                    completed = len(finished) >= max_candidates
                else:
                    lp = lp_dev[:G].cpu()
                    nxt = torch.distributions.Categorical(logits=lp / T).sample()
                    last = torch.tensor([s_[-1] for s_ in seqs])
                    sum_lp += lp[torch.arange(G), nxt] * (last != tok.eot)
                    nxt[last == tok.eot] = tok.eot
                    for s_, t_ in zip(seqs, nxt.tolist()):
                        s_.append(t_)
                    completed = bool((nxt == tok.eot).all())
                cur = len(seqs[0])
                if completed or cur > n_ctx:
                    break
                if i + 1 == setup.sample_len:
                    break
                # ---- device state follows the host: caches of the source hypotheses, new token rows, next logits
                if source != list(range(G)):
                    src = torch.as_tensor(source, dtype=torch.long, device=dev)
                    for li in range(L):
                        for name in ("sk", "sv"):
                            t = st8[name][li]
                            t[:G, :, :cur - 1] = t[src, :, :cur - 1]
                th = np.zeros((G, n_ctx + 1), dtype=np.int32)
                for r, s_ in enumerate(seqs):
                    th[r, :cur] = s_
                ses["tokens"][:G].copy_(torch.from_numpy(th))
                ses["n_tokens"][:G].fill_(cur)
                self._step_logits(ses)
        # ---- finalize + rank (upstream BeamSearchDecoder.finalize / GreedyDecoder.finalize, MaximumLikelihoodRanker)
        if beam:
            if len(finished) < beam:
                for j in list(np.argsort(sum_lp.numpy()))[::-1]:
                    finished[tuple(seqs[j] + [tok.eot])] = sum_lp[j].item()
                    if len(finished) >= beam:
                        break
            cands = [list(k) for k in finished.keys()]
            cand_lp = list(finished.values())
        else:
            cands = [s_ + [tok.eot] for s_ in seqs]
            cand_lp = sum_lp.tolist()
        cut = []
        for c in cands:
            body = c[P:]
            cut.append(body[:body.index(tok.eot)])
        lp_len = [len(c) for c in cut]
        if setup.length_penalty is None:
            score = [lp / n if n else (float("-inf") if lp < 0 else float("inf")) for lp, n in zip(cand_lp, lp_len)]
        else:
            score = [lp / (((5 + n) / 6) ** setup.length_penalty) for lp, n in zip(cand_lp, lp_len)]
        best = int(np.argmax(score))
        torch.cuda.synchronize(dev)
        return WindowRecord(seek=job["seek"], segment_size=job["segment_size"], prompt=prompt, tokens=cut[best], logprobs=None,
                            ended_by_eot=True, no_speech_prob=float(no_speech.cpu()[0]), qk_window=-1, temperature=T,
                            language=tok.language, sum_logprob=float(cand_lp[best]))

    # ------------------------------------------------------------------ teacher-forced pass (two-pass strategy)
    @torch.no_grad()
    def teacher_forced(self, mel, tokens_in, i_start, pairs):
        """Second pass of the two-pass strategy for ONE segment (T.py:1213-1249): encoder on the segment's own mel,
        decoder teacher-forced on `tokens_in` (sot sequence + <|0.00|> + text tokens).  The alignment heads' cross-
        attention rows from position i_start-1 on become a new alignment window; returns (window id, float32
        log_softmax(logits[step])[token] for every (step, token) in `pairs`)."""
        d, dev, st, w = self.dims, self.dev, self._st(), self.w
        tokens_in = [int(t) for t in tokens_in]
        R, D, V = len(tokens_in), d.n_text_state, d.n_vocab
        assert 0 < R <= d.n_text_ctx, f"{R} tokens do not fit the decoder context ({d.n_text_ctx})"
        size = min(N_FRAMES, int(mel.shape[0]))
        with self.phase("encoder"):
            xa = self.encode([dict(mel=mel, seek=0, segment_size=size)])
        st8 = getattr(self, "_tf_state", None)
        if st8 is None:
            st8 = self._tf_state = self._alloc_decoder_state(1, d.n_text_ctx)
        with self.phase("cross_kv"):
            self._cross_kv(xa, st8, 1)
        del xa
        rows = R - (i_start - 1)
        qk_buf = torch.zeros((1, len(self.heads), rows, N_CTX_AUDIO), dtype=torch.float32, device=dev)
        row_seq = _i32([0] * R, dev)
        row_pos = _i32(list(range(R)), dev)
        row_tok = _i32(tokens_in, dev)
        qk_row = _i32([p - (i_start - 1) if p >= i_start - 1 else -1 for p in range(R)], dev)
        x = torch.empty((R, D), dtype=torch.float32, device=dev)
        with self.phase("prefill"):
            nat.check(nat.lib.wts_embed(row_tok.data_ptr(), row_pos.data_ptr(), w.emb.data_ptr(), w.dec_pos.data_ptr(), R, D,
                                        x.data_ptr(), st), "wts_embed")
            self.launches += 1
            self._decoder_rows(st8, x, R, row_seq, row_pos, qk_row, qk_buf)
            vals = np.zeros(0, dtype=np.float32)
            if pairs:
                steps = sorted({int(s_) for (s_, _) in pairs})
                index = {s_: i for i, s_ in enumerate(steps)}
                sel = _i32(steps, dev)
                xr = torch.empty((len(steps), D), dtype=torch.float32, device=dev)
                nat.check(nat.lib.wts_gather_rows(x.data_ptr(), D, sel.data_ptr(), len(steps), D, xr.data_ptr(), st),
                          "wts_gather_rows")
                logits = torch.empty((len(steps), V), dtype=torch.float32, device=dev)
                self._final_logits(xr, len(steps), logits)
                d_rows = _i32([index[int(s_)] for (s_, _) in pairs], dev)
                d_tok = _i32([int(t_) for (_, t_) in pairs], dev)
                out = torch.empty(len(pairs), dtype=torch.float32, device=dev)
                nat.check(nat.lib.wts_logprob_gather(logits.data_ptr(), V, V, d_rows.data_ptr(), d_tok.data_ptr(),
                                                     out.data_ptr(), len(pairs), st), "wts_logprob_gather")
                self.launches += 2
                vals = out.cpu().numpy()
        return self._keep_rows(qk_buf), vals

    # ------------------------------------------------------------------ language detection
    def detect_language(self, mel, tokenizer):
        """Upstream detect_language on the first 30 s: logits at <|startoftranscript|>, softmax over the
        language tokens (T.py:862-867 exposes the same numbers as language_probs)."""
        return self.detect_languages([mel], tokenizer)[0]

    @torch.no_grad()
    def detect_languages(self, mels, tokenizer):
        """detect_language for many recordings: one encoder pass over their first windows (in batches of at most
        `max_batch`, fewer when that many windows would not fit in 85 % of the free device memory, as batch_limit
        sizes a decode batch), then one decoder row per recording at <|startoftranscript|>.  Returns [(language, probs)]."""
        d, dev, st, w = self.dims, self.dev, self._st(), self.w
        ids = list(tokenizer.all_language_tokens)
        torch.cuda.empty_cache()
        free, _ = torch.cuda.mem_get_info(dev)
        step = max(1, min(self.max_batch, int(0.85 * free) // self.window_bytes(1)))
        out = []
        for i in range(0, len(mels), step):
            part = mels[i:i + step]
            B = len(part)
            xa = self.encode([dict(mel=m, seek=0, segment_size=min(N_FRAMES, int(m.shape[0]))) for m in part])
            st8 = self._alloc_decoder_state(B, B)
            self._cross_kv(xa, st8, B)
            del xa
            qk_buf = torch.zeros((B, len(self.heads), 1, N_CTX_AUDIO), dtype=torch.float32, device=dev)
            x = torch.empty((B, d.n_text_state), dtype=torch.float32, device=dev)
            seq, pos = _i32(list(range(B)), dev), _i32([0] * B, dev)
            t = _i32([tokenizer.sot] * B, dev)
            nat.check(nat.lib.wts_embed(t.data_ptr(), pos.data_ptr(), w.emb.data_ptr(), w.dec_pos.data_ptr(), B,
                                        d.n_text_state, x.data_ptr(), st), "wts_embed")
            self._decoder_rows(st8, x, B, seq, pos, _i32([-1] * B, dev), qk_buf)
            logits = torch.empty((B, d.n_vocab), dtype=torch.float32, device=dev)
            self._final_logits(x, B, logits)
            self.launches += 1
            del st8
            for row in torch.softmax(logits[:, ids].cpu().float(), dim=-1).tolist():
                probs = dict(zip(tokenizer.all_language_codes, row))
                out.append((max(probs, key=probs.get), probs))
        return out

    # ------------------------------------------------------------------ alignment
    def align(self, items, disfluencies=False):
        """items: dicts(window=global window id, row0, last_row, T, f0, F, max_dur) -> list of jumps arrays; with
        disfluencies=True a second list: per token -1 or the start offset found by the peak analysis (T.py:1656-1683)."""
        out = [None] * len(items)
        lefts = [None] * len(items)
        groups = {}
        for i, it in enumerate(items):
            buf, b = self.window_index[it["window"]]
            groups.setdefault(buf, []).append((i, b, it))
        queued = []
        for buf, lst in groups.items():
            plan = plan_segments([(b, it["row0"], it["last_row"], it["T"], it["f0"], it["F"], it["max_dur"])
                                  for (_, b, it) in lst], nonpositive=True)
            qk = self.qk_buffers[buf]
            with self.phase("align_prep"):
                cost = attn_prep(qk, plan)
            with self.phase("align_dtw"):
                res = dtw(cost, plan)
            self.launches += 3
            dl = None
            if disfluencies:
                from .alignment import disfluency_starts
                dl = disfluency_starts(cost, plan, res["jumps"])
                self.launches += 1
            queued.append((lst, plan, res["jumps"], dl))
        for lst, plan, d_jumps, dl in queued:                # all launches are queued: the device->host copies come last
            jumps = split_jumps(d_jumps.cpu().numpy(), plan)
            for (i, _, _), j in zip(lst, jumps):
                out[i] = j
            if dl is not None:
                for (i, _, _), l_ in zip(lst, split_jumps(dl.cpu().numpy(), plan)):
                    lefts[i] = l_[:-1]
        return (out, lefts) if disfluencies else out

    def _keep_rows(self, rows):
        """Keeps the alignment rows [windows, heads, rows, 1500] of a decode batch, a collection or a teacher-forced
        segment as one buffer for align(); returns the window id of its first window (the others follow in order)."""
        buf, first = len(self.qk_buffers), len(self.window_index)
        self.qk_buffers.append(rows)
        for b in range(rows.shape[0]):
            self.window_index.append((buf, b))
        return first

    def free_alignment_rows(self, windows):
        """Drop the alignment rows of the decode batches holding these (already aligned) windows."""
        for gid in windows:
            if gid >= 0:
                self.qk_buffers[self.window_index[gid][0]] = None

    def release(self):
        self.qk_buffers.clear()
        self.window_index.clear()
        self.full_logprobs.clear()

"""Which GEMMs of the large-v3 forward need the 3-term split-bf16 product to keep logits / alignment `qk` within 1e-3?

CPU experiment on the oracle stand-in (float32 torch): every Linear / Conv of the chosen group is replaced by an
emulation of what the tensor cores compute — operands split into bf16 hi + lo planes, products accumulated in float32 —
with 3 terms (hi*hi + lo*hi + hi*lo: what gemm_tc_kernel does), 2 terms (activation low part dropped,
or weight low part dropped) or 1 term (plain bf16).  Reports max |delta| against the float32 forward of: encoder
output, teacher-forced decoder logits, pre-softmax cross-attention rows of the alignment heads.

    python tools/precision_scan.py [--model large-v3] [--seconds 30]

Test / design infrastructure: imports the oracle, never used by the product.  Results: DESIGN.md §4.
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle", "upstream"), os.path.join(ROOT, "whisper-timestamped_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def split(x):
    hi = x.to(torch.bfloat16).float()
    lo = (x - hi).to(torch.bfloat16).float()
    return hi, lo


def emu_matmul(a, w, mode):
    """a [.., K] x w[N, K]^T with split-bf16 operands, float32 accumulation (torch CPU matmul in float32)."""
    if mode == "f32":
        return a @ w.t()
    ah, al = split(a)
    wh, wl = split(w)
    y = ah @ wh.t()
    if mode in ("x3", "x2_keep_act_lo"):
        y = y + al @ wh.t()
    if mode in ("x3", "x2_keep_w_lo"):
        y = y + ah @ wl.t()
    return y


class Emu:
    def __init__(self):
        self.mode_of = {}          # module id -> mode

    def linear(self, mod, x):
        mode = self.mode_of.get(id(mod), "f32")
        y = emu_matmul(x, mod.weight, mode)
        return y if mod.bias is None else y + mod.bias


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--threads", type=int, default=8)
    args = ap.parse_args()
    torch.set_num_threads(args.threads)
    import whisper
    from whisper.model import disable_sdpa
    from whisper_timestamped import model_zoo as zoo
    from whisper_timestamped.synthetic_audio import synthetic_speech
    dims = zoo.DIMS[args.model]
    sd = zoo.synthetic_state_dict(dims, seed=1234, ts_offset=4.5, eot_logit=14.5)
    model = whisper.Whisper(whisper.ModelDimensions(**dims.asdict()))
    model.load_state_dict(sd)
    model.eval()
    heads = zoo.ALIGNMENT_HEADS[args.model]
    emu = Emu()
    # route every nn.Linear of the model through the emulation
    for mod in model.modules():
        if isinstance(mod, torch.nn.Linear):
            mod.forward = (lambda x, m=mod: emu.linear(m, x))
    groups = {
        "enc_mlp": [m for blk in model.encoder.blocks for m in (blk.mlp[0], blk.mlp[2])],
        "enc_attn_proj": [m for blk in model.encoder.blocks for m in (blk.attn.query, blk.attn.key, blk.attn.value, blk.attn.out)],
        "dec_cross_kv": [m for blk in model.decoder.blocks for m in (blk.cross_attn.key, blk.cross_attn.value)],
    }
    audio = torch.from_numpy(synthetic_speech(args.seconds, seed=1234))
    mel = whisper.pad_or_trim(whisper.log_mel_spectrogram(audio, dims.n_mels), 3000)[None]
    eot, sot, n_lang, ts0 = zoo.special_token_layout(dims.n_vocab)
    g = torch.Generator().manual_seed(3)
    text = torch.randint(300, 40000, (40,), generator=g).tolist()
    tokens = torch.tensor([[sot, sot + 1, sot + 1 + n_lang + 2, ts0] + text[:20] + [ts0 + 200, ts0 + 200] + text[20:] + [ts0 + 700]])

    def forward():
        captured = []
        hooks = [blk.cross_attn.register_forward_hook(lambda m, i, o: captured.append(o[-1])) for blk in model.decoder.blocks]
        with torch.no_grad(), disable_sdpa():
            xa = model.encoder(mel)
            logits = model.decoder(tokens, xa)
        for h in hooks:
            h.remove()
        qk = torch.stack([captured[l][0, h] for (l, h) in heads])
        return xa, logits, qk

    def run(label, setting):
        emu.mode_of = {}
        for gname, mode in setting.items():
            for m in groups[gname]:
                emu.mode_of[id(m)] = mode
        t0 = time.time()
        out = forward()
        return label, out, time.time() - t0

    _, ref, dt = run("f32", {})
    print(f"float32 forward: {dt:.0f} s; |xa| max {ref[0].abs().max():.2f}, |logits| max {ref[1].abs().max():.2f}, |qk| max {ref[2].abs().max():.2f}",
          flush=True)
    rows = []
    settings = [
        ("all three groups x3 (today)", {"enc_mlp": "x3", "enc_attn_proj": "x3", "dec_cross_kv": "x3"}),
        ("enc MLP x2 (activation lo kept)", {"enc_mlp": "x2_keep_act_lo", "enc_attn_proj": "x3", "dec_cross_kv": "x3"}),
        ("enc MLP x2 (weight lo kept)", {"enc_mlp": "x2_keep_w_lo", "enc_attn_proj": "x3", "dec_cross_kv": "x3"}),
        ("enc MLP bf16", {"enc_mlp": "bf16", "enc_attn_proj": "x3", "dec_cross_kv": "x3"}),
        ("enc MLP + attention projections x2 (activation lo kept)", {"enc_mlp": "x2_keep_act_lo", "enc_attn_proj": "x2_keep_act_lo", "dec_cross_kv": "x3"}),
        ("cross K/V projection x2 (activation lo kept)", {"enc_mlp": "x3", "enc_attn_proj": "x3", "dec_cross_kv": "x2_keep_act_lo"}),
    ]
    for label, setting in settings:
        _, out, dt = run(label, setting)
        row = {"setting": label, "d_encoder": float((out[0] - ref[0]).abs().max()), "d_logits": float((out[1] - ref[1]).abs().max()),
               "d_qk": float((out[2] - ref[2]).abs().max()), "seconds": round(dt)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"model": args.model, "rows": rows}))


if __name__ == "__main__":
    main()

"""One decoder step, kernel by kernel, against a float64 reference of the same step.

Both step implementations share one session state: the lean small-batch step (`wts_decode_step_kernels`, at most 32
active windows; MT = 1 below 17 rows, MT = 2 above) and the per-operator step (`CudaEngine._step`).  They run from one
seeded state on reduced-depth models (2 decoder layers) at every official width, and are compared with a float64 step
built from exactly what the kernels read: the SB16 weight planes, the float32 self-attention caches, fp16 cross K/V
(float32 K for the alignment heads).  The reference itself is pinned to upstream's `TextDecoder` on the CPU.

The remaining per-operator decode kernels (decoder attention kinds 0 and 2, KV append, LayerNorm, softmax pick,
log-prob gather, embed, row gather, step inputs) are compared directly at D = 384 and 1280.

Observed maxima on an NVIDIA H100 80GB HBM3 are noted next to each bound (TOL)."""
import ctypes
import gc
import math

import numpy as np
import pytest
import torch

from whisper_timestamped import model_zoo as zoo

import oracle_engine  # noqa: F401  (puts oracle/upstream on sys.path: `whisper` below is the oracle stand-in)
from test_gpu_decode_select import upstream_filtered

N_CTX, N_AUDIO = 448, 1500

# name: (D, H, n_vocab, n_mels, alignment heads of the 2 decoder layers).  Every width has one layer with a single
# head other than 0 and one with several heads including the last; `small` has a layer without alignment heads, and
# `medium` puts the several-head layer first (its single-head layer starts at slot 3).
WIDTHS = {
    "tiny": (384, 6, 51865, 80, [(0, 4), (1, 0), (1, 3), (1, 5)]),
    "base": (512, 8, 51865, 80, [(0, 1), (1, 2), (1, 6), (1, 7)]),
    "small": (768, 12, 51865, 80, [(1, 0), (1, 5), (1, 11)]),
    "medium": (1024, 16, 51865, 80, [(0, 0), (0, 7), (0, 15), (1, 11)]),
    "large-v3": (1280, 20, 51866, 128, [(0, 7), (1, 0), (1, 13), (1, 19)]),
}

# Bounds per width and quantity: max abs error against the float64 reference of the logits, the appended self K/V,
# the alignment rows (qk_buf) and the chosen token's log-probability, the same for both step paths.  Each is about 4x
# the largest error observed over every row count, cap and path (test_step_matches_float64_reference, and for
# large-v3 also test_consecutive_steps_match_float64_reference; `pytest -s` prints them) on an NVIDIA H100 80GB HBM3
# at 700 W:
#   tiny      logits 3.55e-4  kv 5.2e-5  qk 1.55e-4  logprob 8.0e-5
#   base      logits 3.73e-4  kv 6.4e-5  qk 1.57e-4  logprob 1.26e-4
#   small     logits 3.66e-4  kv 5.5e-5  qk 1.27e-4  logprob 9.4e-5
#   medium    logits 4.33e-4  kv 5.0e-5  qk 1.28e-4  logprob 1.00e-4
#   large-v3  logits 5.59e-4  kv 5.6e-5  qk 1.45e-4  logprob 1.18e-4
TOL = {
    "tiny": dict(logits=1.4e-3, kv=2.0e-4, qk=6.0e-4, logprob=3.2e-4),
    "base": dict(logits=1.5e-3, kv=2.5e-4, qk=6.0e-4, logprob=5.0e-4),
    "small": dict(logits=1.5e-3, kv=2.2e-4, qk=5.0e-4, logprob=3.8e-4),
    "medium": dict(logits=1.7e-3, kv=2.0e-4, qk=5.0e-4, logprob=4.0e-4),
    "large-v3": dict(logits=2.2e-3, kv=2.2e-4, qk=5.8e-4, logprob=4.7e-4),
}


def _dims(name):
    D, H, V, M, _ = WIDTHS[name]
    return zoo.ModelDimensions(n_mels=M, n_audio_ctx=N_AUDIO, n_audio_state=D, n_audio_head=H, n_audio_layer=1,
                               n_vocab=V, n_text_ctx=N_CTX, n_text_state=D, n_text_head=H, n_text_layer=2)


# ---------------------------------------------------------------------------------------------- float64 reference
def _ln(x, g, b):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-5) * g + b


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def ref_weights_from_model(m):
    """float64 weights exactly as the kernels read them: SB16 planes recombined (q/k scale already folded in)."""
    w = m.w

    def f(sb):
        return sb.to_f32().double()

    def v(t):
        return t.double()
    layers = []
    for blk in w.dec:
        a, c = blk.attn, blk.cross
        layers.append(dict(ln1=(v(a.ln_g), v(a.ln_b)), wqkv=f(a.qkv), bqkv=v(a.qkv_b), wo=f(a.out), bo=v(a.out_b),
                           ln2=(v(c.ln_g), v(c.ln_b)), wq=f(c.q), bq=v(c.q_b), wco=f(c.out), bco=v(c.out_b),
                           ln3=(v(blk.mlp_ln_g), v(blk.mlp_ln_b)), w1=f(blk.fc1), b1=v(blk.fc1_b), w2=f(blk.fc2),
                           b2=v(blk.fc2_b)))
    return dict(layers=layers, emb=v(w.emb), emb_out=f(w.emb_sb), pos=v(w.dec_pos), ln=(v(w.ln_g), v(w.ln_b)))


def ref_weights_from_state_dict(sd, dims):
    """The same weights from an openai-whisper state dict (float64, the d_head^-1/4 scale folded into q and k)."""
    s = (dims.n_text_state // dims.n_text_head) ** -0.25

    def g(k):
        return sd[k].double()
    layers = []
    for i in range(dims.n_text_layer):
        p = f"decoder.blocks.{i}."
        layers.append(dict(
            ln1=(g(p + "attn_ln.weight"), g(p + "attn_ln.bias")),
            wqkv=torch.cat([g(p + "attn.query.weight") * s, g(p + "attn.key.weight") * s, g(p + "attn.value.weight")]),
            bqkv=torch.cat([g(p + "attn.query.bias") * s, torch.zeros_like(g(p + "attn.query.bias")),
                            g(p + "attn.value.bias")]),
            wo=g(p + "attn.out.weight"), bo=g(p + "attn.out.bias"),
            ln2=(g(p + "cross_attn_ln.weight"), g(p + "cross_attn_ln.bias")),
            wq=g(p + "cross_attn.query.weight") * s, bq=g(p + "cross_attn.query.bias") * s,
            wco=g(p + "cross_attn.out.weight"), bco=g(p + "cross_attn.out.bias"),
            ln3=(g(p + "mlp_ln.weight"), g(p + "mlp_ln.bias")),
            w1=g(p + "mlp.0.weight"), b1=g(p + "mlp.0.bias"), w2=g(p + "mlp.2.weight"), b2=g(p + "mlp.2.bias")))
    emb = g("decoder.token_embedding.weight")
    return dict(layers=layers, emb=emb, emb_out=emb, pos=g("decoder.positional_embedding"),
                ln=(g("decoder.ln.weight"), g("decoder.ln.bias")))


def ref_step(W, H, tok, pos, self_k, self_v, cross_k, cross_v):
    """One decoder step of R rows in float64.  tok/pos: [R] ints; self_k/self_v[l]: [R, H, >= max(pos), 64] (positions
    < pos[r] are read); cross_k/cross_v[l]: [R, H, 1500, 64].  Returns (logits [R, V], appended K and V per layer
    [R, H, 64], pre-softmax cross-attention rows per layer [R, H, 1500])."""
    R = len(tok)
    x = W["emb"][torch.as_tensor(tok)] + W["pos"][torch.as_tensor(pos)]
    D = x.shape[1]
    k_new, v_new, qk = [], [], []
    for li, L in enumerate(W["layers"]):
        qkv = _ln(x, *L["ln1"]) @ L["wqkv"].T + L["bqkv"]
        q, k, v = (t.reshape(R, H, 64) for t in qkv.split(D, -1))
        att = torch.empty_like(q)
        for r in range(R):
            p = int(pos[r])
            K = torch.cat([self_k[li][r, :, :p], k[r, :, None]], 1)
            V = torch.cat([self_v[li][r, :, :p], v[r, :, None]], 1)
            att[r] = torch.einsum("hj,hjc->hc", torch.softmax(torch.einsum("hc,hjc->hj", q[r], K), -1), V)
        x = x + att.reshape(R, D) @ L["wo"].T + L["bo"]
        q = (_ln(x, *L["ln2"]) @ L["wq"].T + L["bq"]).reshape(R, H, 64)
        s = torch.einsum("rhc,rhjc->rhj", q, cross_k[li])
        y = torch.einsum("rhj,rhjc->rhc", torch.softmax(s, -1), cross_v[li]).reshape(R, D)
        x = x + y @ L["wco"].T + L["bco"]
        x = x + _gelu(_ln(x, *L["ln3"]) @ L["w1"].T + L["b1"]) @ L["w2"].T + L["b2"]
        k_new.append(k)
        v_new.append(v)
        qk.append(s)
    return _ln(x, *W["ln"]) @ W["emb_out"].T, k_new, v_new, qk


def test_reference_step_matches_upstream_decoder(monkeypatch):
    """CPU: the hand-written float64 step, fed token by token with its own K/V, reproduces upstream's TextDecoder (run
    in float64 from the same state dict on the whole prefix, cross K/V from the same encoder output): the logits of
    every position and the pre-softmax cross-attention rows of every head."""
    from whisper.model import LayerNorm, TextDecoder, disable_sdpa
    monkeypatch.setattr(LayerNorm, "forward", torch.nn.LayerNorm.forward)     # float64 LayerNorm (upstream: float32)
    dims = _dims("tiny")
    D, H, L = dims.n_text_state, dims.n_text_head, dims.n_text_layer
    sd = zoo.synthetic_state_dict(dims, seed=7)
    dec = TextDecoder(dims.n_vocab, N_CTX, D, H, L)
    dec.load_state_dict({k[len("decoder."):]: v for k, v in sd.items() if k.startswith("decoder.")})
    dec = dec.double()
    g = torch.Generator().manual_seed(3)
    xa = torch.randn((1, N_AUDIO, D), generator=g, dtype=torch.float64)
    tokens = [50258, 50259, 50359, 50364, 1000, 2345, 50380, 777]
    rows = []
    hooks = [b.cross_attn.register_forward_hook(lambda mod, i, o: rows.append(o[1])) for b in dec.blocks]
    with torch.no_grad(), disable_sdpa():
        want = dec(torch.tensor([tokens]), xa)[0]
    for h in hooks:
        h.remove()
    W = ref_weights_from_state_dict(sd, dims)
    s = (D // H) ** -0.25
    ck = [(xa[0] @ (sd[f"decoder.blocks.{i}.cross_attn.key.weight"].double() * s).T).reshape(N_AUDIO, H, 64)
          .permute(1, 0, 2)[None] for i in range(L)]
    cv = [(xa[0] @ sd[f"decoder.blocks.{i}.cross_attn.value.weight"].double().T
           + sd[f"decoder.blocks.{i}.cross_attn.value.bias"].double()).reshape(N_AUDIO, H, 64).permute(1, 0, 2)[None]
          for i in range(L)]
    sk = [torch.zeros((1, H, N_CTX, 64), dtype=torch.float64) for _ in range(L)]
    sv = [torch.zeros((1, H, N_CTX, 64), dtype=torch.float64) for _ in range(L)]
    for p, t in enumerate(tokens):
        logits, kn, vn, qk = ref_step(W, H, [t], [p], sk, sv, ck, cv)
        for li in range(L):
            sk[li][:, :, p], sv[li][:, :, p] = kn[li], vn[li]
            # upstream computes these rows in float32 (qk.float())
            assert float((qk[li][0] - rows[li][0, :, p]).abs().max()) <= 1e-4, (p, li)
        assert float((logits[0] - want[p]).abs().max()) <= 1e-4, p


# ------------------------------------------------------------------------------------------- models and sessions
_MODELS, _SESSIONS = {}, {}


def _release():
    """Drop the cached models and sessions (an engine and its model reference each other: collect the cycle)."""
    _MODELS.clear()
    _SESSIONS.clear()
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


def _model(name):
    """(model, float64 weights from its SB16 planes, float64 weights from its state dict); one width is cached at a
    time (the tests run width by width)."""
    if name not in _MODELS:
        _release()
        from whisper_timestamped.model import WhisperB200
        dims = _dims(name)
        sd = zoo.synthetic_state_dict(dims, seed=17)
        m = WhisperB200(dims, sd, "cuda", name=name, alignment_heads=WIDTHS[name][4])
        _MODELS[name] = (m, ref_weights_from_model(m), ref_weights_from_state_dict(sd, dims))
    return _MODELS[name]


def _session(name, cap):
    """(engine, session, setup) of a decode session with exactly `cap` slots (one engine per width and cap)."""
    key = (name, cap)
    if key not in _SESSIONS:
        from whisper_timestamped.engine import CudaEngine
        from whisper_timestamped.tokenizer import get_tokenizer
        from whisper_timestamped.windows import make_decode_setup
        m = _model(name)[0]
        eng = CudaEngine(m, max_batch=cap, small_batch_rows=32)
        tok = get_tokenizer(m.is_multilingual, num_languages=m.num_languages, language="en", task="transcribe")
        setup = make_decode_setup(tok, N_CTX)
        ses = eng._decoder_session(setup, cap)
        assert ses["cap"] == cap and ses["steps"] is not None
        eng._set_masks(ses, setup)
        _SESSIONS[key] = (eng, ses, setup)
    return _SESSIONS[key]


def _lean_rows(n_active):
    return 4 if n_active <= 4 else 8 if n_active <= 8 else 16 if n_active <= 16 else 32


def _run_lean(eng, ses, max_rows):
    from whisper_timestamped import _native as nat
    sd = ses["steps"]
    p = sd["args"]
    p.max_rows = max_rows
    nat.check(nat.lib.wts_decode_step_kernels(ctypes.byref(p), ctypes.byref(sd["host_layers"]), eng._st()),
              "wts_decode_step_kernels")
    torch.cuda.synchronize()


def _state_keys(eng):
    L = eng.dims.n_text_layer
    return [("tokens",), ("n_tokens",), ("n_prompt",), ("done",), ("logprobs",), ("qk_buf",)] + \
        [("st8", n, li) for n in ("sk", "sv") for li in range(L)]


def _get(ses, key):
    t = ses
    for k in key:
        t = t[k]
    return t


def _snapshot(eng, ses):
    return {k: _get(ses, k).clone() for k in _state_keys(eng)}


def _restore(ses, snap):
    for k, v in snap.items():
        _get(ses, k).copy_(v)
    torch.cuda.synchronize()


def _seed(eng, ses, setup, slots, seed, kinds=None):
    """Random caches, cross K/V, float32 alignment K, token histories; `slots` active, every other slot finished
    (done 1 or 2).  Row kinds (cycled unless given): 0 first sampled position (n_tokens == n_prompt); 1 a window
    carrying a 40-token prompt; 2 a prompt-carrying window at position n_ctx - 1 = 447."""
    d = eng.dims
    tok = setup.tokenizer
    L, cap = d.n_text_layer, ses["cap"]
    g = torch.Generator(device="cuda").manual_seed(seed)
    rng = np.random.default_rng(seed)
    st8 = ses["st8"]
    for li in range(L):
        for n in ("ck", "cv"):
            t = st8[n][li]
            t.copy_((torch.randn(t.shape, device="cuda", generator=g) * 0.5).to(t.dtype))
        for n in ("sk", "sv"):
            st8[n][li].normal_(0, 0.5, generator=g)
        if st8["ckal"][li] is not None:
            st8["ckal"][li].normal_(0, 0.5, generator=g)
    ses["qk_buf"].normal_(0, 1, generator=g)
    ses["logprobs"].normal_(0, 1, generator=g)
    sot = list(tok.sot_sequence)
    tsb = tok.timestamp_begin
    tokens = np.zeros((cap, N_CTX + 1), dtype=np.int32)
    n_tok = np.zeros(cap, dtype=np.int32)
    n_pr = np.zeros(cap, dtype=np.int32)
    done = 1 + (np.arange(cap) % 2).astype(np.int32)

    def history(n):
        out, ts = [], tsb
        for _ in range(n):
            if rng.random() < 0.15:
                ts = min(ts + int(rng.integers(0, 30)), tsb + 1500)
                out.append(ts)
            else:
                out.append(int(rng.integers(300, 30000)))
        return out
    rank = {b: r for r, b in enumerate(slots)}
    kinds = kinds or [0, 1, 2]
    for i in range(cap):
        kind = kinds[rank.get(i, i) % len(kinds)]
        if kind == 0:
            prompt, n = sot, 0
        elif kind == 1:
            prompt, n = [tok.sot_prev] + history(40) + sot, int(rng.integers(1, 60))
        else:
            prompt = [tok.sot_prev] + [int(t) for t in rng.integers(300, 30000, 222)] + sot
            n = N_CTX - len(prompt)
        row = prompt + history(n)
        tokens[i, :len(row)] = row
        n_tok[i], n_pr[i] = len(row), len(prompt)
    done[list(slots)] = 0
    ses["tokens"].copy_(torch.from_numpy(tokens))
    ses["n_tokens"].copy_(torch.from_numpy(n_tok))
    ses["n_prompt"].copy_(torch.from_numpy(n_pr))
    ses["done"].copy_(torch.from_numpy(done))
    torch.cuda.synchronize()


def _ref_inputs(eng, ses, slots):
    """float64 copies of what the step of `slots` reads (cross K of the alignment heads from the float32 copy)."""
    st8 = ses["st8"]
    idx = torch.as_tensor(slots, device="cuda")
    sk = [st8["sk"][li][idx].double() for li in range(eng.dims.n_text_layer)]
    sv = [st8["sv"][li][idx].double() for li in range(eng.dims.n_text_layer)]
    ck, cv = [], []
    for li in range(eng.dims.n_text_layer):
        k = st8["ck"][li][idx].double()
        s0, n_l = eng.layer_slots[li]
        for h in range(eng.dims.n_text_head):
            s = int(eng.head_slot[li, h])
            if s >= 0:
                k[:, h] = st8["ckal"][li][idx, s - s0].double()
        ck.append(k)
        cv.append(st8["cv"][li][idx].double())
    return sk, sv, ck, cv


def _select_ref(snap, setup, logits, slot, tol):
    """Upstream's choice from the float64 logits of one slot (token state of the snapshot before the step), its filtered
    log-softmax row, and whether the choice is clear of the error bound: a top-2 gap above 4 x TOL, and the same
    choice with every timestamp logit moved by +-4 x TOL (the timestamp-mass switch is not a near tie)."""
    tok = setup.tokenizer
    nt, n_prompt = int(snap[("n_tokens",)][slot]), int(snap[("n_prompt",)][slot])
    args = (snap[("tokens",)][slot, :nt].tolist(), n_prompt, tok, list(setup.suppress_tokens),
            setup.max_initial_timestamp_index)
    raw = logits.cpu()
    filt = upstream_filtered(raw, *args)
    choice = int(filt.argmax())
    top = torch.topk(filt, 2).values
    clear = float(top[0] - top[1]) > 4 * tol
    for sign in (1.0, -1.0):
        shifted = raw.clone()
        shifted[tok.timestamp_begin:] += sign * 4 * tol
        clear = clear and int(upstream_filtered(shifted, *args).argmax()) == choice
    return choice, torch.log_softmax(filt, -1), clear


def _check_step(eng, ses, setup, slots, snap, ref, errs, path, choices):
    """Compare the state after one step of `path` with the float64 reference `ref` for the active `slots`, and the
    finished slots with the snapshot taken before the step."""
    logits_ref, k_new, v_new, qk_ref = ref
    tol = TOL[eng.m.name]
    d = eng.dims
    H = d.n_text_head
    idx = torch.as_tensor(slots, device="cuda")
    n_tok0 = snap[("n_tokens",)][idx].cpu()
    n_pr = snap[("n_prompt",)][idx].cpu()
    got = ses["logits"][idx].double()
    e = float((got - logits_ref).abs().max())
    errs["logits"] = max(errs.get("logits", 0.0), e)
    assert e <= tol["logits"], (path, "logits", e)
    for li in range(d.n_text_layer):
        pos = (n_tok0 - 1).long().cuda()
        for n, want in (("sk", k_new[li]), ("sv", v_new[li])):
            c = ses["st8"][n][li][idx, :, pos]          # [R, H, 64]
            e = float((c.double() - want).abs().max())
            errs["kv"] = max(errs.get("kv", 0.0), e)
            assert e <= tol["kv"], (path, n, li, e)
        for h in range(H):
            s = int(eng.head_slot[li, h])
            if s < 0:
                continue
            rows = ses["qk_buf"][idx, s, (n_tok0 - n_pr).long().cuda()]    # [R, 1500]
            e = float((rows.double() - qk_ref[li][:, h]).abs().max())
            errs["qk"] = max(errs.get("qk", 0.0), e)
            assert e <= tol["qk"], (path, "qk", li, h, e)
    # the choice, the token state and the log-probability of each active row
    for r, b in enumerate(slots):
        if b not in choices:                                 # one reference choice per slot and state
            choices[b] = _select_ref(snap, setup, logits_ref[r], b, tol["logits"])
        choice, lp, clear = choices[b]
        nt = int(n_tok0[r])
        n = nt - int(n_pr[r])
        done = int(ses["done"][b])
        picked = setup.tokenizer.eot if done == 1 else int(ses["tokens"][b, nt])
        if clear:
            assert picked == choice, (path, b, picked, choice)
        if done == 1:
            assert int(ses["n_tokens"][b]) == nt
        else:
            assert int(ses["n_tokens"][b]) == nt + 1
            assert done == (2 if (n + 1 >= setup.sample_len or nt + 1 > N_CTX) else 0), (path, b, done)
        if math.isfinite(float(lp[picked])):
            e = abs(float(ses["logprobs"][b, n]) - float(lp[picked]))
            errs["logprob"] = max(errs.get("logprob", 0.0), e)
            if clear:
                assert e <= tol["logprob"], (path, b, e)
    # finished slots: untouched, bit for bit
    others = torch.as_tensor([b for b in range(ses["cap"]) if b not in set(slots)], dtype=torch.long, device="cuda")
    if len(others):
        for k, v in snap.items():
            t = _get(ses, k)
            assert torch.equal(t[others], v[others]), (path, "finished slot changed", k)


def _spread_slots(n_active, cap, rng):
    """Active slots spread over the session, with some above slot 31 when the session has more than 32 slots."""
    if cap <= 32:
        return sorted(rng.choice(cap, n_active, replace=False).tolist())
    hi = max(1, n_active // 2)
    lo = n_active - hi
    return sorted(rng.choice(32, lo, replace=False).tolist() + (32 + rng.choice(cap - 32, hi, replace=False)).tolist())


def _ref_for(eng, ses, slots, W):
    sk, sv, ck, cv = _ref_inputs(eng, ses, slots)
    nt = ses["n_tokens"][torch.as_tensor(slots, device="cuda")].cpu()
    tok = [int(ses["tokens"][b, int(nt[r]) - 1]) for r, b in enumerate(slots)]
    pos = [int(x) - 1 for x in nt]
    return ref_step(W, eng.dims.n_text_head, tok, pos, sk, sv, ck, cv)


@pytest.mark.gpu
def test_reference_weights_are_the_model_weights():
    """The weights the step reference reads (SB16 planes recombined) are the state dict's, with the scale folded in
    as the reference's own CPU pin assumes."""
    m, Wm, Ws = _model("tiny")
    for a, b in zip(Wm["layers"], Ws["layers"]):
        for k in a:
            x, y = (a[k], b[k]) if not isinstance(a[k], tuple) else (torch.stack(a[k]), torch.stack(b[k]))
            assert float((x.cpu() - y).abs().max()) <= 1e-5 * max(1.0, float(y.abs().max())), k
    assert float((Wm["emb_out"].cpu() - Ws["emb"]).abs().max()) <= 1e-5 * float(Ws["emb"].abs().max())


@pytest.mark.gpu
@pytest.mark.parametrize("cap", ["fit", 64])
@pytest.mark.parametrize("n_active", [1, 4, 5, 9, 16, 17, 32])
@pytest.mark.parametrize("name", list(WIDTHS))
def test_step_matches_float64_reference(name, n_active, cap):
    """Lean step (grid bound = the smallest of 4/8/16/32 rows that fits, as the engine picks it) and per-operator
    step from one state: logits, appended self K/V, alignment rows, the choice and the token state of the active rows
    against the float64 step; finished slots unchanged bit for bit.  With at most 4 active rows, the lean step's row
    bound (4, 8, 16, 32: MT = 1 and MT = 2) does not change a bit of the logits."""
    cap = _lean_rows(n_active) if cap == "fit" else cap
    eng, ses, setup = _session(name, cap)
    W = _model(name)[1]
    rng = np.random.default_rng(1000 * n_active + cap)
    slots = _spread_slots(n_active, cap, rng)
    _seed(eng, ses, setup, slots, seed=n_active * 7 + cap)
    snap = _snapshot(eng, ses)
    ref = _ref_for(eng, ses, slots, W)
    errs = {}
    _run_lean(eng, ses, _lean_rows(n_active))
    choices = {}
    _check_step(eng, ses, setup, slots, snap, ref, errs, "lean", choices)
    lean_logits = ses["logits"][torch.as_tensor(slots, device="cuda")].clone()
    _restore(ses, snap)
    eng._step(ses)
    torch.cuda.synchronize()
    _check_step(eng, ses, setup, slots, snap, ref, errs, "per-operator", choices)
    if n_active <= 4:
        for rows in (8, 16, 32):
            _restore(ses, snap)
            _run_lean(eng, ses, rows)
            assert torch.equal(ses["logits"][torch.as_tensor(slots, device="cuda")], lean_logits), rows
    _restore(ses, snap)
    print(f"\nERR {name} n_active={n_active} cap={cap} " + " ".join(f"{k}={v:.3e}" for k, v in sorted(errs.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("n_active", [5, 17])
def test_consecutive_steps_match_float64_reference(n_active):
    """Three lean steps, then three per-operator steps, from one state at large-v3 width: after every step the state
    (appended K/V read back by the next step, the advancing alignment row, n_tokens, done) matches the float64 step
    teacher-forced on the tokens the kernels chose."""
    name = "large-v3"
    eng, ses, setup = _session(name, 64)
    W = _model(name)[1]
    rng = np.random.default_rng(n_active)
    slots = _spread_slots(n_active, 64, rng)
    _seed(eng, ses, setup, slots, seed=5 + n_active, kinds=[0, 1])
    start = _snapshot(eng, ses)
    errs = {}
    for path in ("lean", "per-operator"):
        _restore(ses, start)
        sk, sv, ck, cv = _ref_inputs(eng, ses, slots)
        active = list(slots)
        for step in range(3):
            if not active:
                break
            snap = _snapshot(eng, ses)
            r_idx = [slots.index(b) for b in active]
            nt = [int(ses["n_tokens"][b]) for b in active]
            tok = [int(ses["tokens"][b, n - 1]) for b, n in zip(active, nt)]
            pos = [n - 1 for n in nt]
            ref = ref_step(W, eng.dims.n_text_head, tok, pos, [t[r_idx] for t in sk], [t[r_idx] for t in sv],
                           [t[r_idx] for t in ck], [t[r_idx] for t in cv])
            if path == "lean":
                _run_lean(eng, ses, _lean_rows(len(active)))
            else:
                eng._step(ses)
                torch.cuda.synchronize()
            _check_step(eng, ses, setup, active, snap, ref, errs, f"{path} step {step}", {})
            for li in range(eng.dims.n_text_layer):           # the reference keeps its own float64 K/V
                for j, (r, p) in enumerate(zip(r_idx, pos)):
                    sk[li][r, :, p], sv[li][r, :, p] = ref[1][li][j], ref[2][li][j]
            active = [b for b in active if int(ses["done"][b]) == 0]
    _restore(ses, start)
    print(f"\nERR consecutive n_active={n_active} " + " ".join(f"{k}={v:.3e}" for k, v in sorted(errs.items())))


# ------------------------------------------------------------------------------ the other per-operator decode kernels
def _sb(rows, cols):
    from whisper_timestamped.model import SB16
    return SB16(rows, cols, "cuda")


def _attn_ref(q, K, V):
    """q [H, 64], K/V [H, n, 64] float64 -> [H, 64]."""
    return torch.einsum("hj,hjc->hc", torch.softmax(torch.einsum("hc,hjc->hj", q, K), -1), V)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 1280])
def test_decoder_attention_prefill_after_kv_append(D):
    """kind 0 over a ragged prefill (prompts of 1, 3 and 221 rows in one call) after wts_kv_append: the cache holds
    every row's K/V exactly, the causal attention matches float64."""
    from whisper_timestamped import _native as nat
    H = D // 64
    g = torch.Generator(device="cuda").manual_seed(D)
    lens, seqs = [1, 3, 221], [2, 0, 3]
    R = sum(lens)
    row_seq = torch.tensor([s for s, n in zip(seqs, lens) for _ in range(n)], dtype=torch.int32, device="cuda")
    row_pos = torch.tensor([i for n in lens for i in range(n)], dtype=torch.int32, device="cuda")
    qkv = torch.randn((R, 3 * D), device="cuda", generator=g) * 0.7
    kc = torch.full((4, H, N_CTX, 64), 9.0, device="cuda")
    vc = torch.full((4, H, N_CTX, 64), 9.0, device="cuda")
    st = nat.stream_ptr("cuda")
    nat.check(nat.lib.wts_kv_append(qkv.data_ptr() + 4 * D, qkv.data_ptr() + 8 * D, 3 * D, row_seq.data_ptr(),
                                    row_pos.data_ptr(), R, H, N_CTX, kc.data_ptr(), vc.data_ptr(), H * N_CTX * 64, st),
              "wts_kv_append")
    out = _sb(R, D)
    nat.check(nat.lib.wts_decoder_attention(0, qkv.data_ptr(), 3 * D, kc.data_ptr(), vc.data_ptr(), H * N_CTX * 64, N_CTX,
                                            row_seq.data_ptr(), row_pos.data_ptr(), R, H, out.ptr, out.ld, out.plane,
                                            None, None, 0, 0, None, None, st), "wts_decoder_attention")
    torch.cuda.synchronize()
    q, k, v = (t.reshape(R, H, 64) for t in qkv.split(D, -1))
    r0 = 0
    err = 0.0
    for s, n in zip(seqs, lens):
        assert torch.equal(kc[s, :, :n], k[r0:r0 + n].permute(1, 0, 2))
        assert torch.equal(vc[s, :, :n], v[r0:r0 + n].permute(1, 0, 2))
        assert bool((kc[s, :, n:] == 9.0).all())
        K, V = k[r0:r0 + n].permute(1, 0, 2).double(), v[r0:r0 + n].permute(1, 0, 2).double()
        for i in range(n):
            want = _attn_ref(q[r0 + i].double(), K[:, :i + 1], V[:, :i + 1]).reshape(D)
            err = max(err, float((out.to_f32()[r0 + i].double() - want).abs().max()))
        r0 += n
    assert bool((kc[1] == 9.0).all())
    assert err <= 4e-5, err                                  # observed 1.52e-5 (H100)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 1280])
def test_decoder_attention_fused_append_with_holes(D):
    """kind 2 (one row per sequence, the kernel appends K/V first) with inactive rows: active rows append and attend
    over positions 0..pos, inactive rows touch neither the cache nor their output."""
    from whisper_timestamped import _native as nat
    H = D // 64
    B = 12
    g = torch.Generator(device="cuda").manual_seed(D + 1)
    pos = torch.tensor([0, 5, 447, 100, 31, 32, 1, 300, 64, 446, 2, 200], dtype=torch.int32, device="cuda")
    active = torch.tensor([1, 1, 1, 0, 1, 0, 1, 1, 0, 1, 1, 0], dtype=torch.int32, device="cuda")
    seq = torch.arange(B, dtype=torch.int32, device="cuda")
    qkv = torch.randn((B, 3 * D), device="cuda", generator=g) * 0.7
    kc = torch.randn((B, H, N_CTX, 64), device="cuda", generator=g) * 0.5
    vc = torch.randn((B, H, N_CTX, 64), device="cuda", generator=g)
    kc0, vc0 = kc.clone(), vc.clone()
    out = _sb(B, D)
    out.t.fill_(3.0)
    nat.check(nat.lib.wts_decoder_attention(2, qkv.data_ptr(), 3 * D, kc.data_ptr(), vc.data_ptr(), H * N_CTX * 64, N_CTX,
                                            seq.data_ptr(), pos.data_ptr(), B, H, out.ptr, out.ld, out.plane, None, None,
                                            0, 0, None, active.data_ptr(), nat.stream_ptr("cuda")), "wts_decoder_attention")
    torch.cuda.synchronize()
    q, k, v = (t.reshape(B, H, 64) for t in qkv.split(D, -1))
    y = out.to_f32()
    err = 0.0
    for b in range(B):
        p = int(pos[b])
        if not int(active[b]):
            assert torch.equal(kc[b], kc0[b]) and torch.equal(vc[b], vc0[b]) and bool((out.t[:, b] == 3.0).all())
            continue
        assert torch.equal(kc[b, :, p], k[b]) and torch.equal(vc[b, :, p], v[b])
        mask = torch.ones(N_CTX, dtype=torch.bool, device="cuda")
        mask[p] = False
        assert torch.equal(kc[b][:, mask], kc0[b][:, mask]) and torch.equal(vc[b][:, mask], vc0[b][:, mask])
        want = _attn_ref(q[b].double(), kc[b, :, :p + 1].double(), vc[b, :, :p + 1].double()).reshape(D)
        err = max(err, float((y[b].double() - want).abs().max()))
    assert err <= 4e-5, err                                  # observed 1.48e-5 (H100)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 1280])
def test_layernorm_pitch_and_large_mean(D):
    """SB16 and float32 outputs at a row pitch ldx > D, on rows with a large mean, against float64."""
    from whisper_timestamped import _native as nat
    M, ldx = 7, D + 36
    g = torch.Generator(device="cuda").manual_seed(D + 2)
    x = torch.randn((M, ldx), device="cuda", generator=g)
    x[:, D:] = float("nan")                                   # the pitch padding must not be read
    x[1, :D] += 1000.0
    x[4, :D] = x[4, :D] * 0.5 - 300.0
    x[6, :D] *= 50.0
    gam = 1.0 + 0.1 * torch.randn(D, device="cuda", generator=g)
    bet = 0.1 * torch.randn(D, device="cuda", generator=g)
    sb = _sb(M, D)
    f = torch.full((M, D + 8), 5.0, device="cuda")
    nat.check(nat.lib.wts_layernorm(x.data_ptr(), ldx, gam.data_ptr(), bet.data_ptr(), M, D, sb.ptr, sb.ld, sb.plane,
                                    f.data_ptr(), D + 8, nat.stream_ptr("cuda")), "wts_layernorm")
    torch.cuda.synchronize()
    want = _ln(x[:, :D].double(), gam.double(), bet.double())
    e_f = (f[:, :D].double() - want).abs().amax(1)
    e_sb = (sb.to_f32().double() - want).abs().amax(1)
    assert bool((f[:, D:] == 5.0).all())
    # observed on an H100 (D = 384 / 1280): float32 out 4.5e-7 on the ordinary rows, 2.8e-5 / 4.7e-5 on the rows with a
    # large mean (float32 statistics: torch's float32 layer_norm is off by 3e-5 there too); SB16 out 1.6e-5 / 5.4e-5
    large = torch.tensor([False, True, False, False, True, False, False], device="cuda")
    assert float(e_f[~large].max()) <= 2e-6 and float(e_f[large].max()) <= 2e-4, e_f.tolist()
    assert float(e_sb[~large].max()) <= 6.4e-5 and float(e_sb[large].max()) <= 2.2e-4, e_sb.tolist()


@pytest.mark.gpu
def test_softmax_pick_and_logprob_gather():
    """At V = 51866, a row with one dominant logit and a flat row: the picked probability and gathered log-probability
    against float64."""
    from whisper_timestamped import _native as nat
    V, ldl = 51866, 51866 + 6
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.zeros((3, ldl), device="cuda")
    x[0, :V] = torch.randn(V, device="cuda", generator=g) * 2
    x[0, 50362] = 40.0                                        # dominant
    x[1, :V] = 0.25                                           # flat
    x[2, :V] = torch.randn(V, device="cuda", generator=g) * 3
    x[2, V - 1] = 12.0                                        # the last column of the ragged tail
    x[:, V:] = 1e4                                            # padding past n must not be read
    st = nat.stream_ptr("cuda")
    picks = [(0, 50362), (1, 17), (2, V - 1)]
    out = torch.zeros(3, device="cuda")
    err_p = err_l = 0.0
    for r, t in picks:
        nat.check(nat.lib.wts_softmax_pick(x[r].data_ptr(), ldl, V, t, out[r:].data_ptr(), 1, st), "wts_softmax_pick")
    rows = torch.tensor([0, 0, 1, 2, 2], dtype=torch.int32, device="cuda")
    toks = torch.tensor([50362, 3, 17, V - 1, 0], dtype=torch.int32, device="cuda")
    lp = torch.zeros(5, device="cuda")
    nat.check(nat.lib.wts_logprob_gather(x.data_ptr(), ldl, V, rows.data_ptr(), toks.data_ptr(), lp.data_ptr(), 5, st),
              "wts_logprob_gather")
    torch.cuda.synchronize()
    ref = torch.log_softmax(x[:, :V].double(), -1)
    for r, t in picks:
        err_p = max(err_p, abs(float(out[r]) - math.exp(float(ref[r, t]))))
    for i in range(5):
        err_l = max(err_l, abs(float(lp[i]) - float(ref[int(rows[i]), int(toks[i])])))
    assert err_p <= 5e-9 and err_l <= 4e-6, (err_p, err_l)   # observed 1.3e-9 and 1.07e-6 (H100)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [384, 1280])
def test_embed_gather_rows_step_inputs_exact(D):
    from whisper_timestamped import _native as nat
    V = 51866
    g = torch.Generator(device="cuda").manual_seed(D + 3)
    st = nat.stream_ptr("cuda")
    emb = torch.randn((V, D), device="cuda", generator=g)
    pos = torch.randn((N_CTX, D), device="cuda", generator=g)
    tok = torch.tensor([0, V - 1, 50257, 7, 7, 30000], dtype=torch.int32, device="cuda")
    p = torch.tensor([0, 447, 3, 3, 200, 1], dtype=torch.int32, device="cuda")
    out = torch.empty((6, D), device="cuda")
    nat.check(nat.lib.wts_embed(tok.data_ptr(), p.data_ptr(), emb.data_ptr(), pos.data_ptr(), 6, D, out.data_ptr(), st),
              "wts_embed")
    idx = torch.tensor([5, 0, 0, 3], dtype=torch.int32, device="cuda")
    ldx = D + 20
    xs = torch.randn((6, ldx), device="cuda", generator=g)
    gat = torch.empty((4, D), device="cuda")
    nat.check(nat.lib.wts_gather_rows(xs.data_ptr(), ldx, idx.data_ptr(), 4, D, gat.data_ptr(), st), "wts_gather_rows")
    B, ld = 70, N_CTX + 1
    tokens = torch.randint(0, V, (B, ld), dtype=torch.int32, device="cuda", generator=g)
    n_tokens = torch.randint(1, ld, (B,), dtype=torch.int32, device="cuda", generator=g)
    n_prompt = torch.minimum(n_tokens, torch.randint(1, 230, (B,), dtype=torch.int32, device="cuda", generator=g))
    done = torch.randint(0, 3, (B,), dtype=torch.int32, device="cuda", generator=g)
    s = [torch.full((B,), -7, dtype=torch.int32, device="cuda") for _ in range(4)]
    nat.check(nat.lib.wts_step_inputs(tokens.data_ptr(), ld, n_tokens.data_ptr(), n_prompt.data_ptr(), done.data_ptr(), B,
                                      *(t.data_ptr() for t in s), st), "wts_step_inputs")
    torch.cuda.synchronize()
    assert torch.equal(out, emb[tok.long()] + pos[p.long()])
    assert torch.equal(gat, xs[idx.long(), :D])
    last = n_tokens.long() - 1
    assert torch.equal(s[0], tokens[torch.arange(B, device="cuda"), last])
    assert torch.equal(s[1], n_tokens - 1)
    assert torch.equal(s[2], torch.where(done != 0, torch.full_like(done, -1), n_tokens - n_prompt))
    assert torch.equal(s[3], (done == 0).int())

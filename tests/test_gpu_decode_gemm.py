"""The decode-time GEMM of a session of at most 64 windows (gemm_tc_split_kernel<1>: one 64-row A box, weights fetched
before the dependency wait) against the 128-row instance, bit for bit, and against a float64 product.

The 128-row instance (gemm_tc_split_kernel<2>) runs every one-tile GEMM of 65..128 rows, so the same rows padded to
M = 65 with zero rows (masked) give its arithmetic to compare with."""
import gc

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# (d_model, vocabulary) of the widths a decode step runs at
WIDTHS = {"tiny": (384, 51865), "medium": (1024, 51865), "large-v3": (1280, 51866)}
SHAPES = ("qkv", "out", "fc1", "fc2", "vocab")
ROWS = (1, 9, 17, 33, 64)


@pytest.fixture(autouse=True, scope="module")
def _free_device_memory():
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    yield
    gc.collect()
    if torch.cuda.is_available():
        torch.cuda.empty_cache()


def _eng():
    from whisper_timestamped.engine import CudaEngine
    eng = CudaEngine.__new__(CudaEngine)
    eng.dev, eng.backend, eng.launches = torch.device("cuda:0"), 0, 0
    return eng


def _sb(x):
    from whisper_timestamped.model import SB16
    return SB16.from_f32(x.contiguous())


def _f64(A):
    return A.to_f32().double()


def _mask(M):
    """active rows with finished rows in between (every third row from row 1), the last row active"""
    m = (torch.arange(M) % 3 != 1).to(torch.int32)
    m[-1] = 1
    return m


def _problem(shape, D, V, g):
    """(N, K, bias or None, GELU, residual in place, SB16 output) of one decode GEMM"""
    N, K = {"qkv": (3 * D, D), "out": (D, D), "fc1": (4 * D, D), "fc2": (D, 4 * D), "vocab": (V, D)}[shape]
    bias = None if shape == "vocab" else torch.randn(N, generator=g)
    return N, K, bias, shape == "fc1", shape in ("out", "fc2"), shape == "fc1"


def _run(eng, A, W, M, N, K, bias, act, residual, sb_out, mask, init, b_const):
    """One GEMM the way the decode step issues it; returns the output as float32 [M, N] (SB16: hi + lo planes)."""
    from whisper_timestamped.model import SB16
    dev = eng.dev
    kw = dict(bias=bias, act=1 if act else 0, row_mask=mask, b_const=b_const)
    if sb_out:
        out = SB16(M, N, dev)
        out.t.copy_(init)
        eng.gemm(A, W, M, N, K, out_sb=out, **kw)
        torch.cuda.synchronize()
        return out.t.clone()
    x = init.clone()
    if residual:
        eng.gemm(A, W, M, N, K, residual=x, ldr=N, out_f32=x, ldc=N, **kw)
    else:
        eng.gemm(A, W, M, N, K, out_f32=x, ldc=N, **kw)
    torch.cuda.synchronize()
    return x


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("width", list(WIDTHS))
def test_rows_equal_128_row_kernel_bitwise(width, shape):
    """Rows 1..64 of every decode GEMM shape: bit-identical to the same rows of the 128-row kernel (M = 65), masked
    rows untouched, active rows within the float64 bound of the tensor-core GEMM tests."""
    eng = _eng()
    dev = eng.dev
    D, V = WIDTHS[width]
    g = torch.Generator(device="cpu").manual_seed(100 * list(WIDTHS).index(width) + SHAPES.index(shape))
    N, K, bias, act, residual, sb_out = _problem(shape, D, V, g)
    W = _sb((torch.randn(N, K, generator=g) / K ** 0.5).to(dev))
    bias = bias.to(dev) if bias is not None else None
    a = torch.randn(64, K, generator=g).to(dev)
    x0 = torch.randn(64, N, generator=g).to(dev)
    torch.cuda.synchronize()                    # the weights are written before any GEMM may read them early
    for M in ROWS:
        A, A65 = _sb(a[:M]), _sb(torch.cat([a[:M], torch.zeros(65 - M, K, device=dev)]))
        mask = _mask(M).to(dev)
        mask65 = torch.cat([mask, torch.zeros(65 - M, dtype=torch.int32, device=dev)])
        if sb_out:
            init = torch.full((2, M, N), 3.0, dtype=torch.bfloat16, device=dev)
            init65 = torch.full((2, 65, N), 3.0, dtype=torch.bfloat16, device=dev)
        else:
            init, init65 = x0[:M].clone(), torch.cat([x0[:M], torch.zeros(65 - M, N, device=dev)])
        torch.cuda.synchronize()
        old = _run(eng, A65, W, 65, N, K, bias, act, residual, sb_out, mask65, init65, False)
        old = old[:, :M] if sb_out else old[:M]
        for b_const in (True, False):
            got = _run(eng, A, W, M, N, K, bias, act, residual, sb_out, mask, init, b_const)
            assert torch.equal(got, old), (width, shape, M, b_const)
        act_rows = mask.bool()
        if sb_out:
            assert torch.equal(got[:, ~act_rows], init[:, ~act_rows])
            val = got[0].float() + got[1].float()
        else:
            assert torch.equal(got[~act_rows], init[~act_rows])
            val = got
        ref = _f64(A) @ _f64(W).T
        if bias is not None:
            ref = ref + bias.double()
        if act:
            ref = torch.nn.functional.gelu(ref)
        if residual:
            ref = ref + init.double()
        scale = max(1.0, ref[act_rows].abs().max().item())
        err = (val[act_rows].double() - ref[act_rows]).abs().max().item()
        assert err <= (3e-4 if sb_out else 2e-4) * scale, (width, shape, M, err, scale)


# ---------------------------------------------------------------------------------------------- one whole step
N_ACTIVE = 40


def _fill(eng, ses, tok, seed):
    """Seeded state in slots 0..63 (the same values whatever the session's capacity): caches, cross K/V, float32
    alignment K, token histories; N_ACTIVE of them decoding, every other slot finished."""
    d = eng.dims
    g = torch.Generator(device="cuda").manual_seed(seed)
    rng = np.random.default_rng(seed)
    st8 = ses["st8"]
    for li in range(d.n_text_layer):
        for n in ("ck", "cv", "sk", "sv", "ckal"):
            t = st8[n][li]
            if t is None:
                continue
            t[:64].copy_((torch.randn((64,) + tuple(t.shape[1:]), device="cuda", generator=g) * 0.5).to(t.dtype))
    ses["qk_buf"][:64].copy_(torch.randn((64,) + tuple(ses["qk_buf"].shape[1:]), device="cuda", generator=g))
    ses["logprobs"][:64].copy_(torch.randn((64,) + tuple(ses["logprobs"].shape[1:]), device="cuda", generator=g))
    cap, n_ctx = ses["cap"], d.n_text_ctx
    tokens = np.zeros((cap, n_ctx + 1), dtype=np.int32)
    n_tok = np.ones(cap, dtype=np.int32)
    n_pr = np.ones(cap, dtype=np.int32)
    done = np.ones(cap, dtype=np.int32)
    sot = list(tok.sot_sequence)
    slots = sorted(rng.choice(64, N_ACTIVE, replace=False).tolist())
    for i in range(64):
        prompt = sot if i % 2 else [tok.sot_prev] + [int(t) for t in rng.integers(300, 30000, 30)] + sot
        row = prompt + [int(t) for t in rng.integers(300, 30000, int(rng.integers(0, 50)))]
        tokens[i, :len(row)] = row
        n_tok[i], n_pr[i] = len(row), len(prompt)
    done[:64] = 1 + (np.arange(64) % 2)
    done[slots] = 0
    ses["tokens"].copy_(torch.from_numpy(tokens))
    ses["n_tokens"].copy_(torch.from_numpy(n_tok))
    ses["n_prompt"].copy_(torch.from_numpy(n_pr))
    ses["done"].copy_(torch.from_numpy(done))
    torch.cuda.synchronize()
    return slots


def _one_step(m, cap):
    """Everything of the active rows that one per-operator step of a `cap`-slot session writes."""
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.tokenizer import get_tokenizer
    from whisper_timestamped.windows import make_decode_setup
    eng = CudaEngine(m, max_batch=cap, small_batch_rows=8)
    tok = get_tokenizer(m.is_multilingual, num_languages=m.num_languages, language="en", task="transcribe")
    setup = make_decode_setup(tok, m.dims.n_text_ctx)
    ses = eng._decoder_session(setup, cap)
    assert ses["cap"] == cap
    eng._set_masks(ses, setup)
    slots = _fill(eng, ses, tok, seed=77)
    idx = torch.as_tensor(slots, device="cuda")
    n0, p0 = ses["n_tokens"][idx].long(), ses["n_prompt"][idx].long()
    eng._step(ses)
    torch.cuda.synchronize()
    out = {"logits": ses["logits"][idx], "tokens": ses["tokens"][idx], "n_tokens": ses["n_tokens"][idx],
           "done": ses["done"][idx], "logprobs": ses["logprobs"][idx], "qk": ses["qk_buf"][idx, :, n0 - p0]}
    for li in range(m.dims.n_text_layer):
        for n in ("sk", "sv"):
            out[f"{n}{li}"] = ses["st8"][n][li][idx, :, n0 - 1]
    out = {k: v.cpu() for k, v in out.items()}
    del ses, eng
    gc.collect()
    torch.cuda.empty_cache()
    return slots, out


def test_step_cap64_equals_cap128_bitwise():
    """One per-operator decode step at large-v3 width: a 64-slot session (64-row GEMMs) and a 128-slot session (128-row
    GEMMs) holding the same 64 windows write bit-identical logits, self K/V, alignment rows, choices and log-probs."""
    import whisper_timestamped as wt
    m = wt.load_model("synthetic:large-v3", device="cuda")
    slots64, got = _one_step(m, 64)
    slots128, want = _one_step(m, 128)
    assert slots64 == slots128
    for k in want:
        assert torch.equal(got[k], want[k]), k
    del m
    gc.collect()
    torch.cuda.empty_cache()

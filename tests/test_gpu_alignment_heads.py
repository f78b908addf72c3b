"""GPU: `word_alignment_most_top_layers=k`, models without an alignment-head table, the per-layer compacted float32 K
copy of the cross-attention entries and the head-parallel attention prep."""
import glob
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = sorted(glob.glob(os.path.join(HERE, "golden", "heads", "*.json")))


def _model(g, tmp_path):
    import whisper_timestamped as wt
    from whisper_timestamped import model_zoo as zoo
    if g["table_heads"]:
        return wt.load_model("synthetic:" + g["model"], device="cuda", synthetic_kwargs=g["model_kwargs"])
    dims = zoo.DIMS[g["model"]]
    path = os.path.join(str(tmp_path), f"finetuned-{g['model']}.pt")       # a name outside the table
    torch.save({"dims": dims.asdict(), "model_state_dict": zoo.synthetic_state_dict(dims, seed=g["model_seed"],
                                                                                    **g["model_kwargs"])}, path)
    return wt.load_model(path, device="cuda")


@pytest.mark.parametrize("path", CASES, ids=[os.path.basename(p)[:-5] for p in CASES])
def test_transcribe_matches_heads_golden(path, tmp_path):
    import whisper_timestamped as wt
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from test_host_e2e import compare, stitch_cuts
    g = json.load(open(path))
    m = _model(g, tmp_path)
    kw = dict(g["transcribe_kwargs"])
    if "chunks" in g:
        kw["chunks"] = g["chunks"]
    res = wt.transcribe(m, synthetic_speech(*g["audio"]), **kw)
    if "chunks" in g:
        compare(res, stitch_cuts(g)[0], conf_tol=2e-3, time_tol=1e-6)
    else:
        compare(res, g["result"], conf_tol=2e-3)


def _cross(nat, q, k16, v16, kal, slot, n_slots, s0, n_l, row_seq, R, H, out, qk_out, qk_rows, qk_row, legacy=False):
    D = H * 64
    if legacy:
        return nat.lib.wts_cross_attention_f16(q.data_ptr(), D, k16.data_ptr(), v16.data_ptr(), kal.data_ptr(),
                                               slot.data_ptr(), n_slots, 1500, row_seq.data_ptr(), R, H, out.ptr, out.ld,
                                               out.plane, qk_out.data_ptr(), qk_rows, qk_row.data_ptr(), None, None)
    return nat.lib.wts_cross_attention_f16_layer(q.data_ptr(), D, k16.data_ptr(), v16.data_ptr(),
                                                 kal.data_ptr() if kal is not None else None, slot.data_ptr(), n_slots,
                                                 s0, n_l, 1500, row_seq.data_ptr(), R, H, out.ptr, out.ld, out.plane,
                                                 qk_out.data_ptr(), qk_rows, qk_row.data_ptr(), None, None)


def test_compacted_cross_attention_layers_vs_torch():
    """Two layers of a 9-slot head set: layer A holds slots 2..6 (5 heads), layer B none.  Pack + attention through
    the per-layer entries against torch; the old entry (s0 = 0, n_l = n_slots) on a full-size copy writes the same
    rows bit for bit."""
    from whisper_timestamped import _native as nat
    from whisper_timestamped.model import SB16
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(5)
    B, H, ctx, n_slots, qk_rows = 3, 6, 1500, 9, 4
    D = H * 64
    slot_a = torch.tensor([2, -1, 3, 4, 5, 6], dtype=torch.int32, device=dev)
    slot_b = torch.full((H,), -1, dtype=torch.int32, device=dev)
    src = torch.randn((B, H, ctx, 64), device=dev, generator=g)
    k16 = torch.empty((B, H, ctx, 64), dtype=torch.float16, device=dev)
    v16 = (torch.randn((B, H, ctx, 64), device=dev, generator=g) * 0.5).half()
    kal = torch.full((B, 5, ctx, 64), -9.0, device=dev)
    st = nat.stream_ptr(dev)
    nat.check(nat.lib.wts_cross_kv_pack_layer(src.data_ptr(), k16.data_ptr(), kal.data_ptr(), slot_a.data_ptr(), 2, 5,
                                              B, H, ctx, st), "pack")
    kal_full = torch.full((B, n_slots, ctx, 64), -9.0, device=dev)
    k16b = torch.empty_like(k16)
    nat.check(nat.lib.wts_cross_kv_pack(src.data_ptr(), k16b.data_ptr(), kal_full.data_ptr(), slot_a.data_ptr(), n_slots,
                                        B, H, ctx, st), "pack old")
    torch.cuda.synchronize()
    assert torch.equal(k16, src.half()) and torch.equal(k16, k16b)
    for h in range(H):
        s = int(slot_a[h])
        if s >= 0:
            assert torch.equal(kal[:, s - 2], src[:, h]) and torch.equal(kal_full[:, s], src[:, h])
    R = 4
    row_seq = torch.tensor([2, 0, 1, 2], dtype=torch.int32, device=dev)
    qk_row = torch.tensor([0, 3, 1, 2], dtype=torch.int32, device=dev)
    q = torch.randn((R, D), device=dev, generator=g) * 0.3
    ref_rows = torch.einsum("rhc,rhfc->rhf", q.view(R, H, 64), src[row_seq.long()])
    ref_out = torch.einsum("rhf,rhfc->rhc", torch.softmax(torch.einsum("rhc,rhfc->rhf", q.view(R, H, 64),
                                                                       k16[row_seq.long()].float()), -1),
                           v16[row_seq.long()].float()).reshape(R, D)
    outs = {}
    for name, args in (("a", (kal, slot_a, 2, 5, False)), ("b", (None, slot_b, 0, 0, False)),
                       ("old", (kal_full, slot_a, 0, n_slots, True))):
        kl, sl, s0, n_l, legacy = args
        out = SB16(R, D, dev)
        qk_out = torch.full((B, n_slots, qk_rows, ctx), -77.0, device=dev)
        nat.check(_cross(nat, q, k16, v16, kl, sl, n_slots, s0, n_l, row_seq, R, H, out, qk_out, qk_rows, qk_row,
                         legacy=legacy), name)
        torch.cuda.synchronize()
        outs[name] = (out.to_f32(), qk_out)
        assert torch.allclose(out.to_f32(), ref_out, atol=2e-3, rtol=2e-3), name
    assert torch.equal(outs["a"][0], outs["old"][0]) and torch.equal(outs["a"][1], outs["old"][1])
    # layer B reads fp16 K for every head: the same output as layer A for the heads that are not alignment heads
    for h in range(H):
        if int(slot_a[h]) < 0:
            assert torch.equal(outs["b"][0][:, h * 64:(h + 1) * 64], outs["a"][0][:, h * 64:(h + 1) * 64])
    assert bool((outs["b"][1] == -77.0).all())                       # a layer without alignment heads writes no row
    qa = outs["a"][1]
    for r in range(R):
        for h in range(H):
            s = int(slot_a[h])
            if s >= 0:
                got = qa[int(row_seq[r]), s, int(qk_row[r])]
                assert torch.allclose(got, ref_rows[r, h], atol=1e-4, rtol=1e-4), (r, h)


@pytest.mark.parametrize("small_batch_rows", [0, 32])
def test_lean_and_per_operator_steps_top_layers(small_batch_rows):
    """A top-layers head set (layers without alignment heads next to layers with all of theirs) through the per-operator
    step only (0) and through the lean small-batch step whenever at most 32 windows are left (32): both reproduce the
    reference golden."""
    import whisper_timestamped as wt
    from whisper_timestamped.engine import CudaEngine
    from whisper_timestamped.synthetic_audio import synthetic_speech
    from test_host_e2e import compare, stitch_cuts
    g = json.load(open(os.path.join(HERE, "golden", "heads", "tiny_top2_chunks.json")))
    m = wt.load_model("synthetic:tiny", device="cuda")
    eng = CudaEngine(m, small_batch_rows=small_batch_rows)
    res = wt.transcribe(m, synthetic_speech(*g["audio"]), engine=eng, chunks=g["chunks"], **g["transcribe_kwargs"])
    compare(res, stitch_cuts(g)[0], conf_tol=2e-3, time_tol=1e-6)
    if small_batch_rows:
        assert eng.small_batch_steps > 0


@pytest.mark.parametrize("N", [120, 320])
def test_prep_many_heads_matches_oracle(N):
    import oracle
    from oracle.prep import attn_cost
    from whisper_timestamped import _native as nat
    from whisper_timestamped.alignment import attn_prep, cost_matrix, dtw, plan_segments, split_jumps
    rng = np.random.default_rng(N)
    rows = 40
    qk = (3 * rng.standard_normal((2, N, rows, 1500))).astype(np.float32)
    items = [(0, 0, None, 24, 100, 300, 0), (1, 3, None, 30, 0, 500, 450), (0, 24, None, 12, 700, 160, 0)]
    plan = plan_segments(items)
    d_qk = torch.from_numpy(qk).cuda()
    cost = attn_prep(d_qk, plan)
    jl = split_jumps(dtw(cost, plan)["jumps"].cpu().numpy(), plan)
    ch = cost.cpu().numpy()
    # the serial kernel on the same input: same numbers up to the summation order over heads
    cost1 = torch.empty_like(cost)
    from whisper_timestamped.alignment import _segs_to_device
    nat.check(nat.lib.wts_attn_prep_batch_kernel(d_qk.data_ptr(), N, rows, 1500, _segs_to_device(plan.segs, torch.device("cuda")).data_ptr(),
                                                 plan.nseg, plan.max_T, plan.max_F, cost1.data_ptr(), 1,
                                                 nat.stream_ptr("cuda")), "prep serial")
    torch.cuda.synchronize()
    assert np.max(np.abs(cost1.cpu().numpy() - ch)) <= 1e-6
    for k, (w, row0, _, T, f0, F, md) in enumerate(items):
        c = np.ascontiguousarray(cost_matrix(ch, plan.segs[k]))
        ref = attn_cost(qk[w][:, row0:row0 + T], f0, f0 + F, max_duration=md or None)
        assert np.max(np.abs(c - ref)) <= 1e-6, k
        _, _, j, _ = oracle.dtw_symmetric1(c.astype(np.float64))
        assert np.array_equal(jl[k], j), k


def test_default_then_top_layers_then_default():
    import whisper_timestamped as wt
    from whisper_timestamped.synthetic_audio import synthetic_speech
    m = wt.load_model("synthetic:tiny", device="cuda")
    audio = synthetic_speech(75.0, seed=11)
    a = wt.transcribe(m, audio, language="en")
    b = wt.transcribe(m, audio, language="en", word_alignment_most_top_layers=6)
    c = wt.transcribe(m, audio, language="en")
    assert json.dumps(a, sort_keys=True) == json.dumps(c, sort_keys=True)
    assert [s["tokens"] for s in a["segments"]] == [s["tokens"] for s in b["segments"]]
    assert m.engine().heads == sorted(m.heads)


def test_many_heads_memory_is_bounded(tmp_path):
    """large-v3 shape without a table (320 heads) at the auto-sized batch: 40 minutes in 30-s chunks (80 windows, two
    decode batches per round) peak within 5 % of 20 minutes (40 windows, one batch per round): the alignment rows of
    one decode batch are alive at a time.  (5 minutes would be a 10-window batch, a smaller session.)"""
    import whisper_timestamped as wt
    from whisper_timestamped.synthetic_audio import synthetic_speech
    g = dict(model="large-v3", model_seed=1234, model_kwargs={"ts_offset": 4.5, "eot_logit": 14.5}, table_heads=False)
    m = _model(g, tmp_path)
    assert len(m.heads) == 320
    peaks = []
    for minutes in (20, 40):
        audio = np.concatenate([synthetic_speech(300.0, seed=1234 + k) for k in range(minutes // 5)])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        wt.transcribe(m, audio, language="en", chunks=30.0)
        peaks.append(torch.cuda.max_memory_allocated())
    assert peaks[1] <= 1.05 * peaks[0], peaks

"""GPU parity tests proper for the alignment numerics (run with -m gpu on an H100).

All calls go through the C-ABI (libwts.so via ctypes); the oracle is only the checker.
Bars: DTW jumps / paths bit-exact; attention post-processing within 1e-6 absolute of the
oracle (values are O(1)), and bit-exact jumps when the oracle's DTW is fed the GPU-made cost.
"""
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from oracle.prep import attn_cost

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PREP_ATOL = 1e-6


def _dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def run_dtw(mats, dtype=np.float32, want_path=False, want_status=False):
    """mats: list of [T,F] arrays -> list of jumps (and paths) from the CUDA kernel."""
    from whisper_timestamped.alignment import plan_segments, dtw, split_jumps, put_cost_matrix
    plan = plan_segments([(0, 0, None, m.shape[0], 0, m.shape[1], 0) for m in mats])
    host = np.zeros(plan.cost_elems, dtype=dtype)
    for s, m in zip(plan.segs, mats):
        put_cost_matrix(host, s, m.astype(dtype))
    cost = torch.from_numpy(host).to(_dev())
    out = dtw(cost, plan, want_path=want_path, want_status=want_status)
    torch.cuda.synchronize()
    jumps = split_jumps(out["jumps"].cpu().numpy(), plan)
    res = {"jumps": jumps}
    if want_path:
        p = out["path"].cpu().numpy()
        plen = out["path_len"].cpu().numpy()
        paths = [None] * len(mats)
        for k, seg_idx in enumerate(out["path_order"]):
            T, F = mats[seg_idx].shape
            o = out["path_off"][k]
            paths[seg_idx] = (p[o:o + plen[k]], p[o + T + F:o + T + F + plen[k]])
        res["paths"] = paths
    if want_status:
        st = out["status"].cpu().numpy()
        status = [0] * len(mats)
        for k, seg_idx in enumerate(out["status_order"]):
            status[seg_idx] = int(st[k])
        res["status"] = status
    return res


def test_dtw_golden_vectors_bit_exact():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden
    g = np.load(os.path.join(HERE, "golden", "dtw_golden.npz"))
    cases = make_golden.dtw_cases()
    mats = [c for _, c in cases]
    res = run_dtw(mats, want_path=True)
    for n, m in enumerate(mats):
        assert np.array_equal(res["jumps"][n], g[f"dtw{n}_jumps"]), (n, m.shape, cases[n][0])
        i1, i2 = res["paths"][n]
        assert np.array_equal(i1, g[f"dtw{n}_i1"]) and np.array_equal(i2, g[f"dtw{n}_i2"]), (n, m.shape)


def test_dtw_random_mixed_batch_vs_oracle():
    rng = np.random.default_rng(2024)
    mats = []
    for k in range(1500):
        T = int(rng.integers(1, 70))
        F = int(min(1500, T * rng.integers(1, 13) + rng.integers(0, 5)))
        F = max(F, T)
        kind = k % 5
        if kind == 0:
            c = -rng.random((T, F), dtype=np.float32)
        elif kind == 1:
            c = -rng.integers(0, 2, (T, F)).astype(np.float32)
        elif kind == 2:
            c = rng.standard_normal((T, F)).astype(np.float32)
        elif kind == 3:
            c = -np.abs(rng.standard_normal((T, F)).astype(np.float32)) * 1e-6
        else:
            c = -(rng.random((T, F), dtype=np.float32) ** 8)
        mats.append(c)
    res = run_dtw(mats)
    for n, m in enumerate(mats):
        _, _, j, _ = oracle.dtw_symmetric1(m.astype(np.float64))
        assert np.array_equal(res["jumps"][n], j), (n, m.shape)


def test_dtw_float64_input():
    rng = np.random.default_rng(5)
    mats = [rng.standard_normal((T, F)) for (T, F) in [(3, 9), (24, 300), (40, 77), (100, 160)]]
    res = run_dtw(mats, dtype=np.float64, want_path=True)
    for n, m in enumerate(mats):
        i1, i2, j, _ = oracle.dtw_symmetric1(m)
        assert np.array_equal(res["jumps"][n], j)
        assert np.array_equal(res["paths"][n][0], i1) and np.array_equal(res["paths"][n][1], i2)


def test_dtw_worst_case_size():
    rng = np.random.default_rng(11)
    mats = [-rng.random((224, 1500), dtype=np.float32) for _ in range(6)]
    mats.append(mats[0].copy())
    res = run_dtw(mats)
    for n in (0, 3, 5):
        _, _, j, _ = oracle.dtw_symmetric1(mats[n].astype(np.float64))
        assert np.array_equal(res["jumps"][n], j)
    assert np.array_equal(res["jumps"][0], res["jumps"][6])


def test_dtw_full_size_batch_properties():
    """BASELINE-size batch (4096 typical matrices): size-independent properties + sampled oracle."""
    rng = np.random.default_rng(3)
    base = [-rng.random((24, 300), dtype=np.float32) for _ in range(64)]
    mats = [base[k % 64] for k in range(4096)]
    res = run_dtw(mats)
    for n in range(4096):
        j = res["jumps"][n]
        assert j[0] == 0 and j[-1] == 299 and np.all(np.diff(j) >= 0)
        assert np.array_equal(j, res["jumps"][n % 64])          # idempotent across the batch
    for n in range(0, 64, 7):
        _, _, j, _ = oracle.dtw_symmetric1(base[n].astype(np.float64))
        assert np.array_equal(res["jumps"][n], j)


def test_dtw_nonpositive_fast_path_vs_oracle():
    """Integer-compare fast path (flags bit 0) on strictly negative costs, incl. multi-strip and worst-case sizes."""
    from whisper_timestamped.alignment import plan_segments, dtw, split_jumps
    rng = np.random.default_rng(17)
    shapes = [(1, 5), (2, 9), (24, 300), (31, 64), (32, 70), (63, 200), (100, 380), (224, 1500), (12, 12)]
    mats = []
    for (T, F) in shapes:
        for kind in range(3):
            if kind == 0:
                c = -(rng.random((T, F), dtype=np.float32) + 1e-3)
            elif kind == 1:
                c = -np.ones((T, F), np.float32)                      # all ties
            else:
                c = -(rng.integers(1, 4, (T, F)).astype(np.float32))   # many ties
            mats.append(c)
    plan = plan_segments([(0, 0, None, m.shape[0], 0, m.shape[1], 0) for m in mats], nonpositive=True)
    host = np.zeros(plan.cost_elems, dtype=np.float32)
    from whisper_timestamped.alignment import put_cost_matrix
    for s, m in zip(plan.segs, mats):
        put_cost_matrix(host, s, m)
    out = dtw(torch.from_numpy(host).to(_dev()), plan)
    torch.cuda.synchronize()
    jl = split_jumps(out["jumps"].cpu().numpy(), plan)
    for n, m in enumerate(mats):
        _, _, j, _ = oracle.dtw_symmetric1(m.astype(np.float64))
        assert np.array_equal(jl[n], j), (n, m.shape)


@pytest.mark.parametrize("chains,bands", [(4, 2), (2, 4), (2, 2), (2, 1), (4, 1)])
@pytest.mark.parametrize("max_rows", [8, 16, 24, 32, 70])
def test_dtw_lane_kernel_vs_oracle(max_rows, chains, bands, monkeypatch):
    """The lane-per-matrix kernel (large batches; forced here with WTS_DTW_LANE_MIN=1) on ragged batches: every row
    unrolling (8/16/24/32), matrices above 32 rows falling back to the general kernel in the same call, heavy ties."""
    from whisper_timestamped.alignment import plan_segments, dtw, split_jumps, put_cost_matrix
    monkeypatch.setenv("WTS_DTW_LANE_MIN", "1")
    monkeypatch.setenv("WTS_DTW_LANE_NC", str(chains))
    monkeypatch.setenv("WTS_DTW_LANE_G", str(bands))
    rng = np.random.default_rng(100 + max_rows)
    shapes = [(1, 1), (1, 2), (2, 2), (min(max_rows, 32), 7), (min(max_rows, 32), 8), (min(max_rows, 32), 9), (3, 16), (3, 17),
              (min(max_rows, 24), 300), (min(max_rows, 31), 354), (min(max_rows, 32), 1500), (5, 1499)]
    shapes += [(int(rng.integers(1, max_rows + 1)), int(rng.integers(1, 420))) for _ in range(150)]
    mats = []
    for n, (T, F) in enumerate(shapes):
        if n % 3 == 0:
            c = -(rng.random((T, F), dtype=np.float32) + 1e-3)
        elif n % 3 == 1:
            c = -np.ones((T, F), np.float32)
        else:
            c = -(rng.integers(1, 4, (T, F)).astype(np.float32))
        mats.append(c)
    plan = plan_segments([(0, 0, None, m.shape[0], 0, m.shape[1], 0) for m in mats], nonpositive=True)
    host = np.zeros(plan.cost_elems, dtype=np.float32)
    for s, m in zip(plan.segs, mats):
        put_cost_matrix(host, s, m)
    out = dtw(torch.from_numpy(host).to(_dev()), plan)
    torch.cuda.synchronize()
    jl = split_jumps(out["jumps"].cpu().numpy(), plan)
    for n, m in enumerate(mats):
        _, _, j, _ = oracle.dtw_symmetric1(m.astype(np.float64))
        assert np.array_equal(jl[n], j), (n, m.shape)


def test_dtw_lane_kernel_equals_wavefront_kernel_at_full_size(monkeypatch):
    """BASELINE-size batch (16384 x 24 x 300, what bench.py --workload align times): both kernels, identical jumps."""
    from whisper_timestamped.alignment import plan_segments, dtw, put_cost_matrix
    rng = np.random.default_rng(8)
    base = [-(rng.random((24, 300), dtype=np.float32) + 1e-3) for _ in range(256)]
    plan = plan_segments([(0, 0, None, 24, 0, 300, 0)] * 16384, nonpositive=True)
    host = np.zeros(plan.cost_elems, dtype=np.float32)
    for k, s in enumerate(plan.segs):
        put_cost_matrix(host, s, base[k % 256])
    cost = torch.from_numpy(host).to(_dev())
    monkeypatch.setenv("WTS_DTW_LANE_MIN", "0")
    a = dtw(cost, plan)["jumps"].cpu().numpy()
    monkeypatch.setenv("WTS_DTW_LANE_MIN", "1")
    b = dtw(cost, plan)["jumps"].cpu().numpy()
    assert np.array_equal(a, b)
    for n in range(0, 256, 37):
        _, _, j, _ = oracle.dtw_symmetric1(base[n].astype(np.float64))
        assert np.array_equal(b[plan.segs[n]["jumps_off"]: plan.segs[n]["jumps_off"] + 25], j)


def test_dtw_status_flags_non_finite():
    a = -np.ones((4, 9), np.float32)
    b = a.copy()
    b[2, 3] = np.nan
    res = run_dtw([a, b], want_status=True)
    assert res["status"] == [0, 1]


def _prep_case(qk_full, N, T, F, f0, max_dur, last_row=None):
    """qk_full [N, Trows, 1500] float32 -> (gpu cost [T,F] float32, gpu jumps).  The DTW runs twice — generic
    float64 compares and the integer-compare fast path for non-positive costs — and both must agree."""
    from whisper_timestamped.alignment import plan_segments, attn_prep, dtw, split_jumps, cost_matrix
    qk = torch.from_numpy(qk_full[None]).to(_dev()).contiguous()
    plan = plan_segments([(0, 0, last_row, T, f0, F, max_dur)])
    cost = attn_prep(qk, plan)
    out = dtw(cost, plan)
    plan_fast = plan_segments([(0, 0, last_row, T, f0, F, max_dur)], nonpositive=True)
    out_fast = dtw(cost, plan_fast)
    torch.cuda.synchronize()
    c = np.ascontiguousarray(cost_matrix(cost.cpu().numpy(), plan.segs[0]))
    j = split_jumps(out["jumps"].cpu().numpy(), plan)[0]
    assert np.array_equal(j, split_jumps(out_fast["jumps"].cpu().numpy(), plan_fast)[0])
    return c, j


def test_prep_golden_vectors():
    g = np.load(os.path.join(HERE, "golden", "prep_golden.npz"))
    n = 0
    while f"prep{n}_spec" in g:
        N, T, F, f0, max_dur = g[f"prep{n}_spec"].tolist()
        qk_full = np.zeros((N, T, 1500), np.float32)
        qk_full[:, :, f0:f0 + F] = g[f"prep{n}_qk"]
        c, jumps = _prep_case(qk_full, N, T, F, f0, max_dur)
        ref = g[f"prep{n}_cost"]
        assert np.max(np.abs(c - ref)) <= PREP_ATOL, (n, np.max(np.abs(c - ref)))
        assert np.array_equal(c == 0, ref == 0)                       # padding mask, exact zeros
        assert c[0, 0] == c.min()
        # bit-exact at the DTW boundary: oracle DTW on the GPU-made cost gives the GPU's jumps
        _, _, j, _ = oracle.dtw_symmetric1(c.astype(np.float64))
        assert np.array_equal(jumps, j), n
        n += 1
    assert n >= 10


def test_prep_random_vs_oracle_and_truncation_row():
    rng = np.random.default_rng(77)
    N, rows = 10, 30
    qk_full = (3 * rng.standard_normal((N, rows, 1500))).astype(np.float32)
    # regular segment
    c, jumps = _prep_case(qk_full, N, 20, 260, 100, 0)
    ref = attn_cost(qk_full[:, :20], 100, 360)
    assert np.max(np.abs(c - ref)) <= PREP_ATOL
    # truncated text (T.py:1516-1535): rows 0..T-2 then the LAST row of the window's rows
    T = 12
    c, jumps = _prep_case(qk_full, N, T, 11 + 2, 50, 0, last_row=rows - 1)
    sel = np.concatenate([qk_full[:, :T - 1], qk_full[:, rows - 1:rows]], axis=1)
    ref = attn_cost(sel, 50, 63)
    assert np.max(np.abs(c - ref)) <= PREP_ATOL
    _, _, j, _ = oracle.dtw_symmetric1(c.astype(np.float64))
    assert np.array_equal(jumps, j)


def test_prep_batch_many_segments_one_launch():
    from whisper_timestamped.alignment import plan_segments, attn_prep, dtw, split_jumps, cost_matrix
    rng = np.random.default_rng(8)
    N, W, rows = 6, 3, 64
    qk = (2 * rng.standard_normal((W, N, rows, 1500))).astype(np.float32)
    items = []
    for k in range(40):
        T = int(rng.integers(2, 40))
        row0 = int(rng.integers(0, rows - T))
        F = int(rng.integers(T, 400))
        f0 = int(rng.integers(0, 1500 - F))
        md = int(rng.integers(1, F + 60)) if k % 3 == 0 else 0
        items.append((k % W, row0, None, T, f0, F, md))
    plan = plan_segments(items, nonpositive=True)
    d_qk = torch.from_numpy(qk).to(_dev())
    cost = attn_prep(d_qk, plan)
    out = dtw(cost, plan)
    torch.cuda.synchronize()
    ch = cost.cpu().numpy()
    jl = split_jumps(out["jumps"].cpu().numpy(), plan)
    for k, (w, row0, _, T, f0, F, md) in enumerate(items):
        s = plan.segs[k]
        c = np.ascontiguousarray(cost_matrix(ch, s))
        ref = attn_cost(qk[w][:, row0:row0 + T], f0, f0 + F, max_duration=md or None)
        assert np.max(np.abs(c - ref)) <= PREP_ATOL, k
        _, _, j, _ = oracle.dtw_symmetric1(c.astype(np.float64))
        assert np.array_equal(jl[k], j), k

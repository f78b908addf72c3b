"""Host side of the batched alignment numerics: descriptor planning + libwts launches.

Replaces, for a batch of segments, the numerical part of `perform_word_alignment`
(/root/reference/whisper_timestamped/transcribe.py:1510-1581 and 1648-1652): attention
post-processing (`wts_attn_prep_batch`) and monotonic DTW (`wts_dtw_batch`).
"""
from dataclasses import dataclass

import numpy as np
import torch

from . import _native as nat

SEG_NONPOSITIVE, SEG_PITCH16 = 1, 2            # WtsSegDesc.flags (include/wts.h)


@dataclass
class AlignPlan:
    segs: np.ndarray          # structured SEG_DTYPE, in caller order
    cost_elems: int
    jumps_elems: int
    dir_words: int
    bnd_doubles: int
    max_T: int
    max_F: int
    dtw_order: np.ndarray     # launch order of the DTW warps (largest matrices first)

    @property
    def nseg(self):
        return len(self.segs)


def plan_segments(items, nonpositive=False) -> AlignPlan:
    """items: iterable of dicts/tuples (window, row0, last_row, T, f0, F, max_dur).

    Lays the per-segment cost matrices, jumps and DTW workspaces back to back.
    nonpositive=True promises that the float32 costs are <= 0 with cost[0,0] < 0 — what wts_attn_prep_batch
    produces — and lets the DTW kernel use integer compares in its dependent chain (flags bit 0)."""
    items = list(items)
    segs = np.zeros(len(items), dtype=nat.SEG_DTYPE)
    cost = jumps = dirw = bnd = 0
    max_T = max_F = 0
    for i, it in enumerate(items):
        if isinstance(it, dict):
            window, row0, last_row, T, f0, F, max_dur = (it["window"], it["row0"], it.get("last_row"),
                                                         it["T"], it["f0"], it["F"], it.get("max_dur", 0))
        else:
            window, row0, last_row, T, f0, F, max_dur = it
        if last_row is None:
            last_row = row0 + T - 1
        if T < 1 or F < 1:
            raise ValueError(f"segment {i}: empty alignment problem T={T} F={F}")
        s = segs[i]
        s["window"], s["row0"], s["last_row"], s["T"], s["f0"], s["F"] = window, row0, last_row, T, f0, F
        s["max_dur"] = max_dur or 0
        s["flags"] = (SEG_NONPOSITIVE if nonpositive else 0) | SEG_PITCH16
        s["cost_off"], s["jumps_off"], s["dir_off"], s["bnd_off"] = cost, jumps, dirw, bnd
        cost += T * seg_pitch(s)                    # rows padded to 16 bytes: every row (hence every matrix) is 16-byte aligned
        jumps += T + 1
        dirw += nat.lib.wts_dtw_dir_words(T, F)
        bnd += nat.lib.wts_dtw_bnd_doubles(T, F)
        max_T, max_F = max(max_T, T), max(max_F, F)
    work = segs["T"].astype(np.int64) * segs["F"].astype(np.int64)
    order = np.argsort(-work, kind="stable")
    return AlignPlan(segs, cost, jumps, max(dirw, 1), max(bnd, 1), max_T, max_F, order)


def seg_pitch(seg) -> int:
    """Row pitch (float32 elements) of a segment's cost matrix: WtsSegDesc.flags bit 1 = rows padded to 16 bytes."""
    F = int(seg["F"])
    return (F + 3) & ~3 if int(seg["flags"]) & SEG_PITCH16 else F


def cost_matrix(cost_host: np.ndarray, seg) -> np.ndarray:
    """[T, F] view of one segment's matrix inside a host copy of the cost buffer."""
    T, F, P = int(seg["T"]), int(seg["F"]), seg_pitch(seg)
    off = int(seg["cost_off"])
    return cost_host[off: off + T * P].reshape(T, P)[:, :F]


def put_cost_matrix(cost_host: np.ndarray, seg, m) -> None:
    """Writes a [T, F] matrix into a host cost buffer laid out by plan_segments (padding columns zeroed)."""
    T, F, P = int(seg["T"]), int(seg["F"]), seg_pitch(seg)
    off = int(seg["cost_off"])
    view = cost_host[off: off + T * P].reshape(T, P)
    view[:, F:] = 0
    view[:, :F] = np.asarray(m).reshape(T, F)


def _segs_to_device(arr: np.ndarray, device) -> torch.Tensor:
    host = torch.from_numpy(arr.view(np.uint8).reshape(-1).copy())
    if device.type == "cuda":
        host = host.pin_memory()
    return host.to(device, non_blocking=True)


def attn_prep(qk: torch.Tensor, plan: AlignPlan, cost: torch.Tensor = None,
              d_segs: torch.Tensor = None, kernel: int = 0) -> torch.Tensor:
    """qk: float32 [n_windows, N, Tmax, Fmax] on the GPU.  Returns the float32 cost buffer.
    kernel: 0 = chosen by N, 1 = serial over heads, 2 = head-parallel (wts_attn_prep_batch_kernel)."""
    nat.require_cuda(qk, "qk")
    assert qk.dtype == torch.float32 and qk.dim() == 4 and qk.is_contiguous()
    _, N, Tmax, Fmax = qk.shape
    if cost is None:
        cost = torch.empty(plan.cost_elems, dtype=torch.float32, device=qk.device)
    if d_segs is None:
        d_segs = _segs_to_device(plan.segs, qk.device)
    rc = nat.lib.wts_attn_prep_batch_kernel(nat.ptr(qk), N, Tmax, Fmax, nat.ptr(d_segs), plan.nseg, plan.max_T,
                                            plan.max_F, nat.ptr(cost), kernel, nat.stream_ptr(qk.device))
    nat.check(rc, "wts_attn_prep_batch_kernel")
    return cost


def dtw_descriptors(plan: AlignPlan, device) -> torch.Tensor:
    """Device copy of the descriptors in DTW launch order (largest matrices first)."""
    return _segs_to_device(plan.segs[plan.dtw_order], device)


def dtw(cost: torch.Tensor, plan: AlignPlan, want_path=False, want_status=False, workspace=None, d_segs=None,
        jumps=None):
    """cost: float32 or float64 buffer laid out by `plan`.  Returns dict with device tensors
    `jumps` (int32, plan.jumps_elems) and optionally `path`, `path_off`, `path_len`, `status`."""
    nat.require_cuda(cost, "cost")
    assert cost.dtype in (torch.float32, torch.float64)
    dev = cost.device
    segs_sorted = plan.segs[plan.dtw_order]
    if d_segs is None:
        d_segs = _segs_to_device(segs_sorted, dev)
    if workspace is None:
        workspace = (torch.empty(plan.dir_words, dtype=torch.int32, device=dev),
                     torch.empty(plan.bnd_doubles, dtype=torch.float64, device=dev))
    d_dir, d_bnd = workspace
    if jumps is None:
        jumps = torch.empty(plan.jumps_elems, dtype=torch.int32, device=dev)
    out = {"jumps": jumps}
    d_path = d_poff = d_plen = d_status = None
    if want_path:
        TF = (segs_sorted["T"].astype(np.int64) + segs_sorted["F"].astype(np.int64)) * 2
        poff = np.zeros(plan.nseg, dtype=np.int64)
        poff[1:] = np.cumsum(TF[:-1])
        d_path = torch.empty(int(TF.sum()), dtype=torch.int32, device=dev)
        d_poff = torch.from_numpy(poff).to(dev)
        d_plen = torch.zeros(plan.nseg, dtype=torch.int32, device=dev)
        out.update(path=d_path, path_off=poff, path_len=d_plen, path_order=plan.dtw_order)
    if want_status:
        d_status = torch.zeros(plan.nseg, dtype=torch.int32, device=dev)
        out.update(status=d_status, status_order=plan.dtw_order)
    rc = nat.lib.wts_dtw_batch_sized(nat.ptr(cost), 1 if cost.dtype == torch.float64 else 0, nat.ptr(d_segs),
                                     plan.nseg, nat.ptr(d_dir), nat.ptr(d_bnd), nat.ptr(jumps), nat.ptr(d_path),
                                     nat.ptr(d_poff), nat.ptr(d_plen), nat.ptr(d_status), plan.max_T, plan.max_F,
                                     int(np.bitwise_and.reduce(plan.segs["flags"])) if plan.nseg else 0,
                                     nat.stream_ptr(dev))
    nat.check(rc, "wts_dtw_batch_sized")
    return out


def disfluency_starts(cost: torch.Tensor, plan: AlignPlan, jumps: torch.Tensor, d_segs: torch.Tensor = None) -> torch.Tensor:
    """Per token: -1, or the offset from its jump at which the token really starts (detect_disfluencies,
    T.py:1656-1683).  Same layout as `jumps` (T+1 ints per segment, the last one unused)."""
    nat.require_cuda(cost, "cost")
    assert cost.dtype == torch.float32 and jumps.dtype == torch.int32
    if d_segs is None:
        d_segs = _segs_to_device(plan.segs, cost.device)
    out = torch.empty_like(jumps)
    rc = nat.lib.wts_disfluency_starts(nat.ptr(cost), nat.ptr(d_segs), plan.nseg, nat.ptr(jumps), nat.ptr(out),
                                       nat.stream_ptr(cost.device))
    nat.check(rc, "wts_disfluency_starts")
    return out


def split_jumps(jumps_host: np.ndarray, plan: AlignPlan):
    """Per-segment views of a host copy of the jumps buffer."""
    return [jumps_host[s["jumps_off"]: s["jumps_off"] + s["T"] + 1] for s in plan.segs]


def align(qk: torch.Tensor, items):
    """prep + DTW + one D2H copy.  Returns (list of jumps arrays, plan, cost buffer)."""
    plan = plan_segments(items, nonpositive=True)
    cost = attn_prep(qk, plan)
    out = dtw(cost, plan)
    jumps = out["jumps"].cpu().numpy()
    return split_jumps(jumps, plan), plan, cost

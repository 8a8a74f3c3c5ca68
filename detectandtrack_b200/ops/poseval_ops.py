"""Device-tensor API over csrc/poseval.cu: the PoseTrack evaluation's frame assignment, per-joint AP and CLEAR-MOT
counts (lib/datasets/posetrack/poseval/py/).  Inputs are the flat arrays of datasets.posetrack_eval.PoseTrackPack."""
import ctypes as C

import numpy as np

from .. import _lib as L


def _dev(torch, a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a)).to(device='cuda', dtype=dtype).contiguous()


class DevicePack(object):
    """The pack's arrays on the device (kept alive for the launches that read them)."""

    def __init__(self, pack):
        torch = L.require_cuda()
        self.F = pack.nframes
        self.gt_off = _dev(torch, pack.gt_off, torch.int32)
        self.pr_off = _dev(torch, pack.pr_off, torch.int32)
        self.pair_off = _dev(torch, pack.pair_off, torch.int64)
        self.gt_rect = _dev(torch, pack.gt_rect.reshape(-1, 4) if len(pack.gt_rect) else np.zeros((1, 4)), torch.float64)
        self.gt_kp = _dev(torch, pack.gt_kp if len(pack.gt_kp) else np.zeros((1, L.PT_JOINTS, 3)), torch.float64)
        self.gt_tid = _dev(torch, pack.gt_tid if len(pack.gt_tid) else np.zeros(1), torch.int32)
        self.pr_kp = _dev(torch, pack.pr_kp if len(pack.pr_kp) else np.zeros((1, L.PT_JOINTS, 4)), torch.float64)
        self.pr_tid = _dev(torch, pack.pr_tid if len(pack.pr_tid) else np.zeros(1), torch.int32)
        self.max_gt, self.max_pr = pack.max_gt, pack.max_pr
        self.npairs = int(pack.pair_off[-1]) if pack.nframes else 0


def assign(dp):
    """assignGTmulti for every frame -> (labels [NP, 15] int8, ngt [15, F] int32, dist [npairs, 15] fp64)."""
    torch = L.require_cuda()
    labels = torch.empty((max(dp.pr_kp.shape[0], 1), L.PT_JOINTS), dtype=torch.int8, device='cuda')
    ngt = torch.empty((L.PT_JOINTS, max(dp.F, 1)), dtype=torch.int32, device='cuda')
    dist = torch.empty((max(dp.npairs, 1), L.PT_JOINTS), dtype=torch.float64, device='cuda')
    L.call('dt_posetrack_assign', L.ptr(dp.gt_off), L.ptr(dp.pr_off), L.ptr(dp.pair_off), dp.F, L.ptr(dp.gt_rect),
           L.ptr(dp.gt_kp), L.ptr(dp.pr_kp), dp.max_gt, dp.max_pr, L.ptr(labels), L.ptr(ngt), L.ptr(dist), L.stream_ptr())
    return labels, ngt, dist


def average_precision(dp, labels, ngt, segs, seg_off):
    """computeRPC + VOCap of every segment (joint, first frame, end frame) -> cuda fp64 [nseg, 3] (AP, precision, recall)
    x 100.  seg_off [nseg + 1]: the segments' score counts, prefix-summed."""
    torch = L.require_cuda()
    segs = np.asarray(segs, np.int32).reshape(-1, 3)
    nseg, n = len(segs), int(seg_off[-1])
    out = torch.zeros((max(nseg, 1), 3), dtype=torch.float64, device='cuda')
    if nseg == 0:
        return out[:0]
    need = C.c_size_t(0)
    L.call('dt_posetrack_ap_workspace_bytes', n, C.byref(need))
    ws = torch.empty(max(need.value, 256), dtype=torch.uint8, device='cuda')
    d_segs, d_off = _dev(torch, segs, torch.int32), _dev(torch, seg_off, torch.int32)
    L.call('dt_posetrack_ap', L.ptr(dp.pr_kp), L.ptr(labels), L.ptr(ngt), dp.F, L.ptr(dp.pr_off), L.ptr(d_segs), L.ptr(d_off),
           nseg, n, L.ptr(out), L.ptr(ws), ws.numel(), L.stream_ptr())
    return out


def mot_counts(dp, dist, list_off, list_frames, map_cap):
    """MOTAccumulator.update over every frame list and joint -> (counts cuda int32 [nlists, 15, 4] = MATCH, SWITCH, FP,
    MISS; sumd cuda fp64 [nlists, 15]; status cuda int32 [nlists, 15], non-zero where a bound was exceeded)."""
    torch = L.require_cuda()
    nl = len(list_off) - 1
    counts = torch.zeros((max(nl, 1), L.PT_JOINTS, 4), dtype=torch.int32, device='cuda')
    sumd = torch.zeros((max(nl, 1), L.PT_JOINTS), dtype=torch.float64, device='cuda')
    status = torch.zeros((max(nl, 1), L.PT_JOINTS), dtype=torch.int32, device='cuda')
    if nl == 0:
        return counts[:0], sumd[:0], status[:0]
    d_off = _dev(torch, list_off, torch.int32)
    d_frames = _dev(torch, list_frames if len(list_frames) else np.zeros(1), torch.int32)
    L.call('dt_posetrack_mot', L.ptr(dp.gt_off), L.ptr(dp.pr_off), L.ptr(dp.pair_off), L.ptr(dp.gt_kp), L.ptr(dp.gt_tid),
           L.ptr(dp.pr_kp), L.ptr(dp.pr_tid), L.ptr(dist), L.ptr(d_off), L.ptr(d_frames), nl, dp.max_gt, dp.max_pr,
           int(map_cap), L.ptr(counts), L.ptr(sumd), L.ptr(status), L.stream_ptr())
    return counts, sumd, status


def upper_bound(dp, dist):
    """The upper-bound view of the predictions (assignGTmulti with computeUpperBound) -> a DevicePack-like object whose
    pr_off / pair_off / pr_kp / pr_tid are the view's, plus dist (its distances)."""
    torch = L.require_cuda()
    n = max(dp.pr_kp.shape[0], 1)
    v = DevicePack.__new__(DevicePack)
    v.__dict__.update(dp.__dict__)
    v.pr_off = torch.empty((dp.F + 1,), dtype=torch.int32, device='cuda')
    v.pair_off = torch.empty((dp.F + 1,), dtype=torch.int64, device='cuda')
    v.pr_kp = torch.zeros((n, L.PT_JOINTS, 4), dtype=torch.float64, device='cuda')
    v.pr_tid = torch.full((n,), -1, dtype=torch.int32, device='cuda')
    v.dist = torch.empty_like(dist)
    L.call('dt_posetrack_upper_bound', L.ptr(dp.gt_off), L.ptr(dp.pr_off), L.ptr(dp.pair_off), dp.F, L.ptr(dp.gt_kp),
           L.ptr(dp.gt_tid), L.ptr(dp.pr_kp), L.ptr(dp.pr_tid), L.ptr(dist), dp.max_gt, dp.max_pr, L.ptr(v.pr_off),
           L.ptr(v.pair_off), L.ptr(v.pr_kp), L.ptr(v.pr_tid), L.ptr(v.dist), L.stream_ptr())
    return v

"""Device-tensor API over the box / NMS / assignment kernels (torch tensors are
only the memory container; arithmetic is in csrc/boxes.cu and csrc/lsa.cu)."""
import ctypes as C

from .. import _lib as L

NMS_2D_GE, NMS_TUBE_GT = 0, 1
ORDER_SCORE, ORDER_INDEX = 0, 1
MAX_TRACK_IDS = 999   # lib/core/tracking_engine.py:45
FIRST_TRACK_ID = 0    # lib/core/tracking_engine.py:46


def _f32c(t, torch):
    return t.to(device='cuda', dtype=torch.float32).contiguous()


def bbox_overlaps(boxes, query, T=None):
    """lib/utils/boxes.py:60-69.  boxes [N, >=4T], query [K, >=4T] cuda fp32 -> [N, K]."""
    torch = L.require_cuda()
    boxes, query = _f32c(boxes, torch), _f32c(query, torch)
    if T is None:
        T = boxes.shape[1] // 4
    n, k = boxes.shape[0], query.shape[0]
    out = torch.empty((n, k), dtype=torch.float32, device='cuda')
    L.call('dt_bbox_overlaps', L.ptr(boxes), n, boxes.shape[1], L.ptr(query), k, query.shape[1],
           T, L.ptr(out), max(k, 1), L.stream_ptr())
    return out


def _workspace(nbytes, torch, slot='nms'):
    """Scratch buffer of a call.  Allocated per call (the caching allocator makes that free): a process-wide cached
    buffer that is re-allocated when a later call needs more would be freed under a previously CAPTURED CUDA graph
    that still points at it (two ClipPipelines of different batch sizes) — under capture the allocation comes from
    that graph's own pool and lives as long as the graph."""
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device='cuda')


def nms_batched(dets, counts=None, thresh=0.5, cmp_mode=None, out_order=None, max_keep=0):
    """dets [B, Nmax, 4T+1] cuda fp32, counts [B] int32 (or None).
    Returns (keep [B, Nmax] int32, num_keep [B] int32).  cmp_mode/out_order default to the
    reference's dispatch (nms_wrapper.py:49-57): T == 1 -> '>=' + index order, else tube."""
    torch = L.require_cuda()
    dets = _f32c(dets, torch)
    B, nmax, ld = dets.shape
    T = (ld - 1) // 4
    if cmp_mode is None:
        cmp_mode = NMS_2D_GE if T == 1 else NMS_TUBE_GT
    if out_order is None:
        out_order = ORDER_INDEX if cmp_mode == NMS_2D_GE else ORDER_SCORE
    keep = torch.empty((B, max(nmax, 1)), dtype=torch.int32, device='cuda')
    num = L.zeros((B,), torch.int32)
    if counts is not None:
        counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    need = C.c_size_t(0)
    L.call('dt_nms_workspace_bytes', B, nmax, C.byref(need))
    ws = _workspace(need.value, torch)
    L.call('dt_nms_batched', L.ptr(dets), B, nmax, ld, T, L.ptr(counts), float(thresh), cmp_mode,
           out_order, int(max_keep), L.ptr(keep), L.ptr(num), L.ptr(ws), ws.numel(), L.stream_ptr())
    return keep, num


def soft_nms_batched(dets, counts=None, sigma=0.5, overlap_thresh=0.3, score_thresh=0.001, method='linear'):
    """lib/core/nms_wrapper.py:29-46 soft_nms per list: dets [B, Nmax, >=5] cuda fp32 (2-D boxes + score), counts [B]
    int32 (or None).  Returns (rows [B, Nmax, 5], inds [B, Nmax] int32 source rows, counts [B] int32)."""
    torch = L.require_cuda()
    if method not in L.SOFT_NMS_METHODS:
        raise ValueError('Unknown soft_nms method: {}'.format(method))
    dets = _f32c(dets, torch)
    B, nmax, ld = dets.shape
    out = torch.empty((B, max(nmax, 1), 5), dtype=torch.float32, device='cuda')
    inds = torch.empty((B, max(nmax, 1)), dtype=torch.int32, device='cuda')
    num = L.zeros((B,), torch.int32)
    if counts is not None:
        counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    L.call('dt_soft_nms_batched', L.ptr(dets), B, nmax, ld, L.ptr(counts), float(sigma), float(overlap_thresh),
           float(score_thresh), L.SOFT_NMS_METHODS[method], L.ptr(out), L.ptr(inds), L.ptr(num), L.stream_ptr())
    return out, inds, num


def box_vote(all_dets, all_counts, thresh, top=None, top_counts=None, keep=None, nkeep=None):
    """lib/utils/boxes.py:294-310 box_voting per list: the top rows voted against all_dets [B, Nmax, >=5] (counts
    all_counts [B] or None).  Top rows: keep [B, Nmax] / nkeep [B] (nms_batched's output, rows of all_dets), or
    top [B, Ntop, >=5] / top_counts [B] (soft_nms_batched's output).  Returns (rows [B, Ntop, 5], counts [B] int32)."""
    torch = L.require_cuda()
    all_dets = _f32c(all_dets, torch)
    B, nmax, ld = all_dets.shape
    if keep is not None:
        keep, top_counts, ntop, ld_top = keep.contiguous(), nkeep, nmax, 0
    else:
        top = _f32c(top, torch)
        ntop, ld_top = top.shape[1], top.shape[2]
    out = torch.empty((B, max(ntop, 1), 5), dtype=torch.float32, device='cuda')
    num = L.zeros((B,), torch.int32)
    L.call('dt_box_vote', L.ptr(top), L.ptr(keep), L.ptr(top_counts.contiguous()), ntop, ld_top, L.ptr(all_dets),
           L.ptr(all_counts), B, nmax, ld, float(thresh), L.ptr(out), L.ptr(num), L.stream_ptr())
    return out, num


ALGOS ={'hungarian': 0, 'greedy': 1}


def lsa_batched(cost, nrows, ncols, algo='hungarian'):
    """cost [B, D, D'] cuda (rows prev, cols cur): fp64 costs are solved in fp64 (dt_lsa_batched_f64), anything else as
    fp32.  Returns (matches [B, dmax] int32, status [B] int32: 1 = infeasible or, for hungarian, a NaN / -inf entry)."""
    torch = L.require_cuda()
    f64 = cost.dtype == torch.float64
    cost = cost.to(device='cuda').contiguous() if f64 else _f32c(cost, torch)
    B, P, Q = cost.shape
    dmax = max(P, Q)
    if P != dmax or Q != dmax:
        pad = torch.zeros((B, dmax, dmax), dtype=cost.dtype, device='cuda')
        pad[:, :P, :Q] = cost
        cost = pad
    nrows = nrows.to(device='cuda', dtype=torch.int32).contiguous()
    ncols = ncols.to(device='cuda', dtype=torch.int32).contiguous()
    matches = torch.empty((B, dmax), dtype=torch.int32, device='cuda')
    status = torch.empty((B,), dtype=torch.int32, device='cuda')
    L.call('dt_lsa_batched_f64' if f64 else 'dt_lsa_batched', L.ptr(cost), B, dmax, dmax, L.ptr(nrows), L.ptr(ncols),
           ALGOS[algo], L.ptr(matches), L.ptr(status), L.stream_ptr())
    return matches, status


def match_frames(frames, counts, is_start=None, T=1, weight=1.0, algo='hungarian'):
    """frames [F, Dmax, ld] cuda fp32, counts [F] int32 -> matches [F, Dmax] int32."""
    torch = L.require_cuda()
    frames = _f32c(frames, torch)
    F, dmax, ld = frames.shape
    counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    if is_start is not None:
        is_start = is_start.to(device='cuda', dtype=torch.uint8).contiguous()
    matches = torch.empty((F, dmax), dtype=torch.int32, device='cuda')
    status = torch.empty((F,), dtype=torch.int32, device='cuda')
    L.call('dt_match_frames', L.ptr(frames), F, dmax, ld, T, L.ptr(counts), L.ptr(is_start), float(weight), ALGOS[algo],
           L.ptr(matches), L.ptr(status), L.stream_ptr())
    return matches, status


def pose_pck_cost(a, b, head_top, head_bottom, dist_thresh=0.5):
    """a [P, 4|3, K], b [Q, 4|3, K] fp32 poses -> [P, Q] fp64 'pose-pck' cost (tracking_engine.py:113-129)."""
    torch = L.require_cuda()
    a, b = _f32c(a, torch), _f32c(b, torch)
    P, _, K = a.shape
    Q = b.shape[0]
    out = torch.empty((P, Q), dtype=torch.float64, device='cuda')
    L.call('dt_pose_pck_cost', L.ptr(a), P, L.ptr(b), Q, a.shape[1] * K, K, int(head_top), int(head_bottom), float(dist_thresh),
           L.ptr(out), L.stream_ptr())
    return out


def frame_costs(boxes, counts, is_start, poses=None, T=1, w_iou=1.0, w_pck=0.0, head_top=2, head_bottom=1, dist_thresh=0.5):
    """boxes [F, Dmax, ld], poses [F, Dmax, 4|3, K] (or None) -> cost [F, Dmax, Dmax] fp64 (rows = previous frame)."""
    torch = L.require_cuda()
    boxes = _f32c(boxes, torch)
    F, dmax, ld = boxes.shape
    counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    if is_start is not None:
        is_start = is_start.to(device='cuda', dtype=torch.uint8).contiguous()
    K = ldp = 0
    if poses is not None:
        poses = _f32c(poses, torch)
        K, ldp = poses.shape[3], poses.shape[2] * poses.shape[3]
    cost = torch.empty((F, dmax, dmax), dtype=torch.float64, device='cuda')
    L.call('dt_frame_costs', L.ptr(boxes), ld, T, L.ptr(poses), ldp, K, int(head_top), int(head_bottom), float(dist_thresh),
           L.ptr(counts), L.ptr(is_start), F, dmax, float(w_iou), float(w_pck), L.ptr(cost), L.stream_ptr())
    return cost


def assign_track_ids(matches, counts, video_first, is_start=None,
                     first_id=FIRST_TRACK_ID, max_ids=MAX_TRACK_IDS):
    torch = L.require_cuda()
    F, dmax = matches.shape
    counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    video_first = video_first.to(device='cuda', dtype=torch.int32).contiguous()
    tracks = torch.empty((F, dmax), dtype=torch.int32, device='cuda')
    L.call('dt_assign_track_ids', L.ptr(matches.contiguous()), L.ptr(counts), L.ptr(is_start), F, dmax,
           L.ptr(video_first), video_first.numel(), first_id, max_ids, L.ptr(tracks), L.stream_ptr())
    return tracks


def prune_detections(boxes, counts, hw, conf, T=1, center_only=True, min_area=50.0):
    """boxes [F, Dmax, 4T+1]; hw [F, 2] (height, width).  Returns (out, counts_out, sel)."""
    torch = L.require_cuda()
    boxes = _f32c(boxes, torch)
    F, dmax, ld = boxes.shape
    counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    hw = _f32c(hw, torch)
    T_out = 1 if center_only else T
    out = torch.zeros((F, dmax, 4 * T_out + 1), dtype=torch.float32, device='cuda')
    counts_out = torch.empty((F,), dtype=torch.int32, device='cuda')
    sel = torch.full((F, dmax), -1, dtype=torch.int32, device='cuda')
    L.call('dt_prune_detections', L.ptr(boxes), F, dmax, ld, T, int(bool(center_only)), L.ptr(counts), L.ptr(hw),
           float(conf), float(min_area), L.ptr(out), L.ptr(counts_out), L.ptr(sel), L.stream_ptr())
    return out, counts_out, sel


def gt_frame_costs(boxes, counts, poses=None, T=1, w_iou=1.0, w_pck=0.0, head_top=2, head_bottom=1, dist_thresh=0.5):
    """boxes [2F, Dmax, ld], poses [2F, Dmax, R, K] (or None): the GT of frame f at entry 2f, its detections at 2f + 1 ->
    cost [F, Dmax, Dmax] fp64, rows = GT (tracking_engine.py:287-296 with the frame's GT as the previous frame)."""
    torch = L.require_cuda()
    boxes = _f32c(boxes, torch)
    F2, dmax, ld = boxes.shape
    counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    R = K = 0
    if poses is not None:
        poses = _f32c(poses, torch)
        R, K = poses.shape[2], poses.shape[3]
    cost = torch.empty((F2 // 2, dmax, dmax), dtype=torch.float64, device='cuda')
    L.call('dt_gt_frame_costs', L.ptr(boxes), ld, T, L.ptr(poses), R, K, int(head_top), int(head_bottom), float(dist_thresh),
           L.ptr(counts), F2 // 2, dmax, float(w_iou), float(w_pck), L.ptr(cost), L.stream_ptr())
    return cost


def _rows_arg(m, F, dmax):
    """An int32 matches tensor as (pointer, row stride): [F, ld] as it is, or the detection rows of an interleaved [2F, dmax]."""
    if m is None:
        return None, 0
    assert m.dtype.is_floating_point is False and m.is_contiguous()
    if m.shape[0] == 2 * F:
        return C.c_void_p(m.data_ptr() + dmax * m.element_size()), 2 * m.shape[1]
    assert m.shape[0] == F
    return L.ptr(m), m.shape[1]


def track_upper_bound(boxes, poses, counts, gt_tid, matches=None, matches_gt=None, flags=0):
    """TRACKING.DEBUG.UPPER_BOUND* on the interleaved packing of gt_frame_costs: boxes [2F, Dmax, ld], poses [2F, Dmax, R, K],
    counts [2F], gt_tid [F, Dmax]; matches / matches_gt [F, ld] or the interleaved [2F, Dmax] output of match_frames.
    Returns (boxes [F, Dmax, ld], poses [F, Dmax, R, K], track ids [F, Dmax], counts [F])."""
    torch = L.require_cuda()
    boxes, poses = _f32c(boxes, torch), _f32c(poses, torch)
    F2, dmax, ld = boxes.shape
    F, R, K = F2 // 2, poses.shape[2], poses.shape[3]
    counts = counts.to(device='cuda', dtype=torch.int32).contiguous()
    gt_tid = gt_tid.to(device='cuda', dtype=torch.int32).contiguous()
    out_b = torch.empty((F, dmax, ld), dtype=torch.float32, device='cuda')
    out_p = torch.empty((F, dmax, R, K), dtype=torch.float32, device='cuda')
    out_t = torch.empty((F, dmax), dtype=torch.int32, device='cuda')
    out_n = torch.empty((F,), dtype=torch.int32, device='cuda')
    m, ldm = _rows_arg(matches, F, dmax)
    mg, ldmg = _rows_arg(matches_gt, F, dmax)
    L.call('dt_track_upper_bound', L.ptr(boxes), ld, L.ptr(poses), R, K, L.ptr(counts), L.ptr(gt_tid), F, dmax, m, ldm, mg, ldmg,
           int(flags), L.ptr(out_b), L.ptr(out_p), L.ptr(out_t), L.ptr(out_n), L.stream_ptr())
    return out_b, out_p, out_t, out_n

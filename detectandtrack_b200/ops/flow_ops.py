"""Device-tensor API over csrc/flow.cu: Farneback flow between key frames and the flow-smoothed poses of
TRACKING.FLOW_SMOOTHING_ON (lib/core/tracking_engine.py:401-643)."""
import ctypes as C

from .. import _lib as L


def bgr_to_gray(frames):
    """cv2.cvtColor(BGR2GRAY) of cuda uint8 [..., 3] frames -> uint8 [...], bit for bit."""
    torch = L.require_cuda()
    frames = frames.to(device='cuda', dtype=torch.uint8).contiguous()
    assert frames.shape[-1] == 3, 'frames must be [..., 3] BGR'
    out = torch.empty(frames.shape[:-1], dtype=torch.uint8, device='cuda')
    L.call('dt_bgr_to_gray', L.ptr(frames), out.numel(), L.ptr(out), L.stream_ptr())
    return out


def farneback_flow(frames, pairs, pyr_scale=0.5, levels=10, winsize=None, iterations=10, poly_n=7, poly_sigma=1.5,
                   flags=L.FARNEBACK_GAUSSIAN):
    """cv2.calcOpticalFlowFarneback(gray[a], gray[b], None, pyr_scale, levels, winsize, iterations, poly_n, poly_sigma,
    flags) for every pair (a, b): frames cuda uint8 [N, H, W, 3] BGR, pairs [P, 2] frame indices.  winsize None: the
    tracking engine's min(H, W) // 5 (tracking_engine.py:557).  Returns flows [P, H, W, 2] fp32."""
    torch = L.require_cuda()
    frames = frames.to(device='cuda', dtype=torch.uint8).contiguous()
    N, H, W, ch = frames.shape
    assert ch == 3, 'frames must be [N, H, W, 3] BGR'
    pairs = torch.as_tensor(pairs, dtype=torch.int32).reshape(-1, 2)
    if len(pairs) and (int(pairs.min()) < 0 or int(pairs.max()) >= N):
        raise ValueError('pair indices outside [0, %d)' % N)
    P = pairs.shape[0]
    if winsize is None:
        winsize = min(H, W) // 5
    flows = torch.empty((P, H, W, 2), dtype=torch.float32, device='cuda')
    need = C.c_size_t(0)
    L.call('dt_farneback_workspace_bytes', H, W, N, P, C.byref(need))
    ws = torch.empty(max(need.value, 256), dtype=torch.uint8, device='cuda')
    d_pairs = pairs.to('cuda').contiguous()
    L.call('dt_farneback_flow', L.ptr(frames), N, H, W, L.ptr(d_pairs), P, float(pyr_scale), int(levels), int(winsize),
           int(iterations), int(poly_n), float(poly_sigma), int(flags), L.ptr(flows), L.ptr(ws), ws.numel(), L.stream_ptr())
    return flows


def flow_mean_abs(flows):
    """np.abs(flow).mean() of each flow of cuda fp32 [P, H, W, 2], bit for bit -> [P] fp32."""
    torch = L.require_cuda()
    assert flows.dtype == torch.float32 and flows.dim() == 4 and flows.shape[3] == 2, 'flows must be fp32 [P, H, W, 2]'
    flows = flows.contiguous()
    P, H, W, _ = flows.shape
    out = torch.empty((P,), dtype=torch.float32, device='cuda')
    L.call('dt_flow_mean_abs', L.ptr(flows), P, H, W, L.ptr(out), L.stream_ptr())
    return out


def smooth_poses(poses, boxes, counts, tracks, is_start, flows, no_flow, n_context, out_tracks, out_counts):
    """_shift_poses + _combine_shifted_poses (tracking_engine.py:401-546), bit for bit, for the packed frames of
    one or more videos: poses [F, Dmax, 4, K], boxes [F, Dmax, 5], counts [F], tracks [F, Dmax], is_start [F];
    flows: F cuda fp32 [H, W, 2] tensors (frame f -> f + 1) or None; no_flow [F]: the pair moves nothing;
    out_tracks [F, Omax] / out_counts [F]: the output track order of every frame.
    Returns (poses [F, Omax, 4, K], boxes [F, Omax, 5]) fp32."""
    torch = L.require_cuda()
    if not 0 <= n_context <= L.FLOW_MAX_CONTEXT:
        raise NotImplementedError('N_CONTEXT_FRAMES=%d outside [0, %d]' % (n_context, L.FLOW_MAX_CONTEXT))
    dev = lambda t, dt: torch.as_tensor(t).to(device='cuda', dtype=dt).contiguous()
    poses, boxes = dev(poses, torch.float32), dev(boxes, torch.float32)
    F, dmax, rows, K = poses.shape
    assert rows == 4 and boxes.shape == (F, dmax, 5), 'poses [F, Dmax, 4, K] and boxes [F, Dmax, 5] (T = 1)'
    out_tracks = dev(out_tracks, torch.int32)
    omax = max(out_tracks.shape[1], 1)
    if out_tracks.shape[1] == 0:
        out_tracks = torch.zeros((F, 1), dtype=torch.int32, device='cuda')
    assert len(flows) == F, 'one flow (or None) per frame'
    ptrs = torch.tensor([0 if f is None else f.data_ptr() for f in flows], dtype=torch.int64).cuda()
    hw = torch.tensor([[0, 0] if f is None else list(f.shape[:2]) for f in flows], dtype=torch.int32).reshape(F, 2).cuda()
    for f in flows:
        assert f is None or (f.is_cuda and f.dtype == torch.float32 and f.dim() == 3 and f.shape[2] == 2 and f.is_contiguous())
    # every device input is bound to a name: a temporary would be freed (and its block reused) before the launch
    no_flow = dev(no_flow, torch.uint8)
    counts, tracks = dev(counts, torch.int32), dev(tracks, torch.int32)
    is_start, out_counts = dev(is_start, torch.uint8), dev(out_counts, torch.int32)
    out_poses = torch.empty((F, omax, 4, K), dtype=torch.float32, device='cuda')
    out_boxes = torch.empty((F, omax, 5), dtype=torch.float32, device='cuda')
    L.call('dt_flow_smooth_poses', L.ptr(poses), L.ptr(boxes), L.ptr(counts), L.ptr(tracks), L.ptr(is_start), F, dmax, K,
           L.ptr(ptrs), L.ptr(hw), L.ptr(no_flow), int(n_context), L.ptr(out_tracks), L.ptr(out_counts), omax,
           L.ptr(out_poses), L.ptr(out_boxes), L.stream_ptr())
    return out_poses, out_boxes

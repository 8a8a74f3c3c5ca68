"""Per-clip inference entry points with the reference's signature and return containers
(lib/core/test.py:897-958): ``im_detect_all(model, im, box_proposals, timers)``.

``im`` is the reference's list of T BGR uint8 frames (HxWx3).  Everything between the H2D copy
of the frames and the D2H copy of the (<=100) detections runs on the device
(modeling/engine.py) as ONE captured CUDA graph per batch geometry; with TEST.COMPETITION_MODE that graph runs every
test-time view of core/tta.view_plan and merges them on the device.

``ClipPipeline`` is that device step behind the reference's per-clip containers: B clips per graph
replay, frames staged through pinned host buffers filled by loader threads, the upload of step i+1
and the conversion of step i-1's results overlapping the compute of step i.  ``im_detect_all`` is its
1-clip synchronous form (same signature and return value as the reference);
``test_engine.test_net`` drives the B-clip form (cfg.TEST.CLIPS_PER_STEP)."""
from collections import defaultdict, deque, OrderedDict
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import tta
from .config import cfg
from ..utils.timer import Timer

_MAX_PIPELINES = 4          # captured graphs kept per model (each owns its activation pool)


class ClipPipeline(object):
    """B clips of T frames (H x W x 3 uint8, BGR) per captured device step.

    run(n, fill, on_result): ``fill(i, dst)`` writes clip i into the pinned [T, H, W, 3] view ``dst`` (called on a
    loader thread, ahead of time); ``on_result(i, cls_boxes, cls_segms, cls_keyps)`` receives the reference's
    per-clip containers (lib/core/test.py:897-958) in index order.  A short last batch is padded with its last
    clip and the padding results are dropped.
    run(..., fill_device=f): ``f(i, dev_dst, stream)`` instead produces clip i DIRECTLY in the device view ``dev_dst``
    [T, H, W, 3] with GPU work on ``stream`` (device-side JPEG decode, ops/image_ops.jpeg_decode): no pinned staging, only
    the compressed bytes cross PCIe."""

    def __init__(self, model, B, T, H, W, depth=2, loader_threads=2, plan=None):
        eng = model.engine
        torch = eng.torch
        self.torch, self.eng, self.B, self.T, self.H, self.W, self.depth = torch, eng, B, T, H, W, depth
        self.num_classes = eng.spec.num_classes
        self.static_in, self.replay = eng.capture(B, T, H, W, plan=plan)
        out = self.replay()
        torch.cuda.synchronize()
        self.cap = out['dets'].shape[2]
        self.has_kps = out['xy'] is not None
        pin = lambda t: torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
        self.host_in = [torch.empty((B, T, H, W, 3), dtype=torch.uint8, pin_memory=True) for _ in range(depth)]
        self.np_in = [h.numpy() for h in self.host_in]
        self.dev_in = [torch.empty_like(self.static_in) for _ in range(depth)]
        self.host_out = [dict(dets=pin(out['dets']), cnt=pin(out['det_counts']), xy=pin(out['xy']) if self.has_kps else None)
                         for _ in range(depth)]
        self.copy_stream = torch.cuda.Stream()
        self.device = torch.cuda.current_device()
        self.loader_streams = [torch.cuda.Stream() for _ in range(depth)]      # device-side producers (fill_device) of a slot
        self.dev_ready = [torch.cuda.Event() for _ in range(depth)]
        self.h2d_done = [torch.cuda.Event() for _ in range(depth)]
        self.consumed = [torch.cuda.Event() for _ in range(depth)]
        self.out_done = [torch.cuda.Event() for _ in range(depth)]
        self.pool = ThreadPoolExecutor(max_workers=max(1, loader_threads))
        self.pre_step = None          # optional callable enqueued before each step (bench.py: L2 flush between iterations)
        self.h2d_bytes = int(self.host_in[0].numel())
        self.d2h_bytes = sum(int(v.numel() * v.element_size()) for v in self.host_out[0].values() if v is not None)

    # ---- one device step ---------------------------------------------------------------------------
    def _enqueue(self, slot, from_device=False):
        torch = self.torch
        cur = torch.cuda.current_stream()
        if from_device:                                                   # dev_in[slot] was produced on the loader stream
            cur.wait_event(self.dev_ready[slot])
        else:
            with torch.cuda.stream(self.copy_stream):
                self.copy_stream.wait_event(self.consumed[slot])            # the step that last read dev_in[slot] is past it
                self.dev_in[slot].copy_(self.host_in[slot], non_blocking=True)
                self.h2d_done[slot].record(self.copy_stream)
            cur.wait_event(self.h2d_done[slot])
        if self.pre_step is not None:
            self.pre_step()
        self.static_in.copy_(self.dev_in[slot], non_blocking=True)
        self.consumed[slot].record(cur)
        out = self.replay()
        ho = self.host_out[slot]
        ho['dets'].copy_(out['dets'], non_blocking=True)
        ho['cnt'].copy_(out['det_counts'], non_blocking=True)
        if self.has_kps:
            ho['xy'].copy_(out['xy'], non_blocking=True)
        self.out_done[slot].record(cur)

    def _results(self, slot, nvalid):
        """Pinned outputs of a finished step -> per-clip (cls_boxes, cls_segms, cls_keyps) for its first nvalid clips."""
        self.out_done[slot].synchronize()
        ho = self.host_out[slot]
        C, cap = self.num_classes, self.cap
        cnt = ho['cnt'].numpy().reshape(self.B, C - 1)
        dets = ho['dets'].numpy()
        xy = ho['xy'].numpy() if self.has_kps else None
        res = []
        for b in range(nvalid):
            if cnt[b].max() > cap:
                raise RuntimeError('more than %d detections tie at the DETECTIONS_PER_IM threshold (%s)' % (cap, cnt[b]))
            cls_boxes = [[] for _ in range(C)]
            for j in range(1, C):
                cls_boxes[j] = dets[b, j - 1, :cnt[b, j - 1]].copy()
            cls_keyps = None
            n1 = int(cnt[b, 0])
            if self.has_kps and n1 > 0:
                k = xy[b * cap:b * cap + n1].copy()
                cls_keyps = [[] for _ in range(C)]
                cls_keyps[1] = [k[i] for i in range(n1)]
            res.append((cls_boxes, None, cls_keyps))
        return res

    # ---- public ------------------------------------------------------------------------------------
    def detect_one(self, im):
        """Synchronous single step on a 1-clip pipeline: the body of im_detect_all."""
        assert self.B == 1 and len(im) == self.T
        dst = self.np_in[0][0]
        for t in range(self.T):
            np.copyto(dst[t], im[t])
        self._enqueue(0)
        return self._results(0, 1)[0]

    def run(self, n, fill, on_result, fill_device=None):
        B, depth = self.B, self.depth
        if n <= 0:
            return
        nsteps = (n + B - 1) // B
        torch = self.torch

        def load(step):
            slot = step % depth
            if fill_device is None:
                dst = self.np_in[slot]
                for j in range(B):
                    fill(min(step * B + j, n - 1), dst[j])
                return
            torch.cuda.set_device(self.device)                         # loader threads start on device 0
            st = self.loader_streams[slot]
            st.wait_event(self.consumed[slot])                         # the step that last read dev_in[slot] is past it
            for j in range(B):
                fill_device(min(step * B + j, n - 1), self.dev_in[slot][j], st)
            self.dev_ready[slot].record(st)

        fut = {s: self.pool.submit(load, s) for s in range(min(depth, nsteps))}
        pending = deque()
        for step in range(nsteps):
            slot = step % depth
            fut.pop(step).result()
            self._enqueue(slot, from_device=fill_device is not None)
            pending.append((step, slot))
            if len(pending) > 1:                               # results of the previous step while this one computes
                self._emit(pending.popleft(), n, on_result)
            if step + depth < nsteps:
                if fill_device is None:
                    self.h2d_done[slot].synchronize()          # pinned buffer read out: the loader may refill it
                fut[step + depth] = self.pool.submit(load, step + depth)   # (device path: ordered by the consumed[slot] event)
        while pending:
            self._emit(pending.popleft(), n, on_result)

    def _emit(self, item, n, on_result):
        step, slot = item
        first = step * self.B
        for j, r in enumerate(self._results(slot, min(self.B, n - first))):
            on_result(first + j, *r)


def get_pipeline(model, B, T, H, W):
    """The model's captured pipeline for a batch geometry (built on first use, a few kept).  With TEST.COMPETITION_MODE
    its step runs the test-time views of core/tta.view_plan, which rejects what the device path does not run before
    anything is built."""
    plan = tta.view_plan(cfg, model.engine.spec, H, W) if cfg.TEST.COMPETITION_MODE else None
    cache = model.__dict__.setdefault('_pipelines', OrderedDict())
    key = (B, T, H, W, plan)
    p = cache.get(key)
    if p is None:
        while len(cache) >= _MAX_PIPELINES:
            cache.popitem(last=False)
        p = cache[key] = ClipPipeline(model, B, T, H, W, plan=plan)
    else:
        cache.move_to_end(key)
    return p


def _check_hot_path(box_proposals):
    if box_proposals is not None:
        raise NotImplementedError('precomputed proposals are not on the hot path (FASTER_RCNN models only)')


def im_detect_all(model, im, box_proposals=None, timers=None):
    if timers is None:
        timers = defaultdict(Timer)
    _check_hot_path(box_proposals)
    if not isinstance(im, (list, tuple)):
        im = [im]
    T = cfg.VIDEO.NUM_FRAMES if cfg.MODEL.VIDEO_ON else 1
    assert len(im) == T, 'expected {} frames, got {}'.format(T, len(im))
    timers['im_detect_bbox'].tic()
    H, W = im[0].shape[:2]
    cls_boxes, cls_segms, cls_keyps = get_pipeline(model, 1, T, H, W).detect_one(im)
    timers['im_detect_bbox'].toc()
    return cls_boxes, cls_segms, cls_keyps


def im_detect_all_batch(model, ims, clips_per_step=None):
    """ims: list of clips (each the reference's list of T frames, one geometry) -> list of
    (cls_boxes, cls_segms, cls_keyps), through the batched captured step."""
    _check_hot_path(None)
    if not ims:
        return []
    T = cfg.VIDEO.NUM_FRAMES if cfg.MODEL.VIDEO_ON else 1
    H, W = ims[0][0].shape[:2]
    B = int(clips_per_step or cfg.TEST.CLIPS_PER_STEP)
    pipe = get_pipeline(model, B, T, H, W)
    out = [None] * len(ims)

    def fill(i, dst):
        for t in range(T):
            np.copyto(dst[t], ims[i][t])

    def on_result(i, *r):
        out[i] = r
    pipe.run(len(ims), fill, on_result)
    return out

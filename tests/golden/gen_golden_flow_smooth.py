"""Golden vectors for TRACKING.FLOW_SMOOTHING_ON, from the REFERENCE's own _smooth_pose_video.

    python tests/golden/gen_golden_flow_smooth.py      -> tests/golden/flow_smooth.npz

What runs, from the reference's lib/core/tracking_engine.py source text (the module imports Caffe2-era code):
    _get_boxes/_get_poses/_set_poses/_set_boxes (:70-84), _shift_using_flow ... _combine_shifted_poses (:401-546),
    _compute_neg_flow (:567-570), _smooth_pose_video (:600-643).
Shims: cfg is a plain namespace with the TRACKING.FLOW_SMOOTHING keys; ``zip`` returns a list (py2); and
compute_optical_flow returns the supplied pair flows laid out as :589-597 lays out cv2's (zeros for the last forward and
the first backward flow, _compute_neg_flow of every pair, None where cv2 would have raised).

Case c<k> (one video): inputs poses [F, Dmax, 4, 17], boxes [F, Dmax, 5], counts [F], tracks [F, Dmax], pair flows
flow<q> [H, W, 2] fp32 (absent for a None pair: flow_none[q] = 1), params (N_CONTEXT_FRAMES, EXTEND_TRACKS,
FLOW_SHOT_BOUNDARY_TH); outputs out_poses [F, Omax, 4, 17], out_boxes [F, Omax, 5], out_counts [F], out_tracks
[F, Omax], out_box_f64 [F] (1 where the frame's boxes came back as the reference's fp64 np.zeros((0, 5))).
"""
import copy
import os
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/lib/core/tracking_engine.py'
F32 = np.float32
K = 17


def _reference(n_context, extend, th):
    src = open(REF).read().split('\n')
    cfg = types.SimpleNamespace(TRACKING=types.SimpleNamespace(
        FLOW_SMOOTHING=types.SimpleNamespace(N_CONTEXT_FRAMES=n_context, EXTEND_TRACKS=extend, FLOW_SHOT_BOUNDARY_TH=th),
        DEBUG=types.SimpleNamespace(FLOW_SMOOTHING_COMBINE=False)))
    ns = {'np': np, 'copy': copy, 'cfg': cfg, 'zip': lambda *a: list(zip(*a))}
    for a, b in ((69, 84), (400, 546), (566, 570), (599, 643)):
        exec('\n'.join(src[a:b]), ns)
    return ns


def _video(rng, F, H, W, ids_pool, empty=(), dup_frame=None):
    poses, boxes, tracks = [], [], []
    for f in range(F):
        n = 0 if f in empty else int(rng.randint(1, min(6, len(ids_pool) + 1)))
        ids = list(rng.choice(ids_pool, n, replace=False))
        if f == dup_frame and n >= 2:
            ids[1] = ids[0]
        p = np.stack([rng.uniform(-6, W + 6, (n, K)) + 0.25, rng.uniform(-6, H + 6, (n, K)) + 0.25,
                      rng.normal(1, 2, (n, K)), rng.uniform(0, 1, (n, K))], 1).astype(F32)
        p[:, 0] = np.floor(p[:, 0]) + F32(0.25)
        p[:, 1] = np.floor(p[:, 1]) + F32(0.25)
        if n:
            p[0, 2, :3] = -np.inf
            p[-1, 2, 5] = F32(0.0)
        x1 = rng.uniform(0, W / 2, n); y1 = rng.uniform(0, H / 2, n)
        b = np.stack([x1, y1, x1 + rng.uniform(2, W / 2, n), y1 + rng.uniform(2, H / 2, n), rng.uniform(0, 1, n)], 1)
        poses.append([p[i] for i in range(n)])
        boxes.append(b.astype(F32).reshape(n, 5))
        tracks.append([int(i) for i in ids])
    return poses, boxes, tracks


def _flows(rng, F, H, W, boundary=(), none=()):
    out = []
    for q in range(F - 1):
        if q in none:
            out.append(None)
            continue
        f = (rng.normal(0, 1.2, (H, W, 2)) + rng.uniform(-2, 2, 2)).astype(F32)
        if q in boundary:
            f *= F32(9)
        out.append(f)
    return out


def cases():
    rng = np.random.RandomState(20261016)
    vids = []
    pool = np.array([0, 1, 2, 3, 5, 8, 9, 64, 65, 70, 72, 130, 200, 257, 999])        # >= 64: set order != sorted order
    vids.append(_video(rng, 8, 12, 16, pool, empty=(3,), dup_frame=5) + (_flows(rng, 8, 12, 16, boundary=(4,), none=(1,)),))
    vids.append(_video(rng, 6, 10, 14, pool, dup_frame=2) + (_flows(rng, 6, 10, 14),))
    vids.append(_video(rng, 5, 8, 8, np.arange(3), empty=(0, 4)) + (_flows(rng, 5, 8, 8, none=(2,)),))
    vids.append(_video(rng, 1, 16, 16, pool) + ([],))
    vids.append(_video(rng, 7, 12, 16, pool, empty=(6,)) + (_flows(rng, 7, 12, 16, boundary=(2,)),))
    out = []
    for v, dup in zip(vids, (True, True, False, False, False)):
        # with N_CONTEXT_FRAMES = 0 the reference asserts that the boxes come back unchanged (:635-638), which a
        # frame with a duplicate track id breaks (its second row takes the first row's box), and so does EXTEND_TRACKS
        # whenever list(set(ids)) reorders a frame's ids
        for n in ((1, 3) if dup else (0, 1, 3)):
            for ext in ((True, False) if n else (False,)):
                out.append(v + ((n, ext, 6.0),))
    return out


def run_reference(poses, boxes, tracks, flows, params):
    n_context, ext, th = params
    ns = _reference(n_context, ext, th)
    F = len(poses)
    H, W = next((f.shape[:2] for f in flows if f is not None), (16, 16))

    def compute_optical_flow(video_json_data):                      # :589-597 with the supplied pair flows
        fw, neg = [], [np.zeros((H, W, 2))]
        for f in flows:
            fw.append(f)
            neg.append(ns['_compute_neg_flow'](f))
        fw.append(np.zeros((H, W, 2)))
        return fw, neg
    ns['compute_optical_flow'] = compute_optical_flow
    dets = {'all_boxes': [[], [b.copy() for b in boxes]], 'all_keyps': [[], [[p.copy() for p in ps] for ps in poses]]}
    video = [({}, f) for f in range(F)]
    new_tracks = ns['_smooth_pose_video'](video, dets, [list(t) for t in tracks])
    return dets['all_keyps'][1], dets['all_boxes'][1], new_tracks


def pack_case(k, poses, boxes, tracks, flows, params, out_p, out_b, out_t):
    F = len(poses)
    dmax = max([len(t) for t in tracks] + [1])
    omax = max([len(t) for t in out_t] + [1])
    d = {}
    P = np.zeros((F, dmax, 4, K), F32); B = np.zeros((F, dmax, 5), F32); T = np.full((F, dmax), -1, np.int32)
    OP = np.zeros((F, omax, 4, K), F32); OB = np.zeros((F, omax, 5), F32); OT = np.full((F, omax), -1, np.int32)
    for f in range(F):
        n = len(tracks[f])
        if n:
            P[f, :n] = np.stack(poses[f]); B[f, :n] = boxes[f]; T[f, :n] = tracks[f]
        m = len(out_t[f])
        if m:
            OP[f, :m] = np.stack(out_p[f]); OB[f, :m] = out_b[f]; OT[f, :m] = out_t[f]
        assert all(p.dtype == F32 for p in out_p[f]) and (m == 0 or out_b[f].dtype == F32)
    d.update(poses=P, boxes=B, counts=np.array([len(t) for t in tracks], np.int32), tracks=T, out_poses=OP, out_boxes=OB,
             out_counts=np.array([len(t) for t in out_t], np.int32), out_tracks=OT,
             out_box_f64=np.array([b.dtype == np.float64 for b in out_b], np.uint8),
             flow_none=np.array([f is None for f in flows], np.uint8).reshape(-1),
             params=np.array(params, np.float64))
    for q, f in enumerate(flows):
        if f is not None:
            d['flow%d' % q] = f
    return {'c%d_%s' % (k, n): v for n, v in d.items()}


def main():
    out = {}
    for k, (poses, boxes, tracks, flows, params) in enumerate(cases()):
        out.update(pack_case(k, poses, boxes, tracks, flows, params, *run_reference(poses, boxes, tracks, flows, params)))
    path = os.path.join(HERE, 'flow_smooth.npz')
    np.savez_compressed(path, **out)
    print('wrote flow_smooth.npz: %d cases, %d bytes' % (k + 1, os.path.getsize(path)))


if __name__ == '__main__':
    main()

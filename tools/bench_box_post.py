"""Cost of TEST.SOFT_NMS / TEST.BBOX_VOTE on the device (BASELINE.json configs[3]: 8 clips of 3 x 800 x 1333, R50-FPN3D,
1000 proposals per clip, one foreground class).

    python tools/bench_box_post.py [--reps 5] [--steps 10] [--kernel-iters 20] [--out box_post.json]

1. Kernel times (CUDA events, mean over --kernel-iters launches after one warm-up) of dt_soft_nms_batched per method and of
   dt_box_vote (after hard NMS and after linear soft-NMS), on the decoded rows of a real captured step (its dt_box_decode
   output: 8 lists of up to 1000 rows), and on a V = 4 test-time augmentation union of them (4000 rows per list: the
   step's rows and three jittered copies, the shape dt_aug_merge_dets gives).
2. The captured configs[3] step in clips/s with: off, soft linear, soft gaussian, voting, soft linear + voting; the
   settings alternate within each of --reps rounds of --steps replays.
The card's name and power limit are read in the same call and printed with the numbers (one JSON line)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SETTINGS = [('off', {}),
            ('soft_linear', {'SOFT_NMS': {'ENABLED': True, 'METHOD': 'linear'}}),
            ('soft_gaussian', {'SOFT_NMS': {'ENABLED': True, 'METHOD': 'gaussian'}}),
            ('vote', {'BBOX_VOTE': {'ENABLED': True}}),
            ('soft_linear_vote', {'SOFT_NMS': {'ENABLED': True, 'METHOD': 'linear'}, 'BBOX_VOTE': {'ENABLED': True}})]


def card():
    import torch
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else 'unavailable')


def engine(setting):
    import bench
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.engine import DetectionEngine
    cfg = bench.bench_cfg(800, 1333, 'r50fpn3d')
    for node, kv in setting.items():
        for k, v in kv.items():
            cfg.TEST[node][k] = v
    blobs, spec = P.random_blobs(cfg)
    eng = DetectionEngine(cfg, blobs, spec, dtype='bf16x3')
    return eng, dict(cfg.TEST.SOFT_NMS), dict(cfg.TEST.BBOX_VOTE)


def time_kernel(torch, fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_times(torch, dets, cnt, iters, tag):
    from detectandtrack_b200.ops import box_ops
    out = {}
    for m in ('hard', 'linear', 'gaussian'):
        out['soft_nms_%s_ms' % m] = time_kernel(torch, lambda: box_ops.soft_nms_batched(dets, cnt, 0.5, 0.5, 0.0001, m), iters)
    keep, nkeep = box_ops.nms_batched(dets, cnt, 0.5, box_ops.NMS_2D_GE, box_ops.ORDER_INDEX)
    out['hard_nms_ms'] = time_kernel(torch, lambda: box_ops.nms_batched(dets, cnt, 0.5, box_ops.NMS_2D_GE,
                                                                         box_ops.ORDER_INDEX), iters)
    out['vote_after_hard_ms'] = time_kernel(torch, lambda: box_ops.box_vote(dets, cnt, 0.8, keep=keep, nkeep=nkeep), iters)
    rows, _, n = box_ops.soft_nms_batched(dets, cnt, 0.5, 0.5, 0.0001, 'linear')
    out['vote_after_soft_linear_ms'] = time_kernel(torch, lambda: box_ops.box_vote(dets, cnt, 0.8, top=rows, top_counts=n), iters)
    torch.cuda.synchronize()
    out['rows_per_list'] = cnt.cpu().tolist()
    out['hard_nms_kept'] = nkeep.cpu().tolist()
    out['soft_linear_kept'] = n.cpu().tolist()
    return {tag: out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--kernel-iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    import bench
    if not torch.cuda.is_available():
        raise SystemExit('bench_box_post: needs a CUDA device')
    B, T, H, W = 8, 3, 800, 1333
    frames = torch.from_numpy(bench.synth_frames(B, T, H, W, 7)).cuda()
    res = dict(card=card(), workload='configs[3]: B=%d clips of %dx%dx%d, R50-FPN3D, bf16x3' % (B, T, H, W))
    steps = {}
    for name, setting in SETTINGS:
        eng, soft, vote = engine(setting)
        seen = {}
        inner = eng.box_nms_limit

        def spy(dets, cnt, inner=inner, seen=seen):
            seen['dets'], seen['cnt'] = dets, cnt
            return inner(dets, cnt)
        eng.box_nms_limit = spy
        static_in, run = eng.capture(B, T, H, W)
        static_in.copy_(frames)
        run()
        torch.cuda.synchronize()
        steps[name] = dict(run=run, seen=seen, times=[], keep=(eng, static_in))     # the graph reads their memory
        if name == 'off':
            dets = seen['dets'].view(B, -1, 5).clone()
            cnt = seen['cnt'].clone()
    res['kernels'] = kernel_times(torch, dets, cnt, a.kernel_iters, 'step_rows')
    # a V = 4 union: the step's rows, then three copies jittered by up to 2 px (rows of a list stay contiguous)
    g = torch.Generator(device='cuda').manual_seed(0)
    R = dets.shape[1]
    views = [dets] + [dets + torch.cat([torch.rand(dets.shape[:2] + (4,), device='cuda', generator=g) * 4 - 2,
                                        torch.zeros(dets.shape[:2] + (1,), device='cuda')], 2) for _ in range(3)]
    union = torch.zeros((B, 4 * R, 5), dtype=torch.float32, device='cuda')
    c = cnt.cpu().tolist()
    for b in range(B):
        for v in range(4):
            union[b, v * c[b]:(v + 1) * c[b]] = views[v][b, :c[b]]
    res['kernels'].update(kernel_times(torch, union, (cnt * 4).int(), a.kernel_iters, 'union_v4'))
    for r in range(a.reps):
        for name, _ in SETTINGS:
            run = steps[name]['run']
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.steps):
                run()
            torch.cuda.synchronize()
            steps[name]['times'].append(B * a.steps / (time.perf_counter() - t0))
    res['step_clips_per_s'] = {n: dict(median=float(np.median(s['times'])), min=float(min(s['times'])),
                                       max=float(max(s['times']))) for n, s in steps.items()}
    res['card_after'] = card()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()

"""Cost of test-time augmentation (TEST.COMPETITION_MODE) at the benchmarked size: configs[3] (R50-FPN-3D, slice-center,
T = 3) at 800 x 1333 in bf16x3, the captured ClipPipeline step timed with CUDA events for

  off       augmentation off
  kps_flip  KPS_AUG.H_FLIP
  flip      BBOX_AUG.H_FLIP + KPS_AUG.H_FLIP
  flip_s    the previous plus one extra scale (BBOX_AUG / KPS_AUG.SCALES (--scale,) with SCALE_H_FLIP)

at the largest B up to --max-clips that fits, with the peak max_memory_allocated of each, and the CUDA-event time of each
new kernel (dt_aug_merge_dets, dt_aug_scale_rois, dt_keypoint_decode_aug) at that step's shapes.  Prints one JSON line
with the card name and power limit read in the same run.

    python tools/bench_tta.py [--steps 10] [--warmup 3] [--max-clips 8] [--scale 1000]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SETTINGS = {
    'off': {},
    'kps_flip': {'KPS_AUG.H_FLIP': True},
    'flip': {'BBOX_AUG.H_FLIP': True, 'KPS_AUG.H_FLIP': True},
    'flip_s': {'BBOX_AUG.H_FLIP': True, 'KPS_AUG.H_FLIP': True, 'BBOX_AUG.SCALES': 'S', 'KPS_AUG.SCALES': 'S',
               'BBOX_AUG.SCALE_H_FLIP': True, 'KPS_AUG.SCALE_H_FLIP': True},
}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:                      # noqa: BLE001
        return 'unknown (%s)' % e


def configure(cfg, name, scale):
    cfg.TEST.COMPETITION_MODE = name != 'off'
    cfg.TEST.BBOX_AUG.SCORE_HEUR = 'UNION'; cfg.TEST.BBOX_AUG.COORD_HEUR = 'UNION'
    for stage in (cfg.TEST.BBOX_AUG, cfg.TEST.KPS_AUG):
        stage.H_FLIP, stage.SCALES, stage.SCALE_H_FLIP = False, (), False
    for k, v in SETTINGS[name].items():
        stage, key = k.split('.')
        cfg.TEST[stage][key] = (scale,) if v == 'S' else v


def time_step(torch, model, B, T, H, W, plan, frames, args):
    from detectandtrack_b200.core.test import ClipPipeline
    torch.cuda.reset_peak_memory_stats()
    pipe = ClipPipeline(model, B, T, H, W, plan=plan)
    pipe.static_in.copy_(frames[:B])
    for _ in range(args.warmup):
        pipe.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        out = pipe.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    ndet = out['det_counts'].view(B, -1)[:, 0].tolist()
    peak = torch.cuda.max_memory_allocated()
    del pipe
    return dict(ms_per_step=round(ms, 2), clips_per_s=round(B * 1000. / ms, 3), peak_gib=round(peak / 2. ** 30, 2), ndet=ndet)


def kernel_times(torch, B, R, cap, V, K=17, S=14, n=50):
    """CUDA-event time of each new kernel at the step's shapes (V views, R proposals, cap detections per clip)."""
    from detectandtrack_b200.ops import rpn_ops, dense_ops
    from detectandtrack_b200.core import tta
    g = torch.Generator(device='cuda').manual_seed(0)
    dets = [torch.rand((B, 1, R, 5), device='cuda', generator=g) * 500 for _ in range(V)]
    cnts = [torch.full((B,), R, dtype=torch.int32, device='cuda') for _ in range(V)]
    im_hw = torch.tensor([[800., 1333.]] * B, device='cuda')
    boxes = torch.rand((B * cap, 5), device='cuda', generator=g) * 500
    low = torch.randn((V, B * cap, S, S, 4 * K), device='cuda', generator=g)
    flips = [v % 2 == 0 for v in range(V)]
    calls = dict(aug_merge_dets=lambda: rpn_ops.aug_merge_dets(dets, cnts, flips, im_hw),
                 aug_scale_rois=lambda: dense_ops.aug_scale_rois(boxes, 1.0, True, im_hw, per_image=cap),
                 keypoint_decode_aug=lambda: dense_ops.keypoint_decode_aug(low, flips, tta.COCO_FLIP_PERM, False, boxes, K))
    res = {}
    for name, f in calls.items():
        for _ in range(3):
            f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            f()
        e1.record()
        torch.cuda.synchronize()
        res[name + '_us'] = round(e0.elapsed_time(e1) * 1000. / n, 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--max-clips', type=int, default=8)
    ap.add_argument('--scale', type=int, default=1000)
    ap.add_argument('--height', type=int, default=800)
    ap.add_argument('--width', type=int, default=1333)
    args = ap.parse_args()
    import torch
    import bench
    from detectandtrack_b200.core import tta
    from detectandtrack_b200.modeling import params as P, model_builder
    H, W = args.height, args.width
    cfg = bench.bench_cfg(H, W, 'r50fpn3d')
    T = bench.frames_per_clip(cfg)
    blobs, spec = P.random_blobs(cfg)
    model = model_builder.create(cfg.MODEL.TYPE, train=False, blobs=blobs, dtype='bf16x3')
    frames = torch.from_numpy(bench.synth_frames(args.max_clips, T, H, W, 7)).cuda()
    out = dict(card=card(), size=[H, W], T=T, dtype='bf16x3', steps=args.steps, settings={})
    for name in SETTINGS:
        configure(cfg, name, args.scale)
        plan = tta.view_plan(cfg, spec, H, W) if cfg.TEST.COMPETITION_MODE else None
        r = None
        B = args.max_clips
        while B >= 1 and r is None:
            try:
                r = time_step(torch, model, B, T, H, W, plan, frames, args)
            except torch.cuda.OutOfMemoryError:
                model.__dict__.pop('_pipelines', None)
                torch.cuda.empty_cache()
                B //= 2
        r = r or dict(error='out of memory at B = 1')
        r.update(B=B, box_views=len(plan.box) if plan else 1, kps_views=len(plan.kps) if plan else 1)
        out['settings'][name] = r
        torch.cuda.empty_cache()
        print(name, r, flush=True)
    B = max(s.get('B', 1) for s in out['settings'].values())
    out['kernels'] = kernel_times(torch, B, cfg.TEST.RPN_POST_NMS_TOP_N, model.engine.det_cap, 4)
    out['kernels'].update(B=B, V=4)
    print(json.dumps(out))


if __name__ == '__main__':
    main()

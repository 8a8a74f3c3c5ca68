"""Micro-benchmark of the wgmma filter-gradient kernels on the trainable layer shapes of the keypoint R-CNN training step at
TRAIN.IMS_PER_BATCH = 2 clips (T = 3, 800x1344 blob): dt_wgrad_nhwc (operands straight from NDHWC, the path the trainer uses)
next to the first implementation (dt_to_planes + dt_wgrad).  CUDA events, median of --iters; TFLOP/s = 2*MACs of the conv.
    python tools/bench_wgrad.py [--iters 5] [--only res4] [--planes]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from detectandtrack_b200.ops import train_ops as to

LAYERS = [
    # name, N, T, H, W, Cin, Cout, k
    ('res3 branch2b 128>128 3x3x3', 2, 3, 100, 168, 128, 128, (3, 3, 3)),
    ('res3 branch2c 128>512 1x1x1', 2, 3, 100, 168, 128, 512, (1, 1, 1)),
    ('res4 branch2b 256>256 3x3x3', 2, 3, 50, 84, 256, 256, (3, 3, 3)),
    ('res4 branch2a 1024>256 1x1x1', 2, 3, 50, 84, 1024, 256, (1, 1, 1)),
    ('res5 branch2b 512>512 3x3x3', 2, 3, 25, 42, 512, 512, (3, 3, 3)),
    ('fpn posthoc P2 256>256 3x3x3', 2, 3, 200, 336, 256, 256, (3, 3, 3)),
    ('fpn posthoc P3 256>256 3x3x3', 2, 3, 100, 168, 256, 256, (3, 3, 3)),
    ('rpn conv P2 256>256 1x3x3', 2, 1, 200, 336, 256, 256, (1, 3, 3)),
    ('res3 branch2a 512>128 1x1x1', 2, 3, 100, 168, 512, 128, (1, 1, 1)),
    ('res5 branch2c 512>2048 1x1x1', 2, 3, 25, 42, 512, 2048, (1, 1, 1)),
    ('fpn lateral P2 256>256 1x1x1', 2, 3, 200, 336, 256, 256, (1, 1, 1)),
    ('kps conv_fcn 512>512 1x3x3 (256 RoIs)', 256, 1, 14, 14, 512, 512, (1, 3, 3)),
    ('fc6 12544>1024 (1024 RoIs)', 1, 1, 1, 1024, 12544, 1024, (1, 1, 1)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--only', default='')
    ap.add_argument('--planes', action='store_true', help='also time the plane-copy implementation')
    a = ap.parse_args()
    rows = []
    for name, N, T, H, W, Cin, Cout, k in LAYERS:
        if a.only and a.only not in name:
            continue
        x = torch.randn((N, T, H, W, Cin), device='cuda').bfloat16()
        gz = torch.randn((N, T, H, W, Cout), device='cuda').bfloat16()
        fl = 2.0 * N * T * H * W * Cin * Cout * k[0] * k[1] * k[2]
        dW = to.wgrad_nhwc(gz, x, k)
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.iters):
            e0, e1 = (torch.cuda.Event(enable_timing=True) for _ in range(2))
            e0.record()
            to.wgrad_nhwc(gz, x, k, dW=dW)
            e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[len(ts) // 2]
        row = dict(layer=name, wgrad_nhwc_ms=round(ms, 4), tflops=round(fl / ms / 1e9, 1), gflop=round(fl / 1e9, 1))
        if a.planes:
            pad = (k[1] // 2, k[2] // 2)
            xp = to.to_planes(x, pad=pad, copies=True)
            gp = to.to_planes(gz, pad=pad)
            dW2 = to.wgrad(gp, xp, (H, W), k)
            torch.cuda.synchronize()
            ts, tp = [], []
            for _ in range(a.iters):
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                xp = to.to_planes(x, pad=pad, copies=True); gp = to.to_planes(gz, pad=pad)
                e1.record()
                to.wgrad(gp, xp, (H, W), k, dW2)
                e2.record(); torch.cuda.synchronize()
                tp.append(e0.elapsed_time(e1)); ts.append(e1.elapsed_time(e2))
            row.update(planes_wgrad_ms=round(sorted(ts)[len(ts) // 2], 4), planes_copy_ms=round(sorted(tp)[len(tp) // 2], 4))
        rows.append(row)
        print(json.dumps(rows[-1]), flush=True)
    os.makedirs('gpurun_out', exist_ok=True)
    json.dump(rows, open('gpurun_out/bench_wgrad.json', 'w'), indent=1)


if __name__ == '__main__':
    main()

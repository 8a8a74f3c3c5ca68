"""Micro-benchmark of the wgmma conv kernel on the layer shapes that dominate the
R50-FPN-3D clip (SURVEY.md §8d).  CUDA-event timing, L2 flushed between iterations.
    python tools/bench_conv.py [--dtype bf16|tf32|bf16x3|tf32x3] [--iters 5]
(split modes: [hi | lo] pair inputs / outputs, 3 MMAs per k-block; TFLOP/s are ALGORITHMIC: 2*MACs of the fp32 conv)
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from detectandtrack_b200.ops import conv as cv

LAYERS = [
    # name, T, H, W, Cin, Cout, k, stride, pad
    ('fpn_posthoc_P2 256>256 3x3x3', 3, 200, 336, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ('fpn_posthoc_P3 256>256 3x3x3', 3, 100, 168, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ('rpn_P2 256>256 1x3x3', 1, 200, 336, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ('res2 64>64 1x3x3', 3, 200, 336, 64, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ('res2 64>256 1x1x1', 3, 200, 336, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('res2 64>256 1x1x1 +res', 3, 200, 336, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('res2 256>64 1x1x1', 3, 200, 336, 256, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('res3 128>128 3x3x3', 3, 100, 168, 128, 128, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ('res3 128>512 1x1x1', 3, 100, 168, 128, 512, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('res3 128>512 1x1x1 +res', 3, 100, 168, 128, 512, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('res4 256>256 3x3x3', 3, 50, 84, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ('res4 1024>256 1x1x1', 3, 50, 84, 1024, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('res5 512>512 3x3x3', 3, 25, 42, 512, 512, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ('fpn_posthoc_P5 256>256 3x3x3', 3, 25, 42, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ('fc6 12544>1024 (R=1000)', 1, 1, 1000, 12544, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ('kps conv 512>512 3x3 (D=100)', 100, 14, 14, 512, 512, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dtype', default='bf16')
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--only', default='')
    ap.add_argument('--n', type=int, default=1, help='clips per launch (body layers)')
    a = ap.parse_args()
    dtype = cv.MODE_NAMES[a.dtype]
    split = dtype in cv.SPLIT_MODES
    tdt = torch.bfloat16 if dtype in (cv.BF16, cv.BF16X3) else torch.float32
    of32 = None if split else (dtype == cv.TF32)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    rows = []
    for (name, T, H, W, Cin, Cout, k, s, p) in LAYERS:
        if a.only and a.only not in name:
            continue
        nb = a.n if H > 14 and H * W > 1000 else 1
        x = torch.randn((nb, T, H, W, Cin), device='cuda')
        x = cv.split_for(dtype, x) if split else x.to(tdt)
        w = cv.pack_weight(torch.randn((Cout, Cin) + k) * 0.02, dtype)
        sc = torch.ones(Cout, device='cuda'); bi = torch.zeros(Cout, device='cuda')
        y = cv.conv3d(x, w, k, s, p, sc, bi, relu=True, out_f32=of32, dtype=dtype)
        res = torch.randn_like(y) if name.endswith('+res') else None
        rm = 1 if res is not None else 0
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.iters):
            flush.zero_()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            cv.conv3d(x, w, k, s, p, sc, bi, res, rm, relu=True, out_f32=of32, dtype=dtype, out=y, split_out=split)
            e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[len(ts) // 2]
        flops = 2.0 * (y.numel() // (2 if split else 1)) * Cin * k[0] * k[1] * k[2]
        rows.append(dict(layer=name, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1), gflop=round(flops / 1e9, 1)))
        print(json.dumps(rows[-1]), flush=True)
    os.makedirs('gpurun_out', exist_ok=True)
    json.dump(rows, open('gpurun_out/bench_conv_%s.json' % a.dtype, 'w'), indent=1)


if __name__ == '__main__':
    main()

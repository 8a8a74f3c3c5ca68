"""GPU parity of the training-step kernels (csrc/train_ops.cu, through the C ABI) against torch autograd of the same
op in fp32 on the CPU (the stand-in for Caffe2's ConvGradient / AffineChannelNdGradient / Relu / Sum gradients that
model.AddGradientOperators emits, lib/modeling/model_builder.py:908-951; parity unpinned by the reference).

Tolerances (config 5 trains in bf16, BASELINE.json configs[4]): operands are the SAME bf16-rounded tensors on both
sides and the device accumulates in fp32, so wgrad / dgrad agree to accumulation order: <= 2e-3 * max|ref| for sums over
up to ~10^5 positions (fp32 split-K partials); bf16-stored outputs add 2^-9."""
import numpy as np
import pytest

from detectandtrack_b200.ops import train_ops as to

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('shape', [(2, 3, 20, 28, 128, 256, (3, 3, 3)), (2, 1, 14, 14, 512, 512, (1, 3, 3)), (1, 3, 13, 21, 1024, 256, (1, 1, 1))])
def test_dgrad_is_conv_with_flipped_transposed_filter(shape):
    import torch
    import torch.nn.functional as F
    from detectandtrack_b200.ops import conv as cv, train_ops as to
    N, T, H, W, Cin, Cout, k = shape
    g = torch.Generator().manual_seed(17)
    w = (torch.randn((Cout, Cin) + k, generator=g) * (1.0 / (Cin * k[0] * k[1] * k[2])) ** 0.5).bfloat16().float()
    gz = torch.randn((N, T, H, W, Cout), generator=g).bfloat16()
    pad = (k[0] // 2, k[1] // 2, k[2] // 2)
    x = torch.zeros((N, Cin, T, H, W), requires_grad=True)
    F.conv3d(x, w, None, 1, pad).backward(gz.float().permute(0, 4, 1, 2, 3))
    ref = x.grad.permute(0, 2, 3, 4, 1)
    dx = cv.conv3d(gz.cuda(), to.pack_dgrad_weight(w), k, (1, 1, 1), pad, out_f32=True, dtype=cv.BF16)
    torch.cuda.synchronize()
    assert dx.shape == ref.shape
    assert (dx.cpu() - ref).abs().max().item() <= 2e-4 * ref.abs().max().item()


def test_pointwise_joins():
    import torch
    from detectandtrack_b200.ops import train_ops as to
    g = torch.Generator().manual_seed(23)
    shp = (2, 3, 10, 14, 64)
    g1 = torch.randn(shp, generator=g).bfloat16(); g2 = torch.randn(shp, generator=g).bfloat16()
    y = torch.randn(shp, generator=g).bfloat16(); sc = torch.rand(64, generator=g) + 0.5
    out = to.bwd_pointwise(g1.cuda(), g2.cuda(), y.cuda(), sc.cuda()).cpu().float()
    ref = ((g1.float() + g2.float()) * (y.float() > 0) * sc).bfloat16().float()
    assert torch.equal(out, ref)
    assert torch.equal(to.bwd_pointwise(g1.cuda()).cpu(), g1)
    # two consumers of the same masked sum from one read: (scaled, other scale) and (scaled, unscaled)
    sc3 = torch.rand(64, generator=g) + 0.5
    o1, o2 = to.bwd_pointwise(g1.cuda(), g2.cuda(), y.cuda(), sc.cuda(), second=True, scale2=sc3.cuda())
    assert torch.equal(o1.cpu().float(), ref)
    assert torch.equal(o2.cpu().float(), ((g1.float() + g2.float()) * (y.float() > 0) * sc3).bfloat16().float())
    o1, o2 = to.bwd_pointwise(g1.cuda(), None, y.cuda(), sc.cuda(), second=True)
    assert torch.equal(o1.cpu().float(), (g1.float() * (y.float() > 0) * sc).bfloat16().float())
    assert torch.equal(o2.cpu().float(), (g1.float() * (y.float() > 0)).bfloat16().float())
    # slice-center gradient embedding
    from detectandtrack_b200 import _lib as L
    gc = torch.randn((2, 1, 5, 7, 64), generator=g).bfloat16().cuda()
    full = torch.empty((2, 3, 5, 7, 64), dtype=torch.bfloat16, device='cuda')
    L.call('dt_embed_frame', L.ptr(gc), 2, 3, 5 * 7 * 64, 1, L.ptr(full), L.stream_ptr())
    exp = torch.zeros((2, 3, 5, 7, 64), dtype=torch.bfloat16, device='cuda'); exp[:, 1:2] = gc
    assert torch.equal(full, exp)
    fine = torch.randn((2, 3, 10, 14, 64), generator=g).bfloat16()
    coarse = torch.randn((2, 3, 5, 7, 64), generator=g).bfloat16()
    up = to.upsample_add_bwd(fine.cuda(), coarse.cuda()).cpu().float()
    f = fine.float()
    ref = (coarse.float() + (f[:, :, 0::2, 0::2] + f[:, :, 0::2, 1::2]) + (f[:, :, 1::2, 0::2] + f[:, :, 1::2, 1::2]))
    assert (up - ref).abs().max().item() <= 2 ** -7 * ref.abs().max().item()          # bf16 output rounding, other sum order
    src = torch.randn((2, 3, 7, 11, 64), generator=g).bfloat16()
    sc2 = to.scatter_stride2(src.cuda(), (13, 21)).cpu()
    ref = torch.zeros((2, 3, 13, 21, 64), dtype=torch.bfloat16); ref[:, :, 0::2, 0::2] = src
    assert torch.equal(sc2, ref)


def test_sgd_update_matches_caffe2_momentum_sgd():
    """model_builder.py:954-985: grad += wd * w (WeightedSum), then MomentumSGDUpdate: adj = lr * grad + mu * m; m = adj;
    w -= adj; plus the refreshed bf16 forward / dgrad filters."""
    import torch
    from detectandtrack_b200.ops import train_ops as to, conv as cv
    g = torch.Generator().manual_seed(29)
    taps, Cout, Cin = 27, 24, 16
    w = torch.randn((taps, Cout, Cin), generator=g); gr = torch.randn((taps, Cout, Cin), generator=g); m = torch.randn((taps, Cout, Cin), generator=g) * 0.1
    lr, mu, wd, gs = 0.01, 0.9, 1e-4, 0.125
    adj = lr * (gs * gr + wd * w) + mu * m
    w_ref = w - adj
    wd_, gd, md = w.clone().cuda(), gr.cuda(), m.clone().cuda()
    wf = torch.empty((taps, Cout, Cin), dtype=torch.bfloat16, device='cuda'); wdg = torch.empty((taps, Cin, Cout), dtype=torch.bfloat16, device='cuda')
    to.sgd_update(wd_, gd, md, lr, mu, wd, gs, wf, wdg)
    assert torch.allclose(wd_.cpu(), w_ref, rtol=1e-6, atol=1e-7) and torch.allclose(md.cpu(), adj, rtol=1e-6, atol=1e-7)
    assert torch.equal(wf.cpu(), wd_.cpu().bfloat16())
    # the dgrad filter equals packing the flipped / transposed 5-D filter
    w5 = wd_.cpu().view(3, 3, 3, Cout, Cin).permute(3, 4, 0, 1, 2)
    assert torch.equal(wdg.cpu(), to.pack_dgrad_weight(w5).cpu())


def test_bias_grad_vs_sum():
    import torch
    from detectandtrack_b200 import _lib as L
    rng = np.random.RandomState(8)
    for rows, C, ld in ((1000, 256, 256), (37, 16, 16), (5000, 72, 72), (300, 520, 528)):
        g = torch.from_numpy(rng.randn(rows, ld).astype(np.float32)).to(torch.bfloat16).cuda()
        db = torch.zeros(C, dtype=torch.float32, device='cuda')
        L.call('dt_bias_grad', L.ptr(g), rows, C, ld, L.ptr(db), L.stream_ptr())
        ref = g.float()[:, :C].sum(0)
        assert torch.allclose(db, ref, rtol=1e-4, atol=1e-3), (rows, C)


NHWC_CASES = [
    # N, T, H, W, Cin, Cout, k
    (2, 3, 20, 28, 128, 128, (3, 3, 3)),
    (1, 3, 25, 42, 256, 256, (3, 3, 3)),
    (2, 1, 14, 14, 64, 192, (1, 3, 3)),
    (2, 2, 16, 24, 64, 256, (1, 1, 1)),
    (1, 3, 13, 21, 512, 128, (1, 1, 1)),
    (3, 1, 7, 7, 72, 40, (1, 3, 3)),
    (1, 1, 50, 84, 256, 15, (1, 1, 1)),
    (1, 1, 1, 300, 264, 16, (1, 1, 1)),          # an FC layer: RoIs along W
    (37, 1, 14, 14, 64, 72, (1, 3, 3)),          # keypoint-head maps: many small images per position tile
    (2, 3, 25, 42, 128, 128, (3, 3, 3)),         # ragged tiles in H and W, temporal taps
]


@pytest.mark.parametrize('case', range(len(NHWC_CASES)))
def test_wgrad_nhwc_vs_autograd(case):
    """dt_wgrad_nhwc (operands straight from NDHWC as MN-major wgmma operands) against torch autograd in fp32."""
    import torch
    import torch.nn.functional as F
    N, T, H, W, Cin, Cout, k = NHWC_CASES[case]
    g = torch.Generator().manual_seed(900 + case)
    x = torch.randn((N, T, H, W, Cin), generator=g).bfloat16()
    gz = torch.randn((N, T, H, W, Cout), generator=g).bfloat16()
    pad = (k[0] // 2, k[1] // 2, k[2] // 2)
    w = torch.zeros((Cout, Cin) + k, requires_grad=True)
    F.conv3d(x.float().permute(0, 4, 1, 2, 3), w, None, 1, pad).backward(gz.float().permute(0, 4, 1, 2, 3))
    ref = w.grad.permute(2, 3, 4, 0, 1).reshape(k[0] * k[1] * k[2], Cout, Cin)
    cpad = (Cout + 7) // 8 * 8
    gzd = torch.zeros((N, T, H, W, cpad), dtype=torch.bfloat16)
    gzd[..., :Cout] = gz
    dW = to.wgrad_nhwc(gzd.cuda(), x.cuda(), k, cout=cpad)
    torch.cuda.synchronize()
    got = dW.cpu()[:, :Cout]
    err = (got - ref).abs().max().item()
    assert err <= 2e-3 * ref.abs().max().item(), (err, ref.abs().max().item())
    assert float(dW[:, Cout:].abs().sum()) == 0.0


def test_wgrad_nhwc_strided_pointwise():
    """1x1 stride-2 conv (bottleneck branch2a / branch1 of the first block of a stage, STRIDE_1X1): the input box walks the
    subsampled positions."""
    import torch
    import torch.nn.functional as F
    g = torch.Generator().manual_seed(6)
    x = torch.randn((2, 3, 25, 41, 256), generator=g).bfloat16()
    gz = torch.randn((2, 3, 13, 21, 128), generator=g).bfloat16()
    w = torch.zeros((128, 256, 1, 1, 1), requires_grad=True)
    F.conv3d(x.float().permute(0, 4, 1, 2, 3), w, None, (1, 2, 2)).backward(gz.float().permute(0, 4, 1, 2, 3))
    dW = to.wgrad_nhwc(gz.cuda(), x.cuda(), (1, 1, 1), stride=(2, 2))
    ref = w.grad.reshape(1, 128, 256)
    assert (dW.cpu() - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()

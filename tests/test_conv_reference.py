"""CPU: the fp64 reference the conv value tests (tests/test_gpu_conv.py) compare conv_tc_kernel with.  It is a sum over
filter taps of GEMMs on the zero-padded, tap-shifted input, so it shares nothing with the kernel's implicit GEMM or with
cuDNN, and on the device it runs as DGEMMs, fast enough for problems that fill several waves of the GPU.  Pinned here
once against torch's own fp64 conv3d."""
import torch
import torch.nn.functional as F


def conv_ref(x, w, stride, pad, scale=None, bias=None, residual=None, res_mode=0, relu=False):
    """x [N, T, H, W, Cin], w [Cout, Cin, kT, kH, kW] (any float type, any device) -> fp64 [N, To, Ho, Wo, Cout] =
    relu?(conv(x, w) * scale + bias (+ residual, or its nearest-2x upsample for res_mode 2))."""
    x, w = x.double(), w.double()
    N, T, H, W, Cin = x.shape
    Cout, _, kT, kH, kW = w.shape
    (sT, sH, sW), (pT, pH, pW) = stride, pad
    To, Ho, Wo = (T + 2 * pT - kT) // sT + 1, (H + 2 * pH - kH) // sH + 1, (W + 2 * pW - kW) // sW + 1
    xp = F.pad(x, (0, 0, pW, pW, pH, pH, pT, pT))
    y = torch.zeros((N * To * Ho * Wo, Cout), dtype=torch.float64, device=x.device)
    for kt in range(kT):
        for kh in range(kH):
            for kw in range(kW):
                xs = xp[:, kt:kt + sT * (To - 1) + 1:sT, kh:kh + sH * (Ho - 1) + 1:sH, kw:kw + sW * (Wo - 1) + 1:sW]
                y += xs.reshape(-1, Cin) @ w[:, :, kt, kh, kw].t()
    y = y.view(N, To, Ho, Wo, Cout)
    if scale is not None:
        y = y * scale.double()
    if bias is not None:
        y = y + bias.double()
    if res_mode == 1:
        y = y + residual.double()
    elif res_mode == 2:
        y = y + residual.double().repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    return y.clamp_min(0) if relu else y


def test_tap_sum_reference_equals_torch_conv3d():
    g = torch.Generator().manual_seed(5)
    x = torch.randn((2, 4, 11, 13, 6), generator=g)
    w = torch.randn((5, 6, 3, 3, 3), generator=g)
    scale, bias = torch.rand(5, generator=g) + 0.5, torch.randn(5, generator=g)
    for stride, pad in (((1, 1, 1), (1, 1, 1)), ((1, 2, 2), (0, 1, 1)), ((2, 1, 2), (1, 0, 1))):
        y = conv_ref(x, w, stride, pad, scale, bias)
        ref = F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), None, stride, pad).permute(0, 2, 3, 4, 1)
        ref = ref * scale.double() + bias.double()
        assert y.dtype == torch.float64 and y.shape == ref.shape
        assert (y - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    # residual epilogues: same shape, and the nearest-2x upsample of the FPN top-down add, then ReLU
    y = conv_ref(x, w, (1, 1, 1), (1, 1, 1))
    res = torch.randn(y.shape, generator=g)
    assert torch.equal(conv_ref(x, w, (1, 1, 1), (1, 1, 1), residual=res, res_mode=1, relu=True), (y + res.double()).clamp_min(0))
    x2 = torch.randn((1, 2, 8, 6, 6), generator=g)
    y = conv_ref(x2, w, (1, 1, 1), (1, 1, 1))
    top = torch.randn((1, 2, 4, 3, 5), generator=g)
    up = conv_ref(x2, w, (1, 1, 1), (1, 1, 1), residual=top, res_mode=2)
    assert torch.equal(up[:, :, 5, 3], y[:, :, 5, 3] + top[:, :, 2, 1].double())

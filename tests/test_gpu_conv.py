"""GPU parity of the wgmma implicit-GEMM convolution (through the C ABI) against a plain
PyTorch fp32 reference of the same op (torch.nn.functional.conv3d on the CPU, the stand-in
for the un-vendored Caffe2 ConvNd + AffineChannelNd + Sum + Relu; "parity unpinned" by the
reference, SURVEY.md §8c).

Tolerances (north star: 1e-3 relative fp32):
  bf16 mode: the reference is evaluated on the SAME bf16-rounded x and w, so only fp32
             accumulation order differs: |err| <= 2e-4 * max|y| (fp32 output).
  tf32 mode: fp32 inputs, tf32 multiplies: |err| <= 1e-3 * max|y|.
  tf32x3   : [hi | lo] tf32 pairs, 3 MMAs per k-block (fp32-accurate parity mode): |err| <= 1e-4 * max|y|.
  bf16x3   : [hi | lo] bf16 pairs, 3 bf16 MMAs per k-block (the headline parity mode; operands carry 16 mantissa
             bits, 2^-17 relative): |err| <= 1e-4 * max|y| for both the bf16-pair output and the plain fp32 output.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _ref_conv(x, w, stride, pad, scale, bias, residual, res_mode, relu):
    import torch
    import torch.nn.functional as F
    # x [N,T,H,W,C] -> NCTHW
    y = F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), None, stride, pad)
    if scale is not None:
        y = y * scale.double().view(1, -1, 1, 1, 1)
    if bias is not None:
        y = y + bias.double().view(1, -1, 1, 1, 1)
    y = y.permute(0, 2, 3, 4, 1)
    if res_mode == 1:
        y = y + residual.double()
    elif res_mode == 2:
        y = y + residual.double().repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
    if relu:
        y = y.clamp_min(0)
    return y.float()


CASES = [
    # N, T, H, W, Cin, Cout, k, stride, pad, affine, res_mode, relu
    dict(N=1, T=1, H=16, W=16, Cin=64, Cout=64, k=(1, 1, 1), s=(1, 1, 1), p=(0, 0, 0)),
    dict(N=1, T=1, H=16, W=32, Cin=64, Cout=128, k=(1, 3, 3), s=(1, 1, 1), p=(0, 1, 1), affine=True, relu=True),
    dict(N=2, T=3, H=20, W=28, Cin=128, Cout=256, k=(3, 3, 3), s=(1, 1, 1), p=(1, 1, 1), affine=True, res_mode=1, relu=True),
    dict(N=1, T=3, H=13, W=21, Cin=256, Cout=256, k=(3, 3, 3), s=(1, 1, 1), p=(1, 1, 1)),
    dict(N=1, T=3, H=25, W=42, Cin=256, Cout=512, k=(1, 1, 1), s=(1, 2, 2), p=(0, 0, 0), affine=True),
    dict(N=1, T=2, H=24, W=40, Cin=192, Cout=64, k=(1, 1, 1), s=(1, 1, 1), p=(0, 0, 0), res_mode=2),
    dict(N=1, T=1, H=50, W=84, Cin=256, Cout=12, k=(1, 1, 1), s=(1, 1, 1), p=(0, 0, 0), bias=True),
    dict(N=1, T=1, H=1, W=300, Cin=1000, Cout=1024, k=(1, 1, 1), s=(1, 1, 1), p=(0, 0, 0), bias=True, relu=True),
    dict(N=1, T=1, H=14, W=14, Cin=512, Cout=512, k=(1, 3, 3), s=(1, 1, 1), p=(0, 1, 1), bias=True, relu=True),
    dict(N=3, T=1, H=9, W=7, Cin=72, Cout=40, k=(1, 3, 3), s=(1, 1, 1), p=(0, 1, 1)),
    # strided non-pointwise convs (TMA element strides): conv1 7x7/2 on a channel-padded image, R18 3x3/2
    dict(N=1, T=3, H=64, W=96, Cin=8, Cout=64, k=(1, 7, 7), s=(1, 2, 2), p=(0, 3, 3), affine=True, relu=True),
    dict(N=2, T=3, H=30, W=44, Cin=64, Cout=128, k=(3, 3, 3), s=(1, 2, 2), p=(1, 1, 1), affine=True, relu=True),
    dict(N=1, T=1, H=33, W=47, Cin=64, Cout=64, k=(1, 3, 3), s=(1, 2, 2), p=(0, 1, 1)),
    # small maps: the M tile stacks images / frames (ragged last stack included)
    dict(N=20, T=1, H=14, W=14, Cin=64, Cout=96, k=(1, 3, 3), s=(1, 1, 1), p=(0, 1, 1), affine=True, res_mode=1, relu=True),
    dict(N=2, T=3, H=25, W=42, Cin=64, Cout=64, k=(3, 3, 3), s=(1, 1, 1), p=(1, 1, 1), affine=True, relu=True),
    dict(N=5, T=3, H=7, W=7, Cin=64, Cout=128, k=(3, 3, 3), s=(1, 1, 1), p=(1, 1, 1), bias=True),
    dict(N=7, T=2, H=6, W=10, Cin=96, Cout=64, k=(1, 1, 1), s=(1, 1, 1), p=(0, 0, 0), res_mode=2),
]


@pytest.mark.parametrize('mode', ['bf16', 'tf32', 'tf32x3', 'bf16x3', 'bf16x3-f32out', 'f16'])
@pytest.mark.parametrize('case', range(len(CASES)))
def test_conv_parity(case, mode):
    import torch
    from detectandtrack_b200.ops import conv as cv
    c = CASES[case]
    g = torch.Generator().manual_seed(100 + case)
    N, T, H, W, Cin, Cout = c['N'], c['T'], c['H'], c['W'], c['Cin'], c['Cout']
    k, s, p = c['k'], c['s'], c['p']
    x = torch.randn((N, T, H, W, Cin), generator=g)
    w = torch.randn((Cout, Cin) + k, generator=g) * (2.0 / (Cin * k[0] * k[1] * k[2])) ** 0.5
    scale = (torch.rand(Cout, generator=g) + 0.5) if c.get('affine') else None
    bias = (torch.randn(Cout, generator=g) * 0.1) if (c.get('affine') or c.get('bias')) else None
    To = (T + 2 * p[0] - k[0]) // s[0] + 1
    Ho = (H + 2 * p[1] - k[1]) // s[1] + 1
    Wo = (W + 2 * p[2] - k[2]) // s[2] + 1
    rm = c.get('res_mode', 0)
    res = None
    if rm == 1:
        res = torch.randn((N, To, Ho, Wo, Cout), generator=g)
    elif rm == 2:
        res = torch.randn((N, To, Ho // 2, Wo // 2, Cout), generator=g)
    f32out = mode.endswith('-f32out')
    mode = mode.split('-')[0]
    dtype = cv.F16 if mode == 'f16' else cv.MODE_NAMES[mode]
    if mode == 'f16':
        # fp16 operands (DT_DTYPE_F16: the post-hoc FPN convs of the bf16x3h mode): reference on the SAME fp16-rounded x, w
        if rm:
            pytest.skip('fp16-operand convs take no residual')
        x = x.half().float(); w = w.half().float()
        xd = x.half().cuda()
        tol = 2e-4
    elif mode == 'bf16x3':
        if Cin % 64 or (Cout % 64 and not f32out):
            pytest.skip('bf16-pair storage needs channel counts that are multiples of 64 (true for every layer that uses it)')
        xd = cv.split_bf16(x.cuda())
        tol = 1e-4          # operands exact to 2^-17, lo*lo dropped (2^-18), bf16-pair output 2^-17
    elif mode == 'tf32x3':
        if Cin % 32 or Cout % 32:
            pytest.skip('3xTF32 storage needs channel counts that are multiples of 32 (true for every layer that uses it)')
        xd = cv.split_tf32(x.cuda())
        tol = 1e-4          # fp32 accumulation over K up to 3456 (measured ~2e-5); 10x inside the north star's 1e-3
    elif mode == 'bf16':
        x = x.bfloat16().float(); w = w.bfloat16().float()
        xd = x.bfloat16().cuda()
        tol = 2e-4
    else:
        xd = x.cuda()
        tol = 1e-3
    wp = cv.pack_weight(w, dtype)
    resd = res.cuda().contiguous() if res is not None else None
    if mode in ('tf32x3', 'bf16x3') and resd is not None:
        if f32out:
            pytest.skip('plain fp32 outputs of the split modes are the final head outputs: no residual')
        resd = cv.split_for(dtype, resd)
    out = torch.empty((N, To, Ho, Wo, Cout), dtype=torch.float32, device='cuda') if f32out else None
    y = cv.conv3d(xd.contiguous(), wp, k, s, p,
                  scale.cuda() if scale is not None else None, bias.cuda() if bias is not None else None,
                  resd, rm, bool(c.get('relu')), out_f32=(None if mode == 'bf16x3' else True), dtype=dtype, cin=Cin,
                  round_tf32=False, out=out)
    if mode in ('tf32x3', 'bf16x3') and not f32out:
        y = cv.join_split(y)
    torch.cuda.synchronize()
    ref = _ref_conv(x, w, s, p, scale, bias, res, rm, bool(c.get('relu')))
    err = (y.cpu() - ref).abs().max().item()
    den = ref.abs().max().item()
    assert y.shape == ref.shape
    assert err <= tol * den, (err, den, err / den)


def test_conv_bf16_output_and_channel_slices():
    """bf16 output path, reading a channel slice (in_ld > Cin) and writing into a slice of a
    wider tensor (out_ld > Cout), as the engine does for concatenations."""
    import torch
    from detectandtrack_b200.ops import conv as cv
    g = torch.Generator().manual_seed(7)
    x = torch.randn((1, 1, 12, 20, 128), generator=g).bfloat16()
    w = (torch.randn((64, 64, 1, 3, 3), generator=g) * 0.05).bfloat16()
    out = torch.zeros((1, 1, 12, 20, 192), dtype=torch.bfloat16, device='cuda')
    wp = cv.pack_weight(w.float(), cv.BF16)
    cv.conv3d(x.cuda(), wp, (1, 3, 3), (1, 1, 1), (0, 1, 1), relu=True, out_f32=False, dtype=cv.BF16, cin=64, out=out)
    ref = _ref_conv(x[..., :64].float(), w.float(), (1, 1, 1), (0, 1, 1), None, None, None, 0, True)
    got = out.cpu().float()
    assert torch.all(got[..., 64:] == 0)
    assert (got[..., :64] - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()     # bf16 output rounding (2^-8)


@pytest.mark.parametrize('shape', [(1, 3, 40, 56, 64, 256), (11, 1, 14, 14, 128, 200), (2, 3, 25, 42, 64, 256), (2, 1, 16, 32, 64, 256),
                                   (3, 2, 24, 48, 128, 192)])
@pytest.mark.parametrize('res_mode', [1, 2])
def test_conv_bf16_residual_epilogue(shape, res_mode):
    """The hot-path epilogue: bf16 in / bf16 out, AffineChannel + residual (same shape, or nearest-2x
    top-down add) + ReLU, including stacked M tiles and a ragged channel tail (Cout=200)."""
    import torch
    from detectandtrack_b200.ops import conv as cv
    N, T, H, W, Cin, Cout = shape
    if res_mode == 2 and (H % 2 or W % 2):
        pytest.skip('upsample-add needs even output size')
    g = torch.Generator().manual_seed(H * 131 + Cout + res_mode)
    x = torch.randn((N, T, H, W, Cin), generator=g).bfloat16()
    w = (torch.randn((Cout, Cin, 1, 1, 1), generator=g) * (1.0 / Cin) ** 0.5).bfloat16()
    scale = torch.rand(Cout, generator=g) + 0.5
    bias = torch.randn(Cout, generator=g) * 0.1
    rs = (N, T, H, W, Cout) if res_mode == 1 else (N, T, H // 2, W // 2, Cout)
    res = torch.randn(rs, generator=g).bfloat16()
    wp = cv.pack_weight(w.float(), cv.BF16)
    y = cv.conv3d(x.cuda(), wp, (1, 1, 1), (1, 1, 1), (0, 0, 0), scale.cuda(), bias.cuda(), res.cuda(), res_mode, True,
                  out_f32=False, dtype=cv.BF16, cin=Cin)
    torch.cuda.synchronize()
    ref = _ref_conv(x.float(), w.float(), (1, 1, 1), (0, 0, 0), scale, bias, res.float(), res_mode, True)
    assert y.dtype == torch.bfloat16 and y.shape == ref.shape
    assert (y.cpu().float() - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()   # bf16 output rounding (2^-8)


def test_conv_time_major_output():
    """out_time_major: y stored [To, N, Ho, Wo, C]; the returned [N, To, ...] view equals the normal result and
    a single-frame slice of it is contiguous (the centre-frame link becomes a view)."""
    import torch
    from detectandtrack_b200.ops import conv as cv
    g = torch.Generator().manual_seed(11)
    x = torch.randn((3, 3, 13, 21, 64), generator=g).bfloat16().cuda()
    w = (torch.randn((64, 64, 3, 3, 3), generator=g) * 0.03).bfloat16()
    wp = cv.pack_weight(w.float(), cv.BF16)
    a = cv.conv3d(x, wp, (3, 3, 3), (1, 1, 1), (1, 1, 1), relu=True, out_f32=False, dtype=cv.BF16)
    b = cv.conv3d(x, wp, (3, 3, 3), (1, 1, 1), (1, 1, 1), relu=True, out_f32=False, dtype=cv.BF16, time_major=True)
    torch.cuda.synchronize()
    assert b.shape == a.shape and not b.is_contiguous() and b[:, 1:2].is_contiguous()
    assert torch.equal(a, b.contiguous())


@pytest.mark.parametrize('first,count', [(0, 1), (1, 1), (2, 1), (1, 2)])
def test_conv_output_frame_range(first, count):
    """out_t_first / out_t_count: only the requested output frames are computed, bit-identical to the same
    frames of the full conv (temporal zero padding at the clip borders included)."""
    import torch
    from detectandtrack_b200.ops import conv as cv
    g = torch.Generator().manual_seed(21)
    x = torch.randn((2, 3, 13, 21, 64), generator=g).bfloat16().cuda()
    w = (torch.randn((64, 64, 3, 3, 3), generator=g) * 0.03).bfloat16()
    wp = cv.pack_weight(w.float(), cv.BF16)
    full = cv.conv3d(x, wp, (3, 3, 3), (1, 1, 1), (1, 1, 1), relu=True, out_f32=False, dtype=cv.BF16)
    part = cv.conv3d(x, wp, (3, 3, 3), (1, 1, 1), (1, 1, 1), relu=True, out_f32=False, dtype=cv.BF16, out_frames=(first, count))
    torch.cuda.synchronize()
    assert part.shape == (2, count, 13, 21, 64)
    assert torch.equal(part, full[:, first:first + count])


def test_conv_rejects_bad_arguments():
    import torch
    from detectandtrack_b200.ops import conv as cv
    x = torch.zeros((1, 1, 8, 8, 12), dtype=torch.bfloat16, device='cuda')     # 24-byte rows
    wp = torch.zeros((1, 16, 16), dtype=torch.bfloat16, device='cuda')
    with pytest.raises(RuntimeError, match='16 bytes'):
        cv.conv3d(x, wp, (1, 1, 1), cin=12)


@pytest.mark.parametrize('mode', ['bf16', 'tf32', 'bf16x3'])
def test_conv1_packed_rows_vs_torch(mode):
    """dt_conv1_7x7s2 (filter row packed into K over a zero-bordered blob) == conv 7x7 s2 p3 + affine + relu."""
    import torch
    import torch.nn.functional as F
    from detectandtrack_b200.ops import conv as cv, dense_ops
    g = torch.Generator().manual_seed(11)
    Fr, H, W = 3, 64, 96
    frames = torch.randint(0, 256, (Fr, H, W, 3), generator=g, dtype=torch.uint8)
    means = (102.9801, 115.9465, 122.7717)
    w = torch.randn((64, 3, 1, 7, 7), generator=g) * 0.01
    sc = torch.rand(64, generator=g) + 0.5
    bi = torch.randn(64, generator=g) * 0.1
    dtype = cv.MODE_NAMES[mode]
    cp = 4 if mode == 'tf32' else 8
    x = dense_ops.prep_clip(frames.cuda(), means, 1.0, (H, W), (H, W), cpad=cp, out_f32={'bf16': 0, 'tf32': 1, 'bf16x3': 3}[mode],
                            border=(3, 4), row_planes=True)
    assert x.shape == (Fr, 2, (H + 6) // 2, W + 8, cp)
    wp = cv.pack_conv1_weight(w, dtype)
    if mode == 'bf16x3':
        # split-pixel blob [hi3 | lo3 | 0 0], 14 weight blocks, bf16-pair output: fp32-accurate (<= 1e-4) vs the exact conv
        y = cv.join_split(cv.conv1_7x7s2(x, wp, (H, W), sc.cuda(), bi.cuda(), relu=True, dtype=dtype)).cpu()
        xin = (frames.float() - torch.tensor(means).view(1, 1, 1, 3)).permute(0, 3, 1, 2)
        ref = F.conv2d(xin.double(), w[:, :, 0].double(), None, 2, 3) * sc.double().view(1, -1, 1, 1) + bi.double().view(1, -1, 1, 1)
        ref = ref.clamp_min(0).permute(0, 2, 3, 1).float()
        assert y.shape == ref.shape and (y - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
        return
    y = cv.conv1_7x7s2(x, wp, (H, W), sc.cuda(), bi.cuda(), relu=True, dtype=dtype, out_f32=True).cpu()
    xfull = x.permute(0, 2, 1, 3, 4).reshape(Fr, H + 6, W + 8, cp)             # padded row r = [r & 1][r >> 1]
    xin = xfull[:, 3:3 + H, 4:4 + W, :3].float().cpu().permute(0, 3, 1, 2)      # what the kernel saw (rounded blob)
    wr = w[:, :, 0].bfloat16().float() if mode == 'bf16' else w[:, :, 0]
    ref = F.conv2d(xin.double(), wr.double(), None, 2, 3) * sc.double().view(1, -1, 1, 1) + bi.double().view(1, -1, 1, 1)
    ref = ref.clamp_min(0).permute(0, 2, 3, 1).float()
    tol = 2e-4 if mode == 'bf16' else 1.5e-3
    assert y.shape == ref.shape
    assert (y - ref).abs().max().item() <= tol * ref.abs().max().item()

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


def _within_bf16_output(y, ref):
    """bf16 outputs: |y - ref| <= 2^-8 |ref| + 2e-4 max|ref| elementwise, half a bf16 ulp of output rounding plus the
    fp32 accumulation-order error."""
    y, ref = y.double(), ref.double()
    return bool(((y - ref).abs() <= 2 ** -8 * ref.abs() + 2e-4 * ref.abs().max()).all())


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
    assert _within_bf16_output(got[..., :64], ref)


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
    assert _within_bf16_output(y.cpu().float(), ref)


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
    _check_conv1_packed_rows(mode, 3, 64, 96)


@pytest.mark.parametrize('mode', ['bf16', 'tf32', 'bf16x3'])
def test_conv1_packed_rows_three_tiles_per_cta(mode):
    """The same at three 256 x 336 frames: every CTA walks at least three 128-row tiles."""
    import torch
    Fr, H, W = 3, 256, 336
    assert Fr * (H // 2) * (W // 2) / 128 >= 3 * torch.cuda.get_device_properties(0).multi_processor_count
    _check_conv1_packed_rows(mode, Fr, H, W)


def _check_conv1_packed_rows(mode, Fr, H, W):
    import torch
    import torch.nn.functional as F
    from detectandtrack_b200.ops import conv as cv, dense_ops
    g = torch.Generator().manual_seed(11)
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
    if mode == 'bf16':
        # the engine's bf16 conv1 writes bf16: half a bf16 ulp of rounding on top of the accumulation-order error
        yb = cv.conv1_7x7s2(x, wp, (H, W), sc.cuda(), bi.cuda(), relu=True, dtype=dtype).cpu()
        assert _within_bf16_output(yb, ref)


def test_conv1_exact_fp32_vs_fp64():
    """dt_conv1_7x7s2_f32 (the tf32x3 mode's conv1) is plain fp32: each output is within the fp32 rounding bound of a
    147-term sum, sum_k |x_k w_k| * 147 * 2^-24, plus the affine rounding and the tf32 pair storage (2^-22) of the
    value, against an fp64 conv of the same fp32 blob.  Three 256 x 336 frames: many CTAs of 32 pixels each."""
    import torch
    import torch.nn.functional as F
    from detectandtrack_b200.ops import conv as cv, dense_ops
    g = torch.Generator().manual_seed(12)
    Fr, H, W = 3, 256, 336
    frames = torch.randint(0, 256, (Fr, H, W, 3), generator=g, dtype=torch.uint8)
    blob = dense_ops.prep_clip(frames.cuda(), (102.9801, 115.9465, 122.7717), 1.0, (H, W), (H, W), cpad=4, out_f32=2)
    w = torch.randn((64, 3, 7, 7), generator=g) * 0.01
    sc = torch.rand(64, generator=g) + 0.5
    bi = torch.randn(64, generator=g) * 0.1
    y = cv.join_tf32(cv.conv1_7x7s2_f32(blob, cv.pack_conv1_weight_f32(w), sc.cuda(), bi.cuda())).cpu().double()
    xin = blob[..., :3].cpu().double().permute(0, 3, 1, 2)
    s4, b4 = sc.double().view(1, -1, 1, 1), bi.double().view(1, -1, 1, 1)
    ref = (F.conv2d(xin, w.double(), None, 2, 3) * s4 + b4).clamp_min(0).permute(0, 2, 3, 1)
    mag = (F.conv2d(xin.abs(), w.double().abs(), None, 2, 3) * s4.abs()).permute(0, 2, 3, 1)
    bound = 2 ** -24 * (147 * mag + 5 * ref.abs()) + 1e-30
    assert y.shape == ref.shape
    ratio = ((y - ref).abs() / bound).max().item()
    assert ratio <= 1.0, ratio


def test_pairs_to_f16_rounds_and_saturates_like_torch():
    """dt_pairs_to_f16 == fp16(clamp(hi + lo, +-65504)) bit for bit, from fp16 subnormals to values beyond its range."""
    import torch
    from detectandtrack_b200.ops import conv as cv, dense_ops
    g = torch.Generator().manual_seed(13)
    v = torch.randn((777, 256), generator=g) * 10.0 ** (torch.rand((777, 256), generator=g) * 14 - 8)
    v[0, :8] = torch.tensor([65504., 65519., 65520., 1e5, -65504., -65520., -3e38, 3e38])
    pairs = cv.split_bf16(v.cuda())
    got = dense_ops.pairs_to_f16(pairs).cpu()
    hi, lo = pairs[..., :256].float().cpu(), pairs[..., 256:].float().cpu()
    want = (hi + lo).clamp(-65504, 65504).half()
    assert (want.abs() == 65504).sum() > 8 and torch.isfinite(got).all()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


# ------------------------------------------------------------------ every conv plan of the benchmarked step, multi-tile
from test_conv_plan import R50_FPN_3D, REDUCED, conv_args, layer_modes, step_plan  # noqa: E402
from test_conv_reference import conv_ref  # noqa: E402

STEP_CASES = [(l, m) for l in R50_FPN_3D for m in layer_modes(l)]
# DESIGN.md §4, max-norm.  bf16 / f16: the reference gets the same rounded operands, so only the fp32 accumulation order
# differs; bf16 outputs are checked elementwise instead (below).
STEP_TOL = {'bf16': 2e-4, 'f16': 2e-4, 'tf32': 1e-3, 'tf32x3': 1e-4, 'bf16x3': 1e-4}


def _step_tol(layer, mode):
    """STEP_TOL, except tf32x3 beyond K = 8192 products per output: there the bound grows in proportion to K.  The
    tensor cores do not round to nearest when they add into the fp32 accumulator, so the error is biased and grows
    linearly with the wgmma steps per output rather than with their square root.  tf32x3 takes the most steps (8
    products per step, three products per pair): on an H100 its worst error was 0.51e-4 of max|ref| at K = 6912,
    0.89e-4 at 12544 (fc6) and 1.03e-4 at 13824 (res5 3x3x3), and bf16x3 (16 products per step) exactly half of that."""
    K = layer[5] * layer[7][0] * layer[7][1] * layer[7][2]
    return STEP_TOL[mode] * (max(1.0, K / 8192) if mode == 'tf32x3' else 1.0)


def _epilogue(name):
    """(AffineChannel, ReLU) of a layer as the engine fuses it: the ResNet body convs carry a frozen-BN affine (no
    ReLU on the projection shortcut); everything else a bias, ReLU on the RPN / keypoint convs and the FCs."""
    if name.startswith('res'):
        return True, 'branch1' not in name
    return False, name.startswith(('rpn conv', 'fc6', 'keypoint head'))


def _step_inputs(layer, mode, g):
    """Device tensors of one layer at its reduced shape, stored the way the engine stores them in `mode`, and the
    values the kernel reads from them (rounded operands, hi + lo pairs, the stored residual) for the reference."""
    import torch
    from detectandtrack_b200.ops import conv as cv, dense_ops
    name, _, _, _, _, Cin, Cout, k, s, p, rm = layer
    N, T, H, W = REDUCED[name]
    To, Ho, Wo = (T + 2 * p[0] - k[0]) // s[0] + 1, (H + 2 * p[1] - k[1]) // s[1] + 1, (W + 2 * p[2] - k[2]) // s[2] + 1
    dt = cv.F16 if mode == 'f16' else cv.MODE_NAMES[mode]
    split = dt in cv.SPLIT_MODES
    affine, relu = _epilogue(name)
    x = torch.randn((N, T, H, W, Cin), generator=g, device='cuda')
    w = torch.randn((Cout, Cin) + k, generator=g, device='cuda') * (2.0 / (Cin * k[0] * k[1] * k[2])) ** 0.5
    scale = torch.rand(Cout, generator=g, device='cuda') + 0.5 if affine else None
    bias = torch.randn(Cout, generator=g, device='cuda') * 0.1
    res = None
    if rm:
        res = torch.randn((N, To, Ho // rm, Wo // rm, Cout), generator=g, device='cuda')
    wp = cv.pack_weight(w, dt)
    wr = (cv.join_split(wp) if split else wp.float())[:, :, :Cin]            # [taps, Cout, Cin] as the kernel reads it
    wr = wr.reshape(k + (Cout, Cin)).permute(3, 4, 0, 1, 2)
    if mode == 'f16':
        xd = dense_ops.pairs_to_f16(cv.split_bf16(x))                          # the bf16x3h engine's post-hoc input
    elif split:
        xd = cv.split_for(dt, x)
    else:
        xd = {'bf16': x.bfloat16(), 'tf32': cv.round_tf32(x)}[mode]
    xr = cv.join_split(xd) if split else xd.float()
    if res is not None:
        res = cv.split_for(dt, res) if split else (res.bfloat16() if mode == 'bf16' else res)
    resr = None if res is None else (cv.join_split(res) if split else res.float())
    head = Cout % 64 != 0
    out = None
    if head:                                       # final fp32 head outputs, in a row padded to 16 bytes as the engine does
        out = torch.empty((N, To, Ho, Wo, (Cout + 3) // 4 * 4), dtype=torch.float32, device='cuda')
    run = dict(x=xd, w=wp, k=k, s=s, p=p, scale=scale, bias=bias, res=res, rm=rm, relu=relu, dtype=dt, out=out,
               out_f32=True if head else None, split_out=True if mode == 'f16' else None)
    ref = dict(x=xr, w=wr, scale=scale, bias=bias, residual=resr, res_mode=rm, relu=relu)
    return run, ref


def _locate(idx, shape, o, sms):
    """Output element (n, t, h, w, c) -> its (M tile, column tile), linear tile index, and the CTA that ran it."""
    n, t, h, w, c = idx
    _, To, Ho, Wo, Cout = shape
    tw, th, tt = -(-Wo // o.TW), -(-Ho // o.TH), -(-To // o.TT)
    tn = -(-Cout // o.BN)
    m = ((n // o.TB * tt + t // o.TT) * th + h // o.TH) * tw + w // o.TW
    tile = m * tn + c // o.BN
    return ('M tile %d (image %d, frame %d, row %d, column %d tile), column tile %d: tile %d = tile %d of CTA %d'
            % (m, n // o.TB, t // o.TT, h // o.TH, w // o.TW, c // o.BN, tile, tile // sms, tile % sms))


@pytest.mark.parametrize('layer,mode', STEP_CASES, ids=['%s-%s' % (l[0], m) for l, m in STEP_CASES])
def test_step_layer_over_three_waves_vs_fp64(layer, mode, record_property):
    """Every (layer, mode) of the benchmarked step at its reduced shape (test_conv_plan.REDUCED: the step's plan, three
    or more tiles per CTA, a ragged last wave) with the engine's storage and epilogue, against the fp64 tap-sum
    reference on the values the kernel reads.  bf16 outputs: |y - ref| <= 2^-8 |ref| + 2e-4 max|ref| elementwise (half a
    bf16 ulp of output rounding plus the accumulation-order error); the others _step_tol * max|ref|."""
    import zlib
    import torch
    from detectandtrack_b200.ops import conv as cv
    name, Cout = layer[0], layer[6]
    o = step_plan(layer, mode, reduced=True)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert o.tiles / sms >= 3, (name, mode, o.tiles, sms)
    g = torch.Generator(device='cuda').manual_seed(zlib.crc32(('%s/%s' % (name, mode)).encode()))
    run, ref_in = _step_inputs(layer, mode, g)
    y = cv.conv3d(run['x'], run['w'], run['k'], run['s'], run['p'], run['scale'], run['bias'], run['res'], run['rm'],
                  run['relu'], out_f32=run['out_f32'], dtype=run['dtype'], out=run['out'], split_out=run['split_out'])
    if run['out'] is not None:
        y = y[..., :Cout]
    elif run['split_out'] or run['dtype'] in cv.SPLIT_MODES:
        y = cv.join_split(y)
    bf16_out = y.dtype == torch.bfloat16
    ref = conv_ref(ref_in['x'], ref_in['w'], layer[8], layer[9], ref_in['scale'], ref_in['bias'], ref_in['residual'],
                   ref_in['res_mode'], ref_in['relu'])
    assert y.shape == ref.shape
    err = (y.double() - ref).abs()
    den = ref.abs().max().item()
    bound = 2 ** -8 * ref.abs() + 2e-4 * den if bf16_out else _step_tol(layer, mode) * den
    ratio = err / bound
    worst = ratio.max().item()
    record_property('tiles', o.tiles)
    record_property('tiles_per_cta', round(o.tiles / sms, 2))
    record_property('worst_err_over_tol', worst)
    if not worst <= 1.0:                           # NaN too: a wrong shared-memory read can produce it
        idx = [int(i) for i in torch.unravel_index(ratio.argmax(), ratio.shape)]
        pytest.fail('%s %s: error %.3g x the bound at %s, %s' % (name, mode, worst, idx, _locate(idx, y.shape, o, sms)))


@pytest.mark.parametrize('mode', ['bf16x3', 'f16'])
def test_posthoc_fpn_time_major_and_center_frame_vs_fp64(mode):
    """The post-hoc FPN conv as the slice-center link runs it: frames-outermost output (time_major) and the centre
    output frame alone (out_frames=(1, 1)), in bf16x3 and with fp16 operands writing bf16 pairs (bf16x3h)."""
    import torch
    from detectandtrack_b200.ops import conv as cv
    layer = next(l for l in R50_FPN_3D if l[0] == 'fpn post-hoc P4')
    g = torch.Generator(device='cuda').manual_seed(14)
    run, ref_in = _step_inputs(layer, mode, g)
    ref = conv_ref(ref_in['x'], ref_in['w'], layer[8], layer[9], None, ref_in['bias'])
    kw = dict(dtype=run['dtype'], split_out=run['split_out'])
    tm = cv.conv3d(run['x'], run['w'], run['k'], run['s'], run['p'], None, run['bias'], time_major=True, **kw)
    mid = cv.conv3d(run['x'], run['w'], run['k'], run['s'], run['p'], None, run['bias'], out_frames=(1, 1), **kw)
    assert not tm.is_contiguous() and tm[:, 1:2].is_contiguous() and mid.shape[1] == 1
    tol = STEP_TOL[mode] * ref.abs().max().item()
    assert (cv.join_split(tm).double() - ref).abs().max().item() <= tol
    assert (cv.join_split(mid).double() - ref[:, 1:2]).abs().max().item() <= tol


def test_step_convs_are_all_in_the_table(monkeypatch, record_property):
    """One 800 x 1333 clip of the benchmarked R50-FPN-3D config through DetectionEngine.detect in bf16, bf16x3,
    bf16x3h and tf32x3: every conv_tc launch has a plan key (storage, residual kind, BN, schedule length, ring, staging
    and residual split) of a test_conv_plan.R50_FPN_3D layer, which the value test above checks at three or more tiles
    per CTA; every conv1 launch runs a variant test_conv1_packed_rows_vs_torch / test_conv1_exact_fp32_vs_fp64 check."""
    import ctypes as C
    import torch
    import bench
    from detectandtrack_b200 import _lib as L
    from detectandtrack_b200.modeling import params as P
    from detectandtrack_b200.modeling.engine import DetectionEngine
    from detectandtrack_b200.ops import conv as cv
    from test_conv_plan import plan_key, table_plan_keys
    table = table_plan_keys()
    conv1_tested = {('conv1', 0, 1, 0), ('conv1', 0, 0, 0), ('conv1', 1, 1, 0), ('conv1', 0, 0, 1), ('conv1_f32', 0)}
    calls, launched = {'py': 0, 'c': 0}, []
    orig_call = L.call

    def spy(name, *a):
        if name == 'dt_conv3d':
            d = a[0]._obj
            o = L.ConvPlan()
            aligned = a[5] is None or a[5].value % 16 == 0
            assert L.lib().dt_conv_plan(C.byref(d), int(aligned), C.byref(o)) == 0, L.lib().dt_last_error()
            launched.append((plan_key(d.dtype, d.x3, d.out_f32, d.res_mode, o), (d.N, d.Ti, d.Hi, d.Wi, d.Cin, d.Cout)))
        elif name == 'dt_conv1_7x7s2':
            launched.append((('conv1', a[10], a[11], a[13]), None))
        elif name == 'dt_conv1_7x7s2_f32':
            launched.append((('conv1_f32', a[8]), None))
        if name.startswith(('dt_conv3d', 'dt_conv1_7x7s2')):
            calls['c'] += 1
        return orig_call(name, *a)

    def counted(f):
        def wrapped(*a, **kw):
            calls['py'] += 1
            return f(*a, **kw)
        return wrapped
    monkeypatch.setattr(L, 'call', spy)
    for f in ('conv3d', 'conv1_7x7s2', 'conv1_7x7s2_f32'):
        monkeypatch.setattr(cv, f, counted(getattr(cv, f)))
    cfg = bench.bench_cfg(800, 1333)
    blobs, spec = P.random_blobs(cfg)
    frames = torch.from_numpy(bench.synth_frames(1, bench.frames_per_clip(cfg), 800, 1333, 7)).cuda()
    missing = {}
    for mode in ('bf16', 'bf16x3', 'bf16x3h', 'tf32x3'):
        del launched[:]
        eng = DetectionEngine(cfg, blobs, spec, dtype=mode)
        eng.detect(frames)
        torch.cuda.synchronize()
        assert len(launched) > 50
        record_property('launches_' + mode, len(launched))
        record_property('plan_keys_' + mode, len({k for k, _ in launched}))
        for key, shape in launched:
            if key not in table and key not in conv1_tested:
                missing.setdefault(key, (mode, shape))
        del eng
    assert calls['py'] == calls['c']
    assert not missing, missing

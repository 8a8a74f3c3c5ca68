"""GPU: the two consumer warpgroups of conv_tc_kernel take turns over whole tiles (ping-pong, DESIGN.md §3).  Each one steps
over the other's ring stages, staging slots and residual chunks, so these cases aim at what that bookkeeping depends on:
the number of tiles per CTA (odd, or one, where the second warpgroup has none), tiles without a live group next to live
ones, live counts that differ from tile to tile, the residual and top-down rings, plain and [hi | lo] pair outputs.  Each
is checked against the fp64 tap-sum reference on the values the kernel reads, and on integer operands bit for bit."""
import zlib

import pytest

from test_conv_plan import plan
from test_conv_reference import conv_ref
from test_gpu_conv import _exact_mismatch, _integer_operands, with_operands

pytestmark = pytest.mark.gpu

TOL = {'bf16': 2e-4, 'bf16x3': 1e-4, 'tf32x3': 1e-4}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _frames_alternating(sms):
    """Output frames of a 1x1x1 conv with pT = 1 (first and last frame without a live group) such that a CTA's
    consecutive tiles, sms frames apart, step through the frames two at a time: dead and live tiles alternate."""
    for to in range(5, 64):
        if sms % to == 2:
            return to
    return 5


def _case(kind, sms):
    """(N, T, H, W, Cin, Cout, k, stride, pad, res_mode) of one case; H x W = 128 output positions per frame keeps a tile
    to one frame."""
    pw = ((1, 1, 1), (1, 1, 1), (0, 0, 0))
    if kind == 'one tile per CTA':                              # fewer tiles than SMs: warpgroup 1 idles in every CTA
        return (sms - 5, 1, 8, 16, 64, 128) + pw + (0,)
    if kind == 'odd tiles per CTA':                             # 3 or 4 tiles per CTA, ragged last wave
        return (3 * sms + 7, 1, 8, 16, 64, 128) + pw + (0,)
    if kind == 'dead and live tiles':                           # 1x1x1 with pT = 1: frames 0 and To - 1 have no live group
        to = _frames_alternating(sms)
        return (-(-3 * sms // to) + 1, to - 2, 8, 16, 64, 128, (1, 1, 1), (1, 1, 1), (1, 0, 0), 0)
    if kind == '3x3x3 edge rows':                               # live taps differ between edge and inner tiles
        return (7, 3, 40, 64, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0)
    if kind == 'residual':                                      # two column tiles per M tile, residual ring
        return (sms // 2 + 3, 3, 8, 16, 64, 256) + pw + (1,)
    if kind == 'top-down':                                      # FPN top-down add from the (TH/2 x TW/2) box
        return (sms // 8 + 3, 3, 16, 32, 64, 256) + pw + (2,)
    raise KeyError(kind)


# (kind, mode, output): 'plain' is the mode's single output (bf16 rows in bf16, fp32 in the split modes), 'pair' the
# [hi | lo] pair rows of the split modes' intermediate activations, 'f32' fp32 rows from bf16 operands
CASES = [('one tile per CTA', 'bf16', 'plain'), ('one tile per CTA', 'bf16x3', 'pair'),
         ('odd tiles per CTA', 'bf16', 'plain'), ('odd tiles per CTA', 'bf16', 'f32'),
         ('odd tiles per CTA', 'bf16x3', 'pair'), ('odd tiles per CTA', 'bf16x3', 'plain'),
         ('odd tiles per CTA', 'tf32x3', 'pair'),
         ('dead and live tiles', 'bf16', 'f32'), ('dead and live tiles', 'bf16x3', 'pair'),
         ('3x3x3 edge rows', 'bf16', 'plain'), ('3x3x3 edge rows', 'bf16x3', 'pair'), ('3x3x3 edge rows', 'tf32x3', 'pair'),
         ('residual', 'bf16', 'plain'), ('residual', 'bf16', 'f32'), ('residual', 'bf16x3', 'pair'),
         ('top-down', 'bf16', 'plain'), ('top-down', 'bf16x3', 'pair')]


@with_operands('kind,mode,output', CASES, ['%s-%s-%s' % c for c in CASES])
def test_pingpong_vs_fp64(kind, mode, output, operands):
    import torch
    from detectandtrack_b200.ops import conv as cv
    sms = _sms()
    N, T, H, W, Cin, Cout, k, s, p, rm = _case(kind, sms)
    dt = cv.MODE_NAMES[mode]
    split = dt in cv.SPLIT_MODES
    pair = output == 'pair'
    out_f32 = output == 'f32' or (split and not pair) or (pair and mode == 'tf32x3')
    o = plan(N, T, H, W, Cin, Cout, k, s, p, res_mode=rm, out_f32=int(out_f32), dtype=1 if mode == 'tf32x3' else 0,
             x3=(3 if pair else 1) if split else 0)
    per_cta = o.tiles / min(o.tiles, sms)
    if kind == 'one tile per CTA':
        assert o.tiles < sms
    elif kind == 'dead and live tiles':
        assert (o.TT, o.TB, o.tiles % sms != 0) == (1, 1, True) and per_cta >= 3 and o.mma_kblocks < o.tiles * o.kiters
    else:
        assert per_cta >= 3 and o.tiles % sms != 0, (kind, o.tiles, sms)
    if kind == '3x3x3 edge rows':
        assert o.mma_kblocks < o.tiles * o.kiters
    if rm and not out_f32:
        assert o.nrbuf > 0                                      # the residual arrives through the TMA ring

    g = torch.Generator(device='cuda').manual_seed(zlib.crc32(('pingpong/%s/%s/%s' % (kind, mode, output)).encode()))
    To, Ho, Wo = (T + 2 * p[0] - k[0]) // s[0] + 1, (H + 2 * p[1] - k[1]) // s[1] + 1, (W + 2 * p[2] - k[2]) // s[2] + 1
    if operands == 'integer':
        xd, wp, scale, bias, res, ref = _integer_operands(
            g, (N, T, H, W), Cin, Cout, k, mode, True, (N, To, Ho // rm, Wo // rm, Cout) if rm else None,
            torch.float32 if out_f32 else torch.bfloat16, pair)
        ref.update(res_mode=rm, relu=True,
                   kind=('%s pair' % mode[:4]) if pair else ('f32' if out_f32 else 'bf16'))
        y = cv.conv3d(xd, wp, k, s, p, scale, bias, res, rm, True, out_f32=out_f32, dtype=dt, split_out=pair)
        msg = _exact_mismatch(y, ref, s, p, '%s %s %s' % (kind, mode, output), o)
        assert msg is None, msg
    else:
        x = torch.randn((N, T, H, W, Cin), generator=g, device='cuda')
        w = torch.randn((Cout, Cin) + k, generator=g, device='cuda') * (2.0 / (Cin * k[0] * k[1] * k[2])) ** 0.5
        scale = torch.rand(Cout, generator=g, device='cuda') + 0.5
        bias = torch.randn(Cout, generator=g, device='cuda') * 0.5
        wp = cv.pack_weight(w, dt)
        wr = (cv.join_split(wp) if split else wp.float())[:, :, :Cin].reshape(k + (Cout, Cin)).permute(3, 4, 0, 1, 2)
        xd = cv.split_for(dt, x) if split else x.bfloat16()
        xr = cv.join_split(xd) if split else xd.float()
        res = resr = None
        if rm:
            r = torch.randn((N, To, Ho // rm, Wo // rm, Cout), generator=g, device='cuda')
            res = cv.split_for(dt, r) if pair else (r if out_f32 else r.bfloat16())
            resr = cv.join_split(res) if pair else res.float()
        y = cv.conv3d(xd, wp, k, s, p, scale, bias, res, rm, True, out_f32=out_f32, dtype=dt, split_out=pair)
        if pair:
            y = cv.join_split(y)
        ref = conv_ref(xr, wr, s, p, scale, bias, resr, rm, relu=True)
        torch.cuda.synchronize()
        assert y.shape == ref.shape
        err = (y.double() - ref).abs()
        den = ref.abs().max().item()
        if y.dtype == torch.bfloat16:
            bound = 2 ** -8 * ref.abs() + TOL[mode] * den
        else:
            bound = torch.full_like(ref, TOL[mode] * den)
        worst = (err / bound).max().item()
        assert worst <= 1.0, (kind, mode, output, worst)
    if kind == 'dead and live tiles' and output == 'f32':      # frames without a live group: exactly relu(bias)
        dead = torch.cat([y[:, :1], y[:, -1:]], 1)
        assert torch.equal(dead, bias.clamp_min(0).expand_as(dead))

"""GPU: conv_tc_kernel does not issue the (tap, channel chunk) groups whose activation box lies wholly in the zero padding
(DESIGN.md §3).  Such a group's MMAs would only add zeros, so skipping them must not change a single output bit."""
import zlib

import pytest

from test_conv_dead_taps import EDGES, edge_plan
from test_conv_plan import R50_FPN_3D, REDUCED, conv_args, plan
from test_conv_reference import conv_ref
from test_gpu_conv import _exact_mismatch, _integer_operands, _step_inputs, with_operands
from test_gpu_train_grads import test_dgrad_of_every_step_layer_is_bf16_of_the_exact_sum as _dgrad_is_bf16_of_exact_sum
from test_train_plan import D_REDUCED, ROWS, row_dplan

pytestmark = pytest.mark.gpu

LAYERS = {l[0]: l for l in R50_FPN_3D}
PLAN_FIELDS = ('BN', 'TH', 'TW', 'TT', 'TB', 'tiles', 'kiters', 'stages', 'ks', 'ncbuf', 'nrbuf', 'stage_bytes')
# P2-, res4- and keypoint-head-like launches at their REDUCED shapes (the step's plans, three or more tiles per CTA, a
# ragged last wave): the bf16 P2 plan carries two plain groups per ring stage, the split modes three products per group,
# and res4 also runs with a same-shape residual (the TMA residual ring in bf16 / bf16x3, per-thread loads in tf32)
ZERO_CASES = [(n, m, False) for n in ('fpn post-hoc P2', 'res4 3x3x3', 'keypoint head conv')
              for m in ('bf16', 'tf32', 'tf32x3', 'bf16x3', 'f16')] + \
             [('res4 3x3x3', m, True) for m in ('bf16', 'tf32', 'tf32x3', 'bf16x3')]


def _bits(t):
    import torch
    return t.contiguous().view(-1).view(torch.uint8)


@pytest.mark.parametrize('name,mode,res', ZERO_CASES, ids=['%s-%s%s' % (n, m, '-residual' if r else '') for n, m, r in ZERO_CASES])
def test_skipped_taps_equal_physical_zero_padding(name, mode, res):
    """The conv with its padding (dead taps skipped) == the same conv with pad 0 on an input that carries the padding as
    physical zero frames, rows and columns (same output shape and tile, every box reads real zeros, every MMA issued),
    byte for byte."""
    import torch
    import torch.nn.functional as F
    from detectandtrack_b200.ops import conv as cv
    layer = LAYERS[name]
    _, _, _, _, _, Cin, Cout, k, s, p, _ = layer
    N, T, H, W = REDUCED[name]
    g = torch.Generator(device='cuda').manual_seed(zlib.crc32(('zero/%s/%s' % (name, mode)).encode()))
    run, _ = _step_inputs(layer, mode, g)
    resd, rm = None, 0
    if res:
        To, Ho, Wo = (T + 2 * p[0] - k[0]) // s[0] + 1, (H + 2 * p[1] - k[1]) // s[1] + 1, (W + 2 * p[2] - k[2]) // s[2] + 1
        r = torch.randn((N, To, Ho, Wo, Cout), generator=g, device='cuda')
        resd = cv.split_for(run['dtype'], r) if run['dtype'] in cv.SPLIT_MODES else (r.bfloat16() if mode == 'bf16' else r)
        rm = 1
    a = conv_args(layer, mode)
    skip = plan(N, T, H, W, Cin, Cout, k, s, p, res_mode=rm, **a)
    full = plan(N, T + 2 * p[0], H + 2 * p[1], W + 2 * p[2], Cin, Cout, k, s, (0, 0, 0), res_mode=rm, **a)
    for f in PLAN_FIELDS:
        assert getattr(skip, f) == getattr(full, f), (name, mode, f)
    assert full.mma_kblocks == full.tiles * full.kiters and skip.mma_kblocks < full.mma_kblocks
    xz = F.pad(run['x'], (0, 0, p[2], p[2], p[1], p[1], p[0], p[0])).contiguous()
    kw = dict(out_f32=run['out_f32'], dtype=run['dtype'], split_out=run['split_out'])
    y = cv.conv3d(run['x'], run['w'], k, s, p, run['scale'], run['bias'], resd, rm, run['relu'], **kw)
    z = cv.conv3d(xz, run['w'], k, s, (0, 0, 0), run['scale'], run['bias'], resd, rm, run['relu'], **kw)
    torch.cuda.synchronize()
    assert y.shape == z.shape and bool((y != 0).any())
    bad = _bits(y) != _bits(z)
    assert not bool(bad.any()), (name, mode, res, int(bad.sum()))


EDGE_MODES = ('bf16', 'tf32x3', 'bf16x3')
EDGE_TOL = {'bf16': 2e-4, 'tf32x3': 1e-4, 'bf16x3': 1e-4}
EDGE_CASES = [(e, m) for e in EDGES for m in EDGE_MODES]


@with_operands('e,mode', EDGE_CASES, ['%s-%s' % (e[0], m) for e, m in EDGE_CASES])
def test_edge_geometry_vs_fp64(e, mode, operands):
    """The edge geometries of the dead-tap rule (tests/test_conv_dead_taps.EDGES) against the fp64 tap-sum reference on
    the values the kernel reads (on integer operands: bit for bit), with an affine, a bias of both signs and ReLU.  In
    bf16 (fp32 output) a tile without a live group must give exactly relu(scale * 0 + bias)."""
    import torch
    from detectandtrack_b200.ops import conv as cv
    name, N, T, H, W, Cin, Cout, k, s, p, out_t = e
    dt = cv.MODE_NAMES[mode]
    g = torch.Generator(device='cuda').manual_seed(zlib.crc32(('edge/%s/%s' % (name, mode)).encode()))
    frames = out_t if out_t[1] else None
    if operands == 'integer':
        xd, wp, scale, bias, _, ref = _integer_operands(g, (N, T, H, W), Cin, Cout, k, mode, True)
        ref.update(res=[], res_mode=0, relu=True, kind={'bf16': 'f32', 'tf32x3': 'tf32 pair', 'bf16x3': 'bf16 pair'}[mode])
        y = cv.conv3d(xd, wp, k, s, p, scale, bias, None, 0, True, out_f32=True if mode == 'bf16' else None, dtype=dt,
                      out_frames=frames)
        msg = _exact_mismatch(y, ref, s, p, '%s %s' % (name, mode), edge_plan(e, mode, out_f32=1), frames)
        assert msg is None, msg
    else:
        x = torch.randn((N, T, H, W, Cin), generator=g, device='cuda')
        w = torch.randn((Cout, Cin) + k, generator=g, device='cuda') * (2.0 / (Cin * k[0] * k[1] * k[2])) ** 0.5
        scale = torch.rand(Cout, generator=g, device='cuda') + 0.5
        bias = torch.randn(Cout, generator=g, device='cuda') * 0.5
        wp = cv.pack_weight(w, dt)
        if dt in cv.SPLIT_MODES:
            xd = cv.split_for(dt, x)
            xr, wr = cv.join_split(xd), cv.join_split(wp)[:, :, :Cin]
        else:
            xd = x.bfloat16()
            xr, wr = xd.float(), wp.float()[:, :, :Cin]
        wr = wr.reshape(k + (Cout, Cin)).permute(3, 4, 0, 1, 2)
        y = cv.conv3d(xd, wp, k, s, p, scale, bias, None, 0, True, out_f32=True if mode == 'bf16' else None, dtype=dt,
                      out_frames=frames)
        if dt in cv.SPLIT_MODES:
            y = cv.join_split(y)
        ref = conv_ref(xr, wr, s, p, scale, bias, relu=True)
        if out_t[1]:
            ref = ref[:, out_t[0]:out_t[0] + out_t[1]]
        torch.cuda.synchronize()
        assert y.shape == ref.shape
        err = (y.double() - ref).abs().max().item()
        assert err <= EDGE_TOL[mode] * ref.abs().max().item(), (name, mode, err)
    if mode == 'bf16' and k[0] == 1 and p[0] > 0:      # the padded output frames read only zeros: no live group
        dead = torch.cat([y[:, :p[0]], y[:, -p[0]:]], 1)
        want = bias.clamp_min(0).expand_as(dead)
        assert torch.equal(dead, want), name
        o = edge_plan(e, mode)
        assert o.mma_kblocks < o.tiles * o.kiters


def test_padded_3x3x3_dgrad_is_bf16_of_the_exact_sum():
    """The input gradient of a 3x3x3 layer runs through the same kernel, so its dead taps are skipped too: the res4
    branch2b dgrad on integer operands is still bf16 of the exact sum, bit for bit."""
    r = ROWS['res4 branch2b']
    o = row_dplan(r, D_REDUCED[r[0]])
    assert o.mma_kblocks < o.tiles * o.kiters
    _dgrad_is_bf16_of_exact_sum(r)

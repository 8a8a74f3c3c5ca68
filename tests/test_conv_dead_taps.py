"""CPU: the MMA k-blocks a dt_conv3d launch issues once the taps whose activation box lies wholly in the zero padding
are skipped (dt_conv_plan.mma_kblocks), against a brute-force count over every tile and tap box."""
import numpy as np
import pytest

from test_conv_plan import R50_FPN_3D, conv_args, layer_modes, plan

# (name, N, T, H, W, Cin, Cout, k, stride, pad, out_t): the edge geometries of the dead-tap rule, also run on the GPU
# against the fp64 reference (tests/test_gpu_conv_dead_taps.py)
EDGES = [
    ('T1 kT3 pT1', 2, 1, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (0, 0)),
    ('T2 kT3 pT1', 2, 2, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (0, 0)),
    ('T3 kT3 pT1', 2, 3, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (0, 0)),
    ('T5 kT3 pT1', 2, 5, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (0, 0)),
    ('kT3 pT2', 2, 3, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (2, 1, 1), (0, 0)),
    ('1x1x1 pT1 (all-dead tiles)', 2, 3, 12, 20, 64, 128, (1, 1, 1), (1, 1, 1), (1, 0, 0), (0, 0)),
    ('temporal stride 2', 2, 5, 12, 20, 64, 64, (3, 3, 3), (2, 1, 1), (1, 1, 1), (0, 0)),
    ('out_t (0, 1)', 2, 3, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (0, 1)),
    ('out_t (1, 1)', 2, 3, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (1, 1)),
    ('out_t (2, 1)', 2, 3, 12, 20, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (2, 1)),
    ('frame-stacked', 2, 5, 5, 7, 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), (0, 0)),
    ('image-stacked rows', 67, 1, 14, 14, 64, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), (0, 0)),
    ('strided 3x3 s2', 1, 1, 33, 47, 64, 64, (1, 3, 3), (1, 2, 2), (0, 1, 1), (0, 0)),
    ('strided 3x3x3 s2', 2, 3, 30, 44, 64, 128, (3, 3, 3), (1, 2, 2), (1, 1, 1), (0, 0)),
    ('pointwise s2', 1, 3, 25, 42, 256, 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), (0, 0)),
]
EDGE_MODES = ('bf16', 'tf32', 'bf16x3', 'tf32x3')


def edge_plan(e, mode, **kw):
    name, N, T, H, W, Cin, Cout, k, s, p, out_t = e
    a = dict(dtype={'bf16': 0, 'tf32': 1, 'bf16x3': 0, 'tf32x3': 1}[mode], x3=3 if mode.endswith('x3') else 0,
             out_f32=int(mode.startswith('tf32')))
    a.update(kw)
    return plan(N, T, H, W, Cin, Cout, k, s, p, out_t=out_t, **a)


def brute_kblocks(N, T, H, W, Cin, Cout, k, s, p, out_t, o, dtype, x3):
    """Every (M tile, tap): the tap is live when some position of the tile's whole box (the rows a ragged edge tile has
    beyond the output included) reads an input coordinate inside [0, size) in each of T, H and W."""
    To_full = (T + 2 * p[0] - k[0]) // s[0] + 1
    first, To = (out_t[0], out_t[1]) if out_t[1] else (0, To_full)
    Ho, Wo = (H + 2 * p[1] - k[1]) // s[1] + 1, (W + 2 * p[2] - k[2]) // s[2] + 1

    def dim(out, ext, first, s, pad, k, size):              # [tile, tap]: the box reaches the input
        tiles = -(-out // ext)
        pos = first + np.arange(tiles)[:, None, None] * ext + np.arange(ext)[None, None, :]
        c = pos * s - pad + np.arange(k)[None, :, None]
        return ((c >= 0) & (c < size)).any(axis=2)
    lt = dim(To, o.TT, first, s[0], p[0], k[0], T)
    lh = dim(Ho, o.TH, 0, s[1], p[1], k[1], H)
    lw = dim(Wo, o.TW, 0, s[2], p[2], k[2], W)
    live = lt[:, None, None, :, None, None] & lh[None, :, None, None, :, None] & lw[None, None, :, None, None, :]
    kchunks = -(-Cin // (32 if dtype == 1 else 64))
    nmma = 3 if x3 & 1 else 1
    return float(live.sum()) * -(-N // o.TB) * -(-Cout // o.BN) * kchunks * nmma


STEP = [(l, m) for l in R50_FPN_3D for m in layer_modes(l)]


@pytest.mark.parametrize('layer,mode', STEP, ids=['%s-%s' % (l[0], m) for l, m in STEP])
def test_step_layer_issues_the_brute_force_count(layer, mode):
    name, N, T, H, W, Cin, Cout, k, s, p, rm = layer
    a = conv_args(layer, mode)
    o = plan(N, T, H, W, Cin, Cout, k, s, p, res_mode=rm, **a)
    assert o.mma_kblocks == brute_kblocks(N, T, H, W, Cin, Cout, k, s, p, (0, 0), o, a['dtype'], a['x3'])
    assert o.mma_kblocks <= o.tiles * o.kiters
    if k == (1, 1, 1):
        assert o.mma_kblocks == o.tiles * o.kiters, name


@pytest.mark.parametrize('mode', EDGE_MODES)
@pytest.mark.parametrize('e', EDGES, ids=[e[0] for e in EDGES])
def test_edge_geometry_issues_the_brute_force_count(e, mode):
    o = edge_plan(e, mode)
    dtype = 1 if mode.startswith('tf32') else 0
    x3 = 3 if mode.endswith('x3') else 0
    assert o.mma_kblocks == brute_kblocks(*e[1:], o, dtype, x3), (e[0], mode)


def test_edge_geometries_cover_what_they_name():
    by = {e[0]: e for e in EDGES}
    o = edge_plan(by['1x1x1 pT1 (all-dead tiles)'], 'bf16')        # frames 0 and 4 of 5 read only padding
    assert o.TT == 1 and o.mma_kblocks == o.tiles * o.kiters * 3 / 5
    assert edge_plan(by['frame-stacked'], 'bf16').TT > 1
    o = edge_plan(by['image-stacked rows'], 'bf16')
    assert o.TB > 1 and o.TH == 1
    o = edge_plan(by['T1 kT3 pT1'], 'bf16')                          # one frame: only kt = 1 is live
    assert o.mma_kblocks * 3 <= o.tiles * o.kiters
    o = edge_plan(by['pointwise s2'], 'bf16')
    assert o.mma_kblocks == o.tiles * o.kiters                       # pointwise: nothing is skipped
    for n in ('out_t (0, 1)', 'out_t (2, 1)'):                       # the first / last frame: one temporal tap of three dead
        o = edge_plan(by[n], 'bf16')
        assert o.mma_kblocks * 3 / 2 >= o.tiles * o.kiters > o.mma_kblocks
    o = edge_plan(by['out_t (1, 1)'], 'bf16')
    assert o.mma_kblocks > 7 / 9 * o.tiles * o.kiters               # centre frame: only the H / W borders


def test_pinned_savings_of_the_step():
    """post-hoc P2 (8 x 16 spatial tiles, T = 3 padded by one frame): 7 of the 9 (output frame, temporal tap) pairs are
    live and no spatial tap dies (200 and 336 are multiples of 8 and 16, every box reaches the map); the keypoint head
    (1 x 14 rows x 9 RoIs): the first and last of the 14 rows lose one of their three kh taps, 40 / 42."""
    p2 = next(l for l in R50_FPN_3D if l[0] == 'fpn post-hoc P2')
    for mode in layer_modes(p2):
        o = plan(*p2[1:10], **conv_args(p2, mode))
        assert (o.TH, o.TW, o.TT, o.TB) == (8, 16, 1, 1)
        assert o.mma_kblocks * 9 == o.tiles * o.kiters * 7, mode
    kp = next(l for l in R50_FPN_3D if l[0] == 'keypoint head conv')
    o = plan(*kp[1:10], **conv_args(kp, 'bf16x3'))
    assert (o.TH, o.TW, o.TT, o.TB) == (1, 14, 1, 9)
    assert o.mma_kblocks * 42 == o.tiles * o.kiters * 40

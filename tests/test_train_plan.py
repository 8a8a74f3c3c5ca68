"""CPU: the plans of every filter- and input-gradient launch of the benchmarked keypoint R-CNN training step (2 clips, T=3,
800x1344 blob, R50-FPN-3D, BATCH_SIZE_PER_IM 512, 8 stacked keypoint convs), through the host-only planning queries
dt_wgrad_nhwc_plan / dt_conv_plan.  The reduced shapes below are what tests/test_gpu_train_grads.py runs; these tests pin
that each one takes the step's plan.  Also: the fp64 tap-sum references of that file against torch autograd, and the host
alignment checks of the backward entry points."""
import ctypes as C
import os

import pytest

from detectandtrack_b200 import _lib as L
from test_conv_plan import PLAN_FIELDS, SMS, plan, plan_key

W_FIELDS = ('TW', 'TH', 'TT', 'TB', 'BN', 'taps', 'tiles_m', 'tiles_n', 'ksplit')

# One row per distinct gradient launch of the step: (name, N, T, Hi, Wi, Cin, Cout, k, stride, launches, bias).
# (N, T, Hi, Wi) is the layer's INPUT (the saved activation); the output grid is ceil(Hi / s) x ceil(Wi / s).  launches:
# 'w' filter gradient (dt_wgrad_nhwc), 'd' input gradient (dt_conv3d with the flipped, transposed filter; strided layers
# then dt_scatter_stride2).  Cout is the stored (padded) channel count: the RPN output conv 5A = 15 -> rpn_ld 16, the
# class / box FC 5 * 2 = 10 -> cb_ld 16, the sub-pixel keypoint conv 4 * 17 = 68 -> kp_ld 72.  The FCs are 1x1 convs over
# the RoI axis (W = 2 x 512 sampled RoIs); the keypoint head runs on 2 x 128 keypoint RoIs of 14 x 14.
S2 = (2, 2)
TRAIN_STEP = [
    ('res3_0 branch2a s2', 2, 3, 200, 336, 256, 128, (1, 1, 1), S2, 'w', False),       # res2 is frozen: no dgrad
    ('res3_0 branch1 s2', 2, 3, 200, 336, 256, 512, (1, 1, 1), S2, 'w', False),
    ('res3 branch2a', 2, 3, 100, 168, 512, 128, (1, 1, 1), (1, 1), 'wd', False),
    ('res3 branch2b', 2, 3, 100, 168, 128, 128, (3, 3, 3), (1, 1), 'wd', False),
    ('res3 branch2c', 2, 3, 100, 168, 128, 512, (1, 1, 1), (1, 1), 'wd', False),
    ('res4_0 branch2a s2', 2, 3, 100, 168, 512, 256, (1, 1, 1), S2, 'wd', False),
    ('res4_0 branch1 s2', 2, 3, 100, 168, 512, 1024, (1, 1, 1), S2, 'wd', False),
    ('res4 branch2a', 2, 3, 50, 84, 1024, 256, (1, 1, 1), (1, 1), 'wd', False),
    ('res4 branch2b', 2, 3, 50, 84, 256, 256, (3, 3, 3), (1, 1), 'wd', False),
    ('res4 branch2c', 2, 3, 50, 84, 256, 1024, (1, 1, 1), (1, 1), 'wd', False),
    ('res5_0 branch2a s2', 2, 3, 50, 84, 1024, 512, (1, 1, 1), S2, 'wd', False),
    ('res5_0 branch1 s2', 2, 3, 50, 84, 1024, 2048, (1, 1, 1), S2, 'wd', False),
    ('res5 branch2a', 2, 3, 25, 42, 2048, 512, (1, 1, 1), (1, 1), 'wd', False),
    ('res5 branch2b', 2, 3, 25, 42, 512, 512, (3, 3, 3), (1, 1), 'wd', False),
    ('res5 branch2c', 2, 3, 25, 42, 512, 2048, (1, 1, 1), (1, 1), 'wd', False),
    ('fpn lateral P5', 2, 3, 25, 42, 2048, 256, (1, 1, 1), (1, 1), 'wd', True),
    ('fpn lateral P4', 2, 3, 50, 84, 1024, 256, (1, 1, 1), (1, 1), 'wd', True),
    ('fpn lateral P3', 2, 3, 100, 168, 512, 256, (1, 1, 1), (1, 1), 'wd', True),
    ('fpn lateral P2', 2, 3, 200, 336, 256, 256, (1, 1, 1), (1, 1), 'w', True),        # C2's producer is frozen
    ('fpn post-hoc P5', 2, 3, 25, 42, 256, 256, (3, 3, 3), (1, 1), 'wd', True),
    ('fpn post-hoc P4', 2, 3, 50, 84, 256, 256, (3, 3, 3), (1, 1), 'wd', True),
    ('fpn post-hoc P3', 2, 3, 100, 168, 256, 256, (3, 3, 3), (1, 1), 'wd', True),
    ('fpn post-hoc P2', 2, 3, 200, 336, 256, 256, (3, 3, 3), (1, 1), 'wd', True),
    ('rpn conv P2', 2, 1, 200, 336, 256, 256, (1, 3, 3), (1, 1), 'wd', True),
    ('rpn conv P3', 2, 1, 100, 168, 256, 256, (1, 3, 3), (1, 1), 'wd', True),
    ('rpn conv P4', 2, 1, 50, 84, 256, 256, (1, 3, 3), (1, 1), 'wd', True),
    ('rpn conv P5', 2, 1, 25, 42, 256, 256, (1, 3, 3), (1, 1), 'wd', True),
    ('rpn conv P6', 2, 1, 13, 21, 256, 256, (1, 3, 3), (1, 1), 'wd', True),
    ('rpn out P2', 2, 1, 200, 336, 256, 16, (1, 1, 1), (1, 1), 'wd', True),
    ('rpn out P3', 2, 1, 100, 168, 256, 16, (1, 1, 1), (1, 1), 'wd', True),
    ('rpn out P4', 2, 1, 50, 84, 256, 16, (1, 1, 1), (1, 1), 'wd', True),
    ('rpn out P5', 2, 1, 25, 42, 256, 16, (1, 1, 1), (1, 1), 'wd', True),
    ('rpn out P6', 2, 1, 13, 21, 256, 16, (1, 1, 1), (1, 1), 'wd', True),
    ('fc6', 1, 1, 1, 1024, 12544, 1024, (1, 1, 1), (1, 1), 'wd', True),
    ('fc7', 1, 1, 1, 1024, 1024, 1024, (1, 1, 1), (1, 1), 'wd', True),
    ('cls + bbox', 1, 1, 1, 1024, 1024, 16, (1, 1, 1), (1, 1), 'wd', True),
    ('keypoint conv1', 256, 1, 14, 14, 256, 512, (1, 3, 3), (1, 1), 'wd', True),
    ('keypoint conv', 256, 1, 14, 14, 512, 512, (1, 3, 3), (1, 1), 'wd', True),
    ('keypoint lowres (sub-pixel deconv)', 256, 1, 14, 14, 512, 72, (1, 3, 3), (1, 1), 'wd', True),
]
ROWS = {r[0]: r for r in TRAIN_STEP}


def out_hw(Hi, Wi, s):
    return (Hi + s[0] - 1) // s[0], (Wi + s[1] - 1) // s[1]


def wgrad_plan(N, T, Hi, Wi, Cin, Cout, k, s=(1, 1)):
    """dt_wgrad_nhwc_plan with the arguments TrainConv.backward passes (leading dims = the stored channel counts)."""
    Ho, Wo = out_hw(Hi, Wi, s)
    o = L.WgradPlan()
    rc = L.lib().dt_wgrad_nhwc_plan(Cout, Cin, N, T, Ho, Wo, Hi, Wi, Cout, Cin, k[0], k[1], k[2], s[0], s[1], C.byref(o))
    assert rc == 0, L.lib().dt_last_error()
    return o


def dgrad_plan(N, T, Hi, Wi, Cin, Cout, k, s=(1, 1)):
    """dt_conv_plan of the input-gradient conv: the layer's output gradient (Cout channels, on the output grid) convolved
    with the flipped, transposed filter into Cin bf16 channels (a strided 1x1 conv runs on the coarse grid)."""
    Ho, Wo = out_hw(Hi, Wi, s)
    return plan(N, T, Ho, Wo, Cout, Cin, k, p=tuple(x // 2 for x in k), res_mode=0, out_f32=0, dtype=0, x3=0)


def dgrad_key(o):
    return plan_key(0, 0, 0, 0, o)


def wgrad_key(o):
    return tuple(getattr(o, f) for f in W_FIELDS)


def split_ranges(o):
    """[k0, k1) of every CTA of one (tap, tile) unit, exactly as wgrad_nhwc_kernel computes them."""
    total = o.nW * o.nH * o.nT * o.nN
    return [(total * ks // o.ksplit, total * (ks + 1) // o.ksplit) for ks in range(o.ksplit)]


def dead_blocks(o, T, dt, k0, k1):
    """k-blocks of [k0, k1) whose tap-shifted frames (frame offset dt) all lie outside the clip (wgrad_nhwc_kernel live())."""
    per_t = o.nW * o.nH
    n = 0
    for kb in range(k0, k1):
        t0 = ((kb // per_t) % o.nT) * o.TT + dt
        n += not (t0 + o.TT > 0 and t0 < T)
    return n


def padding_kinds(o, T, kT):
    """(some split range lies wholly in temporally padded k-blocks, some range straddles a padded run) over the taps."""
    whole = straddle = False
    for dt in range(-(kT // 2), kT // 2 + 1):
        if dt == 0:
            continue
        for k0, k1 in split_ranges(o):
            d = dead_blocks(o, T, dt, k0, k1)
            whole |= d == k1 - k0 > 0
            straddle |= 0 < d < k1 - k0
    return whole, straddle


# (N, T, Hi, Wi) of each wgrad row for tests/test_gpu_train_grads.py: the step's plan in every field but the per-axis box
# counts, so the same box, column tile, tile counts and K split.  A kT = 3 layer keeps whether some split range lies wholly
# in temporally padded frames and whether some range straddles a padded run.  Where the full-size ranges are unequal
# (the k-block count is not a multiple of ksplit), so are these; with T = 3 and ksplit = 3 they are equal at every size.
W_REDUCED = {
    'res3_0 branch2a s2': (2, 3, 37, 336),
    'res3_0 branch1 s2': (2, 3, 21, 336),
    'res3 branch2a': (2, 3, 11, 168),
    'res3 branch2b': (2, 3, 4, 168),
    'res3 branch2c': (2, 3, 11, 168),
    'res4_0 branch2a s2': (6, 3, 7, 168),
    'res4_0 branch1 s2': (2, 3, 7, 168),
    'res4 branch2a': (2, 3, 19, 84),
    'res4 branch2b': (2, 3, 10, 24),
    'res4 branch2c': (2, 3, 19, 84),
    'res5_0 branch2a s2': (5, 3, 3, 84),
    'res5_0 branch1 s2': (2, 3, 3, 84),
    'res5 branch2a': (2, 3, 9, 13),
    'res5 branch2b': (2, 3, 2, 42),
    'res5 branch2c': (2, 3, 9, 13),
    'fpn lateral P5': (2, 3, 5, 42),
    'fpn lateral P4': (2, 3, 19, 84),
    'fpn lateral P3': (4, 3, 4, 168),
    'fpn lateral P2': (1, 3, 11, 336),
    'fpn post-hoc P5': (2, 3, 9, 13),
    'fpn post-hoc P4': (2, 3, 10, 24),
    'fpn post-hoc P3': (2, 3, 4, 83),
    'fpn post-hoc P2': (2, 3, 4, 169),
    'rpn conv P2': (1, 1, 8, 336),
    'rpn conv P3': (4, 1, 4, 168),
    'rpn conv P4': (2, 1, 12, 84),
    'rpn conv P5': (2, 1, 21, 42),
    'rpn conv P6': (2, 1, 13, 21),
    'rpn out P2': (1, 1, 49, 336),
    'rpn out P3': (2, 1, 49, 168),
    'rpn out P4': (2, 1, 49, 84),
    'rpn out P5': (2, 1, 25, 42),
    'rpn out P6': (2, 1, 13, 21),
    'fc6': (1, 1, 1, 200),
    'fc7': (1, 1, 1, 769),
    'cls + bbox': (1, 1, 1, 961),
    'keypoint conv1': (15, 1, 14, 14),
    'keypoint conv': (15, 1, 14, 14),
    'keypoint lowres (sub-pixel deconv)': (15, 1, 14, 14),
}

# (N, T, Hi, Wi) of each dgrad row: the step's conv plan (PLAN_FIELDS), at least three tiles per CTA on 132 SMs and a ragged
# last wave.  Rows whose step launch has fewer than three waves of tiles take more images or rows (no plan field changes).
D_REDUCED = {
    'res3 branch2a': (1, 3, 25, 168),
    'res3 branch2b': (2, 3, 49, 168),
    'res3 branch2c': (2, 3, 49, 168),
    'res4_0 branch2a s2': (17, 3, 5, 168),
    'res4_0 branch1 s2': (17, 3, 5, 168),
    'res4 branch2a': (1, 3, 25, 84),
    'res4 branch2b': (2, 3, 49, 84),
    'res4 branch2c': (2, 3, 49, 84),
    'res5_0 branch2a s2': (50, 3, 1, 84),
    'res5_0 branch1 s2': (50, 3, 1, 84),
    'res5 branch2a': (1, 3, 25, 42),
    'res5 branch2b': (4, 3, 25, 42),
    'res5 branch2c': (4, 3, 25, 42),
    'fpn lateral P5': (1, 3, 25, 42),
    'fpn lateral P4': (1, 3, 25, 84),
    'fpn lateral P3': (1, 3, 25, 168),
    'fpn post-hoc P5': (8, 3, 25, 42),
    'fpn post-hoc P4': (2, 3, 49, 84),
    'fpn post-hoc P3': (1, 3, 49, 168),
    'fpn post-hoc P2': (1, 3, 25, 336),
    'rpn conv P2': (1, 1, 73, 336),
    'rpn conv P3': (11, 1, 13, 168),
    'rpn conv P4': (10, 1, 28, 84),
    'rpn conv P5': (25, 1, 22, 42),
    'rpn conv P6': (91, 1, 13, 21),
    'rpn out P2': (1, 1, 73, 336),
    'rpn out P3': (11, 1, 13, 168),
    'rpn out P4': (10, 1, 28, 84),
    'rpn out P5': (25, 1, 22, 42),
    'rpn out P6': (91, 1, 13, 21),
    'fc6': (1, 1, 1, 513),
    'fc7': (1, 1, 1, 6273),
    'cls + bbox': (1, 1, 1, 6273),
    'keypoint conv1': (129, 1, 14, 14),
    'keypoint conv': (65, 1, 14, 14),
    'keypoint lowres (sub-pixel deconv)': (65, 1, 14, 14),
}
W_ROWS = [r for r in TRAIN_STEP if 'w' in r[9]]
D_ROWS = [r for r in TRAIN_STEP if 'd' in r[9]]


def row_wplan(r, shape=None):
    N, T, H, W = shape or r[1:5]
    return wgrad_plan(N, T, H, W, r[5], r[6], r[7], r[8])


def row_dplan(r, shape=None):
    N, T, H, W = shape or r[1:5]
    return dgrad_plan(N, T, H, W, r[5], r[6], r[7], r[8])


def positions(r, shape):
    N, T, H, W = shape
    Ho, Wo = out_hw(H, W, r[8])
    return N * T * Ho * Wo


# ---------------------------------------------------------------------------------------------------- fp64 references
def wgrad_ref(gz, x, k, s=(1, 1)):
    """dW [taps, Cout, Cin] = sum over output positions of gz[pos, co] * x[pos shifted by the tap, ci]: one GEMM per tap over
    the zero-padded, shifted input (NDHWC, any float dtype; computed in float64)."""
    import torch
    import torch.nn.functional as F
    gz, x = gz.double(), x.double()
    N, T, Ho, Wo, Cout = gz.shape
    if s != (1, 1):
        assert k == (1, 1, 1)
        xs = x[:, :, ::s[0], ::s[1]]
        return (gz.reshape(-1, Cout).t() @ xs.reshape(-1, x.shape[-1]))[None]
    pT, pH, pW = (kk // 2 for kk in k)
    xp = F.pad(x, (0, 0, pW, pW, pH, pH, pT, pT))
    g2 = gz.reshape(-1, Cout).t()
    out = []
    for kt in range(k[0]):
        for kh in range(k[1]):
            for kw in range(k[2]):
                xs = xp[:, kt:kt + T, kh:kh + Ho, kw:kw + Wo]
                out.append(g2 @ xs.reshape(-1, x.shape[-1]))
    return torch.stack(out)


def dgrad_ref(gz, w, k, in_hw, s=(1, 1)):
    """dx [N, T, Hi, Wi, Cin] of y = conv(x, w) ('same' padding k // 2, or a strided 1x1 conv) for the output gradient gz
    [N, T, Ho, Wo, Cout]; w [taps, Cout, Cin] (the packed forward order).  float64: dx[q] = sum over taps of gz[q - d_tap] @ w[tap]."""
    import torch
    import torch.nn.functional as F
    gz, w = gz.double(), w.double()
    N, T, Ho, Wo, Cout = gz.shape
    Cin = w.shape[-1]
    if s != (1, 1):
        dx = torch.zeros((N, T) + tuple(in_hw) + (Cin,), dtype=torch.float64, device=gz.device)
        dx[:, :, ::s[0], ::s[1]] = (gz.reshape(-1, Cout) @ w[0]).reshape(N, T, Ho, Wo, Cin)
        return dx
    pT, pH, pW = (kk // 2 for kk in k)
    gp = F.pad(gz, (0, 0, pW, pW, pH, pH, pT, pT))
    dx = torch.zeros((N * T * Ho * Wo, Cin), dtype=torch.float64, device=gz.device)
    tap = 0
    for kt in range(k[0]):
        for kh in range(k[1]):
            for kw in range(k[2]):
                a, b, c = 2 * pT - kt, 2 * pH - kh, 2 * pW - kw
                dx += gp[:, a:a + T, b:b + Ho, c:c + Wo].reshape(-1, Cout) @ w[tap]
                tap += 1
    return dx.reshape(N, T, Ho, Wo, Cin)


# ---------------------------------------------------------------------------------------------------- tests
def test_no_wave_override():
    assert 'DT_WGRAD_WAVES' not in os.environ, 'DT_WGRAD_WAVES changes the K split of every wgrad plan'


def test_table_lists_exactly_the_launches_the_step_makes():
    assert len(ROWS) == len(TRAIN_STEP)
    no_dgrad = {r[0] for r in TRAIN_STEP if 'd' not in r[9]}
    assert no_dgrad == {'res3_0 branch2a s2', 'res3_0 branch1 s2', 'fpn lateral P2'}
    assert set(W_REDUCED) == {r[0] for r in W_ROWS} and set(D_REDUCED) == {r[0] for r in D_ROWS}
    A, classes, K = 3, 2, 17                                   # anchors per level, classes, keypoints
    pads = {'rpn out': (5 * A + 7) // 8 * 8, 'cls + bbox': (5 * classes + 7) // 8 * 8, 'keypoint lowres': (4 * K + 7) // 8 * 8}
    for r in TRAIN_STEP:
        for pre, ld in pads.items():
            if r[0].startswith(pre):
                assert r[6] == ld, r
        assert r[6] % 8 == 0 and r[5] % 8 == 0, r


@pytest.mark.parametrize('r', W_ROWS, ids=[r[0] for r in W_ROWS])
def test_reduced_wgrad_shape_keeps_the_step_plan(r):
    red = W_REDUCED[r[0]]
    full, o = row_wplan(r), row_wplan(r, red)
    for f in W_FIELDS:
        assert getattr(o, f) == getattr(full, f), (r[0], f, getattr(o, f), getattr(full, f))
    assert o.grid == o.taps * o.tiles_m * o.tiles_n * o.ksplit and o.smem_bytes <= 227 * 1024
    assert positions(r, red) <= positions(r, r[1:5]), r[0]
    total, ftotal = o.nW * o.nH * o.nT * o.nN, full.nW * full.nH * full.nT * full.nN
    assert total >= 4 * o.ksplit
    if full.ksplit >= 2 and ftotal % full.ksplit:
        assert total % o.ksplit, (r[0], 'full-size split ranges are unequal, reduced ones must be too', total, o.ksplit)
    if r[7][0] == 3:
        assert padding_kinds(o, red[1], 3) == padding_kinds(full, r[2], 3), r[0]


def test_the_step_splits_and_pads_where_the_reduced_shapes_must():
    """The split branches the GPU tests must reach are reached at full size: ksplit >= 2 with unequal ranges, and res3's
    3x3x3 (ksplit 10 against padded runs of 1/6 of the k-blocks) has a split range made only of padded frames."""
    o = row_wplan(ROWS['res3 branch2b'])
    assert o.ksplit == 10 and o.nN * o.nT == 3 and padding_kinds(o, 3, 3) == (True, True)
    unequal = [r[0] for r in W_ROWS for o in [row_wplan(r)] if o.ksplit >= 2 and (o.nW * o.nH * o.nT * o.nN) % o.ksplit]
    assert len(unequal) >= 20, unequal
    assert any(row_wplan(r).TB > 1 for r in W_ROWS if r[0].startswith('keypoint'))      # boxes spanning several images


@pytest.mark.parametrize('r', D_ROWS, ids=[r[0] for r in D_ROWS])
def test_reduced_dgrad_shape_keeps_the_step_plan_over_three_waves(r):
    red = D_REDUCED[r[0]]
    full, o = row_dplan(r), row_dplan(r, red)
    for f in PLAN_FIELDS:
        assert getattr(o, f) == getattr(full, f), (r[0], f, getattr(o, f), getattr(full, f))
    assert (o.TT > 1, o.TB > 1) == (full.TT > 1, full.TB > 1), r[0]
    assert o.tiles >= 3 * SMS and o.tiles % SMS != 0, (r[0], o.tiles)
    assert positions(r, red) <= positions(r, r[1:5]) or full.tiles < 3 * SMS, r[0]


def test_wgrad_plan_rejects_bad_arguments():
    o = L.WgradPlan()
    lib = L.lib()
    assert lib.dt_wgrad_nhwc_plan(64, 60, 1, 1, 8, 8, 8, 8, 64, 60, 1, 3, 3, 1, 1, C.byref(o)) != 0
    assert b'bad shape' in lib.dt_last_error()
    assert lib.dt_wgrad_nhwc_plan(64, 64, 1, 1, 8, 8, 8, 8, 64, 64, 1, 3, 3, 2, 2, C.byref(o)) != 0
    assert b'pointwise' in lib.dt_last_error()
    assert lib.dt_wgrad_nhwc_plan(64, 64, 1, 1, 8, 8, 8, 8, 64, 64, 1, 3, 3, 1, 1, None) != 0


REF_CASES = [((2, 3, 5, 6), 8, 16, (3, 3, 3), (1, 1)), ((1, 1, 4, 7), 16, 8, (1, 3, 3), (1, 1)),
             ((2, 2, 7, 9), 8, 8, (1, 1, 1), (2, 2)), ((1, 3, 6, 6), 8, 24, (1, 1, 1), (2, 2)), ((3, 1, 1, 10), 16, 8, (1, 1, 1), (1, 1))]


@pytest.mark.parametrize('case', range(len(REF_CASES)))
def test_fp64_references_match_autograd(case):
    """The references of the GPU gradient tests equal torch autograd of F.conv3d in float64 (strided 1x1 included)."""
    import torch
    import torch.nn.functional as F
    (N, T, H, W), Cin, Cout, k, s = REF_CASES[case]
    g = torch.Generator().manual_seed(case)
    x = torch.randn((N, T, H, W, Cin), generator=g, dtype=torch.float64, requires_grad=True)
    w5 = torch.randn((Cout, Cin) + k, generator=g, dtype=torch.float64, requires_grad=True)
    pad = tuple(kk // 2 for kk in k)
    y = F.conv3d(x.permute(0, 4, 1, 2, 3), w5, None, (1,) + s, pad)
    gz = torch.randn(y.shape, generator=g, dtype=torch.float64)
    y.backward(gz)
    gzl = gz.permute(0, 2, 3, 4, 1).contiguous()
    wp = w5.detach().permute(2, 3, 4, 0, 1).reshape(-1, Cout, Cin)
    dW = wgrad_ref(gzl, x.detach(), k, s)
    assert torch.allclose(dW, w5.grad.permute(2, 3, 4, 0, 1).reshape(-1, Cout, Cin), rtol=1e-12, atol=1e-12)
    dx = dgrad_ref(gzl, wp, k, (H, W), s)
    assert torch.allclose(dx, x.grad, rtol=1e-12, atol=1e-12)


def _p(a):
    return C.c_void_p(a)


ALIGN_CASES = [
    ('dt_wgrad_nhwc', (_p(0x1000), 64, _p(0x1000), 64, 1, 1, 8, 8, 8, 8, 64, 64, 1, 1, 1, 1, 1, _p(0x1004), None), b'8-byte'),
    ('dt_wgrad', (_p(0x1000), _p(0x1000), 1, 1, 8, 8, 64, 64, 1, 1, 1, _p(0x1004), None), b'8-byte'),
    ('dt_bias_grad', (_p(0x1008), 10, 16, 16, _p(0x1000), None), b'16-byte'),
    ('dt_bwd_pointwise', (_p(0x1000), _p(0x1008), None, None, 10, 16, _p(0x1000), None), b'16-byte'),
    ('dt_bwd_pointwise2', (_p(0x1000), None, _p(0x1000), None, 10, 16, _p(0x1000), None, _p(0x1002), None), b'16-byte'),
    ('dt_upsample_add_bwd', (_p(0x1000), None, 1, 4, 4, 16, _p(0x1008), None), b'16-byte'),
    ('dt_scatter_stride2', (_p(0x1004), 1, 4, 4, 8, 8, 16, _p(0x1000), None), b'16-byte'),
    ('dt_embed_frame', (_p(0x1000), 2, 3, 64, 1, _p(0x1008), None), b'16-byte'),
    ('dt_grad_join_f32', (None, _p(0x1008), 16, _p(0x1000), None), b'16-byte'),
]


@pytest.mark.parametrize('name,args,msg', ALIGN_CASES, ids=[c[0] for c in ALIGN_CASES])
def test_misaligned_vector_operands_are_rejected_on_the_host(name, args, msg):
    """A view at an odd offset inside a flat buffer would fault the device's vector loads / reductions: every entry point
    rejects it before any CUDA call (the pointers here are never dereferenced)."""
    lib = L.lib()
    rc = getattr(lib, name)(*args)
    err = lib.dt_last_error()
    assert rc != 0 and msg in err and b'aligned' in err, (name, err)
    with pytest.raises(RuntimeError, match=name):
        L.check(rc, name)


def test_roi_align_bwd_rejects_a_misaligned_level_accumulator():
    lib = L.lib()
    fp = (C.c_void_p * 2)(0x1000, 0x1008)
    Hs, Ws = (C.c_int * 2)(4, 2), (C.c_int * 2)(4, 2)
    sc = (C.c_float * 2)(0.25, 0.125)
    rc = lib.dt_roi_align_bwd(_p(0x1000), fp, Hs, Ws, sc, 2, 2, 16, _p(0x1000), 5, None, 1, 1, _p(0x1000), 7, 2, None)
    assert rc != 0 and b'level 1 must be 16-byte aligned' in lib.dt_last_error(), lib.dt_last_error()

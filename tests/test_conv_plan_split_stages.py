"""CPU: the ring depth, schedule table and M tile of every split-operand (bf16x3 / tf32x3) conv launch of the
benchmarked workloads, through dt_conv_plan.  A split ring stage is one whole (tap, channel chunk), 64 KiB at BN = 128.
With two stages the 64 KiB refill of one does not land while the other's MMAs run, so a K-heavy split launch wants
three.  The k-block schedule table shares the 227 KiB with the ring, at 8 bytes per (tap, channel chunk) entry."""
import pytest

from test_conv_dead_taps import brute_kblocks
from test_conv_plan import R50_FPN_3D, SMEM_BUDGET, conv_args, layer_modes, plan, step_plan
from test_conv_plan_workloads import TABLES

C_BYTES = 128 * 128                      # one staged output / residual chunk: 128 rows x 128 B
BAR_BYTES = 384                          # mbarriers

WORKLOADS = {'r50fpn3d': (R50_FPN_3D, layer_modes)}
WORKLOADS.update({wl: (rows, modes) for wl, (rows, _, modes) in TABLES.items()})
LAUNCHES = [(wl, l, m) for wl, (rows, modes) in WORKLOADS.items() for l in rows for m in modes(l)]
SPLIT = [(wl, l, m) for wl, l, m in LAUNCHES if conv_args(l, m)['x3'] & 1]

# Ring stages of every split launch at the parent commit (24-byte schedule entries), as (tf32x3, bf16x3); None where the
# layer does not run in that mode (the bf16x3 keypoint head is a Winograd GEMM in the 2-D step).
PARENT_STAGES = {
    'r50fpn3d': {
        'res2 first 1x1 reduce': (3, 3),
        'res2 branch1': (2, 2),
        'res2 1x1 reduce': (3, 3),
        'res2 3x3': (3, 3),
        'res2 1x1 expand + shortcut': (2, 2),
        'res3 branch1 s2': (3, 3),
        'res3 branch2a s2': (3, 3),
        'res3 1x1 reduce': (3, 3),
        'res3 3x3x3': (3, 3),
        'res3 expand + shortcut': (3, 2),
        'res4 branch2a s2': (3, 3),
        'res4 1x1 reduce': (3, 3),
        'res4 3x3x3': (2, 3),
        'res4 expand + shortcut': (3, 2),
        'res5 branch2a s2': (3, 3),
        'res5 1x1 reduce': (3, 3),
        'res5 3x3x3': (2, 2),
        'res5 expand + shortcut': (3, 2),
        'fpn lateral P5': (3, 3),
        'fpn lateral P4 + top-down': (3, 3),
        'fpn lateral P3 + top-down': (3, 3),
        'fpn lateral P2 + top-down': (3, 2),
        'fpn post-hoc P2': (2, 3),
        'fpn post-hoc P3': (2, 3),
        'fpn post-hoc P4': (2, 3),
        'fpn post-hoc P5': (2, 3),
        'rpn conv P2': (3, 3),
        'rpn conv P6': (3, 3),
        'rpn heads P2': (4, 4),
        'fc6': (2, 2),
        'cls + bbox': (4, 4),
        'keypoint head conv': (2, 3),
        'keypoint lowres (sub-pixel deconv)': (2, 3),
    },
    'r50fpn2d': {
        'res2_0 branch1': (2, 2),
        'res2_0 branch2a': (3, 3),
        'res2 3x3': (3, 3),
        'res2 1x1 expand + shortcut': (2, 2),
        'res2 1x1 reduce': (3, 3),
        'res3_0 branch1 s2': (3, 3),
        'res3_0 branch2a s2': (3, 3),
        'res3 3x3': (3, 3),
        'res3 expand + shortcut': (3, 2),
        'res3 1x1 reduce': (3, 3),
        'res4_0 branch1 s2': (3, 3),
        'res4_0 branch2a s2': (3, 3),
        'res4 3x3': (3, 3),
        'res4 expand + shortcut': (3, 2),
        'res4 1x1 reduce': (3, 3),
        'res5_0 branch1 s2': (3, 3),
        'res5_0 branch2a s2': (3, 3),
        'res5 3x3': (2, 3),
        'res5 expand + shortcut': (3, 2),
        'res5 1x1 reduce': (3, 3),
        'fpn lateral P5': (3, 3),
        'fpn lateral P4 + top-down': (3, 3),
        'fpn lateral P3 + top-down': (3, 3),
        'fpn lateral P2 + top-down': (3, 2),
        'fpn post-hoc P2': (3, 3),
        'fpn post-hoc P3': (3, 3),
        'fpn post-hoc P4': (3, 3),
        'fpn post-hoc P5': (3, 3),
        'rpn conv P2': (3, 3),
        'rpn conv P3': (3, 3),
        'rpn conv P4': (3, 3),
        'rpn conv P5': (3, 3),
        'rpn conv P6': (3, 3),
        'rpn heads P2': (4, 4),
        'rpn heads P3': (4, 4),
        'rpn heads P4': (4, 4),
        'rpn heads P5': (4, 4),
        'rpn heads P6': (4, 4),
        'fc6': (2, 2),
        'fc7': (3, 3),
        'cls + bbox': (4, 4),
        'keypoint head conv1': (3, None),
        'keypoint head conv': (2, None),
        'keypoint lowres (sub-pixel deconv)': (2, 3),
    },
    'r18tube': {
        'res2 3x3': (3, 3),
        'res2 3x3 + shortcut': (3, 2),
        'res3_0 branch1 s2': (2, 2),
        'res3_0 branch2a 3x3x3 s2': (3, 3),
        'res3 3x3x3 + shortcut': (3, 2),
        'res3_1 branch2a 3x3x3': (3, 3),
        'res4_0 branch1 s2': (3, 2),
        'res4_0 branch2a 3x3x3 s2': (3, 3),
        'res4 3x3x3 + shortcut': (2, 2),
        'res4_1 branch2a 3x3x3': (2, 3),
        'rpn conv 3x3x3': (2, 3),
        'rpn heads': (4, 4),
        'res5_0 branch1 (RoI)': (3, 3),
        'res5_0 branch2a (RoI)': (3, 3),
        'res5 3x3 + shortcut (RoI)': (2, 2),
        'res5_1 branch2a (RoI)': (2, 3),
        'cls + bbox': (4, 4),
        'keypoint head conv1 3x3x3': (2, 3),
        'keypoint head conv 3x3x3': (2, 2),
        'keypoint lowres (sub-pixel deconv)': (2, 3),
    },
}

# fp32-pair outputs (tf32x3) keep both (hi, lo) staging slot pairs, and so two stages, above this many groups
F32_PAIRS_KEEP_STAGING = 110


def tab_bytes(groups):
    """The schedule table: one 8-byte entry per group plus padding, in whole 128-byte lines."""
    return ((groups + 2) * 8 + 127) // 128 * 128


def ids(cases):
    return ['%s-%s-%s' % (wl, l[0], m) for wl, l, m in cases]


@pytest.mark.parametrize('wl,layer,mode', SPLIT, ids=ids(SPLIT))
def test_k_heavy_split_launches_take_three_stages(wl, layer, mode):
    o = step_plan(layer, mode)
    if o.kiters < 12 or o.nrbuf > 0:
        return                           # K-light, or a split residual layer (two stages, one residual pair)
    groups = o.kiters // 3
    a = conv_args(layer, mode)
    if a['x3'] & 2 and a['out_f32'] and groups > F32_PAIRS_KEEP_STAGING:
        assert (o.stages, o.ncbuf) == (2, 4), (o.stages, o.ncbuf)
    else:
        assert o.stages >= 3, (o.kiters, o.stages, o.ncbuf)


@pytest.mark.parametrize('wl,layer,mode', SPLIT, ids=ids(SPLIT))
def test_no_split_launch_has_fewer_stages_than_the_parent(wl, layer, mode):
    parent = PARENT_STAGES[wl][layer[0]][('tf32x3', 'bf16x3').index(mode)]
    assert step_plan(layer, mode).stages >= parent


@pytest.mark.parametrize('wl,layer,mode', LAUNCHES, ids=ids(LAUNCHES))
def test_smem_bytes_is_ring_staging_barriers_and_table(wl, layer, mode):
    a = conv_args(layer, mode)
    o = step_plan(layer, mode)
    groups = o.kiters // (3 if a['x3'] & 1 else 1)
    pair = 2 if a['x3'] & 2 else 1       # split output: a residual slot is a (hi, lo) chunk pair
    assert o.smem_bytes == (o.stages * o.stage_bytes + (o.ncbuf + pair * o.nrbuf) * C_BYTES + BAR_BYTES +
                            tab_bytes(groups))
    assert o.smem_bytes <= SMEM_BUDGET


def test_res5_and_fc6_take_a_third_stage_in_bf16x3():
    by = {l[0]: l for l in R50_FPN_3D}
    for name, groups, slack in (('res5 3x3x3', 27 * 8, 896), ('fc6', 196, 1024)):
        o = step_plan(by[name], 'bf16x3')
        assert o.kiters == 3 * groups and tab_bytes(groups) == {216: 1792, 196: 1664}[groups]
        assert (o.BN, o.stages, o.ncbuf, o.nrbuf) == (128, 3, 2, 0), (name, o.stages, o.ncbuf)
        assert SMEM_BUDGET - o.smem_bytes == slack, (name, o.smem_bytes)


@pytest.mark.parametrize('mode', ('bf16x3', 'tf32x3'))
@pytest.mark.parametrize('name', ('res5 3x3x3', 'fpn post-hoc P5'))
def test_split_res5_and_p5_keep_frames_apart_to_skip_dead_temporal_taps(name, mode):
    """On the 25 x 42 map with T = 3, three rows of one frame issue fewer k-blocks than one row of the three stacked
    frames, whose temporal taps all stay live.  Live (kt, kh, kw) taps summed over the M tiles of one clip and column
    tile: 7 (over 3 frames) * 26 (over 9 row tiles) * 3 = 546, against 3 * 73 (over 25 rows) * 3 = 657 stacked."""
    layer = next(l for l in R50_FPN_3D if l[0] == name)
    N, T, H, W, Cin, Cout, k, s, p, rm = layer[1:]
    a = conv_args(layer, mode)
    o = step_plan(layer, mode)
    assert (o.TH, o.TW, o.TT, o.TB) == (3, 42, 1, 1)
    assert o.mma_kblocks == brute_kblocks(N, T, H, W, Cin, Cout, k, s, p, (0, 0), o, a['dtype'], a['x3'])
    per_tap = 3 * Cin // (32 if a['dtype'] == 1 else 64) * N * (Cout // o.BN)    # k-blocks of one live tap, all clips
    assert o.mma_kblocks == 546 * per_tap
    stacked = step_plan(layer, 'bf16' if mode == 'bf16x3' else 'tf32')       # plain operands keep the frame stack
    assert (stacked.TH, stacked.TW, stacked.TT, stacked.TB) == (1, 42, 3, 1)
    assert stacked.mma_kblocks == 657 * per_tap // 3                          # one MMA k-block per group


def test_tf32x3_pairs_keep_their_staging_split():
    """fp32-pair outputs trade a staging slot pair for a third stage up to 110 groups, as with 24-byte entries."""
    o = plan(1, 3, 100, 168, 128, 128, (3, 3, 3), p=(1, 1, 1), out_f32=1, dtype=1, x3=3)      # res3: 108 groups
    assert o.kiters == 3 * 108 and (o.stages, o.ncbuf) == (3, 2)
    o = plan(1, 3, 50, 84, 256, 256, (3, 3, 3), p=(1, 1, 1), out_f32=1, dtype=1, x3=3)        # res4: 216 groups
    assert o.kiters == 3 * 216 and (o.stages, o.ncbuf) == (2, 4)
    o = plan(1, 3, 25, 42, 512, 512, (3, 3, 3), p=(1, 1, 1), x3=3)                          # bf16x3 res5: 216 groups
    assert o.kiters == 3 * 216 and (o.stages, o.ncbuf) == (3, 2)

"""CPU: the host-side planning of dt_conv3d (tile picker, column tile, smem split), through dt_conv_plan — no GPU
needed.  Checks the plan of every conv shape of the benchmarked R50-FPN-3D step (8 clips, 800x1344 blob)."""
import ctypes as C

import pytest

from detectandtrack_b200 import _lib as L

SMEM_BUDGET = 227 * 1024


def plan(N, T, H, W, Cin, Cout, k, s=(1, 1, 1), p=(0, 0, 0), res_mode=0, out_f32=0, dtype=0, x3=0, out_t=(0, 0)):
    d = L.ConvDesc(N=N, Ti=T, Hi=H, Wi=W, Cin=Cin, Cout=Cout, kT=k[0], kH=k[1], kW=k[2], sT=s[0], sH=s[1], sW=s[2],
                   pT=p[0], pH=p[1], pW=p[2], in_ld=0, w_ld=0, out_ld=0, res_ld=0, dtype=dtype, out_f32=out_f32, relu=1,
                   res_mode=res_mode, x3=x3, in_lo_off=0, out_lo_off=0, res_lo_off=0, out_round_tf32=0, out_time_major=0,
                   out_t_first=out_t[0], out_t_count=out_t[1])
    o = L.ConvPlan()
    rc = L.lib().dt_conv_plan(C.byref(d), 1, C.byref(o))
    assert rc == 0, L.lib().dt_last_error()
    return o


# (name, N, T, H, W, Cin, Cout, k, stride, pad, res_mode): the distinct conv shapes of one bench step.  The res3..res5
# first blocks stride their 1x1 branch2a (RESNETS.STRIDE_1X1, the default the bench config keeps).
R50_FPN_3D = [
    ('res2 first 1x1 reduce', 8, 3, 200, 336, 64, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res2 branch1', 8, 3, 200, 336, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res2 1x1 reduce', 8, 3, 200, 336, 256, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res2 3x3', 8, 3, 200, 336, 64, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('res2 1x1 expand + shortcut', 8, 3, 200, 336, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('res3 branch1 s2', 8, 3, 200, 336, 256, 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), 0),
    ('res3 branch2a s2', 8, 3, 200, 336, 256, 128, (1, 1, 1), (1, 2, 2), (0, 0, 0), 0),
    ('res3 1x1 reduce', 8, 3, 100, 168, 512, 128, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res3 3x3x3', 8, 3, 100, 168, 128, 128, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('res3 expand + shortcut', 8, 3, 100, 168, 128, 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('res4 branch2a s2', 8, 3, 100, 168, 512, 256, (1, 1, 1), (1, 2, 2), (0, 0, 0), 0),
    ('res4 1x1 reduce', 8, 3, 50, 84, 1024, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res4 3x3x3', 8, 3, 50, 84, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('res4 expand + shortcut', 8, 3, 50, 84, 256, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('res5 branch2a s2', 8, 3, 50, 84, 1024, 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), 0),
    ('res5 1x1 reduce', 8, 3, 25, 42, 2048, 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res5 3x3x3', 8, 3, 25, 42, 512, 512, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('res5 expand + shortcut', 8, 3, 25, 42, 512, 2048, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('fpn lateral P5', 8, 3, 25, 42, 2048, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('fpn lateral P4 + top-down', 8, 3, 50, 84, 1024, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2),
    ('fpn lateral P3 + top-down', 8, 3, 100, 168, 512, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2),
    ('fpn lateral P2 + top-down', 8, 3, 200, 336, 256, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2),
    ('fpn post-hoc P2', 8, 3, 200, 336, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('fpn post-hoc P3', 8, 3, 100, 168, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('fpn post-hoc P4', 8, 3, 50, 84, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('fpn post-hoc P5', 8, 3, 25, 42, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('rpn conv P2', 8, 1, 200, 336, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('rpn conv P6', 8, 1, 13, 21, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('rpn heads P2', 8, 1, 200, 336, 256, 15, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('fc6', 1, 1, 1, 8000, 12544, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('cls + bbox', 1, 1, 1, 8000, 1024, 10, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('keypoint head conv', 832, 1, 14, 14, 512, 512, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('keypoint lowres (sub-pixel deconv)', 832, 1, 14, 14, 512, 68, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
]

# (N, T, H, W) of each layer for the value tests of tests/test_gpu_conv.py: the same plan as in the step, and enough tiles
# that every CTA of a 132-SM H100 walks at least three of them, the last wave ragged.  Only N, T, H, W change.  Two layers
# run fewer than three waves in the step (the coarsest RPN level, the 8000-row class / box FC); their shapes take
# more images / rows instead, which changes no plan field.
REDUCED = {
    'res2 first 1x1 reduce': (1, 3, 55, 336),
    'res2 branch1': (1, 3, 31, 336),
    'res2 1x1 reduce': (1, 3, 55, 336),
    'res2 3x3': (1, 3, 55, 336),
    'res2 1x1 expand + shortcut': (1, 3, 31, 336),
    'res3 branch1 s2': (1, 3, 51, 336),
    'res3 branch2a s2': (1, 3, 199, 336),
    'res3 1x1 reduce': (1, 3, 100, 168),
    'res3 3x3x3': (1, 3, 100, 168),
    'res3 expand + shortcut': (1, 3, 26, 168),
    'res4 branch2a s2': (2, 3, 97, 168),
    'res4 1x1 reduce': (2, 3, 49, 84),
    'res4 3x3x3': (2, 3, 49, 84),
    'res4 expand + shortcut': (1, 3, 26, 84),
    'res5 branch2a s2': (4, 3, 49, 84),
    'res5 1x1 reduce': (4, 3, 25, 42),
    'res5 3x3x3': (4, 3, 25, 42),
    'res5 expand + shortcut': (1, 3, 25, 42),
    'fpn lateral P5': (8, 3, 25, 42),
    'fpn lateral P4 + top-down': (2, 3, 50, 84),
    'fpn lateral P3 + top-down': (1, 3, 50, 168),
    'fpn lateral P2 + top-down': (1, 3, 32, 336),
    'fpn post-hoc P2': (1, 3, 31, 336),
    'fpn post-hoc P3': (1, 3, 49, 168),
    'fpn post-hoc P4': (2, 3, 49, 84),
    'fpn post-hoc P5': (8, 3, 25, 42),
    'rpn conv P2': (1, 1, 79, 336),
    'rpn conv P6': (91, 1, 13, 21),
    'rpn heads P2': (1, 1, 148, 336),
    'fc6': (1, 1, 1, 6273),
    'cls + bbox': (1, 1, 1, 50689),
    'keypoint head conv': (67, 1, 14, 14),
    'keypoint lowres (sub-pixel deconv)': (253, 1, 14, 14),
}
GROWN = ('rpn conv P6', 'cls + bbox')

MODES = ('bf16', 'tf32', 'tf32x3', 'bf16x3')
PLAN_FIELDS = ('BN', 'kiters', 'stages', 'ks', 'ncbuf', 'nrbuf', 'stage_bytes')
SMS = 132                                       # H100 SXM


def layer_modes(layer):
    """The engine modes of a layer; the four post-hoc FPN convs also run with fp16 operands (the bf16x3h mode)."""
    return MODES + (('f16',) if layer[0].startswith('fpn post-hoc') else ())


def conv_args(layer, mode):
    """dtype / x3 / out_f32 of the layer as the engine launches it in `mode`: bf16 writes bf16, tf32 fp32, the split
    modes [hi | lo] pairs (residual pairs too); head outputs (Cout not a multiple of 64) are plain fp32 in every mode,
    and the fp16-operand post-hoc convs write bf16 pairs for their bf16x3 consumers."""
    head = layer[6] % 64 != 0
    return {'bf16': dict(dtype=0, x3=0, out_f32=int(head)),
            'tf32': dict(dtype=1, x3=0, out_f32=1),
            'tf32x3': dict(dtype=1, x3=1 if head else 3, out_f32=1),
            'bf16x3': dict(dtype=0, x3=1 if head else 3, out_f32=int(head)),
            'f16': dict(dtype=2, x3=2, out_f32=0)}[mode]


def step_plan(layer, mode, reduced=False, shapes=None):
    """The plan of a table row at its step shape, or at its reduced shape in `shapes` (default REDUCED)."""
    name, N, T, H, W, Cin, Cout, k, s, p, rm = layer
    if reduced:
        N, T, H, W = (REDUCED if shapes is None else shapes)[name]
    return plan(N, T, H, W, Cin, Cout, k, s, p, res_mode=rm, **conv_args(layer, mode))


def plan_key(dtype, x3, out_f32, res_mode, o):
    """What selects a conv_tc_kernel code path and schedule: operand / output storage, residual kind, and the plan."""
    return (dtype, x3, out_f32, res_mode) + tuple(getattr(o, f) for f in PLAN_FIELDS)


@pytest.mark.parametrize('layer', R50_FPN_3D, ids=[l[0] for l in R50_FPN_3D])
def test_plan_of_every_bench_layer_fits_and_fills_the_mma(layer):
    name, N, T, H, W, Cin, Cout, k, s, p, rm = layer
    o = plan(N, T, H, W, Cin, Cout, k, s, p, res_mode=rm)
    assert o.TB * o.TT * o.TH * o.TW <= 128
    assert o.smem_bytes <= SMEM_BUDGET and o.stages >= 2 and o.ks in (1, 2) and o.stages * o.ks >= 3
    assert o.BN in (32, 64, 128)                                                # 64 x BN register accumulators per warpgroup
    assert o.ncbuf in (1, 2, 4) and o.nrbuf in (0, 2, 4)
    assert o.kiters == k[0] * k[1] * k[2] * ((Cin + 63) // 64)
    floor = 0.84 if (H, W) == (13, 21) else 0.9                                  # P6 is 273 positions per image
    assert o.useful_rows >= floor, (name, o.useful_rows, (o.TH, o.TW, o.TT, o.TB))
    assert o.tiles >= 1


@pytest.mark.parametrize('layer', R50_FPN_3D, ids=[l[0] for l in R50_FPN_3D])
def test_reduced_shape_keeps_the_step_plan_over_three_waves(layer):
    """The value tests run each layer at its REDUCED shape: that launch must take the step's plan (ring, staging and
    residual split, schedule length), the same top-down tile parity and stacking kind, and give every CTA at least
    three tiles with a ragged last wave, so that the state a CTA carries from tile to tile is exercised."""
    name, N, T, H, W = layer[:5]
    n, t, h, w = REDUCED[name]
    assert (n <= N and t <= T and h <= H and w <= W) or name in GROWN
    for mode in layer_modes(layer):
        full, red = step_plan(layer, mode), step_plan(layer, mode, reduced=True)
        for f in PLAN_FIELDS:
            assert getattr(red, f) == getattr(full, f), (name, mode, f, getattr(red, f), getattr(full, f))
        if layer[10] == 2:                               # even tile: TMA box of the coarser map, odd: per-thread loads
            assert (red.TH % 2, red.TW % 2) == (full.TH % 2, full.TW % 2), (name, mode)
        assert (red.TT > 1, red.TB > 1) == (full.TT > 1, full.TB > 1), (name, mode)
        assert red.tiles >= 3 * SMS and red.tiles % SMS != 0, (name, mode, red.tiles)


def test_small_maps_stack_frames_or_images():
    o = plan(832, 1, 14, 14, 512, 512, (1, 3, 3), p=(0, 1, 1))
    assert (o.TH, o.TW, o.TT, o.TB) == (1, 14, 1, 9) and o.useful_rows > 0.97      # 14x14 RoI maps: 9 images per tile
    o = plan(8, 3, 25, 42, 512, 512, (3, 3, 3), p=(1, 1, 1))
    assert (o.TH, o.TW, o.TT, o.TB) == (1, 42, 3, 1)                                # res5: three frames per tile
    o = plan(8, 3, 200, 336, 256, 256, (3, 3, 3), p=(1, 1, 1))
    assert (o.TH, o.TW, o.TT, o.TB) == (8, 16, 1, 1) and o.useful_rows == 1.0       # big maps: plain spatial tiles
    o = plan(8, 3, 25, 42, 512, 512, (3, 3, 3), s=(2, 1, 1), p=(1, 1, 1))
    assert o.TT == 1                                                                # temporal stride: no frame stacking


def test_residual_layers_get_the_tma_ring_and_narrow_column_tiles():
    o = plan(8, 3, 200, 336, 64, 256, (1, 1, 1), res_mode=1)
    assert o.BN == 128 and o.nrbuf == 4 and o.ncbuf == 4
    o = plan(8, 3, 200, 336, 64, 256, (1, 1, 1), res_mode=0)
    assert o.BN == 128 and o.nrbuf == 0 and o.stages == 5                         # no ring: its room goes to operand stages
    o = plan(8, 3, 200, 336, 256, 256, (1, 1, 1), res_mode=2)                       # even tile: top-down add via the ring
    assert o.nrbuf == 4 and o.TH % 2 == 0 and o.TW % 2 == 0
    o = plan(8, 3, 200, 336, 64, 256, (1, 1, 1), res_mode=1, out_f32=1, dtype=1)    # fp32 modes keep per-thread loads
    assert o.nrbuf == 0


def test_k_heavy_layers_get_a_deep_ring_and_narrow_tiles_two_kblocks_per_stage():
    o = plan(8, 3, 200, 336, 256, 256, (3, 3, 3), p=(1, 1, 1))
    assert o.BN == 128 and o.ks == 2 and o.stages >= 3 and o.ncbuf == 2
    o = plan(8, 3, 100, 168, 128, 128, (3, 3, 3), p=(1, 1, 1))
    assert o.BN == 128 and o.ks == 2 and o.stages >= 3
    o = plan(8, 3, 200, 336, 64, 64, (1, 3, 3), p=(0, 1, 1))
    assert o.BN == 64 and o.ks == 2 and o.ncbuf == 2


def test_output_frame_range_and_x3_plans():
    full = plan(8, 3, 200, 336, 256, 256, (3, 3, 3), p=(1, 1, 1))
    one = plan(8, 3, 200, 336, 256, 256, (3, 3, 3), p=(1, 1, 1), out_t=(1, 1))
    assert one.tiles * 3 == full.tiles and one.kiters == full.kiters
    x3 = plan(1, 3, 50, 84, 256, 256, (3, 3, 3), p=(1, 1, 1), out_f32=1, dtype=1, x3=3)
    assert x3.kiters == 3 * 27 * 8 and x3.ncbuf == 4 and x3.smem_bytes <= SMEM_BUDGET     # 32 tf32 per k-block, hi/lo products


def test_plan_rejects_bad_arguments():
    d = L.ConvDesc(N=0, Ti=1, Hi=1, Wi=1, Cin=1, Cout=1, kT=1, kH=1, kW=1, sT=1, sH=1, sW=1)
    o = L.ConvPlan()
    assert L.lib().dt_conv_plan(C.byref(d), 1, C.byref(o)) != 0
    assert b'bad shape' in L.lib().dt_last_error()


def test_workspace_queries_are_host_only_and_consistent():
    """dt_nms_workspace_bytes / dt_rpn_workspace_bytes need no device: sizes grow with the problem and cover the
    documented contents (one u32 key per anchor per image for the RPN top-k)."""
    lib = L.lib()
    a, b = C.c_size_t(0), C.c_size_t(0)
    assert lib.dt_nms_workspace_bytes(1, 1000, C.byref(a)) == 0 and lib.dt_nms_workspace_bytes(8, 8192, C.byref(b)) == 0
    assert 0 < a.value < b.value
    assert lib.dt_nms_workspace_bytes(-1, 10, C.byref(a)) != 0 and b'bad args' in lib.dt_last_error()
    assert b.value >= 8 * 8192 * (4 + 128 * 8 + 1)                              # order + 64-bit mask rows + flags
    Hs = (C.c_int * 5)(200, 100, 50, 25, 13)
    Ws = (C.c_int * 5)(336, 168, 84, 42, 21)
    n = C.c_size_t(0)
    assert lib.dt_rpn_workspace_bytes(8, 5, Hs, Ws, 3, C.byref(n)) == 0
    anchors = sum(h * w for h, w in zip(Hs, Ws)) * 3
    assert 8 * anchors * 4 <= n.value <= 8 * anchors * 4 + 5 * 256

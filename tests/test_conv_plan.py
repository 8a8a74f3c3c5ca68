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


# (name, N, T, H, W, Cin, Cout, k, stride, pad, res_mode): the distinct conv shapes of one bench step
R50_FPN_3D = [
    ('res2 1x1 reduce', 8, 3, 200, 336, 256, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('res2 3x3', 8, 3, 200, 336, 64, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('res2 1x1 expand + shortcut', 8, 3, 200, 336, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('res3 branch1 s2', 8, 3, 200, 336, 256, 512, (1, 1, 1), (1, 2, 2), (0, 0, 0), 0),
    ('res3 3x3x3', 8, 3, 100, 168, 128, 128, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('res3 expand + shortcut', 8, 3, 100, 168, 128, 512, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('res4 3x3x3', 8, 3, 50, 84, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('res4 expand + shortcut', 8, 3, 50, 84, 256, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('res5 3x3x3', 8, 3, 25, 42, 512, 512, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('res5 expand + shortcut', 8, 3, 25, 42, 512, 2048, (1, 1, 1), (1, 1, 1), (0, 0, 0), 1),
    ('fpn lateral P2 + top-down', 8, 3, 200, 336, 256, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), 2),
    ('fpn post-hoc P2', 8, 3, 200, 336, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('fpn post-hoc P5', 8, 3, 25, 42, 256, 256, (3, 3, 3), (1, 1, 1), (1, 1, 1), 0),
    ('rpn conv P2', 8, 1, 200, 336, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('rpn conv P6', 8, 1, 13, 21, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('rpn heads P2', 8, 1, 200, 336, 256, 15, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('fc6', 1, 1, 1, 8000, 12544, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), 0),
    ('keypoint head conv', 832, 1, 14, 14, 512, 512, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
    ('keypoint lowres (sub-pixel deconv)', 832, 1, 14, 14, 512, 68, (1, 3, 3), (1, 1, 1), (0, 1, 1), 0),
]


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

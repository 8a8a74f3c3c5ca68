"""CPU: dt_conv_plan of the bf16x3 (split-operand) convs of the benchmarked R50-FPN-3D step.  A split ring stage holds
one whole (tap, channel chunk): the hi and lo boxes of the activations and of the weights, each fetched once for the
three products A_hi*W_hi, A_lo*W_hi, A_hi*W_lo."""
import pytest

from test_conv_plan import R50_FPN_3D, SMEM_BUDGET, plan

A_BOX = 128 * 128                       # 128 rows x 128 B


def plan_x3(layer):
    """The layer as the engine runs it in bf16x3: [hi | lo] bf16 pair outputs, except the heads' final fp32 outputs
    (Cout % 64 != 0)."""
    name, N, T, H, W, Cin, Cout, k, s, p, rm = layer
    pair_out = Cout % 64 == 0
    return plan(N, T, H, W, Cin, Cout, k, s, p, res_mode=rm if pair_out else 0, out_f32=0 if pair_out else 1,
                dtype=0, x3=3 if pair_out else 1)


@pytest.mark.parametrize('layer', R50_FPN_3D, ids=[l[0] for l in R50_FPN_3D])
def test_split_plan_fits_two_stages_of_whole_groups(layer):
    name, N, T, H, W, Cin, Cout, k, s, p, rm = layer
    o = plan_x3(layer)
    assert o.smem_bytes <= SMEM_BUDGET and o.stages >= 2, (name, o.stages, o.smem_bytes)
    assert o.ks == 1 and o.stage_bytes == 2 * A_BOX + 2 * o.BN * 128, (name, o.ks, o.stage_bytes)
    assert o.kiters == 3 * k[0] * k[1] * k[2] * ((Cin + 63) // 64)               # MMA k-blocks: 3 per group


def test_split_residual_layers_keep_the_output_staging_and_one_residual_pair():
    # res* expand + shortcut and FPN lateral + top-down: two 64 KiB stages, two (hi, lo) staging slot pairs, one
    # residual slot pair.  The P3 / P4 laterals have odd tiles (3 x 42): their top-down add reads the residual per
    # thread, so they keep no residual ring and plan like any K-heavy split layer (three stages, one staging pair)
    for layer in R50_FPN_3D:
        if layer[10]:
            o = plan_x3(layer)
            if layer[10] == 2 and (o.TH % 2 or o.TW % 2):
                assert (o.BN, o.stages, o.ncbuf, o.nrbuf) == (128, 3, 2, 0), (layer[0], o.stages, o.ncbuf, o.nrbuf)
            else:
                assert (o.BN, o.stages, o.ncbuf, o.nrbuf) == (128, 2, 4, 1), (layer[0], o.stages, o.ncbuf, o.nrbuf)


def test_k_heavy_split_layers_trade_a_staging_pair_for_a_third_stage():
    by_name = {l[0]: l for l in R50_FPN_3D}
    for name in ('res3 3x3x3', 'res4 3x3x3', 'fpn post-hoc P2', 'rpn conv P2', 'keypoint head conv'):
        o = plan_x3(by_name[name])
        assert (o.stages, o.ncbuf) == (3, 2), (name, o.stages, o.ncbuf)
    o = plan_x3(by_name['res2 1x1 reduce'])                                      # K-light: both staging pairs stay
    assert o.ncbuf == 4 and o.stages >= 2


def test_plain_plans_keep_two_kblock_stages():
    o = plan(8, 3, 200, 336, 256, 256, (3, 3, 3), p=(1, 1, 1))
    assert o.ks == 2 and o.stage_bytes == 2 * (A_BOX + o.BN * 128)

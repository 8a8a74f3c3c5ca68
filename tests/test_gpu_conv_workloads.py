"""GPU: every conv plan of the 2-D R50-FPN step (`bench.py --config r50fpn2d`), the R18-3D tube step (`--config r18tube`)
and the forward of the keypoint R-CNN training step, at several tiles per CTA, against the fp64 tap-sum reference; and a
check over those steps and the R50-FPN-3D step (tests/step_launches.py records them) that every launch they make is one
of the value-tested plans, by the stricter key of test_conv_plan_workloads.plan_key_v2 (which tells strided and stacked
launches apart)."""
import pytest

from test_conv_plan import step_plan
from test_conv_plan_workloads import (CASES, STACKED_STRIDED, STACKED_STRIDED_REDUCED, TABLES, plan_key_v2, row_plan,
                                      table_keys)
from test_gpu_conv import _check_step_case, with_operands

pytestmark = pytest.mark.gpu


@with_operands('wl,layer,mode', CASES, ['%s-%s-%s' % (w, l[0], m) for w, l, m in CASES])
def test_workload_layer_over_three_waves_vs_fp64(wl, layer, mode, operands, record_property):
    """Every (row, mode) of the three tables at its reduced shape (test_conv_plan_workloads: the step's plan and tile,
    three or more tiles per CTA, a ragged last wave, the step's partial tiles and skipped padding taps) with the engine's
    storage and epilogue, against the fp64 tap-sum reference on the values the kernel reads.  Among them: the strided
    3x3x3 branch2a of the R18 body on odd maps, the res5 RoI convs on stacks of 6 images x 3 frames of 7 x 7 with a ragged
    last stack, and the 3-D keypoint head on stacks of 3 images x 3 frames with a ragged last stack.  Bounds as in
    test_gpu_conv.test_step_layer_over_three_waves_vs_fp64: bf16 outputs elementwise, the others _step_tol; integer
    operands bit for bit."""
    _check_step_case(layer, mode, row_plan(wl, layer, mode, reduced=True), TABLES[wl][1], '%s/%s/%s' % (wl, layer[0], mode),
                     record_property, operands)


@with_operands('mode', ('bf16', 'tf32', 'tf32x3', 'bf16x3'), ('bf16', 'tf32', 'tf32x3', 'bf16x3'))
def test_strided_conv_on_32_image_stacks_vs_fp64(mode, operands, record_property):
    """A strided 3x3 conv on 7 x 7 maps stacked 32 to an M tile (one output row of four columns each), 283 images: the
    strided activation box over stacked images, the live taps of each tile under stride, a last stack of 27 images."""
    o = step_plan(STACKED_STRIDED, mode, True, STACKED_STRIDED_REDUCED)
    assert (o.TB, o.TH, o.TW) == (32, 1, 4)
    _check_step_case(STACKED_STRIDED, mode, o, STACKED_STRIDED_REDUCED, 'stacked-strided/%s' % mode, record_property,
                     operands)


def test_workload_convs_are_all_in_the_tables(record_property):
    """One 800 x 1333 clip of each bench workload through DetectionEngine.detect in every mode (where the engine takes
    it), and one KeypointRcnnTrainer.step at the bench training config: every dt_conv3d launch (of the training step:
    every forward launch, outside TrainConv.backward) has the plan_key_v2 of a row of test_conv_plan.R50_FPN_3D or of a
    test_conv_plan_workloads table, each value-tested above or in test_gpu_conv.py; every conv1 launch runs a variant the
    conv1 tests of test_gpu_conv.py check."""
    import step_launches as sl
    table = {}
    for wl in ('r50fpn3d',) + tuple(TABLES):
        for k, rows in table_keys(wl).items():
            table.setdefault(k, []).extend(rows)
    conv1_tested = {('conv1', 0, 1, 0), ('conv1', 0, 0, 0), ('conv1', 1, 1, 0), ('conv1', 0, 0, 1), ('conv1_f32', 0)}
    calls = {'py': 0, 'c': 0}
    missing, seen = {}, set()
    for run in sl.ENGINE_RUNS + ('train',):
        rec = sl.record(run)
        tag = 'train_forward' if run == 'train' else '%s_%s' % run
        if not rec.taken:
            assert run[1] not in ('bf16', 'bf16x3'), run
            record_property('not_taken_' + tag, True)
            continue
        calls['py'] += rec.conv_py
        launched = []
        for name, a, in_backward in rec.calls:
            if name.startswith(('dt_conv3d', 'dt_conv1_7x7s2')):
                calls['c'] += 1
            if in_backward:
                continue
            if name == 'dt_conv3d':
                d, o = sl.conv_plan(a)
                key = plan_key_v2(d.dtype, d.x3, d.out_f32, d.res_mode, o, (d.kT, d.kH, d.kW), (d.sT, d.sH, d.sW))
                launched.append((key, (d.N, d.Ti, d.Hi, d.Wi, d.Cin, d.Cout)))
            elif name == 'dt_conv1_7x7s2':
                launched.append((('conv1', a[10], a[11], a[13]), None))
            elif name == 'dt_conv1_7x7s2_f32':
                launched.append((('conv1_f32', a[8]), None))
        assert len(launched) > (50 if run == 'train' or run[0] == 'r50fpn3d' else 20), (run, len(launched))
        record_property('launches_' + tag, len(launched))
        record_property('plan_keys_v2_' + tag, len({k for k, _ in launched}))
        for key, shape in launched:
            seen.add(key)
            if key not in table and key not in conv1_tested:
                missing.setdefault(key, (tag, shape))
    record_property('plan_keys_v2_seen', len(seen))
    assert calls['py'] == calls['c'], calls
    assert not missing, missing

"""CPU: every C-ABI entry point validates its arguments on the host BEFORE touching CUDA and reports through the
return code + dt_last_error() (the RuntimeError the python binding raises) — the CAFFE_ENFORCE behaviour the
reference's tests rely on (tests/test_zero_even_op.py:41-44).  Runs without a GPU."""
import ctypes as C

import pytest

from detectandtrack_b200 import _lib as L


def _bad_conv_desc():
    return L.ConvDesc(N=1, Ti=1, Hi=8, Wi=8, Cin=16, Cout=16, kT=1, kH=1, kW=1, sT=1, sH=1, sW=1, dtype=7)


def _cases():
    f3 = (C.c_float * 3)(0, 0, 0)
    f4 = (C.c_float * 4)(1, 1, 1, 1)
    one = (C.c_int * 1)(1)
    onef = (C.c_float * 1)(1.0)
    ptrs = (C.c_void_p * 1)(None)
    lv = (L.RpnLevel * 1)()
    tl = (L.RpnTargetLevel * 1)()
    return [
        ('dt_bbox_overlaps', (None, 4, 4, None, 4, 4, 99, None, 4, None), b'T=99'),
        ('dt_nms_batched', (None, 1, 9000, 5, 1, None, 0.5, 0, 0, 0, None, None, None, 0, None), b'exceeds'),
        ('dt_lsa_batched', (None, 1, 100000, 100000, None, None, 0, None, None, None), b'dt_lsa_batched'),
        ('dt_match_frames', (None, 2, 100000, 5, 1, None, None, 1.0, 0, None, None, None), b'dt_match_frames'),
        ('dt_assign_track_ids', (None, None, None, 0, -1, None, 0, 0, 0, None, None), b'dt_assign_track_ids'),
        ('dt_prune_detections', (None, -1, 1, 5, 1, 0, None, None, 0.5, 50.0, None, None, None, None), b'dt_prune_detections'),
        ('dt_conv3d', (None, None, None, None, None, None, None, None), b'null descriptor'),
        ('dt_conv3d', (C.byref(_bad_conv_desc()), None, None, None, None, None, None, None), b'dtype 7'),
        ('dt_conv_plan', (None, 1, None), b'null pointer'),
        ('dt_rpn_proposals_multi', (lv, 0, 1, 1, 3, 1, None, 1000, 0.0, 4.135, 0, 1, 0, None, 0, None), b'1..8 levels'),
        ('dt_collect_rpn', (None, None, None, 1, 0, 1000, 1, 1000, None, None, None, 1000, None), b'dt_collect_rpn'),
        ('dt_distribute_fpn', (None, 10, None, 2, 1, 1, 2, 5, 224.0, 4.0, None, None, None, None), b'dt_distribute_fpn'),
        ('dt_box_decode', (None, None, 1, 0, 1, None, 2, None, 8, 2, None, None, f4, 4.135, 0.05, None, None, None), b'dt_box_decode'),
        ('dt_limit_detections', (None, None, None, 1, 1, 10, 1, 100, None, None, 104, None), b'dt_limit_detections'),
        ('dt_prep_clip', (None, 1, 0, 10, f3, 1.0, 10, 10, 10, 10, 8, 0, 0, 0, 0, None, None), b'dt_prep_clip'),
        ('dt_conv1_7x7s2', (None, 1, 7, 8, 8, None, 64, None, None, 1, 0, 0, 0, 0, None, 64, None), b'dt_conv1_7x7s2'),
        ('dt_maxpool2d', (None, 1, 8, 8, 12, 12, 3, 2, 1, 0, 0, None, 12, None), b'multiples of 8'),
        ('dt_roi_align', (ptrs, one, one, onef, 0, 2, 256, 256, 0, None, 5, None, 10, 1, None, 7, 2, 0, 0, None, None), b'dt_roi_align'),
        ('dt_keypoint_decode', (None, 68, 99, 17, 1, None, 4, None, 10, 0, None, None, None), b'S=99'),
        ('dt_conv1_7x7s2_f32', (None, 1, 7, 8, 4, None, None, None, 0, None, None), b'dt_conv1_7x7s2_f32'),
        ('dt_spatial_mean', (None, 1, 7, 7, 10, 10, 1, 0, 0, None, 10, None), b'multiples of 4'),
        ('dt_time_mean', (None, 1, 3, 49, 10, 10, 1, 0, 0, None, 10, None), b'multiples of 4'),
        ('dt_fold_tube_heads', (None, 4, 10, 99, 2, None, None, None), b'dt_fold_tube_heads'),
        ('dt_memset', (None, 0, 16, None), b'dt_memset'),
        ('dt_pose_pck_cost', (None, 2, None, 2, 10, 17, 2, 1, 0.5, None, None), b'dt_pose_pck_cost'),
        ('dt_frame_costs', (None, 3, 1, None, 0, 0, 0, 0, 0.5, None, None, 2, 4, 1.0, 0.0, None, None), b'dt_frame_costs'),
        ('dt_pairs_to_f16', (None, 10, 12, None, None), b'C % 8'),
        ('dt_scale_rois', (None, 2, 10, 4, None, 1, 1.0, None, None), b'dt_scale_rois'),
        ('dt_wgrad_nhwc', (None, 64, None, 64, 1, 1, 8, 8, 8, 8, 64, 64, 1, 3, 3, 2, 2, None, None), b'only pointwise'),
        ('dt_wgrad_nhwc', (None, 64, None, 64, 1, 1, 4, 4, 8, 8, 64, 64, 1, 1, 1, 1, 1, None, None), b'does not match'),
        ('dt_wgrad_nhwc', (None, 64, None, 60, 1, 1, 8, 8, 8, 8, 64, 60, 1, 3, 3, 1, 1, None, None), b'dt_wgrad_nhwc'),
        ('dt_bwd_pointwise', (None, None, None, None, 10, 12, None, None), b'C % 8'),
        ('dt_bwd_pointwise2', (None, None, None, None, 10, 12, None, None, None, None), b'C % 8'),
        ('dt_upsample_add_bwd', (None, None, 1, 4, 4, 12, None, None), b'dt_upsample_add_bwd'),
        ('dt_scatter_stride2', (None, 1, 4, 4, 9, 8, 64, None, None), b'dt_scatter_stride2'),
        ('dt_sgd_update_multi', (None, None, 1, 1, 0.1, 0.9, 0.0, 1.0, None), b'null pointer'),
        ('dt_sgd_update_multi', (None, None, 0, 0, 0.1, 0.9, 0.0, 1.0, None), b'empty table'),
        ('dt_bias_grad', (None, 10, 12, 16, None, None), b'dt_bias_grad'),
        ('dt_rpn_loss_grad', (None, 8, None, None, None, None, 10, 3, 1.0, 1.0, 0.1, None, 16, None, None), b'dt_rpn_loss_grad'),
        ('dt_embed_frame', (None, 2, 3, 64, 5, None, None), b'dt_embed_frame'),
        ('dt_grad_join_f32', (None, None, 12, None, None), b'multiple of 8'),
        ('dt_roi_align_bwd', (None, ptrs, one, one, onef, 1, 2, 12, None, 5, None, 10, 1, None, 7, 2, None), b'multiple of 8'),
        ('dt_frcnn_loss_grad', (None, 8, None, None, None, None, 10, 2, None, 1.0, 1.0, None, 16, None, None, None), b'dt_frcnn_loss_grad'),
        ('dt_kps_loss_grad', (None, 72, 99, 17, 4, None, None, None, 1.0, None, 72, None, None), b'S=99'),
        ('dt_subpixel_grad_fix', (None, None, 17, 8, 60, None), b'ldc=60'),
        ('dt_jpeg_decode', (None, None, 2, 0, 10, None, None), b'dt_jpeg_decode'),
        ('dt_rpn_targets', (tl, 1, 3, 1, 1, None, None, None, 4096, None, 0.0, 0.7, 0.3, 256, 0.5, 3, None, 0, None), b'Gmax'),
        ('dt_sample_rois', (None, None, None, 1, 0, 2000, None, None, None, None, None, 8, 17, 1, None, 2, 512, 0.25, 0.5, 0.5, 0.0, f4, 56, 3,
                            None, None, None, None, None, None, None, None, None, None, 128, None, None), b'dt_sample_rois'),
    ]


@pytest.mark.parametrize('name,args,msg', _cases(), ids=['%s-%d' % (c[0], i) for i, c in enumerate(_cases())])
def test_entry_point_rejects_bad_arguments_without_a_gpu(name, args, msg):
    lib = L.lib()
    rc = getattr(lib, name)(*args)
    err = lib.dt_last_error()
    assert rc != 0, name
    assert msg in err, (name, err)
    with pytest.raises(RuntimeError, match=name):
        L.check(rc, name)


def test_every_compute_entry_point_has_an_error_case():
    covered = {c[0] for c in _cases()}
    host_only = {'dt_abi_version', 'dt_nms_workspace_bytes', 'dt_rpn_workspace_bytes', 'dt_rpn_targets_workspace_bytes'}
    assert set(L.SIGNATURES) - host_only <= covered, set(L.SIGNATURES) - host_only - covered


def test_lsa_batched_f64_argument_checks():
    """dt_lsa_batched_f64 (the fp64 solver of the pose-pck tracking cost) rejects bad shapes, algos and null pointers on
    the host; an empty batch is a no-op."""
    lib = L.lib()
    cases = [
        ((None, 1, 225, 225, None, None, 0, None, None, None), b'dmax=225'),
        ((None, 1, 0, 1, None, None, 0, None, None, None), b'dmax=0'),
        ((None, 1, 100, 99, None, None, 0, None, None, None), b'ldc=99'),
        ((None, -1, 8, 8, None, None, 0, None, None, None), b'batch=-1'),
        ((None, 1, 8, 8, None, None, 2, None, None, None), b'unknown algo 2'),
        ((None, 1, 8, 8, None, None, 0, None, None, None), b'null pointer'),
    ]
    for args, msg in cases:
        rc = lib.dt_lsa_batched_f64(*args)
        assert rc != 0, args
        assert msg in lib.dt_last_error(), (args, lib.dt_last_error())
    assert lib.dt_lsa_batched_f64(None, 0, 8, 8, None, None, 0, None, None, None) == 0
